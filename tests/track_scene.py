"""Seeded scenes for the 3D-2D tracking tests: a synthetic window (okvis_b200.synthetic) whose newest frame B is being
tracked, and a feature store that holds, per frame and camera, the keypoints of the window's observations with
per-landmark descriptors (a few bits flipped per observation) plus unrelated keypoints.  Frame B's observations are
taken out of the window; its keypoints carry no landmarks yet and include look-alike distractors: the descriptor of a
landmark B sees, placed far from where that landmark projects."""
import numpy as np

from okvis_b200 import abi, synthetic


def _flip(rng, d, n_bits):
    d = d.copy()
    for _ in range(n_bits):
        i = rng.integers(0, d.size * 8)
        d[i // 8] ^= np.uint8(1 << (i % 8))
    return d


def make_track_scene(seed, n_kp=400, desc_bytes=48, distortion=abi.DIST_RADTAN, n_frames=8, n_landmarks=1200,
                     uninit_fraction=0.1, dead_fraction=0.02):
    gen = abi.DIST_NONE if distortion == abi.DIST_RADTAN8 else distortion       # the generator projects the other three
    cfg = synthetic.WindowConfig(n_frames=n_frames, n_cams=2, n_landmarks=n_landmarks, distortion=gen)
    w = synthetic.make_window(cfg=cfg, seed=0x7AC0 + seed)
    if distortion == abi.DIST_RADTAN8:
        w.cameras["model"] = abi.DIST_RADTAN8
        w.cameras["dist"] = [1e-3, 0.0, 1e-5, -1e-5, 0.0, 1e-3, 0.0, 0.0]
    rng = np.random.default_rng(seed)
    K, L, Cn = len(w.poses), len(w.landmarks), len(w.cameras)
    B = K - 1
    all_obs = w.obs
    keep = all_obs["pose_idx"] != B
    # some landmarks keep a single observation in the window: doSetup marks them uninitialised (step 4)
    single = np.nonzero(rng.random(L) < 0.05)[0]
    for l in single:
        idx = np.nonzero(keep & (all_obs["lm_idx"] == l))[0]
        keep[idx[:-1]] = False
    w.obs = np.ascontiguousarray(all_obs[keep])
    # a few landmark slots are not in the graph (all-zero estimate) while keypoints still name them
    dead = rng.random(L) < dead_fraction
    w.landmarks[dead] = 0.0
    base = rng.integers(0, 256, (L, desc_bytes), dtype=np.uint8)
    F = K + 3
    feat_of_frame = rng.permutation(F)[:K]          # feature slots are the caller's choice, unrelated to positions
    W, H = int(w.cameras[0]["width"]), int(w.cameras[0]["height"])
    store = {}
    for f in range(K):
        for c in range(Cn):
            o = all_obs[(all_obs["pose_idx"] == f) & (all_obs["cam_idx"] == c)]
            lm = o["lm_idx"].astype(np.int32)
            kp = o["z"].copy()
            desc = np.stack([_flip(rng, base[l], int(rng.integers(0, 6))) for l in lm]) if len(lm) else np.zeros((0, desc_bytes), np.uint8)
            if f == B:
                # look-alikes: a landmark's descriptor 40-80 px away from its observation
                pick = rng.choice(len(lm), size=len(lm) // 10, replace=False) if len(lm) else np.zeros(0, int)
                off = rng.uniform(40, 80, (len(pick), 2)) * rng.choice([-1, 1], (len(pick), 2))
                kp_d = np.clip(kp[pick] + off, 1, [W - 2, H - 2])
                kp = np.concatenate([kp, kp_d])
                desc = np.concatenate([desc, base[lm[pick]]])
                lm = np.concatenate([lm, lm[pick]])
            n_extra = max(0, min(n_kp - len(lm), 60))
            kp = np.concatenate([kp, rng.uniform([0, 0], [W, H], (n_extra, 2))])
            desc = np.concatenate([desc, rng.integers(0, 256, (n_extra, desc_bytes), dtype=np.uint8)])
            lm = np.concatenate([lm, -np.ones(n_extra, np.int32)])
            order = rng.permutation(len(lm))[:n_kp]
            kp, desc, lm = kp[order], desc[order], lm[order]
            n = len(lm)
            size = rng.uniform(6.0, 14.0, n)
            if f == B:
                truth = lm.copy()
                lm = -np.ones(n, np.int32)
                observed = np.zeros(n, np.uint8)
            else:
                observed = (lm >= 0).astype(np.uint8)
            entry = dict(kp=kp.astype(np.float32).astype(np.float64), size=size.astype(np.float32).astype(np.float64),
                         desc=np.ascontiguousarray(desc, np.uint8), lm=lm.astype(np.int32), observed=observed)
            if f == B:
                entry["truth"] = truth
            store[(int(feat_of_frame[f]), c)] = entry
    lm_init = (rng.random(L) >= uninit_fraction).astype(np.uint8)
    kf = [int(feat_of_frame[f]) for f in (B - 1, B - 2, B - 3)]       # keyframes by age 1, 2, 3
    fb = int(feat_of_frame[B])
    rounds = dict(
        keyframes=[(f, im, im) for f in kf for im in range(Cn)],          # matchToKeyframes: 3 keyframes x cameras
        last_frame=[(kf[0], im, im) for im in range(Cn)],                 # matchToLastFrame
        stereo=[(fb, 0, 1), (fb, 1, 0)])                                  # matchStereo's 3D-2D / 2D-3D passes
    return dict(window=w, store=store, lm_init=lm_init, F=F, n_kp=n_kp, desc_bytes=desc_bytes, pose_b=B, sb_b=B, feat_b=fb,
                rounds=rounds, n_cams=Cn)


def load(ctx, win, sc):
    """Uploads the scene's window into slot `win` and fills its feature store."""
    w = sc["window"]
    ctx.reserve(win, len(w.poses), len(w.landmarks), len(w.obs), len(w.imu_samples))
    ctx.reserve_features(win, sc["F"], sc["n_cams"], sc["n_kp"], sc["desc_bytes"])
    ctx.upload(win, w)
    for (f, c), e in sorted(sc["store"].items()):
        ctx.set_features(win, f, c, np.stack([e["kp"][:, 0], e["kp"][:, 1], e["size"]], 1), e["desc"], e["lm"], e["observed"])
        ctx.commit(win, 1)          # one frame's worth per commit, as a tracking host sends them
    L = len(w.landmarks)
    ctx.set_landmark_initialized(win, np.arange(L), sc["lm_init"])
