"""Seeded scenes for the 3D-2D RANSAC tests (okb_ransac_3d2d_batch, tests/ransac_reference.py): a synthetic window at the
true poses and landmarks whose newest frame B holds, per camera, its observations as keypoints (at most 0.5 px off the
true projection) plus unrelated keypoints, and every kind of keypoint the adapter skips or keeps:
  wrong       a landmark slot other than the true one (an injected outlier)
  single      a landmark left with B's observation only (skipped: fewer than 2 observations)
  infinity    a landmark at infinity, hp[3] = 0 (skipped)
  dead        a slot whose landmark is not in the graph, or beyond the window's landmarks (skipped)
  bad_bp      (RADTAN8 only) a keypoint 5 focal lengths off the centre: undistort fails and the bearing is NaN"""
import numpy as np

from okvis_b200 import abi, synthetic

MIN_MARGIN = 1e-7
FEAT = 2            # frame B's feature slot
N_FEAT = 3


def make_scene(seed, distortion=abi.DIST_RADTAN, n_cams=2, wrong_fraction=0.1, n_landmarks=500, n_frames=5,
               specials=True, n_kp=400):
    gen = abi.DIST_NONE if distortion == abi.DIST_RADTAN8 else distortion
    cfg = synthetic.WindowConfig(n_frames=n_frames, n_cams=n_cams, n_landmarks=n_landmarks, distortion=gen,
                                 pixel_sigma=0.0, outlier_fraction=0.0, perturb=False)
    w = synthetic.make_window(cfg=cfg, seed=0x5AC0 + seed)
    if distortion == abi.DIST_RADTAN8:
        w.cameras["model"] = abi.DIST_RADTAN8
        w.cameras["dist"] = [1e-3, 0.0, 1e-5, -1e-5, 0.0, 1e-3, 0.0, 0.0]
    rng = np.random.default_rng(seed)
    K, L = len(w.poses), len(w.landmarks)
    B = K - 1
    obs = w.obs
    cnt = np.bincount(obs["lm_idx"].astype(np.int64), minlength=L)
    inB = obs["pose_idx"] == B
    lmB = np.unique(obs["lm_idx"][inB]).astype(np.int64)
    kinds = {}
    if specials:
        cand = rng.permutation(lmB)
        single, inf = cand[:3], cand[3:6]
        drop = np.isin(obs["lm_idx"], single)
        for l in single:
            drop[np.nonzero((obs["lm_idx"] == l) & inB)[0][0]] = False       # one observation left, in frame B
        w.obs = obs = np.ascontiguousarray(obs[~drop])
        w.landmarks[inf, 3] = 0.0
        dead = cand[6:9]
        w.landmarks[dead] = 0.0
        kinds.update(single=set(single.tolist()), infinity=set(inf.tolist()), dead=set(dead.tolist()))
    cnt = np.bincount(obs["lm_idx"].astype(np.int64), minlength=L)
    good_lm = np.nonzero((cnt >= 2) & np.any(w.landmarks != 0.0, 1) & (w.landmarks[:, 3] != 0.0))[0]
    store = {}
    injected = []
    for c in range(n_cams):
        o = obs[(obs["pose_idx"] == B) & (obs["cam_idx"] == c)]
        lm = o["lm_idx"].astype(np.int32)
        kp = o["z"] + rng.uniform(-0.25, 0.25, o["z"].shape)
        truth = lm.copy()
        wrong = (rng.random(len(lm)) < wrong_fraction) & np.isin(truth, good_lm)
        pose = w.poses[B]
        R_WS, r_WS = synthetic.R_from_quat(pose[3:]), pose[:3]
        R_SC, r_SC = synthetic.R_from_quat(w.extrinsics[c][3:]), w.extrinsics[c][:3]
        for i in np.nonzero(wrong)[0]:
            while True:             # a wrong landmark far (> 20 px at the focal length) from the keypoint's true ray
                l = int(rng.choice(good_lm[good_lm != truth[i]]))
                ray_t = R_SC.T @ (R_WS.T @ (w.landmarks[truth[i], :3] / w.landmarks[truth[i], 3] - r_WS) - r_SC)
                ray_w = R_SC.T @ (R_WS.T @ (w.landmarks[l, :3] / w.landmarks[l, 3] - r_WS) - r_SC)
                if np.linalg.norm(ray_t / np.linalg.norm(ray_t) - ray_w / np.linalg.norm(ray_w)) * float(w.cameras[c]["fu"]) > 20:
                    break
            lm[i] = l
        n_extra = max(0, n_kp - len(lm) - 4)
        W_, H_ = int(w.cameras[c]["width"]), int(w.cameras[c]["height"])
        kp = np.concatenate([kp, rng.uniform([0, 0], [W_, H_], (n_extra, 2))])
        lm = np.concatenate([lm, -np.ones(n_extra, np.int32)])
        truth = np.concatenate([truth, -np.ones(n_extra, np.int32)])
        if specials:
            # slots not in the graph: beyond the window's landmarks; and a bad backProject where the model can fail
            kp = np.concatenate([kp, rng.uniform([0, 0], [W_, H_], (1, 2))])
            lm = np.concatenate([lm, [L + 5]]).astype(np.int32)
            truth = np.concatenate([truth, [-1]])
            if distortion == abi.DIST_RADTAN8:
                cm = w.cameras[c]
                kp = np.concatenate([kp, [[float(cm["cu"]) + 5.0 * float(cm["fu"]), float(cm["cv"])]]])
                lm = np.concatenate([lm, [int(good_lm[0])]]).astype(np.int32)
                truth = np.concatenate([truth, [-2]])
        order = rng.permutation(len(lm))
        kp, lm, truth = kp[order], lm[order], truth[order]
        size = rng.uniform(6.0, 14.0, len(lm))
        store[(FEAT, c)] = dict(kp=kp.astype(np.float32).astype(np.float64), size=size.astype(np.float32).astype(np.float64),
                                lm=lm.astype(np.int32), truth=truth.astype(np.int32))
        injected += [(c, int(k)) for k in np.nonzero((lm != truth) & (truth >= 0))[0]]
    return dict(window=w, store=store, n_cams=n_cams, feat=FEAT, injected=set(injected), kinds=kinds, distortion=distortion)


def restrict(sc, max_assoc=None, empty_cam=None):
    """Variants: only the first `max_assoc` associated keypoints of each camera keep their slot; camera `empty_cam`
    has no keypoints."""
    store = {}
    for (f, c), e in sc["store"].items():
        e = {k: v.copy() for k, v in e.items()}
        if max_assoc is not None:
            idx = np.nonzero(e["lm"] >= 0)[0]
            e["lm"][idx[max_assoc:]] = -1
        if empty_cam is not None and c == empty_cam:
            e = {k: v[:0] for k, v in e.items()}
        store[(f, c)] = e
    return dict(sc, store=store)


def load(ctx, win, sc, n_kp=None):
    """Uploads the scene's window into slot `win` and fills frame B's feature slot."""
    w = sc["window"]
    n_kp = n_kp or max(len(e["lm"]) for e in sc["store"].values())
    ctx.reserve(win, len(w.poses), len(w.landmarks), len(w.obs), len(w.imu_samples))
    ctx.reserve_features(win, N_FEAT, sc["n_cams"], max(n_kp, 1), 48)
    ctx.upload(win, w)
    for (f, c), e in sorted(sc["store"].items()):
        n = len(e["lm"])
        ctx.set_features(win, f, c, np.stack([e["kp"][:, 0], e["kp"][:, 1], e["size"]], 1).reshape(n, 3),
                         np.zeros((n, 48), np.uint8), e["lm"], (e["lm"] >= 0).astype(np.uint8))
    ctx.commit(win, 1)


def state(sc):
    return dict(window=sc["window"], store=sc["store"])
