"""Seeded scenes for the 2D-2D RANSAC tests (okb_ransac_2d2d_batch, tests/ransac2d2d_reference.py): a synthetic window
whose older frame A and current frame B hold, per camera, the projections of the window's landmarks visible in both (at
most 0.25 px off) as keypoints naming their landmark slots, plus unrelated keypoints.  Frame B's pose is set from A's:
  motion      "rotation" (same position, rotated), "small" (2 cm baseline) or "large" (30 cm baseline)
  wrong       a fraction of B's keypoints naming another landmark of A (an injected wrong association when it is B's
              first keypoint naming that landmark)
and every kind of keypoint the adapter skips or keeps: a second B keypoint naming a landmark (the first wins), slots of
landmarks not in the graph, and (RADTAN8) a B keypoint 5 focal lengths off the centre, whose bearing is NaN."""
import numpy as np

from okvis_b200 import abi, synthetic

FEAT_A, FEAT_B = 0, 1
N_FEAT = 2
MIN_MARGIN = 1e-7


def _rot(rng, deg):
    v = rng.normal(size=3)
    v /= np.linalg.norm(v)
    a = np.deg2rad(deg)
    K = np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])
    return np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K


def _project(w, pose, c, X):
    R_WS, r_WS = synthetic.R_from_quat(pose[3:]), pose[:3]
    R_SC, r_SC = synthetic.R_from_quat(w.extrinsics[c][3:]), w.extrinsics[c][:3]
    p_C = (R_SC.T @ (R_WS.T @ (X - r_WS).T - r_SC[:, None])).T
    cam = w.cameras[c].copy()
    if cam["model"] == abi.DIST_RADTAN8:         # the keypoints are generated without distortion
        cam["model"] = abi.DIST_NONE
    return synthetic.project_points(cam, p_C)


def make_scene(seed, distortion=abi.DIST_RADTAN, n_cams=1, motion="large", wrong_fraction=0.1, n_landmarks=400, n_kp=300):
    gen = abi.DIST_NONE if distortion == abi.DIST_RADTAN8 else distortion
    cfg = synthetic.WindowConfig(n_frames=3, n_cams=n_cams, n_landmarks=n_landmarks, distortion=gen, pixel_sigma=0.0,
                                 outlier_fraction=0.0, perturb=False)
    w = synthetic.make_window(cfg=cfg, seed=0x2D2D + seed)
    if distortion == abi.DIST_RADTAN8:
        w.cameras["model"] = abi.DIST_RADTAN8
        w.cameras["dist"] = [1e-3, 0.0, 1e-5, -1e-5, 0.0, 1e-3, 0.0, 0.0]
    rng = np.random.default_rng(seed)
    K, L = len(w.poses), len(w.landmarks)
    A, B = K - 2, K - 1
    R_WA = synthetic.R_from_quat(w.poses[A][3:])
    R_WB = R_WA @ _rot(rng, 3.0)
    base = {"rotation": 0.0, "small": 0.02, "large": 0.3}[motion]
    d = rng.normal(size=3)
    w.poses[B] = np.concatenate([w.poses[A][:3] + base * d / np.linalg.norm(d), synthetic.quat_from_R(R_WB)])
    dead = rng.choice(L, 5, replace=False)
    w.landmarks[dead] = 0.0
    X = w.landmarks[:, :3] / np.where(w.landmarks[:, 3:] != 0.0, w.landmarks[:, 3:], 1.0)
    store, injected = {}, []
    for c in range(n_cams):
        W_, H_ = int(w.cameras[c]["width"]), int(w.cameras[c]["height"])
        pa, oka = _project(w, w.poses[A], c, X)
        pb, okb = _project(w, w.poses[B], c, X)
        vis = np.nonzero(oka & okb)[0]
        vis = vis[rng.permutation(len(vis))][:min(len(vis), n_kp - 20)]
        lmA, lmB = vis.astype(np.int32).copy(), vis.astype(np.int32).copy()
        kpA = pa[vis] + rng.uniform(-0.25, 0.25, (len(vis), 2))
        kpB = pb[vis] + rng.uniform(-0.25, 0.25, (len(vis), 2))
        truthB = lmB.copy()
        alive = ~np.isin(vis, dead)
        wrong = np.nonzero((rng.random(len(vis)) < wrong_fraction) & alive)[0]
        for i in wrong:             # another landmark of A, far (> 20 px) from the keypoint's own
            while True:
                j = int(rng.integers(len(vis)))
                if j != i and alive[j] and np.linalg.norm(pb[vis[j]] - pb[vis[i]]) > 20:
                    break
            lmB[i] = vis[j]
        extra = 10
        kpA = np.concatenate([kpA, rng.uniform([0, 0], [W_, H_], (extra, 2))])
        lmA = np.concatenate([lmA, -np.ones(extra, np.int32)])
        kpB = np.concatenate([kpB, rng.uniform([0, 0], [W_, H_], (extra, 2))])
        lmB = np.concatenate([lmB, -np.ones(extra, np.int32)])
        truthB = np.concatenate([truthB, -np.ones(extra, np.int32)])
        # a second B keypoint naming a landmark (std::map::insert keeps the first), a slot beyond the landmarks
        kpB = np.concatenate([kpB, rng.uniform([0, 0], [W_, H_], (2, 2))])
        lmB = np.concatenate([lmB, [int(vis[0]), L + 3]]).astype(np.int32)
        truthB = np.concatenate([truthB, [-1, -1]])
        if distortion == abi.DIST_RADTAN8:
            cm = w.cameras[c]
            lmB[lmB == int(vis[1])] = -1                # the NaN keypoint is B's only one naming its landmark
            kpB = np.concatenate([kpB, [[float(cm["cu"]) + 5.0 * float(cm["fu"]), float(cm["cv"])]]])
            lmB = np.concatenate([lmB, [int(vis[1])]]).astype(np.int32)
            truthB = np.concatenate([truthB, [-2]])
        oa, ob = rng.permutation(len(lmA)), rng.permutation(len(lmB))
        kpA, lmA = kpA[oa], lmA[oa]
        kpB, lmB, truthB = kpB[ob], lmB[ob], truthB[ob]
        for f, kp, lm, tr in ((FEAT_A, kpA, lmA, lmA), (FEAT_B, kpB, lmB, truthB)):
            size = rng.uniform(6.0, 14.0, len(lm))
            store[(f, c)] = dict(kp=kp.astype(np.float32).astype(np.float64), size=size.astype(np.float32).astype(np.float64),
                                 lm=lm.astype(np.int32), truth=tr.astype(np.int32))
        # a wrong association reaches the adapter when it is B's first keypoint naming that landmark
        e = store[(FEAT_B, c)]
        first = {}
        for k, l in enumerate(e["lm"]):
            first.setdefault(int(l), k)
        injected += [(c, int(k)) for k in np.nonzero((e["lm"] != e["truth"]) & (e["truth"] >= 0) & (e["lm"] >= 0))[0] if first[int(e["lm"][k])] == k]
    return dict(window=w, store=store, n_cams=n_cams, pose_a=A, pose_b=B, injected=set(injected), motion=motion,
                distortion=distortion)


def restrict(sc, cam, max_assoc):
    """Only the first `max_assoc` associated keypoints of frame A in camera `cam` keep their slot."""
    store = {k: {kk: v.copy() for kk, v in e.items()} for k, e in sc["store"].items()}
    e = store[(FEAT_A, cam)]
    e["lm"][np.nonzero(e["lm"] >= 0)[0][max_assoc:]] = -1
    return dict(sc, store=store)


def job(sc, seed, **kw):
    return dict(dict(pose_b=sc["pose_b"], feat_slot_b=FEAT_B, pose_a=sc["pose_a"], feat_slot_a=FEAT_A, n_cams=sc["n_cams"],
                     seed=seed), **kw)


def load(ctx, win, sc):
    """Uploads the scene's window into slot `win` and fills both feature slots."""
    w = sc["window"]
    n_kp = max(len(e["lm"]) for e in sc["store"].values())
    ctx.reserve(win, len(w.poses), len(w.landmarks), len(w.obs), len(w.imu_samples))
    ctx.reserve_features(win, N_FEAT, sc["n_cams"], n_kp, 48)
    ctx.upload(win, w)
    for (f, c), e in sorted(sc["store"].items()):
        n = len(e["lm"])
        ctx.set_features(win, f, c, np.stack([e["kp"][:, 0], e["kp"][:, 1], e["size"]], 1).reshape(n, 3),
                         np.zeros((n, 48), np.uint8), e["lm"], (e["lm"] >= 0).astype(np.uint8))
    ctx.commit(win, 1)


def state(sc):
    return dict(window=sc["window"], store=sc["store"])
