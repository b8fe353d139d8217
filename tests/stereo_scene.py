"""Seeded stereo scenes for the stereo initialisation tests: a synthetic window (okvis_b200.synthetic, EuRoC-like stereo
rig with a 0.11 m baseline) whose newest frame holds, per camera, the keypoints of points at 1-60 m seen by both cameras
(descriptors with a few bits flipped between the cameras), 40 distractors (look-alike descriptors elsewhere in the image,
and random ones), and special pairs:
  - keypoints pre-named to landmarks of the graph: A initialised (skipped), A uninitialised, B uninitialised, both;
  - a border keypoint whose partner is off by a few sigma, so that the reprojection check fails;
  - a pair at 2 km, where triangulateFast finds the rays parallel (determinant below 1e-6);
  - a close pair whose A keypoint is so large that A's term in getUncertainty's H falls below Eigen's rank threshold
    while |r_B|^2 >= 4: the QR decides (the size is found by bisection on the reference's rank, then multiplied by 4).
No decision may lie within 1e-9 relative of its threshold: a scene that has one is re-drawn with the next sub-seed."""
import numpy as np

from okvis_b200 import abi, synthetic
import stereo_init_reference as ref
from track_reference import T_CW, project_homogeneous

MIN_MARGIN = 1e-9


def _flip(rng, d, n_bits):
    d = d.copy()
    for i in rng.integers(0, d.size * 8, n_bits):
        d[i // 8] ^= np.uint8(1 << (i % 8))
    return d


def _window(seed, distortion):
    gen = abi.DIST_NONE if distortion == abi.DIST_RADTAN8 else distortion
    w = synthetic.make_window(cfg=synthetic.WindowConfig(n_frames=6, n_cams=2, n_landmarks=300, distortion=gen), seed=0x57E0 + seed)
    if distortion == abi.DIST_RADTAN8:
        w.cameras["model"] = abi.DIST_RADTAN8
        w.cameras["dist"] = [1e-3, 0.0, 1e-5, -1e-5, 0.0, 1e-3, 0.0, 0.0]
    return w


def _project(w, pose, cam, X):
    R, t = T_CW(w.poses[pose], w.extrinsics[cam])
    ip, _, ok = project_homogeneous(w.cameras[cam], np.concatenate([R @ X + t, [1.0]]))
    return ip, ok


def _draw(seed, sub, distortion, n_kp, desc_bytes):
    rng = np.random.default_rng([seed, sub])
    w = _window(seed, distortion)
    K, L = len(w.poses), len(w.landmarks)
    pose = K - 1
    Wd, Hd = int(w.cameras[0]["width"]), int(w.cameras[0]["height"])
    Rc0, tc0 = T_CW(w.poses[pose], w.extrinsics[0])

    def world(p_c0):
        return Rc0.T @ (p_c0 - tc0)

    pts, kpa, kpb, tags = [], [], [], []

    def add(X, tag, off_b=(0.0, 0.0), noise=0.25):
        pa, oka = _project(w, pose, 0, X)
        pb, okb = _project(w, pose, 1, X)
        if not (oka and okb) or min(pa[0], pa[1], pb[0], pb[1]) < 0.5 or pa[0] > Wd - 1 or pb[0] > Wd - 1 or pa[1] > Hd - 1 or pb[1] > Hd - 1:
            return False
        pts.append(X); kpa.append(pa + rng.normal(0, noise, 2)); kpb.append(pb + rng.normal(0, noise, 2) + off_b); tags.append(tag)
        return True

    n_true = n_kp - 40 - 8
    while len(pts) < n_true:
        z = float(np.exp(rng.uniform(np.log(1.0), np.log(60.0))))
        add(world(np.array([rng.uniform(-0.8, 0.8) * z, rng.uniform(-0.5, 0.5) * z, z])), "plain")
    while not add(world(np.array([rng.uniform(-0.3, 0.3) * 2000.0, rng.uniform(-0.2, 0.2) * 2000.0, 2000.0])), "parallel", noise=0.0):
        pass
    # border keypoint: A at the left edge, B off by ~6 sigma in y
    while True:
        z = rng.uniform(3.0, 8.0)
        ip = np.array([rng.uniform(1.0, 3.0), rng.uniform(100, 380)])
        d = ref.back_project(w.cameras[0], ip[None])[0]
        if add(world(d * z), "border", off_b=(0.0, 6 * 0.8 * 10.0 / 12.0), noise=0.0):
            break
    while not add(world(np.array([rng.uniform(-0.3, 0.3) * 2.0, rng.uniform(-0.2, 0.2) * 2.0, 2.0])), "rank"):
        pass
    n = len(pts)
    base = rng.integers(0, 256, (n, desc_bytes), dtype=np.uint8)
    da = np.stack([_flip(rng, base[i], int(rng.integers(0, 6))) for i in range(n)])
    db = np.stack([_flip(rng, base[i], int(rng.integers(0, 6))) for i in range(n)])
    kpa, kpb = np.array(kpa), np.array(kpb)
    size_a, size_b = rng.uniform(6.0, 14.0, n), rng.uniform(6.0, 14.0, n)
    size_a[[i for i, t in enumerate(tags) if t == "border"]] = 10.0
    size_b[[i for i, t in enumerate(tags) if t == "border"]] = 10.0
    # 40 distractors per image: 20 look-alikes of true points placed elsewhere, 20 random
    def distract(kp, desc):
        src = rng.integers(0, n_true, 20)
        kd = np.stack([rng.uniform(20, Wd - 20, 40), rng.uniform(20, Hd - 20, 40)], 1)
        dd = np.concatenate([np.stack([_flip(rng, base[i], 8) for i in src]), rng.integers(0, 256, (20, desc_bytes), dtype=np.uint8)])
        return np.concatenate([kp, kd]), np.concatenate([desc, dd])
    kpa, da = distract(kpa, da)
    kpb, db = distract(kpb, db)
    size_a = np.concatenate([size_a, rng.uniform(6.0, 14.0, 40)])
    size_b = np.concatenate([size_b, rng.uniform(6.0, 14.0, 40)])
    truth_a = np.concatenate([np.arange(n), -np.ones(40, int)])
    truth_b = np.concatenate([np.arange(n), -np.ones(40, int)])
    # pre-named keypoints: landmarks of the graph (slots 0..L-1 of the synthetic window are live)
    lm_a, lm_b = -np.ones(len(kpa), np.int32), -np.ones(len(kpb), np.int32)
    lm_init = (rng.random(L) < 0.5).astype(np.uint8)
    plain = [i for i, t in enumerate(tags) if t == "plain" and np.linalg.norm(pts[i] - world(np.zeros(3))) < 20.0]
    pick = rng.choice(plain, 32, replace=False)
    slots = rng.choice(L, 40, replace=False)
    lm_init[slots[:8]] = 1                       # A named, initialised: skipped by doSetup
    lm_init[slots[8:40]] = 0
    for k, i in enumerate(pick[:8]):
        lm_a[i] = slots[k]
    for k, i in enumerate(pick[8:16]):           # A named, uninitialised
        lm_a[i] = slots[8 + k]
    for k, i in enumerate(pick[16:24]):          # B named, uninitialised
        lm_b[i] = slots[16 + k]
    for k, i in enumerate(pick[24:32]):          # both named
        lm_a[i] = slots[24 + k]; lm_b[i] = slots[32 + k]
    pa_, pb_ = rng.permutation(len(kpa)), rng.permutation(len(kpb))
    f32 = lambda x: np.asarray(x, np.float32).astype(np.float64)
    feat = 2
    rank_i = tags.index("rank")
    store = {(feat, 0): dict(kp=f32(kpa[pa_]), size=f32(size_a[pa_]), desc=np.ascontiguousarray(da[pa_]), lm=lm_a[pa_], observed=(lm_a[pa_] >= 0).astype(np.uint8)),
             (feat, 1): dict(kp=f32(kpb[pb_]), size=f32(size_b[pb_]), desc=np.ascontiguousarray(db[pb_]), lm=lm_b[pb_], observed=(lm_b[pb_] >= 0).astype(np.uint8))}
    inv_a, inv_b = np.argsort(pa_), np.argsort(pb_)
    state = dict(poses=w.poses, extrinsics=w.extrinsics, cameras=w.cameras, landmarks=np.array(w.landmarks), lm_init=lm_init, store=store)
    sc = dict(window=w, state=state, F=4, n_kp=len(kpa), desc_bytes=desc_bytes, job=dict(pose=pose, feat_slot=feat, cam_a=0, cam_b=1),
              truth_a=truth_a[pa_], truth_b=truth_b[pb_], points=np.array(pts), tags=tags,
              idx_a=inv_a, idx_b=inv_b, rank_pair=(int(inv_a[rank_i]), int(inv_b[rank_i])))
    return sc


def _rank_size(sc):
    """The A keypoint size of the rank pair: 4x the size at which the reference's rank of H drops below 9."""
    a, b = sc["rank_pair"]
    g = ref.setup(sc["state"], sc["job"])

    def full_rank(size):
        g2 = dict(g, size_a=g["size_a"].copy(), rs_a=g["rs_a"].copy())
        g2["size_a"][a] = size
        g2["rs_a"][a] = ref.ray_sigmas(size, float(g["cam_a"]["fu"]))
        ok, hp, par = ref.stereo_triangulate(g2, a, b, [])
        assert ok and not par
        r2, H, *_ = ref.uncertainty_H(g2, a, b, hp)
        assert r2 >= 4.0
        return ref.qr_rank(H) == 9

    lo, hi = 10.0, 1e12
    assert full_rank(lo) and not full_rank(hi)
    for _ in range(80):
        mid = np.sqrt(lo * hi)
        lo, hi = (mid, hi) if full_rank(mid) else (lo, mid)
    return float(np.float32(4.0 * hi))


def make_stereo_scene(seed, distortion=abi.DIST_RADTAN, n_kp=400, desc_bytes=48, oracle=None):
    """The scene and the reference's records; re-drawn until no decision lies within MIN_MARGIN of its threshold."""
    for sub in range(20):
        sc = _draw(seed, sub, distortion, n_kp, desc_bytes)
        a, _ = sc["rank_pair"]
        sc["state"]["store"][(sc["job"]["feat_slot"], 0)]["size"][a] = _rank_size(sc)
        margins, cases, dets = [], [], []
        recs, g = ref.stereo_init(oracle, sc["state"], sc["job"], margins=margins, cases=cases, dets=dets)
        # every gate decision the matcher takes: pairs below the Hamming threshold that neither side skips
        A, B = sc["state"]["store"][(sc["job"]["feat_slot"], 0)], sc["state"]["store"][(sc["job"]["feat_slot"], 1)]
        dist = np.unpackbits(A["desc"][:, None, :] ^ B["desc"][None, :, :], axis=2).sum(2)
        for a, b in zip(*np.nonzero(dist < 60)):
            if not (g["skipA"][a] or g["skipB"][b]):
                ref.stereo_triangulate(g, int(a), int(b), margins)
        if min(m for _, m in margins) > MIN_MARGIN:
            sc.update(records=recs, margins=margins, cases=cases, dets=dets, sub=sub)
            return sc
    raise RuntimeError("no scene without near-threshold decisions")


def load(ctx, win, sc):
    """Uploads the scene's window into slot `win` and fills its feature store and initialised flags."""
    w = sc["window"]
    ctx.reserve(win, len(w.poses), len(w.landmarks), len(w.obs), len(w.imu_samples))
    ctx.reserve_features(win, sc["F"], 2, sc["n_kp"], sc["desc_bytes"])
    ctx.upload(win, w)
    for (f, c), e in sorted(sc["state"]["store"].items()):
        ctx.set_features(win, f, c, np.stack([e["kp"][:, 0], e["kp"][:, 1], e["size"]], 1), e["desc"], e["lm"], e["observed"])
    L = len(w.landmarks)
    ctx.set_landmark_initialized(win, np.arange(L), sc["state"]["lm_init"])
    ctx.commit(win, 1)
