"""Seeded two-frame scenes for the 2D-2D tests against an earlier frame: a synthetic window (okvis_b200.synthetic,
EuRoC-like stereo rig) whose newest frame B and an older frame A are set about one stereo baseline apart (0.12 m, with a
small rotation), and, per camera of both frames, the keypoints of points at 1-60 m seen in all four images (descriptors
with a few bits flipped per image), 40 distractors per image (look-alikes of true points elsewhere, and random ones),
and special pairs:
  - A keypoints of all four kinds: no id, an id on the host only (store -1), an uninitialised landmark of the graph, an
    initialised one (skipped); B keypoints with no id, an uninitialised landmark or an initialised one (skipped), and
    pairs where both name a landmark;
  - a border pair whose B keypoint is off by a few sigma, so that the reprojection check fails;
  - a pair at 2 km, where triangulateFast finds the rays parallel;
  - a close pair whose A keypoint is so large that A's term in H falls below Eigen's rank threshold while |r_B|^2 >= 4:
    the QR decides (4x the larger of the sizes at which the reference's rank drops under the two priors).
The prior moves that size by about 1e-5 relative only (its translation block is far above the rank threshold under
either prior), while R_ii at the threshold carries rounding of order eps |max pivot|, a sizeable fraction of the
threshold itself: no rank decision can sit between the two priors and still be reproducible, so none is planted.
The current frame's speed is 0.4 m/s (the velocity clamp: u = 1e-2) or 3 m/s (u = 9e-2), by seed.  No decision of any
job variant (both cameras, sb_current = -1 and the current frame's block) lies within 1e-9 relative of its threshold."""
import numpy as np

from okvis_b200 import abi
import stereo_init_reference as sref
import stereo_scene
import temporal_init_reference as ref
from track_reference import T_CW, project_homogeneous

MIN_MARGIN = 1e-9
BASELINE = 0.12


def _flip(rng, d, n_bits):
    return stereo_scene._flip(rng, d, n_bits)


def _small_q(rng, angle):
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    return np.concatenate([np.sin(angle / 2) * ax, [np.cos(angle / 2)]])


def jobs(sc, sb=True):
    """The scene's two temporal jobs (camera 0 -> 0 and 1 -> 1), with the current frame's speed/bias block or -1."""
    b = sc["frames"]
    return [dict(b, cam_a=c, cam_b=c, sb_current=sc["sb_b"] if sb else -1) for c in (0, 1)]


def stereo_jobs(sc):
    """The stereo jobs of frame B (A = B, cameras 0 -> 1), as okb_stereo_init_batch and okb_match2d2d_batch take them."""
    f = sc["frames"]
    return (dict(pose=f["pose_b"], feat_slot=f["feat_slot_b"], cam_a=0, cam_b=1),
            dict(pose_a=f["pose_b"], feat_slot_a=f["feat_slot_b"], cam_a=0, pose_b=f["pose_b"], feat_slot_b=f["feat_slot_b"],
                 cam_b=1, sb_current=sc["sb_b"]))


def _draw(seed, sub, distortion, n_kp, desc_bytes):
    rng = np.random.default_rng([seed, sub, 0x2D2D])
    w = stereo_scene._window(seed, distortion)
    K, L = len(w.poses), len(w.landmarks)
    assert len(w.speed_bias) == K
    pb, pa = K - 1, K - 3
    qb = w.poses[pb][3:]
    C_WS = sref.q2R(qb)
    w.poses[pa][:3] = w.poses[pb][:3] + C_WS @ np.array([rng.uniform(-0.03, 0.03), BASELINE, rng.uniform(-0.03, 0.03)])
    w.poses[pa][3:] = sref.qmul(qb, _small_q(rng, 0.02))
    speed = 0.4 if seed % 2 == 0 else 3.0
    v = rng.normal(size=3)
    w.speed_bias[pb][:3] = speed * v / np.linalg.norm(v)
    Wd, Hd = int(w.cameras[0]["width"]), int(w.cameras[0]["height"])
    Rc0, tc0 = T_CW(w.poses[pb], w.extrinsics[0])

    def world(p_c0):
        return Rc0.T @ (p_c0 - tc0)

    def proj(pose, cam, X):
        R, t = T_CW(w.poses[pose], w.extrinsics[cam])
        ip, _, ok = project_homogeneous(w.cameras[cam], np.concatenate([R @ X + t, [1.0]]))
        return ip, ok and min(ip) >= 0.5 and ip[0] <= Wd - 1 and ip[1] <= Hd - 1

    pts, kps, tags = [], {k: [] for k in ((0, 0), (0, 1), (1, 0), (1, 1))}, []     # (frame A=0 / B=1, cam)

    def add(X, tag, off_b=(0.0, 0.0), noise=0.25):
        ps = {k: proj(pa if k[0] == 0 else pb, k[1], X) for k in kps}
        if not all(ok for _, ok in ps.values()):
            return False
        pts.append(X); tags.append(tag)
        for k, (ip, _) in ps.items():
            kps[k].append(ip + rng.normal(0, noise, 2) + (np.asarray(off_b) if k[0] == 1 else 0.0))
        return True

    n_true = n_kp - 40 - 8
    while len(pts) < n_true:
        z = float(np.exp(rng.uniform(np.log(1.0), np.log(60.0))))
        add(world(np.array([rng.uniform(-0.7, 0.7) * z, rng.uniform(-0.45, 0.45) * z, z])), "plain")
    while not add(world(np.array([rng.uniform(-0.3, 0.3) * 2000.0, rng.uniform(-0.2, 0.2) * 2000.0, 2000.0])), "parallel", noise=0.0):
        pass
    while not add(world(np.array([rng.uniform(-0.5, 0.5) * 6.0, rng.uniform(-0.3, 0.3) * 6.0, 6.0])), "border",
                  off_b=(0.0, 6 * 0.8 * 10.0 / 12.0), noise=0.0):
        pass
    while not add(world(np.array([rng.uniform(-0.3, 0.3) * 2.0, rng.uniform(-0.2, 0.2) * 2.0, 2.0])), "rank"):
        pass
    n = len(pts)
    base = rng.integers(0, 256, (n, desc_bytes), dtype=np.uint8)
    store, perm, truth = {}, {}, {}
    fa, fb = 1, 3
    lm_init = (rng.random(L) < 0.5).astype(np.uint8)
    slots = rng.choice(L, 64, replace=False)
    lm_init[slots[:16]] = 1
    lm_init[slots[16:]] = 0
    near = [i for i, t in enumerate(tags) if t == "plain" and np.linalg.norm(pts[i] - world(np.zeros(3))) < 20.0]
    pick = rng.choice(near, 48, replace=False)
    host_only = {}
    for (fr, cam), kp in kps.items():
        kp = np.array(kp)
        desc = np.stack([_flip(rng, base[i], int(rng.integers(0, 5))) for i in range(n)])
        size = rng.uniform(6.0, 14.0, n)
        size[[i for i, t in enumerate(tags) if t == "border"]] = 10.0
        src = rng.integers(0, n_true, 20)
        kd = np.stack([rng.uniform(20, Wd - 20, 40), rng.uniform(20, Hd - 20, 40)], 1)
        dd = np.concatenate([np.stack([_flip(rng, base[i], 8) for i in src]), rng.integers(0, 256, (20, desc_bytes), dtype=np.uint8)])
        kp, desc = np.concatenate([kp, kd]), np.concatenate([desc, dd])
        size = np.concatenate([size, rng.uniform(6.0, 14.0, 40)])
        tr = np.concatenate([np.arange(n), -np.ones(40, int)])
        lm = -np.ones(len(kp), np.int32)
        ho = np.zeros(len(kp), bool)
        if fr == 0:
            lm[pick[0:6]] = slots[0:6]                  # A: initialised landmark (skipped)
            lm[pick[6:14]] = slots[16:24]               # A: uninitialised landmark
            ho[pick[14:24]] = True                      # A: an id on the host only
            lm[pick[40:46]] = slots[32:38]              # both named
        else:
            lm[pick[24:30]] = slots[24:30]              # B: uninitialised landmark
            lm[pick[30:34]] = slots[6:10]               # B: initialised landmark (skipped)
            lm[pick[40:46]] = slots[38:44]              # both named
        p = rng.permutation(len(kp))
        f32 = lambda x: np.asarray(x, np.float32).astype(np.float64)
        key = (fa if fr == 0 else fb, cam)
        store[key] = dict(kp=f32(kp[p]), size=f32(size[p]), desc=np.ascontiguousarray(desc[p]), lm=lm[p],
                          observed=(lm[p] >= 0).astype(np.uint8))
        perm[key] = np.argsort(p)
        truth[key] = tr[p]
        host_only[key] = ho[p]
    state = dict(poses=w.poses, extrinsics=w.extrinsics, cameras=w.cameras, landmarks=np.array(w.landmarks), lm_init=lm_init,
                 store=store, speed_bias=w.speed_bias)
    rank_i = tags.index("rank")
    return dict(window=w, state=state, F=4, n_kp=n + 40, desc_bytes=desc_bytes, speed=speed, sb_b=pb,
                frames=dict(pose_a=pa, feat_slot_a=fa, pose_b=pb, feat_slot_b=fb), truth=truth, host_only=host_only,
                points=np.array(pts), tags=tags, perm=perm,
                rank_pair=(int(perm[(fa, 0)][rank_i]), int(perm[(fb, 0)][rank_i])))


def _rank_threshold(sc, job):
    """The A keypoint size of the rank pair at which the reference's rank of H drops below 9 under this job's prior."""
    a, b = sc["rank_pair"]
    g = ref.setup(sc["state"], job)

    def full_rank(size):
        g2 = dict(g, size_a=g["size_a"].copy(), rs_a=g["rs_a"].copy())
        g2["size_a"][a] = size
        g2["rs_a"][a] = sref.ray_sigmas(size, float(g["cam_a"]["fu"]))
        ok, hp, par = sref.stereo_triangulate(g2, a, b, [])
        assert ok and not par
        r2, H, *_ = sref.uncertainty_H(g2, a, b, hp)
        assert r2 >= 4.0
        return sref.qr_rank(H) == 9

    lo, hi = 10.0, 1e12
    assert full_rank(lo) and not full_rank(hi)
    for _ in range(80):
        mid = np.sqrt(lo * hi)
        lo, hi = (mid, hi) if full_rank(mid) else (lo, mid)
    return hi


def variants(sc):
    return jobs(sc, True) + jobs(sc, False)


def make_temporal_scene(seed, distortion=abi.DIST_RADTAN, n_kp=400, desc_bytes=48, oracle=None):
    """The scene and the reference's records of every job variant; re-drawn until no decision lies within MIN_MARGIN of
    its threshold."""
    for sub in range(20):
        sc = _draw(seed, sub, distortion, n_kp, desc_bytes)
        j_fast, j_slow = jobs(sc, True)[0], jobs(sc, False)[0]
        t_fast, t_slow = _rank_threshold(sc, j_fast), _rank_threshold(sc, j_slow)
        a, _ = sc["rank_pair"]
        sc["state"]["store"][(sc["frames"]["feat_slot_a"], 0)]["size"][a] = float(np.float32(4.0 * max(t_fast, t_slow)))
        margins, records, cases, dets = [], [], [], []
        for j in variants(sc):
            cs, ds = [], []
            recs, g = ref.match2d2d(oracle, sc["state"], j, margins=margins, cases=cs, dets=ds)
            A, B = sc["state"]["store"][(j["feat_slot_a"], j["cam_a"])], sc["state"]["store"][(j["feat_slot_b"], j["cam_b"])]
            dist = np.unpackbits(A["desc"][:, None, :] ^ B["desc"][None, :, :], axis=2).sum(2)
            for aa, bb in zip(*np.nonzero(dist < 60)):
                if not (g["skipA"][aa] or g["skipB"][bb]):
                    sref.stereo_triangulate(g, int(aa), int(bb), margins)
            records.append(recs); cases.append(cs); dets.append(ds)
        if min(m for _, m in margins) > MIN_MARGIN:
            sc.update(records=records, cases=cases, dets=dets, margins=margins, sub=sub, rank_sizes=(t_fast, t_slow))
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
