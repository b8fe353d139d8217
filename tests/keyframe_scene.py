"""Seeded keyframe-decision scenes (okb_keyframe_overlap_batch, tests/keyframe_reference.py): images of keypoints with
a store slot per keypoint (-1: no landmark), and sessions of 1-4 such images (one per camera).

  random_image   400 keypoints uniform over a 752x480 image, in float; a planted matched set: the points inside a
                 random ellipse, each kept with a random probability, plus a few matched points scattered outside
  CASES          the degenerate images: 0, 1, 2 and 3 points; duplicates and collinear rows; all points equal and all
                 collinear (NaN overlap); all matched and none matched; matched points only on their own hull (inside 0,
                 ratio inf); points on a circle (cv::convexHull's cyclic shift); query points on vertices and on
                 horizontal and vertical edges of the matched hull; one image of 65 535 keypoints

make_sessions(seed, n) draws n sessions whose decisions all lie more than 1e-9 relative away from the thresholds."""
import numpy as np

import keyframe_reference as ref

W, H = 752, 480
THR_O, THR_R = 0.6, 0.2


def _f32(p):
    return np.asarray(p, np.float32).astype(np.float64)


def random_image(rng, n=400):
    kp = _f32(np.stack([rng.uniform(0, W, n), rng.uniform(0, H, n)], 1))
    cx, cy = rng.uniform(0.3, 0.7) * W, rng.uniform(0.3, 0.7) * H
    ax, ay = rng.uniform(0.15, 0.6) * W, rng.uniform(0.15, 0.6) * H
    inside = ((kp[:, 0] - cx) / ax) ** 2 + ((kp[:, 1] - cy) / ay) ** 2 < 1.0
    matched = (inside & (rng.uniform(0, 1, n) < rng.uniform(0.05, 0.9))) | (rng.uniform(0, 1, n) < 0.02)
    return kp, np.where(matched, rng.integers(0, 300, n), -1).astype(np.int32)


def _lm(matched, rng):
    matched = np.asarray(matched, bool)
    return np.where(matched, rng.integers(0, 300, len(matched)), -1).astype(np.int32)


def _cases():
    rng = np.random.default_rng(7)
    c = {}
    for n in (0, 1, 2, 3):
        kp = _f32(rng.uniform(0, 100, (n, 2)))
        c["points_%d" % n] = (kp, _lm(np.ones(n, bool), rng))
    # duplicates and collinear rows: integer rows, every third point repeated
    xs = np.repeat(np.arange(0, 40, 4.0), 3)
    rows = np.concatenate([np.stack([xs, np.full_like(xs, y)], 1) for y in (10.0, 20.0, 30.0)])
    rows = np.concatenate([rows, rows[::3]])
    perm = rng.permutation(len(rows))
    c["duplicates_rows"] = (_f32(rows[perm]), _lm(rng.uniform(0, 1, len(rows)) < 0.5, rng))
    c["all_equal"] = (_f32(np.tile([[12.5, 40.25]], (9, 1))), _lm(np.ones(9, bool), rng))
    t = rng.permutation(np.arange(20.0))
    c["all_collinear"] = (_f32(np.stack([3 * t + 1, 2 * t + 5], 1)), _lm(np.ones(20, bool), rng))
    kp, _ = random_image(rng)
    c["all_matched"] = (kp, _lm(np.ones(len(kp), bool), rng))
    c["none_matched"] = (kp, _lm(np.zeros(len(kp), bool), rng))
    # matched: the corners of a square; every other point outside it
    corners = np.array([[100.0, 100.0], [300.0, 100.0], [300.0, 300.0], [100.0, 300.0], [200.0, 100.0]])
    out = np.stack([rng.uniform(400, 700, 40), rng.uniform(0, 480, 40)], 1)
    kp = _f32(np.concatenate([out[:20], corners, out[20:]]))
    c["matched_on_own_hull"] = (kp, _lm(np.r_[np.zeros(20, bool), np.ones(5, bool), np.zeros(20, bool)], rng))
    # a circle in angle order (the hull's indices ascend: cv::convexHull rotates them) and one in reverse
    a = np.linspace(0, 2 * np.pi, 64, endpoint=False)
    circ = np.stack([376 + 200 * np.cos(a), 240 + 200 * np.sin(a)], 1)
    c["circle"] = (_f32(circ), _lm(np.arange(64) % 3 != 1, rng))
    c["circle_reversed"] = (_f32(circ[::-1]), _lm(np.arange(64) % 2 == 0, rng))
    # matched: an axis-aligned rectangle; queries on its vertices, on its horizontal and vertical edges, inside, outside
    rect = np.array([[50.0, 60.0], [250.0, 60.0], [250.0, 200.0], [50.0, 200.0]])
    edges = np.array([[150.0, 60.0], [120.0, 200.0], [50.0, 100.0], [250.0, 150.0], [50.0, 60.0], [250.0, 200.0]])
    inner = np.stack([rng.uniform(60, 240, 30), rng.uniform(70, 190, 30)], 1)
    outer = np.stack([rng.uniform(300, 700, 10), rng.uniform(0, 480, 10)], 1)
    kp = _f32(np.concatenate([edges, rect, inner, outer]))
    c["on_edges"] = (kp, _lm(np.r_[np.zeros(6, bool), np.ones(4, bool), rng.uniform(0, 1, 30) < 0.3, np.zeros(10, bool)], rng))
    return c


CASES = _cases()


def big_image(seed=11, n=65535):
    rng = np.random.default_rng(seed)
    return random_image(rng, n)


def camera_values(kp, lm):
    return ref.camera_overlap(kp, lm >= 0)


def session_values(images):
    cams = [camera_values(kp, lm) for kp, lm in images]
    need, overlap, ratio = ref.keyframe_decision(cams, THR_O, THR_R)
    return dict(cams=cams, need_keyframe=need, overlap=overlap, ratio=ratio)


def _clear(v, thr):
    return not np.isfinite(v) or abs(v - thr) > 1e-9 * abs(thr)


def make_sessions(seed, n_sessions, n_cams=None):
    """n_sessions sessions of 1-4 random images (n_cams: fixed count); the decision values are clear of the thresholds."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n_sessions:
        nc = n_cams or int(rng.integers(1, 5))
        images = [random_image(rng) for _ in range(nc)]
        v = session_values(images)
        if all(_clear(c["overlap"], float(np.float32(THR_O))) and _clear(c["ratio"], float(np.float32(THR_R)))
               for c in v["cams"] if not c["skipped"]):
            out.append(dict(images=images, **v))
    return out


def load(ctx, win, images, feat_slot=1, n_feat=2, window=None):
    """Uploads a small synthetic window into `win` and puts `images` (one per camera) into its feature slot."""
    from okvis_b200 import synthetic
    w = window if window is not None else synthetic.make_window(1, 0)
    ctx.reserve(win, len(w.poses), len(w.landmarks), len(w.obs), len(w.imu_samples))
    n_max = max([len(kp) for kp, _ in images] + [1])
    ctx.reserve_features(win, n_feat, len(images), n_max, 48)
    ctx.upload(win, w)
    for cam, (kp, lm) in enumerate(images):
        n = len(kp)
        k = np.zeros((n, 3))
        if n:
            k[:, :2], k[:, 2] = kp, 12.0
        ctx.set_features(win, feat_slot, cam, k, np.zeros((n, 48), np.uint8), lm, np.zeros(n, np.uint8))
    ctx.commit(win, 1)
