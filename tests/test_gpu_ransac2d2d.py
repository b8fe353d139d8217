"""GPU checks of okb_ransac_2d2d_batch (Frontend::runRansac2d2d on the device) against the restatement
tests/ransac2d2d_reference.py: correspondence counts, per-hypothesis inlier counts of both problems, winners, choice,
ret, rotationOnly and outlier lists identical, models and the initialised pose within 1e-9, on every scene kind; a
batch equal to single calls; no change to the window; host-side errors naming their job; n_jobs == 0; world 2 and 4 on
one device byte-identical to an unsharded context."""
import numpy as np
import pytest

from okvis_b200 import abi, capi, synthetic
import ransac2d2d_reference as rr
import ransac2d2d_scene as S

pytestmark = pytest.mark.gpu

DISTS = [abi.DIST_NONE, abi.DIST_RADTAN, abi.DIST_EQUIDISTANT, abi.DIST_RADTAN8]
MOTIONS = ["rotation", "small", "large"]


def _close(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() <= 1e-9 * max(1.0, np.abs(np.asarray(b)).max())


def assert_same(got, want, degenerate=False):
    """degenerate: a scene without translation or with a short baseline, where the five-point problem has (almost) no
    translation to find and its minimal solutions fit noise, so that a last-bit difference in evaluation order between
    the device and NumPy (with or without fused multiply-adds) can move a solution;
    there the five-point inlier counts may differ in at most 5 hypotheses per camera, and its winner's model is compared
    only when the winners agree.  Everything the decision, the outliers and the pose depend on is compared as always."""
    for k in ("ret", "rotation_only", "pose_set", "n_outliers"):
        assert int(got[k]) == int(want[k]), (k, got[k], want[k])
    if degenerate:
        assert np.array_equal(got["hyp_inliers"][:, 0], want["hyp_inliers"][:, 0])
        diff = (got["hyp_inliers"][:, 1] != want["hyp_inliers"][:, 1]).sum(1)
        assert np.all(diff <= 5), diff
    else:
        assert np.array_equal(got["hyp_inliers"], want["hyp_inliers"])
    assert [tuple(int(v) for v in o) for o in got["outliers"]] == [tuple(o) for o in want["outliers"]]
    for g, w in zip(got["cams"], want["cams"]):
        rel_free = degenerate and not w["applied"] or degenerate and w["rotation_only"]
        for k in ("n_correspondences", "rot_inliers", "rel_inliers", "rot_best", "rel_best", "rotation_only", "applied",
                  "n_outliers"):
            if rel_free and k in ("rel_inliers", "rel_best"):
                continue
            assert int(g[k]) == int(w[k]), (k, g[k], w[k])
        assert _close(g["R_rot"], w["R_rot"])
        if not rel_free or g["rel_best"] == w["rel_best"]:
            assert _close(g["R_rel"], w["R_rel"]) and _close(g["t_rel"], w["t_rel"])
    if want["pose_set"]:
        q, qw = got["T_WS"][3:], want["T_WS"][3:]
        qw = qw if q @ qw >= 0 else -qw
        assert _close(got["T_WS"][:3], want["T_WS"][:3]) and np.abs(q - qw).max() <= 1e-9
    else:
        assert not np.any(got["T_WS"])


def _scenes():
    out = []
    for i, (d, m) in enumerate([(d, m) for m in MOTIONS for d in DISTS]):
        # without a usable baseline at most 10 % wrong: the rotation-only ratio stays above 0.8 and decides
        out.append(S.make_scene(300 + i, d, 1 + i % 2, m, (0.0, 0.1, 0.3 if m == "large" else 0.1)[i % 3]))
    out.append(S.restrict(S.make_scene(399, abi.DIST_RADTAN, 2, "large", 0.1), 1, 8))
    return out


def _check_margins(sc, job):
    m = []
    want = rr.ransac2d2d(S.state(sc), job, margins=m)
    assert not m or min(m) > S.MIN_MARGIN
    return want


def test_scenes_vs_reference():
    scenes = _scenes()
    ctx = capi.Context(0, len(scenes))
    for s, sc in enumerate(scenes):
        S.load(ctx, s, sc)
    jobs = [dict(S.job(sc, 900 + s, initialize_pose=bool(s % 2)), win=s) for s, sc in enumerate(scenes)]
    got = ctx.ransac_2d2d_batch(jobs)
    for s, sc in enumerate(scenes):
        assert_same(got[s], _check_margins(sc, jobs[s]), degenerate=sc["motion"] != "large")
    assert got[-1]["cams"][1]["n_correspondences"] < 10 and got[-1]["cams"][1]["rel_best"] == -1
    ctx.close()


def test_batch_equals_single_calls():
    scenes = _scenes()[:8]
    ctx = capi.Context(0, len(scenes))
    for s, sc in enumerate(scenes):
        S.load(ctx, s, sc)
    jobs = [dict(S.job(sc, 40 + s, initialize_pose=s % 3 == 0, max_iterations=(50, 64, 1, 17)[s % 4]), win=s)
            for s, sc in enumerate(scenes)]
    batch = ctx.ransac_2d2d_batch(jobs)
    for s in range(len(scenes)):
        one = ctx.ransac_2d2d_batch([jobs[s]])[0]
        assert_same(one, batch[s])              # the same device code on the same data: exact, degenerate or not
        assert np.array_equal(one["T_WS"], batch[s]["T_WS"])
        for a, b in zip(one["cams"], batch[s]["cams"]):
            for k in ("R_rot", "R_rel", "t_rel"):
                assert np.array_equal(a[k], b[k])
    ctx.close()


def test_window_unchanged():
    sc = S.make_scene(4, abi.DIST_RADTAN, 2, "large", 0.3)
    ctx = capi.Context(0, 1)
    S.load(ctx, 0, sc)
    before = ctx.download(0)
    first = ctx.ransac_2d2d_batch([dict(S.job(sc, 1, initialize_pose=True), win=0)])[0]
    after = ctx.download(0)
    for k in before:
        if before[k] is not None:
            assert np.array_equal(before[k], after[k]), k
    assert_same(ctx.ransac_2d2d_batch([dict(S.job(sc, 1, initialize_pose=True), win=0)])[0], first)
    ctx.close()


def test_errors_before_device_work():
    sc = S.make_scene(9, abi.DIST_RADTAN, 2, "large", 0.1)
    ctx = capi.Context(0, 3)
    S.load(ctx, 0, sc)
    ctx.upload(1, synthetic.make_window(1, 0))
    good = dict(S.job(sc, 1), win=0)
    bad = [dict(good, win=1), dict(good, win=2), dict(good, win=7), dict(good, win=-1),
           dict(good, feat_slot_a=5), dict(good, feat_slot_b=-1), dict(good, pose_a=9), dict(good, pose_b=-1),
           dict(good, n_cams=3), dict(good, n_cams=0), dict(good, max_iterations=0), dict(good, max_iterations=65),
           dict(good, threshold=0.0), dict(good, threshold=float("nan")), dict(good, out=None), dict(good, outlier_cap=10)]
    for bd in bad:
        with pytest.raises(capi.OkbError) as e:
            ctx.ransac_2d2d_batch([good, bd])
        assert e.value.code == abi.OKB_ERR_INVALID_ARG, bd
        assert "jobs[1]" in str(e.value), (bd, str(e.value))
    assert capi.lib().okb_ransac_2d2d_batch(ctx._h, 0, None) == abi.OKB_OK
    assert capi.lib().okb_ransac_2d2d_batch(ctx._h, -1, None) == abi.OKB_ERR_INVALID_ARG
    assert_same(ctx.ransac_2d2d_batch([good])[0], rr.ransac2d2d(S.state(sc), good))
    ctx.close()


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_equals_the_unsharded_window(world):
    from test_gpu_shard_frontend import Group, call_same
    sc = S.make_scene(12, abi.DIST_RADTAN, 2, "large", 0.1)
    w = sc["window"]
    g = Group(world, len(w.poses))
    try:
        g.upload(0, w, S.N_FEAT, sc["n_cams"], max(len(e["lm"]) for e in sc["store"].values()), 48)
        for (f, c), e in sorted(sc["store"].items()):
            n = len(e["lm"])
            g.edit(0, "set_features", f, c, np.stack([e["kp"][:, 0], e["kp"][:, 1], e["size"]], 1),
                   np.zeros((n, 48), np.uint8), e["lm"], (e["lm"] >= 0).astype(np.uint8))
            g.commit(0)
        r = call_same(g, "ransac_2d2d_batch", [dict(S.job(sc, 3, initialize_pose=True), win=0)])
        assert r[0]["ret"] > 10 and r[0]["pose_set"] == 1
        assert_same(r[0], rr.ransac2d2d(S.state(sc), S.job(sc, 3, initialize_pose=True)))
    finally:
        g.close()
