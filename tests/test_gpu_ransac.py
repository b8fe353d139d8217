"""GPU checks of okb_ransac_3d2d_batch (Frontend::runRansac3d2d on the device) against the restatement
tests/ransac_reference.py: correspondence counts, per-hypothesis inlier counts, winner and outlier lists identical and
models within 1e-9 for 1, 8 and 132 sessions and every scene kind; a batch equal to single calls; injected outliers
rejected; no change to the window, its store or a following optimize; host-side errors."""
import numpy as np
import pytest

from okvis_b200 import abi, capi, synthetic
import ransac_reference as rr
import ransac_scene as S

pytestmark = pytest.mark.gpu

DISTS = [abi.DIST_NONE, abi.DIST_RADTAN, abi.DIST_EQUIDISTANT, abi.DIST_RADTAN8]


def job(win, sc, seed, **kw):
    return dict(win=win, feat_slot=S.FEAT, n_cams=sc["n_cams"], seed=seed, **kw)


def assert_same(got, want):
    for k in ("ret", "n_correspondences", "n_inliers", "best", "n_outliers"):
        assert int(got[k]) == int(want[k]), (k, got[k], want[k])
    assert np.array_equal(got["hyp_inliers"], want["hyp_inliers"])
    assert [tuple(int(v) for v in o) for o in got["outliers"]] == [tuple(o) for o in want["outliers"]]
    if want["best"] >= 0:
        q, qw = got["T_WS"][3:], want["T_WS"][3:]
        qw = qw if q @ qw >= 0 else -qw
        assert np.abs(got["T_WS"][:3] - want["T_WS"][:3]).max() <= 1e-9 * max(1.0, np.abs(want["T_WS"][:3]).max())
        assert np.abs(q - qw).max() <= 1e-9
    else:
        assert not np.any(got["T_WS"])


def _scenes(n):
    return [S.make_scene(200 + i, DISTS[i % 4], 2 + 2 * ((i // 4) % 2), (0.0, 0.1, 0.3, 0.5)[(i // 8) % 4]) for i in range(n)]


@pytest.mark.parametrize("n_sessions", [1, 8, 132])
def test_sessions_vs_reference(n_sessions):
    scenes = _scenes(min(n_sessions, 32))
    ctx = capi.Context(0, n_sessions)
    for s in range(n_sessions):
        S.load(ctx, s, scenes[s % len(scenes)])
    got = ctx.ransac_3d2d_batch([job(s, scenes[s % len(scenes)], 1000 + s) for s in range(n_sessions)])
    for s in range(n_sessions):
        sc = scenes[s % len(scenes)]
        m = []
        want = rr.ransac(S.state(sc), S.FEAT, sc["n_cams"], 1000 + s, margins=m)
        assert min(m) > S.MIN_MARGIN
        assert_same(got[s], want)
    ctx.close()


def test_edge_jobs():
    sc = S.make_scene(5, abi.DIST_RADTAN, 2, 0.0)
    variants = [S.restrict(sc, max_assoc=2), S.restrict(sc, max_assoc=4), S.restrict(sc, empty_cam=1), sc]
    ctx = capi.Context(0, len(variants) + 1)
    for s, v in enumerate(variants):
        S.load(ctx, s, v)
    got = ctx.ransac_3d2d_batch([job(s, v, 3) for s, v in enumerate(variants)])
    for s, v in enumerate(variants):
        assert_same(got[s], rr.ransac(S.state(v), S.FEAT, 2, 3))
    assert got[0]["n_correspondences"] < 5 and got[0]["ret"] == got[0]["n_correspondences"]
    assert 5 <= got[1]["n_correspondences"] and got[1]["n_inliers"] < 10 and got[1]["n_outliers"] == 0
    ctx.close()


def test_one_frame_window():
    # the window keeps only its newest frame: runRansac3d2d returns 1 before building the adapter (Frontend.cpp:579-582)
    sc = S.make_scene(5, abi.DIST_RADTAN, 2, 0.0, n_frames=3)
    w = sc["window"]
    B = len(w.poses) - 1
    obs = w.obs[w.obs["pose_idx"] == B].copy()
    obs["pose_idx"] = 0
    w.poses, w.speed_bias, w.obs = w.poses[B:].copy(), w.speed_bias[B:].copy(), obs
    w.imu_terms = w.imu_terms[:0].copy()
    two = S.make_scene(6, abi.DIST_RADTAN, 2, 0.1)
    ctx = capi.Context(0, 2)
    S.load(ctx, 0, sc)
    S.load(ctx, 1, two)
    got = ctx.ransac_3d2d_batch([job(0, sc, 3), job(1, two, 3)])
    want = rr.ransac(S.state(sc), S.FEAT, 2, 3)
    assert want["ret"] == 1 and want["n_correspondences"] == 0
    assert_same(got[0], want)
    assert_same(got[1], rr.ransac(S.state(two), S.FEAT, 2, 3))
    ctx.close()


def test_batch_equals_single_calls():
    scenes = _scenes(8)
    ctx = capi.Context(0, len(scenes))
    for s, sc in enumerate(scenes):
        S.load(ctx, s, sc)
    jobs = [job(s, sc, 50 + s, max_iterations=(50, 64, 1, 17)[s % 4]) for s, sc in enumerate(scenes)]
    batch = ctx.ransac_3d2d_batch(jobs)
    for s in range(len(scenes)):
        assert_same(ctx.ransac_3d2d_batch([jobs[s]])[0], batch[s])
    ctx.close()


@pytest.mark.parametrize("distortion", DISTS)
def test_injected_outliers_rejected(distortion):
    # the scenes and seed of tests/test_ransac_reference.py::test_scene_outcome; elsewhere a true association scoring
    # just above the threshold under a model from a noisy minimal sample can be rejected, on the device as in OKVIS
    for n_cams in (2, 4):
        for wrong in (0.1, 0.3):
            sc = S.make_scene(11 + n_cams, distortion, n_cams, wrong)
            ctx = capi.Context(0, 1)
            S.load(ctx, 0, sc)
            r = ctx.ransac_3d2d_batch([job(0, sc, 77)])[0]
            assert_same(r, rr.ransac(S.state(sc), S.FEAT, n_cams, 77))
            outs = {(int(o["cam"]), int(o["kp"])) for o in r["outliers"]}
            n_nan = n_cams if distortion == abi.DIST_RADTAN8 else 0
            assert len(outs - sc["injected"]) == n_nan and sc["injected"] <= outs
            ctx.close()


def test_window_unchanged_and_optimize_bit_identical():
    sc = S.make_scene(4, abi.DIST_RADTAN, 2, 0.3)
    a, b = capi.Context(0, 1), capi.Context(0, 1)
    S.load(a, 0, sc); S.load(b, 0, sc)
    before = b.download(0)
    first = b.ransac_3d2d_batch([job(0, sc, 1)])[0]
    after = b.download(0)
    for k in before:
        if before[k] is not None:
            assert np.array_equal(before[k], after[k]), k
    assert_same(b.ransac_3d2d_batch([job(0, sc, 1)])[0], first)         # the store is unchanged too
    sa, sb = a.optimize(0, 1, max_iterations=5)[0], b.optimize(0, 1, max_iterations=5)[0]
    assert sa["final_cost"] == sb["final_cost"] and sa["iterations"] == sb["iterations"]
    a.close(); b.close()


def test_pending_removals_are_committed_first():
    sc = S.make_scene(8, abi.DIST_RADTAN, 2, 0.1)
    ctx = capi.Context(0, 1)
    S.load(ctx, 0, sc)
    e = sc["store"][(S.FEAT, 0)]
    k = np.nonzero(e["lm"] >= 0)[0][:20]
    ctx.set_feature_landmarks(0, S.FEAT, 0, k, np.full(len(k), -1), np.zeros(len(k)))
    sc2 = S.restrict(sc)
    sc2["store"][(S.FEAT, 0)]["lm"][k] = -1
    assert_same(ctx.ransac_3d2d_batch([job(0, sc, 2)])[0], rr.ransac(S.state(sc2), S.FEAT, 2, 2))
    ctx.close()


def test_errors_before_device_work():
    sc = S.make_scene(9, abi.DIST_RADTAN, 2, 0.1)
    ctx = capi.Context(0, 3)
    S.load(ctx, 0, sc)
    ctx.upload(1, synthetic.make_window(1, 0))
    good = job(0, sc, 1)
    bad = [dict(good, win=1), dict(good, win=2), dict(good, win=7), dict(good, win=-1),
           dict(good, feat_slot=5), dict(good, feat_slot=0),
           dict(good, n_cams=3), dict(good, n_cams=0),
           dict(good, max_iterations=0), dict(good, max_iterations=65),
           dict(good, threshold=0.0), dict(good, threshold=float("nan")),
           dict(good, out=None), dict(good, outlier_cap=10)]
    for bd in bad:
        with pytest.raises(capi.OkbError) as e:
            ctx.ransac_3d2d_batch([bd])
        assert e.value.code == abi.OKB_ERR_INVALID_ARG, bd
        assert "jobs[0]" in str(e.value)
    with pytest.raises(capi.OkbError) as e:
        ctx.ransac_3d2d_batch([good, good])
    assert e.value.code == abi.OKB_ERR_INVALID_ARG and "jobs[1]" in str(e.value)
    assert capi.lib().okb_ransac_3d2d_batch(ctx._h, 0, None) == abi.OKB_OK
    assert capi.lib().okb_ransac_3d2d_batch(ctx._h, -1, None) == abi.OKB_ERR_INVALID_ARG
    assert_same(ctx.ransac_3d2d_batch([good])[0], rr.ransac(S.state(sc), S.FEAT, 2, 1))
    ctx.close()
    c0, c1 = capi.Context(0, 1), capi.Context(0, 1)
    capi.Context.shard_connect_local([c0, c1])
    with pytest.raises(capi.OkbError) as e:
        c0.ransac_3d2d_batch([good])
    assert e.value.code == abi.OKB_ERR_UNSUPPORTED
    c0.close(); c1.close()
