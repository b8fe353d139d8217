"""GPU checks of okb_keyframe_overlap_batch (Frontend::doWeNeedANewKeyframe on the device) against the restatement
tests/keyframe_reference.py: every per-camera value, maximum and decision bit-identical for 1, 8 and 132 sessions, for
the degenerate images and for a 65 535-keypoint image; a mixed batch against single calls; no change to the window or
a following optimize; host-side errors."""
import numpy as np
import pytest

from okvis_b200 import abi, capi, synthetic
import keyframe_scene as S

pytestmark = pytest.mark.gpu

_FIELDS = ("n_points", "n_matched", "hull_all", "hull_matched", "inside", "skipped", "area_all", "area_matched", "overlap",
           "ratio")


def _bits(v):
    return np.float64(v).tobytes()


def assert_same(got, want):
    """Integers equal, doubles bit-identical (NaN and inf included)."""
    assert len(got["cams"]) == len(want["cams"])
    for g, w in zip(got["cams"], want["cams"]):
        for k in _FIELDS:
            if isinstance(w[k], float):
                assert _bits(g[k]) == _bits(w[k]), (k, g[k], w[k])
            else:
                assert int(g[k]) == int(w[k]), (k, g[k], w[k])
    assert _bits(got["overlap"]) == _bits(want["overlap"]) and _bits(got["ratio"]) == _bits(want["ratio"])
    assert got["need_keyframe"] == want["need_keyframe"]


def job(win, n_cams, **kw):
    return dict(win=win, feat_slot=1, n_cams=n_cams, overlap_threshold=S.THR_O, matching_ratio_threshold=S.THR_R, **kw)


@pytest.mark.parametrize("n_sessions", [1, 8, 132])
def test_sessions_vs_reference(n_sessions):
    sess = S.make_sessions(100 + n_sessions, min(n_sessions, 16))
    ctx = capi.Context(0, n_sessions)
    for s in range(n_sessions):
        S.load(ctx, s, sess[s % len(sess)]["images"])
    got = ctx.keyframe_overlap_batch([job(s, len(sess[s % len(sess)]["images"])) for s in range(n_sessions)])
    for s in range(n_sessions):
        assert_same(got[s], sess[s % len(sess)])
    if n_sessions > 1:
        assert {bool(x["need_keyframe"]) for x in sess} == {True, False}
    ctx.close()


def test_degenerate_cases():
    names = sorted(S.CASES)
    ctx = capi.Context(0, len(names))
    for s, name in enumerate(names):
        S.load(ctx, s, [S.CASES[name]])
    got = ctx.keyframe_overlap_batch([job(s, 1) for s in range(len(names))])
    for s, name in enumerate(names):
        assert_same(got[s], S.session_values([S.CASES[name]]))
    ctx.close()


def test_nan_and_inf_maxima():
    # camera order decides: a NaN overlap first wins; a NaN running maximum is replaced by the next camera's value
    rng = np.random.default_rng(3)
    img = S.random_image(rng)
    for images in ([S.CASES["all_equal"], img], [img, S.CASES["all_equal"]], [S.CASES["all_collinear"], S.CASES["points_2"], img],
                   [S.CASES["circle"], img, S.CASES["matched_on_own_hull"]]):
        ctx = capi.Context(0, 1)
        S.load(ctx, 0, images)
        assert_same(ctx.keyframe_overlap_batch([job(0, len(images))])[0], S.session_values(images))
        ctx.close()


def test_large_image():
    big = S.big_image()
    rng = np.random.default_rng(5)
    images = [big, S.random_image(rng, 3000)]           # beyond shared memory: global scratch
    ctx = capi.Context(0, 2)
    S.load(ctx, 0, images)
    S.load(ctx, 1, [S.random_image(rng)])
    got = ctx.keyframe_overlap_batch([job(0, 2), job(1, 1)])
    assert_same(got[0], S.session_values(images))
    ctx.close()


def test_batch_equals_single_calls():
    rng = np.random.default_rng(9)
    sets = [[S.random_image(rng) for _ in range(k)] for k in (1, 2, 3, 4)] + [[S.CASES["circle"], S.CASES["on_edges"]],
                                                                         [S.random_image(rng, 2500)]]
    ctx = capi.Context(0, len(sets))
    for s, images in enumerate(sets):
        S.load(ctx, s, images)
    batch = ctx.keyframe_overlap_batch([job(s, len(im)) for s, im in enumerate(sets)])
    for s, images in enumerate(sets):
        single = ctx.keyframe_overlap_batch([job(s, len(images))])[0]
        assert_same(single, batch[s])
        assert_same(single, S.session_values(images))
    ctx.close()


def test_window_unchanged_and_optimize_bit_identical():
    images = [S.random_image(np.random.default_rng(4)) for _ in range(2)]
    a, b = capi.Context(0, 1), capi.Context(0, 1)
    S.load(a, 0, images); S.load(b, 0, images)
    before = b.download(0)
    first = b.keyframe_overlap_batch([job(0, 2)])[0]
    after = b.download(0)
    for k in before:
        if before[k] is not None:
            assert np.array_equal(before[k], after[k]), k
    assert_same(b.keyframe_overlap_batch([job(0, 2)])[0], first)
    sa, sb = a.optimize(0, 1, max_iterations=10)[0], b.optimize(0, 1, max_iterations=10)[0]
    assert sa["final_cost"] == sb["final_cost"] and sa["iterations"] == sb["iterations"]
    da, db = a.download(0), b.download(0)
    for k in da:
        if da[k] is not None:
            assert np.array_equal(da[k], db[k]), k
    a.close(); b.close()


def test_pending_edits_are_committed_first():
    # a RANSAC removal arrives as a store edit just before the decision
    kp, lm = S.random_image(np.random.default_rng(6))
    ctx = capi.Context(0, 1)
    S.load(ctx, 0, [(kp, lm)])
    k = np.nonzero(lm >= 0)[0][:5]
    ctx.set_feature_landmarks(0, 1, 0, k, np.full(len(k), -1), np.zeros(len(k)))
    lm2 = lm.copy()
    lm2[k] = -1
    got = ctx.keyframe_overlap_batch([job(0, 1)])[0]
    assert_same(got, S.session_values([(kp, lm2)]))
    assert got["cams"][0]["n_matched"] == int((lm >= 0).sum()) - 5
    ctx.close()


def test_errors_before_device_work():
    img = S.random_image(np.random.default_rng(8))
    ctx = capi.Context(0, 3)
    S.load(ctx, 0, [img, img])
    ctx.upload(1, synthetic.make_window(1, 0))
    good = job(0, 2)
    bad = [dict(good, win=1),                  # uploaded, no store
           dict(good, win=2),                  # not uploaded
           dict(good, win=7), dict(good, win=-1),
           dict(good, feat_slot=5), dict(good, feat_slot=0),     # out of range; a slot with no keypoints
           dict(good, n_cams=3), dict(good, n_cams=0),
           dict(good, cams=None), dict(good, out=None)]
    for bd in bad:
        with pytest.raises(capi.OkbError) as e:
            ctx.keyframe_overlap_batch([bd])
        assert e.value.code == abi.OKB_ERR_INVALID_ARG, bd
        assert "jobs[0]" in str(e.value)
    with pytest.raises(capi.OkbError) as e:
        ctx.keyframe_overlap_batch([good, good])          # a window listed twice
    assert e.value.code == abi.OKB_ERR_INVALID_ARG and "jobs[1]" in str(e.value)
    assert capi.lib().okb_keyframe_overlap_batch(ctx._h, 0, None) == abi.OKB_OK        # no jobs: no-op
    assert capi.lib().okb_keyframe_overlap_batch(ctx._h, -1, None) == abi.OKB_ERR_INVALID_ARG
    assert_same(ctx.keyframe_overlap_batch([good])[0], S.session_values([img, img]))    # nothing changed
    ctx.close()
    c0, c1 = capi.Context(0, 1), capi.Context(0, 1)
    capi.Context.shard_connect_local([c0, c1])
    with pytest.raises(capi.OkbError) as e:
        c0.keyframe_overlap_batch([good])
    assert e.value.code == abi.OKB_ERR_UNSUPPORTED
    c0.close(); c1.close()
