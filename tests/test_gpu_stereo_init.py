"""GPU checks of okb_stereo_init_batch (Frontend::matchStereo's 2D-2D match on the device) against the CPU reference
tests/stereo_init_reference.py: identical records (hp_W within 1e-12 relative, see assert_same) for 1, 8 and 132 sessions at 48- and
64-byte descriptors; a batch against single calls; no change to the window or a following optimize; host-side errors."""
import ctypes as C

import numpy as np
import pytest

from okvis_b200 import abi, capi
from stereo_scene import load, make_stereo_scene

pytestmark = pytest.mark.gpu

_MODELS = [abi.DIST_RADTAN, abi.DIST_EQUIDISTANT, abi.DIST_NONE, abi.DIST_RADTAN8]
_SCENES = {}


def scene(oracle, i, desc_bytes=48):
    key = (i, desc_bytes)
    if key not in _SCENES:
        _SCENES[key] = make_stereo_scene(i, _MODELS[i % 4], desc_bytes=desc_bytes, oracle=oracle)
    return _SCENES[key]


def job(sc, win):
    return dict(sc["job"], win=win)


def assert_same(got, sc):
    """Integers identical; hp_W within 1e-12 relative.  For far points that are not parallel the bound is widened by
    1e-4 / |det|: triangulateFast solves a 2x2 system with det = 1 - cos^2 of the ray angle, so rounding differences
    (the device contracts multiply-adds) grow like eps / |det|.  Parallel rays (|det| <= 1e-6) solve nothing and keep
    1e-12."""
    ref = sc["records"]
    assert len(got) == len(ref)
    for g, (a, b, la, lb, cbi, hp), det in zip(got, ref, sc["dets"]):
        assert (int(g["kp_a"]), int(g["kp_b"]), int(g["lm_slot_a"]), int(g["lm_slot_b"]), int(g["can_be_initialized"])) == (a, b, la, lb, cbi)
        tol = 1e-12 if det <= 1e-6 else 1e-12 * max(1.0, 1e-4 / det)
        assert np.linalg.norm(g["hp_W"] - hp) <= tol * np.linalg.norm(hp), (g, hp, det)


@pytest.mark.parametrize("desc_bytes", [48, 64])
@pytest.mark.parametrize("n_sessions", [1, 8, 132])
def test_records_vs_reference(oracle, n_sessions, desc_bytes):
    n_scenes = min(n_sessions, 8)
    ctx = capi.Context(0, n_sessions)
    for s in range(n_sessions):
        load(ctx, s, scene(oracle, s % n_scenes, desc_bytes))
    got = ctx.stereo_init_batch([job(scene(oracle, s % n_scenes, desc_bytes), s) for s in range(n_sessions)])
    for s in range(n_sessions):
        assert_same(got[s], scene(oracle, s % n_scenes, desc_bytes))
    ctx.close()


def test_every_branch_is_covered(oracle):
    cases = set()
    for i in range(4):
        sc = scene(oracle, i)
        cases |= set(sc["cases"])
        assert "rank_deficient" in sc["cases"]          # the QR decides one pair of every scene
    assert {"both_named", "parallel", "close_residual", "initialised", "rank_deficient", "initialised_a_named",
            "initialised_b_named"} <= cases


def test_batch_equals_single_calls(oracle):
    scs = [scene(oracle, i) for i in range(4)]
    ctx = capi.Context(0, 4)
    for s, sc in enumerate(scs):
        load(ctx, s, sc)
    batch = ctx.stereo_init_batch([job(sc, s) for s, sc in enumerate(scs)])
    for s, sc in enumerate(scs):
        single = ctx.stereo_init_batch([job(sc, s)])[0]
        assert single.tobytes() == batch[s].tobytes()
    ctx.close()


def test_window_unchanged_and_optimize_bit_identical(oracle):
    sc = scene(oracle, 1)
    a, b = capi.Context(0, 1), capi.Context(0, 1)
    load(a, 0, sc); load(b, 0, sc)
    before = b.download(0)
    first = b.stereo_init_batch([job(sc, 0)])[0]
    after = b.download(0)
    for k in before:
        if before[k] is not None:
            assert np.array_equal(before[k], after[k]), k
    # the store and the flags it read are unchanged: the same call gives the same records
    assert b.stereo_init_batch([job(sc, 0)])[0].tobytes() == first.tobytes()
    sa, sb = a.optimize(0, 1, max_iterations=10)[0], b.optimize(0, 1, max_iterations=10)[0]
    assert sa["final_cost"] == sb["final_cost"] and sa["iterations"] == sb["iterations"]
    da, db = a.download(0), b.download(0)
    for k in da:
        if da[k] is not None:
            assert np.array_equal(da[k], db[k]), k
    a.close(); b.close()


def test_errors_before_device_work(oracle):
    sc = scene(oracle, 2)
    ctx = capi.Context(0, 3)
    load(ctx, 0, sc)
    ctx.upload(1, sc["window"])                      # uploaded, no store
    good = job(sc, 0)
    bad = [dict(good, win=1), dict(good, win=2), dict(good, win=7), dict(good, pose=99), dict(good, feat_slot=99),
           dict(good, feat_slot=0),                                  # a feature slot with no keypoints
           dict(good, cam_b=0), dict(good, cam_a=5), dict(good, num_best=9), dict(good, out_cap=3)]
    for bd in bad:
        with pytest.raises(capi.OkbError) as e:
            ctx.stereo_init_batch([good, bd] if bd["win"] != 0 else [bd])
        assert e.value.code == abi.OKB_ERR_INVALID_ARG, bd
    with pytest.raises(capi.OkbError) as e:
        ctx.stereo_init_batch([good, good])              # a window listed twice
    assert e.value.code == abi.OKB_ERR_INVALID_ARG
    lib = capi.lib()
    n = C.c_int32(-1)
    t = abi.StereoJob()
    t.win, t.pose, t.feat_slot, t.cam_a, t.cam_b, t.threshold, t.num_best = 0, good["pose"], good["feat_slot"], 0, 1, 60.0, 4
    t.out, t.out_cap, t.n_out = None, 1 << 20, None
    assert lib.okb_stereo_init_batch(ctx._h, 1, C.byref(t)) == abi.OKB_ERR_INVALID_ARG      # no out / n_out
    assert lib.okb_stereo_init_batch(ctx._h, 0, None) == abi.OKB_OK                          # no jobs: no-op
    ctx.close()
    ctx = capi.Context(0, 2)
    load(ctx, 0, sc)
    load(ctx, 1, scene(oracle, 2, 64))
    with pytest.raises(capi.OkbError) as e:
        ctx.stereo_init_batch([good, job(scene(oracle, 2, 64), 1)])      # two descriptor lengths in one call
    assert e.value.code == abi.OKB_ERR_INVALID_ARG
    assert_same(ctx.stereo_init_batch([good])[0], sc)         # nothing changed by the refused calls
    ctx.close()
    c0, c1 = capi.Context(0, 1), capi.Context(0, 1)
    capi.Context.shard_connect_local([c0, c1])
    with pytest.raises(capi.OkbError) as e:
        c0.stereo_init_batch([good])
    assert e.value.code == abi.OKB_ERR_UNSUPPORTED
    c0.close(); c1.close()
