"""GPU checks of okb_match2d2d_batch (the 2D-2D rounds of matchToKeyframes / matchToLastFrame on the device) against the
CPU restatement tests/temporal_init_reference.py: identical integers and hp_W within the stereo call's tolerance for 1, 8
and 132 sessions at 48- and 64-byte descriptors, with the current frame's speed/bias block and without; jobs with A = B
bit-identical to okb_stereo_init_batch; a mixed batch against single calls; no change to the window or a following
optimize; host-side errors."""
import ctypes as C

import numpy as np
import pytest

from okvis_b200 import abi, capi
from temporal_scene import jobs, load, make_temporal_scene, stereo_jobs, variants

pytestmark = pytest.mark.gpu

_MODELS = [abi.DIST_RADTAN, abi.DIST_EQUIDISTANT, abi.DIST_NONE, abi.DIST_RADTAN8]
_SCENES = {}


def scene(oracle, i, desc_bytes=48):
    key = (i, desc_bytes)
    if key not in _SCENES:
        _SCENES[key] = make_temporal_scene(i, _MODELS[i % 4], desc_bytes=desc_bytes, oracle=oracle)
    return _SCENES[key]


def assert_same(got, ref, dets):
    """Integers identical; hp_W within 1e-12 relative, widened by 1e-4 / |det| for rays that are not parallel (the
    stereo call's tolerance, DESIGN §6c)."""
    assert len(got) == len(ref)
    for g, (a, b, la, lb, cbi, hp), det in zip(got, ref, dets):
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
    # every job variant of a session: camera 0 and 1, with the current frame's speed/bias block and without
    for v in range(4):
        got = ctx.match2d2d_batch([dict(variants(scene(oracle, s % n_scenes, desc_bytes))[v], win=s) for s in range(n_sessions)])
        for s in range(n_sessions):
            sc = scene(oracle, s % n_scenes, desc_bytes)
            assert_same(got[s], sc["records"][v], sc["dets"][v])
    ctx.close()


def test_same_frame_jobs_equal_stereo_call(oracle):
    scs = [scene(oracle, i) for i in range(4)]
    ctx = capi.Context(0, 4)
    for s, sc in enumerate(scs):
        load(ctx, s, sc)
    st = ctx.stereo_init_batch([dict(stereo_jobs(sc)[0], win=s) for s, sc in enumerate(scs)])
    mm = ctx.match2d2d_batch([dict(stereo_jobs(sc)[1], win=s) for s, sc in enumerate(scs)])
    for s in range(4):
        assert len(st[s]) > 100 and st[s].tobytes() == mm[s].tobytes()
    ctx.close()


def test_mixed_batch_equals_single_calls(oracle):
    scs = [scene(oracle, i) for i in range(4)]
    ctx = capi.Context(0, 4)
    for s, sc in enumerate(scs):
        load(ctx, s, sc)
    js = [dict(stereo_jobs(sc)[1] if s % 2 else jobs(sc)[(s // 2) % 2], win=s) for s, sc in enumerate(scs)]
    batch = ctx.match2d2d_batch(js)
    for s in range(4):
        assert ctx.match2d2d_batch([js[s]])[0].tobytes() == batch[s].tobytes()
    ctx.close()


def test_window_unchanged_and_optimize_bit_identical(oracle):
    sc = scene(oracle, 1)
    a, b = capi.Context(0, 1), capi.Context(0, 1)
    load(a, 0, sc); load(b, 0, sc)
    before = b.download(0)
    j = dict(jobs(sc)[0], win=0)
    first = b.match2d2d_batch([j])[0]
    after = b.download(0)
    for k in before:
        if before[k] is not None:
            assert np.array_equal(before[k], after[k]), k
    # the store and the flags it read are unchanged: the same call gives the same records
    assert b.match2d2d_batch([j])[0].tobytes() == first.tobytes()
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
    good = dict(jobs(sc)[0], win=0)
    K, f = len(sc["window"].poses), sc["frames"]
    bad = [dict(good, win=1), dict(good, win=2), dict(good, win=7),
           dict(good, pose_a=99), dict(good, pose_b=-1), dict(good, sb_current=K), dict(good, sb_current=-2),
           dict(good, feat_slot_a=99), dict(good, feat_slot_b=99),
           dict(good, feat_slot_a=0),                                 # a feature slot with no keypoints
           dict(good, feat_slot_b=2),
           dict(good, pose_a=f["pose_b"]),                            # same pose, different slots
           dict(good, feat_slot_a=f["feat_slot_b"]),                  # same slot, different poses
           dict(good, pose_a=f["pose_b"], feat_slot_a=f["feat_slot_b"]),      # frame B against itself in one camera
           dict(good, cam_a=5), dict(good, cam_b=2), dict(good, num_best=9), dict(good, num_best=0), dict(good, out_cap=3)]
    for bd in bad:
        with pytest.raises(capi.OkbError) as e:
            ctx.match2d2d_batch([good, bd] if bd["win"] != 0 else [bd])
        assert e.value.code == abi.OKB_ERR_INVALID_ARG, bd
    with pytest.raises(capi.OkbError) as e:
        ctx.match2d2d_batch([good, good])              # a window listed twice
    assert e.value.code == abi.OKB_ERR_INVALID_ARG
    lib = capi.lib()
    t = abi.Match2D2DJob()
    t.win, t.pose_a, t.feat_slot_a, t.cam_a = 0, good["pose_a"], good["feat_slot_a"], 0
    t.pose_b, t.feat_slot_b, t.cam_b, t.sb_current, t.threshold, t.num_best = good["pose_b"], good["feat_slot_b"], 0, -1, 60.0, 4
    t.out, t.out_cap, t.n_out = None, 1 << 20, None
    assert lib.okb_match2d2d_batch(ctx._h, 1, C.byref(t)) == abi.OKB_ERR_INVALID_ARG      # no out / n_out
    assert lib.okb_match2d2d_batch(ctx._h, 0, None) == abi.OKB_OK                          # no jobs: no-op
    ctx.close()
    ctx = capi.Context(0, 2)
    load(ctx, 0, sc)
    load(ctx, 1, scene(oracle, 2, 64))
    with pytest.raises(capi.OkbError) as e:
        ctx.match2d2d_batch([good, dict(jobs(scene(oracle, 2, 64))[0], win=1)])      # two descriptor lengths in one call
    assert e.value.code == abi.OKB_ERR_INVALID_ARG
    assert_same(ctx.match2d2d_batch([good])[0], sc["records"][0], sc["dets"][0])     # nothing changed by the refused calls
    ctx.close()
    c0, c1 = capi.Context(0, 1), capi.Context(0, 1)
    capi.Context.shard_connect_local([c0, c1])
    with pytest.raises(capi.OkbError) as e:
        c0.match2d2d_batch([good])
    assert e.value.code == abi.OKB_ERR_UNSUPPORTED
    c0.close(); c1.close()
