"""okb_optimize_slots: one batched solve of a list of slots in any order.  Per slot the result must be BIT-IDENTICAL to
okb_optimize over a contiguous range that holds the same windows in the same order, and the slots that are not listed
must be left alone: not committed, not read, not written."""
import ctypes as C

import numpy as np
import pytest

from okvis_b200 import abi, synthetic

pytestmark = pytest.mark.gpu

N_SLOTS = 8
ITERS = 10


def window(i):
    """Slot i's window: cfg-1 (5 frames, 300 landmarks) on odd slots, cfg-2 (10 frames, 2 000 landmarks) on even ones."""
    return synthetic.make_window(1 if i % 2 else 2, i)


def loaded(okb, slot_windows):
    """A context of N_SLOTS slots (the chunk cap depends on the slot count) with slot_windows {slot: window index}."""
    c = okb.Context(0, N_SLOTS)
    for s, i in slot_windows.items():
        c.upload(s, window(i))
    return c


def outputs(ctx, slot, i):
    w = window(i)
    d = ctx.download(slot, dims=(len(w.poses), len(w.speed_bias), len(w.landmarks)))
    d["imu_cache"] = [ctx.debug_imu_cache(slot, t) for t in range(len(w.imu_terms))]
    return d


def assert_same_summary(a, b):
    for k in ("initial_cost", "final_cost", "iterations", "num_successful_steps", "termination", "imu_redo_count",
              "final_radius"):
        assert a[k] == b[k], (k, a[k], b[k])


def assert_same_outputs(a, b):
    for k in ("poses", "speed_bias", "landmarks", "quality"):
        assert np.array_equal(a[k], b[k]), k
    for (ra, va, na), (rb, vb, nb) in zip(a["imu_cache"], b["imu_cache"]):
        assert np.array_equal(ra, rb) and va == vb and na == nb


def range_reference(okb, order):
    """okb_optimize over slots 0..n-1 holding the windows of `order`, in that order."""
    ref = loaded(okb, {s: i for s, i in enumerate(order)})
    try:
        l0 = ref.kernel_launches
        summ = ref.optimize(0, len(order), max_iterations=ITERS)
        launches = ref.kernel_launches - l0
        outs = [outputs(ref, s, i) for s, i in enumerate(order)]
    finally:
        ref.close()
    return summ, outs, launches


@pytest.mark.parametrize("order", [[6, 1, 4], [7, 0, 3, 5, 2], [3]])
def test_scattered_set_equals_range_and_leaves_other_slots(okb, order):
    ctx = loaded(okb, {s: s for s in range(N_SLOTS)})
    try:
        others = [s for s in range(N_SLOTS) if s not in order]
        before = {s: outputs(ctx, s, s) for s in others}
        summ = ctx.optimize_slots(order, max_iterations=ITERS)
        got = [outputs(ctx, s, s) for s in order]
        after = {s: outputs(ctx, s, s) for s in others}
    finally:
        ctx.close()
    ref_summ, ref_outs, _ = range_reference(okb, order)
    assert len(summ) == len(order)
    for a, b in zip(summ, ref_summ):
        assert a["iterations"] > 0
        assert_same_summary(a, b)
    for a, b in zip(got, ref_outs):
        assert_same_outputs(a, b)
    for s in others:
        assert_same_outputs(before[s], after[s])


def test_pending_edits_of_an_unlisted_slot_stay_pending(okb):
    """Slot 3 holds a pending edit during the set call; applied afterwards it gives what it gives without the call."""
    w3 = window(3)
    moved = w3.poses[2:3].copy()
    moved[0, :3] += 0.01

    def run(with_set_call):
        ctx = loaded(okb, {s: s for s in range(N_SLOTS)})
        try:
            uploaded_bytes = ctx.h2d_bytes(3)         # what the last commit of slot 3 (its full upload) shipped
            ctx.set_states(3, pose_idx=[2], poses=moved)
            if with_set_call:
                ctx.optimize_slots([6, 1, 4], max_iterations=ITERS)
                assert ctx.h2d_bytes(3) == uploaded_bytes, "the set call committed an unlisted slot"
            s = ctx.optimize(3, 1, max_iterations=ITERS)[0]
            assert ctx.h2d_bytes(3) < uploaded_bytes        # now the one-pose edit was committed, and only it
            return s, outputs(ctx, 3, 3)
        finally:
            ctx.close()

    (sa, da), (sb, db) = run(True), run(False)
    assert_same_summary(sa, sb)
    assert_same_outputs(da, db)
    # the edit did reach the solve: the initial cost differs from the unedited window's
    ctx = loaded(okb, {3: 3})
    try:
        plain = ctx.optimize(3, 1, max_iterations=ITERS)[0]
    finally:
        ctx.close()
    assert plain["initial_cost"] != sa["initial_cost"]


def test_two_sets_in_flight_keep_their_own_tables(okb):
    """Two sets of one size (one graph) issued back to back with _async, then both finished."""
    a, b = [6, 1, 4], [0, 5, 2]
    ctx = loaded(okb, {s: s for s in range(N_SLOTS)})
    try:
        ctx.optimize_slots_async(a, max_iterations=ITERS)
        ctx.optimize_slots_async(b, max_iterations=ITERS)
        sa = ctx.optimize_slots_finish(a)
        sb = ctx.optimize_slots_finish(b)
        oa = [outputs(ctx, s, s) for s in a]
        ob = [outputs(ctx, s, s) for s in b]
    finally:
        ctx.close()
    for order, summ, outs in ((a, sa, oa), (b, sb, ob)):
        ref_summ, ref_outs, _ = range_reference(okb, order)
        for x, y in zip(summ, ref_summ):
            assert_same_summary(x, y)
        for x, y in zip(outs, ref_outs):
            assert_same_outputs(x, y)


def test_launch_count_equals_range_call(okb):
    order = [6, 1, 4]
    ctx = loaded(okb, {s: s for s in range(N_SLOTS)})
    try:
        l0 = ctx.kernel_launches
        ctx.optimize_slots(order, max_iterations=ITERS)
        n_set = ctx.kernel_launches - l0
    finally:
        ctx.close()
    _, _, n_range = range_reference(okb, order)
    assert n_set == n_range > 0


def test_errors_change_nothing(okb):
    ctx = loaded(okb, {s: s for s in range(N_SLOTS - 1)})      # slot 7 never uploaded
    lib = okb.lib()
    o = okb.Context._options(ITERS, 0, -1.0, 1)
    try:
        before = {s: outputs(ctx, s, s) for s in range(N_SLOTS - 1)}
        l0 = ctx.kernel_launches

        def call(slots, n=None, opt=o):
            arr = (C.c_int32 * max(1, len(slots)))(*slots) if slots is not None else None
            return lib.okb_optimize_slots(ctx._h, len(slots) if n is None else n, arr,
                                          C.byref(opt) if opt is not None else None, None)

        assert call([1, 2], n=0) == abi.OKB_ERR_INVALID_ARG
        assert call([1, 2], n=-1) == abi.OKB_ERR_INVALID_ARG
        assert call(None, n=2) == abi.OKB_ERR_INVALID_ARG
        assert call([1, 2], opt=None) == abi.OKB_ERR_INVALID_ARG
        assert call([1, N_SLOTS]) == abi.OKB_ERR_INVALID_ARG
        assert call([-1, 2]) == abi.OKB_ERR_INVALID_ARG
        assert call([1, 7]) == abi.OKB_ERR_INVALID_ARG          # not uploaded
        assert "slots[1] = 7" in lib.okb_last_error(ctx._h).decode()
        assert call([1, 2, 1]) == abi.OKB_ERR_INVALID_ARG       # listed twice
        assert "slots[2] = 1" in lib.okb_last_error(ctx._h).decode()
        arr = (C.c_int32 * 2)(1, 2)
        assert lib.okb_optimize_slots_async(ctx._h, 2, arr, None) == abi.OKB_ERR_INVALID_ARG
        assert lib.okb_optimize_slots_finish(ctx._h, 0, arr, None) == abi.OKB_ERR_INVALID_ARG
        assert ctx.kernel_launches == l0
        after = {s: outputs(ctx, s, s) for s in range(N_SLOTS - 1)}
        for s in before:
            assert_same_outputs(before[s], after[s])
        # the context still works
        assert ctx.optimize_slots([2, 1], max_iterations=2)[0]["iterations"] > 0
    finally:
        ctx.close()


def test_landmark_sharded_context_is_unsupported(okb):
    from okvis_b200 import sharding
    w = synthetic.make_window(2, 0)
    ctxs = [okb.Context(0, 1) for _ in range(2)]
    try:
        okb.Context.shard_connect_local(ctxs, max_frames=len(w.poses))
        for r, c in enumerate(ctxs):
            c.upload(0, sharding.shard_window(w, r, 2)[0])
        l0 = ctxs[0].kernel_launches
        with pytest.raises(okb.OkbError) as e:
            ctxs[0].optimize_slots([0], max_iterations=ITERS)
        assert e.value.code == abi.OKB_ERR_UNSUPPORTED
        assert ctxs[0].kernel_launches == l0
    finally:
        for c in ctxs:
            c.close()
