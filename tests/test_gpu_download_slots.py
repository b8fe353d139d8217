"""okb_window_download_slots: the estimates of a list of slots in any order.  Per slot the bytes must equal
okb_window_download_batch over a range and okb_window_download of the same slot, and slots that are not listed must be
left alone: their pending edits stay pending."""
import ctypes as C

import numpy as np
import pytest

from okvis_b200 import abi, synthetic

pytestmark = pytest.mark.gpu

N_SLOTS = 8
ITERS = 4
KEYS = ("poses", "speed_bias", "landmarks", "quality")


def window(i):
    return synthetic.make_window(1 if i % 2 else 2, i)


def loaded(okb):
    c = okb.Context(0, N_SLOTS)
    for s in range(N_SLOTS - 1):                   # slot 7 stays empty
        c.upload(s, window(s))
    c.optimize(0, N_SLOTS - 1, max_iterations=ITERS)
    return c


@pytest.mark.parametrize("order", [[6, 1, 4], [5, 4, 3, 2, 1, 0], [2, 3, 0, 6]])
def test_list_returns_the_bytes_of_batch_and_single_downloads(okb, order):
    ctx = loaded(okb)
    try:
        got = ctx.download_slots(order)
        single = [ctx.download(s) for s in order]
        batch = ctx.download_batch(0, N_SLOTS - 1)
    finally:
        ctx.close()
    assert len(got) == len(order)
    for g, one, s in zip(got, single, order):
        for k in KEYS:
            assert g[k].tobytes() == one[k].tobytes(), (s, k)
            assert g[k].tobytes() == batch[s][k].tobytes(), (s, k)


def test_null_tables_and_entries(okb):
    ctx = loaded(okb)
    try:
        order = [4, 1]
        outs, tables = ctx.alloc_slot_outputs(order)
        tables[1][1] = None                         # slot 1's speed/bias entry
        n, arr = ctx._slot_list(order)
        rc = okb.lib().okb_window_download_slots(ctx._h, n, arr, tables[0], tables[1], None, tables[3])
        assert rc == abi.OKB_OK
        ref = [ctx.download(s) for s in order]
    finally:
        ctx.close()
    for o, r in zip(outs, ref):
        assert o["poses"].tobytes() == r["poses"].tobytes() and o["quality"].tobytes() == r["quality"].tobytes()
        assert not o["landmarks"].any()
    assert outs[0]["speed_bias"].tobytes() == ref[0]["speed_bias"].tobytes()
    assert not outs[1]["speed_bias"].any()


def test_pending_edits_of_an_unlisted_slot_stay_pending(okb):
    """Slot 3 holds a pending edit during the list download; a range download of slots 2..4 would commit it."""
    moved = window(3).poses[2:3].copy()
    moved[0, :3] += 0.01
    ctx = loaded(okb)
    try:
        ctx.download(3)
        committed = ctx.h2d_bytes(3)
        ctx.set_states(3, pose_idx=[2], poses=moved)
        ctx.download_slots([4, 2])
        assert ctx.h2d_bytes(3) == committed, "the list download committed an unlisted slot"
        ctx.download(3)
        assert 0 < ctx.h2d_bytes(3) < committed         # now the one-pose edit was committed, and only it
    finally:
        ctx.close()


def test_errors_return_before_device_work_and_name_the_entry(okb):
    ctx = loaded(okb)
    lib = okb.lib()
    try:
        outs, tables = ctx.alloc_slot_outputs([1, 2, 3])
        before = [o["poses"].copy() for o in outs]
        l0 = ctx.kernel_launches

        def call(slots, n=None):
            arr = (C.c_int32 * max(1, len(slots)))(*slots) if slots is not None else None
            return lib.okb_window_download_slots(ctx._h, len(slots) if n is None else n, arr, *tables)

        assert call([1, 2], n=0) == abi.OKB_ERR_INVALID_ARG
        assert call([1, 2], n=-1) == abi.OKB_ERR_INVALID_ARG
        assert call(None, n=2) == abi.OKB_ERR_INVALID_ARG
        assert call([1, N_SLOTS]) == abi.OKB_ERR_INVALID_ARG
        assert "slots[1] = %d" % N_SLOTS in lib.okb_last_error(ctx._h).decode()
        assert call([-1, 2]) == abi.OKB_ERR_INVALID_ARG
        assert "slots[0] = -1" in lib.okb_last_error(ctx._h).decode()
        assert call([1, 7]) == abi.OKB_ERR_INVALID_ARG          # not uploaded
        assert "slots[1] = 7" in lib.okb_last_error(ctx._h).decode()
        assert call([1, 2, 1]) == abi.OKB_ERR_INVALID_ARG       # listed twice
        assert "slots[2] = 1" in lib.okb_last_error(ctx._h).decode()
        assert ctx.kernel_launches == l0
        for o, b in zip(outs, before):
            assert np.array_equal(o["poses"], b)
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
        with pytest.raises(okb.OkbError) as e:
            ctxs[0].download_slots([0])
        assert e.value.code == abi.OKB_ERR_UNSUPPORTED
    finally:
        for c in ctxs:
            c.close()
