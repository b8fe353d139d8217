"""Window groups of the batched solve (okb_set_solve_groups): a batch split into G groups, each solving on its own
stream, must give every window BIT-IDENTICAL summaries, estimates and ImuError caches to the same batch in one group,
through range and slot-list calls, the captured graph and the profiled stream launches, and must launch each group's
round chain once per round."""
import numpy as np
import pytest

from okvis_b200 import abi, synthetic

pytestmark = pytest.mark.gpu

ITERS = 10


def window(i):
    """cfg-1 (5 frames, 300 landmarks) on odd indices, cfg-2 (10 frames, 2 000 landmarks) on even ones."""
    return synthetic.make_window(1 if i % 2 else 2, i)


def outputs(ctx, slot, w, imu_cache=True):
    d = ctx.download(slot, dims=(len(w.poses), len(w.speed_bias), len(w.landmarks)))
    if imu_cache:
        d["imu_cache"] = [ctx.debug_imu_cache(slot, t) for t in range(len(w.imu_terms))]
    return d


def assert_same_summary(a, b):
    for k in ("initial_cost", "final_cost", "iterations", "num_successful_steps", "termination", "imu_redo_count",
              "final_radius"):
        assert a[k] == b[k], (k, a[k], b[k])


def assert_same_outputs(a, b):
    for k in ("poses", "speed_bias", "landmarks", "quality"):
        assert np.array_equal(a[k], b[k]), k
    for (ra, va, na), (rb, vb, nb) in zip(a.get("imu_cache", []), b.get("imu_cache", [])):
        assert np.array_equal(ra, rb) and va == vb and na == nb


def solve(okb, wins, groups, call, max_iterations=ITERS, profile=False, imu_cache=True):
    """A fresh context holding `wins` in slots 0..n-1, solved once with `groups` window groups by `call(ctx)`; returns
    (summaries, per-slot outputs, kernel launches of the call, profile counters or None)."""
    ctx = okb.Context(0, len(wins))
    try:
        ctx.upload_batch(0, wins)
        ctx.set_solve_groups(groups)
        if profile:
            ctx.profile_enable(True)
        l0 = ctx.kernel_launches
        summ = call(ctx, max_iterations)
        launches = ctx.kernel_launches - l0
        prof = ctx.profile_read() if profile else None
        outs = [outputs(ctx, s, w, imu_cache) for s, w in enumerate(wins)]
    finally:
        ctx.close()
    return summ, outs, launches, prof


def range_call(ctx, it):
    return ctx.optimize(0, ctx.max_windows, max_iterations=it)


def check_same(a, b):
    (sa, oa, _, _), (sb, ob, _, _) = a, b
    assert len(sa) == len(sb)
    for x, y in zip(sa, sb):
        assert x["iterations"] > 0
        assert_same_summary(x, y)
    for x, y in zip(oa, ob):
        assert_same_outputs(x, y)


@pytest.mark.parametrize("profile", [False, True], ids=["graph", "profile"])
def test_groups_bit_identical_mixed_sizes_and_terminations(okb, profile):
    """Windows of two shapes, run to convergence so that they stop in different rounds."""
    wins = [window(i) for i in range(8)]
    ref = solve(okb, wins, 1, range_call, max_iterations=40, profile=profile)
    assert len({s["iterations"] for s in ref[0]}) > 1, "every window stopped in the same round"
    for G in (2, 3):
        got = solve(okb, wins, G, range_call, max_iterations=40, profile=profile)
        check_same(got, ref)
        if profile:       # each round counts once for the whole batch
            for k in ("landmarks_launches", "solve_launches", "quality_launches"):
                assert got[3][k] == ref[3][k] > 0, k


@pytest.mark.parametrize("profile", [False, True], ids=["graph", "profile"])
def test_groups_launch_one_chain_per_group(okb, profile):
    """Per round every group launches the whole chain (k_imu, k_landmarks, k_schur, k_reduce_partials, k_solve); the
    reset before the rounds and the quality pass after them stay one launch each."""
    wins = [window(2 * i) for i in range(6)]
    _, _, n1, _ = solve(okb, wins, 1, range_call, profile=profile, imu_cache=False)
    assert (n1 - 2) % (ITERS + 1) == 0
    for G in (2, 3):
        _, _, nG, _ = solve(okb, wins, G, range_call, profile=profile, imu_cache=False)
        assert nG - 2 == G * (n1 - 2), (G, n1, nG)


@pytest.mark.parametrize("profile", [False, True], ids=["graph", "profile"])
def test_groups_scattered_slot_list(okb, profile):
    wins = [window(i) for i in range(8)]
    order = [7, 0, 3, 5, 2, 6, 1]

    def slots_call(ctx, it):
        return ctx.optimize_slots(order, max_iterations=it)

    ref = solve(okb, wins, 1, slots_call, profile=profile)
    for G in (2, 3):
        check_same(solve(okb, wins, G, slots_call, profile=profile), ref)


def test_groups_off_the_wave_boundary(okb):
    """2 x SMs + 1 windows: one more than two waves of k_solve CTAs at this shape.  The automatic choice splits the
    batch (at least one window per SM), and neither its group boundaries nor those of three groups fall on a wave
    boundary."""
    import torch
    n = 2 * torch.cuda.get_device_properties(0).multi_processor_count + 1
    distinct = [synthetic.make_window(2, i) for i in range(8)]
    wins = [distinct[i % len(distinct)] for i in range(n)]
    ref = solve(okb, wins, 1, range_call, imu_cache=False)
    auto = solve(okb, wins, 0, range_call, imu_cache=False)
    check_same(auto, ref)
    assert auto[2] > ref[2], "the automatic choice kept a batch of more windows than SMs in one group"
    check_same(solve(okb, wins, 3, range_call, imu_cache=False), ref)


def test_automatic_choice_keeps_a_small_batch_in_one_group(okb):
    """Fewer windows than SMs: one group."""
    wins = [window(i) for i in range(8)]
    check_same(solve(okb, wins, 0, range_call), solve(okb, wins, 1, range_call))
    assert solve(okb, wins, 0, range_call, imu_cache=False)[2] == solve(okb, wins, 1, range_call, imu_cache=False)[2]


def test_more_groups_than_windows(okb):
    wins = [window(0), window(1)]
    ref = solve(okb, wins, 1, range_call)
    got = solve(okb, wins, 4, range_call)
    check_same(got, ref)
    assert got[2] - 2 == 2 * (ref[2] - 2)      # two groups of one window


def test_invalid_group_counts(okb):
    ctx = okb.Context(0, 1)
    try:
        for n in (-1, 5):
            assert okb.lib().okb_set_solve_groups(ctx._h, n) == abi.OKB_ERR_INVALID_ARG
        assert okb.lib().okb_set_solve_groups(None, 0) == abi.OKB_ERR_INVALID_ARG
        ctx.upload(0, window(1))
        ctx.set_solve_groups(4)
        assert ctx.optimize(0, 1, max_iterations=2)[0]["iterations"] > 0
    finally:
        ctx.close()
