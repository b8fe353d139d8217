"""The IMU term on the device against its extended-precision reference (tests/imu_reference.py), in all three
instantiations of okb_imu.cuh, at the cases of tests/imu_cases.py:

  * the hook okb_eval_imu (WarpCtx, preintegration variant), on the redo path and on the correction path;
  * okb_imu_propagate / okb_imu_propagate_batch (WarpCtx, propagation variant), every job bit-identical to its single
    call;
  * k_imu (GroupCtx<16>, two terms per warp) through okb_debug_imu_terms after optimize(max_iterations=0), which runs
    one solver round: k_imu linearises every term at the uploaded state and nothing writes its output after that
    round.  Each frame carries its case's speed/bias, so the edges that depend on b_g reach the kernel.  Terms of very
    different lengths share a warp, batches of windows with different term counts share a grid, the first-order bias
    correction and the redo run from each case's earlier preintegration, and caches carried through remove_frame /
    remove_speed_bias are evaluated.  The batch-position and t0 cases reach k_imu only in part (see window_cases).

Every check asserts worst error / bound <= 1; the worst ratio per case group is printed at the end of the module (run
with -s to see the table)."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import imu_cases as ic
import imu_reference as ir
from okvis_b200 import abi, synthetic

pytestmark = pytest.mark.gpu

CASES = ic.cases()
IDS = ic.case_ids()
WORST = {}


def record(kind, group, ratio, name):
    key = (kind, group)
    if ratio > WORST.get(key, (-1.0, ""))[0]:
        WORST[key] = (ratio, name)


@pytest.fixture(scope="module", autouse=True)
def ratio_table():
    yield
    if WORST:
        print("\nworst error / bound per case group")
        for (kind, group), (r, name) in sorted(WORST.items()):
            print("  %-12s %-12s %.3f  (%s)" % (kind, group, r, name))


@pytest.fixture(scope="module")
def ctx(okb):
    c = okb.Context(0, 4)
    yield c
    c.close()


@pytest.fixture(scope="module")
def refs():
    memo = {}

    def get(i, path):
        if (i, path) not in memo:
            memo[(i, path)] = ir.reference_and_bounds(CASES[i], path)
        return memo[(i, path)]
    return get


def check(kind, case, got, ref_bounds, keys=None):
    ref, bounds = ref_bounds
    if keys is not None:
        ref = {k: ref[k] for k in keys}
    ratio, where = ir.compare(got, ref, bounds)
    record(kind, case["group"], ratio, case["name"])
    assert ratio <= 1.0, (kind, case["name"], where, ratio)


# ------------------------------------------------------------------------------------------------ hook and propagation
@pytest.mark.parametrize("i", range(len(CASES)), ids=IDS)
def test_hook_matches_reference(ctx, refs, i):
    c = CASES[i]
    for path in ("eval", "corr"):
        r, J, S, redo = ctx.eval_imu(c["prm"], c["samples"], c["t0"], c["t1"], c["pose0"], c["sb0"], c["pose1"], c["sb1"],
                                     sb_ref=c["sb_ref"] if path == "corr" else None)
        check("hook/" + path, c, ir.eval_quantities(redo, r, np.hstack(J), S), refs(i, path))


def test_propagation_matches_reference(ctx, refs):
    jobs = [(c["prm"], c["samples"], c["t0"], c["t1"], c["pose0"], c["sb0"]) for c in CASES]
    single = [ctx.imu_propagate(*j) for j in jobs]
    batch = ctx.imu_propagate_batch(jobs)
    for i, (c, a, b) in enumerate(zip(CASES, single, batch)):
        assert a[0] == b[0] and all(x.tobytes() == y.tobytes() for x, y in zip(a[1:], b[1:])), c["name"]
        check("propagate", c, ir.prop_quantities(*a), refs(i, "prop"))


# ------------------------------------------------------------------------------------------------ k_imu
def by_length(idx):
    """Ordered so that neighbours in a warp differ most in length: shortest, longest, second shortest, ..."""
    idx = sorted(idx, key=lambda i: len(CASES[i]["samples"]))
    out = []
    while idx:
        out.append(idx.pop(0))
        if idx:
            out.append(idx.pop())
    return out


def default_param_cases():
    """The cases a window can hold (one ImuParams per window)."""
    return by_length([i for i, c in enumerate(CASES) if c["prm"] is ic.PRM_A])


def window_cases():
    """31 terms for one window: every default-parameter case outside the batch_end / t0 / long groups (the rotation,
    saturation, bias, zero-length, epoch, t1 and past-t1 edges), filled with the shortest and the longest of those
    three groups, in warp order (2 samples beside 2 000)."""
    edges = [i for i, c in enumerate(CASES) if c["prm"] is ic.PRM_A and c["group"] not in ("batch_end", "t0", "long")]
    rest = by_length([i for i, c in enumerate(CASES) if c["group"] in ("batch_end", "t0", "long")])
    return by_length(edges + rest[:31 - len(edges)])


def imu_window(case_idx, seed=0, state="sb0"):
    """A 32-frame window whose IMU terms are the listed cases: term t links frames t and t + 1 (pose and speed/bias), and
    frame t's speed/bias is the case's `state` (sb0 or sb_ref), so that the edges that depend on b_g (omega - b_g = 0,
    the series thresholds, the bias offsets) reach the kernel as they are in the case."""
    w = synthetic.make_window(cfg=synthetic.WindowConfig(n_frames=32, n_cams=1, n_landmarks=64), seed=0x1A1 + seed)
    terms = np.zeros(len(case_idx), abi.imu_term_dtype)
    sb = w.speed_bias.copy()
    samples, off = [], 0
    for t, i in enumerate(case_idx):
        c = CASES[i]
        terms[t] = (t, t, t + 1, t + 1, c["t0"], c["t1"], off, len(c["samples"]))
        sb[t] = c[state]
        samples.append(c["samples"])
        off += len(c["samples"])
    return dataclasses.replace(w, imu_terms=terms, imu_samples=np.ascontiguousarray(np.concatenate(samples)),
                               speed_bias=np.ascontiguousarray(sb))


def term_case(w, t, case_idx, sb_ref=None):
    """The case of term t of window w, at the window's states (and an earlier preintegration at sb_ref)."""
    T = w.imu_terms[t]
    return dict(CASES[case_idx[t]], pose0=w.poses[T["pose0"]].copy(), sb0=w.speed_bias[T["sb0"]].copy(),
                pose1=w.poses[T["pose1"]].copy(), sb1=w.speed_bias[T["sb1"]].copy(), sb_ref=sb_ref)


def check_k_imu(ctx, win, w, case_idx, kind, sb_refs=None):
    """okb_debug_imu_terms of the window's last round against the reference of each term; returns the raw outputs."""
    n = len(w.imu_terms)
    H, g, cost = ctx.debug_imu_terms(win, 0, n)
    for t in range(n):
        c = term_case(w, t, case_idx, None if sb_refs is None else sb_refs[t])
        rb = ir.reference_and_bounds(c, "eval" if sb_refs is None else "corr")
        check(kind, c, dict(H30=H[t], g30=g[t], cost=cost[t:t + 1]), rb, keys=("H30", "g30", "cost"))
    return H, g, cost


def test_k_imu_odd_term_count_mixed_lengths(ctx):
    order = window_cases()
    lens = [len(CASES[i]["samples"]) for i in order]
    names = {CASES[i]["name"] for i in order}
    assert len(order) == 31 and lens[0] == 2 and lens[1] == 2000 and lens.count(2000) == 3
    assert {"zero_rate", "jr_1e-4", "sinc_1e-6", "near_g_max", "gyro_ulp", "both_ulp", "interp_ends", "dup7",
            "bg_1.1", "second_boundary"} <= names
    w = imu_window(order)
    ctx.upload(0, w)
    ctx.optimize(0, 1, max_iterations=0)
    check_k_imu(ctx, 0, w, order, "k_imu")
    for t in range(len(order)):
        sb_ref, valid, redo = ctx.debug_imu_cache(0, t)
        assert valid == 1 and redo == 1 and np.array_equal(sb_ref, w.speed_bias[t]), t


def test_k_imu_batch_of_windows(ctx):
    """Four windows with 1, 2, 7 and 31 terms in one launch: the grid follows the largest, the others exit early."""
    pool = default_param_cases()
    rng = np.random.default_rng(5)
    counts = (1, 2, 7, 31)
    orders = [[int(x) for x in rng.choice(pool, n, replace=False)] for n in counts]
    orders[3] = window_cases()
    ws = [imu_window(o, seed=k) for k, o in enumerate(orders)]
    ctx.upload_batch(0, ws)
    ctx.optimize(0, 4, max_iterations=0)
    for k, (w, o) in enumerate(zip(ws, orders)):
        check_k_imu(ctx, k, w, o, "k_imu_batch")


def dt_of(c):
    return (c["t1"] - c["t0"]) * 1e-9


def set_speed_bias(ctx, win, w, sb):
    ctx.set_states(win, sb_idx=np.arange(len(sb)), speed_bias=sb)
    return dataclasses.replace(w, speed_bias=sb)


def preintegrated_then_moved(ctx, win, seed):
    """A window preintegrated at each case's sb_ref (first optimize), then moved to each case's sb0: b_g by
    0.9e-4 / Delta_t (1.1e-4 for bias/bg_1.1), b_a by N(0, 0.02) (0.4 for bias/ba_only), and linearised again.  Checks the
    second round against the reference of each term from its cache and returns (order, window, cache biases)."""
    order = window_cases()
    w = imu_window(order, seed=seed, state="sb_ref")
    ctx.reserve(win, 32, len(w.landmarks), len(w.obs), len(w.imu_samples))
    ctx.upload(win, w)
    ctx.optimize(win, 1, max_iterations=0)
    first = w.speed_bias.copy()
    sb = first.copy()
    for t, i in enumerate(order):
        sb[t] = CASES[i]["sb0"]
    w1 = set_speed_bias(ctx, win, w, sb)
    ctx.commit(win, 1)
    ctx.optimize(win, 1, max_iterations=0)
    out = check_k_imu(ctx, win, w1, order, "k_imu_corr", sb_refs=first)
    redo = [ir.run_eval(term_case(w1, t, order, first[t]), np.float64, True)["redo"] for t in range(len(order))]
    assert sum(redo) == 1 and redo[[CASES[i]["name"] for i in order].index("bg_1.1")] == 1
    bias = []
    for t in range(len(order)):
        sb_ref, valid, count = ctx.debug_imu_cache(win, t)
        assert valid == 1 and count == 1 + redo[t] and np.array_equal(sb_ref, sb[t] if redo[t] else first[t]), t
        bias.append(sb_ref)
    return order, w1, np.array(bias), out


def test_k_imu_first_order_correction_then_redo(ctx):
    order, w1, bias, _ = preintegrated_then_moved(ctx, 0, seed=7)
    before = [ctx.debug_imu_cache(0, t)[2] for t in range(len(order))]
    # past the threshold, from each cache's bias: every term redoes at the new bias
    rng = np.random.default_rng(8)
    sb2 = w1.speed_bias.copy()
    for t, i in enumerate(order):
        u = rng.normal(0, 1, 3)
        sb2[t, 3:6] = bias[t, 3:6] + 1.1e-4 / dt_of(CASES[i]) * u / np.linalg.norm(u)
    w2 = set_speed_bias(ctx, 0, w1, sb2)
    ctx.optimize(0, 1, max_iterations=0)
    check_k_imu(ctx, 0, w2, order, "k_imu_redo", sb_refs=bias)
    for t in range(len(order)):
        sb_ref, valid, redo = ctx.debug_imu_cache(0, t)
        assert valid == 1 and redo == before[t] + 1 and np.array_equal(sb_ref, sb2[t]), t


def test_k_imu_cache_through_graph_edits(ctx):
    """remove_frame (the oldest, then one in the middle) and remove_speed_bias move every surviving term's cache with it;
    the next round evaluates each term from its carried cache, as the reference does, and bit for bit as before."""
    order, w1, bias, (H0, g0, c0) = preintegrated_then_moved(ctx, 0, seed=9)
    caches = [ctx.debug_imu_cache(0, t) for t in range(len(order))]
    ctx.set_priors(0, np.zeros(0, abi.pose_prior_dtype), np.zeros(0, abi.sb_prior_dtype))
    # alive[k] = original term at current position k; frames / sbs: original index at current position
    alive, frames, sbs = list(range(len(order))), list(range(32)), list(range(32))
    for op, arg in (("frame", 0), ("frame", 10), ("sb", 20)):
        if op == "frame":
            f = frames[arg]
            ctx.remove_frame(0, arg, arg)
            frames.pop(arg); sbs.pop(arg)
            alive = [t for t in alive if t != f and t + 1 != f]
        else:
            s = sbs[arg]
            ctx.remove_speed_bias(0, arg)
            sbs.pop(arg)
            alive = [t for t in alive if t != s and t + 1 != s]
        for k, t in enumerate(alive):
            got = ctx.debug_imu_cache(0, k)
            assert np.array_equal(got[0], caches[t][0]) and got[1:] == caches[t][1:], (op, arg, k, t)
        with pytest.raises(Exception):
            ctx.debug_imu_cache(0, len(alive))
    assert len(alive) == 31 - 1 - 2 - 2
    ctx.optimize(0, 1, max_iterations=0)
    H, g, cost = ctx.debug_imu_terms(0, 0, len(alive))
    for k, t in enumerate(alive):
        assert H[k].tobytes() == H0[t].tobytes() and g[k].tobytes() == g0[t].tobytes() and cost[k] == c0[t], (k, t)
        c = term_case(w1, t, order, bias[t])
        check("k_imu_edit", c, dict(H30=H[k], g30=g[k], cost=cost[k:k + 1]), ir.reference_and_bounds(c, "corr"),
              keys=("H30", "g30", "cost"))
    for k, t in enumerate(alive):
        assert ctx.debug_imu_cache(0, k)[1:] == caches[t][1:], (k, t)


# ------------------------------------------------------------------------------------------------ diagnostics, checks
def test_debug_imu_terms_arguments(ctx, okb):
    order = default_param_cases()[:3]
    w = imu_window(order, seed=11)
    ctx.upload(1, w)
    ctx.optimize(1, 1, max_iterations=0)
    H, g, cost = ctx.debug_imu_terms(1, 1, 2)
    H3, g3, c3 = ctx.debug_imu_terms(1, 0, 3)
    assert H.tobytes() == H3[1:].tobytes() and g.tobytes() == g3[1:].tobytes() and cost.tobytes() == c3[1:].tobytes()
    assert np.allclose(H3, H3.transpose(0, 2, 1), rtol=0, atol=1e-12 * np.abs(H3).max()) and (c3 > 0).all()
    before = ctx.kernel_launches
    L = okb.lib()
    buf = np.full((4, abi.IMU_TERM_OUT), 7.0)
    for first, n in ((-1, 1), (0, 4), (3, 1), (2, 2), (0, -1)):
        assert L.okb_debug_imu_terms(ctx._h, 1, first, n, C.c_void_p(buf.ctypes.data)) == abi.OKB_ERR_INVALID_ARG, (first, n)
    assert L.okb_debug_imu_terms(ctx._h, 1, 0, 1, None) == abi.OKB_ERR_INVALID_ARG
    assert L.okb_debug_imu_terms(ctx._h, 4, 0, 1, C.c_void_p(buf.ctypes.data)) == abi.OKB_ERR_INVALID_ARG    # no such slot
    assert np.all(buf == 7.0)
    assert ctx.debug_imu_terms(1, 3, 0)[2].size == 0
    assert ctx.kernel_launches == before


def _bad_window(kind):
    w = synthetic.make_window(1, 0)
    t = w.imu_terms.copy()
    if kind == "ends before t1":
        t["sample_count"][1] -= 2
    elif kind == "starts after t0":
        t["sample_offset"][1] += 2
        t["sample_count"][1] -= 2
    else:
        t["t1_ns"][1] = t["t0_ns"][1]
    return w, dataclasses.replace(w, imu_terms=t)


@pytest.mark.parametrize("kind", ["ends before t1", "starts after t0", "t1 not after t0"])
def test_upload_rejects_term_not_covering_its_interval(ctx, okb, kind):
    good, bad = _bad_window(kind)
    ctx.upload(2, good)
    ctx.optimize(2, 1, max_iterations=0)
    ref = ctx.download(2)
    with pytest.raises(okb.OkbError) as e:
        ctx.upload(2, bad)
    assert e.value.code == abi.OKB_ERR_INVALID_ARG and "IMU term 1" in str(e.value)
    got = ctx.download(2)
    assert all(np.array_equal(got[k], ref[k]) for k in ("poses", "speed_bias", "landmarks"))
    assert [ctx.debug_imu_cache(2, t)[1:] for t in range(len(good.imu_terms))] == [(1, 1)] * len(good.imu_terms)


@pytest.mark.parametrize("kind", ["ends before t1", "starts after t0", "t1 not after t0"])
def test_add_frame_rejects_term_not_covering_its_interval(ctx, okb, kind):
    w = synthetic.make_window(1, 0)
    K = len(w.poses)
    base = dataclasses.replace(w, poses=w.poses[:K - 1].copy(), speed_bias=w.speed_bias[:K - 1].copy(),
                               obs=w.obs[w.obs["pose_idx"] < K - 1].copy(), imu_terms=w.imu_terms[:K - 2].copy())
    ctx.reserve(3, K, len(w.landmarks), len(w.obs), 2 * len(w.imu_samples))
    ctx.upload(3, base)
    term = w.imu_terms[K - 2:K - 1].copy()
    lo, n = int(term["sample_offset"][0]), int(term["sample_count"][0])
    smp = np.ascontiguousarray(w.imu_samples[lo:lo + n])
    term["sample_offset"] = 0
    if kind == "ends before t1":
        smp = smp[:-2].copy()
        term["sample_count"] = n - 2
    elif kind == "starts after t0":
        smp = smp[2:].copy()
        term["sample_count"] = n - 2
    else:
        term["t1_ns"] = term["t0_ns"]
    with pytest.raises(okb.OkbError) as e:
        ctx.add_frame(3, w.poses[K - 1], w.speed_bias[K - 1], term, smp)
    assert e.value.code == abi.OKB_ERR_INVALID_ARG and "IMU term %d" % (K - 2) in str(e.value)
    # the slot is unchanged: the same frame and term, covering their interval, are still accepted at the same place
    term_ok = w.imu_terms[K - 2:K - 1].copy()
    term_ok["sample_offset"] = 0
    ctx.add_frame(3, w.poses[K - 1], w.speed_bias[K - 1], term_ok, np.ascontiguousarray(w.imu_samples[lo:lo + n]))
    ctx.optimize(3, 1, max_iterations=0)
    assert ctx.debug_imu_cache(3, K - 2)[1:] == (1, 1)
    with pytest.raises(okb.OkbError):
        ctx.debug_imu_cache(3, K - 1)
