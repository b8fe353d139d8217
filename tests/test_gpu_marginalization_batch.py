"""Batched device marginalisation (okb_window_marginalize_batch): every slot of a batch gets exactly the bits that
okb_window_marginalize gives on it -- prior, persisted H / b0, block list, x0, ImuError caches and status -- and the
solves that follow stay bit-equal.  The same seeded windows go into two slot ranges of one context: range A gets the
single calls, range B the batch.  Each range is optimized as a batch of the same size, so both start from the same
bits."""
import numpy as np
import pytest

from okvis_b200 import abi, synthetic
from test_gpu_marginalization import at_estimates, compare_prior, first_job, oracle_like_device

pytestmark = pytest.mark.gpu
P, SB = abi.BLOCK_POSE, abi.BLOCK_SPEED_BIAS


def solved(summaries):
    """The summaries without their wall-clock time."""
    return [{k: v for k, v in s.items() if k != "solve_time_s"} for s in summaries]


def load(ctx, base, wins, iters=5, max_marg_dim=80):
    for i, w in enumerate(wins):
        ctx.reserve(base + i, len(w.poses), len(w.landmarks), len(w.obs), len(w.imu_samples), max_marg_dim)
    ctx.upload_batch(base, wins)
    return solved(ctx.optimize(base, len(wins), max_iterations=iters))


def twins(ctx, wins, iters=5, max_marg_dim=80):
    """Uploads `wins` into range A = [0, n) and range B = [n, 2n) and optimizes each range as one batch."""
    n = len(wins)
    sa = load(ctx, 0, wins, iters, max_marg_dim)
    sb = load(ctx, n, wins, iters, max_marg_dim)
    assert sa == sb
    return n


def first_last(obs, L):
    last = np.full(L, -1)
    first = np.full(L, 99)
    np.maximum.at(last, obs["lm_idx"], obs["pose_idx"])
    np.minimum.at(first, obs["lm_idx"], obs["pose_idx"])
    return first, last


def oldest_landmarks(obs, L):
    """Landmarks first seen in frame 0 whose track ended before frame 3 (so that poses 0..2 connect them)."""
    first, last = first_last(obs, L)
    return np.nonzero((first == 0) & (last <= 2))[0].astype(np.uint32)


def sb_prior_list(w):
    return [0] if len(w.sb_priors) and int(w.sb_priors["sb_idx"][0]) == 0 else []


def oldest_job(w, lms, prev=(-1,) * 5, sb_priors=None):
    """Marginalise frame 0 (pose + speed/bias) with IMU term 0, the speed/bias prior on frame 0 and `lms`."""
    return abi.make_marg_job([P, SB, P, SB, P], [0, 0, 1, 1, 2], list(prev), [1, 1, 0, 0, 0], imu_terms=[0],
                             sb_priors=sb_prior_list(w) if sb_priors is None else sb_priors, landmarks=lms)


def sb_only_job(w):
    """The removeAllButPose case: speed/bias 0 is marginalised, pose 0 stays."""
    return abi.make_marg_job([P, SB, P, SB], [0, 0, 1, 1], [-1] * 4, [0, 1, 0, 0], imu_terms=[0], sb_priors=sb_prior_list(w))


def state(ctx, win, n_terms):
    m = ctx.download_marg(win)
    caches = [ctx.debug_imu_cache(win, t) for t in range(n_terms)]
    return m, caches


def bits(x):
    return np.ascontiguousarray(x).tobytes()


def assert_same_state(a, b):
    (ma, ca), (mb, cb) = a, b
    assert ma["n"] == mb["n"]
    for k in ("block_kind", "block_idx", "x0", "J", "e0", "H", "b0", "status"):
        assert bits(ma[k]) == bits(mb[k]), k
    assert len(ca) == len(cb)
    for (ra, va, na), (rb, vb, nb) in zip(ca, cb):
        assert bits(ra) == bits(rb) and va == vb and na == nb


def assert_same_estimates(ctx, a, b, dims):
    ea, eb = ctx.download(a, dims=dims), ctx.download(b, dims=dims)
    for k in ("poses", "speed_bias", "landmarks", "quality"):
        assert bits(ea[k]) == bits(eb[k]), k
    return ea


def mixed_windows():
    return [synthetic.make_window(1, 0), synthetic.make_window(2, 0), synthetic.make_window(1, 1), synthetic.make_window(2, 1),
            synthetic.make_window(1, 2), synthetic.make_window(2, 2), synthetic.make_window(1, 3), synthetic.make_window(2, 3)]


# kind of job per slot of the mixed batch
KINDS = ["oldest", "oldest", "sb_only", "oldest", "no_lm", "sb_only", None, "no_lm"]


def mixed_jobs(wins):
    jobs, cands = [], []
    for w, kind in zip(wins, KINDS):
        lms = oldest_landmarks(w.obs, len(w.landmarks))
        cands.append(lms)
        if kind == "oldest":
            jobs.append(oldest_job(w, lms))
        elif kind == "no_lm":
            jobs.append(oldest_job(w, []))
        elif kind == "sb_only":
            jobs.append(sb_only_job(w))
        else:
            jobs.append(None)
    return jobs, cands


def run_twins(ctx, n, jobs):
    """Single calls on range A, one batch on range B."""
    for i, j in enumerate(jobs):
        if j is not None:
            ctx.marginalize(i, j)
    ctx.marginalize_batch(n, jobs)


def test_batch_matches_single_calls_bit_for_bit_then_chains(okb):
    ctx = okb.Context(0, 16)
    try:
        wins = mixed_windows()
        n = twins(ctx, wins)
        jobs, cands = mixed_jobs(wins)
        assert all(len(cands[i]) > 0 for i, k in enumerate(KINDS) if k == "oldest")
        null = KINDS.index(None)
        before_null = state(ctx, n + null, len(wins[null].imu_terms))
        run_twins(ctx, n, jobs)
        for i, w in enumerate(wins):
            assert_same_state(state(ctx, i, len(w.imu_terms)), state(ctx, n + i, len(w.imu_terms)))
            if KINDS[i] is not None:
                assert ctx.download_marg(n + i)["status"][0] == 0
        assert_same_state(before_null, state(ctx, n + null, len(wins[null].imu_terms)))

        # ---- bookkeeping half on both ranges, commit, optimize: bit-equal
        dims, obs_now = [], []
        for i, (w, kind) in enumerate(zip(wins, KINDS)):
            K, L = len(w.poses), len(w.landmarks)
            if kind in ("oldest", "no_lm"):
                est = ctx.download(i)
                pp = np.zeros(1, abi.pose_prior_dtype)
                pp["pose_idx"], pp["meas"] = 0, est["poses"][1]
                pp["sqrt_info"] = np.diag([1e7, 1e7, 1e7, 0, 0, 1e7]).reshape(-1)
                gone = cands[i]      # linearised, or (no_lm) dropped without linearising: the landmarks frame 0 ends
                for base in (0, n):
                    if len(gone):
                        ctx.remove_landmarks(base + i, gone)
                    ctx.remove_frame(base + i, 0, 0)
                    ctx.set_priors(base + i, pp, np.zeros(0, abi.sb_prior_dtype))
                keep = (w.obs["pose_idx"] != 0) & ~np.isin(w.obs["lm_idx"], gone)
                o = w.obs[keep].copy()
                o["pose_idx"] -= 1
                obs_now.append(o)
                dims.append((K - 1, K - 1, L))
            elif kind == "sb_only":
                for base in (0, n):
                    ctx.remove_speed_bias(base + i, 0)
                obs_now.append(w.obs)
                dims.append((K, K - 1, L))
            else:
                obs_now.append(w.obs)
                dims.append((K, K, L))
        ctx.commit(0, n)
        ctx.commit(n, n)
        assert solved(ctx.optimize(0, n, max_iterations=4)) == solved(ctx.optimize(n, n, max_iterations=4))
        for i in range(n):
            assert_same_estimates(ctx, i, n + i, dims[i])
            assert_same_state(state(ctx, i, 0), state(ctx, n + i, 0))

        # ---- second batch: every job carries the current prior over (block_prev >= 0)
        jobs2 = []
        for i, (w, kind) in enumerate(zip(wins, KINDS)):
            if kind == "oldest":
                jobs2.append(oldest_job(w, oldest_landmarks(obs_now[i], len(w.landmarks)), prev=(0, 1, 2, -1, -1), sb_priors=[]))
            elif kind == "no_lm":
                jobs2.append(oldest_job(w, [], prev=(0, 1, 2, -1, -1), sb_priors=[]))
            elif kind == "sb_only":      # prior blocks (pose 0, pose 1, sb 0): marginalise pose 0
                jobs2.append(abi.make_marg_job([P, P, SB], [0, 1, 0], [0, 1, 2], [1, 0, 0]))
            else:
                jobs2.append(None)
        assert any(j is not None and j.n_landmarks > 0 for j in jobs2)
        run_twins(ctx, n, jobs2)
        for i in range(n):
            a, b = ctx.download_marg(i), ctx.download_marg(n + i)
            assert_same_state((a, []), (b, []))
            if KINDS[i] is not None:
                assert b["status"][0] == 0 and b["n"] > 0
        assert solved(ctx.optimize(0, n, max_iterations=4)) == solved(ctx.optimize(n, n, max_iterations=4))
        for i in range(n):
            assert_same_estimates(ctx, i, n + i, dims[i])
    finally:
        ctx.close()


def test_batch_slot_matches_the_oracle(okb, oracle):
    ctx = okb.Context(0, 3)
    try:
        wins = [synthetic.make_window(1, 0), synthetic.make_window(2, 4), synthetic.make_window(1, 5)]
        load(ctx, 0, wins, iters=6)
        est = ctx.download(0)
        job, lms, _ = first_job(oracle, at_estimates(wins[0], est))
        assert len(lms) > 5
        ref = oracle_like_device(oracle, ctx, 0, wins[0], est)
        others = [oldest_job(w, oldest_landmarks(w.obs, len(w.landmarks))) for w in wins[1:]]
        ctx.marginalize_batch(0, [job] + others)
        compare_prior(ctx.download_marg(0), ref.marginalize(job))
    finally:
        ctx.close()


def test_device_error_stays_with_its_slot(okb):
    ctx = okb.Context(0, 8)
    try:
        wins = [synthetic.make_window(1, 6), synthetic.make_window(2, 5), synthetic.make_window(1, 7), synthetic.make_window(1, 8)]
        n = twins(ctx, wins, iters=3)
        jobs = [oldest_job(w, oldest_landmarks(w.obs, len(w.landmarks))) for w in wins[:3]]
        jobs.append(abi.make_marg_job([P, SB, P], [0, 0, 1], [-1] * 3, [1, 1, 0], imu_terms=[0]))     # sb 1 of the IMU term is missing
        run_twins(ctx, n, jobs)
        for i, w in enumerate(wins):
            assert_same_state(state(ctx, i, len(w.imu_terms)), state(ctx, n + i, len(w.imu_terms)))
        assert ctx.download_marg(n + 3)["status"][0] != 0
        assert all(ctx.download_marg(n + i)["status"][0] == 0 for i in range(3))
        assert solved(ctx.optimize(0, 3, max_iterations=3)) == solved(ctx.optimize(n, 3, max_iterations=3))
        for i in range(3):
            assert_same_estimates(ctx, i, n + i, (len(wins[i].poses), len(wins[i].speed_bias), len(wins[i].landmarks)))
        with pytest.raises(okb.OkbError):
            ctx.optimize(n + 3, 1, max_iterations=2)
    finally:
        ctx.close()


def test_host_rejection_leaves_every_slot_unchanged(okb):
    ctx = okb.Context(0, 4)
    try:
        wins = [synthetic.make_window(1, 9), synthetic.make_window(1, 10), synthetic.make_window(2, 6), synthetic.make_window(1, 11)]
        load(ctx, 0, wins, iters=3)
        before = [state(ctx, i, len(w.imu_terms)) for i, w in enumerate(wins)]
        jobs = [oldest_job(w, oldest_landmarks(w.obs, len(w.landmarks))) for w in wins]
        jobs[2] = oldest_job(wins[2], [len(wins[2].landmarks) + 5])
        launches = ctx.kernel_launches
        with pytest.raises(okb.OkbError) as e:
            ctx.marginalize_batch(0, jobs)
        assert e.value.code == abi.OKB_ERR_INVALID_ARG and "slot 2" in str(e.value)
        assert ctx.kernel_launches == launches
        for i, w in enumerate(wins):
            assert_same_state(before[i], state(ctx, i, len(w.imu_terms)))
        # range checks and an all-NULL range
        for first, js in ((0, []), (-1, jobs[:1]), (2, jobs[:3])):
            with pytest.raises(okb.OkbError) as e:
                ctx.marginalize_batch(first, js)
            assert e.value.code == abi.OKB_ERR_INVALID_ARG
        launches = ctx.kernel_launches
        ctx.marginalize_batch(0, [None] * 4)
        assert ctx.kernel_launches == launches
        for i, w in enumerate(wins):
            assert_same_state(before[i], state(ctx, i, len(w.imu_terms)))
    finally:
        ctx.close()


def test_batch_overlaps_a_solve_of_other_slots_and_waits_for_its_own(okb):
    ctx = okb.Context(0, 16)
    try:
        wins = [synthetic.make_window(2, 10 + i) for i in range(4)]
        # A0 = [0, 4), A1 = [4, 8) sequential; B0 = [8, 12), B1 = [12, 16) overlapped; all four hold the same windows
        for base in (0, 4, 8, 12):
            load(ctx, base, wins, iters=3)
        jobs = [oldest_job(w, oldest_landmarks(w.obs, len(w.landmarks))) for w in wins]
        ctx.marginalize_batch(0, jobs)
        s_seq = solved(ctx.optimize(4, 4, max_iterations=6))
        ctx.optimize_async(12, 4, max_iterations=6)
        ctx.marginalize_batch(8, jobs)
        s_ovl = solved(ctx.optimize_finish(12, 4))
        assert s_seq == s_ovl
        for i, w in enumerate(wins):
            assert_same_state(state(ctx, i, len(w.imu_terms)), state(ctx, 8 + i, len(w.imu_terms)))
            assert_same_estimates(ctx, 4 + i, 12 + i, (len(w.poses), len(w.speed_bias), len(w.landmarks)))
        # a batch on slots whose own solve is still in flight runs after it
        for base in (4, 12):
            load(ctx, base, wins, iters=3)
        s_seq = solved(ctx.optimize(4, 4, max_iterations=6))
        ctx.marginalize_batch(4, jobs)
        ctx.optimize_async(12, 4, max_iterations=6)
        ctx.marginalize_batch(12, jobs)
        assert solved(ctx.optimize_finish(12, 4)) == s_seq
        for i, w in enumerate(wins):
            assert_same_state(state(ctx, 4 + i, len(w.imu_terms)), state(ctx, 12 + i, len(w.imu_terms)))
    finally:
        ctx.close()


def test_scratch_growth_and_launch_count(okb):
    ctx = okb.Context(0, 16)
    try:
        wins = [synthetic.make_window(2, 20 + i) for i in range(8)]
        n = twins(ctx, wins, iters=3, max_marg_dim=160)
        # first use: scratch for up to 256 landmarks per slot
        run_twins(ctx, n, [oldest_job(w, []) for w in wins])
        # a full upload clears the prior and keeps the scratch; the next jobs need more landmark records than it holds
        load(ctx, 0, wins, iters=3, max_marg_dim=160)
        load(ctx, n, wins, iters=3, max_marg_dim=160)
        big = []
        for w in wins:
            K = len(w.poses)
            lms = np.unique(w.obs["lm_idx"]).astype(np.uint32)       # every observed landmark: all frames are in the job
            assert len(lms) > 256
            big.append(abi.make_marg_job([P, SB] * K, np.repeat(np.arange(K), 2), [-1] * (2 * K), [1, 1] + [0] * (2 * K - 2),
                                         imu_terms=[0], sb_priors=sb_prior_list(w), landmarks=lms))
        run_twins(ctx, n, big)
        for i, w in enumerate(wins):
            assert_same_state(state(ctx, i, len(w.imu_terms)), state(ctx, n + i, len(w.imu_terms)))
            assert ctx.download_marg(n + i)["status"][0] == 0
        # launches: a batch of 1 costs what a batch of 8 costs when the job slots have no pending edits
        load(ctx, 0, wins, iters=3, max_marg_dim=160)
        load(ctx, n, wins, iters=3, max_marg_dim=160)
        jobs = [oldest_job(w, oldest_landmarks(w.obs, len(w.landmarks))) for w in wins]
        l0 = ctx.kernel_launches
        ctx.marginalize_batch(0, [jobs[0]] + [None] * 7)
        l1 = ctx.kernel_launches
        ctx.marginalize_batch(n, jobs)
        l2 = ctx.kernel_launches
        ctx.marginalize(1, jobs[1])
        l3 = ctx.kernel_launches
        assert l1 - l0 == l2 - l1 == l3 - l2 == 1
        assert_same_state(state(ctx, 0, len(wins[0].imu_terms)), state(ctx, n, len(wins[0].imu_terms)))
        assert_same_state(state(ctx, 1, len(wins[1].imu_terms)), state(ctx, n + 1, len(wins[1].imu_terms)))
    finally:
        ctx.close()
