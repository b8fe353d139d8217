"""Device marginalisation (k_marginalize) against the extended-precision reference (tests/marg_reference.py) and the
oracle at the shapes its limits admit: stereo windows, the scratch-growth path, a 255-coordinate system with an odd
Jacobi dimension, V = 0, a job that keeps nothing, removed observations, and the host's capacity checks.  Each step is
compared with a reference built from the device's own inputs to it (downloaded estimates, IMU caches before the call)."""
import dataclasses

import numpy as np
import pytest

import marg_reference as mr
from okvis_b200 import abi, synthetic
from test_gpu_marginalization import at_estimates, compare_prior

pytestmark = pytest.mark.gpu
P, SB = abi.BLOCK_POSE, abi.BLOCK_SPEED_BIAS
REPORT = []


@pytest.fixture(scope="module")
def ctx(okb):
    c = okb.Context(0, 10)
    yield c
    c.close()
    for label, r in REPORT:         # observed error / bound per case (pytest -s shows it)
        print("marg shapes", label, r)


def stereo17():
    return synthetic.make_window(2, 0, cfg=synthetic.WindowConfig(**mr.STEREO17))


def device_step(ctx, oracle, win, w, make_job, label, iters=6, use_cauchy=1, upload=True):
    """optimize, then one marginalisation on slot `win`; the prior checked against the reference and the oracle."""
    if upload:
        ctx.reserve(win, len(w.poses), len(w.landmarks), len(w.obs), len(w.imu_samples), 160)
        ctx.upload(win, w)
    ctx.optimize(win, 1, max_iterations=iters, use_cauchy_loss=use_cauchy)
    est = ctx.download(win, dims=(len(w.poses), len(w.speed_bias), len(w.landmarks)))
    we = at_estimates(w, est)
    job = make_job(we)
    cache = {}
    for t in range(len(w.imu_terms)):
        sb_ref, valid, _ = ctx.debug_imu_cache(win, t)
        cache[t] = (sb_ref.copy(), valid)
    ref = mr.reference_marginalize(we, job, imu_cache=cache, use_cauchy=bool(use_cauchy))
    pb = oracle.OracleProblem(we)
    if not use_cauchy:
        pb.solve(0, 1, use_cauchy_loss=0)
    for t, (sb_ref, valid) in cache.items():
        pb.set_imu_cache(t, sb_ref, valid)
    o = pb.marginalize(job)
    ctx.marginalize(win, job)
    g = ctx.download_marg(win)
    assert g["status"][0] == 0
    assert g["status"][3] < 40, "a Jacobi eigen-decomposition stopped at its sweep cap"
    assert g["status"][2] == ref["rank_V"]
    mr.check_prior(g, ref, report=REPORT, label=label + " sweeps %d" % g["status"][3])
    if ref["n"]:
        compare_prior(g, o)
    return g, ref, we, job


def test_a_stereo_oldest_frame_with_and_without_cauchy(ctx, oracle):
    w = synthetic.make_window(2, 0)
    assert len(w.cameras) == 2
    job_of = lambda we: mr.frames_job(we, n_pose=1, n_sb=1, lm_before=3, n_frames=2)     # P0 SB0 P1 SB1 P2
    g, ref, _, _ = device_step(ctx, oracle, 0, w, job_of, "A")
    assert (ref["N"], ref["n_marg"], ref["n"]) == (36, 15, 21)
    g, ref, _, _ = device_step(ctx, oracle, 1, w, job_of, "A no-cauchy", use_cauchy=0)
    assert (ref["N"], ref["n_marg"], ref["n"]) == (36, 15, 21)


def test_b_all_blocks_beyond_the_first_landmark_scratch(ctx, oracle):
    w = synthetic.make_window(2, 0)
    g, ref, _, job = device_step(ctx, oracle, 2, w, lambda we: mr.frames_job(we, n_pose=1, n_sb=1, lm_before=99), "B")
    assert (ref["N"], ref["n_marg"], ref["n"]) == (150, 15, 135)
    assert len(job._keep[6]) > 256


@pytest.mark.parametrize("n_sb,kept,label", [(6, 159, "C"), (7, 150, "C'")])
def test_c_full_system_of_255(ctx, oracle, n_sb, kept, label):
    w = stereo17()
    g, ref, we, _ = device_step(ctx, oracle, 3, w, lambda we: mr.frames_job(we, n_pose=7, n_sb=n_sb, lm_before=7), label)
    assert (ref["N"], ref["n"]) == (255, kept) and ref["n_marg"] == 255 - kept
    assert (ref["n_marg"] % 2 == 1) if label == "C'" else (kept % 2 == 1)     # odd Jacobi dimension on both paths
    if label == "C":
        # row M of the 159-dimensional prior: device against the oracle away from the linearisation point
        marg = dict(block_kind=g["block_kind"], block_idx=g["block_idx"], x0=g["x0"], J=np.ascontiguousarray(g["J"]), e0=g["e0"])
        x = g["x0"].copy()
        rng = np.random.default_rng(7)
        x += 1e-4 * rng.standard_normal(len(x))
        o = 0
        for k in g["block_kind"]:       # re-normalise the perturbed quaternions
            if k == P:
                x[o + 3:o + 7] /= np.linalg.norm(x[o + 3:o + 7])
            o += 7 if k == P else 9
        rd, Jd = ctx.eval_marginalization(marg, x)
        ro, Jo = oracle.eval_marginalization(marg, x)
        # r = e0 + J (x [-] x0), J_eff = J times the 6x7 lift Jacobians: n-term and 6-term sums of rounded products
        dx, o = [], 0
        for k in g["block_kind"]:
            w7 = 7 if k == P else 9
            dx.append(np.abs(oracle.pose_minus(g["x0"][o:o + 7], x[o:o + 7])) if k == P else np.abs(x[o:o + 9] - g["x0"][o:o + 9]))
            o += w7
        dx = np.concatenate(dx)
        n = g["n"]
        assert np.all(np.abs(rd - ro) <= mr.C_ROUND * mr.EPS * n * (np.abs(g["e0"]) + np.abs(g["J"]) @ dx))
        assert np.abs(Jd - Jo).max() <= mr.C_ROUND * mr.EPS * 6 * np.abs(g["J"]).max()
        # row M inside the solver at n = 159 (padded to an even 160): optimize the window carrying this prior
        solve_against_oracle(ctx, oracle, 3, dataclasses.replace(we, marg=marg), 6)


def solve_against_oracle(ctx, oracle, win, wo, iters):
    """optimize(iters) of slot `win` against the oracle's solve of `wo` (the same graph, prior included, at the slot's
    current estimates and IMU caches): iterations, termination, costs and poses as in test_gpu_marginalization.py."""
    pb = oracle.OracleProblem(wo)
    for k in range(len(wo.imu_terms)):        # the IMU caches the marginalisation left on the device
        sb_ref, valid, _ = ctx.debug_imu_cache(win, k)
        pb.set_imu_cache(k, sb_ref, valid)
    s = ctx.optimize(win, 1, max_iterations=iters)[0]
    got = ctx.download(win, dims=(len(wo.poses), len(wo.speed_bias), len(wo.landmarks)))
    so = pb.solve(iters, 1)
    st = pb.state()
    assert s["iterations"] == so["iterations"] and s["termination"] == so["termination"]
    assert abs(s["initial_cost"] - so["initial_cost"]) <= 1e-7 * so["initial_cost"]
    assert abs(s["final_cost"] - so["final_cost"]) <= 1e-6 * so["final_cost"]
    assert np.abs(got["poses"] - st["poses"]).max() < 1e-6
    assert np.abs(got["speed_bias"] - st["speed_bias"]).max() < 1e-6


def test_e_speed_bias_chain_with_carried_blocks(ctx, oracle):
    """The removeAllButPose path 16 times on the 17-frame window: speed/bias s marginalised with its IMU term, every
    kept block carried over (block_prev), remove_speed_bias and optimize(3) between steps so that the estimates move
    away from the prior's x0.  Each step is checked against a reference built from the device's estimates, IMU cache,
    and persisted H / b0 before it; the prior grows from 21 to 111.  Then optimize(6) of the final window against the
    oracle (row M at n = 111)."""
    w = stereo17()
    K, L, win = len(w.poses), len(w.landmarks), 9
    ctx.reserve(win, K, L, len(w.obs), len(w.imu_samples), 160)
    ctx.upload(win, w)
    ctx.optimize(win, 1, max_iterations=1)      # far from converged: the optimize(3) between steps keep moving it
    cur = w
    for s in range(K - 1):
        est = ctx.download(win, dims=(K, K - s, L))
        we = at_estimates(cur, est)
        prior = ctx.download_marg(win) if s else None
        prev = (list(range(s + 1)) + [s + 1]) if s else [-1, -1]
        job = abi.make_marg_job([P] * (s + 1) + [SB, P, SB], list(range(s + 1)) + [0, s + 1, 1], prev + [-1, -1], [0] * (s + 1) + [1, 0, 0],
                                imu_terms=[0], sb_priors=[] if s else [0])
        sb_ref, valid, _ = ctx.debug_imu_cache(win, 0)
        ref = mr.reference_marginalize(we, job, prior=prior, imu_cache={0: (sb_ref.copy(), valid)})
        ctx.marginalize(win, job)
        g = ctx.download_marg(win)
        assert g["status"][0] == 0 and g["status"][3] < 40
        assert (ref["N"], ref["n"]) == (30 + 6 * s, 21 + 6 * s)
        mr.check_prior(g, ref, report=REPORT if s in (0, 1, K - 2) else None, label="E step %d sweeps %d" % (s, g["status"][3]))
        if s:       # the carried blocks keep their first linearisation points while the estimates have moved
            assert any(not np.array_equal(g["x0"][7 * i:7 * i + 7], est["poses"][i]) for i in range(s + 1))
        ctx.remove_speed_bias(win, 0)
        terms = cur.imu_terms[1:].copy()
        terms["sb0"] -= 1
        terms["sb1"] -= 1
        cur = dataclasses.replace(cur, speed_bias=np.ascontiguousarray(cur.speed_bias[1:]), imu_terms=terms, sb_priors=np.zeros(0, abi.sb_prior_dtype))
        ctx.optimize(win, 1, max_iterations=3)
    assert g["n"] == 111
    est = ctx.download(win, dims=(K, 1, L))
    g = ctx.download_marg(win)          # after the last remove_speed_bias: the kept speed/bias is now block 0
    assert g["block_idx"][-1] == 0
    marg = dict(block_kind=g["block_kind"], block_idx=g["block_idx"], x0=g["x0"], J=np.ascontiguousarray(g["J"]), e0=g["e0"])
    solve_against_oracle(ctx, oracle, win, dataclasses.replace(at_estimates(cur, est), marg=marg), 6)


def test_d_v_zero_kept_nothing_and_removed_observations(ctx, oracle):
    w = synthetic.make_window(2, 0)
    # V = 0: speed/bias 0 with no terms; the answer is exact
    g, ref, _, _ = device_step(ctx, oracle, 4, w, lambda we: abi.make_marg_job([P, SB, P], [0, 0, 1], [-1] * 3, [0, 1, 0]), "D V=0")
    assert ref["V_zero"] and g["status"][1] == 0 and g["status"][2] == 0 and np.all(g["H"] == 0) and np.all(g["J"] == 0)
    # every block marginalised: no prior is left, and the window solves like the oracle without one
    g, ref, we, _ = device_step(ctx, oracle, 5, w, lambda we: abi.make_marg_job([SB], [0], [-1], [1], sb_priors=[0]), "D kept 0")
    assert g["n"] == 0 and ref["n"] == 0
    s = ctx.optimize(5, 1, max_iterations=4)[0]
    so = oracle.OracleProblem(we).solve(4, 1)
    assert s["iterations"] == so["iterations"] and s["termination"] == so["termination"]
    assert abs(s["final_cost"] - so["final_cost"]) <= 1e-6 * so["final_cost"]
    # landmarks with some and with all of their observations removed
    first, last = mr.track_ends(w)
    lms = mr.well_conditioned(w, np.nonzero((first == 0) & (last <= 2))[0])[:12]
    keys = []
    for k, l in enumerate(lms[:6]):
        o = w.obs[w.obs["lm_idx"] == l]
        for ob in (o[:1] if k % 2 else o):
            keys.append((int(ob["pose_idx"]), int(ob["lm_idx"]), int(ob["cam_idx"])))
    ctx.reserve(6, len(w.poses), len(w.landmarks), len(w.obs), len(w.imu_samples), 160)
    ctx.upload(6, w)
    ctx.remove_observations(6, keys)
    obs = w.obs.copy()
    for (f, l, c) in keys:
        obs["sqrt_info"][(obs["pose_idx"] == f) & (obs["lm_idx"] == l) & (obs["cam_idx"] == c)] = 0.0
    w2 = dataclasses.replace(w, obs=obs)
    gone = lms[:6:2]           # every observation removed: nothing left to linearise

    def job_of(we):            # the partly removed landmarks that stay well conditioned at the device's estimates
        keep = np.concatenate([gone, mr.well_conditioned(we, lms[1::2][:3]), lms[6:]]).astype(np.uint32)
        assert len(keep) >= 9
        return abi.make_marg_job([P, SB, P, SB, P], [0, 0, 1, 1, 2], [-1] * 5, [1, 1, 0, 0, 0], imu_terms=[0], sb_priors=[0], landmarks=keep)

    device_step(ctx, oracle, 6, w2, job_of, "D removed obs", upload=False)


def test_g_host_capacity_limits(ctx):
    """Jobs beyond the limits return OKB_ERR_CAPACITY before any launch and leave the slot as it was."""
    w = synthetic.make_window(2, 0, cfg=synthetic.WindowConfig(n_frames=18, n_cams=2, n_landmarks=600))
    for win, mm in ((7, 160), (8, 140)):
        ctx.reserve(win, 18, len(w.landmarks), len(w.obs), len(w.imu_samples), mm)
        ctx.upload(win, w)
        ctx.optimize(win, 1, max_iterations=2)
    cases = [(7, abi.make_marg_job([P, SB] * 17 + [P], list(np.repeat(np.arange(17), 2)) + [17], [-1] * 35, [1] * 34 + [0],
                                   imu_terms=list(range(16)))),                                                  # N = 261 > 256
             (7, abi.make_marg_job([P, SB] * 11, list(np.repeat(np.arange(11), 2)), [-1] * 22, [0] * 22)),        # kept 165 > 160
             (8, abi.make_marg_job([P, SB] * 10, list(np.repeat(np.arange(10), 2)), [-1] * 20, [0] * 20))]        # kept 150 > 140 reserved
    for win, job in cases:
        before = ctx.download_marg(win)
        launches = ctx.kernel_launches
        with pytest.raises(Exception) as e:
            ctx.marginalize(win, job)
        assert getattr(e.value, "code", None) == -4         # OKB_ERR_CAPACITY
        assert ctx.kernel_launches == launches
        after = ctx.download_marg(win)
        for k in ("n", "block_kind", "block_idx", "x0", "J", "e0", "H", "b0", "status"):
            assert np.array_equal(np.asarray(before[k]), np.asarray(after[k])), k
