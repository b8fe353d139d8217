"""CPU: the extended-precision marginalisation reference (tests/marg_reference.py) against the oracle's
OracleProblem.marginalize at every shape the device test runs, and the sensitivity of the comparator the device test
uses: each fault below, planted into the oracle's inputs or outputs, must be rejected."""
import dataclasses

import numpy as np
import pytest

import marg_reference as mr
from okvis_b200 import abi, synthetic
from oracle import oracle_py as op

P, SB = abi.BLOCK_POSE, abi.BLOCK_SPEED_BIAS


def test_long_double_is_extended():
    mr.require_long_double()


def window(shape):
    if shape == "cfg2":
        return synthetic.make_window(2, 0)
    return synthetic.make_window(2, 0, cfg=synthetic.WindowConfig(**mr.STEREO17))


# (window, job builder args, N, marginalised, kept) -- cases A, B, C, C' of tests/test_gpu_marginalization_shapes.py
SHAPES = {
    "A": ("cfg2", dict(n_pose=1, n_sb=1, lm_before=3, n_frames=2), 36, 15, 21),
    "B": ("cfg2", dict(n_pose=1, n_sb=1, lm_before=99), 150, 15, 135),
    "C": ("s17", dict(n_pose=7, n_sb=6, lm_before=7), 255, 96, 159),
    "C'": ("s17", dict(n_pose=7, n_sb=7, lm_before=7), 255, 105, 150),
}


@pytest.mark.parametrize("name", list(SHAPES))
@pytest.mark.parametrize("cauchy", [1, 0])
def test_reference_matches_oracle(name, cauchy):
    wname, kw, N, nm, nk = SHAPES[name]
    w = window(wname)
    job = mr.frames_job(w, **kw)
    pb = op.OracleProblem(w)
    if not cauchy:
        pb.solve(0, 1, use_cauchy_loss=0)      # the loss of the last optimize decides the Cauchy correction
    o = pb.marginalize(job)
    ref = mr.reference_marginalize(w, job, use_cauchy=bool(cauchy))
    assert (ref["N"], ref["n_marg"], ref["n"]) == (N, nm, nk)
    if name == "B":
        assert len(job._keep[6]) > 256          # more landmarks than the device's first scratch allocation holds
    if name != "A":
        lo, hi = mr.rank_band(ref)
        assert lo == hi                         # the gauge eigenvalues lie far below the threshold, the rest far above
    mr.check_prior(o, ref, label=name)


def test_reference_matches_oracle_on_removed_observations_and_v_zero():
    """Landmarks with some and with all observations removed (sqrt_info = 0); a dense block V that is zero."""
    w = synthetic.make_window(2, 0)
    first, last = mr.track_ends(w)
    lms = mr.well_conditioned(w, np.nonzero((first == 0) & (last <= 2))[0])[:12]
    obs = w.obs.copy()
    for k, l in enumerate(lms[:6]):
        sel = np.nonzero(obs["lm_idx"] == l)[0]
        obs["sqrt_info"][sel[:1] if k % 2 else sel] = 0.0
    w2 = dataclasses.replace(w, obs=obs)
    lms = np.concatenate([lms[:6:2], mr.well_conditioned(w2, lms[1::2][:3]), lms[6:]]).astype(np.uint32)
    job = abi.make_marg_job([P, SB, P, SB, P], [0, 0, 1, 1, 2], [-1] * 5, [1, 1, 0, 0, 0], imu_terms=[0], sb_priors=[0], landmarks=lms)
    mr.check_prior(op.OracleProblem(w2).marginalize(job), mr.reference_marginalize(w2, job))
    job0 = abi.make_marg_job([P, SB, P], [0, 0, 1], [-1] * 3, [0, 1, 0])
    ref0 = mr.reference_marginalize(w, job0)
    assert ref0["V_zero"] and ref0["n"] == 12 and np.all(np.asarray(ref0["H"]) == 0) and mr.rank_band(ref0) == (0, 0)
    mr.check_prior(op.OracleProblem(w).marginalize(job0), ref0)


# ---- sensitivity: the comparator rejects each planted fault
def _oldest_job(w):
    return mr.frames_job(w, n_pose=1, n_sb=1, lm_before=3, n_frames=2)


def _rejects(g, ref):
    with pytest.raises(AssertionError):
        mr.check_prior(g, ref)


def test_rejects_a_dropped_observation():
    w = synthetic.make_window(2, 0)
    job = _oldest_job(w)
    ref = mr.reference_marginalize(w, job)
    obs = w.obs.copy()
    obs["sqrt_info"][np.nonzero(obs["lm_idx"] == job._keep[6][0])[0][0]] = 0.0
    _rejects(op.OracleProblem(dataclasses.replace(w, obs=obs)).marginalize(job), ref)


def test_rejects_rho_prime_instead_of_its_square_root():
    """rho' for one landmark: its observations weighted by an extra sqrt(rho') (sqrt_info scaled by (1 + |r|^2)^-1/4)."""
    w = synthetic.make_window(2, 0)
    job = _oldest_job(w)
    ref = mr.reference_marginalize(w, job)
    obs = w.obs.copy()
    res = {}
    for i in np.nonzero(np.isin(obs["lm_idx"], job._keep[6]))[0]:
        ob = obs[i]
        r, _, _, _ = op.eval_reprojection(w.cameras[ob["cam_idx"]], w.poses[ob["pose_idx"]][None], w.landmarks[ob["lm_idx"]][None],
                                          w.extrinsics[ob["ext_idx"]][None], ob["z"][None], np.array([ob["sqrt_info"]]))
        res[int(ob["lm_idx"])] = max(res.get(int(ob["lm_idx"]), 0.0), float(r[0] @ r[0]))
    l = max(res, key=res.get)        # where sqrt(rho') and rho' differ most
    for i in np.nonzero(obs["lm_idx"] == l)[0]:
        ob = obs[i]
        r, _, _, _ = op.eval_reprojection(w.cameras[ob["cam_idx"]], w.poses[ob["pose_idx"]][None], w.landmarks[l][None], w.extrinsics[ob["ext_idx"]][None],
                                          ob["z"][None], np.array([ob["sqrt_info"]]))
        obs["sqrt_info"][i] *= (1.0 + r[0] @ r[0]) ** -0.25
    _rejects(op.OracleProblem(dataclasses.replace(w, obs=obs)).marginalize(job), ref)


def _second_step(w):
    """A prior from the oldest-frame step, estimates moved by a solve, and the next step carrying pose 1, sb 1, pose 2."""
    job1 = _oldest_job(w)
    o1 = op.OracleProblem(w).marginalize(job1)
    prior = dict(block_kind=o1["block_kind"], block_idx=o1["block_idx"], x0=o1["x0"], J=np.ascontiguousarray(o1["J"]), e0=o1["e0"],
                 H=o1["H"], b0=o1["b0"])
    pb = op.OracleProblem(w)
    pb.solve(3, 1)
    st = pb.state()
    w2 = dataclasses.replace(w, poses=st["poses"], speed_bias=st["speed_bias"], landmarks=st["landmarks"],
                             marg=dict(block_kind=prior["block_kind"], block_idx=prior["block_idx"], x0=prior["x0"], J=prior["J"], e0=prior["e0"]))
    job2 = abi.make_marg_job([P, SB, P, SB, P], [1, 1, 2, 2, 3], [0, 1, 2, -1, -1], [1, 1, 0, 0, 0], imu_terms=[1], sb_priors=[])
    return w2, prior, job2


def test_rejects_a_carried_block_linearised_at_the_current_estimate():
    w2, prior, job2 = _second_step(synthetic.make_window(2, 0))
    ref = mr.reference_marginalize(w2, job2, prior=prior)
    assert mr.check_prior(op.OracleProblem(w2).marginalize(job2, H_prev=prior["H"], b0_prev=prior["b0"]), ref) is not None
    x0 = prior["x0"].copy()
    x0[16:23] = w2.poses[2]                 # carried block 2 (pose 2) at the current estimate
    wf = dataclasses.replace(w2, marg=dict(w2.marg, x0=x0))
    g = op.OracleProblem(wf).marginalize(job2, H_prev=prior["H"], b0_prev=prior["b0"])
    g["x0"] = ref["x0"]                     # hide the x0 difference: the system itself must give the fault away
    _rejects(g, ref)


def test_rejects_an_imu_term_preintegrated_afresh():
    w = synthetic.make_window(2, 0)
    job = _oldest_job(w)
    # a cache from an earlier bias, close enough for the first-order bias correction (no re-preintegration)
    sb_ref = w.speed_bias[0] + np.r_[np.zeros(3), 3e-5 * np.ones(3), 3e-5 * np.ones(3)]
    ref = mr.reference_marginalize(w, job, imu_cache={0: (sb_ref, 1)})
    pb = op.OracleProblem(w)
    pb.set_imu_cache(0, sb_ref, True)
    mr.check_prior(pb.marginalize(job), ref)
    _rejects(op.OracleProblem(w).marginalize(job), ref)     # preintegrated afresh at the linearisation point


def test_rejects_a_negated_e0_entry():
    w = synthetic.make_window(2, 0)
    job = _oldest_job(w)
    ref = mr.reference_marginalize(w, job)
    g = op.OracleProblem(w).marginalize(job)
    mr.check_prior(g, ref)
    k = int(np.argmax(np.abs(g["e0"])))
    g["e0"][k] = -g["e0"][k]
    _rejects(g, ref)


@pytest.mark.parametrize("name", ["A", "C"])
def test_rejects_one_landmark_weighted_four_times(name):
    wname, kw, _, _, _ = SHAPES[name]
    w = window(wname)
    job = mr.frames_job(w, **kw)
    ref = mr.reference_marginalize(w, job)
    obs = w.obs.copy()
    obs["sqrt_info"][obs["lm_idx"] == job._keep[6][0]] *= 2.0
    _rejects(op.OracleProblem(dataclasses.replace(w, obs=obs)).marginalize(job), ref)


@pytest.mark.parametrize("name", ["B", "C", "C'"])
def test_a_wrong_n_in_the_rank_threshold_cannot_change_a_well_defined_rank(name):
    """The rank threshold eps * n * lambda_max computed with the dimension N of the system before marginalising (or
    any n' with n'/n < RANK_GAP) classifies every eigenvalue as the right one does wherever the rank is well defined:
    no eigenvalue lies between the two thresholds, so J, e0 and the rank are bit-identical and there is no output
    difference for any comparator to reject.  Where the rank is not well defined, eigenvalues near the threshold are
    rounding noise that correct implementations also classify either way."""
    wname, kw, N, _, n = SHAPES[name]
    w = window(wname)
    ref = mr.reference_marginalize(w, mr.frames_job(w, **kw))
    lo, hi = mr.rank_band(ref)
    assert lo == hi
    lam = ref["lam"]
    thr_n, thr_N = mr.EPS * n * lam.max(), mr.EPS * N * lam.max()
    assert not np.any((lam > thr_n) & (lam <= thr_N))
    assert N / n < mr.RANK_GAP
