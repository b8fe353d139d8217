"""Marginalisation of landmark-sharded windows (k_marginalize<true>): every rank linearises its own landmarks, the
ranks sum their Schur terms through the shard mailbox in rank order, and every rank holds the bit-identical prior.
The prior is checked against the oracle's and the extended-precision reference's marginalisation of the UNSHARDED
window; a sliding cfg-5 shaped window is checked step by step against an unsharded context driven through the same
edits.  All rank contexts live in this process on device 0 (okb_shard_connect_local) unless noted."""
import os
import subprocess
import sys

import numpy as np
import pytest

import marg_reference as mr
from okvis_b200 import abi, sharding, synthetic
from test_gpu_marginalization import at_estimates, compare_prior, drop_oldest, first_job, oracle_like_device, well_conditioned

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from shard_slide_worker import PRIOR_KEYS, Slide, slide_problem  # noqa: E402

P, SB = abi.BLOCK_POSE, abi.BLOCK_SPEED_BIAS
MERR_POSE_NOT_CONNECTED, MERR_SHARD_JOB = 4, 6


class Ranks:
    """`world` contexts on device 0 with `slots` window slots each, connected as one landmark-sharded group."""

    def __init__(self, okb, world, max_frames, slots=1):
        self.world = world
        self.ctxs = [okb.Context(0, slots) for _ in range(world)]
        okb.Context.shard_connect_local(self.ctxs, max_frames=max_frames)
        self.idx = {}

    def close(self):
        for c in self.ctxs:
            c.close()

    def upload(self, slot, w):
        for r, c in enumerate(self.ctxs):
            sw, idx = sharding.shard_window(w, r, self.world)
            self.idx[slot, r] = idx
            c.reserve(slot, len(w.poses), len(sw.landmarks), len(sw.obs), len(w.imu_samples), 160)
            c.upload(slot, sw)

    def optimize(self, first, count, iters):
        for c in self.ctxs:          # pending edits of every rank applied before any rank's solver spins
            c.commit(first, count)
        for c in self.ctxs:
            c.optimize_async(first, count, max_iterations=iters)
        return [c.optimize_finish(first, count) for c in self.ctxs]

    def estimates(self, slot, K, NSB, L):
        parts = [(self.idx[slot, r], c.download(slot, dims=(K, NSB, len(self.idx[slot, r])))) for r, c in enumerate(self.ctxs)]
        for _, d in parts[1:]:
            assert d["poses"].tobytes() == parts[0][1]["poses"].tobytes() and d["speed_bias"].tobytes() == parts[0][1]["speed_bias"].tobytes()
        return sharding.merge_shard_results(L, parts)

    def edit(self, slot, op, *args):
        for r, c in enumerate(self.ctxs):
            a = sharding.route_edit(op, r, self.world, *args)
            if a is not None:
                getattr(c, op)(slot, *a)

    def marginalize(self, slot, kw):
        for r, c in enumerate(self.ctxs):
            c.marginalize(slot, sharding.shard_marg_job(r, self.world, **kw))
        return [c.download_marg(slot) for c in self.ctxs]


def job_kwargs(job):
    k = job._keep
    return dict(block_kind=k[0], block_idx=k[1], block_prev=k[2], block_marginalize=k[3], imu_terms=k[4], sb_priors=k[5], landmarks=k[6])


def prior_bytes(g):
    return [np.asarray(g[k]).tobytes() for k in PRIOR_KEYS]


def assert_identical(gs):
    for g in gs[1:]:
        assert prior_bytes(g) == prior_bytes(gs[0])


def checked_step(rk, oracle, slot, w, est, job):
    """One sharded marginalisation of `job` (global landmark slots) on `slot`: identical on every rank, and the
    oracle's and the reference's marginalisation of the unsharded window `w` at the estimates `est`."""
    c0 = rk.ctxs[0]
    cache = {}
    for t in range(len(w.imu_terms)):
        sb_ref, valid, _ = c0.debug_imu_cache(slot, t)
        cache[t] = (sb_ref.copy(), valid)
    we = at_estimates(w, est)
    ref = mr.reference_marginalize(we, job, imu_cache=cache)
    o = oracle_like_device(oracle, c0, slot, w, est).marginalize(job)
    gs = rk.marginalize(slot, job_kwargs(job))
    assert_identical(gs)
    g = gs[0]
    assert g["status"][0] == 0 and g["status"][3] < 40
    mr.check_prior(g, ref)
    if ref["n"]:
        compare_prior(g, o)
    return g, o


@pytest.mark.parametrize("world,rank0_only", [(2, False), (3, False), (2, True)])
def test_oldest_frame_matches_the_unsharded_window(okb, oracle, world, rank0_only):
    w = synthetic.make_window(1, 0)
    K, L = len(w.poses), len(w.landmarks)
    rk = Ranks(okb, world, K)
    try:
        rk.upload(0, w)
        rk.optimize(0, 1, 6)
        est = rk.estimates(0, K, K, L)
        job, lms, _ = first_job(oracle, at_estimates(w, est))
        if rank0_only:                  # rank 1 holds none of the marginalised landmarks and pushes zeros
            kw = job_kwargs(job)
            kw["landmarks"] = lms[lms % world == 0]
            job = abi.make_marg_job(**kw)
            assert sharding.shard_marg_job(1, world, **kw).n_landmarks == 0
        assert job.n_landmarks > 3
        g, _ = checked_step(rk, oracle, 0, w, est, job)
        assert g["n"] == 21
    finally:
        rk.close()


def test_b_stereo_all_blocks_grows_the_scratch(okb, oracle):
    """Case B of test_gpu_marginalization_shapes.py at world 2: 1000 landmarks per rank, after a small job sized the
    scratch for 256, so both ranks grow it while the other rank's kernel may already wait for them."""
    w = synthetic.make_window(2, 0)
    K, L = len(w.poses), len(w.landmarks)
    rk = Ranks(okb, 2, K)
    try:
        rk.upload(0, w)
        rk.optimize(0, 1, 6)
        est = rk.estimates(0, K, K, L)
        small = mr.frames_job(at_estimates(w, est), n_pose=1, n_sb=1, lm_before=3, n_frames=2)
        assert all(g["status"][0] == 0 for g in rk.marginalize(0, job_kwargs(small)))
        rk.upload(0, w)                 # a full upload: no prior, the scratch stays
        rk.optimize(0, 1, 6)
        est = rk.estimates(0, K, K, L)
        job = mr.frames_job(at_estimates(w, est), n_pose=1, n_sb=1, lm_before=99)
        lms = job._keep[6]
        assert min((lms % 2 == r).sum() for r in range(2)) > 256
        g, _ = checked_step(rk, oracle, 0, w, est, job)
        assert g["n"] == 135
    finally:
        rk.close()


def test_c_full_system_of_255_at_world_4(okb, oracle):
    w = synthetic.make_window(2, 0, cfg=synthetic.WindowConfig(**mr.STEREO17))
    K, L = len(w.poses), len(w.landmarks)
    rk = Ranks(okb, 4, K)
    try:
        rk.upload(0, w)
        rk.optimize(0, 1, 6)
        est = rk.estimates(0, K, K, L)
        job = mr.frames_job(at_estimates(w, est), n_pose=7, n_sb=6, lm_before=7)
        g, _ = checked_step(rk, oracle, 0, w, est, job)
        assert g["n"] == 159
    finally:
        rk.close()


def test_second_marginalisation_reuses_the_persisted_system(okb, oracle):
    """As test_gpu_marginalization.py's test of the same name, sharded over 2 ranks: the second step carries the first
    prior's blocks (block_prev >= 0) and starts from the H / b0 the first left on every rank."""
    w = synthetic.make_window(1, 3)
    K, L = len(w.poses), len(w.landmarks)
    rk = Ranks(okb, 2, K)
    try:
        rk.upload(0, w)
        rk.optimize(0, 1, 5)
        est = rk.estimates(0, K, K, L)
        job, lms, cand = first_job(oracle, at_estimates(w, est))
        g1, o1 = checked_step(rk, oracle, 0, w, est, job)
        rk.edit(0, "remove_landmarks", cand)
        rk.edit(0, "remove_frame", 0, 0)
        marg_o = dict(block_kind=o1["block_kind"], block_idx=(o1["block_idx"] - 1).astype(np.uint32), x0=o1["x0"], J=np.ascontiguousarray(o1["J"]), e0=o1["e0"])
        w2, pp = drop_oldest(at_estimates(w, est), cand, marg_o, est["poses"][1])
        rk.edit(0, "set_priors", pp, np.zeros(0, abi.sb_prior_dtype))
        rk.optimize(0, 1, 4)
        est2 = rk.estimates(0, K - 1, K - 1, L)
        first, last = mr.track_ends(w2)
        lms2 = well_conditioned(oracle, at_estimates(w2, est2), np.nonzero((first == 0) & (last <= 2))[0])
        job2 = abi.make_marg_job([P, SB, P, SB, P], [0, 0, 1, 1, 2], [0, 1, 2, -1, -1], [1, 1, 0, 0, 0], imu_terms=[0], sb_priors=[], landmarks=lms2)
        ref2 = oracle_like_device(oracle, rk.ctxs[0], 0, w2, est2)
        gs = rk.marginalize(0, job_kwargs(job2))
        assert_identical(gs)
        o2 = ref2.marginalize(job2, H_prev=o1["H"], b0_prev=o1["b0"])
        compare_prior(gs[0], o2, tol=5e-9)
        assert np.array_equal(gs[0]["x0"][:7], g1["x0"][16:23])
    finally:
        rk.close()


def test_batch_equals_single_calls(okb, oracle):
    """marginalize_batch over two slots on every rank (one exchange per slot) gives, per slot, the bytes of the single
    sharded call."""
    ws = [synthetic.make_window(1, 0), synthetic.make_window(1, 1)]
    K, L = len(ws[0].poses), len(ws[0].landmarks)
    rk = Ranks(okb, 2, K, slots=2)
    try:
        def restore():
            for s, w in enumerate(ws):
                rk.upload(s, w)
            rk.optimize(0, 2, 6)
            return [rk.estimates(s, K, K, L) for s in range(2)]
        est = restore()
        kws = [job_kwargs(first_job(oracle, at_estimates(w, e))[0]) for w, e in zip(ws, est)]
        for r, c in enumerate(rk.ctxs):
            c.marginalize_batch(0, [sharding.shard_marg_job(r, 2, **kw) for kw in kws])
        batch = [[c.download_marg(s) for c in rk.ctxs] for s in range(2)]
        est2 = restore()
        assert all(a["poses"].tobytes() == b["poses"].tobytes() for a, b in zip(est, est2))
        single = [rk.marginalize(s, kws[s]) for s in range(2)]
        for s in range(2):
            assert batch[s][0]["status"][0] == 0 and batch[s][0]["n"] == 21
            assert_identical(batch[s])
            assert prior_bytes(batch[s][0]) == prior_bytes(single[s][0])
    finally:
        rk.close()


def test_a_rank_error_or_a_job_mismatch_stops_every_rank(okb, oracle):
    """Rank 1 with a different IMU-term list: every rank reports MERR_SHARD_JOB.  A landmark only rank 1 holds, seen in
    a frame the job does not list: every rank reports rank 1's MERR_POSE_NOT_CONNECTED.  Both ranks arrive in both
    cases; every rank keeps the prior it held."""
    w = synthetic.make_window(1, 0)
    K, L = len(w.poses), len(w.landmarks)
    rk = Ranks(okb, 2, K)
    try:
        rk.upload(0, w)
        rk.optimize(0, 1, 6)
        est = rk.estimates(0, K, K, L)
        job, _, _ = first_job(oracle, at_estimates(w, est))
        kw = job_kwargs(job)
        before = rk.marginalize(0, kw)
        assert before[0]["status"][0] == 0
        rk.ctxs[0].marginalize(0, sharding.shard_marg_job(0, 2, **kw))
        rk.ctxs[1].marginalize(0, sharding.shard_marg_job(1, 2, **dict(kw, imu_terms=[])))
        after = [c.download_marg(0) for c in rk.ctxs]
        far = np.unique(w.obs["lm_idx"][w.obs["pose_idx"] == K - 1])
        odd = far[far % 2 == 1][:1]
        # the prior of `before` (pose 1, speed/bias 1, pose 2) is still in place: the job carries it
        gs = rk.marginalize(0, dict(kw, block_prev=[-1, -1, 0, 1, 2], landmarks=np.concatenate([kw["landmarks"], odd]).astype(np.uint32)))
        for got, code in ((after, MERR_SHARD_JOB), (gs, MERR_POSE_NOT_CONNECTED)):
            for g, b in zip(got, before):
                assert g["status"][0] == code
                assert prior_bytes(g)[:-1] == prior_bytes(b)[:-1]          # everything but the status word
        assert rk.ctxs[0].download_marg(0)["status"][0] == MERR_POSE_NOT_CONNECTED
    finally:
        rk.close()


def compare_sliding(g, u):
    """The sharded prior against the unsharded context's: the linearisation points are the two contexts' estimates,
    which agree to the solver's parity bound, and H / b0 are formed at them."""
    dx = np.abs(g["x0"] - u["x0"]).max()
    assert dx < 1e-7
    # b0 = -J^T r moves to first order by H dx with the linearisation point: |db0| <= n max|H| max|dx| (+ rounding)
    n = g["n"]
    assert np.abs(g["b0"] - u["b0"]).max() <= n * np.abs(u["H"]).max() * dx + 2e-9 * max(1.0, np.abs(u["b0"]).max())
    compare_prior(dict(g, x0=u["x0"], b0=u["b0"]), dict(u, rank=int(u["status"][1])), tol=1e-8)


def test_sliding_cfg5_window_at_world_4(okb):
    """20 frames, 4 cameras, 2000 landmarks; 3 steps of optimize(6), marginalisation of the oldest frame and its
    finished landmarks, and the edits that slide the window (routed by owner), sharded over 4 ranks and unsharded."""
    full, w0, first_seen = slide_problem(2000, extra=3)
    world = 4
    ctxs = [okb.Context(0, 1) for _ in range(world)]
    uctx = okb.Context(0, 1)
    try:
        okb.Context.shard_connect_local(ctxs, max_frames=len(w0.poses))
        sh = Slide(list(enumerate(ctxs)), world, full, w0, first_seen)
        un = Slide([(0, uctx)], 1, full, w0, first_seen)
        for step in range(3):
            ss, su = sh.optimize(6), un.optimize(6)[0]
            for s in ss:
                assert s["iterations"] == su["iterations"] and s["termination"] == su["termination"] != 6, (step, s, su)
                assert abs(s["final_cost"] - su["final_cost"]) <= 1e-7 * su["final_cost"]
            assert all(c.shard_stats(0)["fault"] == 0 for c in ctxs)
            parts = sh.parts()
            for _, d in parts[1:]:
                assert d["poses"].tobytes() == parts[0][1]["poses"].tobytes() and d["speed_bias"].tobytes() == parts[0][1]["speed_bias"].tobytes()
            eg = sharding.merge_shard_results(sh.L, parts)
            eu = sharding.merge_shard_results(un.L, un.parts())
            assert np.abs(eg["poses"] - eu["poses"]).max() < 1e-7 and np.abs(eg["speed_bias"] - eu["speed_bias"]).max() < 1e-7
            kw, cand = un.job(eu, select=mr.well_conditioned)
            sh.marginalize(kw)
            un.marginalize(kw)
            gs, u = sh.priors(), un.priors()[0]
            assert_identical(gs)
            assert u["status"][0] == 0
            compare_sliding(gs[0], u)
            sh.advance(cand, eg["poses"][1])
            un.advance(cand, eu["poses"][1])
    finally:
        for c in ctxs + [uctx]:
            c.close()


def _free_port():
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_multi_process_slide_over_ipc(okb, tmp_path):
    """tools/shard_slide_worker.py under torchrun (one process per GPU, mailboxes over cudaIpc), 2 steps, against the
    same slide unsharded in this process: needs >= 2 GPUs."""
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs at least 2 GPUs")
    world = 2 if n < 4 else 4
    out = tmp_path / "slide.npz"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(ROOT, "tools", "shard_slide_worker.py"), "--landmarks", "2000", "--steps", "2",
           "--out", str(out)]
    subprocess.run(cmd, check=True, timeout=900, cwd=ROOT)
    z = np.load(out, allow_pickle=True)
    full, w0, first_seen = slide_problem(2000, extra=2)
    uctx = okb.Context(0, 1)
    try:
        un = Slide([(0, uctx)], 1, full, w0, first_seen)
        for step in range(2):
            su = un.optimize(6)[0]
            for s in z["summaries_%d" % step]:
                assert s["iterations"] == su["iterations"] and s["termination"] == su["termination"]
                assert abs(s["final_cost"] - su["final_cost"]) <= 1e-7 * su["final_cost"]
            assert not z["faults_%d" % step].any()
            eu = sharding.merge_shard_results(un.L, un.parts())
            assert np.abs(z["poses_%d" % step] - eu["poses"]).max() < 1e-7
            kw, cand = un.job(eu, select=mr.well_conditioned)
            assert np.array_equal(kw["landmarks"], z["landmarks_%d" % step])
            un.marginalize(kw)
            u = un.priors()[0]
            gs = [{k: z["prior_%d_%d_%s" % (step, r, k)] for k in PRIOR_KEYS} for r in range(world)]
            for g in gs:
                g["n"] = int(g["n"])
            assert_identical(gs)
            compare_sliding(gs[0], u)
            un.advance(cand, eu["poses"][1])
    finally:
        uctx.close()
