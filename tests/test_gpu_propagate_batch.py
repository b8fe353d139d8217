"""Batched IMU propagation (okb_imu_propagate_batch): every job of a batch gives exactly what okb_imu_propagate gives on
the same arguments, agrees with the oracle, and runs beside a solve in flight without changing either."""
import ctypes as C

import numpy as np
import pytest

from okvis_b200 import abi, synthetic
from test_oracle_functors import rand_pose

gpu = pytest.mark.gpu

PRM_A = abi.make_imu_params()
PRM_B = abi.make_imu_params(a_max=60.0, g_max=4.0, sigma_g_c=2.0e-3, sigma_a_c=1.5e-2, sigma_bg=0.05, sigma_ba=0.2,
                            sigma_gw_c=1.0e-5, sigma_aw_c=1.0e-4, tau=1800.0, g=9.80665, a0=(0.01, -0.02, 0.03), rate=100)


def imu_job(rng, prm, n, t0_on_sample, t1_on_sample, cov, jac, saturate=None, beyond=False):
    """n samples at prm.rate of sinusoidal motion (as _imu_case) and a state; t0 / t1 on the first / last sample time
    or between samples.  beyond: t1 lies after the last sample."""
    dt = int(1e9 / prm.rate)
    ts = 1_000_000_000 + int(rng.integers(0, dt)) + np.arange(n, dtype=np.int64) * dt
    s = np.zeros(n, abi.imu_sample_dtype)
    s["t_ns"] = ts
    tt = ts * 1e-9
    s["gyro"] = np.stack([0.3 * np.sin(3 * tt + 0.1), 0.2 * np.cos(2 * tt), 0.25 * np.sin(1.7 * tt + 1)], -1)
    s["acc"] = np.stack([1.0 * np.sin(2 * tt), 0.5 * np.cos(3 * tt), 9.81 + 0.3 * np.sin(tt)], -1)
    s["gyro"] += rng.normal(0, 0.01, s["gyro"].shape)
    s["acc"] += rng.normal(0, 0.05, s["acc"].shape)
    if saturate == "acc":
        s["acc"][n // 2, 2] = 2.0 * prm.a_max
    elif saturate == "gyro":
        s["gyro"][n // 2, 0] = 2.0 * prm.g_max
    t0 = int(ts[0]) if t0_on_sample else int(ts[0]) + dt // 4 + int(rng.integers(0, dt // 8))
    t1 = int(ts[-1]) if t1_on_sample else int(ts[-1]) - dt // 3 - int(rng.integers(0, dt // 8))
    if beyond:
        t1 = int(ts[-1]) + dt // 2
    pose = rand_pose(rng, 1.0, 0.5)
    sb = np.concatenate([rng.normal(0, 0.5, 3), rng.normal(0, 0.01, 3), rng.normal(0, 0.05, 3)])
    return (prm, s, t0, t1, pose, sb, cov, jac)


def mixed_jobs(seed=71):
    """About 40 jobs: 2 to 400 samples, t0 / t1 on and between samples, two parameter sets, accelerometer and gyro
    saturation, every combination of covariance and Jacobian, and one job whose samples end before t1."""
    rng = np.random.default_rng(seed)
    counts = [2, 3, 4, 7, 12, 26, 52, 53, 101, 173, 250, 400]
    jobs = []
    for i in range(40):
        prm = PRM_A if i % 3 else PRM_B
        sat = {5: "acc", 11: "gyro", 17: "acc", 23: "gyro"}.get(i)
        jobs.append(imu_job(rng, prm, counts[i % len(counts)], (i // 2) % 2 == 0, (i // 4) % 2 == 0, i % 4 in (0, 1),
                            i % 4 in (0, 2), saturate=sat, beyond=(i == 29)))
    return jobs


def as_bytes(res):
    n, pose, sb, P, F = res
    return (int(n), pose.tobytes(), sb.tobytes(), P.tobytes(), F.tobytes())


@pytest.fixture(scope="module")
def ctx(okb):
    c = okb.Context(0, 1)
    yield c
    c.close()


@gpu
def test_mixed_batch_equals_single_calls(ctx):
    jobs = mixed_jobs()
    single = [ctx.imu_propagate(*j) for j in jobs]
    got = ctx.imu_propagate_batch(jobs)
    assert len(got) == len(jobs)
    for i, (a, b) in enumerate(zip(got, single)):
        assert as_bytes(a) == as_bytes(b), i
    for i, j in enumerate(jobs):
        assert as_bytes(ctx.imu_propagate_batch([j])[0]) == as_bytes(single[i]), i
    failed = [i for i, r in enumerate(got) if r[0] < 0]
    assert failed == [29]
    n, pose, sb, P, F = got[29]
    assert n == -1 and np.array_equal(pose, jobs[29][4]) and np.array_equal(sb, jobs[29][5])
    assert not P.any() and not F.any()
    assert min(r[0] for r in got if r[0] >= 0) >= 1 and max(r[0] for r in got) >= 300


@gpu
def test_mixed_batch_matches_oracle(ctx, oracle):
    jobs = mixed_jobs()
    got = ctx.imu_propagate_batch(jobs)
    for i, (j, (n1, p1, s1, P1, F1)) in enumerate(zip(jobs, got)):
        prm, s, t0, t1, pose, sb, cov, jac = j
        n0, pose1, sb1, P0, F0 = oracle.imu_propagate(prm, s, t0, t1, pose, sb)
        assert n0 == n1, i
        if n0 < 0:
            continue
        assert np.abs(p1 - pose1).max() < 1e-12 * max(1.0, np.abs(pose1).max()), i
        assert np.abs(s1 - sb1).max() < 1e-12 * max(1.0, np.abs(sb1).max()), i
        if cov:
            assert np.abs(P1 - P0).max() < 1e-11 * np.abs(P0).max(), i
        if jac:
            assert np.abs(F1 - F0).max() < 1e-11 * max(1.0, np.abs(F0).max()), i


@gpu
def test_batch_beside_an_optimize_in_flight(okb):
    c = okb.Context(0, 4)
    try:
        ws = [synthetic.make_window(1, i) for i in range(4)]
        c.upload_batch(0, ws)
        ref = c.optimize(0, 4, max_iterations=6)
        ref_states = c.download_batch(0, 4)
        jobs = mixed_jobs(72)
        prop_ref = [as_bytes(c.imu_propagate(*j)) for j in jobs]
        c.imu_propagate_batch(jobs)          # sizes the batch buffers, so the call below allocates nothing
        c.upload_batch(0, ws)
        c.optimize_async(0, 4, max_iterations=6)
        got = c.imu_propagate_batch(jobs)
        summ = c.optimize_finish(0, 4)
        states = c.download_batch(0, 4)
        assert [as_bytes(r) for r in got] == prop_ref
        for a, b in zip(summ, ref):
            assert {k: v for k, v in a.items() if k != "solve_time_s"} == {k: v for k, v in b.items() if k != "solve_time_s"}
        for a, b in zip(states, ref_states):
            for k in ("poses", "speed_bias", "landmarks", "quality"):
                assert np.array_equal(a[k], b[k]), k
    finally:
        c.close()


@gpu
def test_batch_argument_checks(ctx, okb):
    L = okb.lib()
    jobs = mixed_jobs(73)[:3]
    keep = []

    def table(bad=None):
        """Three jobs over fresh outputs filled with a sentinel; `bad` overrides fields of job 2."""
        arr = (abi.PropagateJob * 3)()
        outs = []
        for j, (prm, s, t0, t1, pose, sb, cov, jac) in zip(arr, jobs):
            o = dict(pose=pose.copy(), sb=sb.copy(), P=np.full((15, 15), 7.0), F=np.full((15, 15), 7.0),
                     n=np.full(1, 99, np.int32), s=np.ascontiguousarray(s))
            j.params, j.samples, j.n_samples, j.t0_ns, j.t1_ns = C.pointer(prm), o["s"].ctypes.data, len(s), t0, t1
            j.pose, j.speed_bias, j.covariance, j.jacobian = (abi.dptr(o["pose"]), abi.dptr(o["sb"]), abi.dptr(o["P"]),
                                                              abi.dptr(o["F"]))
            j.n_used = o["n"].ctypes.data_as(C.POINTER(C.c_int32))
            outs.append(o)
        for k, v in (bad or {}).items():
            setattr(arr[2], k, v)
        keep.append(outs)
        return arr, outs

    def unchanged(outs):
        return all(np.array_equal(o["pose"], j[4]) and np.array_equal(o["sb"], j[5]) and np.all(o["P"] == 7.0)
                   and np.all(o["F"] == 7.0) and o["n"][0] == 99 for o, j in zip(outs, jobs))

    for bad in (dict(params=None), dict(samples=None), dict(pose=None), dict(speed_bias=None), dict(n_samples=1),
                dict(n_samples=0), dict(n_samples=-5)):
        arr, outs = table(bad)
        assert L.okb_imu_propagate_batch(ctx._h, 3, arr) == abi.OKB_ERR_INVALID_ARG, bad
        assert "job 2" in L.okb_last_error(ctx._h).decode(), bad
        assert unchanged(outs), bad
    arr, outs = table()
    assert L.okb_imu_propagate_batch(ctx._h, -1, arr) == abi.OKB_ERR_INVALID_ARG
    assert L.okb_imu_propagate_batch(ctx._h, 3, None) == abi.OKB_ERR_INVALID_ARG
    assert unchanged(outs)
    before = ctx.kernel_launches
    assert L.okb_imu_propagate_batch(ctx._h, 0, arr) == abi.OKB_OK
    assert L.okb_imu_propagate_batch(ctx._h, 0, None) == abi.OKB_OK
    assert unchanged(outs) and ctx.kernel_launches == before
    assert L.okb_imu_propagate_batch(ctx._h, 3, arr) == abi.OKB_OK
    assert all(o["n"][0] > 0 for o in outs)


@gpu
def test_launch_count_and_a_large_batch(ctx):
    jobs = mixed_jobs(74)
    before = ctx.kernel_launches
    ctx.imu_propagate_batch(jobs)
    assert ctx.kernel_launches == before + 1
    ctx.imu_propagate_batch(jobs[:1])
    assert ctx.kernel_launches == before + 2
    ctx.imu_propagate(*jobs[0])
    assert ctx.kernel_launches == before + 3
    rng = np.random.default_rng(75)
    big = [imu_job(rng, PRM_A if i % 5 else PRM_B, 2 + i % 3 if i % 2 else 52, i % 3 == 0, i % 7 == 0, i % 4 < 2,
                   i % 2 == 0) for i in range(2048)]
    before = ctx.kernel_launches
    got = ctx.imu_propagate_batch(big)
    assert ctx.kernel_launches == before + 1
    assert all(r[0] >= 1 for r in got)
    for i in sorted(set(rng.choice(2048, 64, replace=False).tolist()) | {0, 2047}):
        assert as_bytes(got[i]) == as_bytes(ctx.imu_propagate(*big[i])), i


def test_propagate_job_layout():
    J = abi.PropagateJob
    assert C.sizeof(J) == 80
    offsets = dict(params=0, samples=8, n_samples=16, _pad=20, t0_ns=24, t1_ns=32, pose=40, speed_bias=48, covariance=56,
                   jacobian=64, n_used=72)
    assert {k: getattr(J, k).offset for k in offsets} == offsets
