"""Seeded IMU-term cases at the edges of the sample recursion, shared by tests/test_imu_reference.py (oracle and host
build against tests/imu_reference.py) and tests/test_gpu_imu_shapes.py (the device's three instantiations).

Each case is a dict: group, name, prm (abi.ImuParams), samples (abi.imu_sample_dtype), t0, t1 (ns), pose0, sb0, pose1,
sb1 and sb_ref, the bias of an earlier preintegration (the correction path; its b_g lies 0.9e-4 / Delta_t from sb0's
unless the case is about that offset).  The samples of every case cover [t0, t1]."""
import functools

import numpy as np

from okvis_b200 import abi

import imu_reference as ir

PRM_A = abi.make_imu_params()
PRM_B = abi.make_imu_params(a_max=60.0, g_max=4.0, sigma_g_c=2.0e-3, sigma_a_c=1.5e-2, sigma_bg=0.05, sigma_ba=0.2,
                            sigma_gw_c=1.0e-5, sigma_aw_c=1.0e-4, tau=1800.0, g=9.80665, a0=(0.01, -0.02, 0.03), rate=100)
PRM_TINY_WALK = abi.make_imu_params(sigma_aw_c=1.0e-6)     # a badly conditioned P_delta
SEED = 0x1A0


def _unit(rng):
    u = rng.normal(0, 1, 3)
    return u / np.linalg.norm(u)


def _rand_pose(rng):
    q = rng.normal(0, 1, 4)
    return np.concatenate([rng.uniform(-1, 1, 3), q / np.linalg.norm(q)])


def _samples(rng, n, rate, start_ns):
    """n samples at `rate` Hz of sinusoidal motion plus noise (as TestImuError.cpp:80-150)."""
    dt = int(round(1e9 / rate))
    ts = start_ns + np.arange(n, dtype=np.int64) * dt
    s = np.zeros(n, abi.imu_sample_dtype)
    s["t_ns"] = ts
    tt = (ts - start_ns) * 1e-9 + rng.uniform(0, 10)
    s["gyro"] = np.stack([0.3 * np.sin(3 * tt + 0.1), 0.2 * np.cos(2 * tt), 0.25 * np.sin(1.7 * tt + 1)], -1)
    s["acc"] = np.stack([1.0 * np.sin(2 * tt), 0.5 * np.cos(3 * tt), 9.81 + 0.3 * np.sin(tt)], -1)
    s["gyro"] += rng.normal(0, 0.01, (n, 3))
    s["acc"] += rng.normal(0, 0.05, (n, 3))
    return s, dt


def _finish(rng, group, name, prm, s, t0, t1, sb0=None, sb_ref=None):
    """States for a case: a random pose0 / sb0, (pose1, sb1) = the float64 reference's propagation plus noise, and a
    correction-path sb_ref."""
    assert s["t_ns"][0] <= t0 < t1 <= s["t_ns"][-1], name
    pose0 = _rand_pose(rng)
    if sb0 is None:
        sb0 = np.concatenate([rng.normal(0, 0.5, 3), rng.normal(0, 0.01, 3), rng.normal(0, 0.05, 3)])
    case = dict(group=group, name=name, prm=prm, samples=s, t0=int(t0), t1=int(t1), pose0=pose0, sb0=np.asarray(sb0, float))
    pr = ir.propagate(s, prm, t0, t1, pose0, sb0, np.float64)
    d = np.concatenate([rng.normal(0, 0.01, 3), rng.normal(0, 0.005, 3)])
    q = np.asarray(pr["pose"][3:], float)
    dq = np.concatenate([np.sin(np.linalg.norm(d[3:]) / 2) * d[3:] / np.linalg.norm(d[3:]), [np.cos(np.linalg.norm(d[3:]) / 2)]])
    q1 = np.asarray(ir.qmul(dq, q), float)
    case["pose1"] = np.concatenate([np.asarray(pr["pose"][:3], float) + d[:3], q1 / np.linalg.norm(q1)])
    case["sb1"] = np.asarray(pr["sb"], float) + rng.normal(0, 0.01, 9)
    if sb_ref is None:
        Dt = (t1 - t0) * 1e-9
        sb_ref = case["sb0"] - np.concatenate([np.zeros(3), 0.9e-4 / Dt * _unit(rng), rng.normal(0, 0.02, 3)])
    case["sb_ref"] = np.asarray(sb_ref, float)
    return case


@functools.lru_cache(maxsize=None)
def cases(seed=SEED):
    rng = np.random.default_rng(seed)
    out = []
    T0 = 1_000_000_000

    # 1. the last integrated interval at every position of a batch of kImuBatch = 8 records, t1 on / between samples
    for n in list(range(2, 19)) + [25, 26, 33]:
        for on in ((True, False) if n in (9, 10, 17, 18) else ((n <= 9) ^ (n % 2 == 1),)):
            s, dt = _samples(rng, n, 200, T0)
            t0 = int(s["t_ns"][0]) + (0 if n % 2 == 0 else dt // 4)
            t1 = int(s["t_ns"][-1]) if on else int(s["t_ns"][-1]) - dt // 3
            out.append(_finish(rng, "batch_end", "n%d_t1%s" % (n, "on" if on else "in"), PRM_A, s, t0, t1))

    # 2. t0 on the first sample, inside the first interval, and after 1, 7, 8, 9 leading samples (on and between)
    for k, frac in ((0, 0.0), (0, 0.37), (1, 0.37), (7, 0.37), (8, 0.0), (8, 0.37), (9, 0.37)):
        s, dt = _samples(rng, 30, 200, T0)
        t0 = int(s["t_ns"][k]) + int(frac * dt)
        out.append(_finish(rng, "t0", "lead%d_%s" % (k, "on" if frac == 0 else "in"), PRM_A, s, t0, int(s["t_ns"][-1]) - dt // 5))

    # 3. t1 inside the first interval: one step, interpolated at both ends
    for n in (2, 6):
        s, dt = _samples(rng, n, 200, T0)
        out.append(_finish(rng, "t1_first", "n%d" % n, PRM_A, s, int(s["t_ns"][0]) + dt // 5, int(s["t_ns"][0]) + 3 * dt // 4))

    # 4. samples running 1, 8 and 50 past t1 (the early break in the middle of a batch)
    for extra in (1, 8, 50):
        s, dt = _samples(rng, 20 + extra, 200, T0)
        out.append(_finish(rng, "past_t1", "extra%d" % extra, PRM_A, s, int(s["t_ns"][0]) + dt // 3, int(s["t_ns"][19]) + dt // 2))

    # 5. repeated timestamps (zero-length intervals), one straddling a batch boundary (records 7 | 8)
    for dups in ((4,), (7,), (4, 7, 12)):
        s, dt = _samples(rng, 24, 200, T0)
        for d in dups:
            s["t_ns"][d + 1:] -= dt
        out.append(_finish(rng, "repeat", "dup" + "_".join(map(str, dups)), PRM_A, s, int(s["t_ns"][0]) + dt // 4,
                           int(s["t_ns"][-1]) - dt // 4))

    # 6. long terms
    for n in (400, 2000):
        for rate in (100, 200, 1000):
            s, dt = _samples(rng, n, rate, T0)
            out.append(_finish(rng, "long", "n%d_%dHz" % (n, rate), PRM_A, s, int(s["t_ns"][0]) + dt // 3,
                               int(s["t_ns"][-1]) - dt // 2))

    # 7. rotation: omega - b_g exactly zero; |omega - b_g| dt across 1e-4 (rightJacobian series); theta / 2 across 1e-6
    #    (sinc series); rates near g_max
    s, dt = _samples(rng, 20, 200, T0)
    sb0 = np.concatenate([rng.normal(0, 0.5, 3), [0.011, -0.007, 0.003], rng.normal(0, 0.05, 3)])
    s["gyro"] = sb0[3:6]
    out.append(_finish(rng, "rotation", "zero_rate", PRM_A, s, int(s["t_ns"][0]), int(s["t_ns"][-1]), sb0=sb0))
    for name, target in (("jr_1e-4", 1e-4), ("sinc_1e-6", 2e-6)):
        s, dt = _samples(rng, 24, 200, T0)
        u = _unit(rng)
        m = target / (dt * 1e-9) * np.linspace(0.995, 1.005, 24)        # |omega| dt straddles `target`
        sb0 = np.concatenate([rng.normal(0, 0.5, 3), np.zeros(3), rng.normal(0, 0.05, 3)])
        s["gyro"] = m[:, None] * u
        out.append(_finish(rng, "rotation", name, PRM_A, s, int(s["t_ns"][0]), int(s["t_ns"][-1]), sb0=sb0))
    s, dt = _samples(rng, 24, 200, T0)
    s["gyro"] = 0.97 * PRM_A.g_max * np.sign(rng.normal(0, 1, (24, 3)))
    out.append(_finish(rng, "rotation", "near_g_max", PRM_A, s, int(s["t_ns"][0]) + dt // 3, int(s["t_ns"][-1]) - dt // 3))

    # 8. saturation: exactly at the limit (not saturated), one ulp above, both sensors, only in an interpolated end
    up = lambda x: np.nextafter(x, np.inf)
    for name, g, a in (("gyro_at", PRM_A.g_max, None), ("gyro_ulp", up(PRM_A.g_max), None), ("acc_at", None, PRM_A.a_max),
                       ("acc_ulp", None, up(PRM_A.a_max)), ("both_ulp", up(PRM_A.g_max), up(PRM_A.a_max))):
        s, dt = _samples(rng, 20, 200, T0)
        if g is not None:
            s["gyro"][9, 1] = -g
        if a is not None:
            s["acc"][10, 2] = a
        out.append(_finish(rng, "saturation", name, PRM_A, s, int(s["t_ns"][0]) + dt // 4, int(s["t_ns"][-1]) - dt // 4))
    s, dt = _samples(rng, 20, 200, T0)
    s["gyro"][-1, 0] = 3 * PRM_A.g_max             # beyond t1: only the interpolated end at t1 exceeds the limit
    s["acc"][0, 1] = -3 * PRM_A.a_max              # before t0: only the interpolated start exceeds it
    out.append(_finish(rng, "saturation", "interp_ends", PRM_A, s, int(s["t_ns"][0]) + dt // 4, int(s["t_ns"][-1]) - dt // 2))

    # 9. Unix-epoch time stamps; t0 and t1 a few microseconds either side of a second boundary
    E = 1_700_000_000 * 1_000_000_000
    s, dt = _samples(rng, 61, 200, E + 974_123_456)
    out.append(_finish(rng, "epoch", "second_boundary", PRM_A, s, E + 999_999_997, E + 1_150_000_003))
    s, dt = _samples(rng, 220, 200, E + 987_654_321)
    out.append(_finish(rng, "epoch", "one_second", PRM_A, s, int(s["t_ns"][0]) + 1_234, int(s["t_ns"][0]) + 1_000_001_234))

    # 10. the parameter sets of test_gpu_propagate_batch, and a tiny accelerometer random walk
    for name, prm in (("prm_a", PRM_A), ("prm_b", PRM_B), ("tiny_walk", PRM_TINY_WALK)):
        s, dt = _samples(rng, 60, prm.rate, T0)
        out.append(_finish(rng, "params", name, prm, s, int(s["t_ns"][0]) + dt // 3, int(s["t_ns"][-1]) - dt // 3))

    # 11. the bias correction: b_g moved 0.9e-4 / Delta_t (first-order correction) and 1.1e-4 / Delta_t (redo) from the
    #     preintegration's bias, and only b_a moved, by a lot (never a redo)
    for name, k, dba in (("bg_0.9", 0.9e-4, 0.0), ("bg_1.1", 1.1e-4, 0.0), ("ba_only", 0.0, 0.4)):
        s, dt = _samples(rng, 50, 200, T0)
        t0, t1 = int(s["t_ns"][0]) + dt // 3, int(s["t_ns"][-1]) - dt // 3
        sb0 = np.concatenate([rng.normal(0, 0.5, 3), rng.normal(0, 0.01, 3), rng.normal(0, 0.05, 3)])
        Dt = (t1 - t0) * 1e-9
        sb_ref = sb0 - np.concatenate([np.zeros(3), k / Dt * _unit(rng), dba * _unit(rng)])
        out.append(_finish(rng, "bias", name, PRM_A, s, t0, t1, sb0=sb0, sb_ref=sb_ref))
    return tuple(out)


def case_ids(cs=None):
    return ["%s/%s" % (c["group"], c["name"]) for c in (cs or cases())]
