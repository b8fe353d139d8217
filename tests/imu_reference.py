"""Extended-precision reference for the IMU term (ImuError), written from the reference's okvis_ceres/src/ImuError.cpp
independently of the oracle and of the device templates (okb_imu.cuh).

One code path, generic in its floating type: run in np.longdouble it is the reference, run in np.float64 on inputs
perturbed by one rounding (and with sin / cos off by up to the 2 ulp CUDA's double math library allows) it measures
how far an honest double-precision realisation of the same algorithm lands from it, and that sets the comparator's
bound (`reference_and_bounds`).  It follows the reference's algorithm literally, quirks included:

  * the interval that reaches t1 is interpolated with r = dt / interval, dt measured from `time` (t0 for the first
    interval), not from the sample (ImuError.cpp:131-138);
  * the first integrated interval is interpolated after that, with the already interpolated end (:145-150);
  * saturation compares with a strict `>` (:156-173);
  * the propagation variant puts dt * sigma_a * sigma_a_c (the saturated and the unsaturated density) into Q and drops
    the right Jacobian from dalpha_db_g (:412, :438);
  * sinc switches to its series below 1e-6 and rightJacobian below 1e-4 (Transformation.hpp:45-81).

The last sample has no successor; where the reference would read past the end of its deque (only reachable with a
zero-length interval before it) this code uses the sample itself, as the device does.

Time differences are exact int64 nanoseconds, converted as okvis::Duration::toSec / okb::ns_to_sec do: whole seconds
plus 1e-9 times the nanoseconds."""
import numpy as np

LD = np.longdouble
EPS = float(np.finfo(np.float64).eps)
# the comparator's bound: this multiple of the largest deviation of a perturbed float64 run from the long double run
C_MEAS = 16.0
# ... and never below this many roundings of the block's largest reference magnitude
C_FLOOR = 4.0
# perturbed float64 runs per bound: the maximum over 4 depended on the seed by more than the margin absorbs in a few
# off-diagonal blocks of the information (an unchanged implementation went from 0.36 to 1.14 of its bound)
N_RUNS = 8

# planted faults the comparator must reject (tests/test_imu_reference.py); never set outside of that test
FAULTS = ("prop_q_in_preint", "dalpha_without_jr", "no_first_interp", "no_last_interp", "half_dt2",
          "bias_sign", "sat_ge")


def require_long_double():
    """The reference needs an extended format (x87 80-bit or binary128): fail, never skip, where it is not."""
    nmant = np.finfo(np.longdouble).nmant
    assert nmant >= 63, "np.longdouble has %d mantissa bits here; the IMU reference needs >= 63" % nmant


# ------------------------------------------------------------------------------------------------ small algebra
def ns_to_sec(ns, D):
    sec, nsec = divmod(int(ns), 1_000_000_000)
    return D(sec) + D(nsec) * (D(1) / D(1_000_000_000))


def crossmx(v):
    D = v.dtype.type
    z = D(0)
    return np.array([[z, -v[2], v[1]], [v[2], z, -v[0]], [-v[1], v[0], z]])


def qmul(a, b):
    """Hamilton product, coefficients (x, y, z, w) as Eigen stores them."""
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz])


def qconj(q):
    return np.array([-q[0], -q[1], -q[2], q[3]])


def qinv(q):
    return qconj(q) / (q @ q)


def qnormalized(q):
    return q / np.sqrt(q @ q)


def q2R(q):
    """Eigen's toRotationMatrix (no normalisation)."""
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def plus(q):
    """operators.hpp:92-100: q * p = plus(q) p."""
    x, y, z, w = q
    return np.array([[w, -z, y, x], [z, w, -x, y], [-y, x, w, z], [-x, -y, -z, w]])


def oplus(q):
    """operators.hpp:104-112: p * q = oplus(q) p."""
    x, y, z, w = q
    return np.array([[w, z, -y, x], [-z, w, x, y], [y, -x, w, z], [-x, -y, -z, w]])


# sin and cos of the float64 runs that set the bound err by up to LIBM_ULP units in the last place, as CUDA's double
# sin / cos may (CUDA C Programming Guide, mathematical functions: 2 ulp); the long double run is exact to its format.
# (sqrt and division are correctly rounded on both sides.)
LIBM_ULP = 2.0
_libm_rng = [None]


def _sin(x):
    y = np.sin(x)
    return y if _libm_rng[0] is None else y * (1.0 + LIBM_ULP * EPS * _libm_rng[0].uniform(-1.0, 1.0))


def _cos(x):
    y = np.cos(x)
    return y if _libm_rng[0] is None else y * (1.0 + LIBM_ULP * EPS * _libm_rng[0].uniform(-1.0, 1.0))


def sinc(x):
    if abs(x) > 1e-6:
        return _sin(x) / x
    x2 = x * x
    return 1 - x2 / 6 + x2 * x2 / 120 - x2 * x2 * x2 / 5040


def delta_q(a):
    hn = np.sqrt(a @ a) / 2
    return np.concatenate([sinc(hn) * a / 2, [_cos(hn)]])


def right_jacobian(phi):
    P = np.sqrt(phi @ phi)
    X = crossmx(phi)
    X2 = X @ X
    D = phi.dtype.type
    if P < 1e-4:
        return np.eye(3, dtype=D) - X / 2 + X2 / 6
    return np.eye(3, dtype=D) - (1 - _cos(P)) / (P * P) * X + (P - _sin(P)) / (P * P * P) * X2


def cholesky(A):
    """Lower Cholesky factor, column by column (np.linalg has no long double)."""
    n = A.shape[0]
    L = np.zeros_like(A)
    for j in range(n):
        d = A[j, j] - L[j, :j] @ L[j, :j]
        assert d > 0, "matrix is not positive definite at column %d" % j
        L[j, j] = np.sqrt(d)
        L[j + 1:, j] = (A[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return L


def inverse_spd(A):
    """A^-1 = L^-T L^-1, L^-1 by forward substitution on all 15 columns at once."""
    L = cholesky(A)
    n = A.shape[0]
    X = np.zeros_like(A)
    E = np.eye(n, dtype=A.dtype)
    for i in range(n):
        X[i] = (E[i] - L[i, :i] @ X[:i]) / L[i, i]
    return X.T @ X


# ------------------------------------------------------------------------------------------------ the recursion
def integrate(samples, prm, t0, t1, sb, D, preint, want_cov=True, faults=()):
    """The sample loop of redoPreintegration (preint=True, ImuError.cpp:112-264) or of propagation (:327-469).
    Returns None when the samples end before t1, else a dict of the increments, the sub-Jacobians, Delta_t, the step
    count and (want_cov) P_delta."""
    t_ns = samples["t_ns"]
    n = len(samples)
    if not (int(t_ns[-1]) >= t1):
        return None
    gyro, acc = np.asarray(samples["gyro"], D), np.asarray(samples["acc"], D)
    sb = np.asarray(sb, D)
    g_max, a_max = D(prm.g_max), D(prm.a_max)
    sg_c, sa_c, sgw_c, saw_c = D(prm.sigma_g_c), D(prm.sigma_a_c), D(prm.sigma_gw_c), D(prm.sigma_aw_c)
    I3 = np.eye(3, dtype=D)
    Delta_q = np.array([0, 0, 0, 1], D)
    C_int, C_dint = np.zeros((3, 3), D), np.zeros((3, 3), D)
    acc_int, acc_dint = np.zeros(3, D), np.zeros(3, D)
    cross = np.zeros((3, 3), D)
    dalpha, dv, dp = np.zeros((3, 3), D), np.zeros((3, 3), D), np.zeros((3, 3), D)
    P = np.zeros((15, 15), D)
    Delta_t = D(0)
    time = int(t0)
    started = False
    steps = 0
    sat_gt = (lambda x, m: np.any(np.abs(x) >= m)) if "sat_ge" in faults else (lambda x, m: np.any(np.abs(x) > m))
    for it in range(n):
        last = it + 1 == n
        w0, a0 = gyro[it], acc[it]
        w1, a1 = (gyro[it], acc[it]) if last else (gyro[it + 1], acc[it + 1])
        nexttime = int(t1) if last else int(t_ns[it + 1])
        dt = ns_to_sec(nexttime - time, D)
        if t1 < nexttime:
            interval = ns_to_sec(nexttime - int(t_ns[it]), D)
            nexttime = int(t1)
            dt = ns_to_sec(nexttime - time, D)
            r = dt / interval
            if "no_last_interp" not in faults:
                w1, a1 = (1 - r) * w0 + r * w1, (1 - r) * a0 + r * a1
        if dt <= 0:
            continue
        Delta_t += dt
        if not started:
            started = True
            r = dt / ns_to_sec(nexttime - int(t_ns[it]), D)
            if "no_first_interp" not in faults:
                w0, a0 = r * w0 + (1 - r) * w1, r * a0 + (1 - r) * a1
        sigma_g_c, sigma_a_c = sg_c, sa_c
        if sat_gt(w0, g_max) or sat_gt(w1, g_max):
            sigma_g_c = sigma_g_c * 100
        if sat_gt(a0, a_max) or sat_gt(a1, a_max):
            sigma_a_c = sigma_a_c * 100
        om = (w0 + w1) / 2 - sb[3:6]
        th = np.sqrt(om @ om) * dt / 2
        dq = np.concatenate([sinc(th) * om * dt / 2, [_cos(th)]])
        Delta_q1 = qmul(Delta_q, dq)
        C, C1 = q2R(Delta_q), q2R(Delta_q1)
        CC = C + C1
        ac = (a0 + a1) / 2 - sb[6:9]
        C_int1 = C_int + CC * dt / 2
        acc_int1 = acc_int + CC @ ac * dt / 2
        q_dt2 = dt * dt / 2 if "half_dt2" in faults else dt * dt / 4
        C_dint = C_dint + C_int * dt + CC * q_dt2
        add = acc_int * dt + CC @ ac * (dt * dt / 4)
        acc_dint = acc_dint + add
        Jr = right_jacobian(om * dt)
        if preint and "dalpha_without_jr" not in faults:
            dalpha = dalpha + C1 @ Jr * dt
        else:
            dalpha = dalpha + dt * C1
        cross1 = q2R(qinv(dq)) @ cross + Jr * dt
        ax = crossmx(ac)
        sumA = C @ ax @ cross + C1 @ ax @ cross1
        dv1 = dv + dt / 2 * sumA
        F09 = dt * dv + dt * dt / 4 * sumA
        dp = dp + F09
        if want_cov:
            F = np.eye(15, dtype=D)
            F[0:3, 3:6] = -crossmx(add)
            F[0:3, 6:9] = I3 * dt
            F[0:3, 9:12] = F09
            F[0:3, 12:15] = -C_int * dt + CC * (dt * dt / 4)
            F[3:6, 9:12] = -dt * C1
            F[6:9, 3:6] = -crossmx(CC @ ac * dt / 2)
            F[6:9, 9:12] = dt / 2 * sumA
            F[6:9, 12:15] = -CC * dt / 2
            P = F @ P @ F.T
            s2_v = dt * sigma_a_c * (sigma_a_c if preint and "prop_q_in_preint" not in faults else sa_c)
            q = np.repeat([dt * dt / 2 * s2_v, dt * sigma_g_c * sigma_g_c, s2_v, dt * sgw_c * sgw_c, dt * saw_c * saw_c], 3)
            P[np.arange(15), np.arange(15)] += q.astype(D)
        Delta_q, C_int, acc_int, cross, dv = Delta_q1, C_int1, acc_int1, cross1, dv1
        time = nexttime
        steps += 1
        if nexttime == t1:
            break
    return dict(Delta_q=Delta_q, C_integral=C_int, C_doubleintegral=C_dint, acc_integral=acc_int,
                acc_doubleintegral=acc_dint, dalpha_db_g=dalpha, dv_db_g=dv, dp_db_g=dp, Delta_t=Delta_t, steps=steps,
                P=P)


def preintegrate(samples, prm, t0, t1, sb, D, faults=()):
    """redoPreintegration (ImuError.cpp:76-284): the increments at `sb` and sqrt_info = LLT(sym(sym(P)^-1))^T.
    None when the samples end before t1."""
    st = integrate(samples, prm, t0, t1, sb, D, True, True, faults)
    if st is None:
        return None
    P = st["P"] / 2 + st["P"].T / 2
    info = inverse_spd(P)
    info = info / 2 + info.T / 2
    st["sqrt_info"] = cholesky(info).T
    st["sb_ref"] = np.asarray(sb, D).copy()
    return st


def evaluate(samples, prm, t0, t1, pose0, sb0, pose1, sb1, D, cache=None, faults=()):
    """EvaluateWithMinimalJacobians (ImuError.cpp:514-685) with the cache `cache` (None: never preintegrated, as a
    fresh ImuError).  Returns dict(redo, r (15), J (15 x 30: the four minimal Jacobians side by side), S, cache)."""
    pose0, sb0, pose1, sb1 = (np.asarray(x, D) for x in (pose0, sb0, pose1, sb1))
    Delta_t = ns_to_sec(int(t1) - int(t0), D)
    redo = cache is None
    Delta_b = np.zeros(6, D) if redo else sb0[3:9] - cache["sb_ref"][3:9]
    redo = redo or np.sqrt(Delta_b[:3] @ Delta_b[:3]) * Delta_t > 1e-4
    if redo:
        cache = preintegrate(samples, prm, t0, t1, sb0, D, faults)
        Delta_b = np.zeros(6, D)
    q0, q1 = qnormalized(pose0[3:7]), qnormalized(pose1[3:7])
    C_WS0 = q2R(q0)
    C_S0W = C_WS0.T
    g_W = np.array([0, 0, D(prm.g)])
    dp_W = pose0[:3] - pose1[:3] + sb0[:3] * Delta_t - g_W * Delta_t * Delta_t / 2
    dv_W = sb0[:3] - sb1[:3] - g_W * Delta_t
    sgn = 1 if "bias_sign" in faults else -1
    Dq = qmul(delta_q(sgn * cache["dalpha_db_g"] @ Delta_b[:3]), cache["Delta_q"])
    q1i = qconj(q1)
    F0 = np.eye(15, dtype=D)
    F0[0:3, 0:3] = C_S0W
    F0[0:3, 3:6] = C_S0W @ crossmx(dp_W)
    F0[0:3, 6:9] = C_S0W * Delta_t
    F0[0:3, 9:12] = cache["dp_db_g"]
    F0[0:3, 12:15] = -cache["C_doubleintegral"]
    F0[3:6, 3:6] = (plus(qmul(Dq, q1i)) @ oplus(q0))[:3, :3]
    F0[3:6, 9:12] = (oplus(qmul(q1i, q0)) @ oplus(Dq))[:3, :3] @ -cache["dalpha_db_g"]
    F0[6:9, 3:6] = C_S0W @ crossmx(dv_W)
    F0[6:9, 6:9] = C_S0W
    F0[6:9, 9:12] = cache["dv_db_g"]
    F0[6:9, 12:15] = -cache["C_integral"]
    F1 = -np.eye(15, dtype=D)
    F1[0:3, 0:3] = -C_S0W
    F1[3:6, 3:6] = -(plus(Dq) @ oplus(q0) @ plus(q1i))[:3, :3]
    F1[6:9, 6:9] = -C_S0W
    e = np.zeros(15, D)
    e[0:3] = C_S0W @ dp_W + cache["acc_doubleintegral"] + F0[0:3, 9:15] @ Delta_b
    e[3:6] = 2 * qmul(Dq, qmul(q1i, q0))[:3]
    e[6:9] = C_S0W @ dv_W + cache["acc_integral"] + F0[6:9, 9:15] @ Delta_b
    e[9:15] = sb0[3:9] - sb1[3:9]
    S = cache["sqrt_info"]
    return dict(redo=int(bool(redo)), r=S @ e, J=S @ np.hstack([F0, F1]), S=S, cache=cache)


def propagate(samples, prm, t0, t1, pose, sb, D, faults=()):
    """The static ImuError::propagation (:287-504).  Returns dict(n, pose, sb, P, F); n = -1 (pose, sb unchanged, P,
    F zero) when the samples end before t1."""
    pose, sb = np.asarray(pose, D).copy(), np.asarray(sb, D).copy()
    st = integrate(samples, prm, t0, t1, sb, D, False, True, faults)
    if st is None:
        return dict(n=-1, pose=pose, sb=sb, P=np.zeros((15, 15), D), F=np.zeros((15, 15), D))
    q0 = qnormalized(pose[3:7])
    C0 = q2R(q0)
    Dt = st["Delta_t"]
    g_W = np.array([0, 0, D(prm.g)])
    out_pose = np.concatenate([pose[:3] + sb[:3] * Dt + C0 @ st["acc_doubleintegral"] - g_W * Dt * Dt / 2,
                               qnormalized(qmul(q0, st["Delta_q"]))])
    out_sb = sb.copy()
    out_sb[:3] = sb[:3] + C0 @ st["acc_integral"] - g_W * Dt
    F = np.eye(15, dtype=D)
    F[0:3, 3:6] = -crossmx(C0 @ st["acc_doubleintegral"])
    F[0:3, 6:9] = np.eye(3, dtype=D) * Dt
    F[0:3, 9:12] = C0 @ st["dp_db_g"]
    F[0:3, 12:15] = -C0 @ st["C_doubleintegral"]
    F[3:6, 9:12] = -C0 @ st["dalpha_db_g"]
    F[6:9, 3:6] = -crossmx(C0 @ st["acc_integral"])
    F[6:9, 9:12] = C0 @ st["dv_db_g"]
    F[6:9, 12:15] = -C0 @ st["C_integral"]
    T = np.eye(15, dtype=D)
    T[0:3, 0:3] = T[3:6, 3:6] = T[6:9, 6:9] = C0
    return dict(n=st["steps"], pose=out_pose, sb=out_sb, P=T @ st["P"] @ T.T, F=F)


# ------------------------------------------------------------------------------------------------ compared quantities
def eval_quantities(redo, r, J, S):
    """The unique quantities of one evaluation, formed in the precision of the inputs' widest type: redo (exact), the
    information S^T S, the cost, H30 = J^T J and g30 = J^T r (J = [J0 J1 J2 J3], 15 x 30)."""
    D = np.result_type(np.asarray(r).dtype, np.asarray(J).dtype).type
    r, J, S = (np.asarray(x, D) for x in (r, J, S))
    return dict(redo=int(redo), info=S.T @ S, cost=np.array([r @ r / 2]), H30=J.T @ J, g30=J.T @ r)


def prop_quantities(n, pose, sb, P, F):
    pose = np.asarray(pose)
    q = pose[3:7] * (1 if pose[6] >= 0 else -1)       # a quaternion up to its sign
    return dict(n=int(n), p=pose[:3], q=q, v=np.asarray(sb)[:3], bg=np.asarray(sb)[3:6], ba=np.asarray(sb)[6:9],
                P=np.asarray(P), F=np.asarray(F))


def ref_eval_quantities(res):
    return eval_quantities(res["redo"], res["r"], res["J"], res["S"])


def ref_prop_quantities(res):
    return prop_quantities(res["n"], res["pose"], res["sb"], res["P"], res["F"])


def _blocks(x):
    """A quantity's comparison blocks: 3 x 3 blocks of a matrix, 3-vectors of a vector of 3k, else the whole."""
    x = np.asarray(x)
    if x.ndim == 2 and x.shape[0] % 3 == 0 and x.shape[1] % 3 == 0:
        a, b = x.shape[0] // 3, x.shape[1] // 3
        return x.reshape(a, 3, b, 3).transpose(0, 2, 1, 3).reshape(a * b, 9)
    if x.ndim == 1 and x.size % 3 == 0:
        return x.reshape(-1, 3)
    return x.reshape(1, -1)


def block_max(x):
    return np.abs(_blocks(np.asarray(x, LD))).max(axis=1)


# ------------------------------------------------------------------------------------------------ cases and bounds
def _perturb(rng, x, keep=None):
    """x * (1 + u eps), u uniform in [-1, 1]: one rounding of every element (except where `keep`)."""
    x = np.asarray(x, np.float64)
    y = x * (1.0 + EPS * rng.uniform(-1.0, 1.0, x.shape))
    return np.where(keep, x, y) if keep is not None else y


def perturbed_inputs(case, rng):
    """Every floating input of a case perturbed by one rounding.  Sample components that sit exactly on a saturation
    limit or one ulp above it stay exact, so that the branch the case pins is the one every run takes."""
    prm = case["prm"]
    s = case["samples"].copy()
    for key, lim in (("gyro", prm.g_max), ("acc", prm.a_max)):
        a = np.abs(s[key])
        keep = (a == lim) | (a == np.nextafter(lim, np.inf))
        s[key] = _perturb(rng, s[key], keep)
    c = dict(case, samples=s)
    for k in ("pose0", "sb0", "pose1", "sb1", "sb_ref"):
        if case.get(k) is not None:
            c[k] = _perturb(rng, case[k])
    return c


def run_eval(case, D, use_ref, faults=(), cache_from=None):
    """One evaluation of a case in type D.  use_ref: preintegrate at the case's sb_ref first (the correction path,
    or a redo when the bias moved past the threshold); else evaluate a fresh term.  cache_from: preintegrate that
    case's samples / interval instead (the fault `cache of the neighbouring term`)."""
    src = cache_from if cache_from is not None else case
    cache = None
    if use_ref:
        cache = preintegrate(src["samples"], src["prm"], src["t0"], src["t1"], case["sb_ref"], D, faults)
    elif cache_from is not None:
        cache = preintegrate(src["samples"], src["prm"], src["t0"], src["t1"], case["sb0"], D, faults)
    return evaluate(case["samples"], case["prm"], case["t0"], case["t1"], case["pose0"], case["sb0"], case["pose1"],
                    case["sb1"], D, cache, faults)


def run_prop(case, D, faults=()):
    return propagate(case["samples"], case["prm"], case["t0"], case["t1"], case["pose0"], case["sb0"], D, faults)


def reference_and_bounds(case, path, seed=0):
    """The long double quantities of a case and their per-block bounds.  path: 'prop', 'eval' (fresh term) or 'corr'
    (preintegrated at sb_ref first).  delta = the largest deviation of N_RUNS float64 runs on perturbed inputs;
    bound = max(C_MEAS delta, C_FLOOR eps max|x_ref|) per 3 x 3 block / 3-vector."""
    require_long_double()
    if path == "prop":
        run, quant = (lambda c, D: run_prop(c, D)), ref_prop_quantities
    else:
        run, quant = (lambda c, D: run_eval(c, D, path == "corr")), ref_eval_quantities
    ref = quant(run(case, LD))
    rng = np.random.default_rng([seed, 7919])
    delta = {k: np.zeros(len(_blocks(v))) for k, v in ref.items() if not isinstance(v, int)}
    for _ in range(N_RUNS):
        c = perturbed_inputs(case, rng)
        _libm_rng[0] = rng
        try:
            got = quant(run(c, np.float64))
        finally:
            _libm_rng[0] = None
        for k, v in ref.items():
            if isinstance(v, int):
                assert got[k] == v, "%s: a perturbed float64 run takes another branch (%s)" % (case["name"], k)
            else:
                delta[k] = np.maximum(delta[k], np.abs(_blocks(np.asarray(got[k], LD)) - _blocks(v)).max(axis=1))
    bounds = {k: np.maximum(C_MEAS * d.astype(np.float64), C_FLOOR * EPS * block_max(ref[k]).astype(np.float64))
              for k, d in delta.items()}
    return ref, bounds


def compare(got, ref, bounds):
    """Worst ratio |got - ref| / bound over every block of every quantity, and the name of the quantity where it occurs.
    Integers must match, and every element of `got` must be finite: inf otherwise."""
    worst, where = 0.0, None
    for k, v in ref.items():
        if isinstance(v, int):
            if int(got[k]) != v:
                return np.inf, k
            continue
        g = _blocks(np.asarray(got[k], LD))
        if g.shape != _blocks(v).shape or not np.all(np.isfinite(g)):
            return np.inf, k
        err = np.abs(g - _blocks(v)).max(axis=1).astype(np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):      # 0 / 0 where a block and its bound are both 0
            ratio = np.where(err == 0, 0.0, err / bounds[k])
        m = float(np.max(ratio)) if ratio.size else 0.0
        if not np.isfinite(m):
            return np.inf, k
        if m > worst:
            worst, where = m, k
    return worst, where
