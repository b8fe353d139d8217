"""TEST INFRASTRUCTURE ONLY -- CPU restatement of okb_stereo_init_batch: the 2D-2D match of Frontend::matchStereo
(okvis_frontend/src/Frontend.cpp:521-546), one VioKeyframeWindowMatchingAlgorithm Match2D2D match per job with frame
A = frame B:
  setFrames         VioKeyframeWindowMatchingAlgorithm.cpp:76-111
  doSetup           :124-146, 216-232, 256-274 (2D-2D branch), resetFrames ProbabilisticStereoTriangulator.cpp:117-159
  DenseMatcher      oracle.match_hamming_gated (oracle_matcher.hpp / oracle_gate.hpp: Hamming + verifyMatch :304-339)
  setBestMatch      :370-481 up to the landmark bookkeeping: stereoTriangulate (:168-227), getUncertainty (:253-355)
getUncertainty keeps the reference's behaviour: A's Jacobian at the triangulated point, B's residual and Jacobians at
the point moved 20 % towards the baseline centre (parametersB[1] aliases hPA), canBeInitialized = |r_B|^2 >= 4, then
the rank test of H.colPivHouseholderQr() (Eigen's algorithm and rank rule; PARITY UNPINNED, Eigen is not available).
`margins` collects, for every decision taken, its relative distance to the threshold it was compared against."""
import numpy as np

from okvis_b200 import abi
from track_reference import distort, project_homogeneous, q2R

EPS = 2.220446049250313e-16
I7 = np.array([0, 0, 0, 0, 0, 0, 1.0])


class Xf:
    """okvis::kinematics::Transformation: (r, q) with q normalised on construction."""

    def __init__(self, r, q):
        q = np.asarray(q, np.float64)
        self.q = q / np.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
        self.r = np.array(r, np.float64)
        self.C = q2R(self.q)

    def __mul__(self, o):
        return Xf(self.C @ o.r + self.r, qmul(self.q, o.q))

    def inverse(self):
        n2 = self.q[0] * self.q[0] + self.q[1] * self.q[1] + self.q[2] * self.q[2] + self.q[3] * self.q[3]
        return Xf(-(self.C.T @ self.r), np.array([-self.q[0], -self.q[1], -self.q[2], self.q[3]]) / n2)

    def p7(self):
        return np.concatenate([self.r, self.q])


def qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz])


def undistort_gn(cam, d0, d1):
    """The models' Gauss-Newton undistort: 5 iterations, break at chi2 < 1e-15 (success flag ignored)."""
    x0, x1 = d0, d1
    for _ in range(5):
        xt, E, _ = distort(cam, x0, x1)
        e0, e1 = d0 - xt[0], d1 - xt[1]
        a, b, d = E[0] * E[0] + E[2] * E[2], E[0] * E[1] + E[2] * E[3], E[1] * E[1] + E[3] * E[3]
        r0, r1 = E[0] * e0 + E[2] * e1, E[1] * e0 + E[3] * e1
        det = a * d - b * b
        x0 += (d * r0 - b * r1) / det
        x1 += (-b * r0 + a * r1) / det
        if e0 * e0 + e1 * e1 < 1e-15:
            break
    return x0, x1


def back_project(cam, kp):
    """PinholeCamera::backProject: (p - c) * (1 / f), undistort, z = 1."""
    out = np.zeros((len(kp), 3))
    for i, (x, y) in enumerate(kp):
        u = undistort_gn(cam, (x - float(cam["cu"])) * (1.0 / float(cam["fu"])), (y - float(cam["cv"])) * (1.0 / float(cam["fv"])))
        out[i] = [u[0], u[1], 1.0]
    return out


def ray_sigmas(size, f):
    return np.sqrt(np.sqrt(2.0)) * (0.8 * np.asarray(size, np.float64) / 12.0) / f


def _rel(x, thr):
    return abs(x - thr) / max(abs(thr), 1e-300)


def reprojection(cam, pose, hp, z, sqrt_info):
    """ReprojectionError::EvaluateWithMinimalJacobians with fixed identity extrinsics: r, J_pose_min 2x6, J_point_min 2x3."""
    C_WS = q2R(pose[3:])
    w = hp[3]
    p = np.array([hp[0] - pose[0] * w, hp[1] - pose[1] * w, hp[2] - pose[2] * w])
    pc = C_WS.T @ p
    valid = not (abs(w) > 1.0e-8 and pc[2] / w < 0.2)
    ip, Jp, _ = project_homogeneous(cam, np.concatenate([pc, [w]]))
    r = sqrt_info * (np.asarray(z) - ip)
    A = sqrt_info * (Jp @ C_WS.T) if valid else np.zeros((2, 3))
    J0 = np.zeros((2, 6))
    for i in range(2):
        a = A[i]
        J0[i, :3] = w * a
        J0[i, 3:] = [p[1] * a[2] - p[2] * a[1], p[2] * a[0] - p[0] * a[2], p[0] * a[1] - p[1] * a[0]]
    return r, J0, -A


def reproj_err4(cam, kp, size, hp, margins=None):
    ip, _, ok = project_homogeneous(cam, hp)
    if not ok:
        return None
    sd = 0.8 * size / 12.0
    w = 1.0 / (sd * sd)
    d = ip - kp
    return d[0] * (w * d[0]) + d[1] * (w * d[1])


def stereo_triangulate(g, a, b, margins):
    """stereoTriangulate: (valid, hpA, isParallel)."""
    ba, bb = g["bearing_a"][a], g["bearing_b"][b]
    e1 = ba / np.sqrt(ba @ ba)
    eb = g["C_AB"] @ bb
    e2 = eb / np.sqrt(eb @ eb)
    sigma = max(g["rs_a"][a], g["rs_b"][b])
    t12 = g["t_AB"]
    b0, b1 = t12 @ e1, t12 @ e2
    A00, A10, A11 = e1 @ e1, e1 @ e2, -(e2 @ e2)
    A01 = -A10
    if A10 < 0.0:
        A10, A01 = -A10, -A01
    det = A00 * A11 - A01 * A10
    margins.append(("det", _rel(abs(det), 1e-6)))
    if not abs(det) > 1.0e-6:
        parallel = True
        c = np.cross(e1, e2)
        nc = np.sqrt(c @ c)
        margins.append(("6sigma", _rel(nc, 6 * sigma)))
        if not nc < 6 * sigma:
            return False, None, True
        v = np.array([(e1[0] + e2[0]) / 2.0, (e1[1] + e2[1]) / 2.0, (e1[2] + e2[2]) / 2.0, 1e-3])
        hp = v / np.sqrt(v @ v)
    else:
        parallel = False
        i00, i01, i10, i11 = A11 / det, -A01 / det, -A10 / det, A00 / det
        l0, l1 = i00 * b0 + i01 * b1, i10 * b0 + i11 * b1
        xm, xn = l0 * e1, l1 * e2 + t12
        mid = (xm + xn) / 2.0
        err, diff = mid - xm, mid - 0.5 * t12
        chi2 = (err @ err) * (1.0 / ((diff @ diff) * sigma * sigma))
        margins.append(("chi2", _rel(chi2, 9.0)))
        if chi2 > 9:
            return False, None, False
        if diff @ e1 < 0:
            mid = 0.5 * t12 - diff
        n = np.sqrt(mid @ mid + 1.0)
        hp = np.array([mid[0] / n, mid[1] / n, mid[2] / n, 1.0 / n])
    errA = reproj_err4(g["cam_a"], g["kp_a"][a], g["size_a"][a], hp)
    if errA is None:
        return False, None, parallel
    C, t = g["C_AB"], g["t_AB"]
    hpB = np.array([C[:, k] @ hp[:3] - C[:, k] @ t * hp[3] for k in range(3)] + [hp[3]])
    errB = reproj_err4(g["cam_b"], g["kp_b"][b], g["size_b"][b], hpB)
    if errB is None:
        return False, None, parallel
    margins.append(("errA", _rel(errA, 4.0)))
    margins.append(("errB", _rel(errB, 4.0)))
    return not (errA > 4.0 or errB > 4.0), hp, parallel


def _det(g, a, b):
    """|det| of triangulateFast's 2x2 system (1 - cos^2 of the angle between the rays)."""
    ba, bb = g["bearing_a"][a], g["bearing_b"][b]
    e1 = ba / np.sqrt(ba @ ba)
    eb = g["C_AB"] @ bb
    e2 = eb / np.sqrt(eb @ eb)
    c = e1 @ e2
    return abs((e1 @ e1) * -(e2 @ e2) + c * c)


def qr_rank(H, margins=None):
    """Eigen's ColPivHouseholderQR(H).rank(): column pivoting on downdated norms, Householder reflectors, |R_ii| >
    9 eps |max pivot| over the nonzero pivots."""
    n = 9
    M = np.array(H, np.float64, copy=True)
    nu = np.array([np.sqrt(M[:, j] @ M[:, j]) for j in range(n)])
    nd = nu.copy()
    maxn = nd.max()
    thr_helper = (maxn * EPS) * (maxn * EPS) / 9.0
    nonzero, maxpivot = n, 0.0
    for k in range(n):
        p = k + int(np.argmax(nu[k:]))
        if nonzero == n and nu[p] * nu[p] < thr_helper * (n - k):
            nonzero = k
        if p != k:
            M[:, [k, p]] = M[:, [p, k]]
            nu[[k, p]] = nu[[p, k]]
            nd[[k, p]] = nd[[p, k]]
        c0 = M[k, k]
        tail = M[k + 1:, k] @ M[k + 1:, k]
        if tail <= 2.2250738585072014e-308:
            tau, beta = 0.0, c0
            M[k + 1:, k] = 0.0
        else:
            beta = np.sqrt(c0 * c0 + tail)
            if c0 >= 0.0:
                beta = -beta
            M[k + 1:, k] = M[k + 1:, k] / (c0 - beta)
            tau = (beta - c0) / beta
        M[k, k] = beta
        maxpivot = max(maxpivot, abs(beta))
        v = M[k + 1:, k]
        for j in range(k + 1, n):
            w = v @ M[k + 1:, j] + M[k, j]
            M[k, j] -= tau * w
            M[k + 1:, j] -= tau * v * w
            if nu[j] != 0.0:
                t = abs(M[k, j]) / nu[j]
                t = max((1.0 + t) * (1.0 - t), 0.0)
                if t * (nu[j] / nd[j]) ** 2 <= np.sqrt(EPS):
                    nd[j] = nu[j] = np.sqrt(M[k + 1:, j] @ M[k + 1:, j])
                else:
                    nu[j] *= np.sqrt(t)
    thr = maxpivot * (EPS * 9.0)
    diag = np.abs(np.diag(M))[:nonzero]
    if margins is not None:
        margins += [("rank", _rel(d, thr)) for d in diag]
    return int(np.sum(diag > thr))


def prior_H(T_AB):
    """resetFrames: PoseError(T_AB, UOplus^-1) at T_AB, UOplus = diag(4e-8 I3, 1e-8 I3); H_ 9x9 with J^T J in the pose
    block (PoseError.cpp:86-136, sqrt information = sqrt(diag(info)))."""
    S = np.diag([np.sqrt(1.0 / 4e-8)] * 3 + [np.sqrt(1.0 / 1e-8)] * 3)
    q = T_AB.q / np.sqrt(T_AB.q @ T_AB.q)
    qi = np.array([-q[0], -q[1], -q[2], q[3]]) / (q @ q)
    dq = qmul(q, qi)
    dq = dq / np.sqrt(dq @ dq)
    P = np.array([[dq[3], -dq[2], dq[1]], [dq[2], dq[3], -dq[0]], [-dq[1], dq[0], dq[3]]])
    Jm = np.zeros((6, 6))
    Jm[:3, :3] = -np.eye(3)
    Jm[3:, 3:] = -P
    J = S @ Jm
    H = np.zeros((9, 9))
    H[:6, :6] = J.T @ J
    return H


def uncertainty_H(g, a, b, hpA):
    """getUncertainty up to the rank test: (|r_B|^2, H, r_B, JA, JTB, JhB)."""
    sdA, sdB = 0.8 * g["size_a"][a] / 12.0, 0.8 * g["size_b"][b] / 12.0
    _, _, JA = reprojection(g["cam_a"], I7, hpA, g["kp_a"][a], np.sqrt(1.0 / (sdA * sdA)))
    t = g["t_AB"]
    hm = np.concatenate([0.8 * (hpA[:3] - t / 2.0 * hpA[3]) + t / 2.0 * hpA[3], [hpA[3]]])
    rB, JTB, JhB = reprojection(g["cam_b"], g["T_AB"].p7(), hm, g["kp_b"][b], np.sqrt(1.0 / (sdB * sdB)))
    H = g["H_"].copy()
    H[6:, 6:] += JA.T @ JA
    H[:6, :6] += JTB.T @ JTB
    H[:6, 6:] += JTB.T @ JhB
    H[6:, :6] += JhB.T @ JTB
    H[6:, 6:] += JhB.T @ JhB
    return rB @ rB, H, rB, JA, JTB, JhB


def named(state, l):
    l = int(l)
    return l if (0 <= l < len(state["landmarks"]) and bool(np.any(state["landmarks"][l] != 0.0))) else -1


def setup(state, job):
    """setFrames + doSetup (2D-2D): the gate geometry and inputs, skip flags, T_WCa."""
    w = state
    f, ca, cb = job["feat_slot"], job["cam_a"], job["cam_b"]
    P, Ea, Eb = w["poses"][job["pose"]], w["extrinsics"][ca], w["extrinsics"][cb]
    T_WS, T_SCa, T_SCb = Xf(P[:3], P[3:]), Xf(Ea[:3], Ea[3:]), Xf(Eb[:3], Eb[3:])
    T_WCa, T_WCb = T_WS * T_SCa, T_WS * T_SCb
    T_AB = T_WCa.inverse() * T_WCb
    A, B = w["store"][(f, ca)], w["store"][(f, cb)]
    cam_a, cam_b = w["cameras"][ca], w["cameras"][cb]
    g = dict(T_AB=T_AB, C_AB=T_AB.C, t_AB=T_AB.r, T_WCa=T_WCa, cam_a=cam_a, cam_b=cam_b,
             kp_a=A["kp"], kp_b=B["kp"], size_a=A["size"], size_b=B["size"],
             bearing_a=back_project(cam_a, A["kp"]), bearing_b=back_project(cam_b, B["kp"]),
             rs_a=ray_sigmas(A["size"], float(cam_a["fu"])), rs_b=ray_sigmas(B["size"], float(cam_b["fu"])), H_=prior_H(T_AB))

    def skip(e):
        return np.array([1 if (named(w, l) >= 0 and l < len(w["lm_init"]) and w["lm_init"][l]) else 0 for l in e["lm"]], np.uint8)

    g["skipA"], g["skipB"] = skip(A), skip(B)
    return g


def gate_struct(g):
    return abi.make_match_gate(abi.GATE_2D2D, g["kp_b"], g["size_b"], kp_a=g["kp_a"], kp_size_a=g["size_a"],
                               bearing_a=g["bearing_a"], bearing_b=g["bearing_b"], ray_sigma_a=g["rs_a"], ray_sigma_b=g["rs_b"],
                               cam_a=g["cam_a"], cam_b=g["cam_b"], T_AB=g["T_AB"].p7())


def stereo_init(oracle, state, job, threshold=60.0, num_best=4, margins=None, cases=None, dets=None):
    """One job: the records [(kp_a, kp_b, lm_slot_a, lm_slot_b, can_be_initialized, hp_W[4])] in setBestMatch order.
    `cases` (list) receives the branch each winner took, `dets` triangulateFast's determinant of each record."""
    margins = [] if margins is None else margins
    g = setup(state, job)
    A, B = state["store"][(job["feat_slot"], job["cam_a"])], state["store"][(job["feat_slot"], job["cam_b"])]
    out = []
    if not (len(A["lm"]) and len(B["lm"])):
        return out, g
    res = oracle.match_hamming_gated(A["desc"], B["desc"], gate_struct(g), g["skipA"], g["skipB"], threshold=threshold,
                                     num_best=num_best)
    for b, (a, dist) in enumerate(zip(res["pairs"]["index_a"].tolist(), res["pairs"]["distance"].tolist())):
        if a < 0 or not dist < threshold:
            continue
        la, lb = named(state, A["lm"][a]), named(state, B["lm"][b])
        if la >= 0 and lb >= 0:
            cases is not None and cases.append("both_named")
            continue
        valid, hp, parallel = stereo_triangulate(g, a, b, margins)
        if not valid:
            cases is not None and cases.append("invalid")
            continue
        cbi = not parallel
        case = "parallel"
        if cbi:
            r2, H, *_ = uncertainty_H(g, a, b, hp)
            margins.append(("rB", _rel(r2, 4.0)))
            cbi = r2 >= 4.0
            case = "close_residual"
            if cbi:
                cbi = qr_rank(H, margins) == 9
                case = "initialised" if cbi else "rank_deficient"
        cases is not None and cases.append(case + ("_a_named" if la >= 0 else "_b_named" if lb >= 0 else ""))
        C, r = g["T_WCa"].C, g["T_WCa"].r
        hpW = np.concatenate([C @ hp[:3] + r * hp[3], [hp[3]]])
        out.append((a, b, la, lb, int(cbi), hpW))
        if dets is not None:
            dets.append(_det(g, a, b))
    return out, g
