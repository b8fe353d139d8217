"""TEST INFRASTRUCTURE ONLY -- CPU restatement of okb_track_3d2d_batch: the 3D-2D rounds of Frontend::matchToKeyframes
(okvis_frontend/src/Frontend.cpp:389-411) and matchToLastFrame (:484-494), one VioKeyframeWindowMatchingAlgorithm match
per round:
  doSetup           VioKeyframeWindowMatchingAlgorithm.cpp:122-215 (A keypoints), 238-255 (skipB)
  DenseMatcher      oracle.match_hamming_gated (oracle_matcher.hpp / oracle_gate.hpp: Hamming + verifyMatch :304-339)
  setBestMatch      :483-526, 3D-2D branch
Sequential in the reference's order: rounds in list order, A keypoints ascending in doSetup, B ascending in the
setBestMatch callbacks.  The state (TrackState) is what the device keeps: the window's landmark estimates, poses,
speed/bias blocks, extrinsics, cameras and observation list, and the feature store with the initialised flags."""
import numpy as np

from okvis_b200 import abi


def q2R(q):
    """Rotation matrix of a quaternion [x, y, z, w], no normalisation (okb_math.cuh q2R, Eigen toRotationMatrix)."""
    x, y, z, w = q
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return np.array([[1 - (tyy + tzz), txy - twz, txz + twy],
                     [txy + twz, 1 - (txx + tzz), tyz - twx],
                     [txz - twy, tyz + twx, 1 - (txx + tyy)]])


def T_CW(pose, ext):
    """Camera-from-world rotation / translation of (T_WS pose, T_SC ext): (T_WS T_SC)^-1."""
    C_WS, C_SC = q2R(pose[3:]), q2R(ext[3:])
    C_CS, C_SW = C_SC.T, C_WS.T
    R = C_CS @ C_SW
    t = -(C_CS @ (C_SW @ pose[:3])) - C_CS @ ext[:3]
    return R, t


def distort(cam, u0, u1):
    """Distortion of the normalised point and its 2x2 Jacobian (the four Distortion headers of okvis_cv); ok = False where
    RadialTangentialDistortion8::distort fails."""
    model, k = int(cam["model"]), cam["dist"]
    if model == abi.DIST_RADTAN:
        k1, k2, p1, p2 = k[:4]
        mx, my, mxy = u0 * u0, u1 * u1, u0 * u1
        rho = mx + my
        rad = k1 * rho + k2 * rho * rho
        d = (u0 + u0 * rad + 2.0 * p1 * mxy + p2 * (rho + 2.0 * mx), u1 + u1 * rad + 2.0 * p2 * mxy + p1 * (rho + 2.0 * my))
        J00 = 1 + rad + k1 * 2.0 * mx + k2 * rho * 4 * mx + 2.0 * p1 * u1 + 6 * p2 * u0
        J01 = k1 * 2.0 * u0 * u1 + k2 * 4 * rho * u0 * u1 + p1 * 2.0 * u0 + 2.0 * p2 * u1
        J11 = 1 + rad + k1 * 2.0 * my + k2 * rho * 4 * my + 6 * p1 * u1 + 2.0 * p2 * u0
        return d, (J00, J01, J01, J11), True
    if model == abi.DIST_EQUIDISTANT:
        k1, k2, k3, k4 = k[:4]
        r2 = u0 * u0 + u1 * u1
        r = np.sqrt(r2)
        th = np.arctan(r)
        th2 = th * th
        th4, th6, th8 = th2 * th2, th2 * th2 * th2, th2 * th2 * th2 * th2
        poly = 1 + k1 * th2 + k2 * th4 + k3 * th6 + k4 * th8
        thd = th * poly
        if r > 1e-8:
            s = thd / r
            dpoly = 2 * k1 * th + 4 * k2 * th2 * th + 6 * k3 * th4 * th + 8 * k4 * th6 * th
            dthd = (poly + th * dpoly) / (1.0 + r2)
            spr = (dthd * r - thd) / (r2 * r)
            J = (s + spr * u0 * u0, spr * u0 * u1, spr * u0 * u1, s + spr * u1 * u1)
        else:
            s, J = 1.0, (1.0, 0.0, 0.0, 1.0)
        return (s * u0, s * u1), J, True
    if model == abi.DIST_RADTAN8:
        k1, k2, p1, p2, k3, k4, k5, k6 = k[:8]
        mx, my, mxy = u0 * u0, u1 * u1, u0 * u1
        rho = mx + my
        if rho > 9.0:
            return (0.0, 0.0), (0.0, 0.0, 0.0, 0.0), False
        num = 1.0 + ((k3 * rho + k2) * rho + k1) * rho
        den = 1.0 + ((k6 * rho + k5) * rho + k4) * rho
        rad = num / den
        d = (u0 * rad + 2.0 * p1 * mxy + p2 * (rho + 2.0 * mx), u1 * rad + 2.0 * p2 * mxy + p1 * (rho + 2.0 * my))
        dnum = (3 * k3 * rho + 2 * k2) * rho + k1
        dden = (3 * k6 * rho + 2 * k5) * rho + k4
        drad = (dnum * den - num * dden) / (den * den)
        J00 = rad + 2 * u0 * u0 * drad + 2.0 * p1 * u1 + 6.0 * p2 * u0
        J01 = 2 * u0 * u1 * drad + 2.0 * p1 * u0 + 2.0 * p2 * u1
        J11 = rad + 2 * u1 * u1 * drad + 6.0 * p1 * u1 + 2.0 * p2 * u0
        return d, (J00, J01, J01, J11), True
    return (u0, u1), (1.0, 0.0, 0.0, 1.0), True


def project_homogeneous(cam, hp_C):
    """PinholeCamera::projectHomogeneous with the point Jacobian (PinholeCamera.hpp(impl):148-226, 358-378): the image
    point, the 2x3 Jacobian of project() (the homogeneous column is zero) and whether the status is Successful."""
    p = np.array(hp_C[:3], dtype=np.float64)
    if hp_C[3] < 0:
        p = -p
    if abs(p[2]) < 1.0e-12:
        return np.zeros(2), np.zeros((2, 3)), False
    rz = 1.0 / p[2]
    u0, u1 = p[0] * rz, p[1] * rz
    d, Jd, ok = distort(cam, u0, u1)
    fu, fv = float(cam["fu"]), float(cam["fv"])
    rz2 = rz * rz
    J = np.array([[fu * Jd[0] * rz, fu * Jd[1] * rz, -fu * (p[0] * Jd[0] + p[1] * Jd[1]) * rz2],
                  [fv * Jd[2] * rz, fv * Jd[3] * rz, -fv * (p[0] * Jd[2] + p[1] * Jd[3]) * rz2]])
    ip = np.array([fu * d[0] + float(cam["cu"]), fv * d[1] + float(cam["cv"])])
    ok = ok and not (ip[0] < 0.0 or ip[1] < 0.0 or ip[0] >= cam["width"] or ip[1] >= cam["height"]) and p[2] > 0.0
    return ip, J, ok


class TrackState:
    """The window and its feature store.  store[(feat_slot, cam)] = dict(kp [n][2], size [n], desc [n][D] uint8,
    lm [n] int32 (-1: none), observed [n] uint8); lm_init [lm_cap] uint8."""

    def __init__(self, window, store, lm_init):
        self.w = window
        self.lm = np.array(window.landmarks, dtype=np.float64, copy=True)
        self.store = {k: {f: np.array(v, copy=True) for f, v in d.items()} for k, d in store.items()}
        self.lm_init = np.array(lm_init, dtype=np.uint8, copy=True)
        self.counts = np.bincount(np.asarray(window.obs["lm_idx"], dtype=np.int64), minlength=len(self.lm))

    def live(self, l):
        return 0 <= l < len(self.lm) and bool(np.any(self.lm[l] != 0.0))

    def initialised(self, l):
        return 0 <= l < len(self.lm_init) and bool(self.lm_init[l])


def uoplus_scale(state, sb_b, same_frame):
    """Top-left diagonal of UOplus (:127-142)."""
    if sb_b >= 0 and not same_frame:
        v = state.w.speed_bias[sb_b][:3]
        scale = max(1.0, float(np.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])))
        return (scale * scale) * 1.0e-2
    return 4e-8


def setup_round(state, pose_b, sb_b, feat_b, feat_a, cam_a, cam_b):
    """doSetup: skipA, projectionsIntoB_ [nA][2], their uncertainties [nA][4] (2x2 row-major), skipB, and the landmark
    slots set to uninitialised, in order.  Clears those flags in `state`."""
    A, B = state.store[(feat_a, cam_a)], state.store[(feat_b, cam_b)]
    nA, nB = len(A["lm"]), len(B["lm"])
    s = uoplus_scale(state, sb_b, feat_a == feat_b)
    R, t = T_CW(state.w.poses[pose_b], state.w.extrinsics[cam_b])
    cam = state.w.cameras[cam_b]
    skipA = np.ones(nA, np.uint8)
    proj = np.zeros((nA, 2))
    unc = np.zeros((nA, 4))
    uninit = []
    for k in range(nA):
        l = int(A["lm"][k])
        if not state.live(l):                       # 1. no landmark / not added
            continue
        if not state.initialised(l):                # 2. not initialised
            continue
        X = state.lm[l]
        hp = np.concatenate([R @ X[:3] + t * X[3], [X[3]]])
        ip, J, ok = project_homogeneous(cam, hp)    # 3. projection status
        if not ok:
            continue
        if state.counts[l] < 2:                     # 4. fewer than 2 observations: uninitialised, after the projection
            state.lm_init[l] = 0
            uninit.append(l)
            continue
        skipA[k] = 0                                # 5. projection and J P_C J^T, P_C = s I3
        proj[k] = ip
        sJ = s * J
        unc[k] = [sJ[0] @ J[0], sJ[0] @ J[1], sJ[1] @ J[0], sJ[1] @ J[1]]
    skipB = np.array([1 if (B["observed"][b] and state.live(int(B["lm"][b]))) else 0 for b in range(nB)], np.uint8)
    return dict(skipA=skipA, proj=proj, unc=unc, skipB=skipB, uninit=uninit, scale=s)


def set_best_match(state, setup, feat_b, cam_b, feat_a, cam_a, a, b):
    """setBestMatch, 3D-2D (:483-526): None (rejected) or (landmark slot, uncertain)."""
    A, B = state.store[(feat_a, cam_a)], state.store[(feat_b, cam_b)]
    sd = 0.8 * float(B["size"][b]) / 12.0
    P = setup["unc"][a]
    U = np.array([[sd * sd + P[0], P[1]], [P[2], sd * sd + P[3]]])
    e = setup["proj"][a] - B["kp"][b]
    invdet = 1.0 / (U[0, 0] * U[1, 1] - U[1, 0] * U[0, 1])
    i00, i10, i01, i11 = U[1, 1] * invdet, -U[1, 0] * invdet, -U[0, 1] * invdet, U[0, 0] * invdet
    r0, r1 = e[0] * i00 + e[1] * i10, e[0] * i01 + e[1] * i11
    chi2 = r0 * e[0] + r1 * e[1]
    if chi2 > 4.0:
        return None
    nrm = np.sqrt(U[0, 0] * U[0, 0] + U[1, 0] * U[1, 0] + U[0, 1] * U[0, 1] + U[1, 1] * U[1, 1])
    return int(A["lm"][a]), int(nrm > 25.0 / (sd * sd * np.sqrt(2.0)))


def track(oracle, state, pose_b, sb_b, feat_b, rounds, threshold=60.0, num_best=4, keep_setups=False):
    """The rounds of one job, in order.  Mutates `state` (B's store entries, counts, initialised flags) and returns
    dict(assoc [(round, cam_b, kp_b, lm_slot, uncertain)], num_matches, num_uncertain, uninit[, setups])."""
    assoc, nm, nu, uninit, setups = [], [], [], [], []
    for r, (feat_a, cam_a, cam_b) in enumerate(rounds):
        su = setup_round(state, pose_b, sb_b, feat_b, feat_a, cam_a, cam_b)
        uninit += su["uninit"]
        A, B = state.store[(feat_a, cam_a)], state.store[(feat_b, cam_b)]
        m = u = 0
        if len(A["lm"]) and len(B["lm"]):
            gate = abi.make_match_gate(abi.GATE_3D2D, B["kp"], B["size"], proj_into_b=su["proj"], proj_uncertainty=su["unc"])
            res = oracle.match_hamming_gated(A["desc"], B["desc"], gate, su["skipA"], su["skipB"], threshold=threshold,
                                             num_best=num_best)
            for b, (a, dist) in enumerate(zip(res["pairs"]["index_a"].tolist(), res["pairs"]["distance"].tolist())):
                if a < 0 or not dist < threshold:
                    continue
                out = set_best_match(state, su, feat_b, cam_b, feat_a, cam_a, a, b)
                if out is None:
                    continue
                l, unc = out
                B["lm"][b] = l
                B["observed"][b] = 1
                state.counts[l] += 1
                assoc.append((r, cam_b, b, l, unc))
                m += 1
                u += unc
        nm.append(m)
        nu.append(u)
        if keep_setups:
            setups.append(su)
    out = dict(assoc=assoc, num_matches=nm, num_uncertain=nu, uninit=uninit)
    if keep_setups:
        out["setups"] = setups
    return out
