"""TEST INFRASTRUCTURE ONLY -- CPU restatement of okb_match2d2d_batch: one VioKeyframeWindowMatchingAlgorithm Match2D2D
round of Frontend::matchToKeyframes (okvis_frontend/src/Frontend.cpp:413-452) or matchToLastFrame (:499-509),
setFrames(olderFrameId, currentFrameId, im, im) with usePoseUncertainty = false.  It is tests/stereo_init_reference.py
with what differs between the two:
  setFrames   two poses: T_WCa = T_WSa T_SCa, T_WCb = T_WSb T_SCb (VioKeyframeWindowMatchingAlgorithm.cpp:76-111), and
              A's keypoints from A's feature slot
  doSetup     UOplus = diag(u I3, 1e-8 I3) (:127-142), u = max(1, |v_current|)^2 1e-2 when the current frame is in the
              IMU window and A != B, else 4e-8; resetFrames' prior H_ from it
Everything after that -- skip flags, the gated match, stereoTriangulate, getUncertainty and its rank test -- is the
stereo restatement's, called unchanged."""
import numpy as np

import stereo_init_reference as sref
from stereo_init_reference import Xf, back_project, ray_sigmas, qmul, named


def uoplus_t(state, job):
    """The translation variance u of doSetup's UOplus."""
    if job.get("sb_current", -1) >= 0 and job["feat_slot_a"] != job["feat_slot_b"]:
        v = state["speed_bias"][job["sb_current"]][:3]
        scale = max(1.0, float(np.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])))
        return (scale * scale) * 1.0e-2
    return 4e-8


def prior_H(T_AB, u):
    """resetFrames: PoseError(T_AB, UOplus^-1) at T_AB with UOplus = diag(u I3, 1e-8 I3); H_ 9x9, J^T J in the pose
    block.  prior_H(T_AB, 4e-8) is the stereo restatement's prior_H(T_AB)."""
    S = np.diag([np.sqrt(1.0 / u)] * 3 + [np.sqrt(1.0 / 1e-8)] * 3)
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


def setup(state, job):
    """setFrames + doSetup (2D-2D) for frames A and B: the gate geometry and inputs, skip flags, T_WCa."""
    w = state
    ca, cb = job["cam_a"], job["cam_b"]
    Pa, Pb = w["poses"][job["pose_a"]], w["poses"][job["pose_b"]]
    Ea, Eb = w["extrinsics"][ca], w["extrinsics"][cb]
    T_WCa = Xf(Pa[:3], Pa[3:]) * Xf(Ea[:3], Ea[3:])
    T_WCb = Xf(Pb[:3], Pb[3:]) * Xf(Eb[:3], Eb[3:])
    T_AB = T_WCa.inverse() * T_WCb
    A, B = w["store"][(job["feat_slot_a"], ca)], w["store"][(job["feat_slot_b"], cb)]
    cam_a, cam_b = w["cameras"][ca], w["cameras"][cb]
    g = dict(T_AB=T_AB, C_AB=T_AB.C, t_AB=T_AB.r, T_WCa=T_WCa, cam_a=cam_a, cam_b=cam_b,
             kp_a=A["kp"], kp_b=B["kp"], size_a=A["size"], size_b=B["size"],
             bearing_a=back_project(cam_a, A["kp"]), bearing_b=back_project(cam_b, B["kp"]),
             rs_a=ray_sigmas(A["size"], float(cam_a["fu"])), rs_b=ray_sigmas(B["size"], float(cam_b["fu"])),
             u=uoplus_t(state, job), H_=prior_H(T_AB, uoplus_t(state, job)))

    def skip(e):
        return np.array([1 if (named(w, l) >= 0 and l < len(w["lm_init"]) and w["lm_init"][l]) else 0 for l in e["lm"]], np.uint8)

    g["skipA"], g["skipB"] = skip(A), skip(B)
    return g


def match2d2d(oracle, state, job, threshold=60.0, num_best=4, margins=None, cases=None, dets=None):
    """One job: the records [(kp_a, kp_b, lm_slot_a, lm_slot_b, can_be_initialized, hp_W[4])] in setBestMatch order,
    and the setup.  `cases` receives the branch each winner took, `dets` triangulateFast's determinant per record."""
    margins = [] if margins is None else margins
    g = setup(state, job)
    A, B = state["store"][(job["feat_slot_a"], job["cam_a"])], state["store"][(job["feat_slot_b"], job["cam_b"])]
    out = []
    if not (len(A["lm"]) and len(B["lm"])):
        return out, g
    res = oracle.match_hamming_gated(A["desc"], B["desc"], sref.gate_struct(g), g["skipA"], g["skipB"], threshold=threshold,
                                     num_best=num_best)
    for b, (a, dist) in enumerate(zip(res["pairs"]["index_a"].tolist(), res["pairs"]["distance"].tolist())):
        if a < 0 or not dist < threshold:
            continue
        la, lb = named(state, A["lm"][a]), named(state, B["lm"][b])
        if la >= 0 and lb >= 0:
            cases is not None and cases.append("both_named")
            continue
        valid, hp, parallel = sref.stereo_triangulate(g, a, b, margins)
        if not valid:
            cases is not None and cases.append("invalid")
            continue
        cbi = not parallel
        case = "parallel"
        if cbi:
            r2, H, *_ = sref.uncertainty_H(g, a, b, hp)
            margins.append(("rB", sref._rel(r2, 4.0)))
            cbi = r2 >= 4.0
            case = "close_residual"
            if cbi:
                cbi = sref.qr_rank(H, margins) == 9
                case = "initialised" if cbi else "rank_deficient"
        cases is not None and cases.append(case + ("_a_named" if la >= 0 else "_b_named" if lb >= 0 else ""))
        C, r = g["T_WCa"].C, g["T_WCa"].r
        out.append((a, b, la, lb, int(cbi), np.concatenate([C @ hp[:3] + r * hp[3], [hp[3]]])))
        if dets is not None:
            dets.append(sref._det(g, a, b))
    return out, g
