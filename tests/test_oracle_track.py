"""CPU checks of the 3D-2D tracking reference (tests/track_reference.py), which the GPU tests hold okb_track_3d2d_batch
to: its projections against the oracle's reprojection functor, its associations against a replay of the gated matcher
fed those independent projections, and one case per rule of doSetup / setBestMatch."""
import numpy as np
import pytest

import track_reference as tr
from okvis_b200 import abi
from track_scene import make_track_scene

MODELS = [abi.DIST_NONE, abi.DIST_RADTAN, abi.DIST_EQUIDISTANT, abi.DIST_RADTAN8]


def _small(seed, model=abi.DIST_RADTAN, **kw):
    return make_track_scene(seed, n_kp=200, distortion=model, n_frames=6, n_landmarks=400, **kw)


def _state(sc):
    return tr.TrackState(sc["window"], sc["store"], sc["lm_init"])


def _independent(oracle, state, sc, feat_a, cam_a, cam_b, skipA):
    """projectionsIntoB_ and J P_C J^T from the oracle's ReprojectionError (z = 0, sqrt_info = 1: r = -p, J_lm = -dp/dp_C C_CW)."""
    w = sc["window"]
    A = state.store[(feat_a, cam_a)]
    ks = np.nonzero(skipA == 0)[0]
    lms = state.lm[A["lm"][ks]]
    n = len(ks)
    r, _, J1, _ = oracle.eval_reprojection(w.cameras[cam_b], np.tile(w.poses[sc["pose_b"]], (n, 1)), lms,
                                           np.tile(w.extrinsics[cam_b], (n, 1)), np.zeros((n, 2)), np.ones(n))
    R, _ = tr.T_CW(w.poses[sc["pose_b"]], w.extrinsics[cam_b])
    Jp = -J1 @ R                       # dp/dp_C (C_CW orthonormal)
    s = tr.uoplus_scale(state, sc["sb_b"], feat_a == sc["feat_b"])
    unc = s * np.einsum("nik,njk->nij", Jp, Jp).reshape(n, 4)
    return ks, -r, unc


@pytest.mark.parametrize("model", MODELS)
def test_projections_match_oracle_functor(oracle, model):
    sc = _small(1, model)
    st = _state(sc)
    rounds = sc["rounds"]["keyframes"] + sc["rounds"]["stereo"]
    out = tr.track(oracle, st, sc["pose_b"], sc["sb_b"], sc["feat_b"], rounds, keep_setups=True)
    assert sum(out["num_matches"]) > 50
    replay = _state(sc)
    n_checked = 0
    for (fa, ca, cb), su in zip(rounds, out["setups"]):
        ks, proj, unc = _independent(oracle, replay, sc, fa, ca, cb, su["skipA"])
        assert np.allclose(su["proj"][ks], proj, rtol=1e-9, atol=0)
        assert np.allclose(su["unc"][ks], unc, rtol=1e-9, atol=1e-300)
        n_checked += len(ks)
        # the same round replayed through the gated matcher on the independent arrays gives the same associations
        A, B = replay.store[(fa, ca)], replay.store[(sc["feat_b"], cb)]
        p, u = np.zeros_like(su["proj"]), np.zeros_like(su["unc"])
        p[ks], u[ks] = proj, unc
        gate = abi.make_match_gate(abi.GATE_3D2D, B["kp"], B["size"], proj_into_b=p, proj_uncertainty=u)
        res = oracle.match_hamming_gated(A["desc"], B["desc"], gate, su["skipA"], su["skipB"], threshold=60.0, num_best=4)
        su2 = dict(proj=p, unc=u)
        for b, (a, d) in enumerate(zip(res["pairs"]["index_a"].tolist(), res["pairs"]["distance"].tolist())):
            if a >= 0 and d < 60.0:
                m = tr.set_best_match(replay, su2, sc["feat_b"], cb, fa, ca, a, b)
                if m is not None:
                    B["lm"][b], B["observed"][b] = m[0], 1
                    replay.counts[m[0]] += 1
        for l in su["uninit"]:
            replay.lm_init[l] = 0
    assert n_checked > 100
    B0 = st.store[(sc["feat_b"], 0)]
    assert np.array_equal(B0["lm"], replay.store[(sc["feat_b"], 0)]["lm"])


def test_no_distractor_accepted_and_truth_recovered(oracle):
    sc = _small(2)
    st = _state(sc)
    out = tr.track(oracle, st, sc["pose_b"], sc["sb_b"], sc["feat_b"], sc["rounds"]["keyframes"])
    truth = {c: sc["store"][(sc["feat_b"], c)]["truth"] for c in range(2)}
    good = 0
    for r, cb, b, l, _ in out["assoc"]:
        assert truth[cb][b] == l, "a keypoint was associated with a landmark it does not observe"
        good += 1
    assert good > 50


def test_skip_rules_and_flag_clearing(oracle):
    sc = _small(3, uninit_fraction=0.0, dead_fraction=0.0)
    st = _state(sc)
    fa, ca, cb = sc["rounds"]["keyframes"][0]
    A = st.store[(fa, ca)]
    ks = np.nonzero(A["lm"] >= 0)[0]
    k_none, k_dead, k_uninit, k_behind, k_few, k_neg = ks[:6]
    A["lm"][k_none] = -1
    st.lm[A["lm"][k_dead]] = 0.0                               # not in the graph
    st.lm_init[A["lm"][k_uninit]] = 0
    l_b, l_f = A["lm"][k_behind], A["lm"][k_few]
    R, t = tr.T_CW(sc["window"].poses[sc["pose_b"]], sc["window"].extrinsics[cb])
    p_C = R @ st.lm[l_b][:3] / st.lm[l_b][3] + t
    st.lm[l_b] = np.concatenate([R.T @ (np.array([p_C[0], p_C[1], -abs(p_C[2])]) - t), [1.0]])   # behind camera B
    st.counts = np.maximum(st.counts, 2)
    st.counts[l_b] = 1                                         # few observations, but the projection fails first
    st.counts[l_f] = 1
    l_n = A["lm"][k_neg]
    ref_neg = tr.setup_round(_state(sc), sc["pose_b"], sc["sb_b"], sc["feat_b"], fa, ca, cb)
    st.lm[l_n] = -st.lm[l_n]                                   # the same point with w < 0
    su = tr.setup_round(st, sc["pose_b"], sc["sb_b"], sc["feat_b"], fa, ca, cb)
    for k in (k_none, k_dead, k_uninit, k_behind, k_few):
        assert su["skipA"][k] == 1
    assert su["uninit"] == [l_f] and st.lm_init[l_f] == 0 and st.lm_init[l_b] == 1
    assert su["skipA"][k_neg] == 0
    assert np.allclose(su["proj"][k_neg], ref_neg["proj"][k_neg], rtol=1e-12)
    assert np.allclose(su["unc"][k_neg], ref_neg["unc"][k_neg], rtol=1e-12)


def test_skipB_and_same_frame_variance(oracle):
    sc = _small(4)
    st = _state(sc)
    fb = sc["feat_b"]
    assert tr.uoplus_scale(st, sc["sb_b"], True) == 4e-8
    assert tr.uoplus_scale(st, -1, False) == 4e-8
    v = sc["window"].speed_bias[sc["sb_b"]][:3]
    assert tr.uoplus_scale(st, sc["sb_b"], False) == max(1.0, np.linalg.norm(v)) ** 2 * 1e-2
    B = st.store[(fb, 0)]
    l_live = int(st.store[sc["rounds"]["keyframes"][0][:2]]["lm"].max())
    B["lm"][:3] = l_live
    B["observed"][:3] = [1, 0, 1]
    su = tr.setup_round(st, sc["pose_b"], sc["sb_b"], fb, *sc["rounds"]["keyframes"][0])
    assert list(su["skipB"][:3]) == [1, 0, 1]


def test_int_truncated_gate_and_uncertain_matches(oracle):
    """verifyMatch truncates chi2 to int (a chi2 in [4, 5) fails like 4.0); setBestMatch rejects chi2 > 4 in double and
    counts, but keeps, a match whose image uncertainty saturates."""
    kp_b = np.array([[100.0, 100.0], [200.0, 200.0], [300.0, 300.0]])
    size_b = np.array([12.0, 12.0, 12.0])
    sd2 = (0.8 * 12.0 / 12.0) ** 2
    proj = np.array([[100.0 + np.sqrt(3.99 * sd2), 100.0], [200.0 + np.sqrt(4.5 * sd2), 200.0], [300.5, 300.0]])
    unc = np.array([[0, 0, 0, 0], [0, 0, 0, 0], [50.0, 0, 0, 50.0]], np.float64)
    A = np.zeros((3, 48), np.uint8)
    gate = abi.make_match_gate(abi.GATE_3D2D, kp_b, size_b, proj_into_b=proj, proj_uncertainty=unc)
    res = oracle.match_hamming_gated(A, A.copy(), gate, threshold=60.0, num_best=4)
    assert res["pairs"]["index_a"].tolist() == [0, -1, 2]
    st = tr.TrackState.__new__(tr.TrackState)
    st.store = {(0, 0): dict(lm=np.array([5, 6, 7])), (1, 0): dict(kp=kp_b, size=size_b)}
    su = dict(proj=proj, unc=unc)
    assert tr.set_best_match(st, su, 1, 0, 0, 0, 0, 0) == (5, 0)
    assert tr.set_best_match(st, su, 1, 0, 0, 0, 1, 1) is None
    assert tr.set_best_match(st, su, 1, 0, 0, 0, 2, 2) == (7, 1)


def test_landmark_associated_twice_across_rounds(oracle):
    """Two keyframes' keypoints of one landmark can each claim a keypoint of B's same camera in different rounds; both
    associations are reported (the reference does not stop it; the host's one-observation rule decides)."""
    sc = _small(5)
    st = _state(sc)
    fb = sc["feat_b"]
    B = st.store[(fb, 0)]
    truth = sc["store"][(fb, 0)]["truth"]
    (fa1, ca1, _), (fa2, ca2, _) = sc["rounds"]["keyframes"][0], sc["rounds"]["keyframes"][2]
    A1, A2 = st.store[(fa1, ca1)], st.store[(fa2, ca2)]
    common = sorted(l for l in set(A1["lm"].tolist()) & set(A2["lm"].tolist()) & set(truth.tolist()) if l >= 0 and st.lm_init[l])
    dup = [int(np.nonzero(truth == l)[0][0]) for l in common[:20]]
    B["kp"] = np.concatenate([B["kp"], B["kp"][dup] + 0.05])          # a second keypoint on the same spot
    for f in ("size", "desc", "lm", "observed", "truth"):
        B[f] = np.concatenate([B[f], B[f][dup]])
    out = tr.track(oracle, st, sc["pose_b"], sc["sb_b"], fb, [(fa1, ca1, 0), (fa2, ca2, 0)])
    per_lm = {}
    for r, cb, b, l, _ in out["assoc"]:
        per_lm.setdefault(l, []).append((r, b))
    twice = [v for v in per_lm.values() if len(v) == 2]
    assert twice and all(v[0][0] == 0 and v[1][0] == 1 and v[0][1] != v[1][1] for v in twice)
