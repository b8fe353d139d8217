"""CPU: the restatement of okb_stereo_init_batch (tests/stereo_init_reference.py) against the oracle's gate
(stereoTriangulate inside verifyMatch) and reprojection functor, getUncertainty's H against central differences of the
residuals, the rank rule against numpy.linalg.matrix_rank, and the triangulated points against the scene's truth, on
seeded scenes of all four distortion models."""
import numpy as np
import pytest

import stereo_init_reference as ref
from okvis_b200 import abi
from stereo_scene import MIN_MARGIN, make_stereo_scene

_MODELS = [abi.DIST_RADTAN, abi.DIST_EQUIDISTANT, abi.DIST_NONE, abi.DIST_RADTAN8]
_SCENES = {}


def scene(oracle, i):
    if i not in _SCENES:
        _SCENES[i] = make_stereo_scene(i, _MODELS[i], oracle=oracle)
    return _SCENES[i]


@pytest.mark.parametrize("i", range(4))
def test_every_branch_and_no_decision_near_a_threshold(oracle, i):
    sc = scene(oracle, i)
    assert min(m for _, m in sc["margins"]) > MIN_MARGIN
    for case in ("both_named", "parallel", "close_residual", "initialised", "rank_deficient"):
        assert case in sc["cases"], case
    assert any(c.endswith("_a_named") for c in sc["cases"]) and any(c.endswith("_b_named") for c in sc["cases"])
    # the A keypoints naming an initialised landmark are skipped, the border pair fails the reprojection check
    g = ref.setup(sc["state"], sc["job"])
    assert g["skipA"].sum() >= 8
    a_b, b_b = (int(sc["idx_a"][sc["tags"].index("border")]), int(sc["idx_b"][sc["tags"].index("border")]))
    ok, _, _ = ref.stereo_triangulate(g, a_b, b_b, [])
    assert not ok
    assert all(r[0] != a_b for r in sc["records"])


@pytest.mark.parametrize("i", range(4))
def test_triangulation_matches_oracle_gate(oracle, i):
    """stereoTriangulate's verdict equals the oracle's verifyMatch for every truth pair and look-alike pair."""
    sc = scene(oracle, i)
    st, job = sc["state"], sc["job"]
    g = ref.setup(st, job)
    A, B = st["store"][(job["feat_slot"], 0)], st["store"][(job["feat_slot"], 1)]
    pairs = [(a, int(np.nonzero(sc["truth_b"] == sc["truth_a"][a])[0][0])) for a in range(len(A["lm"])) if sc["truth_a"][a] >= 0]
    rng = np.random.default_rng(i)
    pairs += [(int(a), int(b)) for a, b in zip(rng.integers(0, len(A["lm"]), 100), rng.integers(0, len(B["lm"]), 100))]
    n_valid = 0
    for a, b in pairs:
        gate = abi.make_match_gate(abi.GATE_2D2D, B["kp"][b:b + 1], B["size"][b:b + 1], kp_a=A["kp"][a:a + 1], kp_size_a=A["size"][a:a + 1],
                                   bearing_a=g["bearing_a"][a:a + 1], bearing_b=g["bearing_b"][b:b + 1], ray_sigma_a=g["rs_a"][a:a + 1],
                                   ray_sigma_b=g["rs_b"][b:b + 1], cam_a=g["cam_a"], cam_b=g["cam_b"], T_AB=g["T_AB"].p7())
        same = np.zeros((1, sc["desc_bytes"]), np.uint8)
        r = oracle.match_hamming_gated(same, same, gate)
        ok, _, _ = ref.stereo_triangulate(g, a, b, [])
        assert ok == (int(r["pairs"]["index_a"][0]) == 0), (a, b)
        n_valid += ok
    assert n_valid > 200


@pytest.mark.parametrize("i", range(4))
def test_reprojection_and_H_against_oracle_and_differences(oracle, i):
    sc = scene(oracle, i)
    g = ref.setup(sc["state"], sc["job"])
    for (a, b, _, _, _, hpW) in sc["records"][:40:4]:
        ok, hp, par = ref.stereo_triangulate(g, a, b, [])
        if par:
            continue
        r2, H, rB, JA, JTB, JhB = ref.uncertainty_H(g, a, b, hp)
        sdB = 0.8 * g["size_b"][b] / 12.0
        t = g["t_AB"]
        hm = np.concatenate([0.8 * (hp[:3] - t / 2.0 * hp[3]) + t / 2.0 * hp[3], [hp[3]]])
        T7 = g["T_AB"].p7()
        ro, J0o, J1o, _ = oracle.eval_reprojection(g["cam_b"], T7[None], hm[None], ref.I7[None], g["kp_b"][b][None], [np.sqrt(1 / (sdB * sdB))])
        np.testing.assert_allclose(rB, ro[0], rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(JTB, J0o[0], rtol=1e-10, atol=1e-9 * np.abs(J0o[0]).max())
        np.testing.assert_allclose(JhB, J1o[0], rtol=1e-10, atol=1e-9 * np.abs(J1o[0]).max())
        sqa = np.sqrt(1 / (0.8 * g["size_a"][a] / 12.0) ** 2)
        # central differences: B over the pose (pose_plus) and the point (x + [d, 0]), A over the point
        h = 1e-6
        num_T = np.stack([(ref.reprojection(g["cam_b"], oracle.pose_plus(T7, h * e), hm, g["kp_b"][b], np.sqrt(1 / (sdB * sdB)))[0] -
                           ref.reprojection(g["cam_b"], oracle.pose_plus(T7, -h * e), hm, g["kp_b"][b], np.sqrt(1 / (sdB * sdB)))[0]) / (2 * h)
                          for e in np.eye(6)], 1)
        dp = lambda e: np.concatenate([h * e, [0.0]])
        num_hB = np.stack([(ref.reprojection(g["cam_b"], T7, hm + dp(e), g["kp_b"][b], np.sqrt(1 / (sdB * sdB)))[0] -
                            ref.reprojection(g["cam_b"], T7, hm - dp(e), g["kp_b"][b], np.sqrt(1 / (sdB * sdB)))[0]) / (2 * h) for e in np.eye(3)], 1)
        num_hA = np.stack([(ref.reprojection(g["cam_a"], ref.I7, hp + dp(e), g["kp_a"][a], sqa)[0] -
                            ref.reprojection(g["cam_a"], ref.I7, hp - dp(e), g["kp_a"][a], sqa)[0]) / (2 * h) for e in np.eye(3)], 1)
        J = np.zeros((4, 9))
        J[:2, 6:] = num_hA
        J[2:, :6], J[2:, 6:] = num_T, num_hB
        H_num = g["H_"] + J.T @ J
        np.testing.assert_allclose(H, H_num, rtol=1e-5, atol=1e-5 * np.abs(H[6:, 6:]).max())
        # the prior block against the oracle's PoseError
        S = np.diag([np.sqrt(1 / 4e-8)] * 3 + [np.sqrt(1 / 1e-8)] * 3)
        _, Jp = oracle.eval_pose_error(T7, S, T7)
        np.testing.assert_allclose(g["H_"][:6, :6], Jp.T @ Jp, rtol=1e-12, atol=1e-6)


def test_rank_rule_on_clear_cases():
    rng = np.random.default_rng(5)
    for rank in (9, 8, 6, 3):
        for scale in (1.0, 1e8):
            U = rng.normal(size=(9, rank))
            M = scale * (U @ U.T)
            assert ref.qr_rank(M) == np.linalg.matrix_rank(M) == rank


@pytest.mark.parametrize("i", range(4))
def test_points_near_truth(oracle, i):
    sc = scene(oracle, i)
    n_true = len(sc["points"])
    rel = []
    for (a, b, _, _, cbi, hpW) in sc["records"]:
        t = sc["truth_a"][a]
        if cbi and 0 <= t < n_true and sc["truth_b"][b] == t:
            P = sc["points"][t]
            rel.append(np.linalg.norm(hpW[:3] / hpW[3] - P) / np.linalg.norm(P - sc["window"].poses[sc["job"]["pose"]][:3]))
    # 0.25 px keypoint noise over a 0.11 m baseline: about 1 % of the distance at the median, a few % at the far end
    assert len(rel) > 50 and np.median(rel) < 0.025 and max(rel) < 0.15
