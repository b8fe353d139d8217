"""CPU: the restatement of okb_match2d2d_batch (tests/temporal_init_reference.py) -- the 2D-2D round of matchToKeyframes
/ matchToLastFrame between an older frame and the current one -- on seeded two-frame scenes of all four distortion
models: the scaled prior H_ against central differences of the oracle's PoseError, the velocity clamp, the restatement's
gate against the oracle's verifyMatch, and the triangulated points against the scene's truth."""
import numpy as np
import pytest

import stereo_init_reference as sref
import temporal_init_reference as ref
from okvis_b200 import abi
from temporal_scene import MIN_MARGIN, jobs, make_temporal_scene, variants

_MODELS = [abi.DIST_RADTAN, abi.DIST_EQUIDISTANT, abi.DIST_NONE, abi.DIST_RADTAN8]
_SCENES = {}


def scene(oracle, i):
    if i not in _SCENES:
        _SCENES[i] = make_temporal_scene(i, _MODELS[i], oracle=oracle)
    return _SCENES[i]


@pytest.mark.parametrize("i", range(4))
def test_scene_covers_every_kind_and_no_decision_near_a_threshold(oracle, i):
    sc = scene(oracle, i)
    assert min(m for _, m in sc["margins"]) > MIN_MARGIN
    cases = set(sum(sc["cases"], []))
    for case in ("both_named", "parallel", "close_residual", "initialised", "rank_deficient"):
        assert case in cases, case
    assert any(c.endswith("_a_named") for c in cases) and any(c.endswith("_b_named") for c in cases)
    for j in jobs(sc):
        g = ref.setup(sc["state"], j)
        assert g["skipA"].sum() >= 6 and g["skipB"].sum() >= 4        # initialised landmarks of the graph on both sides
    # keypoints named on the host only reach the records (the device cannot see their ids)
    recs, fa = sc["records"][0], sc["frames"]["feat_slot_a"]
    assert sum(bool(sc["host_only"][(fa, 0)][r[0]]) for r in recs) >= 5
    # the rank pair: the QR decides under both priors, which move its threshold size by about 1e-5 relative
    a = sc["rank_pair"][0]
    assert [r[4] for r in sc["records"][0] if r[0] == a] == [r[4] for r in sc["records"][2] if r[0] == a] == [0]
    t_fast, t_slow = sc["rank_sizes"]
    assert abs(t_slow - t_fast) < 1e-3 * t_slow


def test_uoplus_branches_and_velocity_clamp():
    st = dict(speed_bias=np.zeros((3, 9)))
    st["speed_bias"][0, :3] = [0.3, 0.4, 0.0]          # 0.5 m/s: clamped to 1
    st["speed_bias"][1, :3] = [0.0, 3.0, 4.0]          # 5 m/s
    j = dict(feat_slot_a=0, feat_slot_b=1, sb_current=0)
    assert ref.uoplus_t(st, j) == 1e-2
    assert ref.uoplus_t(st, dict(j, sb_current=1)) == 25.0 * 1e-2
    assert ref.uoplus_t(st, dict(j, sb_current=-1)) == 4e-8
    assert ref.uoplus_t(st, dict(j, feat_slot_a=1)) == 4e-8         # same frame: the stereo prior
    T = sref.Xf([0.1, -0.02, 0.03], [0.01, 0.02, -0.03, 1.0])
    np.testing.assert_array_equal(ref.prior_H(T, 4e-8), sref.prior_H(T))


@pytest.mark.parametrize("i", range(4))
def test_prior_against_pose_error_differences(oracle, i):
    sc = scene(oracle, i)
    for j in jobs(sc, True) + jobs(sc, False):
        g = ref.setup(sc["state"], j)
        u = ref.uoplus_t(sc["state"], j)
        assert u == (max(1.0, sc["speed"]) ** 2 * 1e-2 if j["sb_current"] >= 0 else 4e-8)
        T7 = g["T_AB"].p7()
        S = np.diag([np.sqrt(1 / u)] * 3 + [np.sqrt(1 / 1e-8)] * 3)
        r0, Jp = oracle.eval_pose_error(T7, S, T7)
        np.testing.assert_allclose(g["H_"][:6, :6], Jp.T @ Jp, rtol=1e-12, atol=1e-6)
        # central differences of PoseError's residual over pose_plus, at the scaled UOplus
        h = 1e-7
        num = np.stack([(oracle.eval_pose_error(oracle.pose_plus(T7, h * e), S, T7)[0] -
                         oracle.eval_pose_error(oracle.pose_plus(T7, -h * e), S, T7)[0]) / (2 * h) for e in np.eye(6)], 1)
        np.testing.assert_allclose(g["H_"][:6, :6], num.T @ num, rtol=1e-5, atol=1e-5 * np.abs(g["H_"]).max())
        assert not g["H_"][6:].any() and not g["H_"][:, 6:].any()


@pytest.mark.parametrize("i", range(4))
def test_triangulation_matches_oracle_gate(oracle, i):
    """stereoTriangulate's verdict equals the oracle's verifyMatch for every truth pair and look-alike pair of camera 0."""
    sc = scene(oracle, i)
    st, j = sc["state"], jobs(sc)[0]
    g = ref.setup(st, j)
    A, B = st["store"][(j["feat_slot_a"], 0)], st["store"][(j["feat_slot_b"], 0)]
    ta, tb = sc["truth"][(j["feat_slot_a"], 0)], sc["truth"][(j["feat_slot_b"], 0)]
    pairs = [(a, int(np.nonzero(tb == ta[a])[0][0])) for a in range(len(A["lm"])) if ta[a] >= 0]
    rng = np.random.default_rng(i)
    pairs += [(int(a), int(b)) for a, b in zip(rng.integers(0, len(A["lm"]), 100), rng.integers(0, len(B["lm"]), 100))]
    n_valid = 0
    for a, b in pairs:
        gate = abi.make_match_gate(abi.GATE_2D2D, B["kp"][b:b + 1], B["size"][b:b + 1], kp_a=A["kp"][a:a + 1], kp_size_a=A["size"][a:a + 1],
                                   bearing_a=g["bearing_a"][a:a + 1], bearing_b=g["bearing_b"][b:b + 1], ray_sigma_a=g["rs_a"][a:a + 1],
                                   ray_sigma_b=g["rs_b"][b:b + 1], cam_a=g["cam_a"], cam_b=g["cam_b"], T_AB=g["T_AB"].p7())
        same = np.zeros((1, sc["desc_bytes"]), np.uint8)
        r = oracle.match_hamming_gated(same, same, gate)
        ok, _, _ = sref.stereo_triangulate(g, a, b, [])
        assert ok == (int(r["pairs"]["index_a"][0]) == 0), (a, b)
        n_valid += ok
    assert n_valid > 200


@pytest.mark.parametrize("i", range(4))
def test_points_near_truth(oracle, i):
    sc = scene(oracle, i)
    n_true = len(sc["points"])
    rel = []
    for v, j in enumerate(variants(sc)):
        ta, tb = sc["truth"][(j["feat_slot_a"], j["cam_a"])], sc["truth"][(j["feat_slot_b"], j["cam_b"])]
        for (a, b, _, _, cbi, hpW) in sc["records"][v]:
            t = ta[a]
            if cbi and 0 <= t < n_true and tb[b] == t:
                P = sc["points"][t]
                rel.append(np.linalg.norm(hpW[:3] / hpW[3] - P) / np.linalg.norm(P - sc["window"].poses[j["pose_b"]][:3]))
    # 0.25 px keypoint noise over about 0.12 m of motion: about 1 % of the distance at the median; the far points (up to
    # 60 m, rays a few milliradians apart) err by tens of percent
    assert len(rel) > 200 and np.median(rel) < 0.025 and np.percentile(rel, 90) < 0.1 and max(rel) < 1.0
