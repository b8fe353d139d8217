"""CPU checks of the restatement tests/ransac2d2d_reference.py of okb_ransac_2d2d_batch (Frontend::runRansac2d2d): the
five-point and two-point solvers on seeded noise-free samples, both scores against a direct transcription of the
reference headers, the triangulation, every branch of the decision and the return value, and the pose initialisation
against a transcription of Frontend.cpp:756-798."""
import itertools

import numpy as np
import pytest

from okvis_b200 import abi
import ransac2d2d_reference as r
import ransac2d2d_scene as S
from stereo_init_reference import Xf


def _rot(rng, ang):
    v = rng.normal(size=3)
    v /= np.linalg.norm(v)
    a = rng.uniform(-ang, ang)
    K = np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])
    return np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K


def _two_view(rng, N, n_pts=6, baseline=(0.1, 1.0)):
    """N noise-free two-view samples: R, t (point in frame 1 = R p2 + t), bearings f1, f2 [N][n_pts][3]."""
    R = np.array([_rot(rng, 0.5) for _ in range(N)])
    t = rng.normal(size=(N, 3))
    t *= (rng.uniform(*baseline, N) / np.linalg.norm(t, axis=1))[:, None]
    P = np.concatenate([rng.uniform(-2, 2, (N, n_pts, 2)), rng.uniform(3, 10, (N, n_pts, 1))], 2)
    P2 = np.einsum("nji,nkj->nki", R, P - t[:, None])
    return R, t, P / np.linalg.norm(P, axis=2)[..., None], P2 / np.linalg.norm(P2, axis=2)[..., None]


def test_monomial_tables():
    for i, j in itertools.product(range(4), range(4)):
        assert r.QUAD[r.LL[i][j]] == tuple(np.add(r.LIN[i], r.LIN[j]))
    for q, i in itertools.product(range(10), range(4)):
        assert r.CUB[r.QL[q][i]] == tuple(np.add(r.QUAD[q], r.LIN[i]))


def test_fivept_finds_the_true_pose():
    rng = np.random.default_rng(55)
    N = 10000
    R, t, f1, f2 = _two_view(rng, N)
    Rs, ts, ok = r.fivept(f1[:, :5], f2[:, :5])
    tu = t / np.linalg.norm(t, axis=1)[:, None]
    err = np.maximum(np.abs(Rs - R[:, None]).reshape(N, 40, 9).max(2), np.abs(ts - tu[:, None]).max(2))
    err = np.where(ok, err, np.inf).min(1)
    assert np.mean(err < 1e-8) >= 0.999


def test_fivept_essential_constraints():
    rng = np.random.default_rng(56)
    N = 2000
    _, _, f1, f2 = _two_view(rng, N)
    E, ok = r.essential_matrices(f1[:, :5], f2[:, :5])
    assert ok.any(1).all()
    En = np.sqrt((E * E).sum((2, 3)))
    epi = np.abs(np.einsum("nir,nkrc,nic->nki", f1[:, :5], E, f2[:, :5])).max(2)
    assert np.all(epi[ok] <= 1e-9 * En[ok])
    EEt = np.einsum("nkij,nklj->nkil", E, E)
    tr = np.trace(EEt, axis1=2, axis2=3)
    cons = 2 * np.einsum("nkij,nkjl->nkil", EEt, E) - tr[..., None, None] * E
    assert np.all(np.abs(cons).max((2, 3))[ok] <= 1e-9 * En[ok] ** 3)
    det = np.linalg.det(E[ok])
    assert np.all(np.abs(det) <= 1e-9 * En[ok] ** 3)


def test_rotation_two_points():
    rng = np.random.default_rng(57)
    N = 1000
    R = np.array([_rot(rng, 1.0) for _ in range(N)])
    f2 = rng.normal(size=(N, 2, 3))
    f2 /= np.linalg.norm(f2, axis=2)[..., None]
    f1 = np.einsum("nij,nkj->nki", R, f2)
    Rg, ok = r.rotation(f1[:, 0], f2[:, 0], f1[:, 1], f2[:, 1])
    assert ok.all() and np.abs(Rg - R).max() < 1e-12
    # symmetric in the two points
    Rs, _ = r.rotation(f1[:, 1], f2[:, 1], f1[:, 0], f2[:, 0])
    assert np.abs(Rs - Rg).max() < 1e-14


def test_scores_match_the_reference_headers():
    rng = np.random.default_rng(58)
    for _ in range(200):
        R, t = _rot(rng, 0.3), rng.normal(size=3)
        f1, f2 = (v / np.linalg.norm(v) for v in rng.normal(size=(2, 3)))
        s1, s2 = rng.uniform(1e-7, 1e-6, 2)
        # FrameRotationOnlySacProblem.hpp
        e1, e2 = R @ f2 - f1, R.T @ f1 - f2
        assert np.isclose(r.score_rot(R, f1, f2, s1, s2), e1 @ e1 * 0.5 / s1 + e2 @ e2 * 0.5 / s2, rtol=1e-12)
        # FrameRelativePoseSacProblem.hpp with triangulate2's point
        p, _, _ = r.triangulate(R, t, f1, f2)
        inv = np.hstack([R.T, (-R.T @ t)[:, None]])
        rep1, rep2 = p / np.linalg.norm(p), inv @ np.append(p, 1.0)
        rep2 = rep2 / np.linalg.norm(rep2)
        want = (rep1 - f1) @ (rep1 - f1) * 0.5 / s1 + (rep2 - f2) @ (rep2 - f2) * 0.5 / s2
        assert np.isclose(r.score_rel(R, t, f1, f2, s1, s2), want, rtol=1e-10)


def test_triangulation_is_the_least_squares_midpoint():
    rng = np.random.default_rng(59)
    for _ in range(200):
        R, t = _rot(rng, 0.3), rng.normal(size=3)
        f1, f2 = (v / np.linalg.norm(v) for v in rng.normal(size=(2, 3)))
        g = R @ f2
        lam = np.linalg.lstsq(np.stack([f1, -g], 1), t, rcond=None)[0]
        p, l1, l2 = r.triangulate(R, t, f1, f2)
        assert np.allclose([l1, l2], lam, rtol=1e-9, atol=1e-12)
        assert np.allclose(p, 0.5 * (lam[0] * f1 + t + lam[1] * g), rtol=1e-9, atol=1e-12)


def test_real_roots_signed():
    rng = np.random.default_rng(60)
    z = np.sort(rng.uniform(-3, 3, (200, 10)), 1)
    p = np.zeros((200, 11))
    for i in range(200):
        p[i] = np.poly(z[i])[::-1]
    roots, cnt = r.real_roots(p, True)
    assert np.all(cnt == 10)
    assert np.abs(roots - z).max() < 1e-6


def _decide(cams):
    """The decision of :709-733 / :802-808 on (n, rotation-only inliers, five-point inliers) per camera: ret,
    rotationOnly and the applied cameras."""
    rot_s = rel_s = False
    total, rot_only, applied = 0, False, []
    for n, ri, li in cams:
        rr, lr = np.float32(ri) / np.float32(n), np.float32(li) / np.float32(n)
        if rr > lr or rr > np.float32(0.8):
            rot_s |= ri > 10
            rot_only = True
            total += ri
        else:
            rel_s |= li > 10
            total += li
        applied.append(rot_s or rel_s)
    return (total, rot_only, applied) if (rot_s or rel_s) else (-1, True, applied)


def test_decision_branches(monkeypatch):
    """Every branch of the decision and the return value, through ransac2d2d with the RANSACs replaced by fixed
    inlier counts."""
    sc = S.make_scene(3, abi.DIST_RADTAN, 4, "large", 0.0)
    cases = [                                       # (rotation-only, five-point) inliers as fractions of n
        [(0.9, 0.3), (0.3, 0.6), (0.02, 0.02), (0.01, 0.02)],   # rotation wins, then five-point, then failures applied
        [(0.85, 0.9), (0.2, 0.2), (0.5, 0.2), (0.9, 0.9)],      # rotation wins above 0.8 against a higher five-point ratio
        [(0.04, 0.04), (0.01, 0.03), (0.04, 0.01), (0.01, 0.04)],  # no success: ret -1, rotationOnly
        [(0.01, 0.3), (0.2, 0.2), (0.0, 0.0), (0.0, 0.0)],      # five-point success, later failures still applied
    ]
    for case in cases:
        it = iter(case)
        cur = {}

        def fake(cr, cam, prob, seed, H, threshold, margins=None):
            n = len(cr["kp_a"])
            if prob == 0:
                cur["c"] = next(it)
            k = int(cur["c"][prob] * n)
            cur.setdefault("k", {})[(cam, prob)] = k
            hyp = np.zeros(H, np.int64)
            hyp[0] = k
            s = np.full(n, 100.0)
            s[:k] = 0.0
            return hyp, {0: (np.eye(3), np.array([0.0, 0.0, 1.0]))}, {0: s}, 0

        monkeypatch.setattr(r, "run_problem", fake)
        o = r.ransac2d2d(S.state(sc), S.job(sc, 1))
        ns = [c["n_correspondences"] for c in o["cams"]]
        assert all(n >= 10 for n in ns)
        ks = [(cur["k"][(c, 0)], cur["k"][(c, 1)]) for c in range(4)]
        want = _decide([(n, a, b) for n, (a, b) in zip(ns, ks)])
        assert (o["ret"], bool(o["rotation_only"])) == want[:2]
        assert [bool(c["applied"]) for c in o["cams"]] == want[2]
        for c, n, (a, b) in zip(o["cams"], ns, ks):
            if c["applied"]:
                assert c["n_outliers"] == n - (a if c["rotation_only"] else b)


def test_camera_below_ten_correspondences_is_skipped():
    sc = S.restrict(S.make_scene(4, abi.DIST_RADTAN, 2, "large", 0.1), 1, 9)
    o = r.ransac2d2d(S.state(sc), S.job(sc, 2))
    c = o["cams"][1]
    assert 0 < c["n_correspondences"] < 10 and c["rot_best"] == c["rel_best"] == -1 and not c["applied"]
    assert not np.any(o["hyp_inliers"][1])
    assert all(oc[0] == 0 for oc in o["outliers"])


def test_pose_initialisation_transcription():
    """T_WS0 <- T_WSA T_SCA T_C1C2 T_SC0^-1 (:756-798) on random poses, the two-camera chain reading camera 0's result."""
    rng = np.random.default_rng(61)
    for _ in range(50):
        q = lambda: (lambda v: v / np.linalg.norm(v))(rng.normal(size=4))
        T_WSA, T_WS0 = Xf(rng.normal(size=3), q()), Xf(rng.normal(size=3), q())
        T_SC = [Xf(rng.normal(size=3) * 0.1, q()) for _ in range(2)]
        models = [(_rot(rng, 0.3), (lambda v: v / np.linalg.norm(v))(rng.normal(size=3))) for _ in range(2)]
        for use_rel in (True, False):
            cur = T_WS0
            for c in range(2):
                R, t = models[c]
                new = r.pose_init(T_WSA, T_SC[c], cur, R, t, use_rel)
                # transcription with 4x4 matrices
                M = lambda T: np.block([[T.C, T.r[:, None]], [np.zeros((1, 3)), np.ones((1, 1))]])
                T12 = np.eye(4)
                T12[:3, :3] = R
                if use_rel:
                    prior = np.linalg.inv(M(T_SC[c])) @ np.linalg.inv(M(T_WSA)) @ M(cur) @ M(T_SC[c])
                    T12[:3, 3] = t * max(0.0, float(t @ prior[:3, 3]))
                want = M(T_WSA) @ M(T_SC[c]) @ T12 @ np.linalg.inv(M(T_SC[c]))
                assert np.abs(M(new) - want).max() < 1e-9
                cur = new


def test_scene_outcomes():
    """Pure rotation with 10 % wrong associations chooses rotation-only (its ratio is above 0.8) and removes every
    injected association; a large baseline chooses the five-point model, whose unit translation is within a few degrees
    of the truth."""
    for dist in (abi.DIST_NONE, abi.DIST_RADTAN, abi.DIST_EQUIDISTANT, abi.DIST_RADTAN8):
        sc = S.make_scene(20 + dist, dist, 2, "rotation", 0.1)
        m = []
        o = r.ransac2d2d(S.state(sc), S.job(sc, 5), margins=m)
        assert o["rotation_only"] == 1 and o["ret"] > 0 and min(m) > S.MIN_MARGIN
        outs = {(c, kb) for c, _, kb, _ in o["outliers"]}
        assert sc["injected"] <= outs
        n_nan = 2 if dist == abi.DIST_RADTAN8 else 0
        assert len(outs - sc["injected"]) <= n_nan + 8
        sc = S.make_scene(30 + dist, dist, 2, "large", 0.1)
        o = r.ransac2d2d(S.state(sc), S.job(sc, 6, initialize_pose=True))
        assert o["rotation_only"] == 0 and o["pose_set"] == 1
        w = sc["window"]
        for c, cam in enumerate(o["cams"]):
            T_SC = Xf(w.extrinsics[c][:3], w.extrinsics[c][3:])
            TA = Xf(w.poses[sc["pose_a"]][:3], w.poses[sc["pose_a"]][3:]) * T_SC
            TB = Xf(w.poses[sc["pose_b"]][:3], w.poses[sc["pose_b"]][3:]) * T_SC
            t_true = (TA.inverse() * TB).r
            cosang = cam["t_rel"] @ t_true / np.linalg.norm(t_true)
            assert cosang > np.cos(np.deg2rad(5.0))
        outs = {(c, kb) for c, _, kb, _ in o["outliers"]}
        assert len(sc["injected"] & outs) >= 0.9 * len(sc["injected"])


@pytest.mark.parametrize("seed", [1, 2])
def test_nan_bearing_never_sampled_or_inlier(seed):
    sc = S.make_scene(seed, abi.DIST_RADTAN8, 1, "large", 0.0)
    o = r.ransac2d2d(S.state(sc), S.job(sc, seed))
    cr = o["cams"][0]["correspondences"]
    nan = np.nonzero(~np.isfinite(cr["f2"].sum(1)))[0]
    assert len(nan) == 1
    assert (0, int(cr["kp_a"][nan[0]]), int(cr["kp_b"][nan[0]]), int(cr["lm"][nan[0]])) in o["outliers"]
