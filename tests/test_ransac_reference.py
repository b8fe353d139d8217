"""CPU: the restatement of okb_ransac_3d2d_batch (tests/ransac_reference.py) -- the generalised P3P's properties on
seeded rigs, the score against a direct transcription of FrameAbsolutePoseSacProblem.hpp, the sampler, the seeded
scenes' outcomes and margins, and the C structs."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from okvis_b200 import abi
import ransac_reference as rr
import ransac_scene as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rig(rng, N, n_cams):
    """N noise-free problems: ray origins on an n_cams rig (1: central), unit rays to points 2-10 m ahead, and a random
    pose (R, t) mapping the body points into the world."""
    cams = rng.normal(0, 0.2, (N, n_cams, 3)) if n_cams > 1 else np.zeros((N, 1, 3))
    c = np.take_along_axis(cams, rng.integers(0, n_cams, (N, 3))[:, :, None], 1)
    pb = c + np.stack([rng.uniform(-3, 3, (N, 3)), rng.uniform(-3, 3, (N, 3)), rng.uniform(2, 10, (N, 3))], -1)
    f = pb - c
    f /= np.linalg.norm(f, axis=-1, keepdims=True)
    Q, _ = np.linalg.qr(rng.normal(size=(N, 3, 3)))
    Q *= np.sign(np.linalg.det(Q))[:, None, None]
    t = rng.normal(0, 5, (N, 3))
    X = np.einsum("nij,nkj->nki", Q, pb) + t[:, None]
    return c, f, X, Q, t, pb


@pytest.mark.parametrize("n_cams", [1, 2, 4])
def test_gp3p_properties(n_cams):
    rng = np.random.default_rng(100 + n_cams)
    c, f, X, Q, t, pb = _rig(rng, 10000, n_cams)
    R, tt, ok = rr.gp3p(c, f, X)
    assert ok.sum(1).max() <= 8
    # every returned solution satisfies the three distance equations to 1e-9 relative
    for r in range(8):
        m = ok[:, r]
        p = np.einsum("nji,nkj->nki", R[m, r], X[m] - tt[m, r][:, None])          # body points of the solution
        for i, j in ((0, 1), (0, 2), (1, 2)):
            d = np.sum((X[m, i] - X[m, j]) ** 2, 1)
            assert np.all(np.abs(np.sum((p[:, i] - p[:, j]) ** 2, 1) - d) <= 1e-9 * d)
        # the points lie on their rays
        lam = np.einsum("nki,nki->nk", p - c[m], f[m])
        assert np.all(np.abs(p - c[m] - lam[:, :, None] * f[m]) <= 1e-8 * (1 + np.abs(lam[:, :, None])))
    hit = np.zeros(len(c), bool)
    for r in range(8):
        err = np.maximum(np.abs(R[:, r] - Q).reshape(-1, 9).max(1), np.abs(tt[:, r] - t).max(1) / np.abs(t).max(1))
        hit |= ok[:, r] & (err < 1e-8)
    assert hit.mean() >= 0.999
    # the misses are near-degenerate: the distance equations' Jacobian at the true depths is nearly singular (a double root)
    for n in np.nonzero(~hit)[0]:
        lam = np.einsum("ki,ki->k", pb[n] - c[n], f[n])
        J = np.zeros((3, 3))
        for e, (i, j) in enumerate(((0, 1), (0, 2), (1, 2))):
            v = c[n, i] + lam[i] * f[n, i] - c[n, j] - lam[j] * f[n, j]
            J[e, i], J[e, j] = 2 * v @ f[n, i], -2 * v @ f[n, j]
        sv = np.linalg.svd(J, compute_uv=False)
        assert sv[-1] < 1e-4 * sv[0], (n, sv)


def test_gp3p_central_octic_is_even():
    """All three rays from one camera: the octic has only even powers (depths come in +- pairs), and the positive half of
    its roots still gives the true pose."""
    rng = np.random.default_rng(7)
    c, f, X, Q, t, _ = _rig(rng, 200, 1)
    octs = []
    R, tt, ok = rr.gp3p(c, f, X, octic=octs)
    o = octs[0]
    scale = np.abs(o).max(1)
    assert np.all(np.abs(o[:, 1::2]).max(1) <= 1e-9 * scale)
    c2, f2, X2, _, _, _ = _rig(np.random.default_rng(8), 200, 2)
    octs2 = []
    rr.gp3p(c2, f2, X2, octic=octs2)
    assert np.median(np.abs(octs2[0][:, 1::2]).max(1) / np.abs(octs2[0]).max(1)) > 1e-3       # non-central: not even
    hit = np.zeros(len(c), bool)
    for r in range(8):
        hit |= ok[:, r] & (np.abs(R[:, r] - Q).reshape(-1, 9).max(1) < 1e-8)
    assert hit.mean() >= 0.99


def test_score_matches_transcription():
    """FrameAbsolutePoseSacProblem::getSelectedDistancesToModel, written out as the reference writes it."""
    rng = np.random.default_rng(3)
    for _ in range(50):
        Q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        Q *= np.sign(np.linalg.det(Q))
        t = rng.normal(0, 3, 3)
        model = np.concatenate([Q, t[:, None]], 1)
        inv = np.zeros((3, 4))
        inv[:, :3] = model[:, :3].T
        inv[:, 3] = -inv[:, :3] @ model[:, 3]
        X, b = rng.normal(0, 5, 3), rng.normal(size=3)
        b /= np.linalg.norm(b)
        Cs, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        rs, sigma = rng.normal(0, 0.1, 3), rng.uniform(1e-7, 1e-5)
        body = inv @ np.concatenate([X, [1.0]])
        rep = Cs.T @ (body - rs)
        rep = rep / np.linalg.norm(rep)
        want = float((rep - b) @ (rep - b)) / sigma
        got = rr.score(Q, t, X, b, sigma, Cs, rs)
        assert abs(got - want) <= 1e-12 * max(1.0, want)


def test_sampler_distinct_and_position_free():
    for seed in (0, 1, 2 ** 63 + 5, 0xFFFFFFFFFFFFFFFF):
        for n in (5, 6, 37, 1000):
            for h in range(64):
                s = rr.sample(seed, h, n)
                assert s is not None and len(set(s)) == 4 and all(0 <= v < n for v in s)
    # the draws are a function of (seed, hypothesis, counter) only: the known first values pin the generator
    assert rr.draw(0, 0, 0) == 0xE220A8397B1DCDAF
    assert rr.draw(1234, 3, 7) == rr.draw(1234, 3, 7)
    assert rr.sample(99, 5, 400) != rr.sample(100, 5, 400)


@pytest.mark.parametrize("distortion", [abi.DIST_NONE, abi.DIST_RADTAN, abi.DIST_EQUIDISTANT, abi.DIST_RADTAN8])
@pytest.mark.parametrize("n_cams", [2, 4])
@pytest.mark.parametrize("wrong", [0.0, 0.1, 0.3, 0.5])
def test_scene_outcome(distortion, n_cams, wrong):
    sc = S.make_scene(11 + n_cams, distortion, n_cams, wrong)
    m = []
    r = rr.ransac(S.state(sc), S.FEAT, n_cams, seed=77, margins=m)
    assert min(m) > S.MIN_MARGIN
    cr = r["correspondences"]
    kinds = sc["kinds"]
    for l in cr["lm"]:
        assert int(l) not in kinds["single"] | kinds["infinity"] | kinds["dead"]
    assert r["n_inliers"] >= 10 and r["ret"] == r["n_inliers"]
    outs = {(c, k) for c, k, _ in r["outliers"]}
    nan_bearing = {(int(c), int(k)) for c, k, b in zip(cr["cam"], cr["kp"], cr["bearing"]) if not np.all(np.isfinite(b))}
    assert len(nan_bearing) == (n_cams if distortion == abi.DIST_RADTAN8 else 0)
    assert nan_bearing <= outs                         # a failed backProject: a correspondence, never an inlier
    if wrong <= 0.3:
        assert outs - nan_bearing == sc["injected"]    # every injected outlier out, no true association out


def test_scene_edge_jobs():
    sc = S.make_scene(5, abi.DIST_RADTAN, 2, 0.0)
    r = rr.ransac(S.state(S.restrict(sc, max_assoc=2)), S.FEAT, 2, seed=1)
    assert r["n_correspondences"] < 5 and r["ret"] == r["n_correspondences"] and r["outliers"] == []
    r = rr.ransac(S.state(S.restrict(sc, max_assoc=4)), S.FEAT, 2, seed=1)
    assert r["n_correspondences"] >= 5 and r["n_inliers"] < 10 and r["outliers"] == []
    r = rr.ransac(S.state(S.restrict(sc, empty_cam=1)), S.FEAT, 2, seed=1)
    assert set(r["correspondences"]["cam"].tolist()) == {0} and r["n_inliers"] >= 10


def _header_struct(name):
    txt = open(os.path.join(ROOT, "include", "okvis_b200.h")).read()
    m = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), txt, re.S)
    assert m, name
    body = re.sub(r"/\*.*?\*/", "", m.group(1), flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        typ, names = re.match(r"([\w\s\*]+?\*?)\s*((?:\*?\w+(?:\[\d+\])?\s*,\s*)*\*?\w+(?:\[\d+\])?)$", decl).groups()
        for nm in names.split(","):
            nm = nm.strip()
            arr = re.match(r"(\w+)\[(\d+)\]", nm)
            fields.append((arr.group(1) if arr else nm.lstrip("*"), "*" in typ or nm.startswith("*"), typ.replace("*", "").strip(),
                           int(arr.group(2)) if arr else 1))
    return fields


_CT = {"int32_t": C.c_int32, "uint64_t": C.c_uint64, "double": C.c_double}


@pytest.mark.parametrize("cname,py", [("okb_ransac_result", abi.RansacResult), ("okb_ransac_job", abi.RansacJob)])
def test_abi_layout_matches_header(cname, py):
    fields = _header_struct(cname)
    assert [f for f, _, _, _ in fields] == [f for f, _ in py._fields_]
    off, align = 0, 1
    for (nm, is_ptr, typ, n), (pnm, ptyp) in zip(fields, py._fields_):
        ct = C.c_void_p if is_ptr else _CT[typ]
        a = C.alignment(ct)
        off = (off + a - 1) // a * a
        assert getattr(py, pnm).offset == off, nm
        assert C.sizeof(ptyp) == C.sizeof(ct) * n, nm
        off += C.sizeof(ct) * n
        align = max(align, a)
    assert C.sizeof(py) == (off + align - 1) // align * align


def test_outlier_dtype_matches_header():
    assert [f for f, _, _, _ in _header_struct("okb_ransac_outlier")] == list(abi.ransac_outlier_dtype.names)
    assert abi.ransac_outlier_dtype.itemsize == 12
