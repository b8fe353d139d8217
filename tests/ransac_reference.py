"""TEST INFRASTRUCTURE ONLY -- CPU restatement of okb_ransac_3d2d_batch, Frontend::runRansac3d2d
(okvis_frontend/src/Frontend.cpp:575-642) on the window's feature store, step for step as k_ransac_3d2d runs it:
  adapter     FrameNoncentralAbsoluteAdapter.cpp:65-160 (cameras ascending, keypoints ascending)
  sampler     SplitMix64 keyed by (seed, hypothesis, draw), multiply-shift to [0, n), duplicates redrawn (DESIGN.md 6f)
  solver      the generalised P3P of DESIGN.md 6f (octic in the first depth, derivative-bracketed bisection, 2 Gauss-Newton
              steps, triad pose), vectorised over many problems
  score       FrameAbsolutePoseSacProblem.hpp:134-160
  decision    most inliers (ties: lowest hypothesis), outliers reported at >= 10 inliers (:613-640)
`margins` collects every score's relative distance to the threshold."""
import numpy as np

from stereo_init_reference import Xf, undistort_gn

MASK = (1 << 64) - 1
BISECT = 60
POLISH = 2


# ---------------------------------------------------------------------------------------------------------------- sampler
def draw(seed, h, c):
    z = (seed + 0x9E3779B97F4A7C15 * ((h << 32) + c + 1)) & MASK
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK
    return z ^ (z >> 31)


def sample(seed, h, n):
    """4 distinct indices in [0, n), or None after 64 draws."""
    idx = []
    for c in range(64):
        if len(idx) == 4:
            break
        v = ((draw(seed, h, c) >> 32) * n) >> 32
        if v not in idx:
            idx.append(v)
    return idx if len(idx) == 4 else None


# ---------------------------------------------------------------------------------------------------------------- solver
def _horner(c, m, x):
    v = c[:, m].copy()
    for i in range(m - 1, -1, -1):
        v = v * x + c[:, i]
    return v


def _umul(p, q):
    r = np.zeros((p.shape[0], p.shape[1] + q.shape[1] - 1))
    for i in range(p.shape[1]):
        for j in range(q.shape[1]):
            r[:, i + j] += p[:, i] * q[:, j]
    return r


def _bmul(A, B):
    C = np.zeros_like(A)
    for i1 in range(5):
        for j1 in range(5 - i1):
            for i2 in range(5 - i1):
                for j2 in range(5 - i1 - i2 - j1):
                    C[:, i1 + i2, j1 + j2] += A[:, i1, j1] * B[:, i2, j2]
    return C


def positive_roots(p):
    """Roots in (0, bound] of each row of p [N][9] (ascending; NaN-padded [N][8]) and their counts."""
    N = p.shape[0]
    roots = np.full((N, 8), np.nan)
    cnt = np.zeros(N, np.int64)
    finite = np.all(np.isfinite(p), 1)
    mx = np.where(finite, np.max(np.abs(np.where(np.isfinite(p), p, 0.0)), 1), 0.0)
    deg = np.zeros(N, np.int64)
    for i in range(8, 0, -1):
        deg = np.where((deg == 0) & (np.abs(p[:, i]) > 1e-14 * mx), i, deg)
    deg[~finite] = 0
    for n in range(1, 9):
        rows = np.nonzero(deg == n)[0]
        if len(rows) == 0:
            continue
        q = p[rows, :n + 1] / p[rows, n:n + 1]
        bound = np.max(np.abs(q[:, :n]), 1) + 1.0
        M = len(rows)
        r = np.full((M, 8), np.nan)
        nr = np.zeros(M, np.int64)
        for m in range(1, n + 1):
            c = np.zeros((M, m + 1))
            for i in range(m + 1):
                f = q[:, i + n - m].copy()
                for t in range(i + 1, i + n - m + 1):
                    f = f * float(t)
                c[:, i] = f
            nxt = np.full((M, 8), np.nan)
            k = np.zeros(M, np.int64)
            lo = np.zeros(M)
            flo = _horner(c, m, lo)
            for e in range(int(nr.max()) + 1):
                valid = e <= nr
                hi = np.where(e < nr, r[:, min(e, 7)], bound)
                fhi = _horner(c, m, hi)
                has = valid & (((flo < 0) & (fhi >= 0)) | ((flo > 0) & (fhi <= 0)))
                neg = flo < 0
                a, b = lo.copy(), hi.copy()
                for _ in range(BISECT):
                    mid = 0.5 * (a + b)
                    go = (_horner(c, m, mid) < 0) == neg
                    a = np.where(go, mid, a)
                    b = np.where(go, b, mid)
                ii = np.nonzero(has)[0]
                nxt[ii, k[ii]] = 0.5 * (a[ii] + b[ii])
                k += has
                lo = np.where(valid, hi, lo)
                flo = np.where(valid, fhi, flo)
            r, nr = nxt, k
        roots[rows] = r
        cnt[rows] = nr
    return roots, cnt


def _dot(a, b):
    return a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1] + a[..., 2] * b[..., 2]


def gp3p(c, f, X, octic=None):
    """Generalised P3P for N problems: c, f, X [N][3][3] (ray origins and unit directions in the body frame, world points).
    Returns R [N][8][3][3], t [N][8][3] with X = R p + t, and ok [N][8] (admissible solutions, ascending first depth).
    octic: a list that receives the octics [N][9] (scaled problem, before normalisation)."""
    c, f, X = (np.asarray(a, np.float64) for a in (c, f, X))
    N = c.shape[0]
    R_out = np.zeros((N, 8, 3, 3))
    t_out = np.zeros((N, 8, 3))
    ok_out = np.zeros((N, 8), bool)
    dX = np.stack([X[:, 0] - X[:, 1], X[:, 0] - X[:, 2], X[:, 1] - X[:, 2]], 1)
    D01, D02, D12 = _dot(dX[:, 0], dX[:, 0]), _dot(dX[:, 1], dX[:, 1]), _dot(dX[:, 2], dX[:, 2])
    s = np.sqrt(np.maximum(D01, np.maximum(D02, D12)))
    good = (s > 0) & np.isfinite(s)
    s = np.where(good, s, 1.0)
    i_s = 1.0 / s
    c01 = (c[:, 0] - c[:, 1]) * i_s[:, None]
    c02 = (c[:, 0] - c[:, 2]) * i_s[:, None]
    c12 = (c[:, 1] - c[:, 2]) * i_s[:, None]
    d01, d02, d12 = D01 * i_s * i_s, D02 * i_s * i_s, D12 * i_s * i_s
    f0, f1, f2 = f[:, 0], f[:, 1], f[:, 2]
    f01, f02, f12 = _dot(f0, f1), _dot(f0, f2), _dot(f1, f2)
    k01, k02, k12 = _dot(c01, c01) - d01, _dot(c02, c02) - d02, _dot(c12, c12) - d12
    g0_01, g1_01, g0_02, g2_02 = _dot(f0, c01), _dot(f1, c01), _dot(f0, c02), _dot(f2, c02)
    g1_12, g2_12, g2_01 = _dot(f1, c12), _dot(f2, c12), _dot(f2, c01)
    Dp, Dq, R1, P1 = (np.zeros((N, 5, 5)) for _ in range(4))
    Dp[:, 1, 0], Dp[:, 0, 1], Dp[:, 0, 0] = 2.0 * f02, -2.0 * f12, 2.0 * g2_01
    Dq[:, 0, 2], Dq[:, 0, 1], Dq[:, 0, 0], Dq[:, 1, 0], Dq[:, 2, 0] = 1.0, 2.0 * g1_12, k12 - k02, -2.0 * g0_02, -1.0
    R1[:, 2, 0], R1[:, 1, 0], R1[:, 0, 0] = 1.0, 2.0 * g0_02, k02
    P1[:, 1, 0], P1[:, 0, 0] = -2.0 * f02, -2.0 * g2_02
    S = _bmul(Dp, _bmul(Dp, R1) - _bmul(Dq, P1)) + _bmul(Dq, Dq)
    a = np.stack([-2.0 * g1_01, -2.0 * f01], 1)
    b = np.stack([k01, 2.0 * g0_01, np.ones(N)], 1)
    A2, AB, A3, A2B, B2 = _umul(a, a), _umul(a, b), _umul(_umul(a, a), a), _umul(_umul(a, a), b), _umul(b, b)
    r3y, r4y, r4c = A2 - b, 2.0 * AB - A3, B2 - A2B
    sk = [S[:, :5 - k, k] for k in range(5)]          # coefficient of l_1^k: polynomial in l_0 of degree 4 - k
    al = np.zeros((N, 4))
    al += sk[1][:, :4]
    al -= _umul(a, sk[2][:, :3])[:, :4]
    al += _umul(r3y, sk[3][:, :2])[:, :4]
    al += _umul(r4y, sk[4][:, :1])[:, :4]
    be = np.zeros((N, 5))
    be += sk[0][:, :5]
    be -= _umul(b, sk[2][:, :3])[:, :5]
    be += _umul(AB, sk[3][:, :2])[:, :5]
    be += _umul(r4c, sk[4][:, :1])[:, :5]
    oct_ = _umul(_umul(al, al), b) - _umul(_umul(al, be), a) + _umul(be, be)
    oct_[~good] = np.nan
    if octic is not None:
        octic.append(oct_.copy())
    roots, _ = positive_roots(oct_)
    for r in range(8):
        x = roots[:, r]
        alx, bex = _horner(al, 3, x), _horner(be, 4, x)
        live = np.isfinite(x) & (alx != 0.0)
        with np.errstate(all="ignore"):
            y = -bex / alx
            dp = 2.0 * f02 * x - 2.0 * f12 * y + 2.0 * g2_01
            live &= dp != 0.0
            dq = y * y + 2.0 * g1_12 * y + (k12 - k02) - x * x - 2.0 * g0_02 * x
            z = -dq / dp
            go = live.copy()
            for _ in range(POLISH):
                F0 = x * x + y * y - 2.0 * f01 * x * y + 2.0 * g0_01 * x - 2.0 * g1_01 * y + k01
                F1 = x * x + z * z - 2.0 * f02 * x * z + 2.0 * g0_02 * x - 2.0 * g2_02 * z + k02
                F2 = y * y + z * z - 2.0 * f12 * y * z + 2.0 * g1_12 * y - 2.0 * g2_12 * z + k12
                A = 2.0 * x - 2.0 * f01 * y + 2.0 * g0_01
                B = 2.0 * y - 2.0 * f01 * x - 2.0 * g1_01
                C = 2.0 * x - 2.0 * f02 * z + 2.0 * g0_02
                D = 2.0 * z - 2.0 * f02 * x - 2.0 * g2_02
                E = 2.0 * y - 2.0 * f12 * z + 2.0 * g1_12
                G = 2.0 * z - 2.0 * f12 * y - 2.0 * g2_12
                det = -A * D * E - B * C * G
                go = go & (det != 0.0) & np.isfinite(det)
                x = np.where(go, x + (F0 * D * E + B * F1 * G - B * D * F2) / det, x)
                y = np.where(go, y + (-A * F1 * G + A * D * F2 + F0 * C * G) / det, y)
                z = np.where(go, z + (A * F1 * E + B * C * F2 - F0 * C * E) / det, z)
            live &= (x > 0) & (y > 0) & (z > 0) & np.isfinite(x + y + z)
            lam = np.stack([x, y, z], 1)
            pp = c * i_s[:, None, None] + lam[:, :, None] * f
            for (i, j), dd in zip(((0, 1), (0, 2), (1, 2)), (d01, d02, d12)):
                v = pp[:, i] - pp[:, j]
                live &= np.abs(_dot(v, v) - dd) <= 1e-10 * dd
            p = c + (lam * s[:, None])[:, :, None] * f
            frames = []
            for P in (p, X):
                u1, u2 = P[:, 1] - P[:, 0], P[:, 2] - P[:, 0]
                nn = np.stack([u1[:, 1] * u2[:, 2] - u1[:, 2] * u2[:, 1], u1[:, 2] * u2[:, 0] - u1[:, 0] * u2[:, 2],
                               u1[:, 0] * u2[:, 1] - u1[:, 1] * u2[:, 0]], 1)
                e1 = u1 * (1.0 / np.sqrt(_dot(u1, u1)))[:, None]
                e3 = nn * (1.0 / np.sqrt(_dot(nn, nn)))[:, None]
                e2 = np.stack([e3[:, 1] * e1[:, 2] - e3[:, 2] * e1[:, 1], e3[:, 2] * e1[:, 0] - e3[:, 0] * e1[:, 2],
                               e3[:, 0] * e1[:, 1] - e3[:, 1] * e1[:, 0]], 1)
                frames.append(np.stack([e1, e2, e3], 1))          # rows e1, e2, n
            Fp, Fx = frames
            R = (Fx[:, 0, :, None] * Fp[:, 0, None, :] + Fx[:, 1, :, None] * Fp[:, 1, None, :] +
                 Fx[:, 2, :, None] * Fp[:, 2, None, :])
            live &= np.isfinite(R.reshape(N, 9).sum(1))
            pc = (p[:, 0] + p[:, 1] + p[:, 2]) / 3.0
            xc = (X[:, 0] + X[:, 1] + X[:, 2]) / 3.0
            t = xc - np.einsum("nij,nj->ni", R, pc)
        R_out[:, r], t_out[:, r], ok_out[:, r] = R, t, live & good
    return R_out, t_out, ok_out


def quat_from_R(M):
    """Eigen's Quaternion(Matrix3d), [x, y, z, w]."""
    q = np.zeros(4)
    tr = M[0, 0] + M[1, 1] + M[2, 2]
    if tr > 0.0:
        s = np.sqrt(tr + 1.0)
        q[3] = 0.5 * s
        s = 0.5 / s
        q[:3] = [(M[2, 1] - M[1, 2]) * s, (M[0, 2] - M[2, 0]) * s, (M[1, 0] - M[0, 1]) * s]
    else:
        i = 0
        if M[1, 1] > M[0, 0]:
            i = 1
        if M[2, 2] > M[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        s = np.sqrt(M[i, i] - M[j, j] - M[k, k] + 1.0)
        q[i] = 0.5 * s
        s = 0.5 / s
        q[3] = (M[k, j] - M[j, k]) * s
        q[j] = (M[j, i] + M[i, j]) * s
        q[k] = (M[k, i] + M[i, k]) * s
    return q


# ---------------------------------------------------------------------------------------------------------------- score
def score(R, t, X, bearing, sigma, C_SC, r_SC):
    """FrameAbsolutePoseSacProblem::getSelectedDistancesToModel, broadcast over leading axes: R [...][3][3], t [...][3],
    X / bearing [...][3], sigma [...], C_SC [...][3][3], r_SC [...][3]."""
    Ri = np.swapaxes(R, -1, -2)
    ti = -np.einsum("...ij,...j->...i", Ri, t)
    body = np.einsum("...ij,...j->...i", Ri, X) + ti
    rep = np.einsum("...ji,...j->...i", C_SC, body - r_SC)
    with np.errstate(all="ignore"):
        rep = rep / np.sqrt(_dot(rep, rep))[..., None]
        e = rep - bearing
        return _dot(e, e) / sigma


# ---------------------------------------------------------------------------------------------------------------- call
def correspondences(state, feat, n_cams):
    """The adapter's correspondences: dict of arrays X, bearing, ray, sigma, cam, kp, lm (correspondence order)."""
    w = state["window"]
    L = len(w.landmarks)
    cnt = np.bincount(np.asarray(w.obs["lm_idx"][w.obs["sqrt_info"] != 0.0], np.int64), minlength=L)
    ext = [Xf(w.extrinsics[cm][:3], w.extrinsics[cm][3:]) for cm in range(n_cams)]
    out = {k: [] for k in ("X", "bearing", "ray", "sigma", "cam", "kp", "lm")}
    for cam in range(n_cams):
        e = state["store"][(feat, cam)]
        cm = w.cameras[cam]
        fu, fv, cu, cv = (float(cm[k]) for k in ("fu", "fv", "cu", "cv"))
        for k in range(len(e["lm"])):
            l = int(e["lm"][k])
            if not (0 <= l < L and np.any(w.landmarks[l] != 0.0)):
                continue
            if cnt[l] < 2:
                continue
            hp = w.landmarks[l]
            if abs(hp[3]) < 1.0e-8:
                continue
            with np.errstate(all="ignore"):
                u = undistort_gn(cm, (e["kp"][k][0] - cu) * (1.0 / fu), (e["kp"][k][1] - cv) * (1.0 / fv))
                br = np.array([u[0], u[1], 1.0])
                n2 = br @ br
                if n2 > 0:
                    br = br / np.sqrt(n2)
            sd = 0.8 * float(e["size"][k]) / 12.0
            out["X"].append(hp[:3] / hp[3])
            out["bearing"].append(br)
            out["ray"].append(ext[cam].C @ br)
            out["sigma"].append(np.sqrt(2.0) * sd * sd / (fu * fu))
            out["cam"].append(cam)
            out["kp"].append(k)
            out["lm"].append(l)
    res = {k: np.array(v, np.float64) for k, v in out.items() if k in ("X", "bearing", "ray", "sigma")}
    for k in ("X", "bearing", "ray"):
        res[k] = res[k].reshape(-1, 3)
    for k in ("cam", "kp", "lm"):
        res[k] = np.array(out[k], np.int64)
    res["C_SC"] = np.array([ext[cm].C for cm in range(n_cams)]).reshape(-1, 3, 3)
    res["r_SC"] = np.array([ext[cm].r for cm in range(n_cams)]).reshape(-1, 3)
    return res


def ransac(state, feat, n_cams, seed, max_iterations=50, threshold=9.0, margins=None):
    """One job.  state: dict(window, store {(feat, cam): dict(kp, size, lm)}).  Returns the okb_ransac_result fields plus
    hyp_inliers and outliers [(cam, kp, lm)]."""
    w = state["window"]
    out = dict(ret=0, n_correspondences=0, n_inliers=0, best=-1, n_outliers=0, T_WS=np.zeros(7),
               hyp_inliers=np.zeros(max_iterations, np.int64), outliers=[])
    if len(w.poses) < 2:
        out["ret"] = 1
        return out
    cr = correspondences(state, feat, n_cams)
    n = len(cr["cam"])
    out["n_correspondences"] = out["ret"] = n
    if n < 5:
        return out
    H = max_iterations
    samples = [sample(seed, h, n) for h in range(H)]
    use = [h for h in range(H) if samples[h] is not None and np.all(np.isfinite(cr["bearing"][samples[h]]))]
    models = {}
    if use:
        idx = np.array([samples[h] for h in use])
        c = cr["r_SC"][cr["cam"][idx[:, :3]]]
        R, t, ok = gp3p(c, cr["ray"][idx[:, :3]], cr["X"][idx[:, :3]])
        k4 = idx[:, 3]
        sc4 = score(R, t, cr["X"][k4][:, None], cr["bearing"][k4][:, None], cr["sigma"][k4][:, None],
                    cr["C_SC"][cr["cam"][k4]][:, None], cr["r_SC"][cr["cam"][k4]][:, None])
        for u, h in enumerate(use):
            best, pick = np.inf, -1
            for r in range(8):
                if ok[u, r] and sc4[u, r] < best:
                    best, pick = sc4[u, r], r
            if pick >= 0:
                models[h] = (R[u, pick], t[u, pick])
    cam = cr["cam"]
    scores = {}
    for h, (R, t) in models.items():
        s = score(R[None], t[None], cr["X"], cr["bearing"], cr["sigma"], cr["C_SC"][cam], cr["r_SC"][cam])
        scores[h] = s
        out["hyp_inliers"][h] = int(np.sum(s < threshold))
        if margins is not None:
            fin = s[np.isfinite(s)]
            margins.extend((np.abs(fin - threshold) / threshold).tolist())
    best, bc = -1, -1
    for h in range(H):
        if h in models and out["hyp_inliers"][h] > bc:
            best, bc = h, out["hyp_inliers"][h]
    out["best"] = best
    out["n_inliers"] = out["ret"] = int(bc) if best >= 0 else 0
    if best >= 0:
        R, t = models[best]
        out["T_WS"] = np.concatenate([t, quat_from_R(R)])
        out["R"] = R
        if out["n_inliers"] >= 10:
            bad = ~(scores[best] < threshold)
            out["outliers"] = [(int(cr["cam"][k]), int(cr["kp"][k]), int(cr["lm"][k])) for k in np.nonzero(bad)[0]]
    out["n_outliers"] = len(out["outliers"])
    out["correspondences"] = cr
    return out
