"""TEST INFRASTRUCTURE ONLY -- CPU restatement of okb_ransac_2d2d_batch, Frontend::runRansac2d2d
(okvis_frontend/src/Frontend.cpp:645-810) on the window's feature store, step for step as k_ransac_2d2d runs it:
  adapter     FrameRelativeAdapter.cpp:139-244 (per camera: B's first keypoint per landmark of the graph, then A's
              keypoints ascending)
  sampler     ransac_reference.draw keyed by (seed, (2 cam + problem) 64 + hypothesis, draw), k distinct indices
  solvers     the two-point rotation (bearing triads) and the five-point relative pose of DESIGN.md 6i (Householder null
              space, 10 x 20 Gauss-Jordan, degree-10 polynomial, derivative-bracketed bisection, E -> 4 (R, t)),
              vectorised over many problems
  scores      FrameRotationOnlySacProblem.hpp / FrameRelativePoseSacProblem.hpp (triangulate2 as a closed-form midpoint)
  decision    :709-733 (float ratios, success flags kept across cameras), ret :802-808, outliers :735-753 (the B keypoint
              of the correspondence), pose initialisation :756-798
`margins` collects every score's relative distance to the threshold."""
import numpy as np

from ransac_reference import BISECT, draw, quat_from_R
from stereo_init_reference import Xf, undistort_gn

MAX_HYP = 64
POLISH = 2
CONS_TOL = 1e-10

# monomials (exponents of x, y, z) of the linear, quadratic and cubic polynomials, and the product tables
LIN = [(1, 0, 0), (0, 1, 0), (0, 0, 1), (0, 0, 0)]
QUAD = [(2, 0, 0), (0, 2, 0), (0, 0, 2), (1, 1, 0), (1, 0, 1), (0, 1, 1), (1, 0, 0), (0, 1, 0), (0, 0, 1), (0, 0, 0)]
CUB = [(3, 0, 0), (0, 3, 0), (2, 1, 0), (1, 2, 0), (2, 0, 1), (2, 0, 0), (0, 2, 1), (0, 2, 0), (1, 1, 1), (1, 1, 0),
       (1, 0, 2), (1, 0, 1), (1, 0, 0), (0, 1, 2), (0, 1, 1), (0, 1, 0), (0, 0, 3), (0, 0, 2), (0, 0, 1), (0, 0, 0)]
LL = [[0, 3, 4, 6], [3, 1, 5, 7], [4, 5, 2, 8], [6, 7, 8, 9]]
QL = [[0, 2, 4, 5], [3, 1, 6, 7], [10, 13, 16, 17], [2, 3, 8, 9], [4, 8, 10, 11], [8, 6, 13, 14], [5, 9, 11, 12],
      [9, 7, 14, 15], [11, 14, 17, 18], [12, 15, 18, 19]]


def sample(seed, key, n, k):
    """k distinct indices in [0, n), or None after 64 draws."""
    idx = []
    for c in range(64):
        if len(idx) == k:
            break
        v = ((draw(seed, key, c) >> 32) * n) >> 32
        if v not in idx:
            idx.append(v)
    return idx if len(idx) == k else None


def _dot(a, b):
    return a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1] + a[..., 2] * b[..., 2]


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _horner(c, x):
    v = c[:, -1].copy()
    for i in range(c.shape[1] - 2, -1, -1):
        v = v * x + c[:, i]
    return v


def _umul(p, q):
    r = np.zeros((p.shape[0], p.shape[1] + q.shape[1] - 1))
    for i in range(p.shape[1]):
        for j in range(q.shape[1]):
            r[:, i + j] += p[:, i] * q[:, j]
    return r


# ---------------------------------------------------------------------------------------------------------------- roots
def real_roots(p, signed):
    """rs_real_roots<D, signed> for each row of p [N][D + 1]: the roots in (0, B] (signed: (-B, B]), ascending,
    NaN-padded [N][D], and their counts."""
    N, D = p.shape[0], p.shape[1] - 1
    roots = np.full((N, D), np.nan)
    cnt = np.zeros(N, np.int64)
    finite = np.all(np.isfinite(p), 1)
    mx = np.where(finite, np.max(np.abs(np.where(np.isfinite(p), p, 0.0)), 1), 0.0)
    deg = np.zeros(N, np.int64)
    for i in range(D, 0, -1):
        deg = np.where((deg == 0) & (np.abs(p[:, i]) > 1e-14 * mx), i, deg)
    deg[~finite] = 0
    for n in range(1, D + 1):
        rows = np.nonzero(deg == n)[0]
        if len(rows) == 0:
            continue
        q = p[rows, :n + 1] / p[rows, n:n + 1]
        bound = np.max(np.abs(q[:, :n]), 1) + 1.0
        M = len(rows)
        r = np.full((M, D), np.nan)
        nr = np.zeros(M, np.int64)
        for m in range(1, n + 1):
            c = np.zeros((M, m + 1))
            for i in range(m + 1):
                f = q[:, i + n - m].copy()
                for t in range(i + 1, i + n - m + 1):
                    f = f * float(t)
                c[:, i] = f
            nxt = np.full((M, D), np.nan)
            k = np.zeros(M, np.int64)
            lo = -bound if signed else np.zeros(M)
            flo = _horner(c, lo)
            for e in range(int(nr.max()) + 1):
                valid = e <= nr
                hi = np.where(e < nr, r[:, min(e, D - 1)], bound)
                fhi = _horner(c, hi)
                has = valid & (((flo < 0) & (fhi >= 0)) | ((flo > 0) & (fhi <= 0)))
                neg = flo < 0
                a, b = lo.copy(), hi.copy()
                for _ in range(BISECT):
                    mid = 0.5 * (a + b)
                    go = (_horner(c, mid) < 0) == neg
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


# ---------------------------------------------------------------------------------------------------------------- models
def triad(u1, nn):
    """rs_triad: rows e1 = u1 / |u1|, e2 = n x e1, n = nn / |nn| ([...][3][3])."""
    e1 = u1 * (1.0 / np.sqrt(_dot(u1, u1)))[..., None]
    e3 = nn * (1.0 / np.sqrt(_dot(nn, nn)))[..., None]
    e2 = np.stack([e3[..., 1] * e1[..., 2] - e3[..., 2] * e1[..., 1], e3[..., 2] * e1[..., 0] - e3[..., 0] * e1[..., 2],
                   e3[..., 0] * e1[..., 1] - e3[..., 1] * e1[..., 0]], -1)
    return np.stack([e1, e2, e3], -2)


def rotation(a0, b0, a1, b1):
    """Two-point rotation for N problems (A bearings a, B bearings b, [N][3]): R [N][3][3] with R b = a, and ok."""
    with np.errstate(all="ignore"):
        FA = triad(a0 + a1, _cross(a0, a1))
        FB = triad(b0 + b1, _cross(b0, b1))
        R = FA[:, 0, :, None] * FB[:, 0, None, :] + FA[:, 1, :, None] * FB[:, 1, None, :] + FA[:, 2, :, None] * FB[:, 2, None, :]
    return R, np.isfinite(R.reshape(-1, 9).sum(1))


def triangulate(R, t, f1, f2):
    """triangulate2 as specified: the midpoint of the common perpendicular of l1 f1 and t + l2 R f2 (broadcast).
    Returns the point and (l1, l2)."""
    g = np.einsum("...ij,...j->...i", R, f2)
    a, b, c, d1, d2 = _dot(f1, f1), _dot(f1, g), _dot(g, g), _dot(f1, t), _dot(g, t)
    with np.errstate(all="ignore"):
        det = a * c - b * b
        l1 = (c * d1 - b * d2) / det
        l2 = (b * d1 - a * d2) / det
        p = 0.5 * (l1[..., None] * f1 + (t + l2[..., None] * g))
    return p, l1, l2


def score_rot(R, f1, f2, s1, s2):
    """FrameRotationOnlySacProblem::getSelectedDistancesToModel (broadcast)."""
    e1 = np.einsum("...ij,...j->...i", R, f2) - f1
    e2 = np.einsum("...ji,...j->...i", R, f1) - f2
    with np.errstate(all="ignore"):
        return _dot(e1, e1) * 0.5 / s1 + _dot(e2, e2) * 0.5 / s2


def score_rel(R, t, f1, f2, s1, s2):
    """FrameRelativePoseSacProblem::getSelectedDistancesToModel (broadcast)."""
    p, _, _ = triangulate(R, t, f1, f2)
    ti = -np.einsum("...ji,...j->...i", R, t)
    q = np.einsum("...ji,...j->...i", R, p) + ti
    with np.errstate(all="ignore"):
        e1 = p / np.sqrt(_dot(p, p))[..., None] - f1
        e2 = q / np.sqrt(_dot(q, q))[..., None] - f2
        return _dot(e1, e1) * 0.5 / s1 + _dot(e2, e2) * 0.5 / s2


def essential_matrices(f1, f2, details=None):
    """The E of every real root for N five-point problems (f1, f2 [N][5][3], f1^T E f2 = 0): E [N][10][3][3] (scaled to
    |E|_F = sqrt 2) and ok [N][10], roots ascending.  details: a dict that receives the null basis and the polynomial."""
    N = f1.shape[0]
    M = np.einsum("nir,nic->nrci", f1, f2).reshape(N, 9, 5).copy()
    V = np.zeros((N, 5, 9))
    beta = np.zeros((N, 5))
    for j in range(5):
        nx = np.sqrt(np.sum(M[:, j:, j] * M[:, j:, j], 1))
        alpha = np.where(M[:, j, j] < 0.0, nx, -nx)
        V[:, j, j:] = M[:, j:, j]
        V[:, j, j] -= alpha
        b = np.sum(V[:, j, j:] * V[:, j, j:], 1)
        beta[:, j] = b
        live = b > 0.0
        with np.errstate(all="ignore"):
            for k in range(j, 5):
                s = 2.0 * np.sum(V[:, j, j:] * M[:, j:, k], 1) / b
                M[:, j:, k] = np.where(live[:, None], M[:, j:, k] - s[:, None] * V[:, j, j:], M[:, j:, k])
    Nb = np.zeros((N, 4, 9))
    for b4 in range(4):
        Nb[:, b4, 5 + b4] = 1.0
        for j in range(4, -1, -1):
            live = beta[:, j] > 0.0
            with np.errstate(all="ignore"):
                s = 2.0 * np.sum(V[:, j, j:] * Nb[:, b4, j:], 1) / beta[:, j]
            Nb[:, b4, j:] = np.where(live[:, None], Nb[:, b4, j:] - s[:, None] * V[:, j, j:], Nb[:, b4, j:])
    G = np.zeros((N, 10, 20))
    EE = np.zeros((N, 3, 3, 10))
    for r in range(3):
        for c in range(3):
            for k in range(3):
                for i in range(4):
                    for j in range(4):
                        EE[:, r, c, LL[i][j]] += Nb[:, i, 3 * r + k] * Nb[:, j, 3 * c + k]
    tr = EE[:, 0, 0] + EE[:, 1, 1] + EE[:, 2, 2]
    for r in range(3):
        for c in range(3):
            S = np.zeros((N, 20))
            T = np.zeros((N, 20))
            for k in range(3):
                for q in range(10):
                    for i in range(4):
                        S[:, QL[q][i]] += EE[:, r, k, q] * Nb[:, i, 3 * k + c]
            for q in range(10):
                for i in range(4):
                    T[:, QL[q][i]] += tr[:, q] * Nb[:, i, 3 * r + c]
            G[:, 1 + 3 * r + c] = 2.0 * S - T
    cof = [(4, 8, 5, 7), (3, 8, 5, 6), (3, 7, 4, 6)]
    for e, sg in zip(range(3), (1.0, -1.0, 1.0)):
        mq = np.zeros((N, 10))
        for i in range(4):
            for j in range(4):
                mq[:, LL[i][j]] += Nb[:, i, cof[e][0]] * Nb[:, j, cof[e][1]] - Nb[:, i, cof[e][2]] * Nb[:, j, cof[e][3]]
        for q in range(10):
            for i in range(4):
                G[:, 0, QL[q][i]] += sg * (Nb[:, i, e] * mq[:, q])
    G0 = G.copy()
    good = np.ones(N, bool)
    ar = np.arange(N)
    with np.errstate(all="ignore"):
        for j in range(10):
            p = np.full(N, j)
            for i in range(j + 1, 10):
                p = np.where(np.abs(G[:, i, j]) > np.abs(G[ar, p, j]), i, p)
            piv = G[ar, p, j]
            good &= (piv != 0.0) & np.isfinite(piv)
            rowp = G[ar, p].copy()
            G[ar, p] = G[:, j]
            G[:, j] = rowp
            G[:, j, j:] = G[:, j, j:] / piv[:, None]
            for i in range(10):
                if i == j:
                    continue
                f = G[:, i, j].copy()
                G[:, i, j:] -= f[:, None] * G[:, j, j:]
    P = np.zeros((N, 3, 3, 5))
    for r in range(3):
        a, b = G[:, 4 + 2 * r], G[:, 5 + 2 * r]
        P[:, r, 0, :4] = np.stack([a[:, 12], a[:, 11] - b[:, 12], a[:, 10] - b[:, 11], -b[:, 10]], 1)
        P[:, r, 1, :4] = np.stack([a[:, 15], a[:, 14] - b[:, 15], a[:, 13] - b[:, 14], -b[:, 13]], 1)
        P[:, r, 2] = np.stack([a[:, 19], a[:, 18] - b[:, 19], a[:, 17] - b[:, 18], a[:, 16] - b[:, 17], -b[:, 16]], 1)
    d3, d4 = (lambda r, v: P[:, r, v, :4]), (lambda r, v: P[:, r, v, :5])
    t1 = _umul(d3(1, 1), d4(2, 2)) - _umul(d4(1, 2), d3(2, 1))
    t2 = _umul(d3(1, 0), d4(2, 2)) - _umul(d4(1, 2), d3(2, 0))
    t3 = _umul(d3(1, 0), d3(2, 1)) - _umul(d3(1, 1), d3(2, 0))
    dz = _umul(d3(0, 0), t1) - _umul(d3(0, 1), t2) + _umul(d4(0, 2), t3)
    dz[~good] = np.nan
    if details is not None:
        details.update(null=Nb, poly=dz, good=good)
    roots, _ = real_roots(dz, True)
    E_out = np.zeros((N, 10, 3, 3))
    ok_out = np.zeros((N, 10), bool)
    with np.errstate(all="ignore"):
        for ir in range(10):
            z = roots[:, ir]
            row = np.stack([np.stack([_horner(P[:, r, v], z) for v in range(3)], -1) for r in range(2)], 1)
            u = _cross(row[:, 0], row[:, 1])
            live = np.isfinite(z) & (u[:, 2] != 0.0) & np.isfinite(u.sum(1))
            x, y = u[:, 0] / u[:, 2], u[:, 1] / u[:, 2]
            x, y, z = polish(G0, x, y, z)
            E = x[:, None] * Nb[:, 0] + y[:, None] * Nb[:, 1] + z[:, None] * Nb[:, 2] + Nb[:, 3]
            ss = np.zeros(N)
            for e in range(9):
                ss = ss + E[:, e] * E[:, e]
            live &= (ss > 0.0) & np.isfinite(ss)
            E = E * (np.sqrt(2.0) / np.sqrt(ss))[:, None]
            live &= constraints_hold(E.reshape(N, 3, 3))
            E_out[:, ir] = E.reshape(N, 3, 3)
            ok_out[:, ir] = live
    return E_out, ok_out


def polish(G0, x, y, z):
    """POLISH Gauss-Newton steps of (x, y, z) [N] on the 10 cubic constraints G0 [N][10][20] (before elimination), the
    3x3 normal equations solved by Cramer's rule; a step stops at a singular or non-finite system."""
    go = np.isfinite(x + y + z)
    for _ in range(POLISH):
        px = np.stack([np.ones_like(x), x, x * x, x * x * x], 1)
        py = np.stack([np.ones_like(y), y, y * y, y * y * y], 1)
        pz = np.stack([np.ones_like(z), z, z * z, z * z * z], 1)
        g = np.zeros((len(x), 10))
        J = np.zeros((len(x), 10, 3))
        for m, (a, b, c) in enumerate(CUB):
            mon = px[:, a] * py[:, b] * pz[:, c]
            dx = a * px[:, max(a - 1, 0)] * py[:, b] * pz[:, c]
            dy = b * px[:, a] * py[:, max(b - 1, 0)] * pz[:, c]
            dw = c * px[:, a] * py[:, b] * pz[:, max(c - 1, 0)]
            g += G0[:, :, m] * mon[:, None]
            J[:, :, 0] += G0[:, :, m] * dx[:, None]
            J[:, :, 1] += G0[:, :, m] * dy[:, None]
            J[:, :, 2] += G0[:, :, m] * dw[:, None]
        A = np.einsum("nki,nkj->nij", J, J)
        bb = np.einsum("nki,nk->ni", J, g)
        det = (A[:, 0, 0] * (A[:, 1, 1] * A[:, 2, 2] - A[:, 1, 2] * A[:, 2, 1]) - A[:, 0, 1] * (A[:, 1, 0] * A[:, 2, 2] - A[:, 1, 2] * A[:, 2, 0]) +
               A[:, 0, 2] * (A[:, 1, 0] * A[:, 2, 1] - A[:, 1, 1] * A[:, 2, 0]))
        go = go & (det != 0.0) & np.isfinite(det)
        d = []
        for v in range(3):
            Av = A.copy()
            Av[:, :, v] = bb
            d.append((Av[:, 0, 0] * (Av[:, 1, 1] * Av[:, 2, 2] - Av[:, 1, 2] * Av[:, 2, 1]) -
                      Av[:, 0, 1] * (Av[:, 1, 0] * Av[:, 2, 2] - Av[:, 1, 2] * Av[:, 2, 0]) +
                      Av[:, 0, 2] * (Av[:, 1, 0] * Av[:, 2, 1] - Av[:, 1, 1] * Av[:, 2, 0])) / det)
        x = np.where(go, x - d[0], x)
        y = np.where(go, y - d[1], y)
        z = np.where(go, z - d[2], z)
    return x, y, z


def constraints_hold(E):
    """E [N][3][3] (|E|_F = sqrt 2) meets det E = 0 and 2 E E^T E - tr(E E^T) E = 0 to CONS_TOL |E|_F^3, each entry
    summed in the kernel's order."""
    worst = np.zeros(E.shape[0])
    EEt = np.zeros(E.shape)
    for i in range(3):
        for j in range(3):
            EEt[:, i, j] = E[:, i, 0] * E[:, j, 0] + E[:, i, 1] * E[:, j, 1] + E[:, i, 2] * E[:, j, 2]
    tr = EEt[:, 0, 0] + EEt[:, 1, 1] + EEt[:, 2, 2]
    for i in range(3):
        for j in range(3):
            v = 2.0 * (EEt[:, i, 0] * E[:, 0, j] + EEt[:, i, 1] * E[:, 1, j] + EEt[:, i, 2] * E[:, 2, j]) - tr * E[:, i, j]
            worst = np.maximum(worst, np.abs(v))
    det = (E[:, 0, 0] * (E[:, 1, 1] * E[:, 2, 2] - E[:, 1, 2] * E[:, 2, 1]) - E[:, 0, 1] * (E[:, 1, 0] * E[:, 2, 2] - E[:, 1, 2] * E[:, 2, 0]) +
           E[:, 0, 2] * (E[:, 1, 0] * E[:, 2, 1] - E[:, 1, 1] * E[:, 2, 0]))
    worst = np.maximum(worst, np.abs(det))
    return worst <= CONS_TOL * 2.0 * np.sqrt(2.0)


def decompose(E):
    """The 4 (R, t) candidates of E [...][3][3] (|E|_F = sqrt 2): R [...][4][3][3], t [...][4][3], order (R1, t), (R1, -t),
    (R2, t), (R2, -t), R1 = cof(E) - [t]x E, R2 = cof(E) + [t]x E; and whether t exists."""
    cols = [E[..., :, c] for c in range(3)]
    best = np.full(E.shape[:-2], -1.0)
    t = np.zeros(E.shape[:-2] + (3,))
    with np.errstate(all="ignore"):
        for a, b in ((0, 1), (0, 2), (1, 2)):
            w = _cross(cols[a], cols[b])
            wn = np.sqrt(_dot(w, w))
            pick = wn > best
            best = np.where(pick, wn, best)
            t = np.where(pick[..., None], w, t)
        ok = best > 0.0
        t = t / best[..., None]
    cf = np.zeros(E.shape)
    tx = np.zeros(E.shape)
    for i in range(3):
        for j in range(3):
            i1, i2, j1, j2 = (i + 1) % 3, (i + 2) % 3, (j + 1) % 3, (j + 2) % 3
            cf[..., i, j] = E[..., i1, j1] * E[..., i2, j2] - E[..., i1, j2] * E[..., i2, j1]
            tx[..., i, j] = t[..., i1] * E[..., i2, j] - t[..., i2] * E[..., i1, j]
    R1, R2 = cf - tx, cf + tx
    R = np.stack([R1, R1, R2, R2], -3)
    T = np.stack([t, -t, t, -t], -2)
    return R, T, ok


def fivept(f1, f2):
    """Every admissible (R, t) of N five-point problems: R [N][40][3][3], t [N][40][3], ok [N][40] (roots ascending,
    then candidates in decompose's order)."""
    N = f1.shape[0]
    E, okE = essential_matrices(f1, f2)
    R, t, okT = decompose(E)
    ok = np.repeat((okE & okT)[:, :, None], 4, 2)
    for i in range(5):
        _, l1, l2 = triangulate(R, t, f1[:, None, None, i], f2[:, None, None, i])
        ok &= (l1 > 0.0) & (l2 > 0.0)
    return R.reshape(N, 40, 3, 3), t.reshape(N, 40, 3), ok.reshape(N, 40)


# ---------------------------------------------------------------------------------------------------------------- call
def correspondences(state, feat_a, feat_b, cam):
    """FrameRelativeAdapter for camera `cam`: dict of f1, f2 [n][3], s1, s2 [n], kp_a, kp_b, lm [n]."""
    w = state["window"]
    L = len(w.landmarks)
    eA, eB = state["store"][(feat_a, cam)], state["store"][(feat_b, cam)]
    cm = w.cameras[cam]
    fu, fv, cu, cv = (float(cm[k]) for k in ("fu", "fv", "cu", "cv"))
    first = {}
    for k in range(len(eB["lm"])):
        l = int(eB["lm"][k])
        if 0 <= l < L and np.any(w.landmarks[l] != 0.0) and l not in first:
            first[l] = k
    out = {k: [] for k in ("f1", "f2", "s1", "s2", "kp_a", "kp_b", "lm")}

    def bearing(e, k):
        with np.errstate(all="ignore"):
            u = undistort_gn(cm, (e["kp"][k][0] - cu) * (1.0 / fu), (e["kp"][k][1] - cv) * (1.0 / fv))
            br = np.array([u[0], u[1], 1.0])
            n2 = br @ br
            if n2 > 0:
                br = br / np.sqrt(n2)
        sd = 0.8 * float(e["size"][k]) / 12.0
        return br, np.sqrt(2.0) * sd * sd / (fu * fu)

    for k in range(len(eA["lm"])):
        l = int(eA["lm"][k])
        if l not in first:
            continue
        kb = first[l]
        b1, s1 = bearing(eA, k)
        b2, s2 = bearing(eB, kb)
        for key, v in (("f1", b1), ("f2", b2), ("s1", s1), ("s2", s2), ("kp_a", k), ("kp_b", kb), ("lm", l)):
            out[key].append(v)
    res = {k: np.array(out[k], np.float64).reshape(-1, 3) for k in ("f1", "f2")}
    res.update({k: np.array(out[k], np.float64) for k in ("s1", "s2")})
    res.update({k: np.array(out[k], np.int64) for k in ("kp_a", "kp_b", "lm")})
    return res


def run_problem(cr, cam, prob, seed, H, threshold, margins=None):
    """One RANSAC of one camera: per-hypothesis inliers [H], the models {h: (R, t)} and the winner (or -1)."""
    n = len(cr["kp_a"])
    k = 6 if prob else 2
    samples = [sample(seed, (2 * cam + prob) * MAX_HYP + h, n, k) for h in range(H)]
    fin = np.isfinite(cr["f1"].sum(1) + cr["f2"].sum(1))
    use = [h for h in range(H) if samples[h] is not None and np.all(fin[samples[h]])]
    models = {}
    if use:
        idx = np.array([samples[h] for h in use])
        if prob == 0:
            R, ok = rotation(cr["f1"][idx[:, 0]], cr["f2"][idx[:, 0]], cr["f1"][idx[:, 1]], cr["f2"][idx[:, 1]])
            for u, h in enumerate(use):
                if ok[u]:
                    models[h] = (R[u], np.zeros(3))
        else:
            R, t, ok = fivept(cr["f1"][idx[:, :5]], cr["f2"][idx[:, :5]])
            k6 = idx[:, 5]
            sc6 = score_rel(R, t, cr["f1"][k6][:, None], cr["f2"][k6][:, None], cr["s1"][k6][:, None], cr["s2"][k6][:, None])
            for u, h in enumerate(use):
                best, pick = np.inf, -1
                for r in range(40):
                    if ok[u, r] and sc6[u, r] < best:
                        best, pick = sc6[u, r], r
                if pick >= 0:
                    models[h] = (R[u, pick], t[u, pick])
    hyp = np.zeros(H, np.int64)
    scores = {}
    for h, (R, t) in models.items():
        s = (score_rel(R[None], t[None], cr["f1"], cr["f2"], cr["s1"], cr["s2"]) if prob else
             score_rot(R[None], cr["f1"], cr["f2"], cr["s1"], cr["s2"]))
        scores[h] = s
        hyp[h] = int(np.sum(s < threshold))
        if margins is not None:
            f = s[np.isfinite(s)]
            margins.extend((np.abs(f - threshold) / threshold).tolist())
    best, bc = -1, -1
    for h in range(H):
        if h in models and hyp[h] > bc:
            best, bc = h, hyp[h]
    return hyp, models, scores, best


def pose_init(T_WSA, T_SC, T_WS0, R, t, use_rel):
    """Frontend.cpp:756-798 for one camera: the new T_WS0 (Xf).  use_rel: rel_pose_success; R, t: that model (None:
    missing, T_C1C2 stays the identity)."""
    Rm, tm = np.eye(3), np.zeros(3)
    if R is not None:
        Rm = R
        if use_rel:
            prior = T_SC.inverse() * T_WSA.inverse() * T_WS0 * T_SC
            tm = t * max(0.0, float(t[0] * prior.r[0] + t[1] * prior.r[1] + t[2] * prior.r[2]))
    return T_WSA * T_SC * Xf(tm, quat_from_R(Rm)) * T_SC.inverse()


def ransac2d2d(state, job, margins=None):
    """One job (dict with pose_b, feat_slot_b, pose_a, feat_slot_a, n_cams, seed and optionally initialize_pose,
    max_iterations, threshold).  Returns okb_ransac2d_result's fields plus cams, hyp_inliers [n_cams][2][H] and
    outliers [(cam, kp_a, kp_b, lm)]."""
    w = state["window"]
    H, thr = int(job.get("max_iterations", 50)), float(job.get("threshold", 9.0))
    seed, n_cams = int(job["seed"]), int(job["n_cams"])
    out = dict(ret=0, rotation_only=0, pose_set=0, n_outliers=0, T_WS=np.zeros(7), cams=[],
               hyp_inliers=np.zeros((n_cams, 2, H), np.int64), outliers=[])
    rot_success = rel_success = False
    total = 0
    T_WSA = Xf(w.poses[job["pose_a"]][:3], w.poses[job["pose_a"]][3:])
    T_WS0 = Xf(w.poses[job["pose_b"]][:3], w.poses[job["pose_b"]][3:])
    for cam in range(n_cams):
        cr = correspondences(state, job["feat_slot_a"], job["feat_slot_b"], cam)
        n = len(cr["kp_a"])
        c = dict(n_correspondences=n, rot_inliers=0, rel_inliers=0, rot_best=-1, rel_best=-1, rotation_only=0, applied=0,
                 n_outliers=0, R_rot=np.eye(3), R_rel=np.eye(3), t_rel=np.zeros(3), correspondences=cr)
        out["cams"].append(c)
        if n < 10:
            continue
        runs = [run_problem(cr, cam, p, seed, H, thr, margins) for p in (0, 1)]
        for p in (0, 1):
            out["hyp_inliers"][cam, p] = runs[p][0]
        (_, mrot, srot, brot), (_, mrel, srel, brel) = runs
        c["rot_best"], c["rel_best"] = brot, brel
        c["rot_inliers"] = int(runs[0][0][brot]) if brot >= 0 else 0
        c["rel_inliers"] = int(runs[1][0][brel]) if brel >= 0 else 0
        if brot >= 0:
            c["R_rot"] = mrot[brot][0]
        if brel >= 0:
            c["R_rel"], c["t_rel"] = mrel[brel]
        rot_ratio = np.float32(c["rot_inliers"]) / np.float32(n)
        rel_ratio = np.float32(c["rel_inliers"]) / np.float32(n)
        if rot_ratio > rel_ratio or rot_ratio > np.float32(0.8):
            if c["rot_inliers"] > 10:
                rot_success = True
            out["rotation_only"] = c["rotation_only"] = 1
            total += c["rot_inliers"]
            b, sc = brot, srot
        else:
            if c["rel_inliers"] > 10:
                rel_success = True
            total += c["rel_inliers"]
            b, sc = brel, srel
        if not (rot_success or rel_success):
            continue
        c["applied"] = 1
        inl = sc[b] < thr if b >= 0 else np.zeros(n, bool)
        outl = [(cam, int(cr["kp_a"][k]), int(cr["kp_b"][k]), int(cr["lm"][k])) for k in np.nonzero(~inl)[0]]
        c["n_outliers"] = len(outl)
        out["outliers"] += outl
        if job.get("initialize_pose", False):
            e = w.extrinsics[cam]
            T_SC = Xf(e[:3], e[3:])
            if rel_success:
                R, t = (c["R_rel"], c["t_rel"]) if brel >= 0 else (None, None)
            else:
                R, t = (c["R_rot"], None) if brot >= 0 else (None, None)
            T_WS0 = pose_init(T_WSA, T_SC, T_WS0, R, t, rel_success)
            out["pose_set"] = 1
    if rot_success or rel_success:
        out["ret"] = total
    else:
        out["ret"], out["rotation_only"] = -1, 1
    if out["pose_set"]:
        out["T_WS"] = T_WS0.p7()
    out["n_outliers"] = len(out["outliers"])
    return out
