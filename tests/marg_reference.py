"""Extended-precision reference for one marginalisation step (the operation of okb_window_marginalize and of the
oracle's oracle_marg_apply.hpp), written independently of both.

Assembly evaluates every residual through the oracle's single-functor hooks (pinned by the golden NumPy vectors) and
follows the device's semantics: blocks carried over from the previous prior (block_prev >= 0) are linearised at its
x0, every IMU term at the bias of the preintegration cache the step starts from, the Cauchy correction sqrt(rho') only
when the last optimize used the Cauchy loss, and the previous prior's (H, b0) is scattered into the new ordering.
Products and sums run in np.longdouble.  Elimination is in np.longdouble too: one explicit 3x3 inverse per landmark,
then a Cholesky factorisation of the preconditioned dense block V.  Neither shares code with the oracle's or the
device's eigen pseudo-inverses.

The prior (J, e0) is not unique (any orthogonal transform of the residual space), so `check_prior` compares it through
quantities that are: the rank, J^T J against H', J^T e0 + b' on the range of H', x0 and the block list.  Every bound is
a first-order rounding-error model whose magnitudes and condition numbers are taken from the reference."""
import numpy as np

from okvis_b200 import abi
from oracle import oracle_py as op

P, SB = abi.BLOCK_POSE, abi.BLOCK_SPEED_BIAS
LD = np.longdouble
EPS = float(np.finfo(np.float64).eps)
# rounding-error model constant: a handful of roundings per product and per sum of the model's first-order terms
C_ROUND = 8.0
# H', b': multiple of the measured error of a double-precision realisation of the step (`bounds`)
C_MEAS = 16.0
# a rank is well defined when no eigenvalue of the preconditioned H' lies within this factor of the threshold
RANK_GAP = 1e3


def require_long_double():
    """The reference needs an extended format (x87 80-bit or binary128): fail, never skip, where it is not."""
    nmant = np.finfo(np.longdouble).nmant
    assert nmant >= 63, "np.longdouble has %d mantissa bits here; the marginalisation reference needs >= 63" % nmant


def precond(d):
    """p = sqrt(diag) where diag > 1e-9, else 1e-3 (MarginalizationError.cpp:618, 695, 816)."""
    d = np.asarray(d, np.float64)
    return np.where(d > 1e-9, np.sqrt(np.maximum(d, 0.0)), 1e-3)


def job_lists(job):
    """The index lists of an abi.make_marg_job object."""
    k = job._keep
    return dict(kind=[int(x) for x in k[0]], idx=[int(x) for x in k[1]], prev=[int(x) for x in k[2]], marg=[bool(x) for x in k[3]],
                imu=[int(x) for x in k[4]], sbp=[int(x) for x in k[5]], lms=[int(x) for x in k[6]])


def _inv3(V):
    """Inverse of a 3x3 long-double matrix by cofactors."""
    a = V
    c = np.empty((3, 3), LD)
    for i in range(3):
        for j in range(3):
            r = [x for x in range(3) if x != j]
            s = [x for x in range(3) if x != i]
            c[i, j] = (-1) ** (i + j) * (a[r[0], s[0]] * a[r[1], s[1]] - a[r[0], s[1]] * a[r[1], s[0]])
    det = a[0, 0] * c[0, 0] + a[0, 1] * c[1, 0] + a[0, 2] * c[2, 0]
    return c / det


def _cholesky(A):
    """Lower Cholesky factor of a symmetric positive definite long-double matrix (column by column)."""
    n = A.shape[0]
    L = np.zeros((n, n), LD)
    for j in range(n):
        d = A[j, j] - L[j, :j] @ L[j, :j]
        assert d > 0, "dense block V is not positive definite at column %d" % j
        L[j, j] = np.sqrt(d)
        L[j + 1:, j] = (A[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return L


def _forward(L, B):
    """L^-1 B for lower-triangular L (long double, B is n x m)."""
    X = np.zeros(B.shape, LD)
    for i in range(L.shape[0]):
        X[i] = (B[i] - L[i, :i] @ X[:i]) / L[i, i]
    return X


def _pinv64(A):
    """Double-precision pseudo-inverse of a symmetric block as a double-precision implementation forms it: eigen
    decomposition of the diagonally preconditioned block, eigenvalues <= eps * n * lambda_max dropped."""
    p = precond(np.diag(A))
    lam, Q = np.linalg.eigh(0.5 * (A + A.T) / np.outer(p, p))
    keep = lam > EPS * len(lam) * lam.max(initial=0.0)
    return ((Q[:, keep] / lam[keep]) @ Q[:, keep].T) / np.outer(p, p)


def _cond_sym(A):
    ev = np.linalg.eigvalsh(np.asarray(A, np.float64))
    return np.inf if ev[0] <= 0 else ev[-1] / ev[0]


def reference_marginalize(w, job, prior=None, imu_cache=None, use_cauchy=True):
    """The reduced system (H', b') of one marginalisation step.

    w          window at the estimates the step sees (obs with sqrt_info == 0 are removed observations)
    job        abi.make_marg_job object
    prior      None, or the previous prior as okb_window_download_marg returns it: block_kind / block_idx / x0 and the
               persisted system H / b0 (what block_prev indexes)
    imu_cache  {term: (sb_ref, valid)} of the caches before the step; a missing or invalid entry preintegrates afresh
    """
    require_long_double()
    jl = job_lists(job)
    NB = len(jl["kind"])
    dims = [6 if k == P else 9 for k in jl["kind"]]
    col = np.concatenate([[0], np.cumsum(dims)]).astype(int)
    Nd = int(col[-1])
    pose_blk = {i: b for b, (k, i) in enumerate(zip(jl["kind"], jl["idx"])) if k == P}
    sb_blk = {i: b for b, (k, i) in enumerate(zip(jl["kind"], jl["idx"])) if k == SB}
    # linearisation points
    if prior is not None:
        pw = [9 if k == SB else 7 for k in prior["block_kind"]]
        pd = [9 if k == SB else 6 for k in prior["block_kind"]]
        poff, pcol = np.concatenate([[0], np.cumsum(pw)]).astype(int), np.concatenate([[0], np.cumsum(pd)]).astype(int)
    xlin = []
    for b in range(NB):
        pv, k, i = jl["prev"][b], jl["kind"][b], jl["idx"][b]
        if pv >= 0:
            xlin.append(np.array(prior["x0"][poff[pv]:poff[pv + 1]], np.float64))
        else:
            xlin.append(np.array(w.poses[i] if k == P else w.speed_bias[i], np.float64))
    H = np.zeros((Nd, Nd), LD)
    bv = np.zeros(Nd, LD)
    # the same step carried out a second time in double precision, the way a double-precision implementation does it
    # (sums in double, eigen pseudo-inverses of the preconditioned blocks): its distance from the long-double result
    # measures the rounding error such an implementation makes on this very system (see `bounds`)
    # Its residuals and Jacobians are evaluated at the states perturbed by one rounding (relative 2 eps, fixed signs):
    # a stable functor evaluation is one at inputs perturbed that much, so the measurement also covers the error of the
    # implementation's own functors, and it propagates through both eliminations like any other rounding.
    H64, b64 = np.zeros((Nd, Nd)), np.zeros(Nd)
    kappa_lm = 1.0
    rng = np.random.default_rng(0)

    def pert(x):
        x = np.asarray(x, np.float64)
        return x * (1.0 + 2.0 * EPS * rng.choice([-1.0, 1.0], size=x.shape))
    # the previous prior in the new ordering
    if prior is not None:
        Hp, bp = np.asarray(prior["H"], np.float64), np.asarray(prior["b0"], np.float64)
        carried = [b for b in range(NB) if jl["prev"][b] >= 0]
        for bi in carried:
            ri = slice(pcol[jl["prev"][bi]], pcol[jl["prev"][bi] + 1])
            bv[col[bi]:col[bi + 1]] = bp[ri]
            for bj in carried:
                H[col[bi]:col[bi + 1], col[bj]:col[bj + 1]] = Hp[ri, pcol[jl["prev"][bj]]:pcol[jl["prev"][bj] + 1]]
        H64[:], b64[:] = np.asarray(H, np.float64), np.asarray(bv, np.float64)

    def add(offs, Js, r, J64, r64):
        Js, r = [np.asarray(J, np.float64).astype(LD) for J in Js], np.asarray(r, np.float64).astype(LD)
        for oi, Ji, Ji64 in zip(offs, Js, J64):
            bv[oi:oi + Ji.shape[1]] -= Ji.T @ r
            b64[oi:oi + Ji.shape[1]] -= Ji64.T @ r64
            for oj, Jj, Jj64 in zip(offs, Js, J64):
                H[oi:oi + Ji.shape[1], oj:oj + Jj.shape[1]] += Ji.T @ Jj
                H64[oi:oi + Ji.shape[1], oj:oj + Jj.shape[1]] += Ji64.T @ Jj64

    for i in jl["sbp"]:
        pr = w.sb_priors[i]
        blk = sb_blk[int(pr["sb_idx"])]
        r, J = op.eval_speed_bias_error(pr["meas"], pr["sqrt_info"], xlin[blk])
        r2, J2 = op.eval_speed_bias_error(pr["meas"], pr["sqrt_info"], pert(xlin[blk]))
        add([col[blk]], [J], r, [J2], r2)
    for t in jl["imu"]:
        T = w.imu_terms[t]
        smp = w.imu_samples[T["sample_offset"]:T["sample_offset"] + T["sample_count"]]
        blks = [pose_blk[int(T["pose0"])], sb_blk[int(T["sb0"])], pose_blk[int(T["pose1"])], sb_blk[int(T["sb1"])]]
        ref = None
        if imu_cache is not None and t in imu_cache and imu_cache[t][1]:
            ref = imu_cache[t][0]
        r, J, _, _ = op.eval_imu(w.imu_params, smp, T["t0_ns"], T["t1_ns"], *[xlin[b] for b in blks], sb_ref=ref)
        r2, J2, _, _ = op.eval_imu(w.imu_params, smp, T["t0_ns"], T["t1_ns"], *[pert(xlin[b]) for b in blks], sb_ref=ref)
        add([col[b] for b in blks], J, r, J2, r2)
    # landmarks: per landmark, its pose blocks W (6 per frame x 3), V, b_l; eliminated with an explicit 3x3 inverse
    obs = w.obs
    lms = jl["lms"]
    sel = np.isin(obs["lm_idx"], np.asarray(lms, np.uint32)) & (obs["sqrt_info"] != 0.0)
    oi = np.nonzero(sel)[0]
    R = np.zeros((len(obs), 2))
    J0 = np.zeros((len(obs), 2, 6))
    J1 = np.zeros((len(obs), 2, 3))
    R2, J02, J12 = np.zeros_like(R), np.zeros_like(J0), np.zeros_like(J1)
    for c in np.unique(obs["cam_idx"][oi]):
        s = oi[obs["cam_idx"][oi] == c]
        o = obs[s]
        poses = np.array([xlin[pose_blk[int(f)]][:7] for f in o["pose_idx"]])
        r, j0, j1, _ = op.eval_reprojection(w.cameras[c], poses, w.landmarks[o["lm_idx"]], w.extrinsics[o["ext_idx"]], o["z"], o["sqrt_info"])
        R[s], J0[s], J1[s] = r, j0, j1
        r, j0, j1, _ = op.eval_reprojection(w.cameras[c], pert(poses), pert(w.landmarks[o["lm_idx"]]), w.extrinsics[o["ext_idx"]], o["z"], o["sqrt_info"])
        R2[s], J02[s], J12[s] = r, j0, j1
    if use_cauchy and len(oi):       # Corrector with rho'' < 0: residual and Jacobians scaled by sqrt(rho')
        for Rx, J0x, J1x in ((R, J0, J1), (R2, J02, J12)):
            wq = np.sqrt(1.0 / (1.0 + (Rx[oi] ** 2).sum(1)))
            Rx[oi] *= wq[:, None]
            J0x[oi] *= wq[:, None, None]
            J1x[oi] *= wq[:, None, None]
    by_lm = {}
    for i in oi:
        by_lm.setdefault(int(obs["lm_idx"][i]), []).append(i)
    for l in lms:
        ids = by_lm.get(l, [])
        if not ids:
            continue            # every observation removed: nothing to eliminate
        frames = sorted({int(obs["pose_idx"][i]) for i in ids})
        fpos = {f: k for k, f in enumerate(frames)}
        V = np.zeros((3, 3), LD)
        bl = np.zeros(3, LD)
        Wl = np.zeros((6 * len(frames), 3), LD)
        V64, bl64, Wl64 = np.zeros((3, 3)), np.zeros(3), np.zeros((6 * len(frames), 3))
        for i in ids:
            j0, j1, r = J0[i].astype(LD), J1[i].astype(LD), R[i].astype(LD)
            f = int(obs["pose_idx"][i])
            o6 = col[pose_blk[f]]
            V += j1.T @ j1
            bl -= j1.T @ r
            Wl[6 * fpos[f]:6 * fpos[f] + 6] += j0.T @ j1
            H[o6:o6 + 6, o6:o6 + 6] += j0.T @ j0
            bv[o6:o6 + 6] -= j0.T @ r
            V64 += J12[i].T @ J12[i]
            bl64 -= J12[i].T @ R2[i]
            Wl64[6 * fpos[f]:6 * fpos[f] + 6] += J02[i].T @ J12[i]
            H64[o6:o6 + 6, o6:o6 + 6] += J02[i].T @ J02[i]
            b64[o6:o6 + 6] -= J02[i].T @ R2[i]
        Vi = _inv3(V)
        CH, Cb = Wl @ Vi @ Wl.T, Wl @ (Vi @ bl)
        rows = np.concatenate([np.arange(col[pose_blk[f]], col[pose_blk[f]] + 6) for f in frames])
        H[np.ix_(rows, rows)] -= CH
        bv[rows] -= Cb
        pv = precond(np.diag(np.asarray(V, np.float64)))
        kl = _cond_sym(np.asarray(V, np.float64) / np.outer(pv, pv))
        assert kl < 1e12, "landmark %d: its 3x3 block is singular (pass the job's landmarks through well_conditioned)" % l
        kappa_lm = max(kappa_lm, kl)
        Vi64 = _pinv64(V64)
        H64[np.ix_(rows, rows)] -= Wl64 @ Vi64 @ Wl64.T
        b64[rows] -= Wl64 @ (Vi64 @ bl64)
    # dense stage
    gone = np.concatenate([np.arange(col[b], col[b + 1]) for b in range(NB) if jl["marg"][b]] or [np.zeros(0, int)]).astype(int)
    keep = np.concatenate([np.arange(col[b], col[b + 1]) for b in range(NB) if not jl["marg"][b]] or [np.zeros(0, int)]).astype(int)
    U, Wd, V = H[np.ix_(keep, keep)], H[np.ix_(keep, gone)], H[np.ix_(gone, gone)]
    ba, bb = bv[keep], bv[gone]
    kappa_V, rank_V, V_zero = 1.0, 0, True
    if len(gone):
        Vi64 = _pinv64(H64[np.ix_(gone, gone)])
        W64 = H64[np.ix_(keep, gone)]
        Hn64, bn64 = H64[np.ix_(keep, keep)] - W64 @ Vi64 @ W64.T, b64[keep] - W64 @ (Vi64 @ b64[gone])
    else:
        Hn64, bn64 = H64[np.ix_(keep, keep)], b64[keep]
    if len(gone) and np.abs(V).max() > 0:
        V_zero = False
        pb = precond(np.diag(np.asarray(V, np.float64))).astype(LD)
        Vp = 0.5 * (V + V.T) / np.outer(pb, pb)
        kappa_V = _cond_sym(Vp)
        rank_V = len(gone)
        Lc = _cholesky(Vp)
        X = _forward(Lc, (Wd / pb[None, :]).T)          # L^-1 P_b^-1 W^T
        y = _forward(Lc, (bb / pb)[:, None])[:, 0]
        Hn, bn = U - X.T @ X, ba - X.T @ y
    else:
        assert len(gone) == 0 or (np.abs(Wd).max(initial=0) == 0 and np.abs(bb).max(initial=0) == 0), "V = 0 with W or b_b nonzero"
        Hn, bn = U.copy(), ba.copy()       # V^+ = 0: exact
    n = len(keep)
    out = dict(n=n, N=Nd, n_marg=len(gone), H=Hn, b0=bn, kappa_V=kappa_V, kappa_lm=kappa_lm, rank_V=rank_V, V_zero=V_zero)
    # max-norm error bounds of H' and b' (see `bounds`)
    out["err_H"] = C_MEAS * max(float(np.abs(Hn64 - np.asarray(Hn, np.float64)).max(initial=0.0)), EPS * float(np.abs(H64).max(initial=0.0)))
    out["err_b"] = C_MEAS * max(float(np.abs(bn64 - np.asarray(bn, np.float64)).max(initial=0.0)), EPS * float(np.abs(b64).max(initial=0.0)))
    pk = precond(np.diag(np.asarray(Hn, np.float64))) if len(keep) else np.ones(0)
    out["err_b_pre"] = C_MEAS * max(float(np.linalg.norm((bn64 - np.asarray(bn, np.float64)) / pk)), EPS * float(np.linalg.norm(b64[keep] / pk)))
    out["block_kind"] = np.array([k for k, m in zip(jl["kind"], jl["marg"]) if not m], np.int32)
    out["block_idx"] = np.array([i for i, m in zip(jl["idx"], jl["marg"]) if not m], np.uint32)
    out["x0"] = np.concatenate([x[:9 if k == SB else 7] for x, k, m in zip(xlin, jl["kind"], jl["marg"]) if not m] or [np.zeros(0)])
    # spectrum of the preconditioned H' (what the rank threshold eps * n * lambda_max is applied to)
    Hf = np.asarray(Hn, np.float64)
    p = precond(np.diag(Hf)) if n else np.zeros(0)
    if n:
        Hp = 0.5 * (Hn + Hn.T) / np.outer(p.astype(LD), p.astype(LD))
        _, Uv = np.linalg.eigh(np.asarray(Hp, np.float64))
        # eigenvalues as long-double Rayleigh quotients of the double-precision eigenvectors: their error is second order
        # in the eigenvector error, so the gauge eigenvalues resolve far below the rank threshold eps * n * lambda_max
        Ul = Uv.astype(LD)
        lam = np.asarray(np.einsum("ik,ik->k", Ul, Hp @ Ul) / np.einsum("ik,ik->k", Ul, Ul), np.float64)
    else:
        lam, Uv = np.zeros(0), np.zeros((0, 0))
    out.update(p=p, lam=lam, evecs=Uv)
    return out


def rank_band(ref, d=0.0):
    """(lo, hi): the ranks an implementation may report whose preconditioned H' differs from the reference's by at most
    d in the 2-norm.  The threshold is eps * n * lambda_max; by Weyl's theorem each of the implementation's eigenvalues
    lies within d of the reference's, so an eigenvalue is classified exactly unless it lies within d of the threshold
    or within a factor RANK_GAP of it (rounding level).  lo == hi where the rank is well defined."""
    n, lam = ref["n"], ref["lam"]
    if n == 0 or lam.max() <= 0:
        return 0, 0
    thr_lo, thr_hi = EPS * n * max(lam.max() - d, 0.0), EPS * n * (lam.max() + d)
    return int((lam > max(thr_hi * RANK_GAP, thr_hi + d)).sum()), int((lam > min(thr_lo / RANK_GAP, thr_lo - d)).sum())


def bounds(ref):
    """Error bounds of a double-precision implementation against the reference.
      H', b'   C_MEAS times the measured error of the step redone in double precision, with every functor evaluated at
               the states perturbed by one rounding (sums in double, eigen pseudo-inverses of the preconditioned landmark
               and dense blocks), at least C_MEAS * eps times the largest entry summed.  Every double-precision implementation (the device, the oracle, this realisation)
               makes rounding errors of the same first-order size on the same system -- the same condition numbers of
               the same blocks amplify them -- and differs only in summation order and inversion method; C_MEAS covers
               that spread.  A worst-case model (eps * kappa * |term| per inverted block) lies up to 1e6 above the
               errors actually made and lets whole-observation faults through.
      J^T J    the eigen-decomposition of the preconditioned H' has backward error ~ eps * n * lambda_max, and directions
               below the rank threshold (also eps * n * lambda_max) are dropped: C_ROUND * eps * n * lambda_max * p_i p_j
               on top of the H' bound.
      J^T e0   see `check_prior`."""
    return dict(H=ref["err_H"], b=ref["err_b"])


def _ratio(err, bound):
    """max(err / bound); an error where the bound is zero (exact arithmetic) is infinitely over it."""
    if np.any((bound == 0) & (err > 0)):
        return np.inf
    return float((err / np.where(bound > 0, bound, 1.0)).max(initial=0.0))


def check_prior(g, ref, report=None, label=""):
    """Assert that the prior g (download_marg of the device, or OracleProblem.marginalize) is the reference's step.
    Returns {quantity: observed error / bound}; every entry is <= 1."""
    n = ref["n"]
    assert g["n"] == n, (g["n"], n)
    assert np.array_equal(g["block_kind"], ref["block_kind"]) and np.array_equal(g["block_idx"], ref["block_idx"])
    assert np.array_equal(g["x0"], ref["x0"]), "linearisation points differ"
    rank = int(g["status"][1]) if "status" in g else int(g["rank"])
    ratios = {}
    if n == 0:
        assert rank == 0
        return ratios
    # the implementation's rank comes from the eigenvalues of its own preconditioned H' (Weyl: within d of ours), with
    # an eigensolver backward error of a few eps * n * lambda_max
    p = ref["p"]
    Hr = np.asarray(ref["H"], np.float64)
    d = np.linalg.norm((np.asarray(g["H"]) - Hr) / np.outer(p, p), 2) + C_ROUND * EPS * n * max(ref["lam"].max(), 0.0)
    lo, hi = rank_band(ref, d)
    assert lo <= rank <= hi, "%s rank %d outside [%d, %d]" % (label, rank, lo, hi)
    bd = bounds(ref)
    br = np.asarray(ref["b0"], np.float64)
    Hg, bg = np.asarray(g["H"]), np.asarray(g["b0"])
    ratios["H"] = _ratio(np.abs(Hg - Hr), bd["H"])
    ratios["b0"] = _ratio(np.abs(bg - br), bd["b"])
    lam, Uv = ref["lam"], ref["evecs"]
    lmax = max(lam.max(), 0.0)
    JtJ = g["J"].T @ g["J"]
    ratios["JtJ"] = _ratio(np.abs(JtJ - Hr), bd["H"] + C_ROUND * EPS * n * lmax * np.outer(p, p))
    # J^T e0 + b' on the range of the reference (preconditioned coordinates)
    if lo > 0:
        Ur = Uv[:, lam > EPS * n * lmax * RANK_GAP]
        lam_r = lam[lam > EPS * n * lmax * RANK_GAP].min()
        y = Ur.T @ ((g["J"].T @ g["e0"] + br) / p)
        # y = U_r^T P^-1 (b' - b_g) + U_r^T (I - Pi_g) P^-1 b_g, Pi_g the implementation's range.  The first term is the
        # b' error in preconditioned coordinates (err_b_pre, measured like err_H); by Davis-Kahan the implementation's
        # range turns from ours by sin(theta) <= d / lam_r, so the second is at most sin(theta) times the part of b_g
        # outside its range: our null-space part of b', sin(theta) |P^-1 b'| and the b' error.  The sin^2(theta) term
        # assumes the worst alignment of the perturbation; it dominates the bound, about 1e8 above the observed error.
        st = d / lam_r
        bn_null = np.linalg.norm(Uv[:, lam <= EPS * n * lmax * RANK_GAP].T @ (br / p))
        be = ref["err_b_pre"] + st * (bn_null + st * np.linalg.norm(br / p) + ref["err_b_pre"])
        ratios["Jte0"] = np.abs(y).max() / be
    else:
        ratios["Jte0"] = 0.0 if np.abs(g["J"]).max() == 0 else np.inf
    for k, v in ratios.items():
        assert v <= 1.0, "%s %s: error is %.3g x its bound" % (label, k, v)
    if report is not None:
        report.append((label, dict(N=ref["N"], marg=ref["n_marg"], kept=n, rank=rank, band=(lo, hi), rank_defined=rank_band(ref), kappa_V=ref["kappa_V"],
                                   **{k: float(v) for k, v in ratios.items()})))
    return ratios


# ---- the job shapes the tests run (windows from okvis_b200.synthetic, fixed seeds)
STEREO17 = dict(n_frames=17, n_cams=2, n_landmarks=1200)


def well_conditioned(w, lms, limit=1e7):
    """Landmarks whose Cauchy-weighted, preconditioned 3x3 block V has a condition number below `limit` (DESIGN 4b:
    a numerically rank-deficient V amplifies rounding noise by 1/lambda_min in any implementation)."""
    keep = []
    for l in lms:
        o = w.obs[(w.obs["lm_idx"] == l) & (w.obs["sqrt_info"] != 0.0)]
        if len(o) == 0:
            continue
        V = np.zeros((3, 3))
        for c in np.unique(o["cam_idx"]):
            s = o[o["cam_idx"] == c]
            r, _, J1, _ = op.eval_reprojection(w.cameras[c], w.poses[s["pose_idx"]], w.landmarks[s["lm_idx"]], w.extrinsics[s["ext_idx"]], s["z"],
                                               s["sqrt_info"])
            V += np.einsum("nki,nkj,n->ij", J1, J1, 1.0 / (1.0 + (r ** 2).sum(1)))
        d = np.sqrt(np.diag(V))
        if d.min() <= 0:
            continue
        ev = np.linalg.eigvalsh(V / np.outer(d, d))
        if ev[0] > 0 and ev[-1] / ev[0] < limit:
            keep.append(l)
    return np.array(keep, np.uint32)


def track_ends(w):
    L = len(w.landmarks)
    first, last = np.full(L, 1 << 30), np.full(L, -1)
    np.minimum.at(first, w.obs["lm_idx"], w.obs["pose_idx"])
    np.maximum.at(last, w.obs["lm_idx"], w.obs["pose_idx"])
    return first, last


def frames_job(w, n_pose, n_sb, lm_before, n_frames=None, sb_priors=(0,)):
    """Blocks P0 SB0 P1 SB1 ... of the first `n_frames` frames (all by default); poses < n_pose and speed/biases < n_sb
    marginalised, every IMU term between them, and the well-conditioned landmarks whose track ends before frame
    `lm_before`."""
    K = len(w.poses) if n_frames is None else n_frames
    kinds, idx, marg = [], [], []
    for f in range(K):
        kinds += [P, SB]
        idx += [f, f]
        marg += [int(f < n_pose), int(f < n_sb)]
    if n_frames is not None and n_frames < len(w.poses):      # the window continues: end on the next pose
        kinds.append(P)
        idx.append(K)
        marg.append(0)
    _, last = track_ends(w)
    lms = well_conditioned(w, np.nonzero((last >= 0) & (last < lm_before))[0])
    terms = [t for t in range(len(w.imu_terms)) if w.imu_terms[t]["pose1"] < K]
    return abi.make_marg_job(kinds, idx, [-1] * len(kinds), marg, imu_terms=terms, sb_priors=list(sb_priors), landmarks=lms)
