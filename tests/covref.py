"""Reference tools for the marginal covariances (test infrastructure, CPU only).

* `selected_inverse`: a long-double restatement of the natural-order band + arrow Cholesky and its Takahashi selected
  inverse (what cov_selinv_kernel computes): every entry of S^-1 on the block band of half-width beta, the arrow and the
  corner, after equilibration D = diag(S)^-1/2 and with constant dofs masked; the smallest equilibrated pivot;
* `dense_inverse_ld` / `dense_inverse_mp`: Gauss-Jordan in long double, LU in mpmath (small n), over the non-constant dofs;
* `landmark_marginals`: Sigma_ll = V^-1 + V^-1 W^T Sigma_pp W V^-1 from the per-factor outputs (asmref.problem);
* `full_gauss_newton`: the pose + landmark Gauss-Newton matrix (no Schur complement), to check the landmark marginals;
* `pose_jacobian`: J(t), the Jacobian of the interpolated pose [theta | p] (global rotation tangent) with respect to the
  tangents of its k control points, and `interpolated`: J(t) Sigma J(t)^T;
* `cov_error`: max |dSigma_ij| / sqrt(Sigma_ii Sigma_jj) over a set of entries, compared with sysref.forward_bound;
* the conversions of a device-tangent SE3 block to Ceres' quaternion tangent (delta = theta / 2) and to ambient
  coordinates (P T Sigma T^T P^T, P = PlusJacobian).
"""
from __future__ import annotations

import numpy as np

import sysref as sr
from hyperslam_b200 import synthetic

LD = np.longdouble
MIN_PIVOT = 1e-10     # kCovMinPivot (hb200_cov.cuh)


# ---- selected inverse -----------------------------------------------------------------------------------------------
def _chol_ld(A):
    n = A.shape[0]
    L = np.zeros_like(A)
    piv = []
    for k in range(n):
        p = A[k, k] - (L[k, :k] * L[k, :k]).sum()
        piv.append(p)
        if not p > 0:
            return None, piv
        L[k, k] = np.sqrt(p)
        L[k + 1:, k] = (A[k + 1:, k] - L[k + 1:, :k] @ L[k, :k]) / L[k, k]
    return L, piv


def _tri_inv_ld(L):
    n = L.shape[0]
    Li = np.zeros_like(L)
    for c in range(n):
        Li[c, c] = 1 / L[c, c]
        for i in range(c + 1, n):
            Li[i, c] = -(L[i, c:i] @ Li[c:i, c]) / L[i, i]
    return Li


def equilibrated(S, fixed):
    """(d, A_hat) in long double: D = diag(S)^-1/2 (1 on constant dofs), constant rows / columns -> identity."""
    S = np.asarray(S, dtype=LD)
    fixed = np.asarray(fixed, dtype=bool)
    dg = np.diagonal(S).copy()
    d = np.where(fixed | ~(dg > 0), LD(1), 1 / np.sqrt(np.where(dg > 0, dg, 1)))
    A = S * d[:, None] * d[None, :]
    A[fixed, :] = 0
    A[:, fixed] = 0
    A[fixed, fixed] = 1
    return d, A


def selected_inverse(S, K, beta, m, fixed):
    """Band + arrow entries of Sigma = S^-1 (constant dofs 0).  Returns (Sigma dense n x n with zeros off the pattern,
    pattern mask, min pivot, first failing dof or -1)."""
    n = 6 * K + m
    np_ = 6 * K
    d, A = equilibrated(S, fixed)
    A = A.copy()
    L = np.zeros((n, n), LD)
    minpiv = np.inf
    rows = lambda j: np.r_[6 * j + 6:min(6 * (j + beta + 1), np_), np_:n]
    for j in range(K):
        c = slice(6 * j, 6 * j + 6)
        Ljj, piv = _chol_ld(A[c, c])
        minpiv = min([minpiv] + [float(p) for p in piv if p > MIN_PIVOT])
        bad = [i for i, p in enumerate(piv) if not p > MIN_PIVOT]
        if bad:
            return None, None, float(piv[bad[0]]), 6 * j + bad[0]
        R = rows(j)
        L[c, c] = Ljj
        L[R, c] = A[R, c] @ _tri_inv_ld(Ljj).T
        A[np.ix_(R, R)] -= L[R, c] @ L[R, c].T
    Lc, piv = _chol_ld(A[np_:, np_:])
    bad = [i for i, p in enumerate(piv) if not p > MIN_PIVOT]
    if bad:
        return None, None, float(piv[bad[0]]), np_ + bad[0]
    minpiv = min([minpiv] + [float(p) for p in piv])
    Z = np.zeros((n, n), LD)
    Yc = _tri_inv_ld(Lc)
    Z[np_:, np_:] = Yc.T @ Yc
    for j in range(K - 1, -1, -1):
        c = slice(6 * j, 6 * j + 6)
        R = rows(j)
        Li = _tri_inv_ld(L[c, c])
        X = L[R, c] @ Li
        ZS = -Z[np.ix_(R, R)] @ X
        Z[R, c] = ZS
        Z[c, R] = ZS.T
        Zjj = Li.T @ Li - X.T @ ZS
        Z[c, c] = (Zjj + Zjj.T) / 2
    Sig = Z * d[:, None] * d[None, :]
    fixed = np.asarray(fixed, dtype=bool)
    Sig[fixed, :] = 0
    Sig[:, fixed] = 0
    return Sig, pattern(K, beta, m), minpiv, -1


def pattern(K, beta, m):
    """Entries the selected inverse computes: pose pairs within beta blocks, the arrow and the corner."""
    n, np_ = 6 * K + m, 6 * K
    blk = np.arange(n) // 6
    P = np.abs(blk[:, None] - blk[None, :]) <= beta
    P[np_:, :] = True
    P[:, np_:] = True
    return P


def packed_to_dense(packed, K, beta, m):
    """P | A | C of the packed layout -> dense symmetric n x n (zeros off the pattern)."""
    Lay = sr.layout(K, beta, m)
    buf = np.zeros(Lay["total"])
    buf[:Lay["oC"] + m * m] = packed
    S, *_ = sr.unpack_system(buf, K, beta, m)
    return S


def dense_to_packed(Sig, K, beta, m):
    """Dense Sigma -> what hb200_get_covariance returns (diagonal blocks and corner full, padding 0)."""
    Lay = sr.layout(K, beta, m)
    Sig = np.asarray(Sig, dtype=np.float64)
    buf = np.zeros(Lay["oC"] + m * m)
    idx, row, col = sr._band_slots(Lay)
    buf[idx] = Sig[row, col]
    np_ = 6 * K
    buf[Lay["oA"]:Lay["oC"]] = Sig[np_:, :np_].ravel()
    buf[Lay["oC"]:] = Sig[np_:, np_:].ravel()
    return buf


# ---- dense inverses over the non-constant dofs ------------------------------------------------------------------------
def dense_inverse_ld(S, fixed):
    """Gauss-Jordan (partial pivoting) in long double of S over the non-constant dofs; zeros elsewhere."""
    fixed = np.asarray(fixed, dtype=bool)
    keep = np.nonzero(~fixed)[0]
    A = np.asarray(S, dtype=LD)[np.ix_(keep, keep)].copy()
    k = A.shape[0]
    M = np.concatenate([A, np.eye(k, dtype=LD)], axis=1)
    for c in range(k):
        p = c + int(np.argmax(np.abs(M[c:, c])))
        if p != c:
            M[[c, p]] = M[[p, c]]
        M[c] /= M[c, c]
        f = M[:, c].copy()
        f[c] = 0
        M -= f[:, None] * M[c][None, :]
    out = np.zeros(S.shape, LD)
    out[np.ix_(keep, keep)] = M[:, k:]
    return out


def dense_inverse_mp(S, fixed, dps=50):
    import mpmath
    fixed = np.asarray(fixed, dtype=bool)
    keep = np.nonzero(~fixed)[0]
    with mpmath.workdps(dps):
        A = mpmath.matrix([[mpmath.mpf(float(v)) for v in row] for row in np.asarray(S, np.float64)[np.ix_(keep, keep)]])
        Ai = A ** -1
        inv = np.array([[float(Ai[i, j]) for j in range(len(keep))] for i in range(len(keep))])
    out = np.zeros(S.shape)
    out[np.ix_(keep, keep)] = inv
    return out


# ---- metrics ----------------------------------------------------------------------------------------------------------
def cov_error(Sig, Sig_ref, mask=None):
    """max |Sig - Sig_ref|_ij / sqrt(Sig_ref_ii Sig_ref_jj) over mask (entries with a zero diagonal excluded)."""
    ref = np.asarray(Sig_ref, dtype=LD)
    dg = np.sqrt(np.abs(np.diagonal(ref)).astype(np.float64))
    E = np.abs(np.asarray(Sig, dtype=LD) - ref).astype(np.float64)
    ok = (dg[:, None] > 0) & (dg[None, :] > 0)
    if mask is not None:
        ok &= mask
    if not ok.any():
        return 0.0
    return float((E[ok] / (dg[:, None] * dg[None, :])[ok]).max())


def kappa(S, fixed):
    """1-norm condition number of the equilibrated, masked S."""
    _, A = equilibrated(S, fixed)
    return float(np.linalg.cond(A.astype(np.float64), 1))


# ---- landmarks ------------------------------------------------------------------------------------------------------
def _landmark_terms(p):
    """Per landmark: (first control point, V (3 x 3), W (rows x 3), observations) in long double from asmref.problem."""
    import asmref as ar
    fams = ar._families(p, LD)
    k = p["order"]
    obs = []
    if "pixel" in fams:
        J, r, w, _, _ = fams["pixel"]
        obs.append((J, p["out"]["v_Jl"].astype(LD), w, np.asarray(p["vb"]), np.asarray(p["v_lm"])))
    if "bearing" in fams:
        J, r, w, _, _ = fams["bearing"]
        obs.append((J, p["out"]["b_Jl"].astype(LD)[:, None, :], w, np.asarray(p["bb"]), np.asarray(p["b_lm"])))
    L = p["L"]
    # each family's factors grouped by landmark (stable: factor order kept within a landmark)
    groups = []
    for Jp, Jl, w, base, lm in obs:
        order = np.argsort(lm, kind="stable")
        cuts = np.searchsorted(lm[order], np.arange(L + 1))
        groups.append((Jp, Jl, w, base, order, cuts))
    out = []
    for l in range(L):
        sel = []
        for Jp, Jl, w, base, order, cuts in groups:
            i = order[cuts[l]:cuts[l + 1]]
            sel.append((Jp[i], Jl[i], w[i], base[i]))
        bases = np.concatenate([s[3] for s in sel]) if sel else np.zeros(0, np.int64)
        if bases.size == 0:
            out.append(None)
            continue
        lo = int(bases.min())
        rows = 6 * (int(bases.max()) - lo + k)
        V = np.zeros((3, 3), LD)
        W = np.zeros((rows, 3), LD)
        for Jp, Jl, w, base in sel:
            for f in range(len(w)):
                wJl = Jl[f] * w[f]
                V += wJl.T @ Jl[f]
                o = 6 * (int(base[f]) - lo)
                W[o:o + 6 * k] += Jp[f].T @ wJl
        out.append((lo, V, W))
    return out


def landmark_marginals(p, Sig):
    """(L, 3, 3) Sigma_ll = V^-1 + V^-1 W^T Sigma_pp W V^-1 (zero for unobserved landmarks); drop_pp leaves Sigma_pp out."""
    return _landmark_marginals(p, Sig, False)


def _landmark_marginals(p, Sig, drop_pp):
    terms = _landmark_terms(p)
    Sig = np.asarray(Sig, dtype=LD)
    out = np.zeros((p["L"], 3, 3), LD)
    for l, t in enumerate(terms):
        if t is None:
            continue
        lo, V, W = t
        Vi = _inv3(V)
        r = slice(6 * lo, 6 * lo + W.shape[0])
        M = Vi if drop_pp else Vi + Vi @ W.T @ Sig[r, r] @ W @ Vi
        out[l] = (M + M.T) / 2
    return out


def _inv3(V):
    L, _ = _chol_ld(V)
    Li = _tri_inv_ld(L)
    return Li.T @ Li


def full_gauss_newton(p):
    """The pose + landmark Gauss-Newton matrix (n + 3L), undamped, in long double; landmark dofs follow the reduced ones."""
    import asmref as ar
    ref = ar.assemble(p, np.inf, skip_landmarks=range(p["L"]))
    n, L = ref["n"], p["L"]
    H = np.zeros((n + 3 * L, n + 3 * L), LD)
    H[:n, :n] = ref["S"]
    for l, t in enumerate(_landmark_terms(p)):
        if t is None:
            continue
        lo, V, W = t
        c = slice(n + 3 * l, n + 3 * l + 3)
        r = slice(6 * lo, 6 * lo + W.shape[0])
        H[c, c] = V
        H[r, c] = W
        H[c, r] = W.T
    return H


# ---- interpolated pose --------------------------------------------------------------------------------------------------
def _quat_to_rot(q):
    return synthetic.quat_to_rot(np.asarray(q, np.float64)[None])[0]


def pose_jacobian(knots, order, t):
    """(base, J (6, 6k)) of the pose [theta | p] at stamp t with respect to the tangents [phi | rho] of control points
    base .. base+k-1 (global rotation tangent): J_m = [D_m 0 ; 0 (lambda_m - lambda_{m+1}) I]."""
    k = order
    base, u, inv_dt = synthetic.segment(knots[:, 7], k, np.array([t], np.float64))
    base = int(base[0])
    if base < 0 or base + k > knots.shape[0]:
        return -1, None
    Mc = synthetic.blending_matrix(k)                 # cumulative: lambda_j(u) = sum_n Mc[j, n] u^n, lambda_0 = 1
    uu = float(u[0])
    lam = np.append(Mc @ (uu ** np.arange(k)), 0.0)
    R = [_quat_to_rot(knots[base + j, :4]) for j in range(k)]
    P = R[0].copy()
    Ms = []
    for j in range(1, k):
        d = synthetic.so3_log((R[j - 1].T @ R[j])[None])[0]
        w = lam[j] * d
        A = synthetic.so3_exp(w[None])[0]
        Jr = _so3_Jr(w)
        G = _so3_Jr_inv(d) @ R[j].T
        Pn = P @ A
        Ms.append(lam[j] * Pn @ Jr @ G)
        P = Pn
    J = np.zeros((6, 6 * k))
    for mm in range(k):
        D = (np.eye(3) if mm == 0 else Ms[mm - 1]) - (Ms[mm] if mm + 1 < k else 0.0)
        J[:3, 6 * mm:6 * mm + 3] = D
        J[3:, 6 * mm + 3:6 * mm + 6] = (lam[mm] - lam[mm + 1]) * np.eye(3)
    return base, J


def _hat(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


# Jr = I - b W + c W^2 and Jr^-1 = I + W/2 + e W^2.  b = 2 sin^2(t/2)/t^2 does not cancel; t - sin t and
# 1 - (t/2) cot(t/2) do, so c and e take their Taylor series below t^2 = 0.05, where the long-double closed forms would
# lose more than a tenth of a double's ulp.
_C_SERIES = np.array([LD(1) / 39916800, LD(-1) / 362880, LD(1) / 5040, LD(-1) / 120, LD(1) / 6])       # highest power first
_E_SERIES = np.array([LD(691) / 1307674368000, LD(1) / 47900160, LD(1) / 1209600, LD(1) / 30240, LD(1) / 720, LD(1) / 12])


def _so3_Jr(w):
    w = np.asarray(w, LD)
    t2 = w @ w
    t = np.sqrt(t2)
    H = _hat(w)
    b = LD(0.5) - t2 / 24 if t2 < 1e-16 else 2 * np.sin(t / 2) ** 2 / t2
    c = np.polyval(_C_SERIES, t2) if t2 < 0.05 else (t - np.sin(t)) / (t2 * t)
    return (np.eye(3, dtype=LD) - b * H + c * H @ H).astype(np.float64)


def _so3_Jr_inv(w):
    w = np.asarray(w, LD)
    t2 = w @ w
    t = np.sqrt(t2)
    H = _hat(w)
    e = np.polyval(_E_SERIES, t2) if t2 < 0.05 else 1 / t2 - (1 + np.cos(t)) / (2 * t * np.sin(t))
    return (np.eye(3, dtype=LD) + H / 2 + e * H @ H).astype(np.float64)


def interpolated(knots, order, t, Sig):
    """J(t) Sigma_{span} J(t)^T (6 x 6) in long double, or (None) outside the valid span."""
    base, J = pose_jacobian(knots, order, t)
    if base < 0:
        return None
    r = slice(6 * base, 6 * (base + order))
    Jl = J.astype(LD)
    out = Jl @ np.asarray(Sig, LD)[r, r] @ Jl.T
    return (out + out.T) / 2


def untouched_knots(win):
    """Knots no factor of the window reaches (outside every factor's control-point span): their rows of J^T J are zero,
    so a covariance needs them constant.  The synthetic windows keep factor stamps inside the valid span, which leaves
    the last knot untouched."""
    k, K = win.order, win.knots.shape[0]
    stamps = np.concatenate([win.v_stamp, win.i_stamp, win.b_stamp, win.m_stamp])
    hit = np.zeros(K, bool)
    if stamps.size:
        base = synthetic.segment(win.knots[:, 7], k, stamps)[0]
        for a in range(k):
            hit[base + a] = True
    return ~hit


# ---- Ceres conventions ------------------------------------------------------------------------------------------------
T_CERES = np.diag([0.5, 0.5, 0.5, 1.0, 1.0, 1.0])   # device tangent [theta | rho] -> Ceres' quaternion tangent [theta / 2 | rho]


def ceres_tangent(S6):
    """Covariance of an SE3 block in Ceres' tangent (delta = theta / 2): T S T^T."""
    return T_CERES @ S6 @ T_CERES.T


def ambient(S6, plus_jacobian):
    """Ambient (7 x 7) covariance of an SE3 block: P T S T^T P^T with P = the block's PlusJacobian (7 x 6)."""
    return plus_jacobian @ ceres_tangent(S6) @ plus_jacobian.T
