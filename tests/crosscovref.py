"""Reference of the covariance blocks outside the selected inverse's pattern (test infrastructure, CPU only), in long
double, from a Sigma on the pattern and the factor of the selected inversion:

* `band_factor`: D and the band + arrow factor L of the equilibrated, masked system (the forward sweep of
  covref.selected_inverse / cov_selinv_kernel);
* `far_columns`: the march of cov_far_column_kernel -- Z = A_hat^-1, for i < j - beta
  Z_ij = -L_ii^-T (sum_{k=i+1..i+beta} L_ki^T Z_kj + L_Ci^T Z_Cj), seeded with the band and arrow of column j -- and
  Sigma_ij = D Z D on the far knot pairs (constant dofs 0);
* `landmark_cross` / `landmark_pair`: Sigma_lq = -V_l^-1 W_l^T Sigma_{span(l), q} and
  Sigma_lm = V_l^-1 W_l^T Sigma_{span(l), span(m)} W_m V_m^-1 from the per-factor outputs (asmref.problem).
"""
from __future__ import annotations

import numpy as np

import covref as cr

LD = np.longdouble


def band_factor(S, K, beta, m, fixed):
    """(d, L): D = diag(S)^-1/2 (1 on constant dofs) and the lower factor of A_hat = D S D (n x n, zero off the band and
    the arrow) in long double."""
    n, np_ = 6 * K + m, 6 * K
    d, A = cr.equilibrated(S, fixed)
    A = A.copy()
    L = np.zeros((n, n), LD)
    for j in range(K):
        c = slice(6 * j, 6 * j + 6)
        Ljj, _ = cr._chol_ld(A[c, c])
        assert Ljj is not None, f"block {j} is not positive definite"
        R = np.r_[6 * j + 6:min(6 * (j + beta + 1), np_), np_:n]
        L[c, c] = Ljj
        L[R, c] = A[R, c] @ cr._tri_inv_ld(Ljj).T
        A[np.ix_(R, R)] -= L[R, c] @ L[R, c].T
    Lc, _ = cr._chol_ld(A[np_:, np_:])
    assert Lc is not None, "corner is not positive definite"
    L[np_:, np_:] = Lc
    return d, L


def all_far(K, beta):
    """Every far column down to row 0: {column block j: lowest row block}."""
    return {j: 0 for j in range(beta + 1, K)}


def far_columns(Sig, d, L, K, beta, m, fixed, cols):
    """Sigma (dense, the pattern filled) with the far knot pairs (i, j), lo <= i < j - beta, of every column j in `cols`
    ({j: lo}) added by the back-substitution march; long double."""
    np_ = 6 * K
    fixed = np.asarray(fixed, bool)
    d = np.asarray(d, LD)
    out = np.asarray(Sig, LD).copy()
    Z = out / (d[:, None] * d[None, :])
    for j, lo in cols.items():
        cj = slice(6 * j, 6 * j + 6)
        col = {k: Z[6 * k:6 * k + 6, cj] for k in range(j - beta, j)}
        ZC = Z[np_:, cj]
        for i in range(j - beta - 1, lo - 1, -1):
            ci = slice(6 * i, 6 * i + 6)
            T = L[np_:, ci].T @ ZC
            for k in range(i + 1, i + beta + 1):
                T = T + L[6 * k:6 * k + 6, ci].T @ col[k]
            Zi = -(cr._tri_inv_ld(L[ci, ci]).T @ T)
            col[i] = Zi
            blk = Zi * d[ci][:, None] * d[cj][None, :]
            blk[fixed[ci], :] = 0
            blk[:, fixed[cj]] = 0
            out[ci, cj] = blk
            out[cj, ci] = blk.T
    return out


def landmark_terms(p):
    """Per landmark (first control point, V, W) or None (unobserved), as covref uses them."""
    return cr._landmark_terms(p)


def landmark_cross(terms, Sig, l, dofs):
    """Sigma_lq (3 x len(dofs)) = -V_l^-1 W_l^T Sigma_{span(l), dofs}; zero for an unobserved landmark."""
    t = terms[l]
    if t is None:
        return np.zeros((3, len(dofs)), LD)
    lo, V, W = t
    r = np.arange(6 * lo, 6 * lo + W.shape[0])
    return -(cr._inv3(V) @ W.T @ np.asarray(Sig, LD)[np.ix_(r, np.asarray(dofs))])


def landmark_pair(terms, Sig, l, m):
    """Sigma_lm (3 x 3) = V_l^-1 W_l^T Sigma_{span(l), span(m)} W_m V_m^-1 for l != m; zero when either is unobserved."""
    if terms[l] is None or terms[m] is None:
        return np.zeros((3, 3), LD)
    (la, Va, Wa), (lb, Vb, Wb) = terms[l], terms[m]
    ra = np.arange(6 * la, 6 * la + Wa.shape[0])
    rb = np.arange(6 * lb, 6 * lb + Wb.shape[0])
    return cr._inv3(Va) @ Wa.T @ np.asarray(Sig, LD)[np.ix_(ra, rb)] @ Wb @ cr._inv3(Vb)
