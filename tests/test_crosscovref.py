"""The reference of the covariance blocks outside the selected inverse's pattern (tests/crosscovref.py), CPU only.

* the far-column march from the long-double selected inverse and its factor equals the dense long-double inverse on
  every knot pair more than beta apart, for beta = 1 .. 6, m = 2 and m = 26, with constant knots at both ends; a march
  stopped early gives the same rows; the far entries it checks are far from zero;
* landmark x state and landmark x landmark blocks from the landmark formulas equal the blocks of the inverse of the
  full pose + landmark Gauss-Newton matrix built from oracle Jacobians (orders 4 and 6); leaving the far knot pairs out
  of Sigma_{span(l), span(m)} is caught.
"""
import numpy as np
import pytest

import asmref as ar
import covref as cr
import crosscovref as xr
import sysref as sr
from test_covref import oracle_window, problem


def ends_fixed(K, m):
    f = np.zeros(6 * K + m, bool)
    f[:6] = True
    f[6 * (K - 1):6 * K] = True
    return f


SHAPES = [(beta, m) for beta in range(1, 7) for m in (2, 26)]


@pytest.mark.parametrize("beta,m", SHAPES, ids=[f"b{b}-m{m}" for b, m in SHAPES])
def test_far_columns_equal_dense(beta, m):
    K = 3 * beta + 5
    n = 6 * K + m
    S, *_ = sr.make_system(K, beta, m, seed=300 + 10 * beta + m)
    fixed = ends_fixed(K, m)
    Sig, P, _, bad = cr.selected_inverse(S, K, beta, m, fixed)
    assert bad == -1
    d, L = xr.band_factor(S, K, beta, m, fixed)
    full = xr.far_columns(Sig, d, L, K, beta, m, fixed, xr.all_far(K, beta))
    ref = cr.dense_inverse_ld(S, fixed)
    bound = sr.forward_bound(n, cr.kappa(S, fixed))
    far = ~P
    err = cr.cov_error(full, ref, far)
    dg = np.sqrt(np.abs(np.diagonal(ref)).astype(np.float64))
    with np.errstate(divide="ignore", invalid="ignore"):
        corr = np.abs(ref.astype(np.float64)) / np.outer(dg, dg)
    biggest = float(np.nanmax(np.where(far, corr, 0)))
    print(f"beta {beta} m {m}: far error {err:.3e}, bound {bound:.3e}, largest far correlation {biggest:.3e}")
    assert err < bound, (err, bound)
    assert biggest >= 1e3 * bound, (biggest, bound)
    assert np.all(full[fixed] == 0) and np.all(full[:, fixed] == 0)
    # the pattern is left as it was; a march that stops early gives the same rows
    assert np.array_equal(full[P], np.asarray(Sig, np.longdouble)[P])
    j, lo = K - 1, K // 2 - beta
    part = xr.far_columns(Sig, d, L, K, beta, m, fixed, {j: lo})
    cj = slice(6 * j, 6 * j + 6)
    assert np.array_equal(part[6 * lo:6 * (j - beta), cj], full[6 * lo:6 * (j - beta), cj])
    assert np.all(part[:6 * lo, cj] == 0)


@pytest.mark.parametrize("order", [4, 6])
def test_landmark_blocks_equal_full_inverse(order):
    win = oracle_window(order, order, num_knots=24, num_landmarks=40, num_imu=240)   # landmark spans more than beta apart
    p = problem(win)
    K, Kbg, Kba, L = p["K"], p["Kbg"], p["Kba"], p["L"]
    m = 3 * (Kbg + Kba) + 2
    n = 6 * K + m
    fixed = sr.fixed_mask(K, Kbg, Kba, win.knot_const, win.bias_const, win.gravity_const)
    S = ar.assemble(p, np.inf)["S"]
    beta = sr.block_bandwidth(S.astype(np.float64), K)
    assert K > beta + 2
    Sig, P, _, bad = cr.selected_inverse(S, K, beta, m, fixed)
    assert bad == -1
    d, Lf = xr.band_factor(S, K, beta, m, fixed)
    full = xr.far_columns(Sig, d, Lf, K, beta, m, fixed, xr.all_far(K, beta))
    terms = xr.landmark_terms(p)
    H = cr.full_gauss_newton(p)
    hfixed = np.concatenate([fixed, np.zeros(3 * L, bool)])
    inv = cr.dense_inverse_ld(H, hfixed)
    bound = sr.forward_bound(n + 3 * L, cr.kappa(H, hfixed))

    def assembled(Sg):
        """The landmark rows of the joint covariance from the formulas (diagonal blocks from the inverse)."""
        G = inv.copy()
        for l in range(L):
            rl = slice(n + 3 * l, n + 3 * l + 3)
            G[rl, :n] = xr.landmark_cross(terms, Sg, l, np.arange(n))
            G[:n, rl] = G[rl, :n].T
            for mm in range(L):
                if mm != l:
                    G[rl, n + 3 * mm:n + 3 * mm + 3] = xr.landmark_pair(terms, Sg, l, mm)
        return G

    mask = np.zeros(H.shape, bool)
    mask[n:, :] = True
    mask[:, n:] = True
    err = cr.cov_error(assembled(full), inv, mask)
    # the far knot pairs left out of Sigma: the landmark blocks whose spans are far apart go wrong
    err_band_only = cr.cov_error(assembled(Sig), inv, mask)
    print(f"order {order}: beta {beta}, landmark blocks error {err:.3e}, bound {bound:.3e}; without far pairs {err_band_only:.3e}")
    assert err < bound, (err, bound)
    assert err_band_only > 1e3 * bound, (err_band_only, bound)
