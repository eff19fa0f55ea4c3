"""The covariance reference (tests/covref.py) checked on its own, CPU only.

* the long-double band + arrow selected inverse equals the dense inverse (mpmath at 50 digits for small n, long-double
  Gauss-Jordan above) on the pattern, with constant knots at both ends and in the middle;
* the Schur landmark marginal equals the landmark block of the inverse of the full pose + landmark Gauss-Newton matrix
  built from oracle Jacobians;
* J(t) equals central differences of the oracle spline under the global retraction;
* the comparison metric rejects a transposed block, a band block shifted by one control point, a rotation block off by
  the factor 4 between theta and Ceres' delta, and a landmark marginal without its Sigma_pp term;
* the Ceres-tangent and ambient conversions agree with the oracle's manifold_plus / manifold_plus_jacobian.
"""
import numpy as np
import pytest

import asmref as ar
import covref as cr
import oracle_lib as ol
import sysref as sr
from hyperslam_b200 import synthetic


def const_mask(K, m):
    f = np.zeros(6 * K + m, bool)
    for j in (0, K // 2, K - 1):
        f[6 * j:6 * j + 6] = True
    return f


SHAPES = [(K, beta, m) for beta in (3, 5, 12) for m in (26, 53) for K in sorted({beta + 1, 2 * beta + 3, 40})]


@pytest.mark.parametrize("K,beta,m", SHAPES, ids=[f"b{b}-m{m}-K{K}" for K, b, m in SHAPES])
def test_selected_inverse_equals_dense(K, beta, m):
    S, *_ = sr.make_system(K, beta, m, seed=K + 100 * beta + m)
    fixed = const_mask(K, m)
    Sig, P, minpiv, bad = cr.selected_inverse(S, K, beta, m, fixed)
    assert bad == -1 and minpiv > 1e6 * cr.MIN_PIVOT
    n = 6 * K + m
    ref = cr.dense_inverse_mp(S, fixed) if n <= 80 else cr.dense_inverse_ld(S, fixed)
    kap = cr.kappa(S, fixed)
    err = cr.cov_error(Sig, ref, P)
    assert err < sr.forward_bound(n, kap), (err, kap)
    assert np.all(Sig[fixed] == 0) and np.all(Sig[:, fixed] == 0)
    # packing round trip
    buf = cr.dense_to_packed(Sig, K, beta, m)
    assert np.array_equal(cr.packed_to_dense(buf, K, beta, m), sr.lower_symmetric(np.where(P, Sig, 0).astype(np.float64)))


def test_selected_inverse_rejects_singular():
    """No constant dofs on a system with a null direction: the failing pivot is far below the threshold."""
    K, beta, m = 10, 3, 26
    S, *_ = sr.make_system(K, beta, m, seed=5)
    v = np.zeros(6 * K + m)
    v[24:30] = np.random.default_rng(5).normal(size=6)   # a null direction inside one control point (keeps the band)
    P = np.eye(len(v)) - np.outer(v, v) / (v @ v)
    S0 = P @ S @ P
    _, _, piv, bad = cr.selected_inverse(S0, K, beta, m, np.zeros(len(v), bool))
    print("singular: failing pivot", piv, "dof", bad)
    assert bad >= 0 and abs(piv) < 1e-3 * cr.MIN_PIVOT


def oracle_window(order, seed, num_knots=12, num_landmarks=30, num_imu=120, bearing=20, pose=6):
    base = synthetic.make_window(order=order, num_knots=num_knots, num_landmarks=num_landmarks, num_imu=num_imu, seed=synthetic.SEED_BASE + 1600 + seed)
    win = synthetic.add_bearing_and_pose_factors(base, num_bearing=bearing, num_pose=pose, seed=synthetic.SEED_BASE + 1650 + seed)
    win.knot_const = np.zeros(num_knots, np.uint8)
    win.knot_const[:order] = 1
    win.knot_const[cr.untouched_knots(win)] = 1
    return win


def problem(win):
    ow = ol.OracleWindow(win)
    assert ow.bad == 0
    return ar.problem(ow.evaluate(), win, ow.index_maps())


@pytest.mark.parametrize("order", [4, 6])
def test_landmark_marginal_equals_full_inverse(order):
    win = oracle_window(order, order)
    p = problem(win)
    K, Kbg, Kba, L = p["K"], p["Kbg"], p["Kba"], p["L"]
    n = 6 * K + 3 * (Kbg + Kba) + 2
    fixed = sr.fixed_mask(K, Kbg, Kba, win.knot_const, win.bias_const, win.gravity_const)
    red = ar.assemble(p, np.inf)
    S = red["S"]
    beta = sr.block_bandwidth(S.astype(np.float64), K)
    Sig, P, minpiv, bad = cr.selected_inverse(S, K, beta, n - 6 * K, fixed)
    assert bad == -1
    lm = cr.landmark_marginals(p, Sig)
    H = cr.full_gauss_newton(p)
    full = cr.dense_inverse_ld(H, np.concatenate([fixed, np.zeros(3 * L, bool)]))
    ref = np.stack([full[n + 3 * l:n + 3 * l + 3, n + 3 * l:n + 3 * l + 3] for l in range(L)])
    kap = cr.kappa(H, np.concatenate([fixed, np.zeros(3 * L, bool)]))
    errs = [cr.cov_error(lm[l], ref[l]) for l in range(L)]
    print(f"order {order}: landmark marginal error {max(errs):.3e}, kappa(full) {kap:.3e}, min pivot {minpiv:.3e}")
    assert max(errs) < sr.forward_bound(n + 3 * L, kap)
    # the pose part of the full inverse is the selected inverse on the pattern
    assert cr.cov_error(Sig, full[:n, :n], P) < sr.forward_bound(n + 3 * L, kap)
    # mutation: a landmark marginal without its Sigma_pp term
    bad_lm = cr._landmark_marginals(p, Sig, drop_pp=True)
    assert max(cr.cov_error(bad_lm[l], ref[l]) for l in range(L)) > 100 * sr.forward_bound(n + 3 * L, kap)


def _global_plus(cp, dphi, drho):
    R = synthetic.quat_to_rot(cp[None, :4])[0]
    out = cp.copy()
    out[:4] = synthetic.rot_to_quat((synthetic.so3_exp(dphi[None])[0] @ R)[None])[0]
    if np.dot(out[:4], cp[:4]) < 0:
        out[:4] *= -1
    out[4:7] = cp[4:7] + drho
    return out


@pytest.mark.parametrize("order", [4, 6])
def test_pose_jacobian_central_differences(order):
    win = synthetic.make_window(order=order, num_knots=14, num_landmarks=0, num_imu=0, seed=synthetic.SEED_BASE + 1700)
    kt = win.knots[:, 7]
    left = (order - 1) // 2
    lo, hi = kt[left], kt[len(kt) - 1 - (order - 1 - left)]
    h = 1e-6
    for t in (lo, 0.5 * (kt[5] + kt[6]), kt[7], np.nextafter(hi, -np.inf)):
        base, J = cr.pose_jacobian(win.knots, order, t)
        cps = win.knots[base:base + order].copy()
        v0 = ol.state_evaluate(cps, t, derivative=0, jac=False)[0]
        R0 = synthetic.quat_to_rot(v0[None, :4])[0]
        num = np.zeros((6, 6 * order))
        for mm in range(order):
            for c in range(6):
                vals = []
                for s in (1, -1):
                    d = np.zeros(6)
                    d[c] = s * h
                    q = cps.copy()
                    q[mm] = _global_plus(cps[mm], d[:3], d[3:])
                    v = ol.state_evaluate(q, t, derivative=0, jac=False)[0]
                    th = synthetic.so3_log((synthetic.quat_to_rot(v[None, :4])[0] @ R0.T)[None])[0]
                    vals.append(np.concatenate([th, v[4:7] - v0[4:7]]))
                num[:, 6 * mm + c] = (vals[0] - vals[1]) / (2 * h)
        assert np.abs(num - J).max() < 1e-7, (t, np.abs(num - J).max())


def test_so3_jacobians_against_mpmath():
    """Jr and Jr^-1 of the J(t) reference, entry by entry against 50 digits, for angles from 1e-9 to pi: a few ulps of
    the matrix (whose largest entry is 1) everywhere, including where 1 - cos t and t - sin t cancel."""
    mp = pytest.importorskip("mpmath")
    mp.mp.dps = 50
    rng = np.random.default_rng(3)
    worst = 0.0
    for t in np.concatenate([np.geomspace(1e-9, 3.1, 400), [1e-4, 1.0001e-4, 1e-3, 1.0001e-3, 1e-8, 1e-7, 1.5, 2.0, np.pi]]):
        axis = rng.normal(size=3)
        w = t * axis / np.linalg.norm(axis)
        W = mp.matrix([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
        th = mp.sqrt(mp.mpf(w[0]) ** 2 + mp.mpf(w[1]) ** 2 + mp.mpf(w[2]) ** 2)
        b, c = (1 - mp.cos(th)) / th ** 2, (th - mp.sin(th)) / th ** 3
        e = 1 / th ** 2 - (1 + mp.cos(th)) / (2 * th * mp.sin(th))
        for got, ref in ((cr._so3_Jr(w), mp.eye(3) - b * W + c * W * W), (cr._so3_Jr_inv(w), mp.eye(3) + W / 2 + e * W * W)):
            err = max(abs(mp.mpf(got[i, j]) - ref[i, j]) for i in range(3) for j in range(3))
            worst = max(worst, float(err) / 2.0 ** -53)
    assert worst < 4, worst


def test_metric_rejects_mutations():
    K, beta, m = 12, 3, 26
    S, *_ = sr.make_system(K, beta, m, seed=11)
    fixed = const_mask(K, m)
    Sig, P, _, _ = cr.selected_inverse(S, K, beta, m, fixed)
    ref = cr.dense_inverse_ld(S, fixed)
    n = 6 * K + m
    bound = sr.forward_bound(n, cr.kappa(S, fixed))
    assert cr.cov_error(Sig, ref, P) < bound
    # a transposed off-diagonal block (both copies of the pair)
    T = Sig.copy()
    a, b = slice(18, 24), slice(24, 30)
    T[a, b], T[b, a] = Sig[a, b].T, Sig[b, a].T
    assert cr.cov_error(T, ref, P) > 1e3 * bound
    # the band shifted by one control point: block (j+1, j) read from (j+2, j)
    Sh = Sig.copy()
    for j in range(K - 2):
        Sh[6 * (j + 1):6 * (j + 2), 6 * j:6 * j + 6] = Sig[6 * (j + 2):6 * (j + 3), 6 * j:6 * j + 6]
    assert cr.cov_error(Sh, ref, P) > 1e3 * bound
    # a rotation block off by the factor 4 between theta and Ceres' delta = theta / 2
    R4 = Sig.copy()
    R4[24:27, 24:27] *= 4
    assert cr.cov_error(R4, ref, P) > 1e3 * bound


def test_ceres_conversions_against_oracle_manifold():
    """Ceres' SE3 block (q, p) with the quaternion tangent delta: Plus(x, [theta / 2 | rho]) = (Exp(theta) R, p + rho) to
    first order, so a device-tangent covariance S is T S T^T in Ceres' tangent and P T S T^T P^T in ambient coordinates."""
    rng = np.random.default_rng(3)
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    x = np.concatenate([q, rng.normal(size=3)])
    h = 1e-6
    for c in range(6):
        d_dev = np.zeros(6)
        d_dev[c] = h
        y = ol.manifold_plus(ol.M_SE3, x, cr.T_CERES @ d_dev)
        want = _global_plus(np.concatenate([x, [0.0]]), d_dev[:3], d_dev[3:])[:7]
        assert np.abs(y - want).max() < 1e-11, (c, y - want)
    Pj = ol.manifold_plus_jacobian(ol.M_SE3, x)
    A = rng.normal(size=(6, 6))
    S6 = A @ A.T
    amb = cr.ambient(S6, Pj)
    # ambient covariance = the linear map of device-tangent samples through Plus
    num = np.zeros((7, 6))
    for c in range(6):
        e = np.zeros(6)
        e[c] = h
        num[:, c] = (ol.manifold_plus(ol.M_SE3, x, cr.T_CERES @ e) - ol.manifold_plus(ol.M_SE3, x, -cr.T_CERES @ e)) / (2 * h)
    assert np.abs(num @ S6 @ num.T - amb).max() < 1e-8 * np.abs(amb).max()
    assert np.allclose(cr.ceres_tangent(S6)[:3, :3], S6[:3, :3] / 4)
