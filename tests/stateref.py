"""Reference for the joint covariance of the interpolated state (test infrastructure, CPU only).

x(t) = [theta p | omega v | b_g b_a] (18 rows): the pose [theta | p] of covref.pose_jacobian (global rotation tangent,
p <- p + rho), the body velocity of hb200_interpolate (omega the body rate, v = R^T pdot) and the two bias splines at t.

* `state_jacobian`: J(t) (18 x (6k + 24)) with respect to the tangents [phi | rho] of the stamp's k control points and
  the 4 knots of each bias spline, in long double.  The pose rows are covref.pose_jacobian's; the rate rows come from a
  long-double restatement of the Sommer recursion written as one forward sweep, with P_j = R_0 A_1 .. A_j,
  A_j = Exp(lambda_j d_j), G_j = Jr^-1(d_j) R_j^T:
      d omega / d phi_m = R^T (Y_m - Y_{m+1}),  Y_j = P_j (hat(A_j^T w_{j-1}) lambda_j Jr(lambda_j d_j) + lamd_j I) G_j,
      d v / d phi_m = hat(v) R^T D_m,  d v / d rho_m = (lamd_m - lamd_{m+1}) R^T,
  the bias rows are the bias basis weights (lb_m - lb_{m+1}) I;
* `interpolated_state`: J(t) Sigma_span J(t)^T in long double, symmetrised; None outside the valid spans.
"""
from __future__ import annotations

import numpy as np

import covref as cr
from hyperslam_b200 import synthetic

LD = np.longdouble
BIAS_ORDER = 4
DIM = 18


def _hat(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]], dtype=LD)


def _quat_to_rot(q):
    x, y, z, w = (LD(float(c)) for c in q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]], dtype=LD)


def _increment(qa, qb):
    """d = Log(R_a^T R_b) from the quaternions, in long double (sign-independent)."""
    a = np.asarray(qa, LD)
    b = np.asarray(qb, LD)
    ac = np.array([-a[0], -a[1], -a[2], a[3]], LD)
    q = np.array([ac[3] * b[0] + ac[0] * b[3] + ac[1] * b[2] - ac[2] * b[1],
                  ac[3] * b[1] - ac[0] * b[2] + ac[1] * b[3] + ac[2] * b[0],
                  ac[3] * b[2] + ac[0] * b[1] - ac[1] * b[0] + ac[2] * b[3],
                  ac[3] * b[3] - ac[0] * b[0] - ac[1] * b[1] - ac[2] * b[2]], LD)
    if q[3] < 0:
        q = -q
    n = np.sqrt(q[:3] @ q[:3])
    if n == 0:
        return np.zeros(3, LD)
    return 2 * np.arctan2(n, q[3]) / n * q[:3]


def _exp(w):
    t2 = w @ w
    t = np.sqrt(t2)
    H = _hat(w)
    a = LD(1) - t2 / 6 + t2 * t2 / 120 if t2 < 1e-8 else np.sin(t) / t
    b = LD(0.5) - t2 / 24 + t2 * t2 / 720 if t2 < 1e-8 else 2 * np.sin(t / 2) ** 2 / t2
    return np.eye(3, dtype=LD) + a * H + b * H @ H


def _Jr(w):
    """covref._so3_Jr without its final rounding to double (the same series below t^2 = 0.05)."""
    t2 = w @ w
    t = np.sqrt(t2)
    H = _hat(w)
    b = LD(0.5) - t2 / 24 if t2 < 1e-16 else 2 * np.sin(t / 2) ** 2 / t2
    c = np.polyval(cr._C_SERIES, t2) if t2 < 0.05 else (t - np.sin(t)) / (t2 * t)
    return np.eye(3, dtype=LD) - b * H + c * H @ H


def _Jr_inv(w):
    t2 = w @ w
    t = np.sqrt(t2)
    H = _hat(w)
    e = np.polyval(cr._E_SERIES, t2) if t2 < 0.05 else 1 / t2 - (1 + np.cos(t)) / (2 * t * np.sin(t))
    return np.eye(3, dtype=LD) + H / 2 + e * H @ H


def segment_base(stamps, k, t):
    """hb200's segment_base: the base knot of t, or -1 outside the valid span."""
    K = len(stamps)
    j = int(np.searchsorted(stamps, t, side="right")) - 1
    if K < k or j < 0 or j > K - 2:
        return -1
    base = j - (k - 1) // 2
    return base if base >= 0 and base + k <= K else -1


def _basis(k, stamps, base, t):
    """lambda_j, lamd_j (j = 0..k, lambda_0 = 1, lambda_k = 0) in long double at t in the segment of `base`."""
    left = (k - 1) // 2
    t0, t1 = LD(float(stamps[base + left])), LD(float(stamps[base + left + 1]))
    inv_dt = 1 / (t1 - t0)
    u = (LD(float(t)) - t0) * inv_dt
    Mc = synthetic.blending_matrix(k).astype(LD)
    pw = np.array([u ** n for n in range(k)], LD)
    dpw = np.array([n * u ** (n - 1) if n else LD(0) for n in range(k)], LD)
    lam = np.append(Mc @ pw, LD(0))
    lamd = np.append(Mc @ dpw * inv_dt, LD(0))
    lam[0], lamd[0] = 1, 0
    return lam, lamd


def state_jacobian(knots, gyro, accel, order, t):
    """(base, gb, ab, J (18, 6k + 24)) at stamp t; base = -1 outside the pose spline's valid span or outside that of a bias
    spline with knots.  gb / ab = -1 (and zero rows) for a bias spline without knots."""
    k = order
    knots = np.asarray(knots, np.float64)
    base = segment_base(knots[:, 7], k, t)
    gb = segment_base(gyro[:, 3], BIAS_ORDER, t) if len(gyro) else -1
    ab = segment_base(accel[:, 3], BIAS_ORDER, t) if len(accel) else -1
    if base < 0 or (len(gyro) and gb < 0) or (len(accel) and ab < 0):
        return -1, gb, ab, None
    NC = 6 * k + 24
    J = np.zeros((DIM, NC), LD)
    _, Jpose = cr.pose_jacobian(knots, k, t)
    J[:6, :6 * k] = Jpose
    lam, lamd = _basis(k, knots[:, 7], base, t)
    Rk = [_quat_to_rot(knots[base + j, :4]) for j in range(k)]
    P = Rk[0]
    w = np.zeros(3, LD)
    pd = np.zeros(3, LD)
    Y = [np.zeros((3, 3), LD)]
    for j in range(1, k):
        d = _increment(knots[base + j - 1, :4], knots[base + j, :4])
        A = _exp(lam[j] * d)
        P = P @ A
        aw = A.T @ w
        X = _hat(aw) @ (lam[j] * _Jr(lam[j] * d)) + lamd[j] * np.eye(3, dtype=LD)
        Y.append(P @ X @ _Jr_inv(d) @ Rk[j].T)
        w = aw + lamd[j] * d
        pd += lamd[j] * (knots[base + j, 4:7].astype(LD) - knots[base + j - 1, 4:7].astype(LD))
    Y.append(np.zeros((3, 3), LD))
    R = P
    v = R.T @ pd
    H = _hat(v) @ R.T
    for m in range(k):
        c = 6 * m
        J[6:9, c:c + 3] = R.T @ (Y[m] - Y[m + 1])
        J[9:12, c:c + 3] = H @ J[0:3, c:c + 3]
        J[9:12, c + 3:c + 6] = (lamd[m] - lamd[m + 1]) * R.T
    for s, (bk, b0) in enumerate(((gyro, gb), (accel, ab))):
        if not len(bk):
            continue
        lb, _ = _basis(BIAS_ORDER, bk[:, 3], b0, t)
        for m in range(BIAS_ORDER):
            c = 6 * k + 12 * s + 3 * m
            J[12 + 3 * s:15 + 3 * s, c:c + 3] = (lb[m] - lb[m + 1]) * np.eye(3, dtype=LD)
    return base, gb, ab, J


def state_dofs(K, Kbg, Kba, order, base, gb, ab):
    """Reduced-system dof of each column of J (-1: a bias spline without knots)."""
    np_ = 6 * K
    cols = list(range(6 * base, 6 * (base + order)))
    cols += [np_ + 3 * gb + c for c in range(12)] if Kbg else [-1] * 12
    cols += [np_ + 3 * Kbg + 3 * ab + c for c in range(12)] if Kba else [-1] * 12
    return np.array(cols)


def interpolated_state(knots, gyro, accel, order, t, Sig):
    """J(t) Sigma_span J(t)^T (18 x 18) in long double, or None outside the valid spans.  Sig: dense reduced-system Sigma
    (covref.packed_to_dense)."""
    gyro, accel = np.asarray(gyro, np.float64).reshape(-1, 4), np.asarray(accel, np.float64).reshape(-1, 4)
    base, gb, ab, J = state_jacobian(knots, gyro, accel, order, t)
    if base < 0:
        return None
    cols = state_dofs(len(knots), len(gyro), len(accel), order, base, gb, ab)
    ok = cols >= 0
    Z = np.zeros((cols.size, cols.size), LD)
    Z[np.ix_(ok, ok)] = np.asarray(Sig, LD)[np.ix_(cols[ok], cols[ok])]
    out = J @ Z @ J.T
    return (out + out.T) / 2
