"""Reference of the joint and relative covariance of the poses at two stamps (test infrastructure, CPU only), in long
double.

* `pose_value`: R(t), p(t) of the split cumulative spline (R_0 Exp(lambda_1 d_1) .. , p_0 + sum lambda_j (p_j - p_{j-1}));
* `relative_jacobian`: A (6 x 12), the first-order map from [theta_a rho_a | theta_b rho_b] (global rotation tangent,
  p <- p + rho) to the tangent of T_ab = T_a^-1 T_b in frame a (R_ab <- Exp(dtheta) R_ab, p_ab <- p_ab + dp):
      dtheta = R_a^T (theta_b - theta_a),  dp = R_a^T (rho_b - rho_a + hat(p_b - p_a) theta_a);
* `far_plan`: the far columns the compute marches for a list of stamp spans (the host planner of cov_blocks_enqueue):
  for every knot pair of span(a) x span(b) more than beta apart, its column (the larger block) down to the lowest row;
* `pose_pair`: joint = [J_a; J_b] Sigma_{span(a) u span(b)} [J_a; J_b]^T (12 x 12, J covref.pose_jacobian) and
  relative = A joint A^T, both symmetrised; (None, None) outside the valid span.
"""
from __future__ import annotations

import numpy as np

import covref as cr
import stateref as st

LD = np.longdouble


def pose_value(knots, order, t):
    """(base, R, p) of the interpolated pose at t in long double; base = -1 (R, p None) outside the valid span."""
    k = order
    knots = np.asarray(knots, np.float64)
    base = st.segment_base(knots[:, 7], k, t)
    if base < 0:
        return -1, None, None
    lam, _ = st._basis(k, knots[:, 7], base, t)
    R = st._quat_to_rot(knots[base, :4])
    p = knots[base, 4:7].astype(LD)
    for j in range(1, k):
        d = st._increment(knots[base + j - 1, :4], knots[base + j, :4])
        R = R @ st._exp(lam[j] * d)
        p = p + lam[j] * (knots[base + j, 4:7].astype(LD) - knots[base + j - 1, 4:7].astype(LD))
    return base, R, p


def relative_jacobian(Ra, pa, pb):
    """A = [[-R_a^T, 0, R_a^T, 0], [R_a^T hat(p_b - p_a), -R_a^T, 0, R_a^T]] (6 x 12) in long double."""
    Rt = np.asarray(Ra, LD).T
    A = np.zeros((6, 12), LD)
    A[:3, 0:3], A[:3, 6:9] = -Rt, Rt
    A[3:, 0:3] = Rt @ st._hat(np.asarray(pb, LD) - np.asarray(pa, LD))
    A[3:, 3:6], A[3:, 9:12] = -Rt, Rt
    return A


def far_plan(spans, order, beta):
    """{column block j: lowest row block} over every pair of control points of span(a) x span(b) more than beta apart;
    spans: [(base_a, base_b)], pairs with a negative base skipped."""
    need = {}
    for ba, bb in spans:
        if ba < 0 or bb < 0:
            continue
        for a in range(ba, ba + order):
            for b in range(bb, bb + order):
                if abs(a - b) > beta:
                    j, i = max(a, b), min(a, b)
                    need[j] = min(need.get(j, i), i)
    return need


def stacked_jacobian(knots, order, ta, tb):
    """(base_a, base_b, J (12 x 12k)) = blockdiag(J(t_a), J(t_b)) over the columns [span(a) | span(b)]; bases -1 (J None)
    when a stamp is outside the valid span."""
    ba, Ja = cr.pose_jacobian(knots, order, ta)
    bb, Jb = cr.pose_jacobian(knots, order, tb)
    if ba < 0 or bb < 0:
        return ba, bb, None
    NC = 6 * order
    J = np.zeros((12, 2 * NC), LD)
    J[:6, :NC], J[6:, NC:] = Ja, Jb
    return ba, bb, J


def pose_pair(knots, order, ta, tb, Sig):
    """(joint (12 x 12), relative (6 x 6)) in long double from a dense Sigma whose entries over span(a) u span(b) are set;
    (None, None) outside the valid span."""
    ba, bb, J = stacked_jacobian(knots, order, ta, tb)
    if J is None:
        return None, None
    cols = np.r_[6 * ba:6 * (ba + order), 6 * bb:6 * (bb + order)]
    Z = np.asarray(Sig, LD)[np.ix_(cols, cols)]
    joint = J @ Z @ J.T
    joint = (joint + joint.T) / 2
    _, Ra, pa = pose_value(knots, order, ta)
    _, _, pb = pose_value(knots, order, tb)
    A = relative_jacobian(Ra, pa, pb)
    rel = A @ joint @ A.T
    return joint, (rel + rel.T) / 2
