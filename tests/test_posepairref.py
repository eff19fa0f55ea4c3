"""tests/posepairref.py, CPU only.

* relative-pose Jacobian: A [J(t_a); J(t_b)] (mapped onto the knots of both spans, which may share control points)
  equals central differences (h = 1e-20, 80 digits) of T_a^-1 T_b along the knots' tangents (make_golden.pose of the
  perturbed knots, make_golden.perturbed: R <- Exp(phi) R, p <- p + rho), on the edge_knots windows of
  tests/test_stateref.py at orders 4 and 6 with stamps at the small-angle switches, at u = 0 and at the last double below
  a segment end.  Every entry within C u scale(row), C = 150 and scale(row) the row's largest entry of |A| |[J_a; J_b]|:
  the entries are differences of the two stamps' terms, which cancel for close stamps (0.754 and 0.7546 at order 6 lose
  three digits), so the terms, not their difference, set the rounding;
* joint block: from the selected inverse plus crosscovref.far_columns over far_plan's columns it equals
  J_a Sigma_dense J_b^T of covref.dense_inverse_ld within sysref.forward_bound, for beta = 1 .. 6 and stamp pairs in one
  segment, adjacent, k - 1 apart, more than beta apart and at opposite ends of the window; leaving the far columns out
  is caught;
* identical stamps: the joint's off-diagonal blocks equal its diagonal ones and the relative covariance is zero to
  rounding.
"""
import importlib.util
import os

import mpmath as mp
import numpy as np
import pytest

import covref as cr
import crosscovref as xr
import posepairref as pp
import sysref as sr
from hyperslam_b200 import synthetic
from test_stateref import edge_case

U = 2.0 ** -53
C = 150.0
_spec = importlib.util.spec_from_file_location("make_golden", os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_golden.py"))
mg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mg)


def relative_pose(state, ta, tb):
    """(R_ab, p_ab) of make_golden.pose at 80 digits."""
    Ra, pa = mg.pose(state["knots"], state["k"], ta)
    Rb, pb = mg.pose(state["knots"], state["k"], tb)
    return Ra.T * Rb, Ra.T * (pb - pa)


def numeric_relative_jacobian(knots, order, ta, tb, cols):
    """d [dtheta | dp] / d (knot g, component c) for g in cols, by central differences in mpmath at 80 digits."""
    with mp.workdps(80):
        state = dict(k=order, knots=[[mp.mpf(float(x)) for x in row] for row in np.asarray(knots)])
        tam, tbm = mp.mpf(float(ta)), mp.mpf(float(tb))
        h = mg.H_X
        R0, _ = relative_pose(state, tam, tbm)
        out = np.zeros((6, 6 * len(cols)))
        for q, g in enumerate(cols):
            for c in range(6):
                Rp, pp_ = relative_pose(mg.perturbed(state, "knot", g, c, h), tam, tbm)
                Rm, pm = relative_pose(mg.perturbed(state, "knot", g, c, -h), tam, tbm)
                w = mg.vee((Rp - Rm) * R0.T / (2 * h))
                v = (pp_ - pm) / (2 * h)
                out[:, 6 * q + c] = [float(w[i]) for i in range(3)] + [float(v[i]) for i in range(3)]
        return out


@pytest.mark.parametrize("order", [4, 6])
def test_relative_jacobian_against_central_differences(order, record_property):
    knots, _, _, stamps = edge_case(order)
    pairs = [(stamps[i], stamps[j]) for i in range(len(stamps)) for j in range(len(stamps)) if (i + 2 * j) % 5 == 0 and i != j]
    pairs += [(stamps[0], stamps[-1]), (stamps[-1], stamps[0])]
    worst = 0.0
    for ta, tb in pairs:
        ba, bb, J = pp.stacked_jacobian(knots, order, ta, tb)
        assert ba >= 0 and bb >= 0
        _, Ra, pa = pp.pose_value(knots, order, ta)
        _, _, pb = pp.pose_value(knots, order, tb)
        A = pp.relative_jacobian(Ra, pa, pb)
        AJ = A @ J
        terms = np.abs(np.asarray(A, np.float64)) @ np.abs(np.asarray(J, np.float64))
        cols = sorted(set(range(ba, ba + order)) | set(range(bb, bb + order)))
        got = np.zeros((6, 6 * len(cols)), np.longdouble)
        for s, b0 in enumerate((ba, bb)):
            for m in range(order):
                q = cols.index(b0 + m)
                got[:, 6 * q:6 * q + 6] += AJ[:, 6 * order * s + 6 * m:6 * order * s + 6 * m + 6]
        ref = numeric_relative_jacobian(knots, order, ta, tb, cols)
        for i in range(6):
            scale = terms[i].max()
            assert np.abs(ref[i]).max() > 0
            worst = max(worst, float(np.abs(got[i].astype(np.float64) - ref[i]).max() / (U * scale)))
    record_property("worst_ratio", worst)
    print(f"order {order}: {len(pairs)} pairs, worst |A J - mpmath| / (u scale) = {worst:.3f}")
    assert worst <= C, worst


def window_knots(K, seed, dt=0.1):
    """K knots dt apart with random rotations and positions (every other quaternion stored as -q)."""
    rng = np.random.default_rng(seed)
    R = synthetic.so3_exp(rng.normal(0, 0.4, (K, 3)))
    knots = np.zeros((K, 8))
    knots[:, :4] = synthetic.rot_to_quat(R)
    knots[1::2, :4] *= -1
    knots[:, 4:7] = rng.normal(0, 1.0, (K, 3))
    knots[:, 7] = dt * np.arange(K)
    return knots


def stamp_pairs(knots, order, beta):
    """In one segment, adjacent segments, k - 1 apart, more than beta apart, opposite ends, and the same stamp twice."""
    kt, K, left = knots[:, 7], knots.shape[0], (order - 1) // 2
    first, last = left, K - order + left          # first and last valid segment
    at = lambda s, u: kt[s] + u * (kt[s + 1] - kt[s])
    far = min(first + beta + 2, last)
    return [(at(first + 1, 0.2), at(first + 1, 0.7)), (at(first + 2, 0.3), at(first + 3, 0.6)),
            (at(first, 0.5), at(min(first + order - 1, last), 0.25)), (at(far, 0.9), at(first, 0.1)),
            (at(first, 0.0), float(np.nextafter(kt[last + 1], -np.inf))), (at(last, 0.4), at(first, 0.6)), (at(first + 1, 0.3), at(first + 1, 0.3))]


SHAPES = [(beta, order) for beta in range(1, 7) for order in (4, 6)]


@pytest.mark.parametrize("beta,order", SHAPES, ids=[f"b{b}-k{k}" for b, k in SHAPES])
def test_joint_equals_dense(beta, order):
    K, m = max(3 * beta + 5, order + beta + 4), 8
    n = 6 * K + m
    S, *_ = sr.make_system(K, beta, m, seed=500 + 10 * beta + order)
    fixed = np.zeros(n, bool)
    fixed[:6] = True
    Sig, P, _, bad = cr.selected_inverse(S, K, beta, m, fixed)
    assert bad == -1
    d, L = xr.band_factor(S, K, beta, m, fixed)
    ref = cr.dense_inverse_ld(S, fixed)
    bound = sr.forward_bound(n, cr.kappa(S, fixed))
    knots = window_knots(K, 700 + beta + order)
    pairs = stamp_pairs(knots, order, beta)
    spans = [(pp.pose_value(knots, order, a)[0], pp.pose_value(knots, order, b)[0]) for a, b in pairs]
    plan = pp.far_plan(spans, order, beta)
    assert plan, "no pair needs a far column"
    full = xr.far_columns(Sig, d, L, K, beta, m, fixed, plan)
    err = err_band = 0.0
    for (ta, tb), (ba, bb) in zip(pairs, spans):
        assert ba >= 0 and bb >= 0
        joint, rel = pp.pose_pair(knots, order, ta, tb, full)
        want, _ = pp.pose_pair(knots, order, ta, tb, ref)
        band_only, _ = pp.pose_pair(knots, order, ta, tb, Sig)
        s = np.sqrt(np.abs(np.diagonal(want)).astype(np.float64))
        norm = np.outer(s, s)
        err = max(err, float((np.abs(np.asarray(joint - want, np.float64)) / norm).max()))
        if max(abs(a - b) for a in range(ba, ba + order) for b in range(bb, bb + order)) > beta:
            err_band = max(err_band, float((np.abs(np.asarray(band_only - want, np.float64)) / norm).max()))
        assert np.array_equal(joint, joint.T) and np.array_equal(rel, rel.T)
        # (t_b, t_a) permutes the joint block
        swapped, _ = pp.pose_pair(knots, order, tb, ta, full)
        perm = np.r_[6:12, 0:6]
        assert np.allclose(np.asarray(swapped, np.float64), np.asarray(joint, np.float64)[np.ix_(perm, perm)], rtol=1e-15, atol=0)
    print(f"beta {beta} order {order}: joint error {err:.3e}, bound {bound:.3e}; without far columns {err_band:.3e}; plan {plan}")
    assert err < bound, (err, bound)
    assert err_band > 1e3 * bound, (err_band, bound)


def test_identical_stamps():
    order, beta = 4, 3
    K, m = 14, 8
    S, *_ = sr.make_system(K, beta, m, seed=77)
    fixed = np.zeros(6 * K + m, bool)
    fixed[:6] = True
    ref = cr.dense_inverse_ld(S, fixed)
    knots = window_knots(K, 78)
    for t in (0.25, 0.4, float(np.nextafter(knots[K - order + 2, 7], -np.inf))):
        joint, rel = pp.pose_pair(knots, order, t, t, ref)
        assert joint is not None
        assert np.array_equal(joint[:6, 6:], joint[:6, :6]) and np.array_equal(joint[6:, 6:], joint[:6, :6])
        assert np.abs(np.asarray(rel, np.float64)).max() <= 1e-15 * np.abs(np.asarray(joint, np.float64)).max()
    # outside the valid span
    assert pp.pose_pair(knots, order, knots[0, 7], 0.5, ref) == (None, None)
