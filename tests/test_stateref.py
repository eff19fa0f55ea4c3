"""tests/stateref.py against central differences in mpmath (CPU only).

On the edge_knots windows of tests/golden/make_golden.py (knot increments on both sides of the small-angle switches of
the SO(3) coefficients, every other knot stored as -q) at orders 4 and 6, with bias splines whose knots are spaced
unlike the pose knots, at switch stamps, u = 0 and the last double below a segment end from edge_stamps:
* the omega and v rows are central differences (h = 1e-20, 80 digits) of make_golden.interpolate_answer's body
  velocity -- itself time differences of the value formula, not the Sommer recursion -- along the control points'
  tangents (make_golden.perturbed: R <- Exp(phi) R, p <- p + rho); the bias rows are central differences of
  make_golden.bias along the bias knots.  Every entry within C u scale(row), C = 150 and scale(row) the row's largest
  entry, as in tests/test_gpu_spline_edges.py;
* the pose rows are covref.pose_jacobian's;
* outside the pose span, or outside a bias span, there is no Jacobian.
"""
import importlib.util
import os

import mpmath as mp
import numpy as np
import pytest

import covref as cr
import stateref as st

U = 2.0 ** -53
C = 150.0
_spec = importlib.util.spec_from_file_location("make_golden", os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_golden.py"))
mg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mg)


def bias_knots(seed, dt, n, t0):
    rng = np.random.default_rng(seed)
    b = np.zeros((n, 4))
    b[:, :3] = rng.uniform(-0.05, 0.05, (n, 3))
    b[:, 3] = t0 + dt * np.arange(n)
    return b


def edge_case(order):
    seed = {4: 914, 6: 916}[order] + mg.synthetic.SEED_BASE
    knots = mg.edge_knots(seed)
    gyro = bias_knots(seed + 1, 0.3, 9, -0.45)     # valid span [-0.15, 1.65) covers the pose span
    accel = bias_knots(seed + 2, 0.2, 12, -0.4)    # [-0.2, 1.6)
    stamps = mg.edge_stamps(knots, order)
    return knots, gyro, accel, stamps[:3] + stamps[-4:]


def velocity(state, t):
    """[omega | v] of make_golden.interpolate_answer at full precision (its rounding to double lifted)."""
    fl = mg.fl
    mg.fl = lambda v: [v[i] for i in range(3)]
    try:
        return mg.interpolate_answer(state, t)["vel"]
    finally:
        mg.fl = fl


def numeric_jacobian(knots, gyro, accel, order, t):
    """Rows omega, v (6 x 6k) and b_g, b_a (6 x 24) by central differences in mpmath at make_golden's 80 digits (other
    tests change the global precision; nested differences at h = 1e-20 and 1e-18 need all of them)."""
    with mp.workdps(80):
        return _numeric_jacobian(knots, gyro, accel, order, t)


def _numeric_jacobian(knots, gyro, accel, order, t):
    f = lambda a: [[mp.mpf(float(x)) for x in row] for row in np.asarray(a)]
    state = dict(k=order, knots=f(knots), bg=f(gyro), ba=f(accel))
    tm = mp.mpf(float(t))
    h = mg.H_X
    base = st.segment_base(knots[:, 7], order, t)
    rate = np.zeros((6, 6 * order))
    for m in range(order):
        for c in range(6):
            vp = velocity(mg.perturbed(state, "knot", base + m, c, h), tm)
            vm = velocity(mg.perturbed(state, "knot", base + m, c, -h), tm)
            rate[:, 6 * m + c] = [float((a - b) / (2 * h)) for a, b in zip(vp, vm)]
    bias = np.zeros((6, 24))
    for s, kind in enumerate(("bg", "ba")):
        b0 = st.segment_base(np.asarray(state[kind], float)[:, 3], st.BIAS_ORDER, t)
        for m in range(st.BIAS_ORDER):
            for c in range(3):
                bp = mg.bias(mg.perturbed(state, kind, b0 + m, c, h)[kind], st.BIAS_ORDER, tm)
                bm = mg.bias(mg.perturbed(state, kind, b0 + m, c, -h)[kind], st.BIAS_ORDER, tm)
                bias[3 * s:3 * s + 3, 12 * s + 3 * m + c] = [float((bp[i] - bm[i]) / (2 * h)) for i in range(3)]
    return rate, bias


@pytest.mark.parametrize("order", [4, 6])
def test_state_jacobian_against_central_differences(order, record_property):
    knots, gyro, accel, stamps = edge_case(order)
    worst = 0.0
    for t in stamps:
        base, gb, ab, J = st.state_jacobian(knots, gyro, accel, order, t)
        assert base >= 0 and gb >= 0 and ab >= 0
        rate, bias = numeric_jacobian(knots, gyro, accel, order, t)
        ref = np.zeros((12, 6 * order + 24))
        ref[:6, :6 * order] = rate
        ref[6:, 6 * order:] = bias
        got = J[6:].astype(np.float64)
        for i in range(12):
            scale = np.abs(ref[i]).max()
            assert scale > 0
            worst = max(worst, float(np.abs(got[i] - ref[i]).max() / (U * scale)))
        _, Jp = cr.pose_jacobian(knots, order, t)
        assert np.array_equal(J[:6, :6 * order].astype(np.float64), Jp)
        assert np.all(J[:6, 6 * order:] == 0) and np.all(J[6:12, 6 * order:] == 0) and np.all(J[12:, :6 * order] == 0)
    record_property("worst_ratio", worst)
    print(f"order {order}: worst |stateref - mpmath| / (u scale) = {worst:.3f}")
    assert worst <= C, worst


def test_validity_and_missing_bias_splines():
    order = 4
    knots, gyro, accel, _ = edge_case(order)
    kt = knots[:, 7]
    lo, hi = kt[1], kt[len(kt) - order + 2]
    assert st.state_jacobian(knots, gyro, accel, order, np.nextafter(lo, -np.inf))[0] == -1
    assert st.state_jacobian(knots, gyro, accel, order, hi)[0] == -1
    late = gyro.copy()
    late[:, 3] += 0.5                                # gyro span starts at 0.35, inside the pose span
    assert st.state_jacobian(knots, late, accel, order, 0.3)[0] == -1
    assert st.state_jacobian(knots, late, accel, order, 0.4)[0] >= 0
    none = np.zeros((0, 4))
    t = 0.5 * (lo + hi)
    base, gb, ab, J = st.state_jacobian(knots, none, none, order, t)
    assert base >= 0 and gb == ab == -1 and np.all(J[12:] == 0)
    Sig = np.eye(6 * len(knots) + 2)
    S = st.interpolated_state(knots, none, none, order, t, Sig)
    assert np.all(S[12:] == 0) and np.all(S[:, 12:] == 0) and np.all(np.diag(S)[:12] > 0)
