"""The window's three splines through the C ABI: the setters' validation and reshape rule, hb200_optimize's stamp
checks against the host stamp mirrors, and the mirrors following knots that hb200_append_knots and
hb200_append_bias_knots create on the device.

A refused call must leave the window as it was: the same knot counts and, bit for bit, the same state.
"""
import numpy as np
import pytest

from hyperslam_b200 import runtime, synthetic
from test_gpu_stereo_window import error_code

pytestmark = pytest.mark.gpu

STRIDE = {"knots": 8, "gyro_bias": 4, "accel_bias": 4}


def small_window():
    return synthetic.make_window(order=4, num_knots=16, num_landmarks=60, num_imu=200, seed=synthetic.SEED_BASE + 77)


@pytest.fixture
def ctx():
    c = runtime.Context(0)
    c.load_window(small_window())
    yield c
    c.close()


def snapshot(c):
    c._refresh_sizes()   # (the wrappers record the sizes they pass before the call is refused)
    return (c.K, c.Kbg, c.Kba), c.state()


def assert_unchanged(c, before):
    sizes, st = snapshot(c)
    assert sizes == before[0]
    for key, v in before[1].items():
        assert np.array_equal(st[key], v, equal_nan=True), key


def call_setter(c, target, arrays, order=None):
    if target == "knots":
        c.set_spline(4 if order is None else order, arrays["knots"])
    else:
        c.set_bias_splines(4 if order is None else order, arrays["gyro_bias"], arrays["accel_bias"])


def corrupt(a, stride, case):
    """A copy of the knot array `a` broken in one way; the stamp is each knot's last component."""
    a = a.copy()
    s = stride - 1
    if case == "too_few":
        return a[:3]
    if case == "repeated":
        a[2, s] = a[1, s]
    elif case == "non_uniform":
        a[-1, s] += 0.25 * (a[1, s] - a[0, s])
    elif case == "nan_at_3":
        a[3, s] = np.nan
    return a


@pytest.mark.parametrize("target", ["knots", "gyro_bias", "accel_bias"])
@pytest.mark.parametrize("case,code", [("wrong_order", -4), ("too_few", -1), ("repeated", -1), ("non_uniform", -1), ("nan_at_3", -1)])
def test_setter_refusals(ctx, target, case, code):
    before = snapshot(ctx)
    arrays = {k: v.copy() for k, v in before[1].items()}
    # the other bias spline gets new, valid values: a refused call must not set it either
    other = {"gyro_bias": "accel_bias", "accel_bias": "gyro_bias"}.get(target)
    if other:
        arrays[other][:, :3] += 0.5
    order = None
    if case == "wrong_order":
        order = 5 if target == "knots" else 6
    else:
        arrays[target] = corrupt(arrays[target], STRIDE[target], case)
    assert error_code(call_setter, ctx, target, arrays, order) == code
    assert_unchanged(ctx, before)
    ctx.iterate(1)   # still bound


@pytest.mark.parametrize("target", ["knots", "bias"])
def test_reshape_rule(ctx, target):
    st = ctx.state()
    if target == "knots":
        ctx.set_spline(4, st["knots"])
    else:
        ctx.set_bias_splines(4, st["gyro_bias"], st["accel_bias"])
    ctx.iterate(1)   # identical stamps: the window stays bound
    st = ctx.state()
    if target == "knots":
        shifted = st["knots"].copy()
        shifted[:, 7] += shifted[1, 7] - shifted[0, 7]
        ctx.set_spline(4, shifted)
    else:
        shifted = st["accel_bias"].copy()
        shifted[:, 3] += shifted[1, 3] - shifted[0, 3]
        ctx.set_bias_splines(4, st["gyro_bias"], shifted)
    assert (ctx.K, ctx.Kbg, ctx.Kba) == (st["knots"].shape[0], st["gyro_bias"].shape[0], st["accel_bias"].shape[0])
    assert error_code(ctx.iterate, 1) == -2   # the same counts with other stamps unbind it


@pytest.mark.parametrize("key,stride", [("knots", 8), ("gyro_bias", 4), ("accel_bias", 4)])
def test_optimize_refuses_changed_stamp(ctx, key, stride):
    before = snapshot(ctx)
    arrays = {k: v.copy() for k, v in before[1].items()}
    arrays[key][2, stride - 1] += 1e-3
    passed = {k: v.copy() for k, v in arrays.items()}
    rc = error_code(ctx.optimize, 1, arrays["knots"], arrays["gyro_bias"], arrays["accel_bias"], arrays["gravity"], arrays["landmarks"])
    assert rc == -2
    assert_unchanged(ctx, before)
    for k, v in passed.items():
        assert np.array_equal(arrays[k], v), k


def test_optimize_after_appends(ctx):
    ctx.append_knots(2)
    g0 = ctx.state()["gyro_bias"][:, 3]
    added = ctx.append_bias_knots(g0[-1] + 3.5 * (g0[-1] - g0[-2]))
    assert added[0] > 0 and added[1] > 0
    st = ctx.state()
    assert st["knots"].shape[0] == 18 and st["gyro_bias"].shape[0] == g0.size + added[0]
    ctx.optimize(1, st["knots"], st["gyro_bias"], st["accel_bias"], st["gravity"], st["landmarks"])
    ctx.set_bias_splines(4, st["gyro_bias"], st["accel_bias"])   # the mirrors hold the device's stamps: no reshape
    ctx.iterate(1)
