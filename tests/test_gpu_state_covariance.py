"""Joint covariance of the interpolated state [theta p | omega v | b_g b_a] on the device (need an H100):
hb200_interpolate_state_covariance against tests/stateref.py on the device's own Sigma (covariance_packed ->
covref.packed_to_dense), in covref's correlation metric.

* end to end (orders 4 and 6, bias splines spaced unlike the pose knots and starting inside the pose span, as after a
  slide that dropped bias knots): valid blocks within 1e-11, invalid stamps (outside the pose span, before a bias span)
  zero and counted, output exactly symmetric and positive semidefinite after equilibration; the pose block equals
  hb200_interpolate_covariance value for value (one Jacobian builder; the bias columns only add z * 0 terms, so zeros
  may differ in sign); one launch per call, two calls bit-identical;
* omega and b_g against the device's own inertial factor (identity IMU calibration): Sigma_omega,omega + Sigma_omega,bg
  + Sigma_bg,omega + Sigma_bg,bg equals the sandwich of the factor's gyro rows of Jp and wg;
* knot increments across the small-angle switches of the SO(3) coefficients; bias_const, constant knots, no bias splines;
* results belong to the last compute: iterations, appends and a slide with DROP_BIAS change nothing;
* error codes, a call between build and compute, deterministic reruns, the iteration's kernel list;
* sharded contexts (2 and 3 ranks through the all-reduce hook): bit-identical across ranks and within 1e-11 of stateref.
"""
import math

import numpy as np
import pytest

import covref as cr
import stateref as st
from hyperslam_b200 import runtime
from test_gpu_covariance import NEAR_STATIONARY, e2e_window
from test_gpu_sharded import HostReducer, on_ranks, open_ranks, shard_by_owner
from hyperslam_b200 import synthetic

pytestmark = pytest.mark.gpu

TOL = 1e-11


def late_bias(win, seed, gyro_dt=0.7, accel_dt=0.45, gyro_start=0.8, accel_start=1.1):
    """Bias splines whose valid spans start gyro_start / accel_start s into the pose span and end just past the last
    inertial factor (so that every bias knot reaches one); inertial factors outside both spans are dropped."""
    rng = np.random.default_rng(seed)
    kt, k = win.knots[:, 7], win.order
    lo, last = kt[(k - 1) // 2], win.i_stamp.max()
    out = []
    for dt, start in ((gyro_dt, gyro_start), (accel_dt, accel_start)):
        first = lo + start
        n = int(math.floor((last - first) / dt)) + 3
        b = np.zeros((n, 4))
        b[:, :3] = rng.uniform(-0.02, 0.02, (n, 3))
        b[:, 3] = first - dt + dt * np.arange(n)
        out.append(b)
    win.gyro_bias, win.accel_bias = out
    keep = np.ones(win.i_stamp.size, bool)
    for b in out:
        keep &= (win.i_stamp >= b[1, 3]) & (win.i_stamp < b[-2, 3])
    win.i_stamp, win.i_meas = np.ascontiguousarray(win.i_stamp[keep]), np.ascontiguousarray(win.i_meas[keep])
    return win


def snapshot(ctx):
    packed, _, (K, beta, m, _) = ctx.covariance_packed()
    s = ctx.state()
    return dict(Sig=cr.packed_to_dense(packed, K, beta, m), knots=s["knots"], gyro=s["gyro_bias"], accel=s["accel_bias"])


def compare(cov, bad, stamps, snap, order, report=None, name="err"):
    """Every block against stateref; returns the worst correlation error."""
    refs = [st.interpolated_state(snap["knots"], snap["gyro"], snap["accel"], order, t, snap["Sig"]) for t in stamps]
    invalid = [i for i, r in enumerate(refs) if r is None]
    assert bad == len(invalid)
    assert np.all(cov[invalid] == 0)
    assert np.array_equal(cov, cov.transpose(0, 2, 1))
    worst = 0.0
    for i, r in enumerate(refs):
        if r is None:
            continue
        worst = max(worst, cr.cov_error(cov[i], r))
        d = np.sqrt(np.diag(cov[i]))
        nz = d > 0
        if nz.any():
            E = cov[i][np.ix_(nz, nz)] / d[nz][:, None] / d[nz][None, :]
            assert np.linalg.eigvalsh(E).min() >= -1e-10
    if report:
        report(name, worst)
    assert worst < TOL, worst
    return worst, invalid


def compute(ctx, win):
    ctx.load_window(win)
    ctx.build_covariance()
    info = ctx.compute_covariance()
    assert info["status"] == 0, info


@pytest.mark.parametrize("order", [4, 6])
def test_end_to_end(built, record_property, order):
    win = late_bias(e2e_window(order, seed=80 + order), seed=order)
    kt, k = win.knots[:, 7], order
    left = (k - 1) // 2
    lo, hi = kt[left], kt[len(kt) - k + left + 1]
    g0, a0 = win.gyro_bias[1, 3], win.accel_bias[1, 3]
    end = min(hi, win.gyro_bias[-2, 3], win.accel_bias[-2, 3])
    stamps = np.concatenate([kt[left + 15:left + 20], 0.5 * (kt[20:25] + kt[21:26]), np.nextafter(kt[26:30], -np.inf),
                             [max(g0, a0), np.nextafter(end, -np.inf)],                            # both ends of the joint span
                             [np.nextafter(lo, -np.inf), hi, lo, np.nextafter(g0, -np.inf), 0.5 * (g0 + a0)]])   # invalid
    ctx = runtime.Context(0)
    try:
        compute(ctx, win)
        snap = snapshot(ctx)
        l0 = ctx.launch_count
        cov, bad = ctx.interpolate_state_covariance(stamps)
        assert ctx.launch_count - l0 == 1
        cov2, _ = ctx.interpolate_state_covariance(stamps)
        pose, _ = ctx.interpolate_covariance(stamps)
    finally:
        ctx.close()
    assert np.array_equal(cov.view(np.int64), cov2.view(np.int64))
    _, invalid = compare(cov, bad, stamps, snap, order, record_property)
    assert invalid == list(range(len(stamps) - 5, len(stamps)))
    for i in range(len(stamps)):
        if i not in invalid:
            assert np.array_equal(cov[i][:6, :6], pose[i]), i


def test_gyro_rows_against_inertial_factor(built, record_property):
    """With I_g = I, S_g = 0 and R_bs = I the gyro residual is omega + b_g: its Jacobian rows sandwich Sigma to the sum of
    the omega / b_g blocks."""
    win = e2e_window(4, num_knots=30, num_landmarks=300, num_imu=800, bearing=100, pose=10, seed=91)
    assert np.array_equal(win.imu[:4], [0, 0, 0, 1]) and np.array_equal(win.imu[7:13], [1, 1, 1, 0, 0, 0]) and not win.imu[19:28].any()
    ctx = runtime.Context(0)
    try:
        compute(ctx, win)
        snap = snapshot(ctx)
        cov, bad = ctx.interpolate_state_covariance(win.i_stamp)
        ctx.evaluate(jacobians=True)
        out = ctx.outputs()
        _, ib, ig, _ = ctx.index_maps()
    finally:
        ctx.close()
    assert bad == 0
    K, k = win.knots.shape[0], win.order
    worst = 0.0
    for f in range(win.i_stamp.size):
        Jg = np.hstack([out["i_Jp"][f][:3], np.kron(out["i_wg"][f][None], np.eye(3))])
        cols = np.r_[6 * ib[f]:6 * (ib[f] + k), 6 * K + 3 * ig[f] + np.arange(12)]
        want = Jg.astype(cr.LD) @ snap["Sig"][np.ix_(cols, cols)].astype(cr.LD) @ Jg.T.astype(cr.LD)
        c = cov[f]
        got = c[6:9, 6:9] + c[6:9, 12:15] + c[12:15, 6:9] + c[12:15, 12:15]
        worst = max(worst, cr.cov_error(got, want))
    record_property("err_inertial", worst)
    assert worst < TOL, worst


@pytest.mark.parametrize("order", [4, 6])
def test_near_stationary(built, record_property, order):
    win = e2e_window(order, num_knots=30, num_landmarks=300, num_imu=600, bearing=100, pose=10, seed=40 + order)
    rng = np.random.default_rng(order)
    for i, inc in enumerate(NEAR_STATIONARY, start=10):
        axis = rng.normal(size=3)
        R = synthetic.quat_to_rot(win.knots[i - 1, None, :4])[0] @ synthetic.so3_exp(inc * axis[None] / np.linalg.norm(axis))[0]
        q = win.knots[i - 1, :4] if inc == 0 else synthetic.rot_to_quat(R[None])[0]
        win.knots[i, :4] = q if np.dot(q, win.knots[i - 1, :4]) >= 0 else -q
    kt = win.knots[:, 7]
    stamps = np.concatenate([kt[10:21], kt[10:21] + 0.3 * (kt[11:22] - kt[10:21]), np.nextafter(kt[11:22], -np.inf)])
    ctx = runtime.Context(0)
    try:
        compute(ctx, win)
        snap = snapshot(ctx)
        cov, bad = ctx.interpolate_state_covariance(stamps)
    finally:
        ctx.close()
    assert bad == 0
    compare(cov, bad, stamps, snap, order, record_property)


def test_constants_and_missing_bias_splines(built, record_property):
    win = e2e_window(4, num_knots=30, num_landmarks=300, num_imu=800, bearing=100, pose=10, seed=92, bias_const=1)
    kt = win.knots[:, 7]
    stamps = np.concatenate([[kt[1]], kt[2:6] + 0.01, 0.5 * (kt[10:14] + kt[11:15])])   # kt[1]: every control point constant
    ctx = runtime.Context(0)
    try:
        compute(ctx, win)
        snap = snapshot(ctx)
        cov, bad = ctx.interpolate_state_covariance(stamps)
        # no bias splines (and so no IMU factors): zero bias rows and columns
        plain = e2e_window(4, num_knots=30, num_landmarks=300, num_imu=0, bearing=100, pose=10, seed=93)
        none = runtime.Context(0)
        try:
            none.set_spline(plain.order, plain.knots)
            none.set_gravity(plain.gravity)
            none.set_cameras(plain.cameras)
            none.set_landmarks(plain.landmarks)
            none.set_pixel_factors(plain.v_stamp, plain.v_cam, plain.v_lm, plain.v_pixel)
            none.set_bearing_factors(plain.b_stamp, plain.b_cam, plain.b_lm, plain.b_bearing, plain.huber_bearing)
            none.set_pose_sensors(plain.pose_sensors)
            none.set_manifold_factors(plain.m_stamp, plain.m_sensor, plain.m_pose)
            assert none.bind() == 0
            none.set_constant(plain.knot_const, 1, 0)
            none.build_covariance()
            assert none.compute_covariance()["status"] == 0
            snap0 = snapshot(none)
            cov0, bad0 = none.interpolate_state_covariance(stamps)
        finally:
            none.close()
    finally:
        ctx.close()
    assert bad == 0 and np.all(cov[:, 12:] == 0) and np.all(cov[:, :, 12:] == 0)
    assert np.all(cov[0] == 0)
    compare(cov, bad, stamps, snap, 4, record_property, "err_bias_const")
    assert bad0 == 0 and np.all(cov0[:, 12:] == 0) and np.all(cov0[:, :, 12:] == 0)
    assert snap0["gyro"].shape == (0, 4)
    compare(cov0, bad0, stamps, snap0, 4, record_property, "err_no_bias")


def test_results_belong_to_the_last_compute(built, record_property):
    win = late_bias(e2e_window(4, num_knots=30, num_landmarks=300, num_imu=800, bearing=100, pose=10, seed=94), seed=94,
                    gyro_dt=0.3, accel_dt=0.25, gyro_start=0.3, accel_start=0.4)
    kt = win.knots[:, 7]
    stamps = np.concatenate([kt[6:20] + 0.013, [kt[1]]])
    ctx = runtime.Context(0)
    try:
        compute(ctx, win)
        snap = snapshot(ctx)
        ref, bad = ctx.interpolate_state_covariance(stamps)
        compare(ref, bad, stamps, snap, 4, record_property)

        def same(what):
            cov, b = ctx.interpolate_state_covariance(stamps)
            assert b == bad and np.array_equal(cov.view(np.int64), ref.view(np.int64)), what
        ctx.iterate(2)
        same("iterate")
        ctx.append_knots(2)
        same("append_knots")
        g, a = ctx.append_bias_knots(float(ctx.state()["knots"][-1, 7]) + 1.0)
        assert g > 0 and a > 0
        same("append_bias_knots")
        ctx.slide(kt[8], drop_inertial=True, drop_bias=True)
        b = ctx.bias_knots()
        record_property("bias_knots_dropped", (b["gyro_dropped"], b["accel_dropped"]))
        assert b["gyro_dropped"] > 0, b
        same("slide")
    finally:
        ctx.close()


def test_error_codes_and_pending_build(built):
    win = e2e_window(4, num_knots=30, num_landmarks=300, num_imu=800, bearing=100, pose=10, seed=95)
    stamps = win.knots[5:10, 7] + 0.01
    ctx = runtime.Context(0)
    try:
        ctx.load_window(win)
        with pytest.raises(runtime.HB200Error, match="hb200 error -2"):
            ctx.interpolate_state_covariance(stamps)
        lib, h = ctx.lib, ctx.h
        out = np.zeros((1, 18, 18))
        t = np.array([stamps[0]])
        assert lib.hb200_interpolate_state_covariance(h, -1, runtime._d(t), runtime._d(out), None) == -1
        assert lib.hb200_interpolate_state_covariance(h, 1, None, runtime._d(out), None) == -1
        assert lib.hb200_interpolate_state_covariance(h, 1, runtime._d(t), None, None) == -1
        assert lib.hb200_interpolate_state_covariance(None, 1, runtime._d(t), runtime._d(out), None) == -1
        compute(ctx, win)
        assert lib.hb200_interpolate_state_covariance(h, 0, None, None, None) == 0
        first, _ = ctx.interpolate_state_covariance(stamps)
        ctx.build_covariance()                     # build -> this call -> compute
        between, _ = ctx.interpolate_state_covariance(stamps)
        assert np.array_equal(between.view(np.int64), first.view(np.int64))
        assert ctx.compute_covariance()["status"] == 0
    finally:
        ctx.close()


def test_determinism_and_iteration_path(built):
    win = e2e_window(6, num_knots=30, num_landmarks=300, num_imu=800, bearing=100, pose=10, seed=96)
    stamps = win.knots[6:20, 7] + 0.017
    runs = []
    for _ in range(2):
        ctx = runtime.Context(0)
        try:
            ctx.set_deterministic(True)
            compute(ctx, win)
            runs.append(ctx.interpolate_state_covariance(stamps)[0])
        finally:
            ctx.close()
    assert np.array_equal(runs[0].view(np.int64), runs[1].view(np.int64))
    ctx = runtime.Context(0)
    try:
        ctx.load_window(win)
        kernels0 = [nm for nm, _ in ctx.profile_iteration(reps=1)]
        compute(ctx, win)
        ctx.interpolate_state_covariance(stamps)
        kernels1 = [nm for nm, _ in ctx.profile_iteration(reps=1)]
    finally:
        ctx.close()
    assert kernels1 == kernels0
    assert not any(nm.startswith("cov_") for nm in kernels1)


@pytest.mark.parametrize("world", [2, 3])
def test_sharded(built, record_property, world):
    win = e2e_window(4 if world == 2 else 6, num_knots=30, num_landmarks=300, num_imu=800, bearing=150, pose=10, seed=97 + world)
    owner = np.random.default_rng(world).integers(0, world, win.landmarks.shape[0])
    shards, _ = shard_by_owner(win, owner, world)
    kt = win.knots[:, 7]
    stamps = np.concatenate([kt[4:20] + 0.021, [kt[0]]])
    ctxs, _, _ = open_ranks(shards)
    try:
        red = HostReducer(world)
        red.attach(ctxs)
        infos = on_ranks(red, ctxs, lambda r, c: (c.build_covariance(), c.compute_covariance())[1])
        assert all(i["status"] == 0 for i in infos), infos
        res = [c.interpolate_state_covariance(stamps) for c in ctxs]
        snap = snapshot(ctxs[0])
    finally:
        for c in ctxs:
            c.close()
    for cov, bad in res[1:]:
        assert bad == res[0][1] and np.array_equal(cov.view(np.int64), res[0][0].view(np.int64))
    compare(res[0][0], res[0][1], stamps, snap, win.order, record_property)
