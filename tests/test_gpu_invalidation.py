"""Which cached products each mutating C-ABI call makes stale.

A context caches the evaluated Jacobians, the built reduced system, the covariance build, the snapshot and the bound
window.  Every mutating call must drop exactly the products it invalidates: a product kept too long is a silent stale
read, one dropped too eagerly refuses a valid call.  Each row applies one mutating call to a freshly prepared window
that has all five products, then records the return code of every call that depends on one of them:

  factor_evaluate     evaluated Jacobians    (bound window + hb200_evaluate with Jacobians)
  get_system, solve   built system           (hb200_build_system)
  compute_covariance  fresh covariance build (hb200_build_covariance, nothing launched since)
  restore             snapshot
  evaluate            bound window

Only return codes are compared, so the table does not depend on floating-point results.  A covariance status
(not positive definite, degenerate landmarks) counts as an accepted build: only -2 means a stale one.
"""
import ctypes as C

import numpy as np
import pytest

from hyperslam_b200 import runtime, synthetic

pytestmark = pytest.mark.gpu

PROBES = ("factor_evaluate", "get_system", "solve", "compute_covariance", "restore", "evaluate")


def make_window():
    win = synthetic.make_window(order=4, num_knots=16, num_landmarks=40, num_imu=60, seed=synthetic.SEED_BASE + 1400)
    return synthetic.add_bearing_and_pose_factors(win, num_bearing=30, num_pose=8, seed=synthetic.SEED_BASE + 1401)


def last_of(stamps):
    return int(np.argmax(stamps))


def mutations(win):
    """name -> call on a prepared Context; every call is expected to succeed."""
    knots_shifted = win.knots.copy()
    knots_shifted[:, 7] += win.knots[1, 7] - win.knots[0, 7]
    cams_more = np.vstack([win.cameras, win.cameras[:1]])
    lms_more = np.vstack([win.landmarks, win.landmarks[:1]])
    v, b, i, m = last_of(win.v_stamp), last_of(win.b_stamp), last_of(win.i_stamp), last_of(win.m_stamp)
    vis_last = max(win.v_stamp[v], win.b_stamp[b])
    bias_dt = win.gyro_bias[1, 3] - win.gyro_bias[0, 3]
    return {
        "none": lambda x: None,
        "set_spline(same stamps)": lambda x: x.set_spline(win.order, win.knots),
        "set_spline(shifted stamps)": lambda x: x.set_spline(win.order, knots_shifted),
        "set_bias_splines": lambda x: x.set_bias_splines(win.bias_order, win.gyro_bias, win.accel_bias),
        "set_gravity": lambda x: x.set_gravity(win.gravity),
        "set_cameras(same C)": lambda x: x.set_cameras(win.cameras),
        "set_cameras(other C)": lambda x: x.set_cameras(cams_more),
        "set_imu": lambda x: x.set_imu(win.imu),
        "set_landmarks(same L)": lambda x: x.set_landmarks(win.landmarks),
        "set_landmarks(other L)": lambda x: x.set_landmarks(lms_more),
        "set_constant": lambda x: x.set_constant(win.knot_const, win.gravity_const, win.bias_const),
        "set_reference_quirks": lambda x: x.set_reference_quirks(1),
        "set_options": lambda x: x.set_options(win.huber_pixel, win.imu_loss_scale, 1e3),
        "set_bearing_loss": lambda x: x._check(x.lib.hb200_set_bearing_loss(x.h, C.c_double(2 * win.huber_bearing))),
        "set_pixel_factors": lambda x: x.set_pixel_factors(win.v_stamp, win.v_cam, win.v_lm, win.v_pixel),
        "set_bearing_factors": lambda x: x.set_bearing_factors(win.b_stamp, win.b_cam, win.b_lm, win.b_bearing),
        "set_inertial_factors": lambda x: x.set_inertial_factors(win.i_stamp, win.i_meas),
        "set_manifold_factors": lambda x: x.set_manifold_factors(win.m_stamp, win.m_sensor, win.m_pose),
        "set_pose_sensors": lambda x: x.set_pose_sensors(win.pose_sensors),
        "evaluate(trial)": lambda x: x.evaluate(jacobians=True, trial=True),
        "iterate": lambda x: x.iterate(1),
        "restore": lambda x: x.restore(),
        "profile_iteration": lambda x: x.profile_iteration(reps=1),
        "append_knots": lambda x: x.append_knots(1),
        "append_landmarks": lambda x: x.append_landmarks(win.landmarks[:1]),
        "append_pixel_factors": lambda x: x.append_pixel_factors(win.v_stamp[v:v + 1], win.v_cam[v:v + 1], win.v_lm[v:v + 1], win.v_pixel[v:v + 1]),
        "append_bearing_factors": lambda x: x.append_bearing_factors([vis_last], win.v_cam[v:v + 1], win.v_lm[v:v + 1], [[0.0, 0.0, 1.0]]),
        "append_inertial_factors": lambda x: x.append_inertial_factors(win.i_stamp[i:i + 1], win.i_meas[i:i + 1]),
        "append_manifold_factors": lambda x: x.append_manifold_factors(win.m_stamp[m:m + 1], win.m_sensor[m:m + 1], win.m_pose[m:m + 1]),
        "append_stereo_tracks": lambda x: x.append_stereo_tracks([vis_last], [0], [1], win.v_pixel[v:v + 1], win.v_pixel[v:v + 1], win.v_lm[v:v + 1]),
        "append_bias_knots": lambda x: x.append_bias_knots(win.gyro_bias[-1, 3] + bias_dt),
        "slide": lambda x: x.slide(win.knots[4, 7], drop_inertial=True, drop_manifold=True, drop_bias=True),
    }


# Return codes of PROBES after each mutation, read off the library's rules:
#   outputs changed  (evaluated Jacobians, system and covariance build dropped):  -2 -2 -2 -2  0  0
#   system changed   (system and covariance build dropped):                        0 -2 -2 -2  0  0
#   window unbound   (the above, and the window must be bound again):             -2 -2 -2 -2  0 -2
#   window reshaped  (outputs dropped, snapshot dropped, still bound):            -2 -2 -2 -2 -2  0
#   all dropped:                                                                  -2 -2 -2 -2 -2 -2
OUTPUTS, SYSTEM, UNBOUND, RESHAPED, ALL = (-2, -2, -2, -2, 0, 0), (0, -2, -2, -2, 0, 0), (-2, -2, -2, -2, 0, -2), (-2, -2, -2, -2, -2, 0), (-2,) * 6
EXPECTED = {
    "none": (0, 0, 0, 0, 0, 0),
    "set_spline(same stamps)": OUTPUTS,
    "set_spline(shifted stamps)": ALL,
    "set_bias_splines": OUTPUTS,
    "set_gravity": OUTPUTS,
    "set_cameras(same C)": OUTPUTS,
    "set_cameras(other C)": UNBOUND,
    "set_imu": OUTPUTS,
    "set_landmarks(same L)": OUTPUTS,
    "set_landmarks(other L)": ALL,
    "set_constant": SYSTEM,
    "set_reference_quirks": OUTPUTS,
    "set_options": OUTPUTS,
    "set_bearing_loss": OUTPUTS,
    "set_pixel_factors": UNBOUND,
    "set_bearing_factors": UNBOUND,
    "set_inertial_factors": UNBOUND,
    "set_manifold_factors": UNBOUND,
    "set_pose_sensors": OUTPUTS,
    "evaluate(trial)": OUTPUTS,
    "iterate": OUTPUTS,
    "restore": OUTPUTS,
    "profile_iteration": OUTPUTS,
    "append_knots": RESHAPED,
    "append_landmarks": RESHAPED,
    "append_pixel_factors": RESHAPED,
    "append_bearing_factors": RESHAPED,
    "append_inertial_factors": RESHAPED,
    "append_manifold_factors": RESHAPED,
    "append_stereo_tracks": RESHAPED,
    "append_bias_knots": RESHAPED,
    "slide": RESHAPED,
}


def prepared(win, covariance):
    """A bound window with a snapshot and evaluated Jacobians, then either a built system or a covariance build (a
    covariance build consumes the built system, and building the system after it makes the covariance build stale).
    One iteration first, so that the trial state an evaluate(trial) mutation reads has been written."""
    ctx = runtime.Context(0)
    ctx.load_window(win)
    ctx.iterate(1)
    ctx.snapshot()
    if covariance:
        ctx.build_covariance()
    else:
        ctx.evaluate(jacobians=True)
        ctx.build_system()
    return ctx


def probe(ctx, name):
    lib, h = ctx.lib, ctx.h
    if name == "factor_evaluate":
        params = (C.POINTER(C.c_double) * 16)()
        r = np.zeros(2)
        return lib.hb200_factor_evaluate(h, runtime.PIXEL, 0, params, r.ctypes.data_as(C.POINTER(C.c_double)), None)
    if name == "get_system":
        return lib.hb200_get_system(h, None, None)
    if name == "solve":
        return lib.hb200_solve(h)
    if name == "compute_covariance":
        rc = lib.hb200_compute_covariance(h, C.byref(runtime.CovarianceInfo()))
        return 0 if rc in (runtime.COV_NOT_POSITIVE_DEFINITE, runtime.COV_DEGENERATE_LANDMARKS) else rc
    if name == "restore":
        return lib.hb200_restore(h)
    if name == "evaluate":
        return lib.hb200_evaluate(h, runtime.EVAL_JACOBIANS)
    raise ValueError(name)


def test_invalidation_table(built):
    win = make_window()
    got = {}
    for name, mutate in mutations(win).items():
        codes = {}
        # the covariance compute on a window of its own; the other probes in an order in which none of them changes
        # what a later one reads (restore drops the outputs, so only evaluate follows it)
        ctx = prepared(win, covariance=True)
        mutate(ctx)
        codes["compute_covariance"] = probe(ctx, "compute_covariance")
        ctx.close()
        ctx = prepared(win, covariance=False)
        mutate(ctx)
        for p in ("factor_evaluate", "get_system", "solve", "restore", "evaluate"):
            codes[p] = probe(ctx, p)
        ctx.close()
        got[name] = tuple(codes[p] for p in PROBES)
    wrong = {n: (got[n], EXPECTED[n]) for n in EXPECTED if got[n] != EXPECTED[n]}
    assert not wrong, "(got, expected) in the order " + ", ".join(PROBES) + ": " + repr(wrong)
