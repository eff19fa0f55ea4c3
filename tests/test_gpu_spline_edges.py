"""Factor evaluation and spline interpolation against the 80-digit known answers in tests/golden/, entry by entry.

The k*_spline_edges windows put knot increments d_j and blended increments lambda_j d_j on both sides of the
small-angle switches of the SO(3) coefficients (hb200_math.cuh), store every other knot as -q, and place stamps at
u = 0 and at the last double below a segment end.  Every residual, Jacobian row and interpolated pose, velocity and
acceleration of every fixture must satisfy |got - ref| <= C u scale(row), u = 2^-53.

C = 150: a Jacobian entry ends a chain of about 25 dependent roundings (knot increment and its Jr^-1, k - 1 blended
exponentials and right Jacobians, the rotation product, the sensor model and its chain rule), each accurate to a few
ulps of the row's scale.  The oracle's worst ratio is 11; with the cancelling closed forms the coefficients had before
(1 - cos t at t = 1e-4 is 1e8 ulps wrong) the edge windows reach 3200 (k = 4) and 5600 (k = 6).

scale(row):
  * Jacobian row: its largest entry over every block; a bearing row divided by its angle (when below a radian),
    because rounding p_s by u tilts the plane of the angle, and so the gradient, by u / angle;
  * residual: the largest of the residual, its measurement and its Jacobian row (rounding a stored rotation moves it
    by u radians); a bearing's measurement is a unit direction;
  * interpolation: quaternion and position rows on their own size and the span's largest knot position; a rate or
    acceleration row on its own size and on what a unit change of the knots moves it by: inv_dt^n for rotation,
    inv_dt^n times the largest knot position for translation.
"""
import glob
import json
import os

import numpy as np
import pytest

import oracle_lib as ol
from test_oracle import window_from_golden

U = 2.0 ** -53
C = 150.0
GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "*.json")))


def load(path):
    with open(path) as f:
        return json.load(f)


def _worst(got, ref, scale):
    return float(np.max(np.abs(np.asarray(got, float) - np.asarray(ref, float)) / (U * scale)))


def factor_ratios(case, out):
    """Worst |got - ref| / (u scale) of each factor family's residuals and Jacobians."""
    worst = {}

    def put(key, v):
        worst[key] = max(worst.get(key, 0.0), v)

    for f, p in enumerate(case["pixel"]):
        J = np.hstack([np.array(p["Jp"]), np.array(p["Jl"])])
        got = np.hstack([out["v_Jp"][f], out["v_Jl"][f]])
        for i in range(2):
            s = np.abs(J[i]).max()
            put("pixel_J", _worst(got[i], J[i], s))
            put("pixel_r", _worst(out["v_r"][f][i], p["r"][i], max(s, abs(p["r"][i]), np.abs(p["pixel"]).max())))
    for f, p in enumerate(case.get("bearing", [])):
        J = np.concatenate([p["Jp"], p["Jl"]])
        s = np.abs(J).max()
        put("bearing_J", _worst(np.concatenate([out["b_Jp"][f], out["b_Jl"][f]]), J, s / min(1.0, abs(p["r"][0]))))
        put("bearing_r", _worst(out["b_r"][f], p["r"][0], max(s, abs(p["r"][0]), 1.0)))
    for f, p in enumerate(case.get("pose", [])):
        J = np.array(p["Jp"])
        for i in range(6):
            s = np.abs(J[i]).max()
            put("pose_J", _worst(out["m_Jp"][f][i], J[i], s))
            put("pose_r", _worst(out["m_r"][f][i], p["r"][i], max(s, abs(p["r"][i]), np.abs(p["pose"]).max())))
    for f, p in enumerate(case["inertial"]):
        Jg = np.array(p["Jg"])
        for i in range(6):
            ref_b, got_b = (p["wg"], out["i_wg"][f]) if i < 3 else (p["wa"], out["i_wa"][f])   # a row's bias weights
            J = np.concatenate([p["Jp"][i], ref_b, Jg[i]])
            got = np.concatenate([out["i_Jp"][f][i], got_b, out["i_Jg"][f][i]])
            s = np.abs(J).max()
            put("inertial_J", _worst(got, J, s))
            meas = np.abs(p["meas"][:3] if i < 3 else p["meas"][3:]).max()
            put("inertial_r", _worst(out["i_r"][f][i], p["r"][i], max(s, abs(p["r"][i]), meas)))
    return worst


def interpolate_ratios(case, pose, vel, acc):
    """Worst |got - ref| / (u scale) of hb200_interpolate's pose, velocity and acceleration rows."""
    w = case["window"]
    knots = np.array(w["knots"])
    k = w["order"]
    left = (k - 1) // 2
    worst = dict(interp_pose=0.0, interp_vel=0.0, interp_acc=0.0)
    for n, a in enumerate(case["interpolate"]):
        j = int(np.searchsorted(knots[:, 7], a["stamp"], side="right") - 1)
        inv_dt = 1.0 / (knots[j + 1, 7] - knots[j, 7])
        pmax = np.abs(knots[j - left:j - left + k, 4:7]).max()
        ref_pose, ref_vel, ref_acc = (np.array(a[key]) for key in ("pose", "vel", "acc"))
        worst["interp_pose"] = max(worst["interp_pose"], _worst(pose[n][:4], ref_pose[:4], np.abs(ref_pose[:4]).max()),
                                   _worst(pose[n][4:], ref_pose[4:], max(np.abs(ref_pose[4:]).max(), pmax)))
        for key, got, ref, order in (("interp_vel", vel[n], ref_vel, 1), ("interp_acc", acc[n], ref_acc, 2)):
            rot = max(np.abs(ref[:3]).max(), inv_dt ** order)
            trans = max(np.abs(ref[3:]).max(), inv_dt ** order * pmax)
            worst[key] = max(worst[key], _worst(got[:3], ref[:3], rot), _worst(got[3:], ref[3:], trans))
    return worst


def check(worst, record_property, name):
    for key, v in worst.items():
        record_property(f"{name}:{key}", round(v, 3))
    bad = {key: v for key, v in worst.items() if not v <= C}
    assert not bad, f"{name}: worst |got - ref| / (u scale) above C = {C:g}: {bad}"


def oracle_interpolate(case):
    w = case["window"]
    knots = np.array(w["knots"])
    k = w["order"]
    left = (k - 1) // 2
    pose, vel, acc = [], [], []
    for a in case["interpolate"]:
        j = int(np.searchsorted(knots[:, 7], a["stamp"], side="right") - 1) - left
        v, ve, ac, _ = ol.state_evaluate(knots[j:j + k], a["stamp"], 2, False)
        pose.append(v); vel.append(ve); acc.append(ac)
    return np.array(pose), np.array(vel), np.array(acc)


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_oracle_rows_against_golden(path, record_property):
    """CPU twin of the GPU test: the oracle's factor evaluation and state_evaluate under the same bound."""
    case = load(path)
    win = window_from_golden(case)
    ow = ol.OracleWindow(win)
    assert ow.bad == 0
    worst = factor_ratios(case, ow.evaluate())
    if "interpolate" in case:
        worst.update(interpolate_ratios(case, *oracle_interpolate(case)))
    check(worst, record_property, os.path.basename(path))


@pytest.mark.gpu
@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_gpu_rows_against_golden(built, path, record_property):
    from hyperslam_b200 import runtime
    case = load(path)
    win = window_from_golden(case)
    ctx = runtime.Context(0)
    ctx.load_window(win)
    ctx.evaluate(jacobians=True)
    worst = factor_ratios(case, ctx.outputs())
    if "interpolate" in case:
        stamps = np.array([a["stamp"] for a in case["interpolate"]])
        pose, vel, acc, bad = ctx.interpolate(stamps)
        assert bad == 0
        worst.update(interpolate_ratios(case, pose, vel, acc))
    ctx.close()
    check(worst, record_property, os.path.basename(path))
