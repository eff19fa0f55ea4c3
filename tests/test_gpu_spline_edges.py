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
  * calibration-block row (golden/calib/: hb200_factor_evaluate's camera / IMU / pose-sensor blocks, quirks = 0): the
    same, over the state and calibration blocks together.  Extrinsics come out in the 7-wide ambient layout and are compared in the
    tangent of the known answers (R_bs <- Exp(theta) R_bs, t_bs <- t_bs + rho) through the oracle's Plus Jacobian:
    EigenQuaternionManifold's delta d turns by Exp(2 d), so theta = 2 d.  Worst ratios 10 (oracle) and 4.7 (device);
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


def load_calib(path):
    return load(os.path.join(os.path.dirname(path), "calib", os.path.basename(path)))


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


def ext_tangent(J, T):
    """Ambient extrinsics block (rows x 7) -> the known answers' tangent [theta | rho] (rows x 6)."""
    return np.asarray(J) @ ol.manifold_plus_jacobian(ol.M_SE3, T) @ np.diag([0.5, 0.5, 0.5, 1.0, 1.0, 1.0])


def calibration_ratios(case, calib, evaluate):
    """Worst |got - ref| / (u scale) of the calibration blocks of golden/calib/<case>.json (every pixel, bearing and pose
    factor, the first inertial one).  evaluate(kind, f, stamp, meas, blocks) returns the per-block Jacobians of factor f
    (kind: ol.PIXEL ...) in hb200_factor_evaluate's block order."""
    w = case["window"]
    k, kb = w["order"], w["bias_order"]
    knots, cams, imu = np.array(w["knots"]), np.array(w["cameras"]), np.array(w["imu"])
    worst = {}

    def put(key, got, ref, s):
        worst[key] = max(worst.get(key, 0.0), _worst(got, ref, s))

    for f, (p, c) in enumerate(zip(case["pixel"], calib["pixel"])):
        cam = cams[p["cam"]]
        blocks = [knots[p["base"] + m] for m in range(k)] + [cam[:7], cam[7:11], cam[11:15], np.array(w["landmarks"][p["lm"]])]
        jac = evaluate(ol.PIXEL, f, p["stamp"], p["pixel"], blocks)
        got = np.hstack([ext_tangent(jac[k], cam[:7]), jac[k + 1], jac[k + 2]])
        ref = np.hstack([c["Jext"], c["Jintr"], c["Jdist"]])
        for i in range(2):
            s = max(np.abs(ref[i]).max(), np.abs(p["Jp"][i]).max(), np.abs(p["Jl"][i]).max())
            put("pixel_calib", got[i], ref[i], s)
    for f, (p, c) in enumerate(zip(case.get("bearing", []), calib["bearing"])):
        cam = cams[p["cam"]]
        blocks = [knots[p["base"] + m] for m in range(k)] + [cam[:7], cam[7:11], cam[11:15], np.array(w["landmarks"][p["lm"]])]
        jac = evaluate(ol.BEARING, f, p["stamp"], p["bearing"], blocks)
        s = max(np.abs(c["Jext"]).max(), np.abs(p["Jp"]).max(), np.abs(p["Jl"]).max())
        put("bearing_calib", ext_tangent(jac[k], cam[:7])[0], c["Jext"], s / min(1.0, abs(p["r"][0])))
    for f, (p, c) in enumerate(zip(case.get("pose", []), calib["pose"])):
        T = np.array(w["pose_sensors"][p["sensor"]])
        jac = evaluate(ol.MANIFOLD, f, p["stamp"], p["pose"], [knots[p["base"] + m] for m in range(k)] + [T])
        got = ext_tangent(jac[k], T)
        for i in range(6):
            put("pose_calib", got[i], c["Jext"][i], max(np.abs(c["Jext"][i]).max(), np.abs(p["Jp"][i]).max()))
    gb, ga = np.array(w["gyro_bias"]), np.array(w["accel_bias"])
    for f, (p, c) in enumerate(zip(case["inertial"], calib["inertial"])):
        b = p["bias_base"]
        blocks = ([knots[p["base"] + m] for m in range(k)] + [imu[:7], imu[7:13], imu[13:19], imu[19:28], imu[28:37]]
                  + [gb[b + m] for m in range(kb)] + [ga[b + m] for m in range(kb)] + [np.array(w["gravity"])])
        jac = evaluate(ol.INERTIAL, f, p["stamp"], p["meas"], blocks)
        got = np.hstack([ext_tangent(jac[k], imu[:7])] + [jac[k + j] for j in range(1, 5)])
        ref = np.hstack([c[key] for key in ("Jext", "JIg", "JIa", "JSg", "JXa")])
        for i in range(6):
            state = np.concatenate([p["Jp"][i], p["wg"] if i < 3 else p["wa"], p["Jg"][i]])
            put("inertial_calib", got[i], ref[i], max(np.abs(ref[i]).max(), np.abs(state).max()))
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
    kb = case["window"]["bias_order"]
    worst.update(calibration_ratios(case, load_calib(path), lambda kind, f, stamp, meas, blocks: ol.cost_evaluate(
        kind, stamp, np.asarray(meas, float), np.concatenate(blocks), k=case["window"]["order"], k_bg=kb, k_ba=kb)[1]))
    check(worst, record_property, os.path.basename(path))


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_extrinsics_tangent_matches_golden_perturbation(path):
    """ext_tangent's conversion, checked on the value formula of the known answers: ol.manifold_plus on an SE3 block
    by d (rotation) and rho moves the mpmath residual as the fixtures' R_bs <- Exp(2 d) R_bs, t_bs <- t_bs + rho does."""
    import mpmath as mp
    from test_stateref import mg
    case = load(path)
    win = window_from_golden(case)
    st = mg.to_mp_state(win)
    rng = np.random.default_rng(3)
    fams = [("pixel", mg.pixel_residual, "cam_ext", "cam", lambda p: dict(cam=p["cam"], lm=p["lm"], pixel=[mp.mpf(x) for x in p["pixel"]])),
            ("pose", mg.pose_residual, "sensor_ext", "sensor", lambda p: dict(sensor=p["sensor"], pose=[mp.mpf(x) for x in p["pose"]])),
            ("inertial", mg.inertial_residual, "imu_ext", None, lambda p: dict(meas=[mp.mpf(x) for x in p["meas"]]))]
    checked = 0
    for fam, fn, kind, key, fields in fams:
        for p in case.get(fam, [])[:1]:
            f = dict(stamp=mp.mpf(p["stamp"]), **fields(p))
            index = p[key] if key else 0
            store = {"cam_ext": "cams", "sensor_ext": "pose_sensors", "imu_ext": "imu"}[kind]
            rows = [list(st["imu"])] if store == "imu" else [list(v) for v in st[store]]
            row = rows[0 if store == "imu" else index]
            d = rng.normal(0, 1e-6, 6)
            row[:7] = [mp.mpf(x) for x in ol.manifold_plus(ol.M_SE3, np.array([float(x) for x in row[:7]]), d)]
            a = dict(st, **{store: rows[0] if store == "imu" else rows})
            b = st
            for c in range(6):
                b = mg.perturbed(b, kind, index, c, mp.mpf(2 * d[c] if c < 3 else d[c]))
            ra, rb, r0 = (np.array([float(v) for v in fn(x, f)]) for x in (a, b, st))
            # the moves agree to second order (composing the six single-coordinate moves); Exp(d) would miss by |r - r0| / 2
            assert np.abs(ra - rb).max() < 1e-4 * np.abs(ra - r0).max(), (fam, ra - rb, ra - r0)
            checked += 1
    assert checked


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
    kind = {ol.PIXEL: runtime.PIXEL, ol.INERTIAL: runtime.INERTIAL, ol.BEARING: runtime.BEARING, ol.MANIFOLD: runtime.MANIFOLD}
    worst.update(calibration_ratios(case, load_calib(path), lambda k, f, stamp, meas, blocks: ctx.factor_evaluate(kind[k], f, blocks)[1]))
    ctx.close()
    check(worst, record_property, os.path.basename(path))
