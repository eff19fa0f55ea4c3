#!/usr/bin/env python
"""Generates tests/golden/*.json: known-answer vectors for the hot path at 80 significant digits.

Independent of both the C oracle and the CUDA kernels:
  * only VALUE formulas are implemented (SURVEY.md Appendix A: cumulative B-spline on SO(3) x R^3,
    pinhole + radial-tangential camera, the IMU model of reference inertial.cpp:62-79);
  * body rates come from finite differences of R(t) in time (omega^ = R^T Rdot,
    alpha^ = R^T Rddot - omega^ omega^), NOT from the Sommer recursion the oracle/kernels use;
  * Jacobians come from central differences of the residual along the manifold retractions
    (R <- Exp(theta) R, p <- p + rho, Ceres SphereManifold Plus for gravity), h = 1e-20;
  * calib/<case>.json: calibration blocks (hb200_factor_evaluate) of the case's factors: camera / IMU / pose-sensor
    extrinsics in the tangent R_bs <- Exp(theta) R_bs, t_bs <- t_bs + rho, and intrinsics, distortion, I_g, I_a, S_g,
    X_a in their raw coordinates;
  * the edge windows (k*_spline_edges) also carry hb200_interpolate answers: pose, body velocity and body
    acceleration from the same time differences;
  * ingest/k*_stereo_ingest hold stereo tracks on the edge windows with their bearings (the distortion inverted by
    mp.findroot), the midpoint p_0 in camera 0 and the world landmark.
Run:  python tests/golden/make_golden.py      (takes ~2 minutes)
"""
import dataclasses
import json
import os
import sys

import mpmath as mp
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from hyperslam_b200 import synthetic  # noqa: E402

mp.mp.dps = 80
H_T = mp.mpf(10) ** -18    # time step for body-rate finite differences
H_X = mp.mpf(10) ** -20    # state perturbation


def hat(v):
    return mp.matrix([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


def so3_exp(w):
    t = mp.sqrt(w[0] ** 2 + w[1] ** 2 + w[2] ** 2)
    W = hat(w)
    if t == 0:
        return mp.eye(3)
    return mp.eye(3) + (mp.sin(t) / t) * W + ((1 - mp.cos(t)) / t ** 2) * (W * W)


def quat_to_rot(q):
    x, y, z, w = q
    return mp.matrix([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                      [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                      [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def quat_mul(a, b):
    return [a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1],
            a[3] * b[1] - a[0] * b[2] + a[1] * b[3] + a[2] * b[0],
            a[3] * b[2] + a[0] * b[1] - a[1] * b[0] + a[2] * b[3],
            a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2]]


def quat_exp(d):
    t = mp.sqrt(d[0] ** 2 + d[1] ** 2 + d[2] ** 2)
    if t == 0:
        return [mp.mpf(0)] * 3 + [mp.mpf(1)]
    s = mp.sin(t / 2) / t
    return [s * d[0], s * d[1], s * d[2], mp.cos(t / 2)]


def quat_log(q):
    x, y, z, w = q
    if w < 0:
        x, y, z, w = -x, -y, -z, -w
    n = mp.sqrt(x * x + y * y + z * z)
    if n == 0:
        return [mp.mpf(0)] * 3
    s = 2 * mp.atan2(n, w) / n
    return [s * x, s * y, s * z]


def basis(k, u):
    """lambda_j(u), j = 0..k (cumulative), exact rational blending matrix."""
    Mc = [[mp.mpf(0)] * k for _ in range(k)]
    M = [[mp.mpf(0)] * k for _ in range(k)]
    for s in range(k):
        for n in range(k):
            acc = mp.mpf(0)
            for l in range(s, k):
                acc += (-1) ** (l - s) * mp.binomial(k, l - s) * mp.mpf(k - 1 - l) ** (k - 1 - n)
            M[s][n] = mp.binomial(k - 1, n) / mp.factorial(k - 1) * acc
    for j in range(k):
        for n in range(k):
            Mc[j][n] = sum(M[r][n] for r in range(j, k))
    lam = [sum(Mc[j][n] * u ** n for n in range(k)) for j in range(k)] + [mp.mpf(0)]
    lam[0] = mp.mpf(1)
    return lam


def segment(stamps, k, t, pin=None):
    """Base knot and u of t in the segment holding `pin` (default t): time differences stay on the segment of the
    stamp they differentiate at, as the kernels do, even where t +- h crosses a knot."""
    j = max(i for i in range(len(stamps)) if stamps[i] <= (t if pin is None else pin))
    return j - (k - 1) // 2, (t - stamps[j]) / (stamps[j + 1] - stamps[j])


def pose_q(knots, k, t, pin=None):
    """q(t) [x y z w], p(t) of the split cumulative spline; knots: list of [q(4) p(3) stamp]."""
    stamps = [kn[7] for kn in knots]
    base, u = segment(stamps, k, t, pin)
    lam = basis(k, u)
    q = list(knots[base][:4])
    p = mp.matrix(knots[base][4:7])
    for j in range(1, k):
        qa, qb = knots[base + j - 1][:4], knots[base + j][:4]
        d = quat_log(quat_mul([-qa[0], -qa[1], -qa[2], qa[3]], qb))
        q = quat_mul(q, quat_exp([lam[j] * c for c in d]))
        p = p + lam[j] * (mp.matrix(knots[base + j][4:7]) - mp.matrix(knots[base + j - 1][4:7]))
    return q, p


def pose(knots, k, t, pin=None):
    """R(t), p(t) of the split cumulative spline."""
    q, p = pose_q(knots, k, t, pin)
    return quat_to_rot(q), p


def bias(bknots, kb, t):
    stamps = [b[3] for b in bknots]
    base, u = segment(stamps, kb, t)
    lam = basis(kb, u)
    return sum(((lam[m] - lam[m + 1]) * mp.matrix(bknots[base + m][:3]) for m in range(kb)), mp.matrix([0, 0, 0]))


def vee(M):
    return mp.matrix([(M[2, 1] - M[1, 2]) / 2, (M[0, 2] - M[2, 0]) / 2, (M[1, 0] - M[0, 1]) / 2])


def pixel_residual(st, f):
    R, p = pose(st["knots"], st["k"], f["stamp"])
    cam = st["cams"][f["cam"]]
    R_bs = quat_to_rot(cam[:4]); t_bs = mp.matrix(cam[4:7])
    p_b = R.T * (mp.matrix(st["landmarks"][f["lm"]]) - p)
    p_s = R_bs.T * (p_b - t_bs)
    x, y = p_s[0] / p_s[2], p_s[1] / p_s[2]
    cx, cy, fx, fy, k1, k2, p1, p2 = cam[7:15]
    r2 = x * x + y * y
    rad = 1 + k1 * r2 + k2 * r2 * r2
    dx = x * rad + 2 * p1 * x * y + p2 * (r2 + 2 * x * x)
    dy = y * rad + p1 * (r2 + 2 * y * y) + 2 * p2 * x * y
    return [fx * dx + cx - f["pixel"][0], fy * dy + cy - f["pixel"][1]]


def bearing_residual(st, f):
    """AngularMetric<Bearing>: angle between p_s (reference bearing.cpp:58-60) and the measured direction."""
    R, p = pose(st["knots"], st["k"], f["stamp"])
    cam = st["cams"][f["cam"]]
    R_bs = quat_to_rot(cam[:4]); t_bs = mp.matrix(cam[4:7])
    p_s = R_bs.T * (R.T * (mp.matrix(st["landmarks"][f["lm"]]) - p) - t_bs)
    b = mp.matrix(f["bearing"])
    cr = mp.matrix([p_s[1] * b[2] - p_s[2] * b[1], p_s[2] * b[0] - p_s[0] * b[2], p_s[0] * b[1] - p_s[1] * b[0]])
    return [mp.atan2(mp.sqrt(cr[0] ** 2 + cr[1] ** 2 + cr[2] ** 2), p_s[0] * b[0] + p_s[1] * b[1] + p_s[2] * b[2])]


def rot_log(R):
    c = (R[0, 0] + R[1, 1] + R[2, 2] - 1) / 2
    t = mp.acos(c)
    v = vee(R - R.T)         # vee() averages the two off-diagonal entries: vee(R - R^T) = 2 sin(t) axis
    return v * (t / (2 * mp.sin(t))) if t != 0 else mp.matrix([0, 0, 0])


def pose_residual(st, f):
    """ManifoldMetric<SE3> of T_ws = T_wb (+) T_bs (reference manifold.cpp:38) against the measured pose."""
    R, p = pose(st["knots"], st["k"], f["stamp"])
    T_bs = st["pose_sensors"][f["sensor"]]
    R_ws = R * quat_to_rot(T_bs[:4])
    p_ws = p + R * mp.matrix(T_bs[4:7])
    th = rot_log(R_ws * quat_to_rot(f["pose"][:4]).T)
    d = p_ws - mp.matrix(f["pose"][4:7])
    return [th[0], th[1], th[2], d[0], d[1], d[2]]


def imu_matrix(c):
    return mp.matrix([[c[0], 0, 0], [c[3], c[1], 0], [c[4], c[5], c[2]]])


def inertial_residual(st, f):
    t = f["stamp"]
    R0, p0 = pose(st["knots"], st["k"], t)
    Rp, pp = pose(st["knots"], st["k"], t + H_T, pin=t)
    Rm, pm = pose(st["knots"], st["k"], t - H_T, pin=t)
    Rd = (Rp - Rm) / (2 * H_T)
    Rdd = (Rp - 2 * R0 + Rm) / H_T ** 2
    pdd = (pp - 2 * p0 + pm) / H_T ** 2
    wx = R0.T * Rd
    w = vee(wx)
    al = vee(R0.T * Rdd - hat(w) * hat(w))
    imu = st["imu"]
    R_sb = quat_to_rot(imu[:4]).T; t_bs = mp.matrix(imu[4:7])
    I_g, I_a = imu_matrix(imu[7:13]), imu_matrix(imu[13:19])
    S_g = mp.matrix(3, 3); X_a = mp.matrix(3, 3)
    for i in range(3):
        for j in range(3):
            S_g[i, j] = imu[19 + i + 3 * j]; X_a[i, j] = imu[28 + i + 3 * j]
    a_i = R0.T * (pdd - mp.matrix(st["gravity"]))
    F = hat(w) * hat(w) + hat(al)
    a_m = mp.matrix([a_i[r] + sum(F[r, c] * (X_a[c, r] + t_bs[c]) for c in range(3)) for r in range(3)])
    gyro = I_g * R_sb * w + S_g * a_m + bias(st["bg"], st["kb"], t)
    acc = I_a * R_sb * a_m + bias(st["ba"], st["kb"], t)
    z = f["meas"]
    return [gyro[i] - z[i] for i in range(3)] + [acc[i] - z[3 + i] for i in range(3)]


def sphere_plus(x, d):
    x = [mp.mpf(v) for v in x]
    nd = mp.sqrt(d[0] ** 2 + d[1] ** 2)
    if nd == 0:
        return x
    sigma = x[0] ** 2 + x[1] ** 2
    v = [x[0], x[1], mp.mpf(1)]
    beta = mp.mpf(0)
    if sigma == 0:
        if x[2] < 0:
            beta = mp.mpf(2)
    else:
        mu = mp.sqrt(x[2] ** 2 + sigma)
        vp = x[2] - mu if x[2] <= 0 else -sigma / (x[2] + mu)
        beta = 2 * vp * vp / (sigma + vp * vp)
        v[0] /= vp; v[1] /= vp
    nx = mp.sqrt(sigma + x[2] ** 2)
    y = [mp.sin(nd) / nd * d[0], mp.sin(nd) / nd * d[1], mp.cos(nd)]
    vy = sum(a * b for a, b in zip(v, y))
    return [nx * (y[i] - v[i] * beta * vy) for i in range(3)]


def perturbed(st, kind, index, comp, h):
    """Copy of st with one tangent coordinate moved by h."""
    out = dict(st)
    if kind == "knot":
        knots = [list(kn) for kn in st["knots"]]
        kn = knots[index]
        if comp < 3:
            d = [mp.mpf(0)] * 3; d[comp] = h
            kn[:4] = quat_mul(quat_exp(d), kn[:4])
        else:
            kn[4 + comp - 3] += h
        out["knots"] = knots
    elif kind == "landmark":
        lm = [list(v) for v in st["landmarks"]]
        lm[index][comp] += h
        out["landmarks"] = lm
    elif kind in ("bg", "ba"):
        b = [list(v) for v in st[kind]]
        b[index][comp] += h
        out[kind] = b
    elif kind == "gravity":
        d = [mp.mpf(0)] * 2; d[comp] = h
        out["gravity"] = sphere_plus(st["gravity"], d)
    elif kind in ("cam_ext", "sensor_ext", "imu_ext"):
        # extrinsics T_bs in the tangent of hb200_calib.cuh: R_bs <- Exp(theta) R_bs, t_bs <- t_bs + rho
        key = {"cam_ext": "cams", "sensor_ext": "pose_sensors", "imu_ext": "imu"}[kind]
        rows = [list(st["imu"])] if key == "imu" else [list(v) for v in st[key]]
        T = rows[0 if key == "imu" else index]
        if comp < 3:
            d = [mp.mpf(0)] * 3; d[comp] = h
            T[:4] = quat_mul(quat_exp(d), T[:4])
        else:
            T[4 + comp - 3] += h
        out[key] = rows[0] if key == "imu" else rows
    elif kind in ("cam_intr", "cam_dist"):
        cams = [list(v) for v in st["cams"]]
        cams[index][(7 if kind == "cam_intr" else 11) + comp] += h
        out["cams"] = cams
    elif kind in IMU_BLOCKS:
        # I_g, I_a (6 raw entries, imu_matrix's order), S_g, X_a (9, column-major): raw coordinates
        imu = list(st["imu"])
        imu[IMU_BLOCKS[kind][0] + comp] += h
        out["imu"] = imu
    return out


IMU_BLOCKS = {"I_g": (7, 6), "I_a": (13, 6), "S_g": (19, 9), "X_a": (28, 9)}   # offset in the imu row, size


def numdiff(fn, st, f, kind, index, comp):
    rp = fn(perturbed(st, kind, index, comp, H_X), f)
    rm = fn(perturbed(st, kind, index, comp, -H_X), f)
    return [(a - b) / (2 * H_X) for a, b in zip(rp, rm)]


def to_mp_state(w):
    f = lambda a: [[mp.mpf(float(x)) for x in row] for row in np.asarray(a)]
    return dict(k=w.order, kb=w.bias_order, knots=f(w.knots), cams=f(w.cameras), imu=[mp.mpf(float(x)) for x in w.imu],
                landmarks=f(w.landmarks), bg=f(w.gyro_bias), ba=f(w.accel_bias), gravity=[mp.mpf(float(x)) for x in w.gravity],
                pose_sensors=f(w.pose_sensors))


def make_case(name, n_pix=3, n_imu=3, **kw):
    w = synthetic.make_window(**kw)
    st = to_mp_state(w)
    rng = np.random.default_rng(7)
    pix_idx = sorted(rng.choice(w.v_stamp.size, n_pix, replace=False).tolist()) if w.v_stamp.size else []
    imu_idx = sorted(rng.choice(w.i_stamp.size, n_imu, replace=False).tolist())
    case = dict(name=name, window=window_json(w), pixel=[], inertial=[], digits=mp.mp.dps)
    for f_ in pix_idx:
        case["pixel"].append(pixel_answer(st, w, f_))
        print(name, "pixel", f_, case["pixel"][-1]["r"])
    for f_ in imu_idx:
        case["inertial"].append(inertial_answer(st, w, f_))
        print(name, "inertial", f_, case["inertial"][-1]["r"][:3])
    write_case(name, case)
    write_calibration(name, st, case)


def make_widened_case(name, n_bearing=3, n_pose=3, **kw):
    """Bearing + pose factors (the two other residual families of reference optimizer.cpp:189-251)."""
    w = synthetic.add_bearing_and_pose_factors(synthetic.make_window(**kw), num_bearing=8, num_pose=8, seed=kw["seed"] + 50)
    st = to_mp_state(w)
    case = dict(name=name, window=window_json(w), pixel=[], inertial=[], bearing=[], pose=[], digits=mp.mp.dps)
    for f_ in range(n_bearing):
        case["bearing"].append(bearing_answer(st, w, f_))
        print(name, "bearing", f_, case["bearing"][-1]["r"])
    for f_ in range(n_pose):
        case["pose"].append(pose_answer(st, w, f_))
        print(name, "pose", f_, case["pose"][-1]["r"][:3])
    write_case(name, case)
    write_calibration(name, st, case)


fl = lambda v: [float(x) for x in v]


def calib_block(fn, st, f, kind, index, n):
    """Rows x n Jacobian of fn along the n coordinates of one calibration block (perturbed())."""
    cols = [numdiff(fn, st, f, kind, index, c) for c in range(n)]
    return [[float(col[row]) for col in cols] for row in range(len(cols[0]))]


def write_calibration(name, st, case):
    """calib/<name>.json: the calibration blocks (hb200_factor_evaluate's sensor blocks) of every pixel, bearing and pose
    factor of a case and of its first inertial factor (216 entries each), in perturbed()'s coordinates."""
    mpl = lambda v: [mp.mpf(x) for x in v]
    out = dict(pixel=[], bearing=[], pose=[], inertial=[])
    for a in case["pixel"]:
        f = dict(stamp=mp.mpf(a["stamp"]), cam=a["cam"], lm=a["lm"], pixel=mpl(a["pixel"]))
        out["pixel"].append(dict(Jext=calib_block(pixel_residual, st, f, "cam_ext", a["cam"], 6), Jintr=calib_block(pixel_residual, st, f, "cam_intr", a["cam"], 4),
                                 Jdist=calib_block(pixel_residual, st, f, "cam_dist", a["cam"], 4)))
    for a in case.get("bearing", []):
        f = dict(stamp=mp.mpf(a["stamp"]), cam=a["cam"], lm=a["lm"], bearing=mpl(a["bearing"]))
        out["bearing"].append(dict(Jext=calib_block(bearing_residual, st, f, "cam_ext", a["cam"], 6)[0]))
    for a in case.get("pose", []):
        f = dict(stamp=mp.mpf(a["stamp"]), sensor=a["sensor"], pose=mpl(a["pose"]))
        out["pose"].append(dict(Jext=calib_block(pose_residual, st, f, "sensor_ext", a["sensor"], 6)))
    for a in case["inertial"][:1]:
        f = dict(stamp=mp.mpf(a["stamp"]), meas=mpl(a["meas"]))
        out["inertial"].append(dict(Jext=calib_block(inertial_residual, st, f, "imu_ext", 0, 6),
                                    **{"J" + b.replace("_", ""): calib_block(inertial_residual, st, f, b, 0, n) for b, (_, n) in IMU_BLOCKS.items()}))
    write_case(os.path.join("calib", name), out)


def pixel_answer(st, w, i):
    k = st["k"]
    f = dict(stamp=mp.mpf(float(w.v_stamp[i])), cam=int(w.v_cam[i]), lm=int(w.v_lm[i]), pixel=[mp.mpf(float(x)) for x in w.v_pixel[i]])
    base, _ = segment([kn[7] for kn in st["knots"]], k, f["stamp"])
    r = pixel_residual(st, f)
    Jp = [numdiff(pixel_residual, st, f, "knot", base + m, c) for m in range(k) for c in range(6)]   # columns
    Jl = [numdiff(pixel_residual, st, f, "landmark", f["lm"], c) for c in range(3)]
    return dict(stamp=float(w.v_stamp[i]), cam=f["cam"], lm=f["lm"], pixel=w.v_pixel[i].tolist(), base=base, r=fl(r),
                Jp=[[float(Jp[c][row]) for c in range(6 * k)] for row in range(2)], Jl=[[float(Jl[c][row]) for c in range(3)] for row in range(2)])


def inertial_answer(st, w, i):
    k, kb = st["k"], st["kb"]
    f = dict(stamp=mp.mpf(float(w.i_stamp[i])), meas=[mp.mpf(float(x)) for x in w.i_meas[i]])
    base, _ = segment([kn[7] for kn in st["knots"]], k, f["stamp"])
    gb, _ = segment([b[3] for b in st["bg"]], kb, f["stamp"])
    r = inertial_residual(st, f)
    Jp = [numdiff(inertial_residual, st, f, "knot", base + m, c) for m in range(k) for c in range(6)]
    wg = [numdiff(inertial_residual, st, f, "bg", gb + m, 0)[0] for m in range(kb)]
    wa = [numdiff(inertial_residual, st, f, "ba", gb + m, 0)[3] for m in range(kb)]
    Jg = [numdiff(inertial_residual, st, f, "gravity", 0, c) for c in range(2)]
    return dict(stamp=float(w.i_stamp[i]), meas=w.i_meas[i].tolist(), base=base, bias_base=gb, r=fl(r),
                Jp=[[float(Jp[c][row]) for c in range(6 * k)] for row in range(6)], wg=fl(wg), wa=fl(wa),
                Jg=[[float(Jg[c][row]) for c in range(2)] for row in range(6)])


def bearing_answer(st, w, i):
    k = st["k"]
    f = dict(stamp=mp.mpf(float(w.b_stamp[i])), cam=int(w.b_cam[i]), lm=int(w.b_lm[i]), bearing=[mp.mpf(float(x)) for x in w.b_bearing[i]])
    base, _ = segment([kn[7] for kn in st["knots"]], k, f["stamp"])
    r = bearing_residual(st, f)
    Jp = [numdiff(bearing_residual, st, f, "knot", base + m, c) for m in range(k) for c in range(6)]
    Jl = [numdiff(bearing_residual, st, f, "landmark", f["lm"], c) for c in range(3)]
    return dict(stamp=float(w.b_stamp[i]), cam=f["cam"], lm=f["lm"], bearing=w.b_bearing[i].tolist(), base=base, r=fl(r),
                Jp=[float(Jp[c][0]) for c in range(6 * k)], Jl=[float(Jl[c][0]) for c in range(3)])


def pose_answer(st, w, i):
    k = st["k"]
    f = dict(stamp=mp.mpf(float(w.m_stamp[i])), sensor=int(w.m_sensor[i]), pose=[mp.mpf(float(x)) for x in w.m_pose[i]])
    base, _ = segment([kn[7] for kn in st["knots"]], k, f["stamp"])
    r = pose_residual(st, f)
    Jp = [numdiff(pose_residual, st, f, "knot", base + m, c) for m in range(k) for c in range(6)]
    return dict(stamp=float(w.m_stamp[i]), sensor=f["sensor"], pose=w.m_pose[i].tolist(), base=base, r=fl(r),
                Jp=[[float(Jp[c][row]) for c in range(6 * k)] for row in range(6)])


def window_json(w):
    out = dict(order=w.order, bias_order=w.bias_order, knots=w.knots.tolist(), gyro_bias=w.gyro_bias.tolist(), accel_bias=w.accel_bias.tolist(),
               gravity=w.gravity.tolist(), cameras=w.cameras.tolist(), imu=w.imu.tolist(), landmarks=w.landmarks.tolist())
    if w.pose_sensors.size:
        out["pose_sensors"] = w.pose_sensors.tolist()
    return out


def write_case(name, case):
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), f"{name}.json")
    with open(out, "w") as fh:
        json.dump(case, fh)
    print("wrote", out)


# ---- windows at the spline's numerical edges --------------------------------------------------------
# The SO(3) coefficient functions take w = d_j (a knot increment) or lambda_j d_j (a blended one).  They switch to series
# at |w| = 1e-7 (quaternion exp and log) and |w|^2 = 1e-8 (sin t / t, (1 - cos t)/t^2), and their closed forms cancel
# for small |w| (1 - cos t, t - sin t, 1 - (t/2) cot(t/2)).  The edge window steps its knots by these increments (0 =
# identical knots), so d_j and lambda_j d_j fall on both sides of 1e-7, 1e-4 and 1e-3; stores every other knot as -q;
# and puts stamps where lambda_j |d_j| equals each target, at u = 0 and at the last double below a segment end.
INCREMENTS = [1e-9, 0.0, 5e-8, 1.5e-7, 8e-5, 1.2e-4, 5e-4, 1.5e-3, 1e-2, 0.3, 1.05e-4, 2e-3]
SWITCH_TARGETS = [1.05e-4, 1.2e-4, 9.5e-5, 1.05e-3, 9.5e-4, 1.05e-7, 9.5e-8]


def edge_knots(seed):
    """Knots 0.125 s apart (a binary fraction: every segment has the same dt, so the time differences see a spline that
    is C^(k-2) across knots) whose rotations step by INCREMENTS about random axes while the positions drift slowly."""
    rng = np.random.default_rng(seed)
    q = synthetic.rot_to_quat(synthetic.so3_exp(rng.normal(0, 1.0, (1, 3))))[0]
    quats = [q]
    for inc in INCREMENTS:
        axis = rng.normal(size=3)
        if inc:
            q = np.array(quat_mul(list(q), list(np.append(np.sin(inc / 2) * axis / np.linalg.norm(axis), np.cos(inc / 2)))))
            q /= np.linalg.norm(q)
        quats.append(q)
    kt = np.arange(len(quats)) * 0.125
    knots = np.zeros((len(quats), 8))
    knots[:, :4] = quats
    knots[1::2, :4] *= -1
    knots[:, 4:7] = 0.2 * np.stack([np.sin(0.45 * kt), np.sin(0.3 * kt + 0.7), 0.5 * np.sin(0.6 * kt + 0.2)], -1)
    knots[:, 7] = kt
    return knots


def edge_stamps(knots, k):
    """For each target, the stamp where some lambda_j(u) |d_j| equals it with the largest lambda_j; then u = 0 and the
    last double below the end of every other valid segment."""
    Mc, left, K = synthetic.blending_matrix(k), (k - 1) // 2, knots.shape[0]
    R = synthetic.quat_to_rot(knots[:, :4])
    inc = [np.linalg.norm(synthetic.so3_log((R[i].T @ R[i + 1])[None])[0]) for i in range(K - 1)]
    lam = lambda j, u: float(Mc[j] @ (u ** np.arange(k)))
    segs = range(left, K - k + left + 1)
    out = []
    for target in SWITCH_TARGETS:
        best = (0.0, None)
        for s in segs:
            for j in range(1, k):
                d = inc[s - left + j - 1]
                if d == 0 or not lam(j, 0.0) <= target / d < lam(j, 1.0):
                    continue
                lo, hi = 0.0, 1.0
                for _ in range(80):
                    lo, hi = (0.5 * (lo + hi), hi) if lam(j, 0.5 * (lo + hi)) * d < target else (lo, 0.5 * (lo + hi))
                best = max(best, (lam(j, lo), knots[s, 7] + lo * (knots[s + 1, 7] - knots[s, 7])), key=lambda b: b[0])
        if best[1] is not None:
            out.append(best[1])
    for s in list(segs)[::2]:
        out += [knots[s, 7], float(np.nextafter(knots[s + 1, 7], -np.inf))]
    return out


def interpolate_answer(st, t):
    """hb200_interpolate's outputs at t: pose [q | p], body velocity [omega | R^T p'] and acceleration [alpha | R^T p'']
    from time differences of the value formula."""
    q, p0 = pose_q(st["knots"], st["k"], t)
    R0 = quat_to_rot(q)
    Rp, pp = pose(st["knots"], st["k"], t + H_T, pin=t)
    Rm, pm = pose(st["knots"], st["k"], t - H_T, pin=t)
    w = vee(R0.T * (Rp - Rm) / (2 * H_T))
    al = vee(R0.T * (Rp - 2 * R0 + Rm) / H_T ** 2 - hat(w) * hat(w))
    v = R0.T * ((pp - pm) / (2 * H_T))
    a = R0.T * ((pp - 2 * p0 + pm) / H_T ** 2)
    return dict(stamp=float(t), pose=fl(q) + fl(p0), vel=fl(w) + fl(v), acc=fl(al) + fl(a))


def make_edge_case(name, order, seed, n_pix=5, n_bearing=2, n_pose=2, n_imu=2):
    """Pixel, bearing, pose and inertial factors (stamps taken from edge_stamps, switch stamps first) and interpolation
    answers at every edge stamp.  Each visual factor observes its own landmark, placed in front of its camera;
    measurements are the model's prediction plus noise."""
    rng = np.random.default_rng(seed)
    k = order
    knots = edge_knots(seed)
    base_win = synthetic.make_window(order=k, num_knots=knots.shape[0], num_landmarks=0, num_imu=0, seed=seed, generic_calibration=True)
    cams = base_win.cameras
    stamps = edge_stamps(knots, k)
    v_stamp, b_stamp = np.array(stamps[:n_pix]), np.array(stamps[-n_bearing:])
    m_stamp, i_stamp = np.array(stamps[:n_pose]), np.array([stamps[0], stamps[-2]][:n_imu])
    vis_stamp = np.concatenate([v_stamp, b_stamp])
    vis_cam = (np.arange(vis_stamp.size) % cams.shape[0]).astype(np.int32)
    R, p, *_ = synthetic.spline_eval(knots, k, vis_stamp)
    c = cams[vis_cam]
    px = np.stack([rng.uniform(150, 600, vis_stamp.size), rng.uniform(120, 360, vis_stamp.size)], -1)
    p_s = np.stack([(px[:, 0] - c[:, 7]) / c[:, 9], (px[:, 1] - c[:, 8]) / c[:, 10], np.ones(vis_stamp.size)], -1)
    p_s *= rng.uniform(2.0, 8.0, (vis_stamp.size, 1))
    p_b = (synthetic.quat_to_rot(c[:, :4]) @ p_s[..., None])[..., 0] + c[:, 4:7]
    landmarks = (R @ p_b[..., None])[..., 0] + p
    lm = np.arange(vis_stamp.size, dtype=np.int32)
    v_pixel = synthetic.pixel_model(knots, k, cams, landmarks, v_stamp, vis_cam[:n_pix], lm[:n_pix])[0] + rng.normal(0, 2.0, (n_pix, 2))
    b = p_s[n_pix:] / np.linalg.norm(p_s[n_pix:], axis=1, keepdims=True) + rng.normal(0, 3e-2, (n_bearing, 3))
    sensors = np.zeros((2, 7))
    sensors[:, :4] = synthetic.rot_to_quat(synthetic.so3_exp(rng.normal(0, 0.3, (2, 3))))
    sensors[:, 4:] = rng.normal(0, 0.1, (2, 3))
    m_sensor = (np.arange(n_pose) % 2).astype(np.int32)
    Rm, pm, *_ = synthetic.spline_eval(knots, k, m_stamp)
    ang = np.array([1.05e-4, 1.05e-3])[np.arange(n_pose) % 2]                # pose residual angles about 1e-4 and 1e-3
    axis = rng.normal(size=(n_pose, 3))
    R_ws = synthetic.so3_exp(ang[:, None] * axis / np.linalg.norm(axis, axis=1, keepdims=True)) @ Rm @ synthetic.quat_to_rot(sensors[m_sensor, :4])
    p_ws = pm + (Rm @ sensors[m_sensor, 4:, None])[..., 0] + rng.normal(0, 5e-3, (n_pose, 3))
    i_meas = synthetic.inertial_model(knots, k, base_win.imu, base_win.gyro_bias, base_win.accel_bias, base_win.bias_order, base_win.gravity, i_stamp)
    i_meas += np.concatenate([rng.normal(0, 2e-3, (n_imu, 3)), rng.normal(0, 3e-2, (n_imu, 3))], axis=1)
    w = dataclasses.replace(base_win, knots=knots, landmarks=landmarks, v_stamp=v_stamp, v_cam=vis_cam[:n_pix], v_lm=lm[:n_pix], v_pixel=v_pixel,
                            i_stamp=i_stamp, i_meas=i_meas, knot_const=np.zeros(knots.shape[0], dtype=np.uint8),
                            b_stamp=b_stamp, b_cam=vis_cam[n_pix:], b_lm=lm[n_pix:], b_bearing=b, pose_sensors=sensors, m_stamp=m_stamp,
                            m_sensor=m_sensor, m_pose=np.concatenate([synthetic.rot_to_quat(R_ws), p_ws], axis=1))
    st = to_mp_state(w)
    case = dict(name=name, window=window_json(w), digits=mp.mp.dps,
                pixel=[pixel_answer(st, w, i) for i in range(n_pix)], bearing=[bearing_answer(st, w, i) for i in range(n_bearing)],
                pose=[pose_answer(st, w, i) for i in range(n_pose)], inertial=[inertial_answer(st, w, i) for i in range(n_imu)],
                interpolate=[interpolate_answer(st, mp.mpf(float(t))) for t in stamps])
    write_case(name, case)
    write_calibration(name, st, case)


# ---- stereo ingest (hb200_ingest_stereo, hb200_append_stereo_tracks) ---------------------------------------------
INGEST_DEPTHS = [0.5, 2.0, 10.0, 100.0, 1000.0]


def distort(cam, x, y):
    k1, k2, p1, p2 = cam[11:15]
    r2 = x * x + y * y
    rad = 1 + k1 * r2 + k2 * r2 * r2
    return [x * rad + 2 * p1 * x * y + p2 * (r2 + 2 * x * x), y * rad + p1 * (r2 + 2 * y * y) + 2 * p2 * x * y]


def pixel_bearing(cam, px):
    """Unit bearing of a pixel: the distortion inverted by mp.findroot, started at the distorted point.  Asserts that
    the forward model is monotone (positive Jacobian determinant) on the ray from the centre to the root."""
    cx, cy, fx, fy = cam[7:11]
    d = [(px[0] - cx) / fx, (px[1] - cy) / fy]
    x, y = mp.findroot(lambda x, y: [a - b for a, b in zip(distort(cam, x, y), d)], d)
    for s in mp.linspace(0, 1, 41)[1:]:
        J = mp.jacobian(lambda a, b: distort(cam, a, b), [s * x, s * y])
        assert J[0, 0] * J[1, 1] - J[0, 1] * J[1, 0] > 0, (px, s)
    assert max(abs(a - b) for a, b in zip(distort(cam, x, y), d)) < mp.mpf(10) ** -70
    n = mp.sqrt(x * x + y * y + 1)
    return mp.matrix([x / n, y / n, 1 / n])


def stereo_answer(st, stamp, c0, c1, px0, px1):
    """Bearings of both views, the midpoint p_0 of the common perpendicular in camera 0 (None for parallel rays) and
    the world landmark R (R_b0 p_0 + t_b0) + p at the stamp, from the stored double inputs."""
    ca, cb = st["cams"][c0], st["cams"][c1]
    b0, b1 = pixel_bearing(ca, px0), pixel_bearing(cb, px1)
    Ra, Rb = quat_to_rot(ca[:4]), quat_to_rot(cb[:4])
    t = Ra.T * (mp.matrix(cb[4:7]) - mp.matrix(ca[4:7]))
    d1 = Ra.T * Rb * b1
    dot = lambda u, v: sum(u[i] * v[i] for i in range(3))
    det = dot(b0, b0) * dot(d1, d1) - dot(b0, d1) ** 2
    out = dict(stamp=float(stamp), cam0=c0, cam1=c1, px0=fl(px0), px1=fl(px1), b0=fl(b0), b1=fl(b1), p0=None, lm=None)
    if det != 0:
        s = (dot(b0, t) * dot(d1, d1) - dot(b0, d1) * dot(d1, t)) / det
        u = (dot(b0, d1) * dot(b0, t) - dot(b0, b0) * dot(d1, t)) / det
        p0 = (s * b0 + t + u * d1) / 2
        R, p = pose(st["knots"], st["k"], stamp)
        out.update(p0=fl(p0), lm=fl(R * (Ra * p0 + mp.matrix(ca[4:7])) + p))
    return out


def make_ingest_case(name, edges, seed):
    """Stereo tracks on the window of the edges fixture, at its edge stamps: the EuRoC pair (cameras 0, 1), a generic
    pair (2, 3: rotated rig, other intrinsics, barrel-free distortion with large tangential terms, 0.2 m baseline) and a
    parallel pair (4, 5: identity rotations, no distortion, principal points).  Camera-0 pixels at the image centre,
    the four corners and four points beyond the image, each with two of INGEST_DEPTHS along its ray (every depth three
    or four times per pair); camera-1 pixels from the forward model in doubles."""
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), f"{edges}.json")) as fh:
        w = json.load(fh)["window"]
    k, knots = w["order"], np.array(w["knots"])
    rng = np.random.default_rng(seed)
    gen0 = synthetic.EUROC_CAM0.copy()
    gen0[:4] = synthetic.rot_to_quat(synthetic.so3_exp(rng.normal(0, 0.2, (1, 3))) @ synthetic.quat_to_rot(gen0[None, :4]))[0]
    gen0[7:11] = [330.0, 260.0, 420.0, 425.0]
    gen0[11:15] = [0.05, -0.01, 1.5e-3, -1.2e-3]
    gen1 = gen0.copy()
    gen1[:4] = synthetic.rot_to_quat(synthetic.so3_exp(rng.normal(0, 0.05, (1, 3))) @ synthetic.quat_to_rot(gen0[None, :4]))[0]
    gen1[4:7] += synthetic.quat_to_rot(gen0[None, :4])[0] @ np.array([0.2, 0.01, -0.005])
    gen1[7:11] = [345.0, 250.0, 430.0, 428.0]
    gen1[11:15] = [0.04, -0.008, -1.1e-3, 9e-4]
    par0 = np.concatenate([[0, 0, 0, 1, 0, 0, 0], gen0[7:11], [0, 0, 0, 0]])
    par1 = par0.copy()
    par1[4] = 0.11
    cams = np.stack([synthetic.EUROC_CAM0, synthetic.EUROC_CAM1, gen0, gen1, par0, par1])
    stamps = edge_stamps(knots, k)
    pixels = [(376.0, 240.0), (0.0, 0.0), (751.0, 0.0), (0.0, 479.0), (751.0, 479.0), (-150.0, -100.0), (950.0, -80.0), (-120.0, 620.0),
              (900.0, 640.0)]
    mpm = lambda a: [[mp.mpf(float(x)) for x in row] for row in a]
    st = dict(k=k, knots=mpm(knots), cams=mpm(cams))
    inputs = []
    for c0, c1 in ((0, 1), (2, 3)):
        for i, px0 in enumerate(pixels):
            b0 = np.array(fl(pixel_bearing(st["cams"][c0], [mp.mpf(v) for v in px0])))
            for depth in (INGEST_DEPTHS[(i + c0) % 5], INGEST_DEPTHS[(i + c0 + 2) % 5]):
                ca, cb = cams[c0], cams[c1]
                p_s1 = synthetic.quat_to_rot(cb[None, :4])[0].T @ (synthetic.quat_to_rot(ca[None, :4])[0] @ (depth * b0) + ca[4:7] - cb[4:7])
                assert p_s1[2] > 0
                inputs.append((stamps[len(inputs) % len(stamps)], c0, c1, px0, synthetic.project(cams, np.array([c1]), p_s1[None])[0]))
    inputs.append((stamps[0], 4, 5, par0[7:9], par1[7:9]))
    inputs.sort(key=lambda a: a[0])                     # arrival order, as hb200_append_stereo_tracks requires
    case = dict(name=name, edges=edges, digits=mp.mp.dps, cameras=cams.tolist(),
                tracks=[stereo_answer(st, mp.mpf(float(t)), c0, c1, [mp.mpf(float(v)) for v in p0], [mp.mpf(float(v)) for v in p1])
                        for t, c0, c1, p0, p1 in inputs])
    write_case(os.path.join("ingest", name), case)


if __name__ == "__main__":
    if "--ingest-only" in sys.argv:
        make_ingest_case("k4_stereo_ingest", "k4_spline_edges", seed=synthetic.SEED_BASE + 924)
        make_ingest_case("k6_stereo_ingest", "k6_spline_edges", seed=synthetic.SEED_BASE + 926)
        sys.exit(0)
    if "--widened-only" in sys.argv:
        make_widened_case("k4_bearing_pose", order=4, num_knots=10, num_landmarks=12, num_imu=0, seed=synthetic.SEED_BASE + 905)
        make_widened_case("k6_bearing_pose", order=6, num_knots=12, num_landmarks=12, num_imu=0, seed=synthetic.SEED_BASE + 906, n_bearing=2, n_pose=2)
        sys.exit(0)
    make_case("k4_euroc", order=4, num_knots=10, num_landmarks=12, num_imu=20, seed=synthetic.SEED_BASE + 901)
    make_case("k6_euroc", order=6, num_knots=12, num_landmarks=12, num_imu=20, seed=synthetic.SEED_BASE + 902)
    make_case("k4_generic_calibration", order=4, num_knots=10, num_landmarks=12, num_imu=20, generic_calibration=True, seed=synthetic.SEED_BASE + 903)
    make_case("k6_generic_calibration", order=6, num_knots=12, num_landmarks=12, num_imu=20, generic_calibration=True, seed=synthetic.SEED_BASE + 904, n_pix=2, n_imu=2)
    make_widened_case("k4_bearing_pose", order=4, num_knots=10, num_landmarks=12, num_imu=0, seed=synthetic.SEED_BASE + 905)
    make_widened_case("k6_bearing_pose", order=6, num_knots=12, num_landmarks=12, num_imu=0, seed=synthetic.SEED_BASE + 906, n_bearing=2, n_pose=2)
    make_edge_case("k4_spline_edges", order=4, seed=synthetic.SEED_BASE + 914)
    make_edge_case("k6_spline_edges", order=6, seed=synthetic.SEED_BASE + 916)
    make_ingest_case("k4_stereo_ingest", "k4_spline_edges", seed=synthetic.SEED_BASE + 924)
    make_ingest_case("k6_stereo_ingest", "k6_spline_edges", seed=synthetic.SEED_BASE + 926)
