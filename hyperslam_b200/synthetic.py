"""Seeded synthetic sliding windows for the BASELINE.json configurations (SURVEY.md section 8d).

Produces the flat "window" the C-ABI consumes: control points, calibration, landmarks and the two
factor lists (stereo pixel reprojection + raw 6-DoF inertial), i.e. the data products of the
reference's window manager (reference internal/hyper/optimizers/abstract.cpp:74-147,186-292)
without its pointer graph.  Calibration constants are the reference's EuRoC setup
(reference resources/datasets/euroc/setups/stereo_inertial/settings.yaml:34-45,61-72,83-109).

Measurements are generated with a vectorised numpy forward model (values only), independent of
both the CUDA path and the test oracle.
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np

SEED_BASE = 0x48595045  # "HYPE"

# reference settings.yaml:34-45 (cam0) and :61-72 (cam1): [qx qy qz qw px py pz | cx cy fx fy | k1 k2 p1 p2]
EUROC_CAM0 = np.array([-0.007707179755532, 0.010499323370595, 0.701752800292141, 0.712301460668946,
                       -0.0216401454975, -0.064676986768, 0.00981073058949,
                       367.215, 248.375, 458.654, 457.296,
                       -0.28340811, 0.07395907, 1.76187114e-05, 0.00019359])
EUROC_CAM1 = np.array([-0.002550236745188, 0.015323927487975, 0.702486685782579, 0.711527321918909,
                       -0.0198435579556, 0.0453689425024, 0.00786212447038,
                       379.999, 255.238, 457.587, 456.134,
                       -0.28368365, 0.07451284, -3.55590700e-05, -0.00010473])
IMAGE_SIZE = (752, 480)  # reference tests/include/tests/sensors/camera.hpp:24
GYRO_NOISE_DENSITY = 1.6968e-04  # settings.yaml:96-97
ACCEL_NOISE_DENSITY = 2.0e-3     # settings.yaml:108-109
IMU_RATE = 200.0


@dataclasses.dataclass
class Window:
    order: int
    knots: np.ndarray         # (K, 8)  [qx qy qz qw px py pz | stamp]
    bias_order: int
    gyro_bias: np.ndarray     # (Kb, 4) [bx by bz | stamp]
    accel_bias: np.ndarray    # (Kb, 4)
    gravity: np.ndarray       # (3,)
    cameras: np.ndarray       # (C, 15) [T_bs(7) | cx cy fx fy | k1 k2 p1 p2]
    imu: np.ndarray           # (37,)   [T_bs(7) | i_g(6) | i_a(6) | S_g(9, col-major) | X_a(9, col-major)]
    landmarks: np.ndarray     # (L, 3)
    v_stamp: np.ndarray       # (Nv,)
    v_cam: np.ndarray         # (Nv,) int32
    v_lm: np.ndarray          # (Nv,) int32
    v_pixel: np.ndarray       # (Nv, 2)
    i_stamp: np.ndarray       # (Ni,)
    i_meas: np.ndarray        # (Ni, 6) [gyro | accel]
    knot_const: np.ndarray    # (K,) uint8
    gravity_const: int = 0
    bias_const: int = 0
    huber_pixel: float = 0.5          # reference optimizer.cpp:226
    imu_loss_scale: float = 1.6e-5    # reference optimizer.cpp:267
    truth: dict | None = None
    # bearing factors (VisualBearingObservation, reference optimizer.cpp:189-210): same blocks as a pixel factor
    b_stamp: np.ndarray = dataclasses.field(default_factory=lambda: np.zeros(0))
    b_cam: np.ndarray = dataclasses.field(default_factory=lambda: np.zeros(0, dtype=np.int32))
    b_lm: np.ndarray = dataclasses.field(default_factory=lambda: np.zeros(0, dtype=np.int32))
    b_bearing: np.ndarray = dataclasses.field(default_factory=lambda: np.zeros((0, 3)))
    huber_bearing: float = 1.6e-3     # reference optimizer.cpp:204
    # manifold (pose) factors (ManifoldObservation<SE3>, reference optimizer.cpp:234-251)
    pose_sensors: np.ndarray = dataclasses.field(default_factory=lambda: np.zeros((0, 7)))   # (P, 7) T_bs
    m_stamp: np.ndarray = dataclasses.field(default_factory=lambda: np.zeros(0))
    m_sensor: np.ndarray = dataclasses.field(default_factory=lambda: np.zeros(0, dtype=np.int32))
    m_pose: np.ndarray = dataclasses.field(default_factory=lambda: np.zeros((0, 7)))         # (Nm, 7) measured T_ws
    # family weight matrices (CostConfiguration::weights, reference exteroceptive.cpp:162-178): {kind: (d, d) array} with
    # kind runtime.PIXEL (2x2) / BEARING (1x1) / INERTIAL (6x6) / MANIFOLD (6x6); None (the reference default) sets none
    weights: dict | None = None

    @property
    def num_factors(self) -> int:
        return int(self.v_stamp.size + self.i_stamp.size + self.b_stamp.size + self.m_stamp.size)

    def reduced_size(self) -> int:
        return 6 * self.knots.shape[0] + 3 * self.gyro_bias.shape[0] + 3 * self.accel_bias.shape[0] + 2

    def shard(self, rank: int, world: int) -> "Window":
        """Factor shard of this window for one rank: visual factors partitioned by landmark owner
        (landmark l -> rank l % world... block-wise), inertial factors block-distributed by index.
        State (knots, calibration, landmarks, biases, gravity) is replicated (SURVEY.md section 8e)."""
        L = self.landmarks.shape[0]
        owner_lo = (L * rank) // world
        owner_hi = (L * (rank + 1)) // world
        vm = (self.v_lm >= owner_lo) & (self.v_lm < owner_hi)
        Ni = self.i_stamp.size
        i_lo, i_hi = (Ni * rank) // world, (Ni * (rank + 1)) // world
        bm = (self.b_lm >= owner_lo) & (self.b_lm < owner_hi)
        Nm = self.m_stamp.size
        m_lo, m_hi = (Nm * rank) // world, (Nm * (rank + 1)) // world
        return dataclasses.replace(
            self, b_stamp=np.ascontiguousarray(self.b_stamp[bm]), b_cam=np.ascontiguousarray(self.b_cam[bm]),
            b_lm=np.ascontiguousarray(self.b_lm[bm]), b_bearing=np.ascontiguousarray(self.b_bearing[bm]),
            m_stamp=np.ascontiguousarray(self.m_stamp[m_lo:m_hi]), m_sensor=np.ascontiguousarray(self.m_sensor[m_lo:m_hi]),
            m_pose=np.ascontiguousarray(self.m_pose[m_lo:m_hi]), v_stamp=np.ascontiguousarray(self.v_stamp[vm]), v_cam=np.ascontiguousarray(self.v_cam[vm]),
            v_lm=np.ascontiguousarray(self.v_lm[vm]), v_pixel=np.ascontiguousarray(self.v_pixel[vm]),
            i_stamp=np.ascontiguousarray(self.i_stamp[i_lo:i_hi]), i_meas=np.ascontiguousarray(self.i_meas[i_lo:i_hi]))


# ------------------------------------------------------------------------------------------------
# numpy forward model (values only)
# ------------------------------------------------------------------------------------------------
def blending_matrix(k: int) -> np.ndarray:
    """Cumulative blending matrix Mc[j, n] of the uniform B-spline of order k (SURVEY.md A.3)."""
    M = np.zeros((k, k))
    for s in range(k):
        for n in range(k):
            acc = 0.0
            for l in range(s, k):
                acc += (-1) ** (l - s) * math.comb(k, l - s) * float(k - 1 - l) ** (k - 1 - n)
            M[s, n] = math.comb(k - 1, n) / math.factorial(k - 1) * acc
    return np.cumsum(M[::-1], axis=0)[::-1].copy()


def _hat(v):
    z = np.zeros(v.shape[:-1])
    return np.stack([np.stack([z, -v[..., 2], v[..., 1]], -1),
                     np.stack([v[..., 2], z, -v[..., 0]], -1),
                     np.stack([-v[..., 1], v[..., 0], z], -1)], -2)


def so3_exp(w):
    t = np.linalg.norm(w, axis=-1)[..., None, None]
    W = _hat(w)
    small = t < 1e-8
    ts = np.where(small, 1.0, t)
    a = np.where(small, 1.0 - t * t / 6.0, np.sin(ts) / ts)
    b = np.where(small, 0.5 - t * t / 24.0, (1.0 - np.cos(ts)) / (ts * ts))
    return np.eye(3) + a * W + b * (W @ W)


def quat_to_rot(q):
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
                     np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
                     np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)], -2)


def rot_to_quat(R):
    """Rotation matrices -> [x y z w] (w >= 0), robust branch selection."""
    R = np.asarray(R)
    q = np.zeros(R.shape[:-2] + (4,))
    m00, m11, m22 = R[..., 0, 0], R[..., 1, 1], R[..., 2, 2]
    tr = m00 + m11 + m22
    c0 = tr > 0
    c1 = (~c0) & (m00 >= m11) & (m00 >= m22)
    c2 = (~c0) & (~c1) & (m11 >= m22)
    c3 = (~c0) & (~c1) & (~c2)
    with np.errstate(invalid="ignore"):
        s = np.sqrt(np.maximum(tr + 1.0, 1e-300)) * 2
        q0 = np.stack([(R[..., 2, 1] - R[..., 1, 2]) / s, (R[..., 0, 2] - R[..., 2, 0]) / s, (R[..., 1, 0] - R[..., 0, 1]) / s, 0.25 * s], -1)
        s = np.sqrt(np.maximum(1.0 + m00 - m11 - m22, 1e-300)) * 2
        q1 = np.stack([0.25 * s, (R[..., 0, 1] + R[..., 1, 0]) / s, (R[..., 0, 2] + R[..., 2, 0]) / s, (R[..., 2, 1] - R[..., 1, 2]) / s], -1)
        s = np.sqrt(np.maximum(1.0 + m11 - m00 - m22, 1e-300)) * 2
        q2 = np.stack([(R[..., 0, 1] + R[..., 1, 0]) / s, 0.25 * s, (R[..., 1, 2] + R[..., 2, 1]) / s, (R[..., 0, 2] - R[..., 2, 0]) / s], -1)
        s = np.sqrt(np.maximum(1.0 + m22 - m00 - m11, 1e-300)) * 2
        q3 = np.stack([(R[..., 0, 2] + R[..., 2, 0]) / s, (R[..., 1, 2] + R[..., 2, 1]) / s, 0.25 * s, (R[..., 1, 0] - R[..., 0, 1]) / s], -1)
    q = np.where(c0[..., None], q0, q)
    q = np.where(c1[..., None], q1, q)
    q = np.where(c2[..., None], q2, q)
    q = np.where(c3[..., None], q3, q)
    q = q * np.where(q[..., 3:4] < 0, -1.0, 1.0)
    return q / np.linalg.norm(q, axis=-1, keepdims=True)


def so3_log(R):
    q = rot_to_quat(R)
    v = q[..., :3]
    n = np.linalg.norm(v, axis=-1, keepdims=True)
    w = q[..., 3:4]
    small = n < 1e-9
    ns = np.where(small, 1.0, n)
    s = np.where(small, 2.0 / w, 2.0 * np.arctan2(ns, w) / ns)
    return s * v


def segment(knot_stamps: np.ndarray, order: int, t: np.ndarray):
    """Knot base index and normalised time of stamps t (SURVEY.md A.3)."""
    j = np.searchsorted(knot_stamps, t, side="right") - 1
    left = (order - 1) // 2
    base = j - left
    dt = knot_stamps[j + 1] - knot_stamps[j]
    u = (t - knot_stamps[j]) / dt
    return base.astype(np.int64), u, 1.0 / dt


def spline_eval(knots: np.ndarray, order: int, t: np.ndarray):
    """Vectorised value/velocity/acceleration of the split SO(3) x R^3 cumulative B-spline.
    Returns R (N,3,3), p (N,3), omega_b (N,3), alpha_b (N,3), pdd_w (N,3), pd_w (N,3)."""
    k = order
    Mc = blending_matrix(k)
    base, u, inv_dt = segment(knots[:, 7], k, t)
    N = t.size
    pw = np.stack([u ** n for n in range(k)], -1)                                   # (N,k)
    dpw = np.stack([n * u ** max(n - 1, 0) if n >= 1 else np.zeros(N) for n in range(k)], -1)
    ddpw = np.stack([n * (n - 1) * u ** max(n - 2, 0) if n >= 2 else np.zeros(N) for n in range(k)], -1)
    lam = pw @ Mc.T
    lamd = (dpw @ Mc.T) * inv_dt[:, None]
    lamdd = (ddpw @ Mc.T) * (inv_dt ** 2)[:, None]
    Rk = quat_to_rot(knots[:, :4])
    dk = so3_log(np.swapaxes(Rk[:-1], -1, -2) @ Rk[1:])                              # d between knot i and i+1
    R = Rk[base].copy()
    p = knots[base, 4:7].copy()
    pd = np.zeros((N, 3)); pdd = np.zeros((N, 3))
    w = np.zeros((N, 3)); wd = np.zeros((N, 3))
    for j in range(1, k):
        d = dk[base + j - 1]
        A = so3_exp(lam[:, j, None] * d)
        R = R @ A
        At = np.swapaxes(A, -1, -2)
        w_new = (At @ w[..., None])[..., 0] + lamd[:, j, None] * d
        wd = (At @ wd[..., None])[..., 0] + lamd[:, j, None] * np.cross(w_new, d) + lamdd[:, j, None] * d
        w = w_new
        dp = knots[base + j, 4:7] - knots[base + j - 1, 4:7]
        p += lam[:, j, None] * dp
        pd += lamd[:, j, None] * dp
        pdd += lamdd[:, j, None] * dp
    return R, p, w, wd, pdd, pd


def bias_eval(bias_knots: np.ndarray, order: int, t: np.ndarray):
    Mc = blending_matrix(order)
    base, u, _ = segment(bias_knots[:, 3], order, t)
    pw = np.stack([u ** n for n in range(order)], -1)
    lam = pw @ Mc.T
    lam = np.concatenate([lam, np.zeros((t.size, 1))], -1)
    lam[:, 0] = 1.0
    wgt = lam[:, :-1] - lam[:, 1:]
    b = np.zeros((t.size, 3))
    for m in range(order):
        b += wgt[:, m, None] * bias_knots[base + m, :3]
    return b


def project(cams: np.ndarray, cam_idx: np.ndarray, p_s: np.ndarray):
    c = cams[cam_idx]
    x = p_s[:, 0] / p_s[:, 2]; y = p_s[:, 1] / p_s[:, 2]
    k1, k2, p1, p2 = c[:, 11], c[:, 12], c[:, 13], c[:, 14]
    r2 = x * x + y * y
    rad = 1 + k1 * r2 + k2 * r2 * r2
    dx = x * rad + 2 * p1 * x * y + p2 * (r2 + 2 * x * x)
    dy = y * rad + p1 * (r2 + 2 * y * y) + 2 * p2 * x * y
    return np.stack([c[:, 9] * dx + c[:, 7], c[:, 10] * dy + c[:, 8]], -1)


def pixel_model(win_knots, order, cams, landmarks, stamp, cam_idx, lm_idx):
    R, p, *_ = spline_eval(win_knots, order, stamp)
    c = cams[cam_idx]
    R_bs = quat_to_rot(c[:, :4]); t_bs = c[:, 4:7]
    p_b = (np.swapaxes(R, -1, -2) @ (landmarks[lm_idx] - p)[..., None])[..., 0]
    p_s = (np.swapaxes(R_bs, -1, -2) @ (p_b - t_bs)[..., None])[..., 0]
    return project(cams, cam_idx, p_s), p_s


def imu_matrix(c):
    return np.array([[c[0], 0, 0], [c[3], c[1], 0], [c[4], c[5], c[2]]])


def inertial_model(win_knots, order, imu, gyro_bias, accel_bias, bias_order, gravity, stamp):
    """r = prediction (no measurement subtracted), reference inertial.cpp:62-79."""
    R, p, w, wd, pdd, _ = spline_eval(win_knots, order, stamp)
    Rt = np.swapaxes(R, -1, -2)
    R_sb = quat_to_rot(imu[None, :4])[0].T
    t_bs = imu[4:7]
    I_g, I_a = imu_matrix(imu[7:13]), imu_matrix(imu[13:19])
    S_g = imu[19:28].reshape(3, 3).T
    X_a = imu[28:37].reshape(3, 3).T
    a_i = (Rt @ (pdd - gravity)[..., None])[..., 0]
    F = _hat(w) @ _hat(w) + _hat(wd)
    a_m = a_i.copy()
    for r in range(3):
        a_m[:, r] += F[:, r, :] @ (X_a[:, r] + t_bs)
    b_g = bias_eval(gyro_bias, bias_order, stamp)
    b_a = bias_eval(accel_bias, bias_order, stamp)
    gyro = (w @ (I_g @ R_sb).T) + a_m @ S_g.T + b_g
    acc = a_m @ (I_a @ R_sb).T + b_a
    return np.concatenate([gyro, acc], -1)


# ------------------------------------------------------------------------------------------------
# generators
# ------------------------------------------------------------------------------------------------
def _trajectory(t: np.ndarray):
    """Smooth analytic motion: Lissajous translation (amplitude 2 m, <= ~1 m/s), smooth rotation."""
    p = np.stack([2.0 * np.sin(0.45 * t), 2.0 * np.sin(0.3 * t + 0.7), 0.5 * np.sin(0.6 * t + 0.2)], -1)
    rv = np.stack([0.25 * np.sin(0.7 * t), 0.2 * np.sin(0.5 * t + 1.0), 0.6 * np.sin(0.35 * t + 0.3) + 0.15 * t], -1)
    return so3_exp(rv), p


def make_window(order=4, num_knots=50, dt=0.1, num_landmarks=1000, frames_per_landmark=5, num_cameras=2, num_imu=2000,
                seed=SEED_BASE + 2, frame_dt=0.05, generic_calibration=False, perturb=True, bias_dt=10.0,
                pixel_sigma=0.5, noise=True, constant_knots=0) -> Window:
    rng = np.random.Generator(np.random.Philox(seed))
    k, K = order, num_knots
    left = (k - 1) // 2
    kt = np.arange(K) * dt
    t_lo, t_hi = kt[left], kt[K - 1 - (k - 1 - left)]
    Rk, pk = _trajectory(kt)
    knots = np.zeros((K, 8))
    knots[:, :4] = rot_to_quat(Rk)
    for i in range(1, K):  # keep consecutive quaternions in the same hemisphere
        if np.dot(knots[i, :4], knots[i - 1, :4]) < 0:
            knots[i, :4] *= -1
    knots[:, 4:7] = pk
    knots[:, 7] = kt

    # cameras
    cams = [EUROC_CAM0.copy(), EUROC_CAM1.copy()]
    for c in range(2, num_cameras):  # extra rig cameras: copies of the stereo pair with small offsets
        extra = cams[c % 2].copy()
        extra[4:7] += np.array([0.0, 0.0, 0.03 * (c // 2)]) + rng.uniform(-0.005, 0.005, 3)
        extra[7:11] *= 1.0 + rng.uniform(-0.01, 0.01, 4)
        cams.append(extra)
    cams = np.stack(cams[:num_cameras])
    imu = np.zeros(37)
    imu[3] = 1.0
    imu[7:10] = 1.0; imu[13:16] = 1.0
    if generic_calibration:
        rv = rng.uniform(-0.2, 0.2, 3)
        imu[:4] = rot_to_quat(so3_exp(rv[None])[0])
        imu[4:7] = rng.uniform(-0.1, 0.1, 3)
        imu[7:13] += rng.uniform(-0.02, 0.02, 6)
        imu[13:19] += rng.uniform(-0.02, 0.02, 6)
        imu[19:28] = rng.uniform(-1e-3, 1e-3, 9)
        imu[28:37] = rng.uniform(-0.01, 0.01, 9)

    # bias splines (order 4, knots every bias_dt, reference tests/.../inertial.cpp:48-49,66-89)
    kb = 4
    bl = (kb - 1) // 2
    Kb = int(math.ceil((t_hi - t_lo) / bias_dt)) + kb - 1
    bstamps = t_lo + (np.arange(Kb) - bl) * bias_dt
    gyro_bias = np.zeros((Kb, 4)); accel_bias = np.zeros((Kb, 4))
    gyro_bias[:, :3] = rng.uniform(-0.01, 0.01, (Kb, 3)); gyro_bias[:, 3] = bstamps
    accel_bias[:, :3] = rng.uniform(-0.05, 0.05, (Kb, 3)); accel_bias[:, 3] = bstamps
    g = np.array([0.02, -0.03, -1.0]); gravity = 9.81 * g / np.linalg.norm(g)

    # landmarks + stereo observations
    F = frames_per_landmark
    span = (F - 1) * frame_dt
    L = num_landmarks
    landmarks = np.zeros((L, 3))
    todo = np.arange(L)
    t_center = np.zeros(L)
    while todo.size:
        n = todo.size
        tc = rng.uniform(t_lo + span / 2 + 1e-3, t_hi - span / 2 - 1e-3, n)
        px = np.stack([rng.uniform(150, IMAGE_SIZE[0] - 150, n), rng.uniform(120, IMAGE_SIZE[1] - 120, n)], -1)
        depth = rng.uniform(2.0, 10.0, n)
        R, p, *_ = spline_eval(knots, k, tc)
        c0 = cams[0]
        ray = np.stack([(px[:, 0] - c0[7]) / c0[9], (px[:, 1] - c0[8]) / c0[10], np.ones(n)], -1) * depth[:, None]
        R_bs = quat_to_rot(c0[None, :4])[0]
        p_b = ray @ R_bs.T + c0[4:7]
        lm = (R @ p_b[..., None])[..., 0] + p
        ok = np.ones(n, dtype=bool)
        for f in range(F):
            tf = tc + (f - (F - 1) / 2) * frame_dt
            for c in range(num_cameras):
                pix, p_s = pixel_model(knots, k, cams, lm, tf, np.full(n, c), np.arange(n))
                ok &= (p_s[:, 2] > 0.5) & (pix[:, 0] > 0) & (pix[:, 0] < IMAGE_SIZE[0]) & (pix[:, 1] > 0) & (pix[:, 1] < IMAGE_SIZE[1])
        landmarks[todo[ok]] = lm[ok]
        t_center[todo[ok]] = tc[ok]
        todo = todo[~ok]
    lm_idx = np.repeat(np.arange(L), F * num_cameras)
    frame = np.tile(np.repeat(np.arange(F), num_cameras), L)
    cam_idx = np.tile(np.arange(num_cameras), L * F)
    v_stamp = t_center[lm_idx] + (frame - (F - 1) / 2) * frame_dt
    order_idx = np.argsort(v_stamp, kind="stable")  # sorted by stamp => sorted by knot base index
    v_stamp, lm_idx, cam_idx = v_stamp[order_idx], lm_idx[order_idx], cam_idx[order_idx]
    v_pixel, _ = pixel_model(knots, k, cams, landmarks, v_stamp, cam_idx, lm_idx)
    if noise:
        v_pixel = v_pixel + rng.normal(0.0, pixel_sigma, v_pixel.shape)

    # inertial factors, uniformly spaced over the valid span
    i_stamp = t_lo + (np.arange(num_imu) + 0.5) * (t_hi - t_lo) / max(num_imu, 1)
    i_meas = inertial_model(knots, k, imu, gyro_bias, accel_bias, kb, gravity, i_stamp) if num_imu else np.zeros((0, 6))
    if noise and num_imu:
        i_meas[:, :3] += rng.normal(0.0, GYRO_NOISE_DENSITY * math.sqrt(IMU_RATE), (num_imu, 3))
        i_meas[:, 3:] += rng.normal(0.0, ACCEL_NOISE_DENSITY * math.sqrt(IMU_RATE), (num_imu, 3))

    truth = dict(knots=knots.copy(), landmarks=landmarks.copy(), gyro_bias=gyro_bias.copy(), accel_bias=accel_bias.copy(),
                 gravity=gravity.copy())
    if perturb:
        dq = so3_exp(rng.normal(0, 0.004, (K, 3)))
        knots[:, :4] = rot_to_quat(dq @ quat_to_rot(knots[:, :4]))
        for i in range(1, K):
            if np.dot(knots[i, :4], knots[i - 1, :4]) < 0:
                knots[i, :4] *= -1
        knots[:, 4:7] += rng.normal(0, 0.01, (K, 3))
        landmarks = landmarks + rng.normal(0, 0.03, landmarks.shape)
        gyro_bias[:, :3] += rng.normal(0, 1e-3, (Kb, 3))
        accel_bias[:, :3] += rng.normal(0, 5e-3, (Kb, 3))
    knot_const = np.zeros(K, dtype=np.uint8)
    knot_const[:constant_knots] = 1
    return Window(order=k, knots=np.ascontiguousarray(knots), bias_order=kb, gyro_bias=gyro_bias, accel_bias=accel_bias,
                  gravity=gravity, cameras=np.ascontiguousarray(cams), imu=imu, landmarks=np.ascontiguousarray(landmarks),
                  v_stamp=np.ascontiguousarray(v_stamp), v_cam=cam_idx.astype(np.int32), v_lm=lm_idx.astype(np.int32),
                  v_pixel=np.ascontiguousarray(v_pixel), i_stamp=np.ascontiguousarray(i_stamp), i_meas=np.ascontiguousarray(i_meas),
                  knot_const=knot_const, truth=truth)


def add_bearing_and_pose_factors(win: Window, num_bearing=0, num_pose=0, seed=SEED_BASE + 77, convert=True,
                                 bearing_sigma=1e-3, pose_sigma=(2e-3, 5e-3), num_pose_sensors=2) -> Window:
    """Widen a window with the two other factor families the reference optimizer accepts:
    bearing factors (a random subset of the pixel observations re-expressed as unit directions in the sensor
    frame, removed from the pixel list when `convert`) and pose factors (noisy T_ws = T_wb (+) T_bs samples
    of the ground-truth trajectory on `num_pose_sensors` pose sensors)."""
    rng = np.random.Generator(np.random.Philox(seed))
    truth = win.truth
    out = {}
    if num_bearing:
        Nv = win.v_stamp.size
        sel = np.sort(rng.choice(Nv, size=min(num_bearing, Nv), replace=False))
        _, p_s = pixel_model(truth["knots"], win.order, win.cameras, truth["landmarks"], win.v_stamp[sel], win.v_cam[sel], win.v_lm[sel])
        b = p_s / np.linalg.norm(p_s, axis=1, keepdims=True) + rng.normal(0.0, bearing_sigma, p_s.shape)
        b *= rng.uniform(0.5, 2.0, (sel.size, 1))     # the angular metric is scale-free in the measurement
        out.update(b_stamp=np.ascontiguousarray(win.v_stamp[sel]), b_cam=np.ascontiguousarray(win.v_cam[sel]),
                   b_lm=np.ascontiguousarray(win.v_lm[sel]), b_bearing=np.ascontiguousarray(b))
        if convert:
            keep = np.ones(Nv, dtype=bool); keep[sel] = False
            out.update(v_stamp=np.ascontiguousarray(win.v_stamp[keep]), v_cam=np.ascontiguousarray(win.v_cam[keep]),
                       v_lm=np.ascontiguousarray(win.v_lm[keep]), v_pixel=np.ascontiguousarray(win.v_pixel[keep]))
    if num_pose:
        k, kt = win.order, win.knots[:, 7]
        left = (k - 1) // 2
        t_lo, t_hi = kt[left], kt[len(kt) - 1 - (k - 1 - left)]
        sensors = np.zeros((num_pose_sensors, 7))
        sensors[:, :4] = rot_to_quat(so3_exp(rng.normal(0, 0.3, (num_pose_sensors, 3))))
        sensors[:, 4:] = rng.normal(0, 0.1, (num_pose_sensors, 3))
        stamp = t_lo + (np.arange(num_pose) + 0.5) * (t_hi - t_lo) / num_pose
        sidx = rng.integers(0, num_pose_sensors, num_pose).astype(np.int32)
        R, p, *_ = spline_eval(truth["knots"], k, stamp)
        R_bs = quat_to_rot(sensors[sidx, :4]); t_bs = sensors[sidx, 4:]
        R_ws = so3_exp(rng.normal(0, pose_sigma[0], (num_pose, 3))) @ R @ R_bs
        p_ws = p + (R @ t_bs[..., None])[..., 0] + rng.normal(0, pose_sigma[1], (num_pose, 3))
        pose = np.concatenate([rot_to_quat(R_ws), p_ws], axis=1)
        out.update(pose_sensors=sensors, m_stamp=np.ascontiguousarray(stamp), m_sensor=sidx, m_pose=np.ascontiguousarray(pose))
    return dataclasses.replace(win, **out)


def make_stereo_tracks(win: Window, t0: float, t1: float, frame_dt=0.05, new_per_frame=20, frames_per_landmark=4, pixel_sigma=0.5,
                       seed=SEED_BASE + 99) -> dict:
    """Stereo tracks of the reference's live frame loop (VisualTracks, abstract.cpp:243-260) from the truth of `win`:
    camera frames at t0, t0 + frame_dt, ... < t1; every frame `new_per_frame` landmarks appear and each stays visible in
    both cameras (cameras 0 and 1) for `frames_per_landmark` consecutive frames.  Returns the tracks sorted by stamp
    (stamp, cam0, cam1, px0, px1, gid = global landmark id) and the true landmark positions (landmarks[gid])."""
    rng = np.random.Generator(np.random.Philox(seed))
    truth = win.truth if win.truth is not None else dict(knots=win.knots)
    knots, k, cams = truth["knots"], win.order, win.cameras
    nf = int(math.ceil((t1 - t0) / frame_dt - 1e-9))
    F = frames_per_landmark
    birth = np.repeat(np.arange(nf), new_per_frame)
    G = birth.size
    landmarks = np.zeros((G, 3))
    todo = np.arange(G)
    while todo.size:
        n = todo.size
        fr = np.minimum(birth[todo][:, None] + np.arange(F)[None, :], nf - 1)        # (n, F) frames the landmark is seen in
        tc = t0 + fr[:, F // 2] * frame_dt
        px = np.stack([rng.uniform(150, IMAGE_SIZE[0] - 150, n), rng.uniform(120, IMAGE_SIZE[1] - 120, n)], -1)
        depth = rng.uniform(2.0, 10.0, n)
        R, p, *_ = spline_eval(knots, k, tc)
        c0 = cams[0]
        ray = np.stack([(px[:, 0] - c0[7]) / c0[9], (px[:, 1] - c0[8]) / c0[10], np.ones(n)], -1) * depth[:, None]
        p_b = ray @ quat_to_rot(c0[None, :4])[0].T + c0[4:7]
        lm = (R @ p_b[..., None])[..., 0] + p
        ok = np.ones(n, dtype=bool)
        for f in range(F):
            for c in (0, 1):
                pix, p_s = pixel_model(knots, k, cams, lm, t0 + fr[:, f] * frame_dt, np.full(n, c), np.arange(n))
                ok &= (p_s[:, 2] > 0.5) & (pix[:, 0] > 0) & (pix[:, 0] < IMAGE_SIZE[0]) & (pix[:, 1] > 0) & (pix[:, 1] < IMAGE_SIZE[1])
        landmarks[todo[ok]] = lm[ok]
        todo = todo[~ok]
    frame = birth[:, None] + np.arange(F)[None, :]
    gid = np.repeat(np.arange(G), F)[(frame < nf).ravel()]
    frame = frame[frame < nf]
    order = np.lexsort((gid, frame))
    gid, stamp = gid[order], t0 + frame[order] * frame_dt
    n = gid.size
    px0, _ = pixel_model(knots, k, cams, landmarks, stamp, np.zeros(n, dtype=np.int64), gid)
    px1, _ = pixel_model(knots, k, cams, landmarks, stamp, np.ones(n, dtype=np.int64), gid)
    px0 = px0 + rng.normal(0.0, pixel_sigma, px0.shape)
    px1 = px1 + rng.normal(0.0, pixel_sigma, px1.shape)
    return dict(stamp=stamp, cam0=np.zeros(n, np.int32), cam1=np.ones(n, np.int32), px0=np.ascontiguousarray(px0), px1=np.ascontiguousarray(px1),
                gid=gid.astype(np.int64), landmarks=landmarks)


# BASELINE.json configs (index = position in BASELINE.json "configs").
CONFIGS = {
    0: dict(order=4, num_knots=8, num_landmarks=0, num_imu=200, num_cameras=2),
    1: dict(order=4, num_knots=50, num_landmarks=1000, frames_per_landmark=5, num_cameras=2, num_imu=2000),
    2: dict(order=6, num_knots=200, num_landmarks=10000, frames_per_landmark=5, num_cameras=2, num_imu=20000),
    3: dict(order=4, num_knots=500, num_landmarks=25000, frames_per_landmark=5, num_cameras=4, num_imu=0),
    4: dict(order=4, num_knots=500, num_landmarks=83300, frames_per_landmark=5, num_cameras=2, num_imu=167000),
}
CONFIG_NAMES = {
    0: "cfg0: order-4, 8 knots, 200 IMU (plumbing)",
    1: "cfg1: order-4 SE(3) spline, 50 knots, 10k stereo pixel + 2k IMU factors, 1k landmarks",
    2: "cfg2: order-6, 200 knots, 100k pixel + 20k IMU",
    3: "cfg3: 4-camera rig, 500 knots, 500k pixel factors",
    4: "cfg4: 1M-factor window (833k pixel + 167k IMU), 500 knots",
}


def make_config(index: int, scale: float = 1.0, **overrides) -> Window:
    cfg = dict(CONFIGS[index])
    if scale != 1.0:
        cfg["num_landmarks"] = max(1, int(round(cfg["num_landmarks"] * scale))) if cfg["num_landmarks"] else 0
        cfg["num_imu"] = int(round(cfg["num_imu"] * scale))
    cfg.update(overrides)
    cfg.setdefault("seed", SEED_BASE + index + 1)
    return make_window(**cfg)
