// Calibration-block Jacobians (sm_90a), produced on demand -- the sensor blocks are constant in the live
// configuration (reference internal/hyper/optimizers/ceres/optimizer.cpp:59-63), so the iteration kernels never
// carry them; the reference's own gradient tests however run with every sensor manifold non-constant
// (reference tests/internal/tests/optimizers/evaluators/pixel.cpp:57), and hb200_factor_evaluate hands these
// blocks out in the Ceres shape.  One factor per thread, value-only interpolation from the knot table, then
//   pixel   (reference evaluators/pixel.cpp:91-135,141): extrinsics T_bs (tangent 6), intrinsics [cx cy fx fy],
//           radial-tangential distortion [k1 k2 p1 p2]                                   -> Jc[n][2][14]
//   bearing (reference evaluators/bearing.cpp:62-78): extrinsics only (row 0 of the same slot)
//   manifold(reference evaluators/manifold.cpp:57): extrinsics                           -> Jc[n][6][6]
//   inertial(reference evaluators/inertial.cpp:155-194): extrinsics, gyroscope / accelerometer intrinsics,
//           S_g, X_a, with the reference-quirk switches of the oracle                   -> Jc[n][6][36]
// Tangent convention: R_bs <- Exp(theta) R_bs, t_bs <- t_bs + rho; the 6 -> 7 ambient adapter is applied by the
// host copy-out exactly as for the control-point blocks.
#pragma once
#include "hb200_eval.cuh"

namespace hb {

enum {   // == oracle/ho_evaluators.h Quirks (SURVEY.md section 8a "Reference quirks in a6")
  kQuirkGyroIntrinsicsInAccelRows = 1,   // (i)  inertial.cpp:136,142,148,158 use I_g where I_a is meant
  kQuirkNoSgJacobian = 2,                // (ii) S_g a_b_m contributes no state / extrinsics / X_a / gravity Jacobian
  kQuirkLocalExtrinsics = 4,             // (iv) inertial.cpp:157-158 omit R_sb
  kQuirkAxesOffsetsIgnored = 8           // (v)  inertial.cpp:142,148 use t_bs only
};

// pose of the body at the factor's stamp (value only): R (row-major), p
template <int K>
HB_DI void pose_value(const double* __restrict__ T, const Basis& B, int base, double t, double* P, double* p) {
  constexpr int left = (K - 1) / 2;
  const double* row0 = T + static_cast<size_t>(base) * kTabStride;
  const double t0 = row0[left * kTabStride + 24], t1 = row0[(left + 1) * kTabStride + 24];
  const double inv_dt = 1.0 / (t1 - t0);
  double lam[K + 1];
  basis_eval<K, false>(B, (t - t0) * inv_dt, inv_dt, lam, nullptr, nullptr);
#pragma unroll
  for (int i = 0; i < 9; ++i) P[i] = row0[i];
  p[0] = row0[9]; p[1] = row0[10]; p[2] = row0[11];
#pragma unroll
  for (int j = 1; j < K; ++j) {
    const double* rj = row0 + j * kTabStride;
    const double w[3] = {lam[j] * rj[12], lam[j] * rj[13], lam[j] * rj[14]};
    double A[9], Pn[9];
    so3_exp_and_Jr(w, A, nullptr);
    m3_mul(P, A, Pn);
#pragma unroll
    for (int i = 0; i < 9; ++i) P[i] = Pn[i];
#pragma unroll
    for (int c = 0; c < 3; ++c) p[c] += lam[j] * (rj[9 + c] - rj[9 + c - kTabStride]);
  }
}

// row (1x3) times [R_sb hat(v) | -R_sb]: the extrinsics tangent block of anything that depends on p_s = R_sb (p_b - t_bs)
HB_DI void extrinsics_row(const double* a /* = d/dp_s * R_sb, 1x3 */, const double* v /* p_b - t_bs */, double* out /*6*/) {
  out[0] = a[1] * v[2] - a[2] * v[1];
  out[1] = a[2] * v[0] - a[0] * v[2];
  out[2] = a[0] * v[1] - a[1] * v[0];
  out[3] = -a[0]; out[4] = -a[1]; out[5] = -a[2];
}

template <int K>
__global__ void __launch_bounds__(kEvalThreads) pixel_calib_kernel(int n, const double* __restrict__ stamp, const double2* __restrict__ pixel,
                                                                   const double* __restrict__ meas_z, const int4* __restrict__ idx,
                                                                   const double* __restrict__ tab, const double* __restrict__ cam_tab,
                                                                   const double* __restrict__ landmarks, Basis B, double* __restrict__ Jc /*[n][2][14]*/) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  const int4 id = idx[f];
  const double* cam = cam_tab + kCamStride * id.z;
  const double* lmk = landmarks + 3 * static_cast<size_t>(id.y);
  double P[9], p[3];
  pose_value<K>(tab, B, id.x, stamp[f], P, p);
  const double q[3] = {lmk[0] - p[0], lmk[1] - p[1], lmk[2] - p[2]};
  double pb[3], ps[3];
  m3_tvec(P, q, pb);
  const double pbt[3] = {pb[0] - cam[9], pb[1] - cam[10], pb[2] - cam[11]};
  m3_vec(cam, pbt, ps);
  double J[28];
#pragma unroll
  for (int i = 0; i < 28; ++i) J[i] = 0.0;
  double Jps[6] = {0, 0, 0, 0, 0, 0};
  if (id.w == 0) {
    const double iz = 1.0 / ps[2];
    const double x = ps[0] * iz, y = ps[1] * iz;
    const double fx = cam[14], fy = cam[15];
    const double k1 = cam[16], k2 = cam[17], p1 = cam[18], p2 = cam[19];
    const double r2 = x * x + y * y;
    const double rad = 1.0 + k1 * r2 + k2 * r2 * r2;
    const double dx = x * rad + 2.0 * p1 * x * y + p2 * (r2 + 2.0 * x * x);
    const double dy = y * rad + p1 * (r2 + 2.0 * y * y) + 2.0 * p2 * x * y;
    const double g = k1 + 2.0 * k2 * r2;
    const double drx = 2.0 * x * g, dry = 2.0 * y * g;
    const double a00 = fx * (rad + x * drx + 2.0 * p1 * y + 6.0 * p2 * x);
    const double a01 = fx * (x * dry + 2.0 * p1 * x + 2.0 * p2 * y);
    const double a10 = fy * (y * drx + 2.0 * p1 * x + 2.0 * p2 * y);
    const double a11 = fy * (rad + y * dry + 6.0 * p1 * y + 2.0 * p2 * x);
    Jps[0] = a00 * iz; Jps[1] = a01 * iz; Jps[2] = -(a00 * x + a01 * y) * iz;
    Jps[3] = a10 * iz; Jps[4] = a11 * iz; Jps[5] = -(a10 * x + a11 * y) * iz;
    // intrinsics [cx cy fx fy] (pixel.cpp:99-102,125) and distortion [k1 k2 p1 p2] (pixel.cpp:95,114)
    J[6] = 1.0; J[8] = dx; J[14 + 7] = 1.0; J[14 + 9] = dy;
    J[10] = fx * x * r2; J[11] = fx * x * r2 * r2; J[12] = fx * 2.0 * x * y; J[13] = fx * (r2 + 2.0 * x * x);
    J[14 + 10] = fy * y * r2; J[14 + 11] = fy * y * r2 * r2; J[14 + 12] = fy * (r2 + 2.0 * y * y); J[14 + 13] = fy * 2.0 * x * y;
  } else {
    const double z[3] = {pixel[f].x, pixel[f].y, meas_z[f]};
    double cr[3];
    cross(ps, z, cr);
    const double s = sqrt(cr[0] * cr[0] + cr[1] * cr[1] + cr[2] * cr[2]), c = ps[0] * z[0] + ps[1] * z[1] + ps[2] * z[2];
    if (s > 1e-300) {
      const double is = 1.0 / s;
      const double nrm[3] = {cr[0] * is, cr[1] * is, cr[2] * is};
      double zn[3];
      cross(z, nrm, zn);
      const double iden = 1.0 / ((ps[0] * ps[0] + ps[1] * ps[1] + ps[2] * ps[2]) * (z[0] * z[0] + z[1] * z[1] + z[2] * z[2]));
#pragma unroll
      for (int i = 0; i < 3; ++i) Jps[i] = (c * zn[i] - s * z[i]) * iden;
    }
  }
  // extrinsics (pixel.cpp:141 / bearing.cpp:76): J_r_p_s [R_sb hat(p_b - t_bs) | -R_sb]
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    double a[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) a[j] = Jps[3 * i] * cam[j] + Jps[3 * i + 1] * cam[3 + j] + Jps[3 * i + 2] * cam[6 + j];
    extrinsics_row(a, pbt, &J[14 * i]);
  }
  double* out = Jc + 28 * static_cast<size_t>(f);
#pragma unroll
  for (int i = 0; i < 28; ++i) out[i] = J[i];
}

template <int K>
__global__ void __launch_bounds__(kEvalThreads) manifold_calib_kernel(int n, const double* __restrict__ stamp, const double* __restrict__ meas,
                                                                      const int2* __restrict__ idx, const double* __restrict__ tab,
                                                                      const double* __restrict__ sensors, Basis B, double* __restrict__ Jc /*[n][6][6]*/) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  const int2 id = idx[f];
  double P[9], p[3];
  pose_value<K>(tab, B, id.x, stamp[f], P, p);
  const double* T_bs = sensors + 7 * static_cast<size_t>(id.y);
  const double* z = meas + 7 * static_cast<size_t>(f);
  double Rbs[9], Rz[9], Rws[9], Rerr[9], q[4], th[3];
  quat_to_rot(T_bs, Rbs);
  quat_to_rot(z, Rz);
  m3_mul(P, Rbs, Rws);
  m3_mult(Rws, Rz, Rerr);
  rot_to_quat(Rerr, q);
  quat_log(q, th);
  const double nth[3] = {-th[0], -th[1], -th[2]};
  double A[9], AR[9];
  so3_Jr_inv(nth, A);   // Jl^{-1}(theta)
  m3_mul(A, P, AR);
  // manifold.cpp:57: J_metric * J(T_wb (+) T_bs wrt T_bs) = blockdiag(Jl^{-1} R_wb, R_wb)
  double* out = Jc + 36 * static_cast<size_t>(f);
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      out[6 * i + c] = AR[3 * i + c]; out[6 * i + 3 + c] = 0.0;
      out[6 * (3 + i) + c] = 0.0; out[6 * (3 + i) + 3 + c] = P[3 * i + c];
    }
}

template <int K>
__global__ void __launch_bounds__(kEvalThreads) inertial_calib_kernel(int n, const double* __restrict__ stamp, const int4* __restrict__ idx,
                                                                      const double* __restrict__ tab, const double* __restrict__ imu /*raw 37*/,
                                                                      const double* __restrict__ gravity, Basis B, int quirks,
                                                                      double* __restrict__ Jc /*[n][6][36]*/) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  constexpr int left = (K - 1) / 2;
  const double* row0 = tab + static_cast<size_t>(idx[f].x) * kTabStride;
  const double t0 = row0[left * kTabStride + 24], t1 = row0[(left + 1) * kTabStride + 24];
  const double inv_dt = 1.0 / (t1 - t0);
  double lam[K + 1], lamd[K + 1], lamdd[K + 1];
  basis_eval<K, true>(B, (stamp[f] - t0) * inv_dt, inv_dt, lam, lamd, lamdd);
  double P[9], pdd[3] = {0, 0, 0}, w[3] = {0, 0, 0}, wd[3] = {0, 0, 0};
#pragma unroll
  for (int i = 0; i < 9; ++i) P[i] = row0[i];
#pragma unroll
  for (int j = 1; j < K; ++j) {
    const double* rj = row0 + j * kTabStride;
    const double d[3] = {rj[12], rj[13], rj[14]};
    const double lw[3] = {lam[j] * d[0], lam[j] * d[1], lam[j] * d[2]};
    double A[9], Pn[9], aw[3], awd[3], wn[3], cr[3];
    so3_exp_and_Jr(lw, A, nullptr);
    m3_mul(P, A, Pn);
#pragma unroll
    for (int i = 0; i < 9; ++i) P[i] = Pn[i];
    m3_tvec(A, w, aw);
    m3_tvec(A, wd, awd);
#pragma unroll
    for (int c = 0; c < 3; ++c) wn[c] = aw[c] + lamd[j] * d[c];
    cross(wn, d, cr);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      wd[c] = awd[c] + lamd[j] * cr[c] + lamdd[j] * d[c];
      w[c] = wn[c];
      pdd[c] += lamdd[j] * (rj[9 + c] - rj[9 + c - kTabStride]);
    }
  }
  // calibration (inertial.cpp:35-49,114-119)
  double Rbs[9], Rsb[9];
  quat_to_rot(imu, Rbs);
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) Rsb[3 * i + j] = Rbs[3 * j + i];
  const double* t_bs = imu + 4;
  const double* ig = imu + 7;
  const double* ia = imu + 13;
  const double Ig[9] = {ig[0], 0, 0, ig[3], ig[1], 0, ig[4], ig[5], ig[2]};
  const double Ia[9] = {ia[0], 0, 0, ia[3], ia[1], 0, ia[4], ia[5], ia[2]};
  double Sg[9], IaR[9];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) Sg[3 * i + j] = imu[19 + i + 3 * j];
  m3_mul(Ia, Rsb, IaR);
  const bool q_i = quirks & kQuirkGyroIntrinsicsInAccelRows, q_sg = quirks & kQuirkNoSgJacobian, q_loc = quirks & kQuirkLocalExtrinsics;
  // model (inertial.cpp:121-128)
  const double gm[3] = {pdd[0] - gravity[0], pdd[1] - gravity[1], pdd[2] - gravity[2]};
  double a_i[3], a_m[3], Fa[9];
  m3_tvec(P, gm, a_i);
  {
    const double ww = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) Fa[3 * i + j] = w[i] * w[j] - (i == j ? ww : 0.0);
    Fa[1] -= wd[2]; Fa[2] += wd[1]; Fa[3] += wd[2]; Fa[5] -= wd[0]; Fa[6] -= wd[1]; Fa[7] += wd[0];
  }
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double c[3] = {imu[28 + 3 * r] + t_bs[0], imu[28 + 3 * r + 1] + t_bs[1], imu[28 + 3 * r + 2] + t_bs[2]};   // X_a[:, r] + t_bs
    a_m[r] = a_i[r] + Fa[3 * r] * c[0] + Fa[3 * r + 1] * c[1] + Fa[3 * r + 2] * c[2];
  }
  double w_s[3], a_s[3];
  m3_vec(Rsb, w, w_s);
  m3_vec(Rsb, a_m, a_s);
  double J[216];
#pragma unroll 1
  for (int i = 0; i < 216; ++i) J[i] = 0.0;
  // extrinsics (inertial.cpp:155-162): [I_g hat(w_s) (R_sb) , S_g F_a ; I_lin hat(a_s) (R_sb) , I_a R_sb F_a]
  {
    double H[9], t[9], u[9];
    hat(w_s, H);
    m3_mul(Ig, H, t);
    if (!q_loc) { m3_mul(t, Rsb, u); } else {
#pragma unroll
      for (int i = 0; i < 9; ++i) u[i] = t[i];
    }
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int c = 0; c < 3; ++c) J[36 * i + c] = u[3 * i + c];
    hat(a_s, H);
    m3_mul(q_i ? Ig : Ia, H, t);
    if (!q_loc) { m3_mul(t, Rsb, u); } else {
#pragma unroll
      for (int i = 0; i < 9; ++i) u[i] = t[i];
    }
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int c = 0; c < 3; ++c) J[36 * (3 + i) + c] = u[3 * i + c];
    m3_mul(IaR, Fa, t);
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int c = 0; c < 3; ++c) J[36 * (3 + i) + 3 + c] = t[3 * i + c];
    if (!q_sg) {
      m3_mul(Sg, Fa, t);
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int c = 0; c < 3; ++c) J[36 * i + 3 + c] = t[3 * i + c];
    }
  }
  // gyroscope / accelerometer intrinsics [c00 c11 c22 c10 c20 c21] via align() (inertial.cpp:164-174)
  J[36 * 0 + 6 + 0] = w_s[0];
  J[36 * 1 + 6 + 1] = w_s[1]; J[36 * 1 + 6 + 3] = w_s[0];
  J[36 * 2 + 6 + 2] = w_s[2]; J[36 * 2 + 6 + 4] = w_s[0]; J[36 * 2 + 6 + 5] = w_s[1];
  J[36 * 3 + 12 + 0] = a_s[0];
  J[36 * 4 + 12 + 1] = a_s[1]; J[36 * 4 + 12 + 3] = a_s[0];
  J[36 * 5 + 12 + 2] = a_s[2]; J[36 * 5 + 12 + 4] = a_s[0]; J[36 * 5 + 12 + 5] = a_s[1];
  // S_g, column-major 3x3 block (inertial.cpp:176-187): d r_omega[i] / d S_g(i, j) = a_b_m[j]
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) J[36 * i + 18 + i + 3 * j] = a_m[j];
  // X_a, column-major (inertial.cpp:189-194): column r of X_a is the lever arm of axis r
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        J[36 * (3 + i) + 27 + 3 * r + j] = IaR[3 * i + r] * Fa[3 * r + j];
        if (!q_sg) J[36 * i + 27 + 3 * r + j] = Sg[3 * i + r] * Fa[3 * r + j];
      }
  double* out = Jc + 216 * static_cast<size_t>(f);
#pragma unroll 1
  for (int i = 0; i < 216; ++i) out[i] = J[i];
}

}  // namespace hb
