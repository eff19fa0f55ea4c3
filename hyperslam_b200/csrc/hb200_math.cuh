// Device-side fixed-size math for the sm_90a hot path (FP64, row-major 3x3, everything in
// registers after full unrolling).  Conventions are those of DESIGN.md: quaternion [x y z w],
// global rotation tangent R <- Exp(theta) R, split SE3 tangent [theta | rho].
#pragma once
#include <cuda_runtime.h>

namespace hb {

#define HB_DI __device__ __forceinline__

HB_DI void m3_mul(const double* A, const double* B, double* C) {  // C = A B (no aliasing)
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
HB_DI void m3_tmul(const double* A, const double* B, double* C) {  // C = A^T B
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[i] * B[j] + A[3 + i] * B[3 + j] + A[6 + i] * B[6 + j];
}
HB_DI void m3_mult(const double* A, const double* B, double* C) {  // C = A B^T
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[3 * j] + A[3 * i + 1] * B[3 * j + 1] + A[3 * i + 2] * B[3 * j + 2];
}
HB_DI void m3_vec(const double* A, const double* v, double* r) {  // r = A v (no aliasing)
#pragma unroll
  for (int i = 0; i < 3; ++i) r[i] = A[3 * i] * v[0] + A[3 * i + 1] * v[1] + A[3 * i + 2] * v[2];
}
HB_DI void m3_tvec(const double* A, const double* v, double* r) {  // r = A^T v
#pragma unroll
  for (int i = 0; i < 3; ++i) r[i] = A[i] * v[0] + A[3 + i] * v[1] + A[6 + i] * v[2];
}
HB_DI void hat(const double* v, double* A) {
  A[0] = 0; A[1] = -v[2]; A[2] = v[1];
  A[3] = v[2]; A[4] = 0; A[5] = -v[0];
  A[6] = -v[1]; A[7] = v[0]; A[8] = 0;
}
// C = hat(a) * B
HB_DI void hat_mul(const double* a, const double* B, double* C) {
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    C[j] = a[1] * B[6 + j] - a[2] * B[3 + j];
    C[3 + j] = a[2] * B[j] - a[0] * B[6 + j];
    C[6 + j] = a[0] * B[3 + j] - a[1] * B[j];
  }
}
// C = A * hat(b)
HB_DI void mul_hat(const double* A, const double* b, double* C) {
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    C[3 * i] = A[3 * i + 1] * b[2] - A[3 * i + 2] * b[1];
    C[3 * i + 1] = A[3 * i + 2] * b[0] - A[3 * i] * b[2];
    C[3 * i + 2] = A[3 * i] * b[1] - A[3 * i + 1] * b[0];
  }
}
HB_DI void cross(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

HB_DI void quat_to_rot(const double* q, double* R) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
  const double twx = tx * w, twy = ty * w, twz = tz * w;
  const double txx = tx * x, txy = ty * x, txz = tz * x;
  const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
  R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
  R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}
HB_DI void quat_mul(const double* a, const double* b, double* c) {
  const double x = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  const double y = a[3] * b[1] - a[0] * b[2] + a[1] * b[3] + a[2] * b[0];
  const double z = a[3] * b[2] + a[0] * b[1] - a[1] * b[0] + a[2] * b[3];
  const double w = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
  c[0] = x; c[1] = y; c[2] = z; c[3] = w;
}
HB_DI void quat_log(const double* q, double* d) {
  double x = q[0], y = q[1], z = q[2], w = q[3];
  if (w < 0) { x = -x; y = -y; z = -z; w = -w; }
  const double n2 = x * x + y * y + z * z;
  const double n = sqrt(n2);
  double s;
  if (n < 1e-7) s = (2.0 / w) * (1.0 - n2 / (3.0 * w * w));
  else s = 2.0 * atan2(n, w) / n;
  d[0] = s * x; d[1] = s * y; d[2] = s * z;
}
// Rotation matrix -> unit quaternion [x y z w] (Shepperd's method: pivot on the largest of w^2, x^2, y^2, z^2).
HB_DI void rot_to_quat(const double* R, double* q) {
  const double tr = R[0] + R[4] + R[8];
  double x, y, z, w;
  if (tr > 0.0) {
    const double s = 2.0 * sqrt(1.0 + tr);
    w = 0.25 * s; x = (R[7] - R[5]) / s; y = (R[2] - R[6]) / s; z = (R[3] - R[1]) / s;
  } else if (R[0] > R[4] && R[0] > R[8]) {
    const double s = 2.0 * sqrt(1.0 + R[0] - R[4] - R[8]);
    w = (R[7] - R[5]) / s; x = 0.25 * s; y = (R[1] + R[3]) / s; z = (R[2] + R[6]) / s;
  } else if (R[4] > R[8]) {
    const double s = 2.0 * sqrt(1.0 + R[4] - R[0] - R[8]);
    w = (R[2] - R[6]) / s; x = (R[1] + R[3]) / s; y = 0.25 * s; z = (R[5] + R[7]) / s;
  } else {
    const double s = 2.0 * sqrt(1.0 + R[8] - R[0] - R[4]);
    w = (R[3] - R[1]) / s; x = (R[2] + R[6]) / s; y = (R[5] + R[7]) / s; z = 0.25 * s;
  }
  q[0] = x; q[1] = y; q[2] = z; q[3] = w;
}
HB_DI void quat_exp(const double* d, double* q) {
  const double t2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
  const double t = sqrt(t2);
  double s, c;
  if (t < 1e-7) { s = 0.5 - t2 / 48.0; c = 1.0 - t2 / 8.0; }
  else { double sh, ch; sincos(0.5 * t, &sh, &ch); s = sh / t; c = ch; }
  q[0] = s * d[0]; q[1] = s * d[1]; q[2] = s * d[2]; q[3] = c;
}

// a = sin t / t, b = (1 - cos t)/t^2, c = (t - sin t)/t^3
HB_DI void so3_coeffs(double t2, double* a, double* b, double* c) {
  if (t2 < 1e-8) {
    *a = 1.0 - t2 / 6.0 + t2 * t2 / 120.0;
    *b = 0.5 - t2 / 24.0 + t2 * t2 / 720.0;
    *c = 1.0 / 6.0 - t2 / 120.0 + t2 * t2 / 5040.0;
  } else {
    const double t = sqrt(t2);
    double s, co;
    sincos(t, &s, &co);
    const double it2 = 1.0 / t2;
    *a = s / t;
    *b = (1.0 - co) * it2;
    *c = (t - s) * it2 / t;
  }
}
// E = Exp(w) = I + a W + b W^2 and J = Jr(w) = I - b W + c W^2 from one sincos.
HB_DI void so3_exp_and_Jr(const double* w, double* E, double* J) {
  const double xx = w[0] * w[0], yy = w[1] * w[1], zz = w[2] * w[2];
  const double xy = w[0] * w[1], xz = w[0] * w[2], yz = w[1] * w[2];
  double a, b, c;
  so3_coeffs(xx + yy + zz, &a, &b, &c);
  // W^2 = w w^T - |w|^2 I
  const double W2[9] = {-(yy + zz), xy, xz, xy, -(xx + zz), yz, xz, yz, -(xx + yy)};
  const double W[9] = {0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0};
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    const double id = (i % 4 == 0) ? 1.0 : 0.0;
    E[i] = id + a * W[i] + b * W2[i];
    if (J) J[i] = id - b * W[i] + c * W2[i];
  }
}
HB_DI void so3_Jr_inv(const double* w, double* J) {
  const double xx = w[0] * w[0], yy = w[1] * w[1], zz = w[2] * w[2];
  const double xy = w[0] * w[1], xz = w[0] * w[2], yz = w[1] * w[2];
  const double t2 = xx + yy + zz;
  double e;
  if (t2 < 1e-6) e = 1.0 / 12.0 + t2 / 720.0 + t2 * t2 / 30240.0;
  else { const double t = sqrt(t2); double s, co; sincos(t, &s, &co); e = 1.0 / t2 - (1.0 + co) / (2.0 * t * s); }
  const double W2[9] = {-(yy + zz), xy, xz, xy, -(xx + zz), yz, xz, yz, -(xx + yy)};
  const double W[9] = {0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0};
#pragma unroll
  for (int i = 0; i < 9; ++i) J[i] = ((i % 4 == 0) ? 1.0 : 0.0) + 0.5 * W[i] + e * W2[i];
}

}  // namespace hb
