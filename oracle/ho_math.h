// TEST INFRASTRUCTURE ONLY -- CPU oracle for the HyperSLAM Evaluate()/GN hot path.
// PARITY UNPINNED: the reference's Lie-group / spline / sensor arithmetic lives in the
// un-vendored HyperVariables / HyperState / HyperSensors (reference CMakeLists.txt:26-27) and
// Ceres; none of it is on disk, so everything below is a restatement of published formulas
// (Sola 2018, Sommer 2020, Ceres 2.1 manifold docs) anchored on the reference's in-tree call
// sites.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
// legs may use this directory.  Nothing under hyperslam_b200/ links or imports it.
//
// Small fixed-size linear algebra + SO(3) helpers (row-major 3x3).
// Conventions (see DESIGN.md "Conventions"):
//   * quaternion storage [x y z w] (Eigen coefficient order; reference settings.yaml:34-36)
//   * rotation tangent is GLOBAL (left): R <- Exp(theta) R   (reference inertial.cpp:136 is only
//     consistent with a left perturbation; Ceres EigenQuaternionManifold is left-multiplicative too)
//   * SE3 tangent is split [theta(3) | rho(3)], p <- p + rho   (reference inertial.cpp:160)
#pragma once
#include <cmath>
#include <cstring>

namespace ho {

inline void v3_set(double* a, double x, double y, double z) { a[0] = x; a[1] = y; a[2] = z; }
inline void v3_copy(const double* a, double* b) { b[0] = a[0]; b[1] = a[1]; b[2] = a[2]; }
inline double v3_dot(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
inline void v3_cross(const double* a, const double* b, double* c) {
  const double x = a[1] * b[2] - a[2] * b[1], y = a[2] * b[0] - a[0] * b[2], z = a[0] * b[1] - a[1] * b[0];
  c[0] = x; c[1] = y; c[2] = z;
}
inline void m3_identity(double* A) { for (int i = 0; i < 9; ++i) A[i] = (i % 4 == 0) ? 1.0 : 0.0; }
inline void m3_zero(double* A) { for (int i = 0; i < 9; ++i) A[i] = 0.0; }
inline void m3_copy(const double* A, double* B) { std::memcpy(B, A, 9 * sizeof(double)); }
inline void m3_transpose(const double* A, double* B) {
  double T[9];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) T[3 * i + j] = A[3 * j + i];
  m3_copy(T, B);
}
// C = A * B
inline void m3_mul(const double* A, const double* B, double* C) {
  double T[9];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j)
    T[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
  m3_copy(T, C);
}
// C = A^T * B
inline void m3_tmul(const double* A, const double* B, double* C) {
  double T[9];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j)
    T[3 * i + j] = A[i] * B[j] + A[3 + i] * B[3 + j] + A[6 + i] * B[6 + j];
  m3_copy(T, C);
}
// C = A * B^T
inline void m3_mult(const double* A, const double* B, double* C) {
  double T[9];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j)
    T[3 * i + j] = A[3 * i] * B[3 * j] + A[3 * i + 1] * B[3 * j + 1] + A[3 * i + 2] * B[3 * j + 2];
  m3_copy(T, C);
}
inline void m3_vec(const double* A, const double* v, double* r) {
  const double x = A[0] * v[0] + A[1] * v[1] + A[2] * v[2];
  const double y = A[3] * v[0] + A[4] * v[1] + A[5] * v[2];
  const double z = A[6] * v[0] + A[7] * v[1] + A[8] * v[2];
  r[0] = x; r[1] = y; r[2] = z;
}
inline void m3_tvec(const double* A, const double* v, double* r) {
  const double x = A[0] * v[0] + A[3] * v[1] + A[6] * v[2];
  const double y = A[1] * v[0] + A[4] * v[1] + A[7] * v[2];
  const double z = A[2] * v[0] + A[5] * v[1] + A[8] * v[2];
  r[0] = x; r[1] = y; r[2] = z;
}
inline void m3_scale(double* A, double s) { for (int i = 0; i < 9; ++i) A[i] *= s; }
inline void m3_add(const double* A, const double* B, double* C) { for (int i = 0; i < 9; ++i) C[i] = A[i] + B[i]; }
inline void m3_sub(const double* A, const double* B, double* C) { for (int i = 0; i < 9; ++i) C[i] = A[i] - B[i]; }
inline void hat(const double* v, double* A) {
  A[0] = 0; A[1] = -v[2]; A[2] = v[1];
  A[3] = v[2]; A[4] = 0; A[5] = -v[0];
  A[6] = -v[1]; A[7] = v[0]; A[8] = 0;
}

// Quaternion [x y z w] -> rotation matrix (unit quaternion assumed, as Eigen's toRotationMatrix).
inline void quat_to_rot(const double* q, double* R) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
  const double twx = tx * w, twy = ty * w, twz = tz * w;
  const double txx = tx * x, txy = ty * x, txz = tz * x;
  const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
  R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
  R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}
// Hamilton product c = a (x) b, [x y z w].
inline void quat_mul(const double* a, const double* b, double* c) {
  const double x = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  const double y = a[3] * b[1] - a[0] * b[2] + a[1] * b[3] + a[2] * b[0];
  const double z = a[3] * b[2] + a[0] * b[1] - a[1] * b[0] + a[2] * b[3];
  const double w = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
  c[0] = x; c[1] = y; c[2] = z; c[3] = w;
}
inline void quat_conj(const double* a, double* b) { b[0] = -a[0]; b[1] = -a[1]; b[2] = -a[2]; b[3] = a[3]; }

// Log of a unit quaternion -> rotation vector (angle in (-pi, pi]).
inline void quat_log(const double* q, double* d) {
  double x = q[0], y = q[1], z = q[2], w = q[3];
  if (w < 0) { x = -x; y = -y; z = -z; w = -w; }
  const double n2 = x * x + y * y + z * z;
  const double n = std::sqrt(n2);
  double s;
  if (n < 1e-7) {
    // 2*atan2(n,w)/n = (2/w) * (1 - n^2/(3 w^2) + ...)
    s = (2.0 / w) * (1.0 - n2 / (3.0 * w * w));
  } else {
    s = 2.0 * std::atan2(n, w) / n;
  }
  d[0] = s * x; d[1] = s * y; d[2] = s * z;
}
// Exp: rotation vector -> unit quaternion.
inline void quat_exp(const double* d, double* q) {
  const double t2 = v3_dot(d, d);
  const double t = std::sqrt(t2);
  double s, c;
  if (t < 1e-7) { s = 0.5 - t2 / 48.0; c = 1.0 - t2 / 8.0; }
  else { s = std::sin(0.5 * t) / t; c = std::cos(0.5 * t); }
  q[0] = s * d[0]; q[1] = s * d[1]; q[2] = s * d[2]; q[3] = c;
}

// (t - sin t)/t^3 = sum_n (-1)^n t^2n / (2n+3)!, n = 0..9: below t^2 = 2.5 the closed form cancels by more than
// 6/t^2 ulps, and the truncated tail stays under 1e-17 relative.
inline double so3_c_series(double t2) {
  static const double k[10] = {1.0 / 6.0, -1.0 / 120.0, 1.0 / 5040.0, -1.0 / 362880.0, 1.0 / 39916800.0, -1.0 / 6227020800.0,
                               1.0 / 1307674368000.0, -1.0 / 355687428096000.0, 1.0 / 121645100408832000.0,
                               -1.0 / 51090942171709440000.0};
  double c = k[9];
  for (int n = 8; n >= 0; --n) c = c * t2 + k[n];
  return c;
}
// 1/t^2 - (1 + cos t)/(2 t sin t) = sum_n |B_2n+2| t^2n / (2n+2)!, n = 0..16: below t^2 = 4 the closed form cancels by
// more than 24/t^2 ulps, and the truncated tail stays under 1e-17 relative.
inline double so3_e_series(double t2) {
  static const double k[17] = {1.0 / 12.0, 1.0 / 720.0, 3.306878306878307e-05, 8.267195767195768e-07, 2.08767569878681e-08,
                               5.284190138687493e-10, 1.3382536530684679e-11, 3.3896802963225827e-13, 8.586062056277845e-15,
                               2.174868698558062e-16, 5.5090028283602295e-18, 1.3954464685812522e-19, 3.534707039629467e-21,
                               8.953517427037546e-23, 2.267952452337683e-24, 5.744790668872202e-26, 1.455172475614865e-27};
  double e = k[16];
  for (int n = 15; n >= 0; --n) e = e * t2 + k[n];
  return e;
}
// Rodrigues coefficients: a = sin(t)/t, b = (1-cos t)/t^2, c = (t - sin t)/t^3.  a and b come from the half angle
// (1 - cos t = 2 sin^2(t/2) does not cancel); c takes its series wherever t - sin t would cancel.
inline void so3_coeffs(double t2, double* a, double* b, double* c) {
  if (t2 < 1e-8) {
    *a = 1.0 - t2 / 6.0 + t2 * t2 / 120.0;
    *b = 0.5 - t2 / 24.0 + t2 * t2 / 720.0;
  } else {
    const double t = std::sqrt(t2);
    const double sh = std::sin(0.5 * t), ch = std::cos(0.5 * t);
    const double h = sh / t;
    *a = 2.0 * h * ch;
    *b = 2.0 * h * h;
  }
  *c = (t2 < 2.5) ? so3_c_series(t2) : (1.0 - *a) / t2;
}
// R = Exp(w) = I + a w^ + b w^^2
inline void so3_exp(const double* w, double* R) {
  double a, b, c;
  const double t2 = v3_dot(w, w);
  so3_coeffs(t2, &a, &b, &c);
  double W[9], W2[9];
  hat(w, W); m3_mul(W, W, W2);
  for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0 ? 1.0 : 0.0) + a * W[i] + b * W2[i];
}
// Right Jacobian Jr(w) = I - b w^ + c w^^2   (Exp(w+dw) = Exp(w) Exp(Jr dw))
inline void so3_Jr(const double* w, double* J) {
  double a, b, c;
  const double t2 = v3_dot(w, w);
  so3_coeffs(t2, &a, &b, &c);
  double W[9], W2[9];
  hat(w, W); m3_mul(W, W, W2);
  for (int i = 0; i < 9; ++i) J[i] = (i % 4 == 0 ? 1.0 : 0.0) - b * W[i] + c * W2[i];
}
// Inverse right Jacobian Jr^{-1}(w) = I + 1/2 w^ + e w^^2, e = 1/t^2 - (1+cos t)/(2 t sin t)
inline void so3_Jr_inv(const double* w, double* J) {
  const double t2 = v3_dot(w, w);
  double e;
  if (t2 < 4.0) {
    e = so3_e_series(t2);
  } else {
    const double t = std::sqrt(t2);
    e = (1.0 - 0.5 * t * std::cos(0.5 * t) / std::sin(0.5 * t)) / t2;   // (1 + cos t)/sin t = cot(t/2)
  }
  double W[9], W2[9];
  hat(w, W); m3_mul(W, W, W2);
  for (int i = 0; i < 9; ++i) J[i] = (i % 4 == 0 ? 1.0 : 0.0) + 0.5 * W[i] + e * W2[i];
}

// General dense helpers (row-major): C(m x n) = A(m x k) * B(k x n)
inline void mat_mul(const double* A, const double* B, double* C, int m, int k, int n) {
  for (int i = 0; i < m; ++i)
    for (int j = 0; j < n; ++j) {
      double s = 0;
      for (int l = 0; l < k; ++l) s += A[i * k + l] * B[l * n + j];
      C[i * n + j] = s;
    }
}

}  // namespace ho
