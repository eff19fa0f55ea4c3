// TEST INFRASTRUCTURE ONLY (see ho_math.h header).  PARITY UNPINNED.
//
// Ingest step in front of the hot path (SURVEY.md section 8f rank 4): what AbstractOptimizer::process(
// VisualTracks) does per stereo frame before it adds bearing factors (reference
// internal/hyper/optimizers/abstract.cpp:186-264):
//   B = C.convertPixelsToBearings(PX)                 (:221-223)
//   p_0 = Camera::Triangulate(T_01, B0[i], B1[i])     (:252)   with T_01 = T_b0^-1 (+) T_b1 (:204)
//   landmark = T_w0.vectorPlus(p_0)                    (:253)   with T_w0 = T_wb(stamp) (+) T_b0 (:203)
// Both camera functions live in HyperSensors (not in the tree): [INFERRED]
//   * pixel -> bearing: denormalise, invert the radial-tangential distortion (Newton on the 2x2 system, the
//     forward model and its Jacobian are the ones of the pixel evaluator), normalise [x y 1];
//   * Triangulate: midpoint of the common perpendicular of the two rays, in the frame of camera 0.
// Pinned by properties only: distort(undistort(d)) = d, and exactness on noise-free rays.
#pragma once
#include "ho_evaluators.h"

namespace ho {

// pixel -> unit bearing in the sensor frame; cam = [T_bs(7) | cx cy fx fy | k1 k2 p1 p2]
inline void pixel_to_bearing(const double* cam, const double* px, double* b) {
  const double* in = cam + 7;
  const double* ds = cam + 11;
  const double d[2] = {(px[0] - in[0]) / in[2], (px[1] - in[1]) / in[3]};
  double nrm[2] = {d[0], d[1]};
  for (int it = 0; it < 10; ++it) {
    double o[2], J[4];
    radtan_distort(ds, nrm, o, J, nullptr);
    const double e0 = o[0] - d[0], e1 = o[1] - d[1];
    const double det = J[0] * J[3] - J[1] * J[2];
    nrm[0] -= (J[3] * e0 - J[1] * e1) / det;
    nrm[1] -= (-J[2] * e0 + J[0] * e1) / det;
  }
  const double inv = 1.0 / std::sqrt(nrm[0] * nrm[0] + nrm[1] * nrm[1] + 1.0);
  b[0] = nrm[0] * inv; b[1] = nrm[1] * inv; b[2] = inv;
}

// midpoint triangulation in the frame of camera 0: rays s b0 and t_01 + u R_01 b1, closest points from n = b0 x d1
// (s = ((t x d1) . n) / |n|^2, u = ((t x b0) . n) / |n|^2), so the error follows depth / baseline rather than its
// square (the Gram determinant a c - b^2 = sin^2 of the parallax cancels).  Parallel rays: n = 0, non-finite point.
inline void triangulate_midpoint(const double* T_01, const double* b0, const double* b1, double* p0) {
  double R[9], d1[3], n[3], td[3], tb[3];
  quat_to_rot(T_01, R);
  m3_vec(R, b1, d1);
  const double* t = T_01 + 4;
  v3_cross(b0, d1, n);
  v3_cross(t, d1, td);
  v3_cross(t, b0, tb);
  const double inn = 1.0 / v3_dot(n, n);
  const double s = v3_dot(td, n) * inn, u = v3_dot(tb, n) * inn;
  for (int i = 0; i < 3; ++i) p0[i] = 0.5 * (s * b0[i] + t[i] + u * d1[i]);
}

// one stereo frame: bearings of both views and the triangulated world point of every track
inline void ingest_stereo_frame(const Basis& basis, const double* const* state_blocks, double stamp, const double* cam0, const double* cam1,
                                int n, const double* px0, const double* px1, double* B0, double* B1, double* landmarks) {
  StateResult S;
  state_evaluate(basis, state_blocks, stamp, 0, false, &S);
  double T_w0[7], T_0b[7], T_01[7];
  se3_group_plus(S.value, cam0, T_w0, nullptr, nullptr);
  se3_group_inverse(cam0, T_0b, nullptr);
  se3_group_plus(T_0b, cam1, T_01, nullptr, nullptr);
  for (int i = 0; i < n; ++i) {
    pixel_to_bearing(cam0, px0 + 2 * i, B0 + 3 * i);
    pixel_to_bearing(cam1, px1 + 2 * i, B1 + 3 * i);
    double p0[3];
    triangulate_midpoint(T_01, B0 + 3 * i, B1 + 3 * i, p0);
    se3_vector_plus(T_w0, p0, landmarks + 3 * i, nullptr);
  }
}

}  // namespace ho
