// The split cumulative spline at a stamp (sm_90a): the knot-table segment and basis, the forward sweep
// P <- P Exp(lam_j d_j), p += lam_j (p_j - p_{j-1}), the rotation Jacobian blocks M_j = lam_j P_j Jr(lam_j d_j) G_j and
// the body-rate recursion.  Every kernel that reads the trajectory at a stamp builds on these, so the factor passes,
// the calibration blocks, the stereo ingest and the stamp covariances all round the same way.
#pragma once
#include "hb200_math.cuh"
#include "hb200_types.cuh"

namespace hb {

// Basis evaluation (Horner), lam[0] = 1, lam[K] = 0.
template <int K, bool DERIV>
HB_DI void basis_eval(const Basis& b, double u, double inv_dt, double* lam, double* lamd, double* lamdd) {
  lam[0] = 1.0; lam[K] = 0.0;
  if (DERIV) { lamd[0] = lamdd[0] = 0.0; lamd[K] = lamdd[K] = 0.0; }
#pragma unroll
  for (int j = 1; j < K; ++j) {
    double v = 0, d1 = 0, d2 = 0;
#pragma unroll
    for (int n = K - 1; n >= 0; --n) {
      if (DERIV) { d2 = d2 * u + 2.0 * d1; d1 = d1 * u + v; }
      v = v * u + b.Mc[j * K + n];
    }
    lam[j] = v;
    if (DERIV) { lamd[j] = d1 * inv_dt; lamdd[j] = d2 * inv_dt * inv_dt; }
  }
}

// Knot-table rows of the segment of control points base .. base + K - 1 at stamp t: returns row 0 and evaluates the
// basis lam (with DERIV, also its first and second time derivatives lamd, lamdd).
template <int K, bool DERIV = false>
HB_DI const double* spline_segment(const double* tab, const Basis& B, int base, double t, double* lam, double* lamd = nullptr,
                                   double* lamdd = nullptr) {
  constexpr int left = (K - 1) / 2;
  const double* row0 = tab + static_cast<size_t>(base) * kTabStride;
  const double t0 = row0[left * kTabStride + 24], t1 = row0[(left + 1) * kTabStride + 24];
  const double inv_dt = 1.0 / (t1 - t0);
  basis_eval<K, DERIV>(B, (t - t0) * inv_dt, inv_dt, lam, lamd, lamdd);
  return row0;
}

// Step j of the forward sweep: A = Exp(lam_j d_j) and, with Jr, Jr(lam_j d_j)   (rj: knot-table row j of the segment)
HB_DI void spline_step_exp(const double* rj, double lj, double* A, double* Jr) {
  const double w[3] = {lj * rj[12], lj * rj[13], lj * rj[14]};
  so3_exp_and_Jr(w, A, Jr);
}

// Rotation block of step j: M_j = lam_j P_j Jr_j G_j   (P_j: pose rotation after step j)
HB_DI void pixel_step_block(const double* rj, double lj, const double* Pj, const double* Jr, double* M) {
  double G[9], JG[9], PJG[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) G[i] = rj[15 + i];
  m3_mul(Jr, G, JG);
  m3_mul(Pj, JG, PJG);
#pragma unroll
  for (int i = 0; i < 9; ++i) M[i] = lj * PJG[i];
}

// Body-rate recursion of step j: aw = A_j^T w, awd = A_j^T wd, then w <- aw + lamd_j d_j, wd <- awd + lamd_j (w x d_j) + lamdd_j d_j
HB_DI void inertial_rate_step(const double* A, const double* d, double ld, double ldd, double* w, double* wd, double* aw, double* awd) {
  double wn[3], cr[3];
  m3_tvec(A, w, aw);
  m3_tvec(A, wd, awd);
#pragma unroll
  for (int c = 0; c < 3; ++c) wn[c] = aw[c] + ld * d[c];
  cross(wn, d, cr);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    wd[c] = awd[c] + ld * cr[c] + ldd * d[c];
    w[c] = wn[c];
  }
}

// Pose at the stamp: R (row-major) into P, p; with WANT_M also M_j into M[(j - 1) * 9], j = 1 .. K - 1.
template <int K, bool WANT_M>
HB_DI void spline_pose(const double* row0, const double* lam, double* P, double* p, double* M) {
#pragma unroll
  for (int i = 0; i < 9; ++i) P[i] = row0[i];
  p[0] = row0[9]; p[1] = row0[10]; p[2] = row0[11];
#pragma unroll
  for (int j = 1; j < K; ++j) {
    const double* rj = row0 + j * kTabStride;
    double A[9], Jr[9], Pn[9];
    spline_step_exp(rj, lam[j], A, WANT_M ? Jr : nullptr);
    m3_mul(P, A, Pn);
    if (WANT_M) pixel_step_block(rj, lam[j], Pn, Jr, &M[(j - 1) * 9]);
#pragma unroll
    for (int i = 0; i < 9; ++i) P[i] = Pn[i];
#pragma unroll
    for (int c = 0; c < 3; ++c) p[c] += lam[j] * (rj[9 + c] - rj[9 + c - kTabStride]);
  }
}

// d theta / d phi_m of the pose at the stamp (global rotation tangent): D_m = M_m - M_{m+1}, M_0 = I, M_K = 0.
template <int K>
HB_DI void pose_theta_block(const double* M, int m, double* D) {
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    const double cur = (m == 0) ? ((i % 4 == 0) ? 1.0 : 0.0) : M[(m - 1) * 9 + i];
    const double nxt = (m + 1 < K) ? M[m * 9 + i] : 0.0;
    D[i] = cur - nxt;
  }
}

}  // namespace hb
