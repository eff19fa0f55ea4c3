// Marginal covariances of the window's estimates (hb200_build_covariance / hb200_compute_covariance), sm_90a, FP64.
//
// Sigma = (J^T W J)^-1 over the non-constant dofs at the current state, the model of ceres::Covariance with its defaults.
// The build assembles the undamped reduced system S (landmark Schur complement with mu = 0) into the packed band-only
// buffer; the kernels here then produce, from S and the landmark factors of that build:
//   cov_selinv_kernel     the entries of S^-1 on the block band, the arrow and the corner (selected inversion);
//   cov_landmark_kernel   the 3 x 3 marginal of every landmark, Sigma_ll = L^-T (I + Y^T Sigma_pp Y) L^-1;
//   cov_stamp_kernel      at arbitrary stamps, J(t) Sigma J(t)^T of the interpolated pose (6 x 6) or of the joint pose,
//                         body velocity and IMU biases (18 x 18);
//   cov_far_column_kernel / cov_cross_landmark_kernel the requested blocks outside the pattern (ceres::Covariance::Compute's
//                         list): knot pairs beyond the band and landmark cross-covariances;
//   cov_pose_pair_kernel  the joint covariance of the poses at two stamps and the covariance of their relative pose.
// All are deterministic: no atomics, every sum in a fixed order.
#pragma once
#include "hb200_solve.cuh"

namespace hb {

// Pivot threshold of the covariance factorisations.  The reduced system is factored after the symmetric diagonal
// equilibration D S D, D = diag(S)^-1/2, so a pivot is its own ratio to the diagonal; a landmark pivot is compared with
// d_j = clamp(diag V_l).  Ceres' Covariance::Options::min_reciprocal_condition_number (1e-14) is too close to rounding
// here: a system that is singular in exact arithmetic but assembled in FP64 keeps an equilibrated pivot of order n eps
// (4e-15 at n = 86 in tests/test_covref.py, ~7e-13 = n eps at K = 500), so the threshold sits at 1e-10, 150 x above
// that at K = 500 and far below the smallest pivot of the positive definite windows the tests run.
constexpr double kCovMinPivot = 1e-10;
constexpr int kCovThreads = 512;
constexpr int kCovFlagThreads = 256;

struct CovStatus {
  int status;        // 0 ok, 1 a pivot of the reduced system failed
  int bad_dof;       // first reduced-system dof whose pivot failed, else -1
  double min_pivot;  // smallest pivot of the equilibrated factor (the failing one when status = 1)
};

// Sliding window of the selected inversion: beta + 1 block slots of 6 rows (block b in slot b mod (beta + 1)) and the
// m arrow rows, stored as a full symmetric square with an odd leading dimension.
__host__ __device__ inline int cov_window(int beta, int m) { return 6 * (beta + 1) + m; }
__host__ __device__ inline int cov_ld(int w) { return w | 1; }
__host__ __device__ inline size_t cov_smem_doubles(int beta, int m) {
  const size_t w = cov_window(beta, m);
  return w * cov_ld(static_cast<int>(w)) + 3 * 6 * w + 3 * 36;
}
// global workspace: factor L in the packed P | A | C layout, D (n), L_C^-1 (m x m)
__host__ __device__ inline long long cov_packed_doubles(const SysLayout& L) { return L.oC + static_cast<long long>(L.m) * L.m; }
__host__ __device__ inline long long cov_workspace_doubles(const SysLayout& L) {
  return cov_packed_doubles(L) + L.n + static_cast<long long>(L.m) * L.m;
}

// Landmarks whose undamped V_l is not numerically positive definite (a pivot of the Schur kernels' factor at or below
// kCovMinPivot d_j; NaN-safe) and landmarks without observations.  One CTA, counts in counts[0] / counts[1].
__global__ void __launch_bounds__(kCovFlagThreads) cov_landmark_flags_kernel(int L, const int* __restrict__ lm_off, const double* __restrict__ Vchol,
                                                                             const double* __restrict__ Dl, int* __restrict__ counts) {
  int degenerate = 0, unobserved = 0;
  for (int l = threadIdx.x; l < L; l += kCovFlagThreads) {
    if (lm_off[l + 1] <= lm_off[l]) { ++unobserved; continue; }
    const double* F = Vchol + 9 * static_cast<size_t>(l);   // packed (1/L00, L10, 1/L11, L20, L21, 1/L22)
    const double* d = Dl + 3 * static_cast<size_t>(l);
    const double f[3] = {F[0], F[2], F[5]};
    bool bad = false;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const double pivot = 1.0 / (f[j] * f[j]);
      if (!(pivot > kCovMinPivot * d[j])) bad = true;
    }
    degenerate += bad ? 1 : 0;
  }
  degenerate = __reduce_add_sync(0xffffffffu, degenerate);
  unobserved = __reduce_add_sync(0xffffffffu, unobserved);
  __shared__ int s[2][kCovFlagThreads / 32];
  if ((threadIdx.x & 31) == 0) { s[0][threadIdx.x >> 5] = degenerate; s[1][threadIdx.x >> 5] = unobserved; }
  __syncthreads();
  if (threadIdx.x == 0) {
    int a = 0, b = 0;
    for (int w = 0; w < kCovFlagThreads / 32; ++w) { a += s[0][w]; b += s[1][w]; }
    counts[0] = a; counts[1] = b;
  }
}

// Sharded contexts: the rank's degenerate-landmark count goes into a tail slot of its partial packed system, which the
// system reduction then sums with everything else (one collective per build).  scal[kCovDegenerateSlot] is written by no
// other kernel of a build (cost_kernel writes scal[0] and scal[1]) and is cleared with the rest of the buffer; the sum of
// small integers is exact in any order.
constexpr int kCovDegenerateSlot = 7;
__global__ void cov_degenerate_slot_kernel(const int* __restrict__ counts, double* sys, SysLayout lay) {
  sys[lay.os + kCovDegenerateSlot] = static_cast<double>(counts[0]);
}

// Entry (i, j) of A_hat = D S D with the constant-dof mask (identity rows / columns), read from the lower triangle.
HB_DI double cov_ahat(const double* __restrict__ sys, const SysLayout& lay, const unsigned char* __restrict__ fixed, const double* __restrict__ d,
                      int i, int j) {
  if (fixed[i] || fixed[j]) return i == j ? 1.0 : 0.0;
  const int hi = max(i, j), lo = min(i, j);
  if (hi < lay.np && hi - 6 * (lo / 6) >= lay.h) return 0.0;
  return d[i] * sys[sys_index(lay, hi, lo)] * d[j];
}

// Global dof of window row p while the window holds blocks lo .. lo + beta; -1 for a slot whose block is past the window.
HB_DI int cov_gdof(int p, int lo, int nb, int wp, int K, int np) {
  if (p >= wp) return np + (p - wp);
  const int s = p / 6;
  const int b = lo + ((s - lo % nb) % nb + nb) % nb;
  return b < K ? 6 * b + (p - 6 * s) : -1;
}

// 6 x 6 lower-triangular inverse (row-major)
HB_DI void cov_tri_inv6(const double* L, double* Li) {
  for (int c = 0; c < 6; ++c) {
    for (int i = 0; i < c; ++i) Li[i * 6 + c] = 0.0;
    Li[c * 6 + c] = 1.0 / L[c * 6 + c];
    for (int i = c + 1; i < 6; ++i) {
      double s = 0.0;
      for (int l = c; l < i; ++l) s += L[i * 6 + l] * Li[l * 6 + c];
      Li[i * 6 + c] = -s / L[i * 6 + i];
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Band + arrow Cholesky of A_hat and its selected inverse, one CTA.
//   Forward: right-looking blocked Cholesky in natural order over 6-wide block columns; the window holds the trailing
//   blocks j .. j+beta and the arrow.  Per column: factor the diagonal block (pivots checked against kCovMinPivot),
//   L_Sj = A_Sj L_jj^-T, trailing update of the window, write column j of L to Lf (packed layout), then block j+beta+1
//   enters the freed slot (it has no fill from columns <= j: it is more than beta blocks from them).  Finally the corner.
//   Backward (Takahashi): Z_CC = L_C^-T L_C^-1; for j = K-1 .. 0, with S = {j+1 .. j+beta} u arrow,
//   X = L_Sj L_jj^-1, Z_Sj = -Z_SS X, Z_jj = L_jj^-T L_jj^-1 - X^T Z_Sj.  The window now holds Z over blocks j .. j+beta
//   and the arrow; every Z entry it needs is within the band.
//   Output: Sigma = D Z D in the packed P | A | C layout (diagonal blocks and corner full, padding rows 0), constant dofs 0.
// Dynamic shared memory: cov_smem_doubles(beta, m) doubles.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kCovThreads) cov_selinv_kernel(const double* __restrict__ sys, SysLayout lay, const unsigned char* __restrict__ fixed,
                                                                 double* __restrict__ ws, double* __restrict__ out, CovStatus* __restrict__ status) {
  extern __shared__ double s_cov[];
  const int K = lay.K, m = lay.m, np = lay.np, n = lay.n, h = lay.h;
  const int nb = lay.beta + 1, wp = 6 * nb, w = wp + m, ld = cov_ld(w);
  double* Wm = s_cov;                               // [w][ld]
  double* Lc = Wm + static_cast<size_t>(w) * ld;    // [w][6]  column j of L (rows of the window)
  double* Xc = Lc + 6 * w;                          // [w][6]
  double* Zc = Xc + 6 * w;                          // [w][6]
  double* Ljj = Zc + 6 * w;                         // [36]
  double* Li = Ljj + 36;                            // [36]
  double* Zjj = Li + 36;                            // [36]
  double* Lf = ws;                                  // factor, packed layout
  double* dv = ws + cov_packed_doubles(lay);        // D
  double* Yc = dv + n;                              // L_C^-1 [m][m]
  __shared__ int s_fail;
  __shared__ double s_minpiv, s_failpiv;
  const int tid = threadIdx.x;

  for (int i = tid; i < n; i += kCovThreads) {
    const double s = sys[sys_index(lay, i, i)];
    dv[i] = (fixed[i] || !(s > 0.0) || !isfinite(s)) ? 1.0 : 1.0 / sqrt(s);   // a non-positive diagonal fails at its pivot
  }
  if (tid == 0) { s_fail = -1; s_minpiv = INFINITY; s_failpiv = 0.0; }
  __syncthreads();
  for (int e = tid; e < w * w; e += kCovThreads) {
    const int p = e / w, q = e - p * w;
    const int gi = cov_gdof(p, 0, nb, wp, K, np), gj = cov_gdof(q, 0, nb, wp, K, np);
    Wm[p * ld + q] = (gi < 0 || gj < 0) ? 0.0 : cov_ahat(sys, lay, fixed, dv, gi, gj);
  }

  // ---- forward sweep ----
  for (int j = 0; j < K; ++j) {
    const int c0 = 6 * (j % nb);
    __syncthreads();
    if (tid == 0) {
      double L[36];
      for (int i = 0; i < 36; ++i) L[i] = 0.0;
      for (int k = 0; k < 6 && s_fail < 0; ++k) {
        double piv = Wm[(c0 + k) * ld + c0 + k];
        for (int l = 0; l < k; ++l) piv -= L[k * 6 + l] * L[k * 6 + l];
        if (!(piv > kCovMinPivot)) { s_fail = 6 * j + k; s_failpiv = piv; break; }
        s_minpiv = fmin(s_minpiv, piv);
        const double lkk = sqrt(piv);
        L[k * 6 + k] = lkk;
        for (int i = k + 1; i < 6; ++i) {
          double s = Wm[(c0 + i) * ld + c0 + k];
          for (int l = 0; l < k; ++l) s -= L[i * 6 + l] * L[k * 6 + l];
          L[i * 6 + k] = s / lkk;
        }
      }
      if (s_fail < 0) {
        for (int i = 0; i < 36; ++i) Ljj[i] = L[i];
        cov_tri_inv6(L, Li);
      }
    }
    __syncthreads();
    if (s_fail >= 0) break;
    // L_pj = A_pj L_jj^-T (rows of the diagonal block: L_jj itself)
    for (int e = tid; e < 6 * w; e += kCovThreads) {
      const int p = e / 6, a = e - 6 * p;
      double v = 0.0;
      if (p >= c0 && p < c0 + 6) v = Ljj[(p - c0) * 6 + a];
      else for (int b = 0; b <= a; ++b) v += Li[a * 6 + b] * Wm[p * ld + c0 + b];
      Lc[e] = v;
    }
    __syncthreads();
    for (int e = tid; e < 6 * w; e += kCovThreads) {
      const int p = e / 6, a = e - 6 * p;
      const int gi = cov_gdof(p, j, nb, wp, K, np);
      if (gi < 0) continue;
      if (gi < np) Lf[(static_cast<size_t>(j) * h + (gi - 6 * j)) * 6 + a] = Lc[e];
      else Lf[lay.oA + static_cast<size_t>(gi - np) * np + 6 * j + a] = Lc[e];
    }
    for (int e = tid; e < w * w; e += kCovThreads) {
      const int p = e / w, q = e - p * w;
      if ((p >= c0 && p < c0 + 6) || (q >= c0 && q < c0 + 6)) continue;
      const double* lp = Lc + 6 * p;
      const double* lq = Lc + 6 * q;
      double s = lp[0] * lq[0];
#pragma unroll
      for (int a = 1; a < 6; ++a) s += lp[a] * lq[a];
      Wm[p * ld + q] -= s;
    }
    __syncthreads();
    // block j + beta + 1 enters slot j % nb (zero past the window)
    const int nbk = j + nb;
    for (int e = tid; e < 6 * w; e += kCovThreads) {
      const int a = e / w, q = e - a * w;
      const bool in_slot = q >= c0 && q < c0 + 6;
      double v = 0.0;
      if (nbk < K) {
        const int gj = in_slot ? 6 * nbk + (q - c0) : cov_gdof(q, j + 1, nb, wp, K, np);
        if (gj >= 0) v = cov_ahat(sys, lay, fixed, dv, 6 * nbk + a, gj);
      }
      Wm[(c0 + a) * ld + q] = v;
      if (!in_slot) Wm[q * ld + c0 + a] = v;
    }
  }
  __syncthreads();

  // ---- corner: right-looking Cholesky in place (lower triangle) ----
  for (int k = 0; k < m && s_fail < 0; ++k) {
    const int kk = wp + k;
    if (tid == 0) {
      const double piv = Wm[kk * ld + kk];
      if (!(piv > kCovMinPivot)) { s_fail = np + k; s_failpiv = piv; }
      else { s_minpiv = fmin(s_minpiv, piv); Wm[kk * ld + kk] = sqrt(piv); }
    }
    __syncthreads();
    if (s_fail >= 0) break;
    const double lkk = Wm[kk * ld + kk];
    for (int i = kk + 1 + tid; i < w; i += kCovThreads) Wm[i * ld + kk] /= lkk;
    __syncthreads();
    const int r = m - k - 1;
    for (int e = tid; e < r * r; e += kCovThreads) {
      const int i = kk + 1 + e / r, l = kk + 1 + e % r;
      if (l <= i) Wm[i * ld + l] -= Wm[i * ld + kk] * Wm[l * ld + kk];
    }
    __syncthreads();
  }
  if (s_fail >= 0) {
    if (tid == 0) { status->status = 1; status->bad_dof = s_fail; status->min_pivot = s_failpiv; }
    return;
  }
  // L_C^-1, one column per thread
  for (int t = tid; t < m; t += kCovThreads) {
    for (int i = 0; i < t; ++i) Yc[i * m + t] = 0.0;
    for (int i = t; i < m; ++i) {
      double s = (i == t) ? 1.0 : 0.0;
      for (int l = t; l < i; ++l) s -= Wm[(wp + i) * ld + wp + l] * Yc[l * m + t];
      Yc[i * m + t] = s / Wm[(wp + i) * ld + wp + i];
    }
  }
  __syncthreads();
  // the window becomes Z: corner Z_CC = L_C^-T L_C^-1, pose slots 0 (blocks past the window)
  for (int e = tid; e < w * w; e += kCovThreads) {
    const int p = e / w, q = e - p * w;
    double v = 0.0;
    if (p >= wp && q >= wp) {
      const int a = p - wp, b = q - wp;
      for (int k = max(a, b); k < m; ++k) v += Yc[k * m + a] * Yc[k * m + b];
      const int gi = np + a, gj = np + b;
      out[lay.oC + static_cast<size_t>(a) * m + b] = (fixed[gi] || fixed[gj]) ? 0.0 : dv[gi] * v * dv[gj];
    }
    Wm[p * ld + q] = v;
  }

  // ---- backward sweep (Takahashi) ----
  for (int j = K - 1; j >= 0; --j) {
    const int c0 = 6 * (j % nb);
    __syncthreads();
    for (int e = tid; e < 6 * w; e += kCovThreads) {
      const int p = e / 6, a = e - 6 * p;
      const int gi = cov_gdof(p, j, nb, wp, K, np);
      double v = 0.0;
      if (gi >= 0) v = gi < np ? Lf[(static_cast<size_t>(j) * h + (gi - 6 * j)) * 6 + a] : Lf[lay.oA + static_cast<size_t>(gi - np) * np + 6 * j + a];
      if (p >= c0 && p < c0 + 6) { Ljj[(p - c0) * 6 + a] = v; v = 0.0; }
      Lc[e] = v;
    }
    __syncthreads();
    if (tid == 0) cov_tri_inv6(Ljj, Li);
    __syncthreads();
    // X = L_Sj L_jj^-1
    for (int e = tid; e < 6 * w; e += kCovThreads) {
      const int p = e / 6, a = e - 6 * p;
      double v = 0.0;
      for (int b = a; b < 6; ++b) v += Lc[6 * p + b] * Li[b * 6 + a];
      Xc[e] = v;
    }
    __syncthreads();
    // Z_Sj = -Z_SS X (the slot of j holds stale entries; its rows of X are 0)
    for (int e = tid; e < 6 * w; e += kCovThreads) {
      const int p = e / 6, a = e - 6 * p;
      double v = 0.0;
      if (!(p >= c0 && p < c0 + 6)) {
        const double* zr = Wm + static_cast<size_t>(p) * ld;
        for (int q = 0; q < w; ++q) v += zr[q] * Xc[6 * q + a];
        v = -v;
      }
      Zc[e] = v;
    }
    __syncthreads();
    // Z_jj = L_jj^-T L_jj^-1 - X^T Z_Sj (lower triangle computed, mirrored)
    if (tid < 36) {
      const int a = tid / 6, b = tid - 6 * a;
      if (b <= a) {
        double s = 0.0, t = 0.0;
        for (int k = a; k < 6; ++k) s += Li[k * 6 + a] * Li[k * 6 + b];
        for (int p = 0; p < w; ++p) t += Xc[6 * p + a] * Zc[6 * p + b];
        Zjj[a * 6 + b] = s - t;
        Zjj[b * 6 + a] = s - t;
      }
    }
    __syncthreads();
    // slot of j <- column j of Z; column j of Sigma to the output
    for (int e = tid; e < 6 * w; e += kCovThreads) {
      const int p = e / 6, a = e - 6 * p;
      const bool in_slot = p >= c0 && p < c0 + 6;
      const double v = in_slot ? Zjj[(p - c0) * 6 + a] : Zc[e];
      Wm[p * ld + c0 + a] = v;
      if (!in_slot) Wm[(c0 + a) * ld + p] = v;
      const int gj = 6 * j + a;
      const int gi = cov_gdof(p, j, nb, wp, K, np);
      const double sv = (gi < 0 || fixed[gi] || fixed[gj]) ? 0.0 : dv[gi] * v * dv[gj];
      if (p >= wp) out[lay.oA + static_cast<size_t>(p - wp) * np + gj] = sv;
      else {
        const int off = ((p / 6 - j % nb) % nb + nb) % nb;   // block offset from j (rows past the last pose dof: padding)
        out[(static_cast<size_t>(j) * h + 6 * off + p % 6) * 6 + a] = sv;
      }
    }
  }
  __syncthreads();
  if (tid == 0) { status->status = 0; status->bad_dof = -1; status->min_pivot = s_minpiv; }
}

// ---------------------------------------------------------------------------------------------
// Landmark marginals, one warp per landmark (the observation loop of lm_backsub_kernel / schur_group_kernel):
//   W = sum w Jp^T Jl over the landmark's control-point span, Y = W L^-T with the build's undamped factor V_l = L L^T,
//   M = Y^T Sigma_pp Y (Sigma_pp from the selected inverse: the span lies inside the band),
//   Sigma_ll = L^-T (I + M) L^-1 = V^-1 + V^-1 W^T Sigma_pp W V^-1.
// Unobserved landmarks get a zero block.  Nothing runs when the selected inversion failed.
// Dynamic shared memory: kLmWarps * 3 * max_rows doubles.
// ---------------------------------------------------------------------------------------------
// Y = W L^-T of an observed landmark into the warp's buffer Y (rows x 3, rows = 6 x its control-point span; the
// observations' first control points are ascending) and its packed factor into F.  Returns the span's first control point.
template <int K>
HB_DI int cov_landmark_Y(int o_lo, int o_hi, const int* __restrict__ lm_obs, const int4* __restrict__ idx, const double* __restrict__ Jp,
                         const double* __restrict__ Jl, const double* __restrict__ wv, const double* __restrict__ Vl, double* Y, int* rows_out,
                         double* F) {
  constexpr int NB = 6 * K;
  const int lane = threadIdx.x & 31;
  const int cp_lo = idx[lm_obs[o_lo]].x, cp_hi = idx[lm_obs[o_hi - 1]].x + K;
  const int rows = 6 * (cp_hi - cp_lo);
  *rows_out = rows;
  for (int e = lane; e < 3 * rows; e += 32) Y[e] = 0.0;
  __syncwarp();
  for (int ob = o_lo; ob < o_hi; ++ob) {
    const int f = lm_obs[ob];
    const double wgt = wv[f];
    const int b0 = 6 * (idx[f].x - cp_lo);
    const double* jp = Jp + static_cast<size_t>(f) * 2 * NB;
    const double* jl = Jl + 6 * static_cast<size_t>(f);
    for (int a = lane; a < NB; a += 32) {
      const double j0 = wgt * jp[a], j1 = wgt * jp[NB + a];
      double* wr = Y + 3 * (b0 + a);
      wr[0] += j0 * jl[0] + j1 * jl[3];
      wr[1] += j0 * jl[1] + j1 * jl[4];
      wr[2] += j0 * jl[2] + j1 * jl[5];
    }
    __syncwarp();
  }
#pragma unroll
  for (int i = 0; i < 6; ++i) F[i] = Vl[i];
  for (int r = lane; r < rows; r += 32) {
    double y[3];
    lm_lsolve(F, Y[3 * r], Y[3 * r + 1], Y[3 * r + 2], y);
    Y[3 * r] = y[0]; Y[3 * r + 1] = y[1]; Y[3 * r + 2] = y[2];
  }
  __syncwarp();
  return cp_lo;
}

// L^-1 (row-major 3 x 3, lower) of a packed landmark factor, columns L^-1 e_c
HB_DI void cov_landmark_Linv(const double* F, double* Li) {
  double y[3];
  lm_lsolve(F, 1.0, 0.0, 0.0, y); Li[0] = y[0]; Li[3] = y[1]; Li[6] = y[2];
  lm_lsolve(F, 0.0, 1.0, 0.0, y); Li[1] = y[0]; Li[4] = y[1]; Li[7] = y[2];
  lm_lsolve(F, 0.0, 0.0, 1.0, y); Li[2] = y[0]; Li[5] = y[1]; Li[8] = y[2];
}

template <int K>
__global__ void __launch_bounds__(kLmWarps * 32) cov_landmark_kernel(int L, const int* __restrict__ lm_off, const int* __restrict__ lm_obs,
                                                                     const int4* __restrict__ idx, const double* __restrict__ Jp,
                                                                     const double* __restrict__ Jl, const double* __restrict__ wv,
                                                                     const double* __restrict__ Vchol, const double* __restrict__ cov, SysLayout lay,
                                                                     const CovStatus* __restrict__ status, double* __restrict__ out, int max_rows) {
  extern __shared__ double s_lw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int l = blockIdx.x * kLmWarps + warp;
  if (status->status != 0 || l >= L) return;
  double* Y = s_lw + static_cast<size_t>(warp) * 3 * max_rows;
  double* o = out + 9 * static_cast<size_t>(l);
  const int o_lo = lm_off[l], o_hi = lm_off[l + 1];
  if (o_lo >= o_hi) {
    if (lane < 9) o[lane] = 0.0;
    return;
  }
  double F[6];
  int rows;
  const int cp_lo = cov_landmark_Y<K>(o_lo, o_hi, lm_obs, idx, Jp, Jl, wv, Vchol + 9 * static_cast<size_t>(l), Y, &rows, F);
  double M[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  const int g0 = 6 * cp_lo;
  for (int r = lane; r < rows; r += 32) {
    double t[3] = {0, 0, 0};
    const int gr = g0 + r;
    for (int s = 0; s < rows; ++s) {
      const int gs = g0 + s;
      const double z = cov[sys_index(lay, max(gr, gs), min(gr, gs))];
      t[0] += z * Y[3 * s]; t[1] += z * Y[3 * s + 1]; t[2] += z * Y[3 * s + 2];
    }
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 3; ++b) M[3 * a + b] += Y[3 * r + a] * t[b];
  }
#pragma unroll
  for (int i = 0; i < 9; ++i)
#pragma unroll
    for (int x = 16; x > 0; x >>= 1) M[i] += __shfl_xor_sync(0xffffffffu, M[i], x);
  if (lane == 0) {
    double Li[9];
    cov_landmark_Linv(F, Li);
    double A[9], T[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) A[i] = 0.5 * (M[i] + M[3 * (i % 3) + i / 3]) + ((i % 4 == 0) ? 1.0 : 0.0);
    m3_mul(A, Li, T);        // (I + M) L^-1
    double S[9];
    m3_tmul(Li, T, S);       // L^-T (I + M) L^-1
#pragma unroll
    for (int i = 0; i < 9; ++i) o[i] = 0.5 * (S[i] + S[3 * (i % 3) + i / 3]);
  }
}

// ---------------------------------------------------------------------------------------------
// Covariance blocks outside the selected inverse's pattern (hb200_set_covariance_blocks), computed inside the compute
// from its factor and its Sigma.  A request is a pair of parameter blocks (kind, index); kinds as HB200_COV_*.
// ---------------------------------------------------------------------------------------------
enum { kCovKnot = 0, kCovGyroBias = 1, kCovAccelBias = 2, kCovGravity = 3, kCovLandmark = 4 };
constexpr int kFarThreads = 64;

// First reduced-system dof and device tangent size of a non-landmark block.
HB_DI void cov_block_dofs(int kind, int index, const SysLayout& lay, int Kbg, int* dof, int* t) {
  if (kind == kCovKnot) { *dof = 6 * index; *t = 6; }
  else if (kind == kCovGyroBias) { *dof = lay.np + 3 * index; *t = 3; }
  else if (kind == kCovAccelBias) { *dof = lay.np + 3 * Kbg + 3 * index; *t = 3; }
  else { *dof = lay.n - 2; *t = 2; }
}

// The far-column plan, one int array: slot[K] (column block -> slot, -1: none), then per slot its column block, its
// lowest row block lo and its first scratch block; the scratch holds Sigma_ij of rows i = lo .. j - beta - 1 (6 x 6 each,
// row-major, rows of block i) at block off + (i - lo).
struct CovFarPlan {
  const int* p;
  int nc;
  HB_DI int slot(int j) const { return p[j]; }
};

// Sigma entry (ga, gb) of two non-landmark dofs: the packed Sigma inside the band, the arrow and the corner, the far
// scratch for knot pairs more than beta blocks apart (which the plan covers).
HB_DI double cov_sigma(const double* __restrict__ cov, const double* __restrict__ far, const CovFarPlan& plan, const SysLayout& lay, int ga, int gb) {
  const int hi = max(ga, gb), lo = min(ga, gb);
  if (hi < lay.np) {
    const int bh = hi / 6, bl = lo / 6;
    if (bh - bl > lay.beta) {
      const int s = plan.slot(bh);
      const int blk = plan.p[lay.K + 2 * plan.nc + s] + (bl - plan.p[lay.K + plan.nc + s]);
      return far[static_cast<size_t>(blk) * 36 + 6 * (lo - 6 * bl) + (hi - 6 * bh)];
    }
  }
  return cov[sys_index(lay, hi, lo)];
}

// Control-point span [first, end) of the landmark on each side of every request, (-1, -1) for a non-landmark side or a
// landmark without observations.  One thread per request.
__global__ void cov_landmark_span_kernel(int n, const int4* __restrict__ req, const int* __restrict__ lm_off, const int* __restrict__ lm_obs,
                                         const int4* __restrict__ idx, int k, int2* __restrict__ span) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  const int4 r = req[q];
  const int kind[2] = {r.x, r.z}, index[2] = {r.y, r.w};
  for (int s = 0; s < 2; ++s) {
    int2 v = make_int2(-1, -1);
    if (kind[s] == kCovLandmark) {
      const int o_lo = lm_off[index[s]], o_hi = lm_off[index[s] + 1];
      if (o_lo < o_hi) v = make_int2(idx[lm_obs[o_lo]].x, idx[lm_obs[o_hi - 1]].x + k);
    }
    span[2 * q + s] = v;
  }
}

// ---------------------------------------------------------------------------------------------
// Knot columns beyond the band, one CTA per planned column block j.  Z = A_hat^-1 (A_hat = D S D) satisfies
// L^T Z = L^-1, whose column j is zero above block j, so for i < j - beta (L_ki = 0 for k > i + beta):
//   Z_ij = -L_ii^-T ( sum_{k=i+1..i+beta} L_ki^T Z_kj + L_Ci^T Z_Cj ),
// with L the factor cov_selinv_kernel left in the workspace.  Seeds: Z_kj (j - beta <= k < j) and the arrow Z_Cj,
// unscaled from the packed Sigma just computed (constant dofs: Sigma = 0 = Z off the diagonal, and their factor rows
// and columns are those of the identity).  The CTA marches i down to the plan's lo with a ring of beta blocks in
// shared memory and writes Sigma_ij = D Z D (constant dofs 0) to the scratch.  Every sum in a fixed order.
// Dynamic shared memory: 36 beta + 6 m + 36 doubles.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kFarThreads) cov_far_column_kernel(const double* __restrict__ ws, const double* __restrict__ cov, SysLayout lay,
                                                                     const unsigned char* __restrict__ fixed, CovFarPlan plan,
                                                                     const CovStatus* __restrict__ status, double* __restrict__ far) {
  extern __shared__ double s_far[];
  if (status->status != 0) return;
  const int beta = lay.beta, m = lay.m, np = lay.np, h = lay.h;
  const int s = blockIdx.x;
  const int j = plan.p[lay.K + s], lo = plan.p[lay.K + plan.nc + s], off = plan.p[lay.K + 2 * plan.nc + s];
  const double* Lf = ws;
  const double* dv = ws + cov_packed_doubles(lay);
  double* ring = s_far;            // [beta][6][6]: Z_kj in slot k mod beta
  double* Zc = ring + 36 * beta;   // [m][6]
  double* T = Zc + 6 * m;          // [6][6]
  const int tid = threadIdx.x;
  for (int e = tid; e < 36 * beta; e += kFarThreads) {
    const int k = j - beta + e / 36, r = (e % 36) / 6, c = e % 6;
    const int gi = 6 * k + r, gj = 6 * j + c;
    ring[36 * (k % beta) + 6 * r + c] = cov[sys_index(lay, gj, gi)] / (dv[gi] * dv[gj]);
  }
  for (int e = tid; e < 6 * m; e += kFarThreads) {
    const int p = e / 6, c = e % 6;
    Zc[e] = cov[lay.oA + static_cast<size_t>(p) * np + 6 * j + c] / (dv[np + p] * dv[6 * j + c]);
  }
  __syncthreads();
  for (int i = j - beta - 1; i >= lo; --i) {
    const size_t col = static_cast<size_t>(i) * h * 6;   // column block i of the factor: row q of block k at (6 (k - i) + q) * 6
    if (tid < 36) {
      const int r = tid / 6, c = tid % 6;
      double t = 0.0;
      for (int k = i + 1; k <= i + beta; ++k) {
        const double* Lk = Lf + col + 36 * (k - i);
        const double* Zk = ring + 36 * (k % beta);
#pragma unroll
        for (int q = 0; q < 6; ++q) t += Lk[6 * q + r] * Zk[6 * q + c];
      }
      const double* LC = Lf + lay.oA + 6 * i + r;
      for (int p = 0; p < m; ++p) t += LC[static_cast<size_t>(p) * np] * Zc[6 * p + c];
      T[tid] = t;
    }
    __syncthreads();
    if (tid < 6) {   // Z_ij = -L_ii^-T T, one column per thread (L_ii^T is upper triangular)
      const double* Li = Lf + col;
      double x[6];
#pragma unroll
      for (int r = 5; r >= 0; --r) {
        double v = T[6 * r + tid];
#pragma unroll
        for (int q = r + 1; q < 6; ++q) v -= Li[6 * q + r] * x[q];
        x[r] = v / Li[6 * r + r];
      }
      double* Zi = ring + 36 * (i % beta);
#pragma unroll
      for (int r = 0; r < 6; ++r) Zi[6 * r + tid] = -x[r];
    }
    __syncthreads();
    if (tid < 36) {
      const int gi = 6 * i + tid / 6, gj = 6 * j + tid % 6;
      const double v = ring[36 * (i % beta) + tid];
      far[(static_cast<size_t>(off) + (i - lo)) * 36 + tid] = (fixed[gi] || fixed[gj]) ? 0.0 : dv[gi] * v * dv[gj];
    }
  }
}

// ---------------------------------------------------------------------------------------------
// The requested blocks, one warp per request, written as t_a x t_b (row-major) into the top-left of a 6 x 6 slot, the
// rest 0.  A request is taken in a canonical order -- a landmark first, the smaller landmark index first -- and written
// transposed when it was given the other way round, so (b, a) is exactly the transpose of (a, b).
//   non-landmark pairs: gathered from the packed Sigma (in the pattern: bit for bit) or the far scratch;
//   landmark l with itself: its marginal, bit for bit;
//   landmark l x knot / bias / gravity q: Sigma_lq = -V_l^-1 W_l^T Sigma_{span(l), q} = -L_l^-T Y_l^T Sigma_{span(l), q};
//   landmarks l != m: Sigma_lm = V_l^-1 W_l^T Sigma_{span(l), span(m)} W_m V_m^-1 = L_l^-T Y_l^T Sigma Y_m L_m^-1;
// with W_l, Y_l = W_l L_l^-T and the undamped factor V_l = L_l L_l^T of the build (cov_landmark_Y).  A landmark
// without observations gives a zero block and status 2, or 1 on a sharded context (its observations are on its owner).
// Lane sums are combined by a fixed butterfly.  Dynamic shared memory: kLmWarps * 6 * max_rows doubles.
// ---------------------------------------------------------------------------------------------
template <int K>
__global__ void __launch_bounds__(kLmWarps * 32) cov_cross_landmark_kernel(
    int n, const int4* __restrict__ req, const int* __restrict__ lm_off, const int* __restrict__ lm_obs, const int4* __restrict__ idx,
    const double* __restrict__ Jp, const double* __restrict__ Jl, const double* __restrict__ wv, const double* __restrict__ Vchol,
    const double* __restrict__ cov, const double* __restrict__ lmcov, const double* __restrict__ far, CovFarPlan plan, SysLayout lay, int Kbg,
    int sharded, const CovStatus* __restrict__ status, int max_rows, double* __restrict__ out, int* __restrict__ out_status) {
  extern __shared__ double s_cw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q = blockIdx.x * kLmWarps + warp;
  if (status->status != 0 || q >= n) return;
  double* o = out + 36 * static_cast<size_t>(q);
  const int4 r = req[q];
  int ka = r.x, ia = r.y, kb = r.z, ib = r.w;
  if (ka != kCovLandmark && kb != kCovLandmark) {
    int ga, ta, gb, tb;
    cov_block_dofs(ka, ia, lay, Kbg, &ga, &ta);
    cov_block_dofs(kb, ib, lay, Kbg, &gb, &tb);
    for (int e = lane; e < 36; e += 32) {
      const int a = e / 6, b = e % 6;
      o[e] = (a < ta && b < tb) ? cov_sigma(cov, far, plan, lay, ga + a, gb + b) : 0.0;
    }
    if (lane == 0) out_status[q] = 0;
    return;
  }
  const bool swap = ka != kCovLandmark || (kb == kCovLandmark && ib < ia);
  if (swap) { const int k0 = ka, i0 = ia; ka = kb; ia = ib; kb = k0; ib = i0; }
  // canonical: a is landmark ia; b is landmark ib or block (gb, tb)
  const bool pair = kb == kCovLandmark;
  const int oa_lo = lm_off[ia], oa_hi = lm_off[ia + 1];
  const int ob_lo = pair ? lm_off[ib] : 0, ob_hi = pair ? lm_off[ib + 1] : 1;
  double R[18];   // canonical block, 3 x tb (row stride 6)
#pragma unroll
  for (int i = 0; i < 18; ++i) R[i] = 0.0;
  int tb = 3, st = 0;
  if (oa_lo >= oa_hi || ob_lo >= ob_hi) {
    st = sharded ? 1 : 2;
    if (!pair) { int gb; cov_block_dofs(kb, ib, lay, Kbg, &gb, &tb); }
  } else if (pair && ia == ib) {
#pragma unroll
    for (int i = 0; i < 9; ++i) R[6 * (i / 3) + i % 3] = lmcov[9 * static_cast<size_t>(ia) + i];
  } else {
    double* Ya = s_cw + static_cast<size_t>(warp) * 6 * max_rows;
    double* Yb = Ya + 3 * max_rows;
    double Fa[6], Fb[6];
    int rows_a, rows_b = 0;
    const int ga0 = 6 * cov_landmark_Y<K>(oa_lo, oa_hi, lm_obs, idx, Jp, Jl, wv, Vchol + 9 * static_cast<size_t>(ia), Ya, &rows_a, Fa);
    int gb = 0;
    if (pair) gb = 6 * cov_landmark_Y<K>(ob_lo, ob_hi, lm_obs, idx, Jp, Jl, wv, Vchol + 9 * static_cast<size_t>(ib), Yb, &rows_b, Fb);
    else cov_block_dofs(kb, ib, lay, Kbg, &gb, &tb);
    // M = Y_a^T Sigma_{span(a), b} (3 x tb), b = Y_b-weighted span(b) for a landmark pair (tb = 3)
    double M[18];
#pragma unroll
    for (int i = 0; i < 18; ++i) M[i] = 0.0;
    for (int rr = lane; rr < rows_a; rr += 32) {
      const int gr = ga0 + rr;
      double t[6] = {0, 0, 0, 0, 0, 0};
      if (pair) {
        for (int s = 0; s < rows_b; ++s) {
          const double z = cov_sigma(cov, far, plan, lay, gr, gb + s);
          t[0] += z * Yb[3 * s]; t[1] += z * Yb[3 * s + 1]; t[2] += z * Yb[3 * s + 2];
        }
      } else {
#pragma unroll
        for (int c = 0; c < 6; ++c) t[c] = c < tb ? cov_sigma(cov, far, plan, lay, gr, gb + c) : 0.0;
      }
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int c = 0; c < 6; ++c) M[6 * a + c] += Ya[3 * rr + a] * t[c];
    }
#pragma unroll
    for (int i = 0; i < 18; ++i)
#pragma unroll
      for (int x = 16; x > 0; x >>= 1) M[i] += __shfl_xor_sync(0xffffffffu, M[i], x);
    if (lane == 0) {
      double La[9];
      cov_landmark_Linv(Fa, La);
      if (pair) {   // L_a^-T M L_b^-1
        double Lb[9], Mm[9], T[9], S[9];
#pragma unroll
        for (int i = 0; i < 9; ++i) Mm[i] = M[6 * (i / 3) + i % 3];
        cov_landmark_Linv(Fb, Lb);
        m3_mul(Mm, Lb, T);
        m3_tmul(La, T, S);
#pragma unroll
        for (int i = 0; i < 9; ++i) R[6 * (i / 3) + i % 3] = S[i];
      } else {      // -L_a^-T M
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
          for (int c = 0; c < 6; ++c) R[6 * a + c] = -(La[a] * M[c] + La[3 + a] * M[6 + c] + La[6 + a] * M[12 + c]);
      }
    }
  }
  if (lane == 0) {
    out_status[q] = st;
#pragma unroll
    for (int e = 0; e < 36; ++e) {
      const int a = e / 6, b = e % 6;
      double v = 0.0;
      if (!swap && a < 3 && b < tb) v = R[6 * a + b];
      if (swap && b < 3 && a < tb) v = R[6 * b + a];
      o[e] = v;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Covariance at arbitrary stamps, one warp per stamp: the pose [theta p] (ROWS = 6, hb200_interpolate_covariance) or
// the joint state x(t) = [theta p | omega v | b_g b_a] (ROWS = 18, hb200_interpolate_state_covariance).  J(t)
// (ROWS x NC) is taken with respect to the tangents [phi | rho] of the stamp's k control points (global rotation
// tangent, R <- Exp(theta) R, p <- p + rho) and, for the state, the 4 knots of each bias spline (NC = 6k + 24, columns
// 6k + 3m + c gyro, 6k + 12 + 3m + c accel; NC = 6k for the pose); Sigma(t) = J Z J^T with Z the span of the packed
// Sigma (control-point pairs in the band, pose x bias in the arrow, bias x bias in the corner).
// Jacobian blocks of control point m, with P_j = R_0 A_1 .. A_j, A_j = Exp(lambda_j d_j), G_j = Jr^-1(d_j) R_j^T:
//   theta: D_m = M_m - M_{m+1},             M_j = lambda_j P_j Jr(lambda_j d_j) G_j   (M_0 = I);  p: (lambda_m - lambda_{m+1}) I on rho_m;
//   omega: R^T (Y_m - Y_{m+1}),             Y_j = P_j X_j G_j, X_j = hat(A_j^T w_{j-1}) lambda_j Jr(lambda_j d_j) + lamd_j I
//          -- inertial_factor's rate rows X -> XG, whose left factor A_{k-1}^T .. A_{j+1}^T is R^T P_j;
//   v = R^T pdot: hat(v) R^T D_m on phi_m and (lamd_m - lamd_{m+1}) R^T on rho_m;
//   b_g / b_a: (lb_m - lb_{m+1}) I on knot gb + m / ab + m (the bias basis, as inertial_factor evaluates it).
// Lane 0 builds J in shared memory (one forward sweep, cov_stamp_jacobian); each lane then forms rows a of T = Z J^T
// from the packed Sigma and entries of J T; the output is 0.5 (S + S^T).  Sums run in a fixed order, no atomics.  The
// pose rows of the state's J are the pose J, and its bias columns only add z * 0 terms to the pose block's sums, so
// the pose block of the state covariance equals the pose covariance value for value.  A stamp outside the pose
// spline's valid span, or outside the span of a bias spline that has knots, gives a zero block and invalid[f] = 1; a
// spline without knots (Kbg or Kba = 0) gives zero rows and columns.  All inputs are the snapshot of the last compute.
// ---------------------------------------------------------------------------------------------
constexpr int kStateDim = 18;
constexpr int kStateWarps = 2;   // stamps per CTA (static shared memory: 2 x 17.5 KB at k = 6, ROWS = 18)

// Rows 0 .. ROWS - 1 of J(t) (row stride NC, zero on entry) over control points base .. base + K - 1 -- every column
// but the bias ones -- and the pose R (row-major), p at t.
template <int K, int ROWS, int NC>
HB_DI void cov_stamp_jacobian(const double* __restrict__ tab, const Basis& B, int base, double t, double* J, double* P, double* p) {
  double lam[K + 1], lamd[K + 1], lamdd[K + 1];
  const double* row0 = spline_segment<K, ROWS == kStateDim>(tab, B, base, t, lam, lamd, lamdd);
  auto add3 = [&](double* b, const double* M, double s) {   // 3 x 3 block at b += s M
    for (int i = 0; i < 3; ++i)
      for (int c = 0; c < 3; ++c) b[i * NC + c] += s * M[3 * i + c];
  };
  for (int i = 0; i < 3; ++i) J[i * NC + i] = 1.0;   // M_0 = I
  double w[3] = {0, 0, 0}, wdot[3] = {0, 0, 0}, pd[3] = {0, 0, 0};
  for (int i = 0; i < 9; ++i) P[i] = row0[i];
  p[0] = row0[9]; p[1] = row0[10]; p[2] = row0[11];
#pragma unroll 1
  for (int j = 1; j < K; ++j) {
    const double* rj = row0 + j * kTabStride;
    double A[9], Jr[9], Pn[9], M[9];
    spline_step_exp(rj, lam[j], A, Jr);
    m3_mul(P, A, Pn);
    // theta rows: + M_j on phi_j, - M_j on phi_{j-1}
    pixel_step_block(rj, lam[j], Pn, Jr, M);
    add3(J + 6 * j, M, 1.0);
    add3(J + 6 * (j - 1), M, -1.0);
    if (ROWS == kStateDim) {   // omega rows (R^T applied below): + Y_j on phi_j, - Y_j on phi_{j-1}
      const double d[3] = {rj[12], rj[13], rj[14]};
      double G[9], lj[9], X[9], XG[9], aw[3], awd[3];
      for (int i = 0; i < 9; ++i) { G[i] = rj[15 + i]; lj[i] = lam[j] * Jr[i]; }
      inertial_rate_step(A, d, lamd[j], lamdd[j], w, wdot, aw, awd);   // the J rows need aw and w only; wdot, awd go unused
      hat_mul(aw, lj, X);
      for (int i = 0; i < 3; ++i) X[4 * i] += lamd[j];
      m3_mul(X, G, XG);
      m3_mul(Pn, XG, M);
      add3(J + 6 * NC + 6 * j, M, 1.0);
      add3(J + 6 * NC + 6 * (j - 1), M, -1.0);
      for (int c = 0; c < 3; ++c) pd[c] += lamd[j] * (rj[9 + c] - rj[9 + c - kTabStride]);
    }
    for (int c = 0; c < 3; ++c) p[c] += lam[j] * (rj[9 + c] - rj[9 + c - kTabStride]);
    for (int i = 0; i < 9; ++i) P[i] = Pn[i];
  }
  // P = R: p rows w_m I; omega rows R^T (Y_m - Y_{m+1}); v rows hat(v) R^T D_m and (lamd_m - lamd_{m+1}) R^T
  double H[9];
  if (ROWS == kStateDim) {
    double v[3], Rt[9];
    m3_tvec(P, pd, v);
    for (int i = 0; i < 3; ++i)
      for (int c = 0; c < 3; ++c) Rt[3 * i + c] = P[3 * c + i];
    hat_mul(v, Rt, H);
  }
#pragma unroll 1
  for (int m = 0; m < K; ++m) {
    const double wm = lam[m] - lam[m + 1];
    for (int i = 0; i < 3; ++i) J[(3 + i) * NC + 6 * m + 3 + i] = wm;
    if (ROWS == kStateDim) {
      double* Jo = J + 6 * NC + 6 * m;   // omega block, then the v blocks three rows below
      double Y[9], Dm[9], Z[9];
      for (int i = 0; i < 3; ++i)
        for (int c = 0; c < 3; ++c) { Y[3 * i + c] = Jo[i * NC + c]; Dm[3 * i + c] = J[i * NC + 6 * m + c]; }
      m3_tmul(P, Y, Z);
      for (int i = 0; i < 3; ++i)
        for (int c = 0; c < 3; ++c) Jo[i * NC + c] = Z[3 * i + c];
      m3_mul(H, Dm, Z);
      add3(Jo + 3 * NC, Z, 1.0);
      const double wd = lamd[m] - lamd[m + 1];
      for (int i = 0; i < 3; ++i)
        for (int c = 0; c < 3; ++c) Jo[(3 + i) * NC + 3 + c] = wd * P[3 * c + i];
    }
  }
}

template <int K, int ROWS>
__global__ void __launch_bounds__(kStateWarps * 32) cov_stamp_kernel(
    int n, const double* __restrict__ stamps, const double* __restrict__ knots, const double* __restrict__ tab, int Kn, Basis B,
    const double* __restrict__ bg, int Kbg, const double* __restrict__ ba, int Kba, Basis BB, const double* __restrict__ cov,
    SysLayout lay, double* __restrict__ out, int* __restrict__ invalid) {
  static_assert(ROWS == 6 || ROWS == kStateDim, "pose or joint state rows");
  constexpr bool STATE = ROWS == kStateDim;
  constexpr int NC = 6 * K + (STATE ? 24 : 0), D = ROWS, KB = 4;
  __shared__ double s_J[kStateWarps][D * NC];   // J (row-major), then S
  __shared__ double s_T[kStateWarps][NC * D];   // T = Z J^T (row a of Z per row)
  __shared__ int s_dof[kStateWarps][NC];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f = blockIdx.x * kStateWarps + warp;
  if (f >= n) return;
  double* J = s_J[warp];
  double* T = s_T[warp];
  int* dof = s_dof[warp];
  double* o = out + D * D * static_cast<size_t>(f);
  const double t = stamps[f];
  const int base = segment_base(knots, 8, 7, Kn, K, t);
  const int gb = STATE && Kbg ? segment_base(bg, 4, 3, Kbg, KB, t) : 0;
  const int ab = STATE && Kba ? segment_base(ba, 4, 3, Kba, KB, t) : 0;
  if (base < 0 || gb < 0 || ab < 0) {
    for (int e = lane; e < D * D; e += 32) o[e] = 0.0;
    if (lane == 0) invalid[f] = 1;
    return;
  }
  if (lane == 0) invalid[f] = 0;
  for (int e = lane; e < D * NC; e += 32) J[e] = 0.0;
  for (int c = lane; c < NC; c += 32) {
    int g;
    if (c < 6 * K) g = 6 * base + c;
    else if (c < 6 * K + 12) g = Kbg ? lay.np + 3 * gb + (c - 6 * K) : -1;
    else g = Kba ? lay.np + 3 * Kbg + 3 * ab + (c - 6 * K - 12) : -1;
    dof[c] = g;
  }
  __syncwarp();
  if (lane == 0) {
    double R[9], p[3];
    cov_stamp_jacobian<K, ROWS, NC>(tab, B, base, t, J, R, p);
    // bias rows
    constexpr int lb = (KB - 1) / 2;
    double lbw[KB + 1];
    for (int s = 0; STATE && s < 2; ++s) {
      const int Kb = s ? Kba : Kbg;
      if (!Kb) continue;
      const double* b0 = (s ? ba + 4 * static_cast<size_t>(ab) : bg + 4 * static_cast<size_t>(gb));
      const double s0 = b0[4 * lb + 3], s1 = b0[4 * (lb + 1) + 3];
      basis_eval<KB, false>(BB, (t - s0) / (s1 - s0), 0.0, lbw, nullptr, nullptr);
      for (int m = 0; m < KB; ++m)
        for (int i = 0; i < 3; ++i) J[(12 + 3 * s + i) * NC + 6 * K + 12 * s + 3 * m + i] = lbw[m] - lbw[m + 1];
    }
  }
  __syncwarp();
  // T = Z J^T, one row a of Z per lane at a time, its entries read once from the packed Sigma
  for (int a = lane; a < NC; a += 32) {
    double acc[D];
#pragma unroll
    for (int r = 0; r < D; ++r) acc[r] = 0.0;
    const int ga = dof[a];
    if (ga >= 0) {
#pragma unroll 2
      for (int b = 0; b < NC; ++b) {
        const int gbb = dof[b];
        if (gbb < 0) continue;
        const double z = cov[sys_index(lay, max(ga, gbb), min(ga, gbb))];
#pragma unroll
        for (int r = 0; r < D; ++r) acc[r] += z * J[r * NC + b];
      }
    }
#pragma unroll
    for (int r = 0; r < D; ++r) T[a * D + r] = acc[r];
  }
  __syncwarp();
  // S = J T, then 0.5 (S + S^T) (S overwrites J once every lane has read it)
  constexpr int PER = (D * D + 31) / 32;
  double s[PER];
#pragma unroll
  for (int q = 0; q < PER; ++q) {
    const int e = lane + 32 * q;
    double v = 0.0;
    if (e < D * D) {
      const int r = e / D, c = e - r * D;
      for (int a = 0; a < NC; ++a) v += J[r * NC + a] * T[a * D + c];
    }
    s[q] = v;
  }
  __syncwarp();
#pragma unroll
  for (int q = 0; q < PER; ++q) {
    const int e = lane + 32 * q;
    if (e < D * D) J[e] = s[q];
  }
  __syncwarp();
  for (int e = lane; e < D * D; e += 32) {
    const int r = e / D, c = e - r * D;
    o[e] = 0.5 * (J[r * D + c] + J[c * D + r]);
  }
}

// ---------------------------------------------------------------------------------------------
// Joint and relative covariance of the poses at two stamps (hb200_set_covariance_stamp_pairs), computed inside the
// compute from its Sigma and the far scratch, at the knots the build linearised at (the snapshot knot table).
//   joint    (12 x 12) of [theta_a p_a | theta_b p_b]: blocks J_s Sigma_{span(s), span(s')} J_s'^T, J(t) the pose
//            Jacobian of cov_stamp_jacobian (global rotation tangent, p <- p + rho);
//   relative (6 x 6) of T_ab = T_a^-1 T_b (R_ab = R_a^T R_b, p_ab = R_a^T (p_b - p_a)) in the same split tangent in frame
//            a: A joint A^T with A = Rb M, Rb = diag(R_a^T, R_a^T), M = [[-I, 0, I, 0], [hat(p_b - p_a), -I, 0, I]].
// ---------------------------------------------------------------------------------------------
constexpr int kPairWarps = 2;   // pairs per CTA (static shared memory: 2 x 21 KB at k = 6)

// Control-point span bases (segment_base on the snapshot knots, -1 outside the valid span) of both stamps of each pair.
__global__ void cov_stamp_span_kernel(int n, const double* __restrict__ stamps, const double* __restrict__ knots, int Kn, int k, int2* __restrict__ span) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  span[q] = make_int2(segment_base(knots, 8, 7, Kn, k, stamps[2 * q]), segment_base(knots, 8, 7, Kn, k, stamps[2 * q + 1]));
}

// One warp per pair.  Lanes 0 and 1 build J_a and J_b (cov_stamp_jacobian, as cov_stamp_kernel<K, 6> does, whose sums
// the diagonal blocks repeat term for term); T = Z J^T over the 2 x 6k span dofs (row a of Z per lane, its
// entries gathered through cov_sigma: band, arrow and the far scratch the plan filled), S = blockdiag(J_a, J_b) T,
// joint = 0.5 (S + S^T); then E = M joint, F = E M^T, relative = 0.5 (Rb F Rb^T + (Rb F Rb^T)^T).  Swapping the stamps
// relabels the blocks of every sum without reordering its terms, so (t_b, t_a) is exactly the permutation of
// (t_a, t_b).  A stamp outside the valid span gives zero blocks and status 1.  No atomics, every sum in a fixed order.
template <int K>
__global__ void __launch_bounds__(kPairWarps * 32) cov_pose_pair_kernel(
    int n, const double* __restrict__ stamps, const int2* __restrict__ span, const double* __restrict__ tab, Basis B, const double* __restrict__ cov,
    const double* __restrict__ far, CovFarPlan plan, SysLayout lay, const CovStatus* __restrict__ status, double* __restrict__ joint,
    double* __restrict__ rel, int* __restrict__ out_status) {
  constexpr int NC = 6 * K;
  __shared__ double s_J[kPairWarps][2][6 * NC];   // J_a, J_b
  __shared__ double s_T[kPairWarps][2 * NC * 12];  // T; then S (144) and the joint (144)
  __shared__ double s_E[kPairWarps][72 + 36 + 36]; // E (6 x 12), F, H = F Rb^T
  __shared__ double s_P[kPairWarps][2][12];        // R (9) and p (3) of each stamp
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q = blockIdx.x * kPairWarps + warp;
  if (status->status != 0 || q >= n) return;
  double* jo = joint + 144 * static_cast<size_t>(q);
  double* ro = rel + 36 * static_cast<size_t>(q);
  const int2 sp = span[q];
  if (sp.x < 0 || sp.y < 0) {
    for (int e = lane; e < 144; e += 32) jo[e] = 0.0;
    for (int e = lane; e < 36; e += 32) ro[e] = 0.0;
    if (lane == 0) out_status[q] = 1;
    return;
  }
  const int base[2] = {sp.x, sp.y};
  double* T = s_T[warp];
  for (int e = lane; e < 2 * 6 * NC; e += 32) s_J[warp][e / (6 * NC)][e % (6 * NC)] = 0.0;
  __syncwarp();
  if (lane < 2) {
    double R[9], p[3];
    cov_stamp_jacobian<K, 6, NC>(tab, B, base[lane], stamps[2 * static_cast<size_t>(q) + lane], s_J[warp][lane], R, p);
    for (int i = 0; i < 9; ++i) s_P[warp][lane][i] = R[i];
    for (int c = 0; c < 3; ++c) s_P[warp][lane][9 + c] = p[c];
  }
  __syncwarp();
  for (int a = lane; a < 2 * NC; a += 32) {
    const int ga = 6 * base[a / NC] + a % NC;
    double acc[12];
#pragma unroll
    for (int c = 0; c < 12; ++c) acc[c] = 0.0;
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const double* Js = s_J[warp][s];
#pragma unroll 2
      for (int b = 0; b < NC; ++b) {
        const double z = cov_sigma(cov, far, plan, lay, ga, 6 * base[s] + b);
#pragma unroll
        for (int r = 0; r < 6; ++r) acc[6 * s + r] += z * Js[r * NC + b];
      }
    }
#pragma unroll
    for (int c = 0; c < 12; ++c) T[a * 12 + c] = acc[c];
  }
  __syncwarp();
  double sv[5];   // S = blockdiag(J_a, J_b) T, 144 entries over the lanes
#pragma unroll
  for (int u = 0; u < 5; ++u) {
    const int e = lane + 32 * u;
    double v = 0.0;
    if (e < 144) {
      const int r = e / 12, c = e % 12, s = r / 6;
      const double* Jr = s_J[warp][s] + (r % 6) * NC;
      const double* Tc = T + s * NC * 12 + c;
      for (int b = 0; b < NC; ++b) v += Jr[b] * Tc[12 * b];
    }
    sv[u] = v;
  }
  __syncwarp();
  double* S = T;
  double* Jn = T + 144;
#pragma unroll
  for (int u = 0; u < 5; ++u)
    if (lane + 32 * u < 144) S[lane + 32 * u] = sv[u];
  __syncwarp();
  for (int e = lane; e < 144; e += 32) {
    const int r = e / 12, c = e % 12;
    const double v = 0.5 * (S[e] + S[12 * c + r]);
    Jn[e] = v;
    jo[e] = v;
  }
  __syncwarp();
  const double* Ra = s_P[warp][0];
  const double dp[3] = {s_P[warp][1][9] - s_P[warp][0][9], s_P[warp][1][10] - s_P[warp][0][10], s_P[warp][1][11] - s_P[warp][0][11]};
  const double hp[9] = {0.0, -dp[2], dp[1], dp[2], 0.0, -dp[0], -dp[1], dp[0], 0.0};   // hat(p_b - p_a)
  double* E = s_E[warp];
  double* F = E + 72;
  double* H = F + 36;
  for (int e = lane; e < 72; e += 32) {   // E = M joint
    const int i = e / 12, c = e % 12;
    double v;
    if (i < 3) v = Jn[12 * (6 + i) + c] - Jn[12 * i + c];
    else v = Jn[12 * (6 + i) + c] - Jn[12 * i + c] + (hp[3 * (i - 3)] * Jn[c] + hp[3 * (i - 3) + 1] * Jn[12 + c] + hp[3 * (i - 3) + 2] * Jn[24 + c]);
    E[e] = v;
  }
  __syncwarp();
  for (int e = lane; e < 36; e += 32) {   // F = E M^T
    const int i = e / 6, j = e % 6;
    const double* Ei = E + 12 * i;
    double v;
    if (j < 3) v = Ei[6 + j] - Ei[j];
    else v = Ei[6 + j] - Ei[j] + (hp[3 * (j - 3)] * Ei[0] + hp[3 * (j - 3) + 1] * Ei[1] + hp[3 * (j - 3) + 2] * Ei[2]);
    F[e] = v;
  }
  __syncwarp();
  for (int e = lane; e < 36; e += 32) {   // H = F Rb^T: (R_a^T)^T = R_a, H_ij = sum_l F_{i, 3 bj + l} R_a[l][j % 3]
    const int i = e / 6, j = e % 6, bj = 3 * (j / 3), jj = j % 3;
    H[e] = F[6 * i + bj] * Ra[jj] + F[6 * i + bj + 1] * Ra[3 + jj] + F[6 * i + bj + 2] * Ra[6 + jj];
  }
  __syncwarp();
  for (int e = lane; e < 36; e += 32) {   // Rb H, symmetrised in registers of the lane pair (e, e^T)
    const int i = e / 6, j = e % 6;
    auto rbh = [&](int r, int c) {
      const int br = 3 * (r / 3), rr = r % 3;
      return Ra[rr] * H[6 * br + c] + Ra[3 + rr] * H[6 * (br + 1) + c] + Ra[6 + rr] * H[6 * (br + 2) + c];
    };
    ro[e] = 0.5 * (rbh(i, j) + rbh(j, i));
  }
  if (lane == 0) out_status[q] = 0;
}

}  // namespace hb
