// Shared host/device declarations for libhyperb200 (sm_90a).
#pragma once
#include <cstdint>

namespace hb {

constexpr int kMaxOrder = 6;
// Knot-table row (one per control point, rebuilt once per evaluation by prep_kernel):
//   [0..8]  R_j        rotation matrix of control point j (row-major)
//   [9..11] p_j
//   [12..14] d_j = Log(R_{j-1}^T R_j)                (row 0: zeros)
//   [15..23] G_j = Jr^{-1}(d_j) R_j^T                (row 0: zeros)
//   [24]    stamp_j ; [25..27] pad  -> 28 doubles = 224 B (16 B multiple for cp.async.bulk)
constexpr int kTabStride = 28;
constexpr int kTileRows = 16;       // knot-table rows staged per CTA (3.6 KB); wider spans read the table from global/L2
constexpr int kEvalThreads = 64;    // factors per CTA tile of the factor kernels (one per thread on large windows)

constexpr int kCamStride = 20;      // R_sb(9) t_bs(3) intrinsics(4) distortion(4)
// IMU derived table: R_sb(9) t_bs(3) IgRsb(9) IaRsb(9) Sg(9,row-major) lever arms c_r (3x3 rows) = 48, then the
// Jacobian-side copies selected by the reference-quirk switches: IlinRsb(9) SgJ(9) leverJ(9) pad = 76
constexpr int kImuStride = 76;

struct Basis {
  int k;
  double Mc[kMaxOrder * kMaxOrder];  // cumulative blending matrix, row j = coefficients of lambda_j(u)
};

// Packed reduced system, band-only (no dense n x n anywhere on the iteration path).  After the landmark Schur
// complement the pose part of S is block-banded (6x6 control-point blocks, block half-bandwidth beta = longest
// landmark track in control points, >= k-1) with an arrowhead of m = 3 Kbg + 3 Kba + 2 rows (bias knots, gravity):
//   P [K][h][6]   block column c holds rows 6c .. 6c+h-1 of columns 6c .. 6c+5 (h = 6 + 6 beta; lower triangle;
//                 rows past the last pose dof are unused)                  -- the band solver's own column layout
//   A [m][np]     arrow rows (np = 6K)        C [m][m] corner (lower)      b, diagH, g [n] each      scal [8]
// scal = [cost at the linearisation point, -, cost at the trial point, dl.g_l, dl.D_l.dl, -, -, -].  The whole
// buffer is what one all-reduce sums across ranks (K = 50, beta = 5: 20 k doubles instead of 107 k dense).
struct SysLayout {
  int n, np, m, K, h, beta;
  long long oA, oC, ob, oD, og, os, total;   // offsets in doubles
};
__host__ __device__ inline SysLayout sys_layout(int K, int beta, int m) {
  SysLayout L;
  L.K = K; L.beta = beta; L.h = 6 + 6 * beta; L.np = 6 * K; L.m = m; L.n = L.np + m;
  L.oA = static_cast<long long>(K) * L.h * 6;
  L.oC = L.oA + static_cast<long long>(m) * L.np;
  L.ob = (L.oC + static_cast<long long>(m) * m + 1) & ~1LL;
  L.oD = (L.ob + L.n + 1) & ~1LL;
  L.og = (L.oD + L.n + 1) & ~1LL;
  L.os = (L.og + L.n + 1) & ~1LL;
  L.total = L.os + 8;
  return L;
}
// index of S[row][col], row >= col (entries outside the band do not exist: the caller guarantees row - 6 (col / 6) < h)
__host__ __device__ inline long long sys_index(const SysLayout& L, int row, int col) {
  if (row < L.np) { const int c = col / 6; return (static_cast<long long>(c) * L.h + (row - 6 * c)) * 6 + (col - 6 * c); }
  if (col < L.np) return L.oA + static_cast<long long>(row - L.np) * L.np + col;
  return L.oC + static_cast<long long>(row - L.np) * L.m + (col - L.np);
}

struct SolverState {  // lives on the device; updated by accept_kernel
  double radius;
  double decrease_factor;
  double cost;        // cost at the current linearisation point
  double cost_new;
  double model_change;
  double rho;
  int accepted;
  int spd;
  int iteration;
  int comm_error;     // a peer-memory exchange timed out (multi-GPU): the records of this solve are invalid
  // ceres::TrustRegionMinimizer termination tests (hb200_set_termination); terminated != 0 turns accept_kernel into a no-op
  int terminated;     // 0 running, 1 function tolerance, 2 parameter tolerance, 3 gradient tolerance, 4 minimum trust-region radius, 5 invalid steps
  int invalid_steps;  // consecutive non-positive-definite systems
  double gradient_max_norm, step_norm, x_norm;
};

}  // namespace hb
