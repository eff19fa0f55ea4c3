// Normal equations, landmark Schur complement, dense Cholesky, back-substitution, retraction and
// LM step control (sm_90a).  Replaces the inside of ceres::Solve for the reference's problem
// (reference internal/hyper/optimizers/ceres/optimizer.cpp:38-54,276-280): loss correction
// (Huber 0.5 / ScaledLoss 1.6e-5, optimizer.cpp:226,267-268), J^T J / J^T r, the linear solve
// (SPARSE_NORMAL_CHOLESKY there, landmark Schur + dense Cholesky here), Manifold::Plus
// (reference manifolds/variables/wrapper.hpp:32-34) and the trust-region update.
#pragma once
#include <cooperative_groups.h>

#include "hb200_eval.cuh"

namespace hb {

namespace cg = cooperative_groups;

// The packed reduced system is band-only: see SysLayout / sys_index (hb200_types.cuh).

// The pixel factors' J^T J / J^T r is accumulated by the factor kernel itself (cta_pixel_hessian, hb200_eval.cuh).
constexpr int kHessThreads = 128;

// Inertial factors: one CTA per (run of identical (pose base, gyro-bias base, accel-bias base), split).
// The factor Jacobian is structured -- pose block 6 x 6K dense, bias blocks wg[m] I3 (gyro rows) /
// wa[m] I3 (accel rows), gravity 6 x 2 -- so J^T J is accumulated block by block instead of as a dense
// 6 x (6K + 6KB + 2) product: pose-pose (lower), bias-pose, gravity-pose, bias-bias (diagonal 3x3
// blocks, gyro-accel coupling is identically zero), gravity-bias, gravity-gravity.  Lower triangle of
// S only (dof order pose < gyro bias < accel bias < gravity).
template <int K, int KB>
struct ImuHessScalar {
  static constexpr int NP = 6 * K;
  static constexpr int NBP = 3 * KB * NP;                // bias-pose entries (per bias spline)
  static constexpr int NGP = 2 * NP;                     // gravity-pose
  static constexpr int NBB = KB * (KB + 1) / 2;          // bias-bias scalar weights (lower), each lands on 3 diagonal entries
  static constexpr int NGB = 2 * 3 * KB;                 // gravity-bias (per bias spline)
  static constexpr int NMISC = 2 * NBB + 2 * NGB + 3 + NP + 2 * 3 * KB + 2;   // + gravity-gravity (3) + gradients
  static constexpr int NT = (NP + 7) / 8, NTL = NT * (NT + 1) / 2;     // pose-pose 8 x 8 tiles (lower) for the FP64 tensor cores
  static constexpr int TPW = (NTL + kHessThreads / 32 - 1) / (kHessThreads / 32);   // tiles per warp
  static constexpr int E2 = (NBP + kHessThreads - 1) / kHessThreads;
  static constexpr int E4 = (NGP + kHessThreads - 1) / kHessThreads;
  static constexpr int E5 = (NMISC + kHessThreads - 1) / kHessThreads;
  // writes per thread of the deterministic flush: 3 per pose tile, 2 per bias-pose entry, 1 per gravity-pose entry, at
  // most 6 per small-block entry (3 bias components, each with its diag(J^T J) entry)
  static constexpr int DET_WRITES = 3 * TPW + 2 * E2 + E4 + 6 * E5;
};

template <int K, int KB, bool DET>
HB_DI void inertial_hessian_body(const int* __restrict__ run_off, const int4* __restrict__ idx, const double* __restrict__ r, const double* __restrict__ Jp,
                                 const double* __restrict__ wg, const double* __restrict__ wa, const double* __restrict__ Jg, double loss_scale, double* sys,
                                 SysLayout lay, int o_bg, int o_ba, int o_g, int splits, const DetOut& det) {
  using H = ImuHessScalar<K, KB>;
  constexpr int NP = H::NP;
  constexpr int CH = 16;
  constexpr int NBP = H::NBP, NGP = H::NGP, NBB = H::NBB, NGB = H::NGB, NMISC = H::NMISC, NTL = H::NTL, TPW = H::TPW;
  constexpr int E2 = H::E2, E4 = H::E4, E5 = H::E5;
  __shared__ double sJ[CH][6][NP + 1];
  __shared__ double sWg[CH][KB], sWa[CH][KB], sG[CH][12], sR[CH][6];
  const int run = blockIdx.x / splits, part = blockIdx.x - run * splits;
  const int rlo = run_off[run], rhi = run_off[run + 1];
  const int len = (rhi - rlo + splits - 1) / splits;
  const int lo = rlo + part * len, hi = min(rhi, lo + len);
  if (lo >= hi) return;
  const int4 id0 = idx[lo];
  const int tid = threadIdx.x;
  double a1[2 * TPW], a2[E2], a3[E2], a4[E4], a5[E5];
#pragma unroll
  for (int e = 0; e < 2 * TPW; ++e) a1[e] = 0.0;
  const int warp = tid >> 5, lm = (tid & 31) >> 2, lk = tid & 3;
#pragma unroll
  for (int e = 0; e < E2; ++e) { a2[e] = 0.0; a3[e] = 0.0; }
#pragma unroll
  for (int e = 0; e < E4; ++e) a4[e] = 0.0;
#pragma unroll
  for (int e = 0; e < E5; ++e) a5[e] = 0.0;
  for (int f0 = lo; f0 < hi; f0 += CH) {
    const int cnt = min(CH, hi - f0);
    __syncthreads();
    for (int e = tid; e < cnt * 6 * NP; e += kHessThreads) {   // contiguous in global memory
      const int ff = e / (6 * NP), rem = e - ff * 6 * NP;
      sJ[ff][rem / NP][rem % NP] = Jp[static_cast<size_t>(f0) * 6 * NP + e];
    }
    for (int e = tid; e < cnt * KB; e += kHessThreads) { sWg[e / KB][e % KB] = wg[static_cast<size_t>(f0) * KB + e]; sWa[e / KB][e % KB] = wa[static_cast<size_t>(f0) * KB + e]; }
    for (int e = tid; e < cnt * 12; e += kHessThreads) sG[e / 12][e % 12] = Jg[static_cast<size_t>(f0) * 12 + e];
    for (int e = tid; e < cnt * 6; e += kHessThreads) sR[e / 6][e % 6] = r[static_cast<size_t>(f0) * 6 + e];
    __syncthreads();
    // (1) pose-pose, lower triangle, on the FP64 tensor cores (mma.sync m8n8k4 -> DMMA.8x8x4): the contraction
    // index is (factor, residual row) = the rows of sJ; lane l holds A[m = l/4][k = l%4] = J[k][m] and
    // B[k = l%4][n = l/4] = J[k][n].  (The scalar loop here issued ~290 instructions per entry-triple.)
    {
      const double* Jf = &sJ[0][0][0];
      const int krows = 6 * cnt;
#pragma unroll
      for (int q = 0; q < TPW; ++q) {
        const int tile = warp + q * (kHessThreads / 32);
        if (tile < NTL) {
          int ti = 0;
          while ((ti + 1) * (ti + 2) / 2 <= tile) ++ti;
          const int tj = tile - ti * (ti + 1) / 2;
          const int ma = 8 * ti + lm, nb = 8 * tj + lm;
          const bool va = ma < NP, vb = nb < NP;
          for (int k0 = 0; k0 < krows; k0 += 4) {
            const bool in = k0 + lk < krows;
            const double av = (in && va) ? Jf[(k0 + lk) * (NP + 1) + ma] : 0.0;
            const double bv = (in && vb) ? Jf[(k0 + lk) * (NP + 1) + nb] : 0.0;
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(a1[2 * q]), "+d"(a1[2 * q + 1]) : "d"(av), "d"(bv));
          }
        }
      }
    }
    // (2)/(3) bias-pose: entry (m, c, a) = sum_f w[f][m] * Jp[f][row c (+3)][a]
#pragma unroll
    for (int e = 0; e < E2; ++e) {
      const int id = tid + e * kHessThreads;
      if (id < NBP) {
        const int a = id % NP, mc = id / NP, m = mc / 3, c = mc - 3 * m;
        double s2 = 0, s3 = 0;
        for (int ff = 0; ff < cnt; ++ff) { s2 += sWg[ff][m] * sJ[ff][c][a]; s3 += sWa[ff][m] * sJ[ff][3 + c][a]; }
        a2[e] += s2; a3[e] += s3;
      }
    }
    // (4) gravity-pose
#pragma unroll
    for (int e = 0; e < E4; ++e) {
      const int id = tid + e * kHessThreads;
      if (id < NGP) {
        const int a = id % NP, gm = id / NP;
        double s = 0;
        for (int ff = 0; ff < cnt; ++ff)
#pragma unroll
          for (int row = 0; row < 6; ++row) s += sG[ff][2 * row + gm] * sJ[ff][row][a];
        a4[e] += s;
      }
    }
    // (5) small blocks and gradients
#pragma unroll
    for (int e = 0; e < E5; ++e) {
      int id = tid + e * kHessThreads;
      if (id < NMISC) {
        double s = 0;
        if (id < 2 * NBB) {                       // bias-bias weights
          const bool acc_b = id >= NBB;
          const int q = acc_b ? id - NBB : id;
          int m = static_cast<int>((sqrtf(8.0f * q + 1.0f) - 1.0f) * 0.5f);
          while (m * (m + 1) / 2 > q) --m;
          while ((m + 1) * (m + 2) / 2 <= q) ++m;
          const int m2 = q - m * (m + 1) / 2;
          for (int ff = 0; ff < cnt; ++ff) s += acc_b ? sWa[ff][m] * sWa[ff][m2] : sWg[ff][m] * sWg[ff][m2];
        } else if ((id -= 2 * NBB) < 2 * NGB) {  // gravity-bias: (which, gm, m, c)
          const bool acc_b = id >= NGB;
          const int q = acc_b ? id - NGB : id;
          const int gm = q / (3 * KB), mc = q - gm * 3 * KB, m = mc / 3, c = mc - 3 * m;
          for (int ff = 0; ff < cnt; ++ff) s += sG[ff][2 * (acc_b ? 3 + c : c) + gm] * (acc_b ? sWa[ff][m] : sWg[ff][m]);
        } else if ((id -= 2 * NGB) < 3) {         // gravity-gravity lower: (0,0) (1,0) (1,1)
          const int ga = (id == 0) ? 0 : 1, gb = (id == 2) ? 1 : 0;
          for (int ff = 0; ff < cnt; ++ff)
#pragma unroll
            for (int row = 0; row < 6; ++row) s += sG[ff][2 * row + ga] * sG[ff][2 * row + gb];
        } else if ((id -= 3) < NP) {              // gradient, pose
          for (int ff = 0; ff < cnt; ++ff)
#pragma unroll
            for (int row = 0; row < 6; ++row) s += sJ[ff][row][id] * sR[ff][row];
        } else if ((id -= NP) < 2 * 3 * KB) {     // gradient, biases
          const bool acc_b = id >= 3 * KB;
          const int q = acc_b ? id - 3 * KB : id, m = q / 3, c = q - 3 * m;
          for (int ff = 0; ff < cnt; ++ff) s += (acc_b ? sWa[ff][m] * sR[ff][3 + c] : sWg[ff][m] * sR[ff][c]);
        } else {                                  // gradient, gravity
          id -= 2 * 3 * KB;
          for (int ff = 0; ff < cnt; ++ff)
#pragma unroll
            for (int row = 0; row < 6; ++row) s += sG[ff][2 * row + id] * sR[ff][row];
        }
        a5[e] += s;
      }
    }
  }
  // ---- flush (loss scaling applied once here: J^T J and J^T r both carry loss_scale) ----
  DetCursor dc = det_cursor(det, blockIdx.x, kHessThreads, tid);
  auto add = [&](long long e, double v) { if constexpr (DET) dc.put(e, v); else atomicAdd(&sys[e], v); };
  double* gv = nullptr;   // (the deterministic variant has no system pointer)
  if constexpr (!DET) gv = sys + lay.og;
  auto addg = [&](int i, double v) { if constexpr (DET) dc.put(lay.og + i, v); else atomicAdd(&gv[i], v); };
  const int cp = 6 * id0.x, cg = o_bg + 3 * id0.y, ca = o_ba + 3 * id0.z;
  const double ls = loss_scale;
#pragma unroll
  for (int q = 0; q < TPW; ++q) {
    const int tile = warp + q * (kHessThreads / 32);
    if (tile < NTL) {
      int ti = 0;
      while ((ti + 1) * (ti + 2) / 2 <= tile) ++ti;
      const int tj = tile - ti * (ti + 1) / 2;
      const int a = 8 * ti + lm, b = 8 * tj + 2 * lk;
      if (a < NP) {
        if (b < NP && b <= a) add(sys_index(lay, cp + a, cp + b), ls * a1[2 * q]);
        if (b + 1 < NP && b + 1 <= a) add(sys_index(lay, cp + a, cp + b + 1), ls * a1[2 * q + 1]);
        if (b == a) add(lay.oD + cp + a, ls * a1[2 * q]);               // diag(J^T J), kept apart from S
        if (b + 1 == a) add(lay.oD + cp + a, ls * a1[2 * q + 1]);
      }
    }
  }
#pragma unroll
  for (int e = 0; e < E2; ++e) {
    const int id = tid + e * kHessThreads;
    if (id < NBP) {
      const int a = id % NP, mc = id / NP;
      add(sys_index(lay, cg + mc, cp + a), ls * a2[e]);
      add(sys_index(lay, ca + mc, cp + a), ls * a3[e]);
    }
  }
#pragma unroll
  for (int e = 0; e < E4; ++e) {
    const int id = tid + e * kHessThreads;
    if (id < NGP) add(sys_index(lay, o_g + id / NP, cp + id % NP), ls * a4[e]);
  }
#pragma unroll
  for (int e = 0; e < E5; ++e) {
    int id = tid + e * kHessThreads;
    if (id < NMISC) {
      const double val = ls * a5[e];
      if (id < 2 * NBB) {
        const bool acc_b = id >= NBB;
        const int q = acc_b ? id - NBB : id;
        int m = static_cast<int>((sqrtf(8.0f * q + 1.0f) - 1.0f) * 0.5f);
        while (m * (m + 1) / 2 > q) --m;
        while ((m + 1) * (m + 2) / 2 <= q) ++m;
        const int m2 = q - m * (m + 1) / 2;
        const int c0 = acc_b ? ca : cg;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          add(sys_index(lay, c0 + 3 * m + c, c0 + 3 * m2 + c), val);
          if (m == m2) add(lay.oD + c0 + 3 * m + c, val);
        }
      } else if ((id -= 2 * NBB) < 2 * NGB) {
        const bool acc_b = id >= NGB;
        const int q = acc_b ? id - NGB : id;
        const int gm = q / (3 * KB), mc = q - gm * 3 * KB;
        add(sys_index(lay, o_g + gm, (acc_b ? ca : cg) + mc), val);
      } else if ((id -= 2 * NGB) < 3) {
        const int ga = (id == 0) ? 0 : 1, gb = (id == 2) ? 1 : 0;
        add(sys_index(lay, o_g + ga, o_g + gb), val);
        if (ga == gb) add(lay.oD + o_g + ga, val);
      } else if ((id -= 3) < NP) {
        addg(cp + id, val);
      } else if ((id -= NP) < 2 * 3 * KB) {
        const bool acc_b = id >= 3 * KB;
        addg((acc_b ? ca : cg) + (acc_b ? id - 3 * KB : id), val);
      } else {
        addg(o_g + id - 2 * 3 * KB, val);
      }
    }
  }
}
// DET (deterministic assembly): the records of det, slot = CTA, instead of atomics into sys
template <int K, int KB, bool DET>
__global__ void __launch_bounds__(kHessThreads) inertial_hessian_kernel(const int* __restrict__ run_off, const int4* __restrict__ idx,
                                                                        const double* __restrict__ r, const double* __restrict__ Jp,
                                                                        const double* __restrict__ wg, const double* __restrict__ wa,
                                                                        const double* __restrict__ Jg, double loss_scale, double* sys,
                                                                        SysLayout lay, int o_bg, int o_ba, int o_g, int splits, DetOut det) {
  inertial_hessian_body<K, KB, DET>(run_off, idx, r, Jp, wg, wa, Jg, loss_scale, sys, lay, o_bg, o_ba, o_g, splits, det);
}

// ---------------------------------------------------------------------------------------------
// Inertial J^T J / J^T r as ONE product on the FP64 tensor cores.  The factor's full Jacobian is written out as an
// augmented row block  Ja = [ Jp (6K) | gyro-bias (3KB: w_g[m] in gyro row c, column 3m+c) | accel-bias (3KB) |
// gravity (2) | r (1) ]  -- NA = 6K + 6KB + 3 columns, 6 rows per factor -- and  H = Ja^T Ja  (lower triangle, 8 x 8
// DMMA tiles) holds every block the scalar kernel above accumulates one loop at a time: pose-pose, bias-pose,
// gravity-pose, bias-bias, gravity-bias, gravity-gravity, and in its last row the gradients J^T r.  The bias columns
// are zero except one entry per row, written once per chunk; the zero pattern of the product (gyro-bias x accel-bias,
// bias components c != c') is skipped at the flush.  k-step-outer loop as in the fused pixel J^T J: the NT column
// fragments of a step are loaded once and feed every tile the warp owns.
// WT (an inertial weight matrix W is set): the bias Jacobian is W [w_g[m] I3 ; 0] / W [0 ; w_a[m] I3], so the bias
// columns are dense -- gyro column 3m+c = w_g[m] W[:, c], accel column 3m+c = w_a[m] W[:, 3+c] over all six rows --
// and the product has no zero pattern: every entry is flushed, the gyro-accel coupling included.  The scalar kernel
// above relies on the unweighted structure, so a set inertial matrix always selects this one (inertial_splits).
// ---------------------------------------------------------------------------------------------
template <int K, int KB>
struct ImuHess {
  static constexpr int NP = 6 * K, NBG = 3 * KB, NA = NP + 2 * NBG + 3, NT = (NA + 7) / 8, NTL = NT * (NT + 1) / 2;
  static constexpr int NW = kHessThreads / 32, PER_WARP = (NTL + NW - 1) / NW;
};
// row pitch of the staged rows: >= 8 NT and = 4 or 12 (mod 16) doubles (conflict-free fragment loads): K = 4: 60, K = 6: 68
template <int K, int KB> struct ImuHessLD { static constexpr int value = 8 * ImuHess<K, KB>::NT + 4; };

template <int K, int KB, int W>
HB_DI void imu_hess_steps(double (&c0)[ImuHess<K, KB>::PER_WARP], double (&c1)[ImuHess<K, KB>::PER_WARP], const double* sJ, int krows, int lm, int lk) {
  using H = ImuHess<K, KB>;
  constexpr int LD = ImuHessLD<K, KB>::value;
#pragma unroll 1
  for (int k0 = 0; k0 < krows; k0 += 4) {
    const bool in = k0 + lk < krows;
    const double* p = sJ + (k0 + lk) * LD + lm;
    double fr[H::NT];
#pragma unroll
    for (int t = 0; t < H::NT; ++t) fr[t] = in ? p[8 * t] : 0.0;   // (columns NA .. 8 NT - 1 are zero in shared memory)
#pragma unroll
    for (int q = 0; q < H::PER_WARP; ++q) {
      if (W + H::NW * q < H::NTL) {
        const double av = fr[tile_row(W + H::NW * q < H::NTL ? W + H::NW * q : 0)], bv = fr[tile_col(W + H::NW * q < H::NTL ? W + H::NW * q : 0)];
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0[q]), "+d"(c1[q]) : "d"(av), "d"(bv));
      }
    }
  }
}

// writes per thread of the deterministic flush: two accumulators per tile, each an entry of S and one of diag(J^T J)
template <int K, int KB>
__host__ __device__ constexpr int imu_hess_mma_det_writes() { return 4 * ImuHess<K, KB>::PER_WARP; }

// CH: factors per chunk (static shared memory: 6 CH rows of pitch 60 / 68 doubles, <= 48 KB -> 16 / 12 at most)
template <int K, int KB, int CH, bool DET, bool WT>
HB_DI void inertial_hessian_mma_body(const int* __restrict__ run_off, const int4* __restrict__ idx, const double* __restrict__ r, const double* __restrict__ Jp,
                                     const double* __restrict__ wg, const double* __restrict__ wa, const double* __restrict__ Jg, double loss_scale, double* sys,
                                     SysLayout lay, int o_bg, int o_ba, int o_g, int splits, const DetOut& det, const double* __restrict__ wt) {
  using H = ImuHess<K, KB>;
  constexpr int NP = H::NP, NBG = H::NBG, NA = H::NA, NT = H::NT, NTL = H::NTL, LD = ImuHessLD<K, KB>::value;
  static_assert(LD >= 8 * NT && (LD % 16 == 4 || LD % 16 == 12), "row pitch: conflict-free fragment loads");
  __shared__ double sJ[6 * CH * LD];
  const int run = blockIdx.x / splits, part = blockIdx.x - run * splits;
  const int rlo = run_off[run], rhi = run_off[run + 1];
  const int len = (rhi - rlo + splits - 1) / splits;
  const int lo = rlo + part * len, hi = min(rhi, lo + len);
  if (lo >= hi) return;
  const int4 id0 = idx[lo];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, lm = lane >> 2, lk = lane & 3;
  // the augmented columns are zero except the entries rewritten per chunk
  for (int e = tid; e < 6 * CH * (LD - NP); e += kHessThreads) { const int row = e / (LD - NP), col = NP + e - row * (LD - NP); sJ[row * LD + col] = 0.0; }
  double c0[H::PER_WARP], c1[H::PER_WARP];
#pragma unroll
  for (int q = 0; q < H::PER_WARP; ++q) { c0[q] = 0.0; c1[q] = 0.0; }
  for (int f0 = lo; f0 < hi; f0 += CH) {
    const int cnt = min(CH, hi - f0);
    __syncthreads();   // previous chunk's fragment loads are done (first pass: the zero fill is complete)
    {   // pose block: the chunk's 6 cnt rows are one contiguous run of global memory
      const double2* src = reinterpret_cast<const double2*>(Jp + static_cast<size_t>(f0) * 6 * NP);
      const int total = cnt * 3 * NP;
#pragma unroll 4
      for (int e = tid; e < total; e += kHessThreads) {
        const double2 v = src[e];
        const int row = (2 * e) / NP, col = 2 * e - row * NP;
        sJ[row * LD + col] = v.x; sJ[row * LD + col + 1] = v.y;
      }
    }
    if constexpr (WT) {
      for (int e = tid; e < cnt * KB * 18; e += kHessThreads) {   // bias columns: factor ff, knot m, component c, row
        const int ff = e / (KB * 18), rem = e - ff * KB * 18, m = rem / 18, rc = rem - 18 * m, c = rc / 6, row = rc - 6 * c;
        sJ[(6 * ff + row) * LD + NP + 3 * m + c] = wg[static_cast<size_t>(f0 + ff) * KB + m] * wt[kWtInertial + 6 * row + c];
        sJ[(6 * ff + row) * LD + NP + NBG + 3 * m + c] = wa[static_cast<size_t>(f0 + ff) * KB + m] * wt[kWtInertial + 6 * row + 3 + c];
      }
    } else {
      for (int e = tid; e < cnt * KB * 3; e += kHessThreads) {   // bias entries: factor ff, knot m, component c
        const int ff = e / (KB * 3), rem = e - ff * KB * 3, m = rem / 3, c = rem - 3 * m;
        sJ[(6 * ff + c) * LD + NP + 3 * m + c] = wg[static_cast<size_t>(f0 + ff) * KB + m];
        sJ[(6 * ff + 3 + c) * LD + NP + NBG + 3 * m + c] = wa[static_cast<size_t>(f0 + ff) * KB + m];
      }
    }
    for (int e = tid; e < cnt * 12; e += kHessThreads) {       // gravity: Jg[ff][row][gm]
      const int ff = e / 12, rem = e - 12 * ff, row = rem >> 1, gm = rem & 1;
      sJ[(6 * ff + row) * LD + NP + 2 * NBG + gm] = Jg[static_cast<size_t>(f0) * 12 + e];
    }
    for (int e = tid; e < cnt * 6; e += kHessThreads) sJ[e * LD + NP + 2 * NBG + 2] = r[static_cast<size_t>(f0) * 6 + e];
    __syncthreads();
    const int krows = 6 * cnt;
    if (warp == 0) imu_hess_steps<K, KB, 0>(c0, c1, sJ, krows, lm, lk);
    else if (warp == 1) imu_hess_steps<K, KB, 1>(c0, c1, sJ, krows, lm, lk);
    else if (warp == 2) imu_hess_steps<K, KB, 2>(c0, c1, sJ, krows, lm, lk);
    else imu_hess_steps<K, KB, 3>(c0, c1, sJ, krows, lm, lk);
  }
  // ---- flush: entry (a, b), a >= b, of the augmented product (loss scaling applied once here) ----
  DetCursor dc = det_cursor(det, blockIdx.x, kHessThreads, tid);
  auto add = [&](long long e, double v) { if constexpr (DET) dc.put(e, v); else atomicAdd(&sys[e], v); };
  const long long gv = lay.og;
  const int cp = 6 * id0.x, cg = o_bg + 3 * id0.y, ca = o_ba + 3 * id0.z;
  const double ls = loss_scale;
  auto dof = [&](int a) -> int {   // augmented column -> reduced-system dof
    if (a < NP) return cp + a;
    if (a < NP + NBG) return cg + (a - NP);
    if (a < NP + 2 * NBG) return ca + (a - NP - NBG);
    return o_g + (a - NP - 2 * NBG);
  };
  auto flush = [&](int a, int b, double v) {
    if (a >= NA || b > a) return;
    if (a == NA - 1) {                         // last row: J^T r
      if (b < NA - 1) add(gv + dof(b), ls * v);
      return;
    }
    if constexpr (!WT) {
      if (a >= NP && a < NP + 2 * NBG && b >= NP) {   // bias x bias: only equal components of the same sensor
        if ((a >= NP + NBG) != (b >= NP + NBG)) return;
        if ((a - NP) % 3 != (b - NP) % 3) return;
      }
    }
    const int da = dof(a), db = dof(b);
    add(sys_index(lay, da, db), ls * v);
    if (a == b) add(lay.oD + da, ls * v);   // diag(J^T J), kept apart from S
  };
#pragma unroll
  for (int q = 0; q < H::PER_WARP; ++q) {
    const int tile = warp + H::NW * q;
    if (tile < NTL) {
      const int ti = tile_row(tile), tj = tile_col(tile);
      const int a = 8 * ti + lm, b = 8 * tj + 2 * lk;
      flush(a, b, c0[q]);
      flush(a, b + 1, c1[q]);
    }
  }
}
// DET: slot = CTA; WT: wt is the context's weight table
template <int K, int KB, int CH, bool DET, bool WT>
__global__ void __launch_bounds__(kHessThreads) inertial_hessian_mma_kernel(const int* __restrict__ run_off, const int4* __restrict__ idx,
                                                                            const double* __restrict__ r, const double* __restrict__ Jp,
                                                                            const double* __restrict__ wg, const double* __restrict__ wa,
                                                                            const double* __restrict__ Jg, double loss_scale, double* sys,
                                                                            SysLayout lay, int o_bg, int o_ba, int o_g, int splits, DetOut det,
                                                                            const double* __restrict__ wt) {
  inertial_hessian_mma_body<K, KB, CH, DET, WT>(run_off, idx, r, Jp, wg, wa, Jg, loss_scale, sys, lay, o_bg, o_ba, o_g, splits, det, wt);
}

// J^T J / J^T r of the manifold (pose) factors: one warp per factor, lower triangle of its 6K x 6K block.
constexpr int kManWarps = 4;
// writes per lane of the deterministic variant: an entry of S and one of diag(J^T J) per pass over the block, the gradient
template <int K>
__host__ __device__ constexpr int manifold_det_writes() { return 2 * ((36 * K * K + 31) / 32) + (6 * K + 31) / 32; }

template <int K, bool DET>
HB_DI void manifold_hessian_body(int nf, const int2* __restrict__ idx, const double* __restrict__ r, const double* __restrict__ Jp, double* sys, SysLayout lay,
                                 const DetOut& det) {
  constexpr int NB = 6 * K;
  __shared__ double sJ[kManWarps][6][NB];
  __shared__ double sr[kManWarps][6];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f = blockIdx.x * kManWarps + warp;
  if (f >= nf) return;
  for (int e = lane; e < 6 * NB; e += 32) sJ[warp][e / NB][e % NB] = Jp[static_cast<size_t>(f) * 6 * NB + e];
  if (lane < 6) sr[warp][lane] = r[6 * static_cast<size_t>(f) + lane];
  __syncwarp();
  DetCursor dc = det_cursor(det, f, 32, lane);   // slot = factor
  auto add = [&](long long e, double v) { if constexpr (DET) dc.put(e, v); else atomicAdd(&sys[e], v); };
  const int c0 = 6 * idx[f].x;
  double* g = nullptr;   // (the deterministic variant has no system pointer)
  if constexpr (!DET) g = sys + lay.og;
  for (int e = lane; e < NB * NB; e += 32) {
    const int a = e / NB, b = e - a * NB;
    if (b > a) continue;
    double s = 0;
#pragma unroll
    for (int q = 0; q < 6; ++q) s += sJ[warp][q][a] * sJ[warp][q][b];
    add(sys_index(lay, c0 + a, c0 + b), s);
    if (a == b) add(lay.oD + c0 + a, s);
  }
  for (int a = lane; a < NB; a += 32) {
    double s = 0;
#pragma unroll
    for (int q = 0; q < 6; ++q) s += sJ[warp][q][a] * sr[warp][q];
    if constexpr (DET) dc.put(lay.og + c0 + a, s);
    else atomicAdd(&g[c0 + a], s);
  }
}
template <int K, bool DET>
__global__ void __launch_bounds__(kManWarps * 32) manifold_hessian_kernel(int nf, const int2* __restrict__ idx, const double* __restrict__ r,
                                                                         const double* __restrict__ Jp, double* sys, SysLayout lay, DetOut det) {
  manifold_hessian_body<K, DET>(nf, idx, r, Jp, sys, lay, det);
}

// cost at the linearisation point = sum of the evaluation kernels' per-block partials (fixed order) -> scal[0] of
// the packed system.  (diag(J^T J) is accumulated by the J^T J kernels themselves, the right-hand side is kept as
// b_schur - g by every consumer: nothing else has to happen between the J^T J kernels and the Schur complement, so
// this kernel runs on the side stream next to them.)
__global__ void cost_kernel(double* sys, SysLayout lay, const double* __restrict__ cp_pix, int n_pix_blocks, const double* __restrict__ cp_imu,
                            int n_imu_blocks) {
  __shared__ double s[256];
  double c = 0;
  for (int i = threadIdx.x; i < n_pix_blocks; i += blockDim.x) c += cp_pix[i];
  for (int i = threadIdx.x; i < n_imu_blocks; i += blockDim.x) c += cp_imu[i];
  s[threadIdx.x] = c;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) { sys[lay.os] = s[0]; sys[lay.os + 1] = 0.0; }
}

// ---------------------------------------------------------------------------------------------
// Landmark Schur complement: one CTA per landmark.
//   V = sum w Jl^T Jl + mu D_l ; W = sum w Jp^T Jl (rows of the control points the landmark's
//   observations touch) ; V = L L^T ; Y = W L^-T ; z = L^-1 g_l ; S -= Y Y^T ; b += Y z.
// Dynamic shared memory: 2 * max_rows * 3 doubles.
//
// The elimination goes through a Cholesky factor of V, never an explicit inverse.  A landmark seen once has a rank-2
// V = w Jl^T Jl, and only the damping mu D_l (mu = 1 / radius, down to 1e-16) makes it invertible: an adjugate inverse
// then loses every digit of W V^-1 W^T, while Y Y^T stays accurate (W is zero along V's null direction).  Each pivot is
// floored at mu d_j, its lower bound in exact arithmetic (V + mu D >= mu D), so cancellation cannot take it to 0.
// ---------------------------------------------------------------------------------------------
constexpr int kSchurThreads = 128;

// Cholesky of the damped landmark block (row-major 3 x 3, diagonal already damped by mu d) with every pivot floored at
// mu d_j.  Packed as f = (1/L00, L10, 1/L11, L20, L21, 1/L22): what lm_backsub_kernel solves with (all zero: dl = 0).
HB_DI void lm_chol3(const double* V, const double* d, double mu, double* f) {
  const double i0 = 1.0 / sqrt(fmax(V[0], mu * d[0]));
  const double l10 = V[3] * i0, l20 = V[6] * i0;
  const double i1 = 1.0 / sqrt(fmax(V[4] - l10 * l10, mu * d[1]));
  const double l21 = (V[7] - l20 * l10) * i1;
  const double i2 = 1.0 / sqrt(fmax(V[8] - l20 * l20 - l21 * l21, mu * d[2]));
  f[0] = i0; f[1] = l10; f[2] = i1; f[3] = l20; f[4] = l21; f[5] = i2;
}
// y = L^-1 x (forward substitution with the packed factor)
HB_DI void lm_lsolve(const double* f, double x0, double x1, double x2, double* y) {
  y[0] = x0 * f[0];
  y[1] = (x1 - f[1] * y[0]) * f[2];
  y[2] = (x2 - f[3] * y[0] - f[4] * y[1]) * f[5];
}

// writes per thread of the deterministic variant: b over the rows, then the lower triangle of Y Y^T
__host__ __device__ inline long long schur_det_writes(int max_rows) {
  return (max_rows + kSchurThreads - 1) / kSchurThreads + (static_cast<long long>(max_rows) * max_rows + kSchurThreads - 1) / kSchurThreads;
}

// DET: every entry the landmark's rows cover is written (zeros included), into the landmark's slot
template <int K, bool DET>
HB_DI void schur_body(const int* __restrict__ lm_off, const int* __restrict__ lm_obs, const int4* __restrict__ idx, const double* __restrict__ r,
                      const double* __restrict__ Jp, const double* __restrict__ Jl, const double* __restrict__ wv, const SolverState* __restrict__ st,
                      double* sys, SysLayout lay, double* __restrict__ Vchol, double* __restrict__ gl, double* __restrict__ Dl, int max_rows,
                      const DetOut& det) {
  constexpr int NB = 6 * K;
  extern __shared__ double s_dyn[];
  double* W = s_dyn;                  // [rows][3]
  double* Y = s_dyn + 3 * max_rows;   // [rows][3]
  __shared__ double sV[12];           // V (9) + g_l (3)
  __shared__ double sF[9];            // packed Cholesky factor (6) + z (3)
  const int l = blockIdx.x;
  const int o_lo = lm_off[l], o_hi = lm_off[l + 1];
  if (o_lo >= o_hi) {
    if (threadIdx.x < 9) Vchol[9 * static_cast<size_t>(l) + threadIdx.x] = 0.0;
    if (threadIdx.x < 3) { gl[3 * static_cast<size_t>(l) + threadIdx.x] = 0.0; Dl[3 * static_cast<size_t>(l) + threadIdx.x] = 1e-6; }
    return;
  }
  const int cp_lo = idx[lm_obs[o_lo]].x;
  const int cp_hi = idx[lm_obs[o_hi - 1]].x + K;
  const int rows = 6 * (cp_hi - cp_lo);
  // V and g_l
  if (threadIdx.x < 12) {
    double s = 0;
    for (int o = o_lo; o < o_hi; ++o) {
      const int f = lm_obs[o];
      const double r0 = r[2 * f], r1 = r[2 * f + 1];
      const double wgt = wv[f];
      const double* jl = Jl + 6 * static_cast<size_t>(f);
      if (threadIdx.x < 9) { const int a = threadIdx.x / 3, b = threadIdx.x % 3; s += wgt * (jl[a] * jl[b] + jl[3 + a] * jl[3 + b]); }
      else { const int a = threadIdx.x - 9; s += wgt * (jl[a] * r0 + jl[3 + a] * r1); }
    }
    sV[threadIdx.x] = s;
  }
  // W rows
  for (int e = threadIdx.x; e < rows * 3; e += kSchurThreads) {
    const int row = e / 3, c = e - 3 * row;
    double s = 0;
    for (int o = o_lo; o < o_hi; ++o) {
      const int f = lm_obs[o];
      const int a = row - 6 * (idx[f].x - cp_lo);
      if (a >= 0 && a < NB) {
        const double wgt = wv[f];
        const double* jp = Jp + static_cast<size_t>(f) * 2 * NB;
        const double* jl = Jl + 6 * static_cast<size_t>(f);
        s += wgt * (jp[a] * jl[c] + jp[NB + a] * jl[3 + c]);
      }
    }
    W[e] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const double mu = 1.0 / st->radius;
    double V[9], d[3];
#pragma unroll
    for (int i = 0; i < 9; ++i) V[i] = sV[i];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      d[a] = fmin(fmax(V[4 * a], 1e-6), 1e32);
      Dl[3 * static_cast<size_t>(l) + a] = d[a];
      V[4 * a] += mu * d[a];
    }
    lm_chol3(V, d, mu, sF);
    lm_lsolve(sF, sV[9], sV[10], sV[11], sF + 6);
#pragma unroll
    for (int i = 0; i < 9; ++i) Vchol[9 * static_cast<size_t>(l) + i] = i < 6 ? sF[i] : 0.0;
#pragma unroll
    for (int i = 0; i < 3; ++i) gl[3 * static_cast<size_t>(l) + i] = sV[9 + i];
  }
  __syncthreads();
  const int r0g = 6 * cp_lo;
  DetCursor dc = det_cursor(det, l, kSchurThreads, threadIdx.x);
  auto add = [&](long long e, double v) { if constexpr (DET) dc.put(e, v); else atomicAdd(&sys[e], v); };
  for (int row = threadIdx.x; row < rows; row += kSchurThreads) {
    double y[3];
    lm_lsolve(sF, W[3 * row], W[3 * row + 1], W[3 * row + 2], y);
    Y[3 * row] = y[0]; Y[3 * row + 1] = y[1]; Y[3 * row + 2] = y[2];
    const double val = y[0] * sF[6] + y[1] * sF[7] + y[2] * sF[8];
    if (DET || val != 0.0) add(lay.ob + r0g + row, val);
  }
  __syncthreads();
  for (int e = threadIdx.x; e < rows * rows; e += kSchurThreads) {
    const int a = e / rows, b = e - a * rows;
    if (b > a) continue;
    const double val = Y[3 * a] * Y[3 * b] + Y[3 * a + 1] * Y[3 * b + 1] + Y[3 * a + 2] * Y[3 * b + 2];
    if (DET || val != 0.0) add(sys_index(lay, r0g + a, r0g + b), -val);
  }
}
template <int K, bool DET>
__global__ void __launch_bounds__(kSchurThreads) schur_kernel(const int* __restrict__ lm_off, const int* __restrict__ lm_obs,
                                                              const int4* __restrict__ idx, const double* __restrict__ r,
                                                              const double* __restrict__ Jp, const double* __restrict__ Jl, const double* __restrict__ wv,
                                                              const SolverState* __restrict__ st, double* sys, SysLayout lay,
                                                              double* __restrict__ Vchol, double* __restrict__ gl, double* __restrict__ Dl,
                                                              int max_rows, DetOut det) {
  schur_body<K, DET>(lm_off, lm_obs, idx, r, Jp, Jl, wv, st, sys, lay, Vchol, gl, Dl, max_rows, det);
}

// ---------------------------------------------------------------------------------------------
// Landmark Schur complement for LARGE windows: a CTA takes a GROUP of landmarks whose control-point ranges fall into
// one window of RT rows (groups are cut on the host from the landmarks ordered by their first knot base) and
// accumulates the whole group's contribution on the FP64 tensor cores before touching the system once.
// Per landmark (one warp each, four in flight): V, g_l, W as in schur_kernel; then with V = L L^T
//   W V^-1 W^T = Y Y^T,  Y = W L^-T (rows x 3)       W V^-1 g_l = Y z,  z = L^-1 g_l
// Y's three columns become three rows of the group's stack Ys[3 G][RT] (zero outside the landmark's rows), so
//   S[tile] -= Ys^T Ys  (mma.sync m8n8k4 -> DMMA, contraction over 3 G)        b[tile] += Ys^T zs
// and the group flushes RT (RT + 1) / 2 lower entries with one atomic each instead of ~rows^2 / 2 per landmark
// (83 k landmarks: 75 M FP64 atomics on a few hundred cache lines were the whole cost of schur_kernel).
// ---------------------------------------------------------------------------------------------
constexpr int kSchurGroup = 32;       // landmarks per group (3 * 32 = 96 contraction rows)
constexpr int kSchurGThreads = 128;
// writes per thread of the deterministic variant: two per tile a warp owns, then b over the window's rows
__host__ __device__ inline long long schur_group_det_writes(int RT) {
  const int NT = RT / 8, ntiles = NT * (NT + 1) / 2;
  return 2 * ((ntiles + kSchurGThreads / 32 - 1) / (kSchurGThreads / 32)) + (RT + kSchurGThreads - 1) / kSchurGThreads;
}

template <int K, bool DET>
HB_DI void schur_group_body(const int* __restrict__ group_off, const int* __restrict__ lm_order, const int* __restrict__ lm_off, const int* __restrict__ lm_obs,
                            const int4* __restrict__ idx, const double* __restrict__ r, const double* __restrict__ Jp, const double* __restrict__ Jl,
                            const double* __restrict__ wv, const SolverState* __restrict__ st, double* sys, SysLayout lay, double* __restrict__ Vchol,
                            double* __restrict__ gl, double* __restrict__ Dl, int RT, const DetOut& det) {
  constexpr int NB = 6 * K;
  extern __shared__ double s_grp[];
  const int LD = RT + 1;
  double* Ys = s_grp;                                  // [3 G][LD]
  double* zs = Ys + 3 * kSchurGroup * LD;              // [3 G]
  double* Ws = zs + 3 * kSchurGroup;                   // per warp: W [RT][3]
  __shared__ int s_lo;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g0 = group_off[blockIdx.x], g1 = group_off[blockIdx.x + 1];
  const int cnt = g1 - g0;
  if (tid == 0) {   // window origin = first knot base of the group's first landmark (the order is ascending in it)
    const int l = lm_order[g0];
    s_lo = idx[lm_obs[lm_off[l]]].x;
  }
  for (int e = tid; e < 3 * kSchurGroup * LD; e += kSchurGThreads) Ys[e] = 0.0;
  for (int e = tid; e < 3 * kSchurGroup; e += kSchurGThreads) zs[e] = 0.0;
  __syncthreads();
  const int tile_lo = s_lo;
  const double mu = 1.0 / st->radius;
  double* W = Ws + warp * RT * 3;
  for (int gi = warp; gi < cnt; gi += kSchurGThreads / 32) {
    const int l = lm_order[g0 + gi];
    const int o_lo = lm_off[l], o_hi = lm_off[l + 1];
    const int cp_lo = idx[lm_obs[o_lo]].x, cp_hi = idx[lm_obs[o_hi - 1]].x + K;
    const int rows = 6 * (cp_hi - cp_lo), roff = 6 * (cp_lo - tile_lo);
    // observation-major: per observation the warp reads the factor's two Jacobian rows coalesced (lane = column) and adds
    // w (jp0 jl_c + jp1 jl_{3+c}) into W's rows of that factor's control points; lanes 0..11 keep V (9) and g_l (3)
    for (int e = lane; e < rows * 3; e += 32) W[e] = 0.0;
    __syncwarp();
    double vg = 0.0;
    const int va = lane < 9 ? lane / 3 : lane - 9, vb = lane % 3;   // this lane's entry of V (lanes 0..8) or of g (9..11)
    // four observations per round: all their loads are issued before anything is accumulated (the loop is a chain of
    // dependent L2 round trips otherwise: lm_obs -> idx / w / Jl / Jp)
    for (int o0 = o_lo; o0 < o_hi; o0 += 4) {
      int fq[4], bq[4];
      double wq[4], jlq[4][6], j0q[4][2], j1q[4][2], rq[4][2];
#pragma unroll
      for (int u = 0; u < 4; ++u) fq[u] = (o0 + u < o_hi) ? lm_obs[o0 + u] : -1;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int f = fq[u];
        const bool on = f >= 0;
        wq[u] = on ? wv[f] : 0.0;
        bq[u] = on ? 6 * (idx[f].x - cp_lo) : 0;
        const double* jlp = Jl + 6 * static_cast<size_t>(on ? f : 0);
#pragma unroll
        for (int c = 0; c < 6; ++c) jlq[u][c] = on ? jlp[c] : 0.0;
        const double* jp = Jp + static_cast<size_t>(on ? f : 0) * 2 * NB;
#pragma unroll
        for (int t = 0; t < 2; ++t) {   // NB <= 64 columns: lane, lane + 32
          const int a = lane + 32 * t;
          j0q[u][t] = (on && a < NB) ? jp[a] : 0.0;
          j1q[u][t] = (on && a < NB) ? jp[NB + a] : 0.0;
        }
        rq[u][0] = (on && lane >= 9 && lane < 12) ? r[2 * f] : 0.0;
        rq[u][1] = (on && lane >= 9 && lane < 12) ? r[2 * f + 1] : 0.0;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (fq[u] < 0) continue;
        const double wgt = wq[u];
        const double* jl = jlq[u];
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          const int a = lane + 32 * t;
          if (a < NB) {
            const double j0 = wgt * j0q[u][t], j1 = wgt * j1q[u][t];
            double* wr = W + (bq[u] + a) * 3;
            wr[0] += j0 * jl[0] + j1 * jl[3];
            wr[1] += j0 * jl[1] + j1 * jl[4];
            wr[2] += j0 * jl[2] + j1 * jl[5];
          }
        }
        // lanes 0..8: V[a][b]; lanes 9..11: g[a].  The row picks are SELECT chains on purpose: `jl[a]` with a lane-dependent
        // index put the whole jlq array into local memory (ncu: 250 M local sectors, a third of the kernel's stall samples)
        if (lane < 12) {
          const double ja0 = va == 0 ? jl[0] : (va == 1 ? jl[1] : jl[2]), ja1 = va == 0 ? jl[3] : (va == 1 ? jl[4] : jl[5]);
          const double x0 = lane < 9 ? (vb == 0 ? jl[0] : (vb == 1 ? jl[1] : jl[2])) : rq[u][0];
          const double x1 = lane < 9 ? (vb == 0 ? jl[3] : (vb == 1 ? jl[4] : jl[5])) : rq[u][1];
          vg += wgt * (ja0 * x0 + ja1 * x1);
        }
        __syncwarp();   // the next observation may touch the same rows of W
      }
    }
    __syncwarp();
    // lane 0: damped V and its Cholesky factor (pivots floored, see schur_kernel); everything the back substitution needs
    // goes to global memory
    double V[9], g3[3];
#pragma unroll
    for (int i = 0; i < 9; ++i) V[i] = __shfl_sync(0xffffffffu, vg, i);
#pragma unroll
    for (int i = 0; i < 3; ++i) g3[i] = __shfl_sync(0xffffffffu, vg, 9 + i);
    double F[6] = {0, 0, 0, 0, 0, 0};   // packed factor of lm_chol3
    if (lane == 0) {
      double d[3], z[3];
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        d[a] = fmin(fmax(V[4 * a], 1e-6), 1e32);
        Dl[3 * static_cast<size_t>(l) + a] = d[a];
        V[4 * a] += mu * d[a];
      }
      lm_chol3(V, d, mu, F);
#pragma unroll
      for (int i = 0; i < 9; ++i) Vchol[9 * static_cast<size_t>(l) + i] = i < 6 ? F[i] : 0.0;
#pragma unroll
      for (int i = 0; i < 3; ++i) gl[3 * static_cast<size_t>(l) + i] = g3[i];
      lm_lsolve(F, g3[0], g3[1], g3[2], z);
      zs[3 * gi] = z[0]; zs[3 * gi + 1] = z[1]; zs[3 * gi + 2] = z[2];
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) F[i] = __shfl_sync(0xffffffffu, F[i], 0);
    __syncwarp();
    // Y = W L^-T into the stack: row k = 3 gi + c holds column c of Y at the landmark's rows
    for (int row = lane; row < rows; row += 32) {
      double y[3];
      lm_lsolve(F, W[3 * row], W[3 * row + 1], W[3 * row + 2], y);
      Ys[(3 * gi) * LD + roff + row] = y[0];
      Ys[(3 * gi + 1) * LD + roff + row] = y[1];
      Ys[(3 * gi + 2) * LD + roff + row] = y[2];
    }
    __syncwarp();
  }
  __syncthreads();
  // the group's Schur complement: lower 8 x 8 tiles of Ys^T Ys on the FP64 tensor cores, contraction over 3 cnt rows
  const int NT = RT / 8, ntiles = NT * (NT + 1) / 2, kk = 3 * cnt;
  const int lm = lane >> 2, lk = lane & 3;
  const int r0g = 6 * tile_lo;
  DetCursor dc = det_cursor(det, blockIdx.x, kSchurGThreads, tid);   // slot = group
  auto add = [&](long long e, double v) { if constexpr (DET) dc.put(e, v); else atomicAdd(&sys[e], v); };
  for (int tile = warp; tile < ntiles; tile += kSchurGThreads / 32) {
    int ti = 0;
    while ((ti + 1) * (ti + 2) / 2 <= tile) ++ti;
    const int tj = tile - ti * (ti + 1) / 2;
    const double* pa = Ys + lk * LD + 8 * ti + lm;
    const double* pb = Ys + lk * LD + 8 * tj + lm;
    double c0 = 0.0, c1 = 0.0;
    for (int k0 = 0; k0 < kk; k0 += 4) {
      const bool in = k0 + lk < kk;
      const double av = in ? pa[k0 * LD] : 0.0, bv = in ? pb[k0 * LD] : 0.0;
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(av), "d"(bv));
    }
    const int m = 8 * ti + lm, n = 8 * tj + 2 * lk;
    const int row = r0g + m;
    if (row < lay.np) {
      if (n <= m && (DET || c0 != 0.0) && row - 6 * ((r0g + n) / 6) < lay.h) add(sys_index(lay, row, r0g + n), -c0);
      if (n + 1 <= m && (DET || c1 != 0.0) && row - 6 * ((r0g + n + 1) / 6) < lay.h) add(sys_index(lay, row, r0g + n + 1), -c1);
    }
  }
  for (int m = tid; m < RT; m += kSchurGThreads) {
    double acc = 0.0;
    for (int k = 0; k < kk; ++k) acc += Ys[k * LD + m] * zs[k];
    if ((DET || acc != 0.0) && r0g + m < lay.np) add(lay.ob + r0g + m, acc);
  }
}
template <int K, bool DET>
__global__ void __launch_bounds__(kSchurGThreads) schur_group_kernel(const int* __restrict__ group_off, const int* __restrict__ lm_order,
                                                                    const int* __restrict__ lm_off, const int* __restrict__ lm_obs,
                                                                    const int4* __restrict__ idx, const double* __restrict__ r,
                                                                    const double* __restrict__ Jp, const double* __restrict__ Jl, const double* __restrict__ wv,
                                                                    const SolverState* __restrict__ st, double* sys, SysLayout lay,
                                                                    double* __restrict__ Vchol, double* __restrict__ gl, double* __restrict__ Dl, int RT,
                                                                    DetOut det) {
  schur_group_body<K, DET>(group_off, lm_order, lm_off, lm_obs, idx, r, Jp, Jl, wv, st, sys, lay, Vchol, gl, Dl, RT, det);
}

// ---------------------------------------------------------------------------------------------
// Deterministic assembly, second half: the entry -> records index and the fixed-order sums (see DetOut, hb200_eval.cuh).
// det_index_kernel runs in every deterministic build but works only on the first after the slots were laid out
// (*ready == 0): it counts the records of every entry, scans the counts, fills each entry's list and sorts it by record
// position (the one-time cost is measured in DESIGN.md §5.4).  The keys it reads are those the J^T J kernels of the same build wrote just before -- the same every build,
// since they follow from the window alone.  Cooperative launch (grid syncs between the phases).
// ---------------------------------------------------------------------------------------------
constexpr int kDetThreads = 256;
__global__ void __launch_bounds__(kDetThreads) det_index_kernel(long long nrec, const int* __restrict__ key, int nent, int* __restrict__ cnt,
                                                                int* __restrict__ off, int* __restrict__ perm, int* __restrict__ ready) {
  if (*ready) return;   // (uniform across the grid: nothing writes it before the last phase)
  cg::grid_group grid = cg::this_grid();
  const long long t0 = static_cast<long long>(blockIdx.x) * kDetThreads + threadIdx.x, nt = static_cast<long long>(gridDim.x) * kDetThreads;
  for (long long e = t0; e < nent; e += nt) cnt[e] = 0;
  grid.sync();
  for (long long p = t0; p < nrec; p += nt) { const int k = key[p]; if (k >= 0) atomicAdd(&cnt[k], 1); }
  grid.sync();
  if (blockIdx.x == 0) {   // exclusive scan of the counts -> off[0 .. nent]
    __shared__ int s_warp[kDetThreads / 32];
    __shared__ int s_carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base < nent; base += kDetThreads) {
      const int i = base + tid;
      const int v = i < nent ? cnt[i] : 0;
      int x = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
      if (lane == 31) s_warp[warp] = x;
      __syncthreads();
      int wsum = 0;
      for (int w = 0; w < warp; ++w) wsum += s_warp[w];
      const int incl = x + wsum + s_carry;
      if (i < nent) off[i] = incl - v;
      __syncthreads();
      if (tid == kDetThreads - 1) s_carry = incl;
      __syncthreads();
    }
    if (tid == 0) off[nent] = s_carry;
  }
  grid.sync();
  for (long long e = t0; e < nent; e += nt) cnt[e] = 0;
  grid.sync();
  for (long long p = t0; p < nrec; p += nt) {
    const int k = key[p];
    if (k >= 0) perm[off[k] + atomicAdd(&cnt[k], 1)] = static_cast<int>(p);
  }
  grid.sync();
  // each entry's list into ascending record position (the fill above is in atomic order).  Heap sort, O(n log n) per
  // list: a list holds one record per slot covering the entry -- a handful for most entries, but one per inertial CTA for
  // the gravity entries and one per landmark for the pose entries under the per-landmark Schur kernel (thousands)
  for (long long e = t0; e < nent; e += nt) {
    int* a = perm + off[e];
    const int n = off[e + 1] - off[e];
    auto sift = [&](int root, int end) {   // max-heap on a[0 .. end)
      const int v = a[root];
      int i = root;
      for (int c = 2 * i + 1; c < end; c = 2 * i + 1) {
        if (c + 1 < end && a[c + 1] > a[c]) ++c;
        if (a[c] <= v) break;
        a[i] = a[c];
        i = c;
      }
      a[i] = v;
    };
    for (int i = n / 2 - 1; i >= 0; --i) sift(i, n);
    for (int end = n - 1; end > 0; --end) {
      const int t = a[0]; a[0] = a[end]; a[end] = t;
      sift(0, end);
    }
  }
  if (t0 == 0) *ready = 1;
}

// every packed entry with records = their sum in ascending record order (the system was cleared by prep_kernel; the
// entries no slot covers stay zero)
__global__ void __launch_bounds__(kDetThreads) det_reduce_kernel(int nent, const int* __restrict__ off, const int* __restrict__ perm,
                                                                 const double* __restrict__ val, double* __restrict__ sys) {
  for (int e = blockIdx.x * kDetThreads + threadIdx.x; e < nent; e += gridDim.x * kDetThreads) {
    const int lo = off[e], hi = off[e + 1];
    if (lo == hi) continue;
    double s = 0.0;
    for (int i = lo; i < hi; ++i) s += val[perm[i]];
    sys[e] = s;
  }
}

// Dense fallback / inspection: expands the band-only raw system into the dense factorisation work copy
// Lw ((32 T + 1) x n, last row = b), applying LM damping mu clamp(diag H) and the constant-dof mask on the way
// (what the band solver does while it gathers).  st == nullptr: no damping.
__global__ void densify_kernel(const double* __restrict__ sys, SysLayout lay, const SolverState* __restrict__ st, const unsigned char* __restrict__ fixed,
                               double* __restrict__ D, double* __restrict__ Lw, int* __restrict__ spd_flag) {
  const int n = lay.n;
  if (blockIdx.x == 0 && threadIdx.x == 0) *spd_flag = 1;
  const size_t brow = static_cast<size_t>((n + 31) / 32) * 32;  // row of Lw holding b (own tile row)
  const double mu = st ? 1.0 / st->radius : 0.0;
  const size_t total = static_cast<size_t>(n + 1) * n;
  for (size_t e = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; e < total; e += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int i = static_cast<int>(e / n), j = static_cast<int>(e - static_cast<size_t>(i) * n);
    if (i < n) {
      const int hi = max(i, j), lo = min(i, j);   // only the lower triangle is stored
      double s = 0.0;
      if (hi >= lay.np || hi - 6 * (lo / 6) < lay.h) s = sys[sys_index(lay, hi, lo)];
      if (i == j) {
        const double d = fmin(fmax(sys[lay.oD + i], 1e-6), 1e32);
        D[i] = d;
        s += mu * d;
      }
      if (fixed[i] || fixed[j]) s = (i == j) ? 1.0 : 0.0;
      Lw[e] = s;
    } else {
      Lw[brow * n + j] = fixed[j] ? 0.0 : sys[lay.ob + j] - sys[lay.og + j];   // rhs = Schur part - gradient
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Dense blocked Cholesky (right-looking, 32 x 32 tiles) of the augmented matrix [S ; b^T] stored
// as (32*T + 1) x n (rows n..32T-1 unused, b^T in row 32T so that it owns a tile row): after the
// call the strictly-lower tiles hold L, Ldiag holds the diagonal tiles and row 32T holds y = L^-1 b.  Cooperative launch (grid sync between panel phases).
// ---------------------------------------------------------------------------------------------
constexpr int kCholNB = 32;
constexpr int kCholThreads = 256;
constexpr int kCholWarps = kCholThreads / 32;
constexpr size_t kCholSmem = sizeof(double) * (kCholNB * (kCholNB + 1)) * (1 + kCholWarps);

HB_DI void chol_tile32(double (*s)[kCholNB + 1], int lane) {
  // In-place Cholesky of a 32x32 SPD tile in shared memory by one warp; lane = row.
  double row[kCholNB];
#pragma unroll
  for (int c = 0; c < kCholNB; ++c) row[c] = s[lane][c];
#pragma unroll
  for (int c = 0; c < kCholNB; ++c) {
    const double dcc = __shfl_sync(0xffffffffu, row[c], c);
    const double inv = rsqrt(dcc);
    const double lrc = (lane == c) ? dcc * inv : row[c] * inv;  // sqrt(dcc) on the diagonal
    row[c] = lrc;
    s[lane][c] = (lane >= c) ? lrc : 0.0;
    __syncwarp();
#pragma unroll
    for (int cc = c + 1; cc < kCholNB; ++cc) row[cc] -= lrc * s[cc][c];
    __syncwarp();
  }
}

__global__ void __launch_bounds__(kCholThreads) cholesky_kernel(double* __restrict__ Lw, double* __restrict__ Ldiag, int n, int* __restrict__ spd_flag) {
  cg::grid_group grid = cg::this_grid();
  extern __shared__ double s_chol[];
  double (*sL)[kCholNB + 1] = reinterpret_cast<double (*)[kCholNB + 1]>(s_chol);
  double (*sA)[kCholNB][kCholNB + 1] = reinterpret_cast<double (*)[kCholNB][kCholNB + 1]>(s_chol + kCholNB * (kCholNB + 1));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int T = (n + kCholNB - 1) / kCholNB;  // column tiles
  const int TR = T + 1;                       // row tiles (last one = augmented row only)
  const int brow = T * kCholNB;
  const int gwarp = blockIdx.x * kCholWarps + warp;
  const int nwarps = gridDim.x * kCholWarps;
  for (int p = 0; p < T; ++p) {
    const int c0 = p * kCholNB;
    // ---- phase A: every CTA with TRSM work factors the diagonal tile, then solves its row tiles ----
    const int ntr = TR - (p + 1);
    const bool has_work = (blockIdx.x == 0) || (blockIdx.x * kCholWarps < ntr);
    if (has_work) {
      for (int e = threadIdx.x; e < kCholNB * kCholNB; e += kCholThreads) {
        const int i = e / kCholNB, j = e - i * kCholNB;
        const int gi = c0 + i, gj = c0 + j;
        double val = (i == j) ? 1.0 : 0.0;
        if (gi < n && gj < n) val = Lw[static_cast<size_t>(gi) * n + gj];
        sL[i][j] = val;
      }
      __syncthreads();
      if (warp == 0) chol_tile32(sL, lane);
      __syncthreads();
      if (blockIdx.x == 0) {
        bool bad = false;
        for (int e = threadIdx.x; e < kCholNB * kCholNB; e += kCholThreads) {
          const int i = e / kCholNB, j = e - i * kCholNB;
          const double val = sL[i][j];
          Ldiag[static_cast<size_t>(p) * kCholNB * kCholNB + e] = val;
          if (i == j && !(val > 0.0)) bad = true;
        }
        if (bad) atomicExch(spd_flag, 0);
      }
      // TRSM: row tile i (> p, incl. the augmented row): X = A_ip L_pp^-T, lane = row of the tile
      for (int it = gwarp; it < ntr; it += nwarps) {
        const int i = p + 1 + it;
        const int gi = i * kCholNB + lane;
        double a[kCholNB];
        if (gi < n || gi == brow) {
#pragma unroll
          for (int c = 0; c < kCholNB; ++c) a[c] = (c0 + c < n) ? Lw[static_cast<size_t>(gi) * n + c0 + c] : 0.0;
        } else {
#pragma unroll
          for (int c = 0; c < kCholNB; ++c) a[c] = 0.0;
        }
#pragma unroll
        for (int c = 0; c < kCholNB; ++c) {
          double x = a[c];
#pragma unroll
          for (int q = 0; q < c; ++q) x -= a[q] * sL[c][q];
          a[c] = x / sL[c][c];
        }
        if (gi < n || gi == brow) {
#pragma unroll
          for (int c = 0; c < kCholNB; ++c)
            if (c0 + c < n) Lw[static_cast<size_t>(gi) * n + c0 + c] = a[c];
        }
      }
    }
    grid.sync();
    // ---- phase B: trailing update A_ij -= A_ip A_jp^T for p < j <= i (i over row tiles) ----
    const int nt = TR - (p + 1);   // row tiles below the panel
    const int ntc = T - (p + 1);   // column tiles right of the panel
    // enumerate (ii, jj) with jj < ntc, ii >= jj, ii < nt
    const long long ntiles = static_cast<long long>(ntc) * nt - static_cast<long long>(ntc) * (ntc - 1) / 2;
    for (long long tix = gwarp; tix < ntiles; tix += nwarps) {
      // decode: column jj has (nt - jj) tiles
      int jj = 0;
      long long rem = tix;
      while (rem >= nt - jj) { rem -= nt - jj; ++jj; }
      const int ii = jj + static_cast<int>(rem);
      const int i = p + 1 + ii, j = p + 1 + jj;
      // stage A_ip into this warp's smem tile, keep row `lane` of A_jp in registers
      double (*sa)[kCholNB + 1] = sA[warp];
      for (int rr = 0; rr < kCholNB; ++rr) {
        const int gi = i * kCholNB + rr;
        sa[rr][lane] = ((gi < n || gi == brow) && c0 + lane < n) ? Lw[static_cast<size_t>(gi) * n + c0 + lane] : 0.0;
      }
      double bj[kCholNB];
      {
        const int gj = j * kCholNB + lane;
#pragma unroll
        for (int q = 0; q < kCholNB; ++q) bj[q] = (gj < n && c0 + q < n) ? Lw[static_cast<size_t>(gj) * n + c0 + q] : 0.0;
      }
      __syncwarp();
      const int gcol = j * kCholNB + lane;
      for (int rr = 0; rr < kCholNB; ++rr) {
        const int gi = i * kCholNB + rr;
        if (!(gi < n || gi == brow)) continue;
        double s = 0;
#pragma unroll
        for (int q = 0; q < kCholNB; ++q) s += sa[rr][q] * bj[q];
        if (gcol < n && (gi >= gcol)) Lw[static_cast<size_t>(gi) * n + gcol] -= s;
      }
      __syncwarp();
    }
    grid.sync();
  }
}

// Back-substitution L^T x = y (y = row n of Lw), single CTA of 1024 threads.
__global__ void __launch_bounds__(1024) backsolve_kernel(const double* __restrict__ Lw, const double* __restrict__ Ldiag, int n,
                                                         double* __restrict__ x) {
  __shared__ double part[32][kCholNB + 1];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int T = (n + kCholNB - 1) / kCholNB;
  for (int p = T - 1; p >= 0; --p) {
    const int c0 = p * kCholNB;
    double acc = 0.0;
    const int col = c0 + lane;
    for (int row = (p + 1) * kCholNB + warp; row < n; row += 32)
      if (col < n) acc += Lw[static_cast<size_t>(row) * n + col] * x[row];
    part[warp][lane] = acc;
    __syncthreads();
    if (warp == 0) {
      double rhs = (col < n) ? Lw[static_cast<size_t>(T) * kCholNB * n + col] : 0.0;
      for (int w = 0; w < 32; ++w) rhs -= part[w][lane];
      const double* Ld = Ldiag + static_cast<size_t>(p) * kCholNB * kCholNB;
      double xv = 0.0;
      for (int q = kCholNB - 1; q >= 0; --q) {
        // x_q = rhs_q / L[q][q]; rhs_c -= L[q][c] x_q for c < q
        const double dq = Ld[q * kCholNB + q];
        const double xq = __shfl_sync(0xffffffffu, rhs, q) / dq;
        if (lane == q) xv = xq;
        if (lane < q) rhs -= Ld[q * kCholNB + lane] * xq;
      }
      if (col < n) x[col] = xv;
    }
    __syncthreads();
  }
}

// Ceres SphereManifold<3>::Plus.
HB_DI void sphere_plus(const double* x, const double* delta, double* out) {
  const double nd = sqrt(delta[0] * delta[0] + delta[1] * delta[1]);
  if (nd == 0.0) { out[0] = x[0]; out[1] = x[1]; out[2] = x[2]; return; }
  const double sigma = x[0] * x[0] + x[1] * x[1];
  double v[3] = {x[0], x[1], 1.0};
  double beta = 0.0;
  const double xp = x[2];
  if (sigma <= 2.220446049250313e-16) {
    if (xp < 0.0) beta = 2.0;
  } else {
    const double mu = sqrt(xp * xp + sigma);
    const double vp = (xp <= 0.0) ? (xp - mu) : (-sigma / (xp + mu));
    beta = 2.0 * vp * vp / (sigma + vp * vp);
    v[0] /= vp; v[1] /= vp;
  }
  const double nx = sqrt(sigma + xp * xp);
  const double s = sin(nd) / nd;
  const double y[3] = {s * delta[0], s * delta[1], cos(nd)};
  const double vy = v[0] * y[0] + v[1] * y[1] + v[2] * y[2];
#pragma unroll
  for (int i = 0; i < 3; ++i) out[i] = nx * (y[i] - v[i] * beta * vy);
}

// Manifold::Plus on every variable block: trial = current (+) delta (and the trial state's knot table).
struct RetractArgs {
  int K, Kbg, Kba, L;
  const double *dp, *dl, *knots, *bg, *ba, *grav, *lms;
  double *knots_t, *bg_t, *ba_t, *grav_t, *lms_t, *tab_t /* or null */;
  int retract_landmarks;
};
HB_DI void retract_body(const RetractArgs& ra, int i) {
  const int K = ra.K, Kbg = ra.Kbg, Kba = ra.Kba, L = ra.L, retract_landmarks = ra.retract_landmarks;
  const double* __restrict__ dp = ra.dp; const double* __restrict__ dl = ra.dl; const double* __restrict__ knots = ra.knots;
  const double* __restrict__ bg = ra.bg; const double* __restrict__ ba = ra.ba; const double* __restrict__ grav = ra.grav;
  const double* __restrict__ lms = ra.lms;
  double* __restrict__ knots_t = ra.knots_t; double* __restrict__ bg_t = ra.bg_t; double* __restrict__ ba_t = ra.ba_t;
  double* __restrict__ grav_t = ra.grav_t; double* __restrict__ lms_t = ra.lms_t; double* __restrict__ tab_t = ra.tab_t;
  if (i < K) {
    const double* kn = knots + 8 * static_cast<size_t>(i);
    const double* d = dp + 6 * static_cast<size_t>(i);
    double qe[4], qn[4];
    const double th[3] = {d[0], d[1], d[2]};
    const double q[4] = {kn[0], kn[1], kn[2], kn[3]};
    quat_exp(th, qe);
    quat_mul(qe, q, qn);
    double* o = knots_t + 8 * static_cast<size_t>(i);
    o[0] = qn[0]; o[1] = qn[1]; o[2] = qn[2]; o[3] = qn[3];
    o[4] = kn[4] + d[3]; o[5] = kn[5] + d[4]; o[6] = kn[6] + d[5]; o[7] = kn[7];
    if (tab_t) {
      // the trial state's knot-table row (same arithmetic as prep_kernel): this thread retracts knot i-1 again
      // for the relative rotation instead of waiting for its neighbour
      double qp[4] = {0, 0, 0, 1};
      if (i > 0) {
        const double thp[3] = {d[-6], d[-5], d[-4]};
        const double qo[4] = {kn[-8], kn[-7], kn[-6], kn[-5]};
        double qep[4];
        quat_exp(thp, qep);
        quat_mul(qep, qo, qp);
      }
      knot_table_row(qn, o + 4, o[7], qp, i > 0, tab_t + static_cast<size_t>(i) * kTabStride);
    }
  }
  if (i < Kbg) {
    const double* d = dp + 6 * static_cast<size_t>(K) + 3 * static_cast<size_t>(i);
    for (int c = 0; c < 3; ++c) bg_t[4 * i + c] = bg[4 * i + c] + d[c];
    bg_t[4 * i + 3] = bg[4 * i + 3];
  }
  if (i < Kba) {
    const double* d = dp + 6 * static_cast<size_t>(K) + 3 * static_cast<size_t>(Kbg) + 3 * static_cast<size_t>(i);
    for (int c = 0; c < 3; ++c) ba_t[4 * i + c] = ba[4 * i + c] + d[c];
    ba_t[4 * i + 3] = ba[4 * i + 3];
  }
  if (i == 0) {
    const double* d = dp + 6 * static_cast<size_t>(K) + 3 * static_cast<size_t>(Kbg) + 3 * static_cast<size_t>(Kba);
    const double x[3] = {grav[0], grav[1], grav[2]};
    const double dd[2] = {d[0], d[1]};
    double o[3];
    sphere_plus(x, dd, o);
    grav_t[0] = o[0]; grav_t[1] = o[1]; grav_t[2] = o[2];
  }
  if (retract_landmarks && i < L) {   // otherwise lm_backsub_kernel has written the trial landmarks already
    for (int c = 0; c < 3; ++c) lms_t[3 * static_cast<size_t>(i) + c] = lms[3 * static_cast<size_t>(i) + c] + dl[3 * static_cast<size_t>(i) + c];
  }
}
__global__ void retract_kernel(RetractArgs ra) { retract_body(ra, blockIdx.x * blockDim.x + threadIdx.x); }

// Landmark back-substitution: V dl = -g_l - W^T dp; also partial sums of dl.g_l and dl.D_l.dl.
// One warp per landmark: 8 observations x 4 column groups in flight per pass.
constexpr int kLmWarps = 4;

template <int K>
__global__ void __launch_bounds__(kLmWarps * 32) lm_backsub_kernel(int L, const int* __restrict__ lm_off, const int* __restrict__ lm_obs,
                                                                  const int4* __restrict__ idx, const double* __restrict__ r,
                                                                  const double* __restrict__ Jp, const double* __restrict__ Jl, const double* __restrict__ wv,
                                                                  const double* __restrict__ Vchol, const double* __restrict__ gl,
                                                                  const double* __restrict__ Dl, const double* __restrict__ dp,
                                                                  double* __restrict__ dl, double* __restrict__ part /*[n_lm_blocks][5]*/,
                                                                  const double* __restrict__ lms, double* __restrict__ lms_t,
                                                                  int n_lm_blocks, RetractArgs ra) {
  // blocks past the landmark range retract the knots / biases / gravity in the same launch (they only need dp)
  if (static_cast<int>(blockIdx.x) >= n_lm_blocks) { retract_body(ra, (blockIdx.x - n_lm_blocks) * blockDim.x + threadIdx.x); return; }
  constexpr int NB = 6 * K;
  constexpr int CG = NB / 4;  // columns per lane group
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int l = blockIdx.x * kLmWarps + warp;
  double s_g = 0, s_d = 0, s_step = 0, s_x = 0, s_gmax = 0;   // + |dl|^2, |x_l|^2, |g_l|_inf of the OBSERVED landmarks (termination tests)
  if (l < L) {
    const int o_lo = lm_off[l], o_hi = lm_off[l + 1];
    const int og = lane >> 2, cg = lane & 3;
    double rhs[3] = {0, 0, 0};
    for (int o0 = o_lo; o0 < o_hi; o0 += 8) {
      const int o = o0 + og;
      double t0 = 0, t1 = 0, wgt = 0, jl[6] = {0, 0, 0, 0, 0, 0};
      if (o < o_hi) {
        const int f = lm_obs[o];
        wgt = wv[f];
        const double* jp = Jp + static_cast<size_t>(f) * 2 * NB + cg * CG;
        const double* d = dp + 6 * idx[f].x + cg * CG;
#pragma unroll
        for (int a = 0; a < CG; ++a) { const double dv = d[a]; t0 += jp[a] * dv; t1 += jp[NB + a] * dv; }
        if (cg == 0) {
#pragma unroll
          for (int c = 0; c < 6; ++c) jl[c] = Jl[6 * static_cast<size_t>(f) + c];
        }
      }
      t0 += __shfl_xor_sync(0xffffffffu, t0, 1); t1 += __shfl_xor_sync(0xffffffffu, t1, 1);
      t0 += __shfl_xor_sync(0xffffffffu, t0, 2); t1 += __shfl_xor_sync(0xffffffffu, t1, 2);
      if (cg == 0) {
#pragma unroll
        for (int c = 0; c < 3; ++c) rhs[c] -= wgt * (jl[c] * t0 + jl[3 + c] * t1);
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      rhs[c] += __shfl_xor_sync(0xffffffffu, rhs[c], 4);
      rhs[c] += __shfl_xor_sync(0xffffffffu, rhs[c], 8);
      rhs[c] += __shfl_xor_sync(0xffffffffu, rhs[c], 16);
    }
    if (lane == 0) {
      const double* g = gl + 3 * static_cast<size_t>(l);
#pragma unroll
      for (int c = 0; c < 3; ++c) rhs[c] -= g[c];
      // V dl = rhs through the Schur kernels' packed factor: y = L^-1 rhs, dl = L^-T y (all zero for an unobserved landmark)
      const double* F = Vchol + 9 * static_cast<size_t>(l);
      double y[3], x[3];
      lm_lsolve(F, rhs[0], rhs[1], rhs[2], y);
      x[2] = y[2] * F[5];
      x[1] = (y[1] - F[4] * x[2]) * F[2];
      x[0] = (y[0] - F[1] * x[1] - F[3] * x[2]) * F[0];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const double v = x[c];
        dl[3 * static_cast<size_t>(l) + c] = v;
        if (lms_t) lms_t[3 * static_cast<size_t>(l) + c] = lms[3 * static_cast<size_t>(l) + c] + v;   // Manifold::Plus of the landmark block
        s_g += v * g[c];
        s_d += v * v * Dl[3 * static_cast<size_t>(l) + c];
        if (o_hi > o_lo) {
          const double xl = lms[3 * static_cast<size_t>(l) + c];
          s_step += v * v; s_x += xl * xl; s_gmax = fmax(s_gmax, fabs(g[c]));
        }
      }
    }
  }
  __shared__ double sg[kLmWarps][5];
  if (lane == 0) { sg[warp][0] = s_g; sg[warp][1] = s_d; sg[warp][2] = s_step; sg[warp][3] = s_x; sg[warp][4] = s_gmax; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a[5] = {0, 0, 0, 0, 0};
    for (int w = 0; w < kLmWarps; ++w) { a[0] += sg[w][0]; a[1] += sg[w][1]; a[2] += sg[w][2]; a[3] += sg[w][3]; a[4] = fmax(a[4], sg[w][4]); }
#pragma unroll
    for (int q = 0; q < 5; ++q) part[5 * blockIdx.x + q] = a[q];
  }
}


// scal = [cost_new, dl.g_l, dl.D_l.dl, |dl|^2, |x_l|^2, 0, 0, 0] (rank-local partials, fixed order).
// The paths that can only SUM across ranks (callback hook, NCCL without a peer mapping) run this before their reduction of
// scal.  A sum of per-rank maxima is not the maximum, so the landmark gradient maximum |g_l|_inf is left at 0: after the
// reduction gradient_max_norm covers the replicated blocks only, and hb200_iterate / hb200_optimize refuse a gradient
// tolerance on these paths (the peer mailbox in accept_kernel takes the true maximum).
__global__ void scalars_kernel(const double* __restrict__ cp_pix, int n_pix_blocks, const double* __restrict__ cp_imu, int n_imu_blocks,
                               const double* __restrict__ lm_part, int n_lm_blocks, double* __restrict__ scal) {
  __shared__ double s[5][256];
  double v[5] = {0, 0, 0, 0, 0};
  for (int i = threadIdx.x; i < n_pix_blocks; i += blockDim.x) v[0] += cp_pix[i];
  for (int i = threadIdx.x; i < n_imu_blocks; i += blockDim.x) v[0] += cp_imu[i];
  for (int i = threadIdx.x; i < n_lm_blocks; i += blockDim.x) {
    v[1] += lm_part[5 * i]; v[2] += lm_part[5 * i + 1]; v[3] += lm_part[5 * i + 2]; v[4] += lm_part[5 * i + 3];
  }
#pragma unroll
  for (int q = 0; q < 5; ++q) s[q][threadIdx.x] = v[q];
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
#pragma unroll
      for (int q = 0; q < 5; ++q) s[q][threadIdx.x] += s[q][threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
#pragma unroll
    for (int q = 0; q < 5; ++q) scal[q] = s[q][0];
    scal[5] = 0.0; scal[6] = 0.0; scal[7] = 0.0;
  }
}

// Step acceptance (Ceres TrustRegionMinimizer + LevenbergMarquardtStrategy::StepAccepted/Rejected).
struct CommitArgs {
  size_t count[5];
  const double* src[5];
  double* dst[5];
};

struct ScalarArgs {   // inputs of scalars_kernel, for the fused single-GPU path
  const double* cp_pix; int n_pix_blocks; const double* cp_imu; int n_imu_blocks; const double* lm_part; int n_lm_blocks;
};

// Multi-GPU step acceptance without a second collective call: every rank's trial-cost / model-decrease partials
// (3 doubles) travel through PEER MEMORY inside accept_kernel itself -- thread p stores this rank's triple and a
// sequence tag into rank p's mailbox over NVLink (st.release.sys) and waits for rank p's triple in its own
// (ld.acquire.sys); the sums are taken in rank order, so every replica computes bit-identical rho / radius.
// Mailbox: [2 parities][kMaxRanks][8] doubles = {cost_new, dl.g_l, dl.D_l.dl, |dl|^2, |x_l|^2, |g_l|_inf, -, tag}
// (sums for the first five, maximum for the sixth: the landmark parts of Ceres' termination tests).  Slots alternate with the
// sequence parity; a slot is not reused before the next system all-reduce has synchronised all ranks.
constexpr int kMaxRanks = 16;
constexpr int kMboxSlot = 8;
struct MailboxArgs {
  int nranks, rank;
  double* const* peers;        // [nranks] mailbox base of every rank, mapped into this process (cudaIpcOpenMemHandle)
  double* local;               // this rank's own mailbox
  unsigned long long* seq;     // exchanges completed so far (device counter, identical on every rank)
};
HB_DI void st_release_sys_u64(unsigned long long* p, unsigned long long v) { asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
HB_DI unsigned long long ld_acquire_sys_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
HB_DI void st_relaxed_sys_f64(double* p, double v) { asm volatile("st.relaxed.sys.global.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory"); }
HB_DI double ld_relaxed_sys_f64(const double* p) {
  double v;
  asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
  return v;
}

// ---------------------------------------------------------------------------------------------
// The system reduction over peer memory: barrier + all-reduce in ONE kernel, no library call.
// Every rank's partial packed system sits in its peer arena (mapped into every process with cudaIpcOpenMemHandle).
// CTA 0 tells every peer "my partial of round `want` is complete" (one st.release.sys per peer into the peer's flag
// row); every CTA waits until all ranks' flags of this round have arrived in the LOCAL flag row, then the grid sums
// the N partials straight out of the peers' HBM over NVLink (ld.relaxed.sys, 16 B per lane) in RANK ORDER -- every
// replica computes bit-identical sums -- into the local reduced system the solver reads.  Nothing is written to a
// peer except the flags, so no second barrier is needed: partials alternate between two arena halves (A / B by
// iteration parity) and a rank cannot run two rounds ahead of a peer it has to wait for.
// The last CTA to finish advances the round counter (all CTAs read it first: no CTA can see the new value early).
// Arena layout (doubles): [mailbox 2 x kMaxRanks x kMboxSlot | flags kMaxRanks | partial A cap | partial B cap].
// ---------------------------------------------------------------------------------------------
constexpr int kArenaFlags = 2 * kMaxRanks * kMboxSlot;        // offset of the flag row
constexpr int kArenaParts = kArenaFlags + 2 * kMaxRanks;      // offset of partial A (16-byte aligned)
constexpr int kReduceThreads = 256;
struct PeerReduceArgs {
  int nranks, rank;
  double* const* peers;          // arena base of every rank in this process' address space
  double* local;                 // own arena
  long long part_offset, total;  // active partial (offset in doubles inside the arena), doubles to reduce
  double* out;                   // local reduced system
  unsigned long long* round;     // rounds completed (device counter, identical on every rank)
  unsigned int* arrive;          // CTAs finished in this launch
  SolverState* st;               // comm_error on a timeout
};
HB_DI double2 ld_relaxed_sys_f64x2(const double* p) {
  double2 v;
  asm volatile("ld.relaxed.sys.global.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "l"(p) : "memory");
  return v;
}
// 16-byte asynchronous copy global -> shared, L2 only (LDGSTS.BYPASS): the eight peers' reads of one element group are all
// in flight before the first one is waited for.  (Plain or asm loads do not achieve that here: ptxas schedules the rank-order
// additions between the STRONG.SYS loads and the in-order issue then serialises the NVLink round trips.)
HB_DI void cp_async_16(void* smem, const void* gptr) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(smem))), "l"(gptr) : "memory");
}
__global__ void __launch_bounds__(kReduceThreads) peer_reduce_kernel(PeerReduceArgs a) {
  __shared__ int s_bad;
  __shared__ const double* s_part[kMaxRanks];   // every rank's active partial (the pointer table is read once, before the wait)
  __shared__ __align__(16) double2 s_v[8][kReduceThreads];
  const unsigned long long want = *reinterpret_cast<volatile unsigned long long*>(a.round) + 1;
  const int tid = threadIdx.x;
  if (tid == 0) s_bad = 0;
  if (tid < a.nranks) s_part[tid] = a.peers[tid] + a.part_offset;
  __syncthreads();
  if (blockIdx.x == 0 && tid < a.nranks)
    st_release_sys_u64(reinterpret_cast<unsigned long long*>(a.peers[tid] + kArenaFlags) + a.rank, want);
  if (tid < a.nranks) {
    const unsigned long long* flag = reinterpret_cast<const unsigned long long*>(a.local + kArenaFlags) + tid;
    const long long t0 = clock64();
    while (ld_acquire_sys_u64(flag) < want) {
      if (clock64() - t0 > 6000000000LL) { s_bad = 1; break; }   // ~3 s: a peer died; report instead of hanging the GPU
    }
  }
  __syncthreads();
  const long long pairs = a.total / 2;   // total is even (SysLayout)
  for (long long e = blockIdx.x * static_cast<long long>(kReduceThreads) + tid; e < pairs; e += static_cast<long long>(gridDim.x) * kReduceThreads) {
    double2 acc = make_double2(0.0, 0.0);
    // eight peers' loads are in flight together (one NVLink round trip per group, not one per rank); the sum stays in rank order
    for (int p0 = 0; p0 < a.nranks; p0 += 8) {
#pragma unroll
      for (int u = 0; u < 8; ++u)
        if (p0 + u < a.nranks) cp_async_16(&s_v[u][tid], s_part[p0 + u] + 2 * e);
      asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
#pragma unroll
      for (int u = 0; u < 8; ++u)
        if (p0 + u < a.nranks) { const double2 v = s_v[u][tid]; acc.x += v.x; acc.y += v.y; }
    }
    reinterpret_cast<double2*>(a.out)[e] = acc;
  }
  __syncthreads();
  if (tid == 0) {
    if (s_bad) a.st->comm_error = 1;
    __threadfence();
    if (atomicAdd(a.arrive, 1u) == gridDim.x - 1) { *a.arrive = 0; __threadfence(); *a.round = want; }
  }
}

constexpr int kAcceptThreads = 1024;   // one CTA; wide so that the fused commit copies the state in a few passes

// ceres::TrustRegionMinimizer termination tests (Ceres 2.x trust_region_minimizer.cc, restated from the public
// sources -- the reference leaves them at their defaults, reference optimizer.cpp:38-54):
//   gradient tolerance   |x - Plus(x, -g)|_inf <= gradient_tolerance at the linearisation point (IterationZero /
//                        HandleSuccessfulStep): the solve ends BEFORE this iteration's step is taken;
//   parameter tolerance  |x - x_trial| <= parameter_tolerance (|x| + parameter_tolerance), ambient norms over the
//                        non-constant parameter blocks: ends without applying the trial step;
//   function tolerance   |cost - cost_trial| <= function_tolerance cost: ends without applying the trial step;
//   minimum trust-region radius, five consecutive invalid (non positive definite) steps.
struct TermArgs {
  int enabled;
  double function_tolerance, gradient_tolerance, parameter_tolerance, min_radius;
  int K, Kbg, Kba;
  const double *knots, *knots_t, *bg, *bg_t, *ba, *ba_t, *grav, *grav_t;
};

__global__ void __launch_bounds__(kAcceptThreads) accept_kernel(const double* __restrict__ sys, SysLayout lay, double* __restrict__ scal, const double* __restrict__ dp,
                              const double* __restrict__ D, const unsigned char* __restrict__ fixed, SolverState* st,
                              const int* __restrict__ spd_flag, SolverState* __restrict__ record, int max_records, int fuse_scalars,
                              ScalarArgs sa, int fuse_commit, CommitArgs ca, MailboxArgs mb, TermArgs ta) {
  // block reductions: shuffle within the warp, one partial per warp, fixed order across warps.
  // v[0..5]: cost_new, dl.g_l, dl.D_l.dl, |dl|^2, |x_l|^2, |g_l|_inf (landmark partials of this rank)
  // v[6..7]: dp.g, dp.D.dp        v[8..10]: |x_trial - x|^2, |x|^2, |x - Plus(x, -g)|_inf of the knots / biases / gravity
  constexpr int NV = 11;
  __shared__ double s[NV][kAcceptThreads / 32];
  __shared__ int s_done;
  const int wl = threadIdx.x & 31, ww = threadIdx.x >> 5;
  if (st->terminated) {   // the solve has ended: later iterations of the same call leave everything alone
    if (threadIdx.x == 0 && mb.nranks > 1 && fuse_scalars) *mb.seq += 1;   // (the peers skip their exchange too: keep the counters aligned)
    return;
  }
  double v[NV];
#pragma unroll
  for (int q = 0; q < NV; ++q) v[q] = 0.0;
  if (fuse_scalars) {   // == scalars_kernel (no all-reduce between the two on a single GPU)
    for (int i = threadIdx.x; i < sa.n_pix_blocks; i += blockDim.x) v[0] += sa.cp_pix[i];
    for (int i = threadIdx.x; i < sa.n_imu_blocks; i += blockDim.x) v[0] += sa.cp_imu[i];
    for (int i = threadIdx.x; i < sa.n_lm_blocks; i += blockDim.x) {
      v[1] += sa.lm_part[5 * i]; v[2] += sa.lm_part[5 * i + 1]; v[3] += sa.lm_part[5 * i + 2]; v[4] += sa.lm_part[5 * i + 3];
      v[5] = fmax(v[5], sa.lm_part[5 * i + 4]);
    }
  }
  const int n = lay.n;
  const double* g = sys + lay.og;
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    if (!fixed[i]) { v[6] += dp[i] * g[i]; v[7] += dp[i] * dp[i] * D[i]; }
  if (ta.enabled) {
    // ambient norms over the non-constant blocks (Stamped<SE3>: 8 coordinates, the stamp included; bias knots 4; gravity 3)
    // and the projected gradient step: Ceres' local rotation coordinate is half of this library's theta, so
    // Plus(x, -g_ceres) is a rotation by -4 g_theta.
    const int i = threadIdx.x;
    for (int j = i; j < ta.K; j += blockDim.x) {
      if (fixed[6 * j]) continue;
      const double* x = ta.knots + 8 * static_cast<size_t>(j);
      const double* t = ta.knots_t + 8 * static_cast<size_t>(j);
#pragma unroll
      for (int c = 0; c < 8; ++c) { const double d = t[c] - x[c]; v[8] += d * d; v[9] += x[c] * x[c]; }
      const double th[3] = {-4.0 * g[6 * j], -4.0 * g[6 * j + 1], -4.0 * g[6 * j + 2]};
      const double q[4] = {x[0], x[1], x[2], x[3]};
      double qe[4], qn[4];
      quat_exp(th, qe);
      quat_mul(qe, q, qn);
#pragma unroll
      for (int c = 0; c < 4; ++c) v[10] = fmax(v[10], fabs(qn[c] - q[c]));
#pragma unroll
      for (int c = 0; c < 3; ++c) v[10] = fmax(v[10], fabs(g[6 * j + 3 + c]));
    }
    const int o_bg = 6 * ta.K, o_ba = o_bg + 3 * ta.Kbg, o_g = o_ba + 3 * ta.Kba;
    for (int j = i; j < ta.Kbg + ta.Kba; j += blockDim.x) {
      const bool acc = j >= ta.Kbg;
      const int jj = acc ? j - ta.Kbg : j, o = (acc ? o_ba : o_bg) + 3 * jj;
      if (fixed[o]) continue;
      const double* x = (acc ? ta.ba : ta.bg) + 4 * static_cast<size_t>(jj);
      const double* t = (acc ? ta.ba_t : ta.bg_t) + 4 * static_cast<size_t>(jj);
#pragma unroll
      for (int c = 0; c < 4; ++c) { const double d = t[c] - x[c]; v[8] += d * d; v[9] += x[c] * x[c]; }
#pragma unroll
      for (int c = 0; c < 3; ++c) v[10] = fmax(v[10], fabs(g[o + c]));
    }
    if (i == 0 && !fixed[o_g]) {
      const double x[3] = {ta.grav[0], ta.grav[1], ta.grav[2]};
      const double dd[2] = {-g[o_g], -g[o_g + 1]};
      double xp[3];
      sphere_plus(x, dd, xp);
#pragma unroll
      for (int c = 0; c < 3; ++c) { const double d = ta.grav_t[c] - x[c]; v[8] += d * d; v[9] += x[c] * x[c]; v[10] = fmax(v[10], fabs(xp[c] - x[c])); }
    }
  }
#pragma unroll
  for (int q = 0; q < NV; ++q) {
    const bool is_max = (q == 5 || q == 10);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const double y = __shfl_xor_sync(0xffffffffu, v[q], o); v[q] = is_max ? fmax(v[q], y) : v[q] + y; }
    if (wl == 0) s[q][ww] = v[q];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double t[NV];
#pragma unroll
    for (int q = 0; q < NV; ++q) t[q] = 0.0;
    for (int w = 0; w < kAcceptThreads / 32; ++w)
#pragma unroll
      for (int q = 0; q < NV; ++q) t[q] = (q == 5 || q == 10) ? fmax(t[q], s[q][w]) : t[q] + s[q][w];
    if (fuse_scalars) {
#pragma unroll
      for (int q = 0; q < 6; ++q) scal[q] = t[q];
      scal[6] = 0.0; scal[7] = 0.0;
    }
#pragma unroll
    for (int q = 0; q < NV; ++q) s[q][0] = t[q];
  }
  __syncthreads();
  if (fuse_scalars && mb.nranks > 1) {
    __shared__ double s_peer[kMaxRanks][6];
    __shared__ int s_timeout;
    const unsigned long long want = *mb.seq + 1;   // every thread reads the counter before thread 0 bumps it (below)
    const int par = static_cast<int>(want & 1);
    if (threadIdx.x == 0) s_timeout = 0;
    __syncthreads();
    if (static_cast<int>(threadIdx.x) < mb.nranks) {
      const int p = threadIdx.x;
      double* dst = mb.peers[p] + (par * kMaxRanks + mb.rank) * kMboxSlot;
#pragma unroll
      for (int q = 0; q < 6; ++q) st_relaxed_sys_f64(dst + q, s[q][0]);
      st_release_sys_u64(reinterpret_cast<unsigned long long*>(dst + 7), want);
      const double* src = mb.local + (par * kMaxRanks + p) * kMboxSlot;
      const long long t0 = clock64();
      bool ok = true;
      while (ld_acquire_sys_u64(reinterpret_cast<const unsigned long long*>(src + 7)) != want) {
        if (clock64() - t0 > 6000000000LL) { ok = false; break; }   // ~3 s: a peer died; report instead of hanging the GPU
      }
      if (!ok) s_timeout = 1;
#pragma unroll
      for (int q = 0; q < 6; ++q) s_peer[p][q] = ld_relaxed_sys_f64(src + q);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      double a[6] = {0, 0, 0, 0, 0, 0};
      for (int p = 0; p < mb.nranks; ++p) {   // rank order: identical on every rank
#pragma unroll
        for (int q = 0; q < 5; ++q) a[q] += s_peer[p][q];
        a[5] = fmax(a[5], s_peer[p][5]);
      }
#pragma unroll
      for (int q = 0; q < 6; ++q) scal[q] = a[q];
      *mb.seq = want;
      if (s_timeout) st->comm_error = 1;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    s_done = 0;
    const double mu = 1.0 / st->radius;
    const double cost = sys[lay.os];
    const double cost_new = scal[0];
    const double dg = s[6][0] + scal[1], dDd = s[7][0] + scal[2];
    const double model = 0.5 * (-dg + mu * dDd);
    const double rho = (cost - cost_new) / model;
    const int spd = *spd_flag;
    int term = 0;
    if (ta.enabled) {
      const double gmax = fmax(s[10][0], scal[5]);
      const double step_norm = sqrt(s[8][0] + scal[3]), x_norm = sqrt(s[9][0] + scal[4]);
      st->gradient_max_norm = gmax; st->step_norm = step_norm; st->x_norm = x_norm;
      if (ta.gradient_tolerance > 0.0 && gmax <= ta.gradient_tolerance) term = 3;
      else if (spd && ta.parameter_tolerance > 0.0 && step_norm <= ta.parameter_tolerance * (x_norm + ta.parameter_tolerance)) term = 2;
      else if (spd && ta.function_tolerance > 0.0 && fabs(cost - cost_new) <= ta.function_tolerance * cost) term = 1;
    }
    if (term) {   // the solve ends here; this iteration's step is not applied and not counted (Ceres returns before IsStepSuccessful)
      st->terminated = term; st->accepted = 0;
      st->cost = cost; st->cost_new = cost_new; st->model_change = model; st->rho = rho; st->spd = spd;
      s_done = 1;
    } else {
      st->cost = cost; st->cost_new = cost_new; st->model_change = model; st->rho = rho; st->spd = spd;
      if (spd && model > 0.0 && rho > 1e-3) {
        st->accepted = 1;
        const double t = 2.0 * rho - 1.0;
        st->radius = fmin(1e16, st->radius / fmax(1.0 / 3.0, 1.0 - t * t * t));
        st->decrease_factor = 2.0;
      } else {
        st->accepted = 0;
        st->radius = st->radius / st->decrease_factor;
        st->decrease_factor *= 2.0;
      }
      st->invalid_steps = spd ? 0 : st->invalid_steps + 1;
      st->iteration += 1;
      if (ta.enabled) {
        if (st->invalid_steps >= 5) st->terminated = 5;
        else if (ta.min_radius > 0.0 && st->radius <= ta.min_radius) st->terminated = 4;
      }
      if (record) record[(st->iteration - 1) % max_records] = *st;   // ring buffer, host tracks the index
    }
  }
  if (fuse_commit) {   // small windows: the accepted trial state is committed by this CTA (== commit_kernel)
    __syncthreads();
    if (st->accepted && !s_done) {
#pragma unroll
      for (int q = 0; q < 5; ++q)
        for (size_t i = threadIdx.x; i < ca.count[q]; i += blockDim.x) ca.dst[q][i] = ca.src[q][i];
    }
  }
}

// start of a solve: clean termination state; reset_radius: ceres::Solve starts every call at initial_trust_region_radius
__global__ void new_solve_kernel(SolverState* st, double radius0, int reset_radius) {
  st->terminated = 0; st->invalid_steps = 0;
  if (reset_radius) { st->radius = radius0; st->decrease_factor = 2.0; }
}

// unconditional segmented copy (host staging buffer <-> variable blocks in hb200_optimize)
__global__ void copy_segments_kernel(CommitArgs a) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
#pragma unroll
  for (int s = 0; s < 5; ++s)
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < a.count[s]; i += stride) a.dst[s][i] = a.src[s][i];
}

__global__ void commit_kernel(const SolverState* __restrict__ st, CommitArgs a) {
  if (!st->accepted) return;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
#pragma unroll
  for (int s = 0; s < 5; ++s)
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < a.count[s]; i += stride) a.dst[s][i] = a.src[s][i];
}

}  // namespace hb
