// Multi-CTA solve of the reduced system for LONG windows (sm_90a): block cyclic reduction.
//
// band_solve_kernel factors the block-banded + arrowhead system (SysLayout) in ONE CTA: K/2 + beta dependent
// block-column steps, which at K = 200 .. 500 takes longer than every other kernel of the iteration together,
// and replicated on every rank of a multi-GPU solve.  Here the chain is replaced by a tree.
// The pose part is cut into super-blocks of beta control points (nb = 6 beta dofs): a half-bandwidth of beta
// blocks makes the super-block matrix block-TRIDIAGONAL (D_j on the diagonal, B_j = A[j+1][j] below it), with the
// arrow rows F_j (m x nb) and the corner C (m x m) attached.  Cyclic reduction eliminates every other
// super-block of the current level at once -- they do not couple to each other -- one CTA per eliminated node:
//
//   phase 1 (odd node i, neighbours a = i - s, c = i + s, s = 2^level):
//       L L^T = D_i ;  [Y_a | Y_c | Y_f | y] = L^-1 [B_a | B_i^T | F_i^T | b_i]          (kept for the way back)
//   phase 2 (even node e): Schur complements of its two eliminated neighbours
//       D_e -= Y_c(e-s)^T Y_c(e-s) + Y_a(e+s)^T Y_a(e+s)        F_e, b_e alike
//       B_e  = -Y_c(e+s)^T Y_a(e+s)                             (new coupling e -> e + 2s)
//
// and the even nodes form the next, half as long, block-tridiagonal level: ceil(log2(K / beta)) levels instead
// of K / 2 steps.  The arrow x arrow corner receives C -= sum_i Y_f(i)^T Y_f(i) once, after the last level
// (per-CTA partial sums reduced in a fixed order), is factored by CTA 0, and the solution flows back down the
// tree: x_i = L^-T (y - Y_a x_a - Y_c x_c - Y_f x_arrow), one level per grid synchronisation.
// LM damping mu clamp(diag H) and the constant-dof mask are applied while gathering, as in band_solve_kernel.
// Cooperative launch; everything between the levels lives in a global-memory workspace (a few MB, L2-resident).
// The reference hands this system to CHOLMOD through SPARSE_NORMAL_CHOLESKY, single-threaded
// (reference internal/hyper/optimizers/ceres/optimizer.cpp:41,46-48).
#pragma once
#include "hb200_band.cuh"

namespace hb {

constexpr int kBcrThreads = 512;
constexpr int kBcrMaxNb = 48;     // 6 * beta <= 48: landmark tracks of up to 8 control points

struct BcrPlan {
  int nb, nsb, m, levels;
  long long oD, oB, oF, ob, oL, oYa, oYc, oYf, oy, oG, node_stride;   // per-node offsets (doubles)
  long long oCC, oCCp, oXa, total;                                 // global part (after nsb nodes)
};
__host__ __device__ inline BcrPlan bcr_plan(int K, int beta, int m, int num_ctas) {
  BcrPlan p;
  p.nb = 6 * beta; p.nsb = (K + beta - 1) / beta; p.m = m;
  p.levels = 0;
  while ((1 << p.levels) < p.nsb) p.levels += 1;
  const long long nn = static_cast<long long>(p.nb) * p.nb, mn = static_cast<long long>(m) * p.nb;
  p.oD = 0; p.oB = nn; p.oF = 2 * nn; p.ob = p.oF + mn; p.oL = p.ob + p.nb; p.oYa = p.oL + nn; p.oYc = p.oYa + nn;
  p.oYf = p.oYc + nn; p.oy = p.oYf + mn;
  // G = Y^T Y (lower, [nc][nc], nc = 2 nb + m + 1): the Schur-complement blocks an eliminated node hands to its
  // even neighbours and to the corner (Gram pass of phase 1)
  p.oG = p.oy + p.nb;
  const long long nc = 2LL * p.nb + m + 1;
  p.node_stride = (p.oG + nc * nc + 1) & ~1LL;
  p.oCC = p.node_stride * p.nsb;
  p.oCCp = p.oCC + static_cast<long long>(m + 1) * m;
  p.oXa = p.oCCp + static_cast<long long>(num_ctas) * (m + 1) * m;
  p.total = p.oXa + m + 2;
  return p;
}

// software grid barrier (all CTAs co-resident: cooperative launch).  Monotonic counter, one arrival per CTA.
HB_DI void bcr_grid_sync(unsigned int* counter, unsigned int* phase_local) {
  __syncthreads();
  if (threadIdx.x == 0) {
    *phase_local += 1;
    const unsigned int target = *phase_local * gridDim.x;
    __threadfence();
    atomicAdd(counter, 1u);
    while (*reinterpret_cast<volatile unsigned int*>(counter) < target) {}
    __threadfence();
  }
  __syncthreads();
}

// In-place Cholesky of the n x n SPD matrix in shared memory (row stride ld, n a multiple of 6) by the whole CTA,
// blocked by 6 so that every inner loop is a fixed-size register kernel (the scalar right-looking form spent
// ~450 cycles per column on exposed shared-memory latency): per block column, thread 0 factors the 6 x 6 diagonal
// block in registers (chol6), one thread per row solves the 6-wide panel, every thread updates its own
// elements of the trailing matrix with a 6-term dot product.  Three barriers per block column.
// inv[] receives the reciprocal diagonal.
__device__ __noinline__ void bcr_chol(double* A, int ld, int n, double* inv, int* s_flag) {
  const int tid = threadIdx.x;
  const int ntri = n * (n + 1) / 2;
  int eu[3], ev[3];   // fixed element ownership of the trailing update (n <= 54: at most 3 elements per thread)
#pragma unroll
  for (int w = 0; w < 3; ++w) {
    const int e = tid + w * kBcrThreads;
    eu[w] = 0; ev[w] = -1;
    if (e < ntri) {
      int u = static_cast<int>((sqrtf(8.0f * e + 1.0f) - 1.0f) * 0.5f);
      while (u * (u + 1) / 2 > e) --u;
      while ((u + 1) * (u + 2) / 2 <= e) ++u;
      eu[w] = u; ev[w] = e - u * (u + 1) / 2;
    }
  }
  for (int k0 = 0; k0 < n; k0 += 6) {
    if (tid == 0) { if (!chol6(A + k0 * ld + k0, ld, inv + k0)) *s_flag = 0; }
    __syncthreads();
    for (int r = k0 + 6 + tid; r < n; r += kBcrThreads) {   // panel: x L_kk^T = a
      double* a = A + r * ld + k0;
      double v[6];
#pragma unroll
      for (int q = 0; q < 6; ++q) v[q] = a[q];
#pragma unroll
      for (int j = 0; j < 6; ++j) {
        v[j] *= inv[k0 + j];
#pragma unroll
        for (int q = j + 1; q < 6; ++q) v[q] -= v[j] * A[(k0 + q) * ld + k0 + j];
      }
#pragma unroll
      for (int q = 0; q < 6; ++q) a[q] = v[q];
    }
    __syncthreads();
#pragma unroll
    for (int w = 0; w < 3; ++w) {
      if (ev[w] >= k0 + 6) {
        const double* pu = A + eu[w] * ld + k0;
        const double* pv = A + ev[w] * ld + k0;
        double acc = 0.0;
#pragma unroll
        for (int j = 0; j < 6; ++j) acc += pu[j] * pv[j];
        A[eu[w] * ld + ev[w]] -= acc;
      }
    }
    __syncthreads();
  }
}

// Forward substitution Y = L^-1 R in place, one right-hand-side column per thread, blocked by 6: the six unknowns of
// a block live in registers (triangular solve, then an axpy sweep over the rows below) -- no dependence through
// shared memory inside a block, four independent rows in flight in the sweep.
__device__ __noinline__ void bcr_forward(const double* L, int ldl, const double* inv, int n, double* R, int ldr, int ncols) {
  for (int t = threadIdx.x; t < ncols; t += kBcrThreads) {
    for (int k0 = 0; k0 < n; k0 += 6) {
      double y[6];
#pragma unroll
      for (int j = 0; j < 6; ++j) y[j] = R[(k0 + j) * ldr + t];
#pragma unroll
      for (int j = 0; j < 6; ++j) {
        y[j] *= inv[k0 + j];
#pragma unroll
        for (int q = j + 1; q < 6; ++q) y[q] -= y[j] * L[(k0 + q) * ldl + k0 + j];
      }
#pragma unroll
      for (int j = 0; j < 6; ++j) R[(k0 + j) * ldr + t] = y[j];
#pragma unroll 2
      for (int r = k0 + 6; r < n; ++r) {
        const double* lr = L + r * ldl + k0;
        double acc = R[r * ldr + t];
#pragma unroll
        for (int j = 0; j < 6; ++j) acc -= lr[j] * y[j];
        R[r * ldr + t] = acc;
      }
    }
  }
}

// x = L^-T v (n <= 64) by one warp: lane holds v_r (and v_{r+32}); the solved component is broadcast with one
// shuffle, everybody subtracts its multiple -- row q of L is contiguous.  Call from all 32 lanes of warp 0.
__device__ __noinline__ void bcr_backward_warp(const double* L, int ldl, int n, const double* v_in, double* x_out) {
  const int lane = threadIdx.x & 31;
  double v0 = (lane < n) ? v_in[lane] : 0.0, v1 = (lane + 32 < n) ? v_in[lane + 32] : 0.0;
  const double d0 = (lane < n) ? 1.0 / L[lane * ldl + lane] : 0.0, d1 = (lane + 32 < n) ? 1.0 / L[(lane + 32) * ldl + lane + 32] : 0.0;
  for (int q = n - 1; q >= 0; --q) {
    const double cand = (q >= 32) ? v1 * d1 : v0 * d0;
    const double xq = __shfl_sync(0xffffffffu, cand, q & 31);
    if (lane == (q & 31)) x_out[q] = xq;
    const double* lq = L + q * ldl;
    if (lane < q) v0 -= lq[lane] * xq;
    if (lane + 32 < q) v1 -= lq[lane + 32] * xq;
  }
}
// y = L^-1 v, same layout (forward): column q of L is strided, so the multiplier comes from L[r][q] of the lane's own row.
__device__ __noinline__ void bcr_forward_warp(const double* L, int ldl, int n, const double* v_in, double* y_out) {
  const int lane = threadIdx.x & 31;
  double v0 = (lane < n) ? v_in[lane] : 0.0, v1 = (lane + 32 < n) ? v_in[lane + 32] : 0.0;
  const double d0 = (lane < n) ? 1.0 / L[lane * ldl + lane] : 0.0, d1 = (lane + 32 < n) ? 1.0 / L[(lane + 32) * ldl + lane + 32] : 0.0;
  for (int q = 0; q < n; ++q) {
    const double cand = (q >= 32) ? v1 * d1 : v0 * d0;
    const double yq = __shfl_sync(0xffffffffu, cand, q & 31);
    if (lane == (q & 31)) y_out[q] = yq;
    if (lane > q && lane < n) v0 -= L[lane * ldl + q] * yq;
    if (lane + 32 > q && lane + 32 < n) v1 -= L[(lane + 32) * ldl + q] * yq;
  }
}

// Gram pass: G = Y^T Y (lower triangle, row-major [nc][nc] in global memory) of the n x nc matrix Y in shared memory
// on the FP64 tensor cores (mma.sync m8n8k4 -> DMMA.8x8x4): one 8 x 8 output tile per warp pass, contraction over
// the n rows in steps of 4.  Deliberately a small out-of-line loop: this code runs once per node, and one-shot
// code is bound by instruction fetch, not issue (tools/microbench).
__device__ __noinline__ void bcr_gram(const double* Y, int ldy, int n, int nc, double* G) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, lr = lane >> 2, lk = lane & 3;
  const int T = (nc + 7) / 8, ntiles = T * (T + 1) / 2;
  for (int tile = warp; tile < ntiles; tile += kBcrThreads / 32) {
    int ti = 0;
    while ((ti + 1) * (ti + 2) / 2 <= tile) ++ti;
    const int tj = tile - ti * (ti + 1) / 2;
    const int ca = 8 * ti + lr, cb = 8 * tj + lr;
    const bool va = ca < nc, vb = cb < nc;
    double c0 = 0.0, c1 = 0.0;
    const double* pa = Y + lk * ldy + (va ? ca : 0);
    const double* pb = Y + lk * ldy + (vb ? cb : 0);
    for (int k0 = 0; k0 < n; k0 += 16) {   // four k-steps per round: eight loads in flight, then the dependent DMMA chain
      double av[4], bv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const bool in = k0 + 4 * u + lk < n;
        av[u] = (in && va) ? pa[(k0 + 4 * u) * ldy] : 0.0;
        bv[u] = (in && vb) ? pb[(k0 + 4 * u) * ldy] : 0.0;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(av[u]), "d"(bv[u]));
    }
    const int row = 8 * ti + lr, col = 8 * tj + 2 * lk;
    if (row < nc) {
      if (col <= row) G[row * nc + col] = c0;
      if (col + 1 <= row) G[row * nc + col + 1] = c1;
    }
  }
}

__global__ void __launch_bounds__(kBcrThreads) bcr_solve_kernel(const double* __restrict__ sys, SysLayout lay, BcrPlan pl, double* ws,
                                                                unsigned int* barrier, double* x_out, int* __restrict__ spd_flag,
                                                                const SolverState* __restrict__ st, const unsigned char* __restrict__ fixed,
                                                                double* __restrict__ Dout, long long* __restrict__ dbg) {
  extern __shared__ double s_bcr[];
  int n_stamp = 0;
  auto stamp = [&]() {   // HB200_BAND_TIMING=1: phase boundaries of CTA 0 in ns (globaltimer)
    if (dbg && blockIdx.x == 0 && threadIdx.x == 0 && n_stamp < 70) { long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); dbg[1 + n_stamp++] = t; }
  };
  stamp();
  __shared__ int s_ok;
  __shared__ unsigned int s_phase;
  const int tid = threadIdx.x, cta = blockIdx.x, nctas = gridDim.x;
  const int nb = pl.nb, nsb = pl.nsb, m = pl.m, np = lay.np, n = lay.n, beta = lay.beta;
  if (tid == 0) { s_ok = 1; s_phase = *reinterpret_cast<volatile unsigned int*>(barrier) / gridDim.x; }   // counter persists across launches (multiple of gridDim.x)
  __syncthreads();
  auto node = [&](int j) -> double* { return ws + pl.node_stride * j; };
  const double mu = 1.0 / st->radius;
  // ---- gather: band-only packed system -> block-tridiagonal nodes, damping + mask applied ----
  for (int j = cta; j < nsb; j += nctas) {
    double* N = node(j);
    const int r0 = nb * j;   // first dof of the super-block
    for (int e = tid; e < nb * nb; e += kBcrThreads) {
      const int u = e / nb, v = e - u * nb;
      const int row = r0 + u, col = r0 + v;
      double d = 0.0;
      if (row < np && col < np) {
        const int hi = max(row, col), lo = min(row, col);
        d = sys[sys_index(lay, hi, lo)];
        if (row == col) d += mu * fmin(fmax(sys[lay.oD + row], 1e-6), 1e32);
        if (fixed[row] | fixed[col]) d = (row == col) ? 1.0 : 0.0;
      } else if (row == col) d = 1.0;   // padding of the last super-block
      N[pl.oD + e] = d;
      // B_j = A[j+1][j]: rows of super-block j + 1, columns of j; inside the band iff row - 6 (col / 6) < h
      const int rowb = r0 + nb + u;
      double b = 0.0;
      if (rowb < np && col < np && rowb - 6 * (col / 6) < lay.h && !(fixed[rowb] | fixed[col])) b = sys[sys_index(lay, rowb, col)];
      N[pl.oB + e] = b;
    }
    for (int e = tid; e < m * nb; e += kBcrThreads) {
      const int r = e / nb, v = e - r * nb;
      const int col = r0 + v;
      double f = 0.0;
      if (col < np && !(fixed[np + r] | fixed[col])) f = sys[lay.oA + static_cast<long long>(r) * np + col];
      N[pl.oF + e] = f;
    }
    for (int v = tid; v < nb; v += kBcrThreads) {
      const int col = r0 + v;
      N[pl.ob + v] = (col < np && !fixed[col]) ? sys[lay.ob + col] - sys[lay.og + col] : 0.0;   // rhs = Schur part - gradient
    }
  }
  if (cta == 0) {
    double* CC = ws + pl.oCC;
    for (int e = tid; e < (m + 1) * m; e += kBcrThreads) {
      const int r = e / m, q = e - r * m;
      double v;
      if (r < m) {
        v = (q <= r) ? sys[sys_index(lay, np + r, np + q)] : 0.0;
        if (q == r) v += mu * fmin(fmax(sys[lay.oD + np + r], 1e-6), 1e32);
        if (fixed[np + r] | fixed[np + q]) v = (q == r) ? 1.0 : 0.0;
      } else v = fixed[np + q] ? 0.0 : sys[lay.ob + np + q] - sys[lay.og + np + q];
      CC[e] = v;
    }
    for (int a = tid; a < n; a += kBcrThreads) Dout[a] = fmin(fmax(sys[lay.oD + a], 1e-6), 1e32);
    if (tid == 0) *spd_flag = 1;   // (cleared at the end by any CTA that met a non-positive pivot)
  }
  stamp();
  bcr_grid_sync(barrier, &s_phase);
  stamp();

  // shared-memory carve-up (doubles): L [nb][ldl] | inv [nb] | R [nb][ldr] | corner accumulator [(m+1) m]
  const int ldl = nb | 1;
  const int ncols = 2 * nb + m + 1;
  const int ldr = ((ncols + 11) / 16) * 16 + 4;   // = 4 (mod 16): the FP64 tensor-core fragment loads of the Gram pass are conflict-free
  double* sL = s_bcr;
  double* sInv = sL + nb * ldl;
  double* sR = sInv + nb + (nb & 1);
  double* sAcc = sR + nb * ldr;                     // Y_f^T [Y_f | y] summed over this CTA's nodes (the corner update, deferred)
  const int nacc = (m + 1) * m;
  for (int e = tid; e < nacc; e += kBcrThreads) sAcc[e] = 0.0;
  // After the forward substitution sR holds Y = [Y_a | Y_c | Y_f | y]; with that column order every product the even
  // neighbours and the corner need is a block of the lower triangle of G = Y^T Y (bcr_gram):
  //   (a,a) (c,c) -> D of the neighbours, (c,a) -> their new coupling, (f,a) (f,c) -> F, (y,a) (y,c) -> b, (f,f) (y,f) -> corner.
  // ---- reduction levels ----
  for (int lv = 0; lv < pl.levels; ++lv) {
    const int s = 1 << lv;
    // phase 1: odd nodes i = s, 3s, 5s, ...
    for (int i = s + 2 * s * cta; i < nsb; i += 2 * s * nctas) {
      double* N = node(i);
      const int a = i - s, c = i + s;
      const bool has_c = c < nsb;
      const double* Ba = node(a) + pl.oB;    // A[i][a]: rows i, columns a
      for (int e = tid; e < nb * nb; e += kBcrThreads) {
        const int u = e / nb, v = e - u * nb;
        sL[u * ldl + v] = N[pl.oD + e];
        sR[u * ldr + v] = Ba[e];                                       // column v of B_a, row u
        sR[u * ldr + nb + v] = has_c ? N[pl.oB + v * nb + u] : 0.0;   // (B_i^T)[u][v] = B_i[v][u]
      }
      for (int e = tid; e < m * nb; e += kBcrThreads) {
        const int r = e / nb, u = e - r * nb;
        sR[u * ldr + 2 * nb + r] = N[pl.oF + e];                       // (F_i^T)[u][r]
      }
      for (int u = tid; u < nb; u += kBcrThreads) sR[u * ldr + 2 * nb + m] = N[pl.ob + u];
      __syncthreads();
      if (lv == 0) stamp();
      bcr_chol(sL, ldl, nb, sInv, &s_ok);
      if (lv == 0) stamp();
      bcr_forward(sL, ldl, sInv, nb, sR, ldr, ncols);   // one right-hand-side column per thread
      __syncthreads();
      if (lv == 0) stamp();
      for (int e = tid; e < nb * nb; e += kBcrThreads) {
        const int u = e / nb, v = e - u * nb;
        N[pl.oL + e] = (v <= u) ? sL[u * ldl + v] : 0.0;
        N[pl.oYa + e] = sR[u * ldr + v];
        N[pl.oYc + e] = sR[u * ldr + nb + v];
      }
      for (int e = tid; e < nb * m; e += kBcrThreads) {
        const int u = e / m, r = e - u * m;
        N[pl.oYf + e] = sR[u * ldr + 2 * nb + r];                      // Y_f [nb][m]
      }
      for (int u = tid; u < nb; u += kBcrThreads) N[pl.oy + u] = sR[u * ldr + 2 * nb + m];
      if (lv == 0) stamp();
      bcr_gram(sR, ldr, nb, ncols, N + pl.oG);
      if (lv == 0) stamp();
      __syncthreads();
      if (lv == 0) stamp();
      for (int e = tid; e < nacc; e += kBcrThreads) {   // (f,f) lower and (y,f): this node's share of the corner update
        const int r = e / m, q = e - r * m;
        if (r == m || q <= r) sAcc[e] += N[pl.oG + (2 * nb + r) * ncols + 2 * nb + q];
      }
      __syncthreads();
    }
    stamp();
    bcr_grid_sync(barrier, &s_phase);
    stamp();
    // phase 2: even nodes e = 0, 2s, 4s, ...: subtract the Schur complements their eliminated neighbours prepared
    for (int e0 = 2 * s * cta; e0 < nsb; e0 += 2 * s * nctas) {
      double* N = node(e0);
      const int i1 = e0 - s, i2 = e0 + s;
      const bool h1 = i1 >= 0, h2 = i2 < nsb;
      if (!h1 && !h2) continue;
      const bool hnext = e0 + 2 * s < nsb;
      const double* N1 = h1 ? node(i1) : N;
      const double* N2 = h2 ? node(i2) : N;
      for (int e = tid; e < nb * nb; e += kBcrThreads) {
        const int u = e / nb, v = e - u * nb;
        if (v <= u) {   // D: lower triangle (all the factorisation reads): (c,c) of the left neighbour, (a,a) of the right one
          const double u1 = h1 ? N1[pl.oG + (nb + u) * ncols + nb + v] : 0.0, u2 = h2 ? N2[pl.oG + u * ncols + v] : 0.0;
          N[pl.oD + e] -= u1 + u2;
        }
        N[pl.oB + e] = (h2 && hnext) ? -N2[pl.oG + (nb + u) * ncols + v] : 0.0;   // new coupling e -> e + 2s = -(c,a): rows = dofs of e + 2s, columns = dofs of e
      }
      for (int e = tid; e < m * nb; e += kBcrThreads) {
        const int r = e / nb, v = e - r * nb;
        const double g1 = h1 ? N1[pl.oG + (2 * nb + r) * ncols + nb + v] : 0.0, g2 = h2 ? N2[pl.oG + (2 * nb + r) * ncols + v] : 0.0;
        N[pl.oF + e] -= g1 + g2;
      }
      for (int v = tid; v < nb; v += kBcrThreads) {
        const double g1 = h1 ? N1[pl.oG + (2 * nb + m) * ncols + nb + v] : 0.0, g2 = h2 ? N2[pl.oG + (2 * nb + m) * ncols + v] : 0.0;
        N[pl.ob + v] -= g1 + g2;
      }
    }
    stamp();
    bcr_grid_sync(barrier, &s_phase);
    stamp();
  }
  // ---- top node 0: factor, its share of the corner update; then every CTA publishes its corner partial ----
  if (cta == 0) {
    double* N = node(0);
    for (int e = tid; e < nb * nb; e += kBcrThreads) { const int u = e / nb, v = e - u * nb; sL[u * ldl + v] = N[pl.oD + e]; }
    for (int e = tid; e < m * nb; e += kBcrThreads) { const int r = e / nb, u = e - r * nb; sR[u * ldr + r] = N[pl.oF + e]; }
    for (int u = tid; u < nb; u += kBcrThreads) sR[u * ldr + m] = N[pl.ob + u];
    __syncthreads();
    bcr_chol(sL, ldl, nb, sInv, &s_ok);
    bcr_forward(sL, ldl, sInv, nb, sR, ldr, m + 1);
    __syncthreads();
    for (int e = tid; e < nb * nb; e += kBcrThreads) { const int u = e / nb, v = e - u * nb; N[pl.oL + e] = (v <= u) ? sL[u * ldl + v] : 0.0; }
    for (int e = tid; e < nb * m; e += kBcrThreads) { const int u = e / m, r = e - u * m; N[pl.oYf + e] = sR[u * ldr + r]; }
    for (int u = tid; u < nb; u += kBcrThreads) N[pl.oy + u] = sR[u * ldr + m];
    bcr_gram(sR, ldr, nb, m + 1, N + pl.oG);
    __syncthreads();
    for (int e = tid; e < nacc; e += kBcrThreads) {
      const int r = e / m, q = e - r * m;
      if (r == m || q <= r) sAcc[e] += N[pl.oG + r * (m + 1) + q];
    }
  }
  __syncthreads();
  {
    double* part = ws + pl.oCCp + static_cast<long long>(cta) * nacc;
    for (int e = tid; e < nacc; e += kBcrThreads) part[e] = sAcc[e];
  }
  stamp();
  bcr_grid_sync(barrier, &s_phase);
  stamp();
  // corner C' = C - sum of the partials, every CTA reduces a slice (CTA order: the same sum on every replica)
  {
    double* CC = ws + pl.oCC;
    const int warp = tid >> 5, lane = tid & 31;
    for (int e = cta + nctas * warp; e < nacc; e += nctas * (kBcrThreads / 32)) {   // one element per warp, lanes over the partials
      double v = 0.0;
      for (int c = lane; c < nctas; c += 32) v += ws[pl.oCCp + static_cast<long long>(c) * nacc + e];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) CC[e] -= v;
    }
  }
  stamp();
  bcr_grid_sync(barrier, &s_phase);
  stamp();
  double* xa = ws + pl.oXa;
  if (cta == 0) {
    // corner: padded to a multiple of 6 with identity, blocked Cholesky, forward + backward substitution by one warp
    double* CCs = s_bcr;
    const int mp = ((m + 5) / 6) * 6, ldc = mp | 1;
    double* cinv = CCs + mp * ldc;
    double* rhs = cinv + mp + (mp & 1);
    double* sol = rhs + mp + (mp & 1);
    const double* CC = ws + pl.oCC;
    for (int e = tid; e < mp * mp; e += kBcrThreads) { const int r = e / mp, q = e - r * mp; if (r >= m || q >= m) CCs[r * ldc + q] = (r == q) ? 1.0 : 0.0; }
    for (int r = m + tid; r < mp; r += kBcrThreads) rhs[r] = 0.0;
    for (int e = tid; e < nacc; e += kBcrThreads) {
      const int r = e / m, q = e - r * m;
      const double v = CC[e];
      if (r < m) CCs[r * ldc + q] = v; else rhs[q] = v;
    }
    __syncthreads();
    bcr_chol(CCs, ldc, mp, cinv, &s_ok);
    if (tid < 32) {
      bcr_forward_warp(CCs, ldc, mp, rhs, sol);
      __syncwarp();
      bcr_backward_warp(CCs, ldc, mp, sol, rhs);
      __syncwarp();
      for (int r = tid; r < m; r += 32) { xa[r] = rhs[r]; x_out[np + r] = rhs[r]; }
    }
  }
  stamp();
  bcr_grid_sync(barrier, &s_phase);
  stamp();
  // ---- way back: x_i = L^-T (y - Y_a x_a - Y_c x_c - Y_f x_arrow); top node first, then level by level ----
  auto backsolve_node = [&](int i, int a, int c) {
    const double* N = node(i);
    double* rv = s_bcr;                              // [nb]
    double* xs = rv + nb + (nb & 1);                 // [nb]
    double* sx = xs + nb + (nb & 1);                 // staged x_a | x_c | x_arrow  [2 nb + m]
    double* sLt = sx + 2 * nb + m + (m & 1);         // L [nb][ldl]
    for (int e = tid; e < nb * nb; e += kBcrThreads) { const int u = e / nb, v = e - u * nb; if (v <= u) sLt[u * ldl + v] = N[pl.oL + e]; }
    for (int v = tid; v < nb; v += kBcrThreads) {
      const int ca = nb * a + v, cc = nb * c + v;
      sx[v] = (a >= 0 && ca < np) ? x_out[ca] : 0.0;
      sx[nb + v] = (c >= 0 && cc < np) ? x_out[cc] : 0.0;
    }
    for (int r = tid; r < m; r += kBcrThreads) sx[2 * nb + r] = xa[r];
    __syncthreads();
    // rv_u = y_u - [Y_a | Y_c | Y_f]_u . [x_a | x_c | x_arrow]: one warp per row, coalesced reads, shuffle reduction
    {
      const int warp = tid >> 5, lane = tid & 31;
      for (int u = warp; u < nb; u += kBcrThreads / 32) {
        double acc = 0.0;
        for (int v = lane; v < nb; v += 32) acc += N[pl.oYa + u * nb + v] * sx[v] + N[pl.oYc + u * nb + v] * sx[nb + v];
        for (int r = lane; r < m; r += 32) acc += N[pl.oYf + u * m + r] * sx[2 * nb + r];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) rv[u] = N[pl.oy + u] - acc;
      }
    }
    __syncthreads();
    if (tid < 32) bcr_backward_warp(sLt, ldl, nb, rv, xs);
    __syncthreads();
    for (int u = tid; u < nb; u += kBcrThreads) { const int col = nb * i + u; if (col < np) x_out[col] = xs[u]; }
    __syncthreads();
  };
  if (cta == 0) backsolve_node(0, -1, -1);
  stamp();
  bcr_grid_sync(barrier, &s_phase);
  stamp();
  for (int lv = pl.levels - 1; lv >= 0; --lv) {
    const int s = 1 << lv;
    for (int i = s + 2 * s * cta; i < nsb; i += 2 * s * nctas) backsolve_node(i, i - s, (i + s < nsb) ? i + s : -1);
    stamp();
    if (lv > 0) bcr_grid_sync(barrier, &s_phase);
    stamp();
  }
  if (tid == 0 && !s_ok) atomicExch(spd_flag, 0);
  if (dbg && blockIdx.x == 0 && threadIdx.x == 0) dbg[0] = n_stamp;
}

}  // namespace hb
