// Block-banded + arrowhead Cholesky solve of the reduced system (sm_90a): a 2-CTA cluster when the workspace is
// resident in shared memory (one elimination chain per SM), one CTA over a global-memory workspace otherwise.
//
// After the landmark Schur complement the reduced system of a spline window is
//   S = [ P  A^T ]   P: 6x6 control-point blocks, block half-bandwidth beta (= longest landmark track
//       [ A  C   ]      measured in control points, >= k-1), A: m x 6K arrow (bias knots + gravity),
//   C: m x m.  The reference hands the same structure to CHOLMOD through SPARSE_NORMAL_CHOLESKY
//   (reference internal/hyper/optimizers/ceres/optimizer.cpp:46-48); here the factorisation,
//   forward and backward substitution run with the whole band resident in shared memory (global-memory
//   workspace, one CTA, when it does not fit).
//
// Two-sided elimination.  The factorisation is a chain of K dependent block-column steps, each bounded
// by FP64 dependent-issue latency (a 6x6 potf2 plus a panel solve), not by throughput.  The chain is cut
// in two: a separator of beta block columns in the middle decouples the columns above it from the
// columns below it, so chain 0 eliminates block columns 0 .. Kt-1 top-down while chain 1 eliminates
// K-1 .. Kt+beta bottom-up IN THE SAME STEPS (resident: chain r on CTA r of a cluster; global workspace:
// same barriers, disjoint warps; one look-ahead warp per chain on its own scheduler).  Chain 1 runs the very same code on the index-reversed matrix J P J
// (still block-banded) and accumulates its Schur updates of the separator and of the separator's
// arrow columns into a private, zero-initialised copy.  The copies are then merged into chain 0, which
// eliminates the beta separator columns, and the back substitution runs outwards from the separator
// in both directions at once.  Sequential depth: ~K/2 + beta steps instead of K.
// The arrow x arrow (corner) part of every step's trailing update is deferred: the corner receives
// C -= sum_c A_c A_c^T in one parallel pass after the last column, which takes 15 of 55 tiles (beta = 5, m = 26) out of
// every step.
//
// Per-chain workspace (doubles): W[ncol][h][6] band block-columns (h = 6 + 6 beta rows each: diagonal
//   block first; ncol = eliminated columns + separator columns), AR[m+1][6 ncol] arrow rows (+ the rhs as
//   last row), LI[ncol][48] reciprocal diagonals (6) and inverses (36, at +8) of the diagonal Cholesky
//   blocks, X[6 ncol].  Shared: CC[m+1][m] corner (+ rhs row), XA[m].
#pragma once
#include "hb200_solve.cuh"

namespace hb {

constexpr int kBandThreads = 512;

struct BandPlan { int Kt, Kb, bs; };   // columns eliminated by chain 0 / chain 1, separator columns
__host__ __device__ inline BandPlan band_plan(int K, int beta) {
  BandPlan p;
  if (K >= 2 * beta + 4) { p.bs = beta; p.Kt = (K - beta + 1) / 2; p.Kb = K - beta - p.Kt; }
  else { p.bs = 0; p.Kt = K; p.Kb = 0; }
  return p;
}

__host__ __device__ inline size_t band_workspace_doubles(int K, int beta, int m) {
  const BandPlan p = band_plan(K, beta);
  const size_t h = 6 + 6 * static_cast<size_t>(beta);
  const size_t n0 = p.Kt + p.bs, n1 = p.Kb ? p.Kb + p.bs : 0;
  size_t d = (n0 + n1) * h * 6;                  // W
  d += static_cast<size_t>(m + 1) * 6 * (n0 + n1);  // AR
  d += (n0 + n1) * 48;                           // LI
  d += 6 * (n0 + n1);                            // X
  d += static_cast<size_t>(m + 1) * (m | 1) + 2 * static_cast<size_t>(m); // CC (odd row stride: conflict-free column access), XA, DG
  d += 6 * static_cast<size_t>(K) + m + (6 * static_cast<size_t>(K) + m) / 8 + 1;   // per-dof damping term and constant-dof mask, staged for the gather
  return d + 8;
}

// Shared-memory budget of one CTA of the band solvers.
constexpr size_t kBandSmemBytes = 220 * 1024;

// Chain of CTA `rank` of the resident solver (band_plan): Ke block columns it eliminates, then the bs separator columns
// it stores (ncol in all); forward from block column 0 (rank 0) or reversed from K (rank 1).  Chain 0 eliminates the
// separator (elim).
struct SegChain { int Ke, ncol, anchor; bool rev, elim; };
__host__ __device__ inline SegChain seg_chain(const BandPlan& pl, int K, int rank) {
  SegChain c;
  c.Ke = rank ? pl.Kb : pl.Kt;
  c.ncol = c.Ke ? c.Ke + pl.bs : 0;
  c.rev = rank == 1;
  c.elim = pl.bs > 0 && rank == 0;
  c.anchor = rank ? K : 0;
  return c;
}

// Per-CTA workspace of the resident solver, offsets in doubles: the CTA's own chain only (W, AR, LI, X as in
// band_workspace_doubles), the receive buffer of the separator copy the other chain stores (elim: RBW band block columns,
// RBA arrow columns + rhs), the corner CC (CTA 0: the corner system; CTA 1: its partial sum of the corner update), XA + DG
// and the staging.
struct CtaLayout { size_t W, AR, LI, X, RBW, RBA, CC, XA, total; };
__host__ __device__ inline CtaLayout cta_layout(const BandPlan& pl, int K, int beta, int m, int rank) {
  const SegChain g = seg_chain(pl, K, rank);
  const size_t h6 = 36 + 36 * static_cast<size_t>(beta), npc = 6 * static_cast<size_t>(g.ncol);
  CtaLayout L;
  size_t p = 0;
  L.W = p; p += g.ncol * h6;
  L.AR = p; p += static_cast<size_t>(m + 1) * npc;
  L.LI = p; p += g.ncol * 48;
  L.X = p; p += npc;
  L.RBW = p; if (g.elim) p += pl.bs * h6;
  L.RBA = p; if (g.elim) p += static_cast<size_t>(m + 1) * 6 * pl.bs;
  L.CC = p; p += static_cast<size_t>(m + 1) * (m | 1);
  L.XA = p; p += 2 * static_cast<size_t>(m);
  p += 6 * static_cast<size_t>(K) + m + (6 * static_cast<size_t>(K) + m) / 8 + 1;
  L.total = p + 8;
  return L;
}

// Dynamic shared memory of each CTA of the resident solver's cluster (the larger CTA workspace).
__host__ __device__ inline size_t band_cluster_doubles(int K, int beta, int m) {
  const BandPlan pl = band_plan(K, beta);
  const size_t d0 = cta_layout(pl, K, beta, m, 0).total, d1 = cta_layout(pl, K, beta, m, 1).total;
  return d0 > d1 ? d0 : d1;
}

// Right-looking Cholesky of a 6x6 SPD block (lower, row-major with stride ld), division-free:
// inv[j] = 1 / L[j][j] comes straight out of rsqrt.  If X != nullptr the block first receives its
// pending trailing update A -= X X^T (X = the 6 panel rows of this block, row-major 6x6), so the
// look-ahead thread does not wait for a separate update pass.
HB_DI bool chol6(double* A, int ld, double* inv /*6*/, const double* X = nullptr) {
  double L[21];  // packed lower: L[i(i+1)/2 + j]
  bool ok = true;
#pragma unroll
  for (int i = 0; i < 6; ++i)
#pragma unroll
    for (int j = 0; j <= i; ++j) L[i * (i + 1) / 2 + j] = A[i * ld + j];
  if (X != nullptr) {
    double x[36];
#pragma unroll
    for (int e = 0; e < 18; ++e) { const double2 t = reinterpret_cast<const double2*>(X)[e]; x[2 * e] = t.x; x[2 * e + 1] = t.y; }
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
      for (int j = 0; j <= i; ++j) {
        double acc = 0.0;
#pragma unroll
        for (int q = 0; q < 6; ++q) acc += x[6 * i + q] * x[6 * j + q];
        L[i * (i + 1) / 2 + j] -= acc;
      }
  }
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    const double d = L[j * (j + 1) / 2 + j];
    if (!(d > 0.0)) ok = false;
    const double iv = rsqrt(d);
    inv[j] = iv;
    L[j * (j + 1) / 2 + j] = d * iv;
#pragma unroll
    for (int i = j + 1; i < 6; ++i) L[i * (i + 1) / 2 + j] *= iv;
#pragma unroll
    for (int i = j + 1; i < 6; ++i)
#pragma unroll
      for (int q = j + 1; q <= i; ++q) L[i * (i + 1) / 2 + q] -= L[i * (i + 1) / 2 + j] * L[q * (q + 1) / 2 + j];
  }
#pragma unroll
  for (int i = 0; i < 6; ++i)
#pragma unroll
    for (int j = 0; j <= i; ++j) A[i * ld + j] = L[i * (i + 1) / 2 + j];
  return ok;
}

// Clock read that waits for `dep` (BAR.SYNC is deferred-blocking: a bare clock read right after a barrier
// reports the barrier's issue time, not its release).
HB_DI long long clock_after(double dep) {
  long long t;
  asm volatile("mov.u64 %0, %%clock64;" : "=l"(t) : "d"(dep) : "memory");
  return t;
}

// Named barriers (ids 1..15; id 0 is __syncthreads): only the warps of one chain's pipeline take part.
HB_DI void nbar_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
HB_DI void nbar_arrive(int id, int count) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory"); }

// 2-CTA cluster of the resident solver.  The cluster barrier orders shared-memory accesses across the cluster
// (release on arrive, acquire on wait); a peer CTA's shared memory is read through mapa + ld.shared::cluster.
HB_DI int cluster_rank() { unsigned r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return static_cast<int>(r); }
HB_DI void cluster_arrive() { asm volatile("barrier.cluster.arrive.release;" ::: "memory"); }
HB_DI void cluster_wait() { asm volatile("barrier.cluster.wait.acquire;" ::: "memory"); }
HB_DI unsigned peer_addr(const void* p, int rank) {
  unsigned a;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(static_cast<unsigned>(__cvta_generic_to_shared(p))), "r"(rank));
  return a;
}
HB_DI double ld_peer(const double* p, int rank) {
  double v;
  asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(peer_addr(p, rank)));
  return v;
}
HB_DI void st_peer(double* p, int rank, double v) {
  asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(peer_addr(p, rank)), "d"(v) : "memory");
}
HB_DI int ld_peer(const int* p, int rank) {
  int v;
  asm volatile("ld.shared::cluster.s32 %0, [%1];" : "=r"(v) : "r"(peer_addr(p, rank)));
  return v;
}

// Update warps per CTA of the cluster kernel (schedulers 0..2; the look-ahead warp has scheduler 3 to itself).  At cfg1
// on an H100, 4 and 8 update warps gave the same step time within noise and 6 was ~1 us slower per solve.
constexpr int kBandUpdWarps = 4;

struct BandChain {
  double *W, *AR, *LI, *X;
  int Ke;     // block columns this chain eliminates in the two-sided phase
  int ncol;   // block columns it stores (Ke + separator)
  int npc;    // 6 * ncol
  int ars;    // row stride of AR in doubles (= npc for a whole chain; the chunk capacity for a shared-memory view)
  int ne;     // block columns whose factor the chain holds (Ke, + the separator if it eliminates it)
};

// Panel of block column s: solve x L^T = a for every row below the diagonal block (band rows, arrow rows,
// rhs row), one row per thread lt, lt += nthreads.
HB_DI void band_panel(const BandChain& C, int s, int h, int m, int lt, int nthreads, int row0 = 0) {
  double* Wc = C.W + static_cast<size_t>(s) * h * 6;
  const double* Lic = C.LI + static_cast<size_t>(s) * 48;
  const int nb = min(h - 6, C.npc - 6 * (s + 1));  // band rows below the diagonal block
  const int R = nb + m + 1;                          // + arrow rows + rhs row
  for (int t = row0 + lt; t < R; t += nthreads) {
    double* a = (t < nb) ? (Wc + static_cast<size_t>(6 + t) * 6) : (C.AR + static_cast<size_t>(t - nb) * C.ars + 6 * s);
    double v[6];
#pragma unroll
    for (int q = 0; q < 6; ++q) v[q] = a[q];
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      v[j] *= Lic[j];
#pragma unroll
      for (int q = j + 1; q < 6; ++q) v[q] -= v[j] * Wc[q * 6 + j];
    }
#pragma unroll
    for (int q = 0; q < 6; ++q) a[q] = v[q];
  }
}

// Trailing update of block column s in 6x6 tiles (band x band lower triangle, then arrow x band; the
// arrow x arrow part is deferred).  Worker = (tile, row i of the tile): 6 dots of length 6.  Items start at
// `first` (6 = tile 0, the next diagonal block, is left to the look-ahead warp).  tile_uv: optional lookup
// table tile -> (gu, gv) valid for full-band steps (nbk == beta): the decode then costs two byte loads.
HB_DI void band_update(const BandChain& C, int s, int h, int m, int first, int worker, int nworkers, const unsigned char* tile_uv, int beta) {
  double* Wc = C.W + static_cast<size_t>(s) * h * 6;
  const int nb = min(h - 6, C.npc - 6 * (s + 1));
  const int nbk = nb / 6;
  const int ng = (m + 1 + 5) / 6;
  const int ntri = nbk * (nbk + 1) / 2;
  const int ntiles = ntri + ng * nbk;
  const bool table = tile_uv != nullptr && nbk == beta;
  for (int t = first + worker; t < ntiles * 6; t += nworkers) {
    const int tile = t / 6, i = t - 6 * tile;
    int gu, gv;
    if (table) {
      gu = tile_uv[2 * tile]; gv = tile_uv[2 * tile + 1];
    } else if (tile < ntri) {
      gu = static_cast<int>((sqrtf(8.0f * tile + 1.0f) - 1.0f) * 0.5f);
      while (gu * (gu + 1) / 2 > tile) --gu;
      while ((gu + 1) * (gu + 2) / 2 <= tile) ++gu;
      gv = tile - gu * (gu + 1) / 2;
    } else {
      const int ta = tile - ntri;
      gu = nbk + ta / nbk;
      gv = ta - (ta / nbk) * nbk;
    }
    const bool ub = gu < nbk;
    const int ru = ub ? 0 : 6 * (gu - nbk) + i;   // arrow row index of u
    if (!ub && ru > m) continue;
    const double* xu = ub ? (Wc + static_cast<size_t>(6 + 6 * gu + i) * 6) : (C.AR + static_cast<size_t>(ru) * C.ars + 6 * s);
    double* tgt = ub ? (C.W + (static_cast<size_t>(s + 1 + gv) * h + (6 * (gu - gv) + i)) * 6)   // band x band
                     : (C.AR + static_cast<size_t>(ru) * C.ars + 6 * (s + 1 + gv));              // arrow x band
    double a[6], sd[6];
    {
      const double2* x2 = reinterpret_cast<const double2*>(xu);   // rows are 48 B: 16-byte aligned
      const double2 a0 = x2[0], a1 = x2[1], a2 = x2[2];
      a[0] = a0.x; a[1] = a0.y; a[2] = a1.x; a[3] = a1.y; a[4] = a2.x; a[5] = a2.y;
    }
    double2* t2 = reinterpret_cast<double2*>(tgt);
    double2 o0 = t2[0], o1 = t2[1], o2 = t2[2];
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      const double2* v2 = reinterpret_cast<const double2*>(Wc + static_cast<size_t>(6 + 6 * gv + j) * 6);
      const double2 b0 = v2[0], b1 = v2[1], b2 = v2[2];
      sd[j] = a[0] * b0.x + a[1] * b0.y + a[2] * b1.x + a[3] * b1.y + a[4] * b2.x + a[5] * b2.y;
    }
    o0.x -= sd[0]; o0.y -= sd[1]; o1.x -= sd[2]; o1.y -= sd[3]; o2.x -= sd[4]; o2.y -= sd[5];
    t2[0] = o0; t2[1] = o1; t2[2] = o2;
  }
}

// Look-ahead warp, one step: lanes 0..5 solve the panel rows of the first band block (the only rows the next
// diagonal block depends on) and publish them (arrive on barrier A, which the update warps wait on); lane 0
// then applies the pending update A -= X X^T to the next diagonal block in registers and factors it.  The
// critical chain potf2 -> first panel block -> potf2 never waits for the rest of the panel or the update.
HB_DI bool band_la_step(const BandChain& C, int s, int h, int lane, bool do_chol, int barA, int countA) {
  double* Wc = C.W + static_cast<size_t>(s) * h * 6;
  const double* Lic = C.LI + static_cast<size_t>(s) * 48;
  const int nb = min(h - 6, C.npc - 6 * (s + 1));
  bool ok = true;
  if (nb >= 6 && lane < 6) {
    double* a = Wc + static_cast<size_t>(6 + lane) * 6;
    double v[6];
#pragma unroll
    for (int q = 0; q < 6; ++q) v[q] = a[q];
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      v[j] *= Lic[j];
#pragma unroll
      for (int q = j + 1; q < 6; ++q) v[q] -= v[j] * Wc[q * 6 + j];
    }
#pragma unroll
    for (int q = 0; q < 6; ++q) a[q] = v[q];
  }
  __syncwarp();
  __threadfence_block();
  nbar_arrive(barA, countA);
  if (nb >= 6) {
    // next diagonal block: lane i < 6 subtracts row i of X X^T (X = the 6 panel rows just solved), everything
    // loaded before anything is stored (no store->load serialisation); lane 0 then factors the block
    double* An = C.W + static_cast<size_t>(s + 1) * h * 6;
    if (lane < 6) {
      double x[36], xi[6], an[6];
#pragma unroll
      for (int e = 0; e < 18; ++e) { const double2 t = reinterpret_cast<const double2*>(Wc + 36)[e]; x[2 * e] = t.x; x[2 * e + 1] = t.y; }
#pragma unroll
      for (int e = 0; e < 3; ++e) { const double2 t = reinterpret_cast<const double2*>(Wc + 36 + 6 * lane)[e]; xi[2 * e] = t.x; xi[2 * e + 1] = t.y; }
#pragma unroll
      for (int j = 0; j < 6; ++j) an[j] = An[6 * lane + j];
#pragma unroll
      for (int j = 0; j < 6; ++j) {
        double acc = 0.0;
#pragma unroll
        for (int q = 0; q < 6; ++q) acc += xi[q] * x[6 * j + q];
        an[j] -= acc;
      }
#pragma unroll
      for (int j = 0; j < 6; ++j)
        if (j <= lane) An[6 * lane + j] = an[j];
    }
    __syncwarp();
    if (do_chol && lane == 0) ok = chol6(An, 6, C.LI + static_cast<size_t>(s + 1) * 48);
  }
  return ok;
}

// Back substitution of block columns c_hi .. c_lo of one chain (one warp) AFTER the row transform
// B <- B L_cc^-1, y <- y L_cc^-1 (band_transform_row): x_c = y~_c - sum_r N_{c,r}^T x_{c+r} -- no triangular
// solve on the chain.  Lane = (component j = lane % 6, band block r = lane / 6): one 6-term dot per lane,
// a five-way shuffle reduction, lanes 0..5 publish x_c.  The loop body is kept small on purpose: this code
// runs once per solve, and one-shot code is bound by instruction fetch, not by issue (tools/microbench).
HB_DI void band_backsub_chain(const BandChain& C, int c_hi, int c_lo, int h, int m, int lane) {
  const int j = lane % 6, g = lane / 6;
  // the panel operands of a column do not depend on the solution: they are fetched one column ahead, so that
  // a workspace in global memory costs no L2 round trip on the sequential chain
  auto fetch = [&](int c, double* nv, double* y) {
    const double* Wc = C.W + static_cast<size_t>(c) * h * 6 + 36 + j;
    const int nbk = min(h - 6, C.npc - 6 * (c + 1)) / 6;
#pragma unroll
    for (int t = 0; t < 6; ++t) nv[t] = (g < 5 && g < nbk) ? Wc[36 * g + 6 * t] : 0.0;
    *y = (lane < 6) ? C.AR[static_cast<size_t>(m) * C.npc + 6 * c + lane] : 0.0;
  };
  double nv[6], yv;
  if (c_hi >= c_lo) fetch(c_hi, nv, &yv);
  for (int c = c_hi; c >= c_lo; --c) {
    double nn[6] = {0, 0, 0, 0, 0, 0}, yn = 0.0;
    if (c - 1 >= c_lo) fetch(c - 1, nn, &yn);
    const int nbk = min(h - 6, C.npc - 6 * (c + 1)) / 6;
    double acc = 0.0;
    if (g < 5 && g < nbk) {
      const double* xr = C.X + 6 * (c + 1 + g);
#pragma unroll
      for (int t = 0; t < 6; ++t) acc += nv[t] * xr[t];
      for (int r = g + 5; r < nbk; r += 5) {   // half-bandwidths above 5 blocks
        const double* nr = C.W + static_cast<size_t>(c) * h * 6 + 36 + j + 36 * r;
        const double* xq = C.X + 6 * (c + 1 + r);
#pragma unroll
        for (int t = 0; t < 6; ++t) acc += nr[6 * t] * xq[t];
      }
    }
    double tot = acc;
    tot += __shfl_sync(0xffffffffu, acc, (lane + 6) & 31);
    tot += __shfl_sync(0xffffffffu, acc, (lane + 12) & 31);
    tot += __shfl_sync(0xffffffffu, acc, (lane + 18) & 31);
    tot += __shfl_sync(0xffffffffu, acc, (lane + 24) & 31);
    if (lane < 6) C.X[6 * c + lane] = yv - tot;
    __syncwarp();
#pragma unroll
    for (int t = 0; t < 6; ++t) nv[t] = nn[t];
    yv = yn;
  }
}

// Row transform v <- v L^-1 (L = the column's diagonal Cholesky block, row-major 6x6, rd = reciprocal
// diagonal): solve x L = v from the last component down.  Applied to every panel row below the diagonal
// and to the rhs row, it turns the back substitution into plain dot products.
HB_DI void band_transform_row(double* v, const double* L, const double* rd) {
  double x[6];
#pragma unroll
  for (int q = 0; q < 6; ++q) x[q] = v[q];
#pragma unroll
  for (int jj = 5; jj >= 0; --jj) {
    double acc = x[jj];
#pragma unroll
    for (int q = jj + 1; q < 6; ++q) acc -= x[q] * L[q * 6 + jj];
    x[jj] = acc * rd[jj];
  }
#pragma unroll
  for (int q = 0; q < 6; ++q) v[q] = x[q];
}

template <bool SMEM>
__global__ void __launch_bounds__(kBandThreads) band_solve_kernel(const double* __restrict__ sys, SysLayout lay,
                                                                  double* __restrict__ ws_global, double* __restrict__ x_out,
                                                                  int* __restrict__ spd_flag, long long* __restrict__ dbg,
                                                                  const SolverState* __restrict__ st, const unsigned char* __restrict__ fixed,
                                                                  double* __restrict__ Dout, int chunk_cols) {
  extern __shared__ double s_band[];
  const long long t_entry = clock64();
  // SMEM: the workspace is resident in shared memory and the kernel runs as a 2-CTA cluster, chain r in CTA r, each
  // chain on its own SM (its own shared-memory crossbar and four schedulers).  Each CTA lays out only its own chain
  // (cta_layout); either CTA can compute the other's layout and the dynamic shared memory starts at the same address in
  // both, so a peer's array sits at the local address mapped to the peer's rank.  CTA 0 (the hub) also owns the corner.
  // !SMEM: one CTA runs both chains on chunked shared-memory views of a global workspace.
  constexpr bool CL = SMEM;
  const int rank = CL ? cluster_rank() : 0;
  const int n = lay.n, K = lay.K, beta = lay.beta;
  const int np = 6 * K, m = n - np, h = 6 + 6 * beta, h6 = h * 6;
  const BandPlan pl = band_plan(K, beta);
  const SegChain g = seg_chain(pl, K, rank);
  const bool hub = !CL || rank == 0;
  const bool has0 = !CL || !g.rev, has1 = !CL || g.rev;   // CL: the CTA's chain is forward (C0) or reversed (C1)
  if (CL && dbg) dbg += 72 * rank;
  double* ws = SMEM ? s_band : ws_global;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // Roles (!CL).  Each chain owns one scheduler for its latency-critical work (the arbiter favours the highest
  // warp id of a scheduler): scheduler 0 = chain 0 (warp 12 look-ahead, warp 8 lane 0 block inverses),
  // scheduler 1 = chain 1 (warp 13, warp 9 lane 0); their other warps idle during the update phase.
  // The warps of schedulers 2 and 3 do the trailing updates: 2,3,6,7 -> chain 0, 10,11,14,15 -> chain 1.
  // Roles (CL).  Warp 15 is the look-ahead warp, alone on scheduler 3 (warps 3, 7, 11 idle in the step loop); the
  // first kBandUpdWarps warps of schedulers 0..2, in the order 0, 1, 2, 4, 5, 6, 8, ..., do panel rows and updates.
  const int sched = warp & 3;
  const int my_chain = CL ? (g.rev ? 1 : 0) : ((sched < 2) ? sched : (warp >> 3));
  BandChain C0, C1;
  int o0 = 0, e1 = K;   // natural block column of C0's column 0; one past the natural block column of C1's column 0
  double* CC;
  int LDc;
  if (CL) {
    const CtaLayout L = cta_layout(pl, K, beta, m, rank);
    BandChain own;
    own.W = ws + L.W; own.AR = ws + L.AR; own.LI = ws + L.LI; own.X = ws + L.X;
    own.Ke = g.Ke; own.ncol = g.ncol; own.npc = own.ars = 6 * g.ncol;
    own.ne = g.elim ? g.ncol : g.Ke;
    BandChain none = own;
    none.Ke = none.ncol = none.npc = none.ars = none.ne = 0;
    C0 = g.rev ? none : own; C1 = g.rev ? own : none;
    (g.rev ? e1 : o0) = g.anchor;
    CC = ws + L.CC;
    LDc = m | 1;
  } else {
    double* p = ws;
    BandChain* cc[2] = {&C0, &C1};
    for (int i = 0; i < 2; ++i) {
      BandChain& C = *cc[i];
      C.Ke = i ? pl.Kb : pl.Kt;
      C.ncol = (i && pl.Kb == 0) ? 0 : C.Ke + pl.bs;
      C.npc = 6 * C.ncol;
      C.ars = C.npc;
      C.ne = i ? C.Ke : C.ncol;
      C.W = p; p += static_cast<size_t>(C.ncol) * h6;
      C.AR = p; p += static_cast<size_t>(m + 1) * C.npc;
      C.LI = p; p += static_cast<size_t>(C.ncol) * 48;
      C.X = p; p += C.npc;
    }
    CC = p;
    LDc = m | 1;
  }
  double* XA = CC + static_cast<size_t>(m + 1) * LDc;   // (both move to shared memory after the factorisation when !SMEM)
  const BandChain C = my_chain ? C1 : C0;           // this thread's chain in the update phase (registers)
  const double* S = sys;                 // band-only storage: P at offset 0 in the chain-0 column layout
  const double* b = sys + lay.ob;
  // Dout != null: the system is the raw accumulation (lower triangle of H with the Schur complement applied,
  // b = -g + ...); LM damping mu * clamp(diag H) and the constant-dof mask are applied while gathering
  // (== finalize_kernel, which then need not run), and D = clamp(diag H) is written out for accept_kernel.
  const bool damp = Dout != nullptr;
  const double* diagH = sys + lay.oD;
  // stage the per-dof damping term and the mask once (the gather would otherwise chase them through L2 per element)
  double* s_dmp = XA + 2 * m;
  unsigned char* s_fix = reinterpret_cast<unsigned char*>(s_dmp + n);
  {
    const double mu = damp ? 1.0 / st->radius : 0.0;
    for (int a = threadIdx.x; a < n; a += kBandThreads) {
      const double dcl = damp ? fmin(fmax(diagH[a], 1e-6), 1e32) : 0.0;
      s_dmp[a] = mu * dcl;
      s_fix[a] = damp ? fixed[a] : 0;
      if (damp && hub) Dout[a] = dcl;
    }
  }
  __syncthreads();
  const long long t_staged = clock64();
  long long t_g[4] = {0, 0, 0, 0};
  auto Sval = [&](int row, int col) -> double {   // row >= col
    double v = S[sys_index(lay, row, col)];
    if (row == col) v += s_dmp[row];
    if (s_fix[row] | s_fix[col]) v = (row == col) ? 1.0 : 0.0;
    return v;
  };
  const double* gvec = sys + lay.og;
  auto bval = [&](int col) -> double { return s_fix[col] ? 0.0 : b[col] - gvec[col]; };   // rhs = Schur part - gradient
  __shared__ int s_ok;
  if (tid == 0) s_ok = 1;
  // ---- gather: chain 0 reads P top-down, chain 1 reads J P J (index reversal) and starts its copy of the
  // separator and of the separator's arrow columns at zero (they only accumulate updates) ----
  {
    // Each element is one dependent L2 access; four per thread are kept in flight (values first, stores after):
    // a one-load-at-a-time loop spent 250 us here at K = 500.
    const int N1 = has1 ? C1.npc : 0;   // (CL: each CTA gathers its own chain only)
    auto gather4 = [&](int total, auto value, auto store) {
      for (int e0 = tid; e0 < total; e0 += 4 * kBandThreads) {
        double v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) { const int e = e0 + u * kBandThreads; v[u] = (e < total) ? value(e) : 0.0; }
#pragma unroll
        for (int u = 0; u < 4; ++u) { const int e = e0 + u * kBandThreads; if (e < total) store(e, v[u]); }
      }
    };
    // band blocks: one unit = 6 contiguous doubles of a row of S (three 128-bit loads), two units in flight
    auto fix6 = [&](int row, int col0, double* v) {   // damping / mask / lower-triangle cut of S[row][col0 .. col0+5]
#pragma unroll
      for (int t = 0; t < 6; ++t) {
        const int col = col0 + t;
        double x = v[t];
        if (col > row) x = 0.0;
        else {
          if (col == row) x += s_dmp[row];
          if (s_fix[row] | s_fix[col]) x = (col == row) ? 1.0 : 0.0;
        }
        v[t] = x;
      }
    };
    auto load6 = [&](int row, int col0, double* v) {   // S[row][col0 .. col0+5], col0 a multiple of 6: one 48-byte row of P
      const double2* p2 = reinterpret_cast<const double2*>(S + (static_cast<size_t>(col0 / 6) * h + (row - col0)) * 6);
      const double2 a0 = p2[0], a1 = p2[1], a2 = p2[2];
      v[0] = a0.x; v[1] = a0.y; v[2] = a1.x; v[3] = a1.y; v[4] = a2.x; v[5] = a2.y;
    };
    {
      // chain 0: unit u = row i of block column c (a 48-byte row of P).  chain 1 = J P J: unit (c, q, j) = column j of the
      // 6-row group q of block column c of the reversed band; its six entries are S[a][b0 .. b0+5] (a = np-1-(6c+j), b
      // descending with the row), contiguous in S.  Two units of each chain per thread and pass: twelve 128-bit loads in
      // flight before the first store.
      const int nu0 = has0 ? C0.ncol * h : 0;
      const int hq = h / 6, nu1 = has1 ? C1.Ke * hq * 6 : 0;
      for (int e = tid; has1 && e < (C1.ncol - C1.Ke) * h6; e += kBandThreads) C1.W[static_cast<size_t>(C1.Ke) * h6 + e] = 0.0;   // separator copy
      for (int u0 = tid; u0 < max(nu0, nu1); u0 += 2 * kBandThreads) {
        double v[2][6], v1[2][6];
        int rowv[2], cv[2], av[2], b0v[2];
#pragma unroll
        for (int w = 0; w < 2; ++w) {
          const int u = u0 + w * kBandThreads;
          const int c = u / h, i = u - c * h;
          rowv[w] = 6 * c + i; cv[w] = c;
          if (u < nu0 && rowv[w] < C0.npc) load6(6 * o0 + rowv[w], 6 * (o0 + c), v[w]);
          else { for (int t = 0; t < 6; ++t) v[w][t] = 0.0; rowv[w] = -1; }
        }
#pragma unroll
        for (int w = 0; w < 2; ++w) {
          const int u = u0 + w * kBandThreads;
          const int c = u / (hq * 6), rem = u - c * hq * 6, q = rem / 6, j = rem - 6 * q;
          av[w] = 6 * e1 - 1 - (6 * c + j);
          b0v[w] = 6 * e1 - 6 * (c + q) - 6;
          if (u < nu1 && b0v[w] >= 0) load6(av[w], b0v[w], v1[w]);
          else { for (int t = 0; t < 6; ++t) v1[w][t] = 0.0; av[w] = -1; }
        }
#pragma unroll
        for (int w = 0; w < 2; ++w) {
          const int u = u0 + w * kBandThreads;
          if (u >= nu0) continue;
          if (rowv[w] >= 0) fix6(6 * o0 + rowv[w], 6 * (o0 + cv[w]), v[w]);
          double* dst = C0.W + static_cast<size_t>(u) * 6;
#pragma unroll
          for (int t = 0; t < 6; ++t) dst[t] = v[w][t];
        }
#pragma unroll
        for (int w = 0; w < 2; ++w) {
          const int u = u0 + w * kBandThreads;
          if (u >= nu1) continue;
          const int c = u / (hq * 6), rem = u - c * hq * 6, q = rem / 6, j = rem - 6 * q;
          if (av[w] >= 0) fix6(av[w], b0v[w], v1[w]);
#pragma unroll
          for (int t = 0; t < 6; ++t) C1.W[(static_cast<size_t>(c) * h + 6 * q + t) * 6 + j] = v1[w][5 - t];   // row 6q+t <-> b = b0 + 5 - t
        }
      }
      t_g[0] = clock64();
    }
    t_g[1] = clock64();
    // arrow rows + the right-hand-side row (row m): one warp per row, lanes along the columns (rows of A are contiguous in
    // the packed system) -- chain 0 reads columns 0 .. N0-1, chain 1 the mirrored ones; six loads per lane in flight.
    // (An element-indexed loop through sys_index() spent most of the gather's time here at K = 50.)
    {
      const int N0 = has0 ? C0.npc : 0, n1v = has1 ? 6 * C1.Ke : 0;
      const double* Arows = sys + lay.oA;
      constexpr int NW = kBandThreads / 32;
      for (int r0 = warp; r0 <= m; r0 += 2 * NW) {   // two rows per warp and pass: 24 loads per lane in flight
        for (int c0 = 0; c0 < max(N0, N1); c0 += 192) {
          double v0[2][6], v1[2][6];
#pragma unroll
          for (int w = 0; w < 2; ++w) {
            const int r = r0 + w * NW;
            const bool on = r <= m, rhs = (r == m);
            const double* src = Arows + static_cast<size_t>((on && !rhs) ? r : 0) * np;
#pragma unroll
            for (int u = 0; u < 6; ++u) {
              const int col = c0 + lane + 32 * u, col0 = 6 * o0 + col;
              v0[w][u] = (on && col < N0) ? (rhs ? b[col0] - gvec[col0] : src[col0]) : 0.0;
              const int col1 = 6 * e1 - 1 - col;
              v1[w][u] = (on && col < n1v) ? (rhs ? b[col1] - gvec[col1] : src[col1]) : 0.0;
            }
          }
#pragma unroll
          for (int w = 0; w < 2; ++w) {
            const int r = r0 + w * NW;
            if (r > m) continue;
            const bool rfix = (r < m) && s_fix[np + r];
#pragma unroll
            for (int u = 0; u < 6; ++u) {
              const int col = c0 + lane + 32 * u, col1 = 6 * e1 - 1 - col;
              if (col < N0) C0.AR[static_cast<size_t>(r) * N0 + col] = (rfix || s_fix[6 * o0 + col]) ? 0.0 : v0[w][u];
              if (col < N1) C1.AR[static_cast<size_t>(r) * N1 + col] = (col < n1v && !(rfix || s_fix[col1])) ? v1[w][u] : 0.0;
            }
          }
        }
      }
    }
    t_g[2] = clock64();
    t_g[3] = clock64();
    for (int e = tid; hub && e < (m + 1) * m; e += kBandThreads) {
      const int r = e / m, q = e - r * m;
      CC[static_cast<size_t>(r) * LDc + q] = (r < m) ? ((q <= r) ? Sval(np + r, np + q) : 0.0) : bval(np + q);
    }
  }
  __syncthreads();
  long long t_mark = clock64(), t_acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const long long t_gathered = t_mark;
#define HB_TICKD(i, addr) do { if (dbg && tid == 0) { const long long now = clock_after(*reinterpret_cast<const volatile double*>(addr)); t_acc[i] += now - t_mark; t_mark = now; } } while (0)
#define HB_TICK(i) do { if (dbg && tid == 0) { const long long now = clock64(); t_acc[i] += now - t_mark; t_mark = now; } } while (0)
  // ---- two-sided factorisation + forward substitution: step s eliminates block column s of BOTH chains.
  // The 6x6 Cholesky of a chain's NEXT diagonal block is done by its look-ahead warp inside the
  // trailing-update phase, as soon as that block has received its update: off the critical path. ----
  if (tid == 0 && has0 && C0.Ke > 0) { if (!chol6(C0.W, 6, C0.LI)) s_ok = 0; }
  if (tid == 32 && has1 && C1.Ke > 0) { if (!chol6(C1.W, 6, C1.LI)) s_ok = 0; }
  __syncthreads();
  HB_TICK(0);
  // Pipeline of one chain: kWorkers update threads (panel rows, then trailing-update tiles) + its
  // look-ahead warp.  Barrier A: panel of step s complete (update warps sync, look-ahead warp arrives after
  // its first panel block); barrier B: step s complete.  The chains never synchronise with each other.
  __shared__ unsigned char s_tile[2 * 192];
  const int ng_full = (m + 1 + 5) / 6;
  const int ntiles_full = beta * (beta + 1) / 2 + ng_full * beta;
  const bool have_table = ntiles_full <= 192;
  if (have_table) {
    for (int tile = tid; tile < ntiles_full; tile += kBandThreads) {
      int gu, gv;
      const int ntri = beta * (beta + 1) / 2;
      if (tile < ntri) {
        gu = 0;
        while ((gu + 1) * (gu + 2) / 2 <= tile) ++gu;
        gv = tile - gu * (gu + 1) / 2;
      } else { gu = beta + (tile - ntri) / beta; gv = (tile - ntri) % beta; }
      s_tile[2 * tile] = static_cast<unsigned char>(gu);
      s_tile[2 * tile + 1] = static_cast<unsigned char>(gv);
    }
  }
  __syncthreads();
  const int uidx = (warp >> 2) * 3 + sched;   // CL: rank of a scheduler-0..2 warp among the update warps
  const bool is_la = CL ? warp == 15 : (sched < 2) && (warp >> 2) == 3;
  const bool is_worker = CL ? sched < 3 && uidx < kBandUpdWarps : sched >= 2;
  const int wid = CL ? uidx * 32 + lane : (((warp >> 2) & 1) * 2 + (sched - 2)) * 32 + lane;   // 0..kWorkers-1
  constexpr int kWorkers = CL ? 32 * kBandUpdWarps : 128;
  const int barA = 1 + 2 * my_chain, barB = 2 + 2 * my_chain, nbar = kWorkers + 32;
  const int rec_upd = CL ? 0 : 2, rec_la = CL ? 15 : 12;   // the update warp and the look-ahead warp whose steps are stamped
  __shared__ long long s_ts[8][8];
  // Two-sided phase: every step has the full band below it (the separator follows the last eliminated
  // column), so a worker's items are the same every step and their addresses are affine in s: decode once.
  constexpr int kMaxRounds = 3;
  const int nitems_full = ntiles_full * 6 - 6;   // tile 0 belongs to the look-ahead warp
  const bool fast = have_table && pl.Kb > 0 && nitems_full <= kMaxRounds * kWorkers;
  // !SMEM: the workspace lives in global memory (it does not fit); the factorisation then runs chunk by chunk
  // on shared-memory VIEWS of chunk_cols block columns per chain (loaded, eliminated, written back), so its
  // steps see shared-memory latency instead of L2 latency.  V0 / V1 are the views, F the chain structure the
  // step loop works on (the resident chain itself when SMEM).
  BandChain V0 = C0, V1 = C1;
  if (!SMEM) {
    double* p = s_band;
    BandChain* vv[2] = {&V0, &V1};
    for (int i = 0; i < 2; ++i) {
      BandChain& V = *vv[i];
      V.ars = 6 * chunk_cols;
      V.W = p; p += static_cast<size_t>(chunk_cols) * h6;
      V.AR = p; p += static_cast<size_t>(m + 1) * V.ars;
      V.LI = p; p += static_cast<size_t>(chunk_cols) * 48;
      V.X = nullptr;
    }
  }
  const BandChain F = SMEM ? C : (my_chain ? V1 : V0);
  const double* f_u[kMaxRounds]; const double* f_v[kMaxRounds]; double* f_t[kMaxRounds]; int f_su[kMaxRounds]; bool f_ok[kMaxRounds];
#pragma unroll
  for (int r = 0; r < kMaxRounds; ++r) {
    const int t = 6 + wid + kWorkers * r;
    f_ok[r] = fast && is_worker && t < ntiles_full * 6;
    f_u[r] = F.W; f_v[r] = F.W; f_t[r] = F.W; f_su[r] = 0;
    if (f_ok[r]) {
      const int tile = t / 6, i = t - 6 * tile;
      const int gu = s_tile[2 * tile], gv = s_tile[2 * tile + 1];
      const bool ub = gu < beta;
      const int ru = ub ? 0 : 6 * (gu - beta) + i;
      if (!ub && ru > m) f_ok[r] = false;
      else {
        f_u[r] = ub ? (F.W + static_cast<size_t>(6 + 6 * gu + i) * 6) : (F.AR + static_cast<size_t>(ru) * F.ars);
        f_su[r] = ub ? h6 : 6;
        f_v[r] = F.W + static_cast<size_t>(6 + 6 * gv) * 6;
        f_t[r] = ub ? (F.W + (static_cast<size_t>(1 + gv) * h + (6 * (gu - gv) + i)) * 6) : (F.AR + static_cast<size_t>(ru) * F.ars + 6 * (1 + gv));
      }
    }
  }
  auto fast_update = [&](int s) {
#pragma unroll
    for (int r = 0; r < kMaxRounds; ++r) {
      if (!f_ok[r]) continue;
      const double2* x2 = reinterpret_cast<const double2*>(f_u[r] + static_cast<size_t>(s) * f_su[r]);
      const double2* v2 = reinterpret_cast<const double2*>(f_v[r] + static_cast<size_t>(s) * h6);
      double2* t2 = reinterpret_cast<double2*>(f_t[r] + static_cast<size_t>(s) * f_su[r]);
      const double2 a0 = x2[0], a1 = x2[1], a2 = x2[2];
      double2 o0 = t2[0], o1 = t2[1], o2 = t2[2];
      double sd[6];
#pragma unroll
      for (int j = 0; j < 6; ++j) {
        const double2 b0 = v2[3 * j], b1 = v2[3 * j + 1], b2 = v2[3 * j + 2];
        sd[j] = a0.x * b0.x + a0.y * b0.y + a1.x * b1.x + a1.y * b1.y + a2.x * b2.x + a2.y * b2.y;
      }
      o0.x -= sd[0]; o0.y -= sd[1]; o1.x -= sd[2]; o1.y -= sd[3]; o2.x -= sd[4]; o2.y -= sd[5];
      t2[0] = o0; t2[1] = o1; t2[2] = o2;
    }
  };
  // chol_last: the look-ahead of the last step also factors the next diagonal block (more columns follow)
  auto run_steps = [&](const BandChain& Q, int s0, int s1, bool use_fast, bool chol_last) {
    for (int s = s0; s < s1; ++s) {
      const bool rec = dbg && (CL || my_chain == 0) && s >= 4 && s < 12 && lane == 0 && (warp == rec_upd || warp == rec_la);
      if (rec) s_ts[s - 4][warp == rec_upd ? 0 : 4] = clock_after(Q.LI[static_cast<size_t>(s) * 48]);   // released (chol(s) visible)
      if (is_worker) {
        const int nb = min(h - 6, Q.npc - 6 * (s + 1));
        band_panel(Q, s, h, m, wid, kWorkers, nb >= 6 ? 6 : 0);
        if (rec) s_ts[s - 4][1] = clock_after(Q.AR[6 * s]);           // own panel row (arrow row 0... wid 0 -> band row 6) done
        nbar_sync(barA, nbar);
        if (rec) s_ts[s - 4][2] = clock_after(Q.W[static_cast<size_t>(s) * h6 + 36]);   // A released
        if (use_fast) fast_update(s);
        else band_update(Q, s, h, m, 6, wid, kWorkers, have_table ? s_tile : nullptr, beta);
        if (rec) s_ts[s - 4][3] = clock_after(Q.W[static_cast<size_t>(s + 1) * h6 + 36]);  // update done (approx)
      } else {
        if (!band_la_step(Q, s, h, lane, s + 1 < s1 || chol_last, barA, nbar)) s_ok = 0;
        if (rec) s_ts[s - 4][5] = clock_after(Q.LI[static_cast<size_t>(s + 1) * 48]);      // chol(s+1) done
      }
      nbar_sync(barB, nbar);
    }
  };
  // chunk transfer between a chain's global workspace G (columns c0 .. c0 + nview) and its view V, by the
  // 256 threads of the chain's half of the CTA
  auto chunk_copy = [&](const BandChain& G, const BandChain& V, int c0, int nview, bool to_view) {
    const int lt = tid & 255;
    double* gw = G.W + static_cast<size_t>(c0) * h6;
    for (int e = lt; e < nview * h6; e += 256) { if (to_view) V.W[e] = gw[e]; else gw[e] = V.W[e]; }
    double* gl = G.LI + static_cast<size_t>(c0) * 48;
    for (int e = lt; e < nview * 48; e += 256) { if (to_view) V.LI[e] = gl[e]; else gl[e] = V.LI[e]; }
    const int w6 = 6 * nview;
    for (int e = lt; e < (m + 1) * w6; e += 256) {
      const int r = e / w6, j = e - r * w6;
      double* g = G.AR + static_cast<size_t>(r) * G.ars + 6 * c0 + j;
      double* v = V.AR + static_cast<size_t>(r) * V.ars + j;
      if (to_view) *v = *g; else *g = *v;
    }
  };
  // chunked elimination of columns [c_begin, c_end) of both chains (lim0 / lim1: their end columns)
  auto run_chunked = [&](int c_begin, int lim0, int lim1, bool use_fast) {
    const int CH = chunk_cols - beta;
    for (int c0 = c_begin; c0 < max(lim0, lim1); c0 += CH) {
      const BandChain& Gh = (tid >> 8) ? C1 : C0;          // chain of this half of the CTA (copies)
      const BandChain& Vh = (tid >> 8) ? V1 : V0;
      const int limh = (tid >> 8) ? lim1 : lim0;
      const int ncur_h = min(max(limh - c0, 0), CH);
      const int nview_h = ncur_h ? min(ncur_h + beta, Gh.ncol - c0) : 0;
      if (nview_h) chunk_copy(Gh, Vh, c0, nview_h, true);
      __syncthreads();
      const int lim = my_chain ? lim1 : lim0;
      const int ncur = min(max(lim - c0, 0), CH);
      if ((is_la || is_worker) && ncur) {
        BandChain Q = F;
        Q.Ke = ncur; Q.ncol = min(ncur + beta, C.ncol - c0); Q.npc = 6 * Q.ncol;
        run_steps(Q, 0, ncur, use_fast, c0 + ncur < lim);
      }
      __syncthreads();
      if (nview_h) chunk_copy(Gh, Vh, c0, nview_h, false);
      __syncthreads();
    }
  };
  if (SMEM) { if (is_la || is_worker) run_steps(C, 0, C.Ke, fast, false); }
  else run_chunked(0, C0.Ke, C1.Ke, fast);
  __syncthreads();
  if (dbg && tid < 64) dbg[8 + tid] = s_ts[tid >> 3][tid & 7];
  HB_TICKD(1, C.W);
  // ---- the deferred corner update CC -= sum over the eliminated columns of (arrow panel)(arrow panel)^T, rhs row
  // included (row m): FP64 tensor-core tiles (mma.sync m8n8k4 -> SASS DMMA.8x8x4), output tile (ub, vb) of 8 x 8
  // corner entries, K = the eliminated columns in steps of 4.  Operand fragments: lane l holds
  // A[row l/4][k l%4] and B[k l%4][col l/4] -- both are AR[row][col0 + l%4] -- and C[row l/4][col 2(l%4)+{0,1}].
  // One warp owns each output tile and contracts every column of Qa, then of Qb, into it, in a fixed order, so the
  // corner, and with it the step, is bit-identical from solve to solve (splitting a tile's contraction across
  // warps and merging the parts with shared-memory atomics made the chunked solver's step vary in the last bits).
  // store: CC = the sum (a partial that CTA 0 subtracts later) instead of CC -= the sum. ----
  auto corner_update = [&](const BandChain& Qa, const BandChain& Qb, bool store) {
    const int nrb = (m + 1 + 7) / 8, ncb = (m + 7) / 8;
    const int lr = lane >> 2, lk = lane & 3;
    for (int tile = warp; tile < nrb * ncb; tile += kBandThreads / 32) {
      const int ub = tile / ncb, vb = tile - ub * ncb;
      if (vb > ub) continue;
      double c0 = 0.0, c1 = 0.0;
#pragma unroll
      for (int ci = 0; ci < 2; ++ci) {
        const BandChain& Q = ci ? Qb : Qa;
        const int hi = 6 * Q.ne;                    // the chain's eliminated columns
        const double* pa = Q.AR + static_cast<size_t>(min(8 * ub + lr, m)) * Q.npc + lk;
        const double* pb = Q.AR + static_cast<size_t>(min(8 * vb + lr, m)) * Q.npc + lk;
        for (int col = 0; col < hi; col += 16) {
          double av[4], bv[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const bool in = col + 4 * u + lk < hi;
            av[u] = in ? pa[col + 4 * u] : 0.0;
            bv[u] = in ? pb[col + 4 * u] : 0.0;
          }
#pragma unroll
          for (int u = 0; u < 4; ++u)
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(av[u]), "d"(bv[u]));
        }
      }
      const int u = 8 * ub + lr, v = 8 * vb + 2 * lk;
      double* cu = CC + static_cast<size_t>(u) * LDc + v;
      const bool in0 = u <= m && v < m && v <= u, in1 = u <= m && v + 1 < m && v + 1 <= u;
      if (in0) cu[0] = store ? c0 : cu[0] - c0;
      if (in1) cu[1] = store ? c1 : cu[1] - c1;
    }
  };
  // row transform of the first ncols columns of a chain (one row per thread): panel rows B <- B L^-1 and/or the rhs y <- y L^-1
  auto row_transform = [&](const BandChain& Q, int ncols, bool panel, bool rhs) {
    const int rows_per_col = (h - 6) + 1;
    for (int e = tid; e < ncols * rows_per_col; e += kBandThreads) {
      const int c = e / rows_per_col, t = e - c * rows_per_col;
      const int nb = min(h - 6, Q.npc - 6 * (c + 1));
      const double* L = Q.W + static_cast<size_t>(c) * h6;
      const double* rd = Q.LI + static_cast<size_t>(c) * 48;
      if (t < nb) { if (panel) band_transform_row(Q.W + (static_cast<size_t>(c) * h + 6 + t) * 6, L, rd); }
      else if (t == h - 6 && rhs) band_transform_row(Q.AR + static_cast<size_t>(m) * Q.npc + 6 * c, L, rd);
    }
  };
  // arrow contribution to every eliminated block's right-hand side, all at once: y_p -= AR^T x_a (row m of AR = y)
  auto arrow_prepass = [&](const BandChain& Q, const double* xa) {
    for (int col = tid; col < 6 * Q.ne; col += kBandThreads) {
      double sacc = 0.0;
      for (int r = 0; r < m; ++r) sacc += Q.AR[static_cast<size_t>(r) * Q.npc + col] * xa[r];
      Q.AR[static_cast<size_t>(m) * Q.npc + col] -= sacc;
    }
  };
  // ---- corner (m x m, rhs carried as row m): right-looking Cholesky by the whole CTA with FIXED element
  // ownership (element (u, v), v <= min(u, m-1), decoded once), two barriers per column and no
  // division / modulo in the column loop.  The pivot's square root goes to XA's neighbour array DG so
  // that nobody overwrites CC[q][q] while others still read it. ----
  auto corner_solve = [&]() {
    double* DG = XA + m;   // diagonal of the corner factor
    const int ntri = m * (m + 1) / 2, nel = ntri + m;
    auto decode = [&](int e, int* pu, int* pv) {
      if (e < ntri) {
        int u = static_cast<int>((sqrtf(8.0f * e + 1.0f) - 1.0f) * 0.5f);
        while (u * (u + 1) / 2 > e) --u;
        while ((u + 1) * (u + 2) / 2 <= e) ++u;
        *pu = u; *pv = e - u * (u + 1) / 2;
      } else { *pu = m; *pv = e - ntri; }
    };
    int u0 = 0, v0 = m;   // this thread's first element (v0 = m: none)
    if (tid < nel) decode(tid, &u0, &v0);
    double* own0 = CC + static_cast<size_t>(u0) * LDc + v0;
    // Leading full blocks of six columns: the diagonal block in registers (chol6, one thread), one thread per row for the
    // panel, the fixed element ownership for the 6-term trailing update -- three barriers per SIX columns instead of two
    // per column (the scalar loop below spent ~560 cycles per column on barriers and exposed shared-memory latency).
    const int q_blocked = (m / 6) * 6;
    double* cinv = DG + m;   // scratch behind DG: reciprocal diagonal of the current block (6 doubles; the staged damping terms are dead by now)
    for (int k0 = 0; k0 < q_blocked; k0 += 6) {
      if (tid == 0) {
        if (!chol6(CC + static_cast<size_t>(k0) * LDc + k0, LDc, cinv)) s_ok = 0;
#pragma unroll
        for (int j = 0; j < 6; ++j) DG[k0 + j] = CC[static_cast<size_t>(k0 + j) * LDc + k0 + j];
      }
      __syncthreads();
      for (int r = k0 + 6 + tid; r <= m; r += kBandThreads) {   // panel rows, the rhs row (r == m) included
        double* a = CC + static_cast<size_t>(r) * LDc + k0;
        double v[6];
#pragma unroll
        for (int q = 0; q < 6; ++q) v[q] = a[q];
#pragma unroll
        for (int j = 0; j < 6; ++j) {
          v[j] *= cinv[j];
#pragma unroll
          for (int q = j + 1; q < 6; ++q) v[q] -= v[j] * CC[static_cast<size_t>(k0 + q) * LDc + k0 + j];
        }
#pragma unroll
        for (int q = 0; q < 6; ++q) a[q] = v[q];
      }
      __syncthreads();
      if (v0 >= k0 + 6 && v0 < m) {
        const double* pu = CC + static_cast<size_t>(u0) * LDc + k0;
        const double* pv = CC + static_cast<size_t>(v0) * LDc + k0;
        double acc = 0.0;
#pragma unroll
        for (int j = 0; j < 6; ++j) acc += pu[j] * pv[j];
        *own0 -= acc;
      }
      for (int e = tid + kBandThreads; e < nel; e += kBandThreads) {   // only for m > 30
        int u, v;
        decode(e, &u, &v);
        if (v >= k0 + 6) {
          double acc = 0.0;
          for (int j = 0; j < 6; ++j) acc += CC[static_cast<size_t>(u) * LDc + k0 + j] * CC[static_cast<size_t>(v) * LDc + k0 + j];
          CC[static_cast<size_t>(u) * LDc + v] -= acc;
        }
      }
      __syncthreads();
    }
    for (int q = q_blocked; q < m; ++q) {   // the remaining (m mod 6) columns, one at a time
      const double d = CC[static_cast<size_t>(q) * LDc + q];
      const double iv = rsqrt(d);
      if (tid == 0) { if (!(d > 0.0)) s_ok = 0; DG[q] = d * iv; }
      for (int r = q + 1 + tid; r <= m; r += kBandThreads) CC[static_cast<size_t>(r) * LDc + q] *= iv;
      __syncthreads();
      if (v0 > q && v0 < m) *own0 -= CC[static_cast<size_t>(u0) * LDc + q] * CC[static_cast<size_t>(v0) * LDc + q];
      for (int e = tid + kBandThreads; e < nel; e += kBandThreads) {   // only for m > 30
        int u, v;
        decode(e, &u, &v);
        if (v > q) CC[static_cast<size_t>(u) * LDc + v] -= CC[static_cast<size_t>(u) * LDc + q] * CC[static_cast<size_t>(v) * LDc + q];
      }
      __syncthreads();
    }
    HB_TICK(4);
    if (warp == 0) {
      // back substitution with the rhs in registers: lane r holds y_r; x_q = y_q / L_qq is broadcast, then
      // y_r -= L_qr x_q for r < q (row q of L is contiguous: conflict-free)
      for (int base = ((m - 1) / 32) * 32; base >= 0; base -= 32) {   // m <= 32: one pass
        const int r = base + lane;
        double y = (r < m) ? CC[static_cast<size_t>(m) * LDc + r] : 0.0;
        const double dinv = (r < m) ? 1.0 / DG[r] : 0.0;
        // contributions of already solved x (rows above this 32-block)
        for (int q = m - 1; q >= base + 32; --q) if (r < m) y -= CC[static_cast<size_t>(q) * LDc + r] * XA[q];
        for (int q = min(m, base + 32) - 1; q >= base; --q) {
          const double lq = (r < q) ? CC[static_cast<size_t>(q) * LDc + r] : 0.0;
          const double xq = __shfl_sync(0xffffffffu, y * dinv, q - base);
          if (r == q) XA[q] = xq;
          y -= lq * xq;
        }
        __syncwarp();
      }
    }
  };
  if (!CL) {
    // ---- merge chain 1's copy of the separator (index-reversed) and of its arrow columns into chain 0,
    // then chain 0's pipeline eliminates the separator columns ----
    if (pl.Kb) {
      const int nsep = 6 * pl.bs, N1 = C1.npc;
      for (int e = tid; e < nsep * nsep; e += kBandThreads) {
        const int u = e / nsep, v = e - u * nsep;
        if (v > u) continue;
        const int ru = N1 - 1 - u, rv = N1 - 1 - v;   // ru <= rv: stored in block column ru / 6
        C0.W[(static_cast<size_t>(C0.Ke + v / 6) * h + (u - 6 * (v / 6))) * 6 + v % 6] +=
            C1.W[(static_cast<size_t>(ru / 6) * h + (rv - 6 * (ru / 6))) * 6 + ru % 6];
      }
      for (int e = tid; e < (m + 1) * nsep; e += kBandThreads) {
        const int r = e / nsep, v = e - r * nsep;
        C0.AR[static_cast<size_t>(r) * C0.npc + 6 * C0.Ke + v] += C1.AR[static_cast<size_t>(r) * N1 + (N1 - 1 - v)];
      }
      __syncthreads();
      if (tid == 0 && !chol6(C0.W + static_cast<size_t>(C0.Ke) * h6, 6, C0.LI + static_cast<size_t>(C0.Ke) * 48)) s_ok = 0;
      __syncthreads();
      run_chunked(C0.Ke, C0.ncol, 0, false);
      __syncthreads();
    }
    HB_TICKD(2, C0.W);
    // the chunk views are dead: the corner system, its solution and (if they fit) both chains' solution vectors
    // move into that shared memory for the latency-bound tail phases
    __syncthreads();
    double* p = s_band;
    const size_t ncc = static_cast<size_t>(m + 1) * LDc + 2 * static_cast<size_t>(m);
    for (size_t e = tid; e < ncc; e += kBandThreads) p[e] = CC[e];
    CC = p; XA = CC + static_cast<size_t>(m + 1) * LDc;
    p += ncc;
    const size_t avail = 2 * static_cast<size_t>(chunk_cols) * (h6 + 6 * static_cast<size_t>(m + 1) + 48);
    if (ncc + C0.npc + C1.npc <= avail) { C0.X = p; C1.X = p + C0.npc; }
    __syncthreads();
    corner_update(C0, C1, false);
    __syncthreads();
    HB_TICKD(3, CC);
    corner_solve();
    __syncthreads();
    HB_TICKD(5, XA);
    arrow_prepass(C0, XA);
    arrow_prepass(C1, XA);
    __syncthreads();
    row_transform(C0, C0.ne, true, true);
    row_transform(C1, C1.ne, true, true);
    __syncthreads();
    HB_TICKD(7, C.AR);
    // separator columns first (chain 0, warp 0), then outwards: chain 0 in warp 0, chain 1 in warp 1
    if (warp == 0 && C0.ncol > C0.Ke) band_backsub_chain(C0, C0.ncol - 1, C0.Ke, h, m, lane);
    __syncthreads();
    if (pl.Kb) {
      for (int v = tid; v < 6 * pl.bs; v += kBandThreads) C1.X[C1.npc - 1 - v] = C0.X[6 * C0.Ke + v];
      __syncthreads();
    }
    if (warp < 2) {
      const BandChain& Q = warp ? C1 : C0;
      band_backsub_chain(Q, Q.Ke - 1, 0, h, m, lane);
    }
    __syncthreads();
    HB_TICKD(6, C.X);
    for (int e = tid; e < C0.npc; e += kBandThreads) x_out[e] = C0.X[e];
    for (int e = tid; e < m; e += kBandThreads) x_out[np + e] = XA[e];
    for (int e = tid; e < 6 * C1.Ke; e += kBandThreads) x_out[np - 1 - e] = C1.X[e];
  } else {
    // ---- cluster: after its chain, each CTA meets the other at cluster barriers (release on arrive, acquire on wait);
    // data crosses by remote shared-memory stores ahead of a barrier, or by CTA 0's remote loads behind one.
    //   1. CTA 1's separator copy -> CTA 0, which merges it and eliminates the separator;
    //   2. CTA 1's partial corner update and SPD flag -> CTA 0, which factors and solves the corner;
    //   3. the corner's and the separator's solutions -> CTA 1.  Then both CTAs solve their chains outwards. ----
    const int nsep = 6 * pl.bs, peer = 1 - rank;
    const SegChain gp = seg_chain(pl, K, peer);
    const CtaLayout Lo = cta_layout(pl, K, beta, m, rank), Lp = cta_layout(pl, K, beta, m, peer);
    BandChain E = C;   // no columns: corner_update's second operand
    E.ne = 0;
    if (!g.elim && g.Ke && nsep) {   // remote stores do not stall the way remote loads in the merge would
      const double* w = C.W + static_cast<size_t>(C.Ke) * h6;
      for (int e = tid; e < pl.bs * h6; e += kBandThreads) st_peer(ws + Lp.RBW + e, peer, w[e]);
      for (int e = tid; e < (m + 1) * nsep; e += kBandThreads) {
        const int r = e / nsep, v = e - r * nsep;
        st_peer(ws + Lp.RBA + e, peer, C.AR[static_cast<size_t>(r) * C.npc + 6 * C.Ke + v]);
      }
    }
    cluster_arrive(); cluster_wait();   // barrier 1
    if (g.elim) {
      // chain 1's copy is index-reversed: separator-local index u <-> nsep - 1 - u
      const double* rbw = ws + Lo.RBW;
      const double* rba = ws + Lo.RBA;
      for (int e = tid; e < nsep * nsep; e += kBandThreads) {
        const int u = e / nsep, v = e - u * nsep;
        if (v > u) continue;
        const int ru = nsep - 1 - u, rv = nsep - 1 - v;   // ru <= rv: stored in block column ru / 6
        C.W[(static_cast<size_t>(C.Ke + v / 6) * h + (u - 6 * (v / 6))) * 6 + v % 6] +=
            rbw[(static_cast<size_t>(ru / 6) * h + (rv - 6 * (ru / 6))) * 6 + ru % 6];
      }
      for (int e = tid; e < (m + 1) * nsep; e += kBandThreads) {
        const int r = e / nsep, v = e - r * nsep;
        C.AR[static_cast<size_t>(r) * C.npc + 6 * C.Ke + v] += rba[static_cast<size_t>(r) * nsep + (nsep - 1 - v)];
      }
      __syncthreads();
      if (tid == 0 && !chol6(C.W + static_cast<size_t>(C.Ke) * h6, 6, C.LI + static_cast<size_t>(C.Ke) * 48)) s_ok = 0;
      __syncthreads();
      if (is_la || is_worker) run_steps(C, C.Ke, C.ncol, false, false);
      __syncthreads();
    }
    HB_TICKD(2, C.W);
    // the CTA's own part of the corner update (CTA 1: stored as a partial for CTA 0), and its panel rows, which do not
    // depend on the solution
    corner_update(C, E, !hub);
    row_transform(C, C.ne, true, false);
    __syncthreads();
    HB_TICKD(3, CC);
    cluster_arrive(); cluster_wait();   // barrier 2
    if (!hub) HB_TICK(4);
    // the CTA's rhs: arrow pre-pass and transform, then (CTA 0) the separator's back substitution, handed to CTA 1
    auto solve_own = [&]() {
      arrow_prepass(C, XA);
      __syncthreads();
      row_transform(C, C.ne, false, true);
      __syncthreads();
      if (g.elim) {
        if (warp == 0) band_backsub_chain(C, C.ncol - 1, C.Ke, h, m, lane);
        __syncthreads();
        for (int i = tid; i < nsep; i += kBandThreads) st_peer(ws + Lp.X + 6 * gp.Ke + (nsep - 1 - i), peer, C.X[6 * C.Ke + i]);
      }
    };
    if (hub) {
      if (tid == 0 && !ld_peer(&s_ok, 1)) s_ok = 0;   // chain 1's SPD flag
      // CTA 1's partial corner update, subtracted after CTA 0's own (no atomics across the cluster: replicas of the
      // solve stay bit-identical); a window too short for two chains leaves CTA 1 without columns
      const double* pc = ws + Lp.CC;
      for (int e = tid; pl.Kb && e < (m + 1) * m; e += kBandThreads) {
        const int r = e / m, q = e - r * m;
        if (r < m && q > r) continue;
        CC[static_cast<size_t>(r) * LDc + q] -= ld_peer(pc + static_cast<size_t>(r) * LDc + q, 1);
      }
      __syncthreads();
      corner_solve();
      __syncthreads();
      solve_own();
      for (int e = tid; e < m; e += kBandThreads) st_peer(ws + Lp.XA + e, 1, XA[e]);
    }
    cluster_arrive(); cluster_wait();   // barrier 3
    HB_TICK(5);
    if (!hub) solve_own();
    HB_TICKD(7, C.AR);
    if (warp == 0) band_backsub_chain(C, C.Ke - 1, 0, h, m, lane);
    __syncthreads();
    HB_TICKD(6, C.X);
    for (int e = tid; e < 6 * C.ne; e += kBandThreads) x_out[g.rev ? 6 * g.anchor - 1 - e : 6 * g.anchor + e] = C.X[e];
    if (hub)
      for (int e = tid; e < m; e += kBandThreads) x_out[np + e] = XA[e];
  }
  if (dbg && tid == 0) { for (int i = 0; i < 8; ++i) dbg[i] = t_acc[i]; dbg[8 + 6] = t_staged - t_entry; dbg[8 + 7] = t_gathered - t_staged; dbg[8 + 14] = clock64() - t_entry; dbg[8 + 15] = t_g[0] - t_staged; dbg[8 + 22] = t_g[1] - t_g[0]; dbg[8 + 23] = t_g[2] - t_g[1]; dbg[8 + 30] = t_g[3] - t_g[2]; dbg[8 + 31] = t_gathered - t_g[3]; }
  if (tid == 0 && hub) {
    *spd_flag = s_ok;
    if (dbg) dbg[70] = s_ok;   // (a word the step stamps leave free)
  }
  // neither CTA may exit while the other can still read or write its shared memory (last cluster barrier)
  if (CL) { cluster_arrive(); cluster_wait(); }
}

}  // namespace hb
