// Device-side sliding-window bookkeeping (sm_90a): what the reference does per message on its pointer graph --
// appending state elements by extrapolation (reference internal/hyper/optimizers/abstract.cpp:118-144), adding
// residual blocks (reference internal/hyper/optimizers/ceres/optimizer.cpp:189-274), dropping landmarks whose
// observation range left the window together with their residuals (optimizer.cpp:360-382), setting state elements
// at or before the window's lower bound constant and removing the ones no residual touches any more
// (optimizer.cpp:286-345) -- here on the flattened window that already lives in HBM: no host re-sort, no re-upload
// of the factor lists.  New factors arrive in stamp order, so appending keeps the bound order (sorted by knot base);
// removal is an order-preserving stream compaction.  All four families: pixel and bearing factors share the visual
// list (kind in idx.w), inertial and manifold factors have their own; stereo tracks (the reference's live frame loop,
// abstract.cpp:243-260) become bearing factors and new landmarks in stereo_track_kernel.  The bias splines grow by the
// same extrapolation (updateSensor, abstract.cpp:272-292) and lose their leading knots by the same removal rule when
// HB200_SLIDE_DROP_BIAS is set.  The incidence lists (landmark
// CSR, inertial runs, longest track) are built by the counting + scan kernels below, after hb200_bind as after every
// append or slide.
#pragma once
#include "hb200_eval.cuh"

namespace hb {

// ---- exclusive scan of n ints by ONE CTA of 1024 threads (chunk by chunk, carry in a register); total -> *total ----
__global__ void __launch_bounds__(1024) scan_kernel(const int* __restrict__ in, int n, int* __restrict__ out, int* __restrict__ total) {
  __shared__ int s_warp[32];
  __shared__ int s_carry;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    const int i = base + tid;
    const int v = (i < n) ? in[i] : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int w = s_warp[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
      s_warp[lane] = w;
    }
    __syncthreads();
    const int carry = s_carry;
    const int incl = x + (warp ? s_warp[warp - 1] : 0) + carry;
    if (i < n) out[i] = incl - v;
    __syncthreads();
    if (tid == 1023) s_carry = incl;
    __syncthreads();
  }
  if (tid == 0) *total = s_carry;
}

// order-preserving key of a double for atomicMax (stamps are finite)
HB_DI unsigned long long stamp_key(double t) {
  const unsigned long long b = static_cast<unsigned long long>(__double_as_longlong(t));
  return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}
HB_DI double stamp_from_key(unsigned long long k) {
  const unsigned long long b = (k & 0x8000000000000000ull) ? (k & 0x7fffffffffffffffull) : ~k;
  return __longlong_as_double(static_cast<long long>(b));
}

// last observation stamp of every landmark (key 0 = never observed)
__global__ void landmark_last_stamp_kernel(int n, const double* __restrict__ stamp, const int4* __restrict__ idx, unsigned long long* __restrict__ last) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f < n) atomicMax(&last[idx[f].y], stamp_key(stamp[f]));
}
// a landmark stays while its observation range intersects the window: last stamp >= lower bound (reference
// optimizer.cpp:366: !p_landmark->range().intersects(range) -> remove); unobserved landmarks are kept (just added)
__global__ void landmark_keep_kernel(int L, const unsigned long long* __restrict__ last, double lower, int* __restrict__ keep) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l < L) keep[l] = (last[l] == 0ull || stamp_from_key(last[l]) >= lower) ? 1 : 0;
}
// visual factors (pixel and bearing) live and die with their landmark; min_base receives the smallest knot base among
// the kept ones, kept_bearing the number of kept bearing factors (idx.w = 1; one atomic per warp)
__global__ void visual_keep_kernel(int n, const int4* __restrict__ idx, const int* __restrict__ lm_keep, int* __restrict__ keep, int* __restrict__ min_base,
                                   int* __restrict__ kept_bearing) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  const int4 id = idx[f];
  const int k = lm_keep[id.y];
  keep[f] = k;
  if (k) atomicMin(min_base, id.x);
  const unsigned active = __activemask();
  const unsigned b = __ballot_sync(active, k && id.w == 1);
  if (b && (threadIdx.x & 31) == __ffs(active) - 1) atomicAdd(kept_bearing, __popc(b));
}
// inertial (int4 index) and manifold (int2 index) factors: kept (the reference never removes them); with drop_base >= 0
// those whose control points ALL lie at or before the lower bound (base + order - 1 <= drop_base: every block the
// residual moves with is constant) go.  min_bias (inertial only, may be null): smallest kept gyro / accel bias base.
template <typename Idx>
__global__ void inertial_keep_kernel(int n, const Idx* __restrict__ idx, int order, int drop_base, int* __restrict__ keep, int* __restrict__ min_base,
                                     int* __restrict__ min_bias = nullptr) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  const Idx id = idx[f];
  const int k = (drop_base >= 0 && id.x + order - 1 <= drop_base) ? 0 : 1;
  keep[f] = k;
  if (k) atomicMin(min_base, id.x);
  if constexpr (sizeof(Idx) == sizeof(int4)) {
    if (k && min_bias) { atomicMin(&min_bias[0], id.y); atomicMin(&min_bias[1], id.z); }
  }
}

// z: third bearing component of bearing factors (idx.w = 1), moved with the pixel pair.  keep == nullptr keeps every
// factor (pos is then a permutation), lm_pos == nullptr keeps the landmark indices.
__global__ void compact_visual_kernel(int n, const int* __restrict__ keep, const int* __restrict__ pos, const int* __restrict__ lm_pos, int knot_shift,
                                      const double* __restrict__ stamp, const double2* __restrict__ pixel, const double* __restrict__ z,
                                      const int4* __restrict__ idx, double* __restrict__ stamp_o, double2* __restrict__ pixel_o,
                                      double* __restrict__ z_o, int4* __restrict__ idx_o) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n || (keep && !keep[f])) return;
  const int p = pos[f];
  int4 id = idx[f];
  id.x -= knot_shift;
  if (lm_pos) id.y = lm_pos[id.y];
  stamp_o[p] = stamp[f]; pixel_o[p] = pixel[f]; z_o[p] = z[f]; idx_o[p] = id;
}
__global__ void compact_manifold_kernel(int n, const int* __restrict__ keep, const int* __restrict__ pos, int knot_shift, const double* __restrict__ stamp,
                                        const double* __restrict__ meas, const int* __restrict__ sensor, const int2* __restrict__ idx,
                                        double* __restrict__ stamp_o, double* __restrict__ meas_o, int* __restrict__ sensor_o, int2* __restrict__ idx_o) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n || !keep[f]) return;
  const int p = pos[f];
  int2 id = idx[f];
  id.x -= knot_shift;
  stamp_o[p] = stamp[f]; sensor_o[p] = sensor[f]; idx_o[p] = id;
#pragma unroll
  for (int q = 0; q < 7; ++q) meas_o[7 * static_cast<size_t>(p) + q] = meas[7 * static_cast<size_t>(f) + q];
}
// keep == nullptr: every factor stays
__global__ void compact_inertial_kernel(int n, const int* __restrict__ keep, const int* __restrict__ pos, int knot_shift, int gyro_shift, int accel_shift,
                                        const double* __restrict__ stamp, const double* __restrict__ meas, const int4* __restrict__ idx,
                                        double* __restrict__ stamp_o, double* __restrict__ meas_o, int4* __restrict__ idx_o) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n || (keep && !keep[f])) return;
  const int p = pos[f];
  int4 id = idx[f];
  id.x -= knot_shift; id.y -= gyro_shift; id.z -= accel_shift;
  stamp_o[p] = stamp[f]; idx_o[p] = id;
#pragma unroll
  for (int q = 0; q < 6; ++q) meas_o[6 * static_cast<size_t>(p) + q] = meas[6 * static_cast<size_t>(f) + q];
}
__global__ void compact_landmarks_kernel(int L, const int* __restrict__ keep, const int* __restrict__ pos, const double* __restrict__ xyz, double* __restrict__ xyz_o) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= L || !keep[l]) return;
  const int p = pos[l];
#pragma unroll
  for (int c = 0; c < 3; ++c) xyz_o[3 * static_cast<size_t>(p) + c] = xyz[3 * static_cast<size_t>(l) + c];
}
// knots of `stride` doubles (8: state elements, 4: bias knots): drop the first `shift`
__global__ void shift_knots_kernel(int K_new, int shift, int stride, const double* __restrict__ knots, double* __restrict__ knots_o) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < stride * K_new) knots_o[e] = knots[stride * shift + e];
}

// process(VisualTracks) on the device (reference abstract.cpp:243-260): track f becomes the bearing factors at visual
// list positions Nv + 2f (view 0) and Nv + 2f + 1 (view 1), kind 1; a new track (landmark < 0) also writes the landmark
// triangulated at the current state to L + rank[f] (rank: exclusive scan of the new-track flags).  bad counts tracks
// with an invalid stamp, camera or landmark index, and new tracks whose triangulation is not finite (parallel rays).
template <int K>
__global__ void stereo_track_kernel(int n, const double* __restrict__ stamps, const int* __restrict__ cam0, const int* __restrict__ cam1,
                                    const double* __restrict__ px0, const double* __restrict__ px1, const int* __restrict__ landmark,
                                    const int* __restrict__ rank, const double* __restrict__ knots, const double* __restrict__ tab, int Kn, Basis B,
                                    const double* __restrict__ cams, int C, int L, int Nv, double* __restrict__ v_stamp, double2* __restrict__ v_pixel,
                                    double* __restrict__ v_z, int4* __restrict__ v_idx, double* __restrict__ lms, int* __restrict__ bad) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  double b0[3], b1[3], lm[3];
  const int base = stereo_track<K>(f, stamps, cam0, cam1, px0, px1, knots, tab, Kn, B, cams, C, b0, b1, lm);
  const double t = stamps[f];
  const int c0 = cam0[f], c1 = cam1[f], given = landmark[f];
  const bool fresh = given < 0;
  if (base < 0 || given >= L || (fresh && !(isfinite(lm[0]) && isfinite(lm[1]) && isfinite(lm[2])))) { atomicAdd(bad, 1); return; }
  const int l = fresh ? L + rank[f] : given;
  const size_t a = static_cast<size_t>(Nv) + 2 * static_cast<size_t>(f);
  v_stamp[a] = t; v_stamp[a + 1] = t;
  v_pixel[a] = make_double2(b0[0], b0[1]); v_pixel[a + 1] = make_double2(b1[0], b1[1]);
  v_z[a] = b0[2]; v_z[a + 1] = b1[2];
  v_idx[a] = make_int4(base, l, c0, 1); v_idx[a + 1] = make_int4(base, l, c1, 1);
  if (fresh) {
#pragma unroll
    for (int i = 0; i < 3; ++i) lms[3 * static_cast<size_t>(l) + i] = lm[i];
  }
}

// reference abstract.cpp:126-136: the new element and the current last one take the variable of the second to last;
// stamps continue at the knot separation.  Knots of `stride` doubles, the variable in the first `comps`, the stamp at
// `comps` (8 / 7: state elements, 4 / 3: bias knots).  New stamp i is fma(i + 1, dt, last stamp), one rounding: the
// host mirrors of the stamps (hb200_append_bias_knots) compute it the same way.
__global__ void append_knots_kernel(int K, int count, int stride, int comps, double* __restrict__ knots) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  const double dt = knots[stride * (K - 1) + comps] - knots[stride * (K - 2) + comps];
  for (int q = 0; q < comps; ++q) knots[stride * (K - 1) + q] = knots[stride * (K - 2) + q];
  for (int i = 0; i < count; ++i) {
    for (int q = 0; q < comps; ++q) knots[stride * (K + i) + q] = knots[stride * (K - 2) + q];
    knots[stride * (K + i) + comps] = fma(static_cast<double>(i + 1), dt, knots[stride * (K - 1) + comps]);
  }
}

// ---- incidence lists -------------------------------------------------------------------------------------------
// observations per landmark (y)
__global__ void count_kernel(int n, const int4* __restrict__ idx, int* __restrict__ cnt) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f < n) atomicAdd(&cnt[idx[f].y], 1);
}
// fill the landmark CSR; within a landmark the observations must come in bound order (ascending factor index): the
// factor list is sorted by base, so a landmark's first / last observation give its control-point span
__global__ void csr_fill_kernel(int n, const int4* __restrict__ idx, const int* __restrict__ off, int* __restrict__ cursor, int* __restrict__ obs) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  const int l = idx[f].y;
  obs[off[l] + atomicAdd(&cursor[l], 1)] = f;
}
__global__ void csr_sort_kernel(int L, const int* __restrict__ off, int* __restrict__ obs, const int4* __restrict__ idx, int order, int* __restrict__ max_rows) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= L) return;
  const int lo = off[l], hi = off[l + 1];
  for (int i = lo + 1; i < hi; ++i) {   // insertion sort: tracks are a handful of observations
    const int v = obs[i];
    int j = i - 1;
    while (j >= lo && obs[j] > v) { obs[j + 1] = obs[j]; --j; }
    obs[j + 1] = v;
  }
  if (hi > lo) atomicMax(max_rows, 6 * (idx[obs[hi - 1]].x + order - idx[obs[lo]].x));
}
// inertial runs: a run starts where (base, gyro bias base, accel bias base) changes
__global__ void run_flag_kernel(int n, const int4* __restrict__ idx, int* __restrict__ flag) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  int s = 1;
  if (f > 0) { const int4 a = idx[f], b = idx[f - 1]; s = (a.x != b.x || a.y != b.y || a.z != b.z) ? 1 : 0; }
  flag[f] = s;
}
__global__ void run_fill_kernel(int n, const int* __restrict__ flag, const int* __restrict__ pos, int nruns, int* __restrict__ run_off) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f < n && flag[f]) run_off[pos[f]] = f;
  if (f == 0) run_off[nruns] = n;
}
// bound-order check of an appended tail: every new base must be >= the last old one and the tail itself ascending
__global__ void tail_sorted_kernel(int n_old, int n_new, const int4* __restrict__ idx, int* __restrict__ bad) {
  const int f = n_old + blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n_old + n_new || f == 0) return;
  if (idx[f].x < idx[f - 1].x) atomicAdd(bad, 1);
}

// ---- agreement of a sharded window's collective sliding-window calls --------------------------------------------
// Every rank fills one payload of doubles, the ranks SUM it, and every rank reads the same answer from the sum:
//   [ header kVoteHeader | its squares kVoteHeader | status 2 | smallest kept knot base K | gyro bias base Kbg |
//     accel bias base Kba | beta K ]
// The header holds exact small integers (1, K, Kbg, Kba, call kind, slide flags, ub, ubg, uba).  After the sum, entry x
// must give sum(x) = n a and sum(x^2) = n a^2 for this rank's own a (n = nranks, the sum of the leading 1): together
// they say sum((x - a)^2) = 0, so either every rank holds a or every rank sees the mismatch (the sum alone would let
// 1, 3, 5 pass on the rank holding 3).  Status: one rank-count per window-wide
// code (bad index: 2, arrival order: 3).  The votes are one-hot: a rank puts a 1 at its own value, so the sum is
// nonzero exactly at the values some rank voted for -- the first nonzero entry is the minimum, the last the maximum.
constexpr int kVoteHeader = 9, kVoteStatus = 2, kVoteHead = 2 * kVoteHeader + kVoteStatus;   // (status at 2 kVoteHeader, votes at kVoteHead)
__host__ __device__ inline int vote_payload_len(int K, int Kbg, int Kba) { return kVoteHead + 2 * K + Kbg + Kba; }
struct VoteHeader { double v[kVoteHeader]; };
// What a rank votes with; a null pointer (or a minimum of INT_MAX, a family without factors) casts no vote.
struct VoteSrc {
  const int* status;       // [2]: bad-index count, arrival-order count of this rank's validation
  const int* knot_min[3];  // smallest kept knot base of the visual, inertial and manifold factors
  const int* bias_min;     // [2]: smallest kept gyro / accel bias base
  const int* max_rows;     // longest landmark track in control-point rows (csr_sort_kernel); 0: no visual factor
};
// agreed values, as window_agree_kernel writes them
enum { kAgreeStatus = 0, kAgreeMismatch = 1, kAgreeBeta = 2, kAgreeKnotMin = 3, kAgreeGyroMin = 4, kAgreeAccelMin = 5, kAgreeOut = 6 };

// one CTA: zero the payload, then place the header, the status and the one-hot votes
__global__ void __launch_bounds__(256) window_vote_kernel(double* __restrict__ pay, int K, int Kbg, int Kba, int order, VoteHeader h, VoteSrc src) {
  const int len = vote_payload_len(K, Kbg, Kba);
  for (int i = threadIdx.x; i < len; i += blockDim.x) pay[i] = 0.0;
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int i = 0; i < kVoteHeader; ++i) { pay[i] = h.v[i]; pay[kVoteHeader + i] = h.v[i] * h.v[i]; }
  if (src.status) {
    pay[2 * kVoteHeader] = src.status[0] ? 1.0 : 0.0;
    pay[2 * kVoteHeader + 1] = (!src.status[0] && src.status[1]) ? 1.0 : 0.0;
  }
  double* votes = pay + kVoteHead;
  auto vote = [](double* region, int n, int v) { if (v != 0x7fffffff && n > 0) region[min(max(v, 0), n - 1)] = 1.0; };
  int m = 0x7fffffff;
  for (int f = 0; f < 3; ++f) if (src.knot_min[f]) m = min(m, *src.knot_min[f]);
  vote(votes, K, m);
  if (src.bias_min) { vote(votes + K, Kbg, src.bias_min[0]); vote(votes + K + Kbg, Kba, src.bias_min[1]); }
  if (src.max_rows && *src.max_rows > 0) vote(votes + K + Kbg + Kba, K, max(order - 1, *src.max_rows / 6 - 1));
}

// one CTA, on the summed payload: out[kAgree*] (status code 0 / 2 / 3, header mismatch 0 / 1, the largest beta vote (0:
// none), the smallest knot / gyro / accel base votes (INT_MAX: none))
__global__ void __launch_bounds__(256) window_agree_kernel(const double* __restrict__ pay, int K, int Kbg, int Kba, VoteHeader h, int* __restrict__ out) {
  __shared__ int s[kAgreeOut];
  const int t = threadIdx.x;
  if (t == 0) {
    s[kAgreeStatus] = pay[2 * kVoteHeader] > 0.0 ? 2 : (pay[2 * kVoteHeader + 1] > 0.0 ? 3 : 0);
    int bad = 0;
    for (int i = 0; i < kVoteHeader; ++i) bad |= (pay[i] != pay[0] * h.v[i]) | (pay[kVoteHeader + i] != pay[0] * (h.v[i] * h.v[i]));
    s[kAgreeMismatch] = bad;
    s[kAgreeBeta] = 0;
    s[kAgreeKnotMin] = s[kAgreeGyroMin] = s[kAgreeAccelMin] = 0x7fffffff;
  }
  __syncthreads();
  const double* votes = pay + kVoteHead;
  const int len = 2 * K + Kbg + Kba;
  for (int i = t; i < len; i += blockDim.x) {
    if (votes[i] == 0.0) continue;
    if (i < K) atomicMin(&s[kAgreeKnotMin], i);
    else if (i < K + Kbg) atomicMin(&s[kAgreeGyroMin], i - K);
    else if (i < K + Kbg + Kba) atomicMin(&s[kAgreeAccelMin], i - K - Kbg);
    else atomicMax(&s[kAgreeBeta], i - K - Kbg - Kba);
  }
  __syncthreads();
  if (t < kAgreeOut) out[t] = s[t];
}
}  // namespace hb
