// libhyperb200.so -- C-ABI (include/hyperb200.h) over the sm_90a kernels.
// Host-side bookkeeping mirrors what the reference's CeresOptimizer keeps in ceres::Problem
// (reference internal/hyper/optimizers/ceres/optimizer.cpp:189-382) but flattened: one set of
// device arrays per variable family and two factor lists.
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <numeric>
#include <string>
#include <type_traits>
#include <vector>

#include <cuda_runtime.h>
#include <dlfcn.h>

#include "../../include/hyperb200.h"
#include "hb200_bcr.cuh"
#include "hb200_calib.cuh"
#include "hb200_cov.cuh"
#include "hb200_window.cuh"

using namespace hb;

namespace {

thread_local std::string g_error;

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_error = buf;
  return code;
}

#define HB_CUDA(expr)                                                                                   \
  do {                                                                                                  \
    cudaError_t err__ = (expr);                                                                         \
    if (err__ != cudaSuccess) return fail(100 + static_cast<int>(err__), "%s: %s", #expr, cudaGetErrorString(err__)); \
  } while (0)

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;
  cudaError_t ensure(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    cudaError_t e = cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T));
    if (e == cudaSuccess) cap = n;
    return e;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
  // capacity for n elements, the first `keep` of them preserved (amortised doubling; device-to-device copy on `stream`)
  cudaError_t grow(size_t n, size_t keep, cudaStream_t stream) {
    if (n <= cap) return cudaSuccess;
    const size_t ncap = std::max<size_t>(n, cap + cap / 2 + 16);
    T* q = nullptr;
    cudaError_t e = cudaMalloc(&q, ncap * sizeof(T));
    if (e != cudaSuccess) return e;
    if (p && keep) e = cudaMemcpyAsync(q, p, keep * sizeof(T), cudaMemcpyDeviceToDevice, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (p) cudaFree(p);
    p = q; cap = ncap;
    return e;
  }
  void swap(DevBuf& o) { std::swap(p, o.p); std::swap(cap, o.cap); }
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }   // scratch buffers of the API calls do not leak on early error returns
};

// The first failure of a series of calls, all of which run.
cudaError_t first_error(std::initializer_list<cudaError_t> es) {
  for (cudaError_t e : es) if (e != cudaSuccess) return e;
  return cudaSuccess;
}

// The factor lists on the device, one buffer per field.  grow: capacity for n factors, the first `keep` preserved
// (DevBuf::grow on every field); swap: switch with another copy of the list.
struct VisualList {
  DevBuf<double> stamp, z;   // z: a bearing's third component (x, y are in `pixel`)
  DevBuf<double2> pixel;
  DevBuf<int4> idx;
  cudaError_t grow(size_t n, size_t keep, cudaStream_t s) { return first_error({stamp.grow(n, keep, s), z.grow(n, keep, s), pixel.grow(n, keep, s), idx.grow(n, keep, s)}); }
  void swap(VisualList& o) { stamp.swap(o.stamp); z.swap(o.z); pixel.swap(o.pixel); idx.swap(o.idx); }
};
struct InertialList {
  DevBuf<double> stamp, meas;   // meas: [gyro | accel] per factor
  DevBuf<int4> idx;
  cudaError_t grow(size_t n, size_t keep, cudaStream_t s) { return first_error({stamp.grow(n, keep, s), meas.grow(6 * n, 6 * keep, s), idx.grow(n, keep, s)}); }
  void swap(InertialList& o) { stamp.swap(o.stamp); meas.swap(o.meas); idx.swap(o.idx); }
};
struct ManifoldList {
  DevBuf<double> stamp, meas;   // meas: a pose [7] per factor
  DevBuf<int> sensor;
  DevBuf<int2> idx;
  cudaError_t grow(size_t n, size_t keep, cudaStream_t s) {
    return first_error({stamp.grow(n, keep, s), meas.grow(7 * n, 7 * keep, s), sensor.grow(n, keep, s), idx.grow(n, keep, s)});
  }
  void swap(ManifoldList& o) { stamp.swap(o.stamp); meas.swap(o.meas); sensor.swap(o.sensor); idx.swap(o.idx); }
};

void compute_basis(Basis* b, int k) {
  // Blending matrix of the uniform B-spline of order k and its cumulative form (DESIGN.md A.3).
  auto binom = [](int n, int r) { double v = 1; if (r < 0 || r > n) return 0.0; for (int i = 1; i <= r; ++i) v = v * (n - r + i) / i; return v; };
  double M[kMaxOrder][kMaxOrder];
  double fact = 1;
  for (int i = 2; i <= k - 1; ++i) fact *= i;
  for (int s = 0; s < k; ++s)
    for (int n = 0; n < k; ++n) {
      double sum = 0;
      for (int l = s; l <= k - 1; ++l) {
        double pw = 1;
        for (int i = 0; i < k - 1 - n; ++i) pw *= static_cast<double>(k - 1 - l);
        sum += ((l - s) % 2 ? -1.0 : 1.0) * binom(k, l - s) * pw;
      }
      M[s][n] = binom(k - 1, n) / fact * sum;
    }
  b->k = k;
  for (int j = 0; j < k; ++j)
    for (int n = 0; n < k; ++n) {
      double s = 0;
      for (int r = j; r < k; ++r) s += M[r][n];
      b->Mc[j * k + n] = s;
    }
}

// One of the window's uniform B-splines: the pose knots (stride 8) or a bias spline (stride 4), each knot's stamp last.
// val: the current and trial state; stamp: the host mirror of the stamps hb200_bind computed its index maps from, and
// the knot count; dropped: the leading knots the last hb200_slide removed.  Launching helpers take the context.
struct Spline {
  int order = 0;
  const int stride;
  Basis basis{};
  DevBuf<double> val[2];
  std::vector<double> stamp;
  int dropped = 0;
  explicit Spline(int stride) : stride(stride) {}
  int n() const { return static_cast<int>(stamp.size()); }
  size_t doubles() const { return static_cast<size_t>(stride) * stamp.size(); }
  double stamp_of(const double* knots, int j) const { return knots[static_cast<size_t>(stride) * j + stride - 1]; }
  // Knots fit for set: at least k of them, stamps strictly increasing and each step within 1e-6 of the first (the
  // reference only ever creates uniformly separated knots, abstract.cpp:89,128), so all finite.  `what` names a knot.
  int check(int k, int count, const double* knots, const char* what) const {
    if (count < k) return fail(-1, "need at least %d %ss, got %d", k, what, count);
    for (int j = 1; j < count; ++j)
      if (!(stamp_of(knots, j) > stamp_of(knots, j - 1))) return fail(-1, "%s stamps must be strictly increasing (%s %d)", what, what, j);
    const double dt0 = stamp_of(knots, 1) - stamp_of(knots, 0);
    for (int j = 1; j < count; ++j)
      if (!(std::fabs((stamp_of(knots, j) - stamp_of(knots, j - 1)) - dt0) <= 1e-6 * dt0)) return fail(-1, "%s stamps must be uniformly spaced (%s %d)", what, what, j);
    return 0;
  }
  // checked knots as the current state; *changed: the order, the count or a stamp changed: the index maps no longer hold
  int set(int k, int count, const double* knots, cudaStream_t s, bool* changed) {
    std::vector<double> t(count);
    for (int j = 0; j < count; ++j) t[j] = stamp_of(knots, j);
    *changed = k != order || t != stamp;
    stamp.swap(t); order = k;
    compute_basis(&basis, k);
    for (DevBuf<double>& v : val) HB_CUDA(v.ensure(doubles()));
    HB_CUDA(cudaMemcpyAsync(val[0].p, knots, sizeof(double) * doubles(), cudaMemcpyHostToDevice, s));
    HB_CUDA(cudaStreamSynchronize(s));
    return 0;
  }
  // room for `count` more knots in both copies, the current knots kept
  int reserve(int count, cudaStream_t s) {
    for (int i = 0; i < 2; ++i) HB_CUDA(val[i].grow(static_cast<size_t>(stride) * (n() + count), i == 0 ? doubles() : 0, s));
    return 0;
  }
  int append(hb200_ctx* c, int count);   // append_knots_kernel, the new stamps read back into the mirror
  int upper(double t) const { return static_cast<int>(std::upper_bound(stamp.begin(), stamp.end(), t) - stamp.begin()); }
  // Leading knots a slide to lower_bound drops: those before the (order - 1) / 2 knots of padding in front of the lower
  // bound's interval (reference optimizer.cpp:289,331-341), none from min_base (a kept factor's base) on, `order` kept.
  int drop_count(double lower_bound, int min_base) const {
    const int sh = std::min(std::max(0, upper(lower_bound) - 1 - (order - 1) / 2), min_base);
    return std::max(0, std::min(sh, n() - order));
  }
  int shift(hb200_ctx* c, int count);   // the rest shifted into the trial copy (shift_knots_kernel), which is switched in
  int mismatch(const double* knots) const {   // the first knot whose stamp differs from the mirror, or -1
    for (int j = 0; j < n(); ++j) if (stamp_of(knots, j) != stamp[j]) return j;
    return -1;
  }
  // a covariance build's copy of s: its order, basis, stamps and current knots
  int freeze(const Spline& s, cudaStream_t st) {
    order = s.order; basis = s.basis; stamp = s.stamp;
    HB_CUDA(val[0].ensure(doubles()));
    if (n()) HB_CUDA(cudaMemcpyAsync(val[0].p, s.val[0].p, sizeof(double) * doubles(), cudaMemcpyDeviceToDevice, st));
    return 0;
  }
};

// Fewest knots append_knots_kernel must append to a bias spline (stamps s, order kb) so that segment_base accepts t:
// s[left] <= t < s'[K' - right] (left = (kb-1)/2, right = kb-1-left) over the K' extended stamps s', where new stamp
// K - 1 + i is fma(i, dt, s[K-1]) with dt = s[K-1] - s[K-2].  0 on success, 2 for t before the span, -1 past HB200_BIAS_APPEND_MAX.
int bias_append_count(const Spline& spline, double t, int* count) {
  const std::vector<double>& s = spline.stamp;
  const int K = spline.n(), kb = spline.order, left = (kb - 1) / 2, right = kb - 1 - left;
  const double dt = s[K - 1] - s[K - 2];
  auto end_of = [&](int added) {   // the valid span's end with `added` knots appended: stamp of knot K + added - right
    const int j = K + added - right;
    return j < K ? s[j] : std::fma(static_cast<double>(j - (K - 1)), dt, s[K - 1]);
  };
  *count = 0;
  if (t < s[left]) return 2;
  if (t < end_of(0)) return 0;
  const double est = std::floor((t - s[K - 1]) / dt) + right;   // first guess; the loops below decide
  if (!(est <= HB200_BIAS_APPEND_MAX + 1.0)) return -1;
  int n = std::max(1, static_cast<int>(est));
  while (n > 1 && t < end_of(n - 1)) --n;
  while (!(t < end_of(n)) && n <= HB200_BIAS_APPEND_MAX) ++n;
  if (n > HB200_BIAS_APPEND_MAX) return -1;
  *count = n;
  return 0;
}

// ---- NCCL, bound at run time ----------------------------------------------------------------------
// libnccl.so.2 is resolved with dlopen when the first communicator call is made: inside a torch process this is
// the copy torch already loaded (same SONAME), in a plain C++ host the system library.  Only the five entry
// points below are used; their prototypes are those of nccl.h 2.x (ncclUniqueId = 128 bytes by value,
// ncclDouble = 8, ncclSum = 0).
struct NcclUid { char internal[128]; };
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(NcclUid*) = nullptr;
  int (*CommInitRank)(void**, int, NcclUid, int) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
NcclApi g_nccl;
int load_nccl() {
  if (g_nccl.lib) return 0;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  void* h = nullptr;
  for (const char* nm : names) { h = dlopen(nm, RTLD_NOW | RTLD_GLOBAL); if (h) break; }
  if (!h) return fail(300, "libnccl.so.2 not found: %s", dlerror());
  NcclApi a;
  a.lib = h;
  a.GetUniqueId = reinterpret_cast<int (*)(NcclUid*)>(dlsym(h, "ncclGetUniqueId"));
  a.CommInitRank = reinterpret_cast<int (*)(void**, int, NcclUid, int)>(dlsym(h, "ncclCommInitRank"));
  a.CommDestroy = reinterpret_cast<int (*)(void*)>(dlsym(h, "ncclCommDestroy"));
  a.AllReduce = reinterpret_cast<int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t)>(dlsym(h, "ncclAllReduce"));
  a.GetErrorString = reinterpret_cast<const char* (*)(int)>(dlsym(h, "ncclGetErrorString"));
  if (!a.GetUniqueId || !a.CommInitRank || !a.CommDestroy || !a.AllReduce || !a.GetErrorString) return fail(300, "libnccl.so.2 lacks an expected symbol");
  g_nccl = a;
  return 0;
}
#define HB_NCCL(expr)                                                                                              \
  do {                                                                                                             \
    const int r__ = (expr);                                                                                        \
    if (r__ != 0) return fail(300 + r__, "%s: %s", #expr, g_nccl.GetErrorString ? g_nccl.GetErrorString(r__) : "nccl error"); \
  } while (0)

// The linearisation point hb200_build_covariance froze: its output shapes, and copies of the splines and the knot table.
struct CovPoint {
  SysLayout lay{};
  int L = 0, Nv = 0, max_rows = 0;
  Spline pose{8}, gyro{4}, accel{4};   // the current copy only
  DevBuf<double> tab;
};

// The results of hb200_compute_covariance: the packed selected inverse, the landmark marginals, and the requested blocks
// (blk_n) and stamp-pair blocks (pair_n), each with its status.  swap: switch with another copy.
struct CovResults {
  DevBuf<double> packed, lm, blk, pair_joint, pair_rel;
  DevBuf<int> blk_st, pair_st;
  int blk_n = 0, pair_n = 0;
  void swap(CovResults& o) {
    packed.swap(o.packed); lm.swap(o.lm); blk.swap(o.blk); pair_joint.swap(o.pair_joint); pair_rel.swap(o.pair_rel);
    blk_st.swap(o.blk_st); pair_st.swap(o.pair_st); std::swap(blk_n, o.blk_n); std::swap(pair_n, o.pair_n);
  }
};

// The factor kernels' outputs, one buffer per field.  ensure: room for n factors (at least one) at spline order k.
struct VisualOut {
  DevBuf<double> r, Jp, Jl, w;   // per factor: [2] residual, [2][6k] state and [2][3] landmark Jacobians, robust-loss weight
  cudaError_t ensure(size_t n, size_t k) { n = std::max<size_t>(n, 1); return first_error({r.ensure(2 * n), Jp.ensure(12 * k * n), Jl.ensure(6 * n), w.ensure(n)}); }
};
struct InertialOut {
  DevBuf<double> r, Jp, wg, wa, Jg;   // per factor: [6] residual, [6][6k] state Jacobian, [4] + [4] bias weights, [6][2] gravity
  cudaError_t ensure(size_t n, size_t k) {
    n = std::max<size_t>(n, 1);
    return first_error({r.ensure(6 * n), Jp.ensure(36 * k * n), wg.ensure(4 * n), wa.ensure(4 * n), Jg.ensure(12 * n)});
  }
};
struct ManifoldOut {
  DevBuf<double> r, Jp;   // per factor: [6] residual, [6][6k] state Jacobian
  cudaError_t ensure(size_t n, size_t k) { n = std::max<size_t>(n, 1); return first_error({r.ensure(6 * n), Jp.ensure(36 * k * n)}); }
};

// Host mirror of the factor outputs for hb200_factor_evaluate in user order, indexed by factor kind (HB200_PIXEL ...):
// residuals, state, landmark and calibration Jacobians (the last on demand: calib_valid), inertial bias weights and gravity.
struct OutputMirror {
  std::vector<double> r[4], Jp[4], Jl[4], Jc[4], wg, wa, Jg;
  bool valid = false, calib_valid = false;
};

// One capture of the LM iteration.  release: destroy both handles and mark it stale.
struct IterationGraph {
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  bool valid = false;
  void release() { if (exec) cudaGraphExecDestroy(exec); if (graph) cudaGraphDestroy(graph); exec = nullptr; graph = nullptr; valid = false; }
};

}  // namespace

struct hb200_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  // side stream: the inertial / manifold factor kernels (and their J^T J) are independent of the visual ones and
  // run concurrently with them -- a fork / join inside the iteration (and inside its CUDA graph)
  cudaStream_t stream2 = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr, ev_mid = nullptr;
  bool forked = false;
  // hb200_optimize on small windows: the five variable blocks travel as ONE pinned staging buffer each way
  double* h_stage = nullptr;
  size_t h_stage_cap = 0;
  DevBuf<double> d_stage;
  bool own_stream = false;
  bool use_graph = true;
  int num_sms = 0;
  long long launches = 0;
  long long launches_per_iteration = 0;
  long long iter_total = 0, snap_iter_total = 0;   // host mirror of SolverState.iteration (record ring index)
  int last_terminated = 0, last_performed = 0;     // outcome of the last hb200_iterate / hb200_optimize that fetched records
  double last_gmax = 0, last_step_norm = 0, last_x_norm = 0;

  // window state (index 0 = current, 1 = trial): the pose knots and their table, and the two bias splines of one order
  Spline pose{8}, gyro{4}, accel{4};
  int C = 0, L = 0;
  DevBuf<double> grav[2], lms[2], tab[2];
  DevBuf<double> cams, imu, cam_tab, imu_tab;
  DevBuf<unsigned char> fixed;
  std::vector<unsigned char> h_knot_const;
  int k() const { return pose.order; }
  int K() const { return pose.n(); }
  int Kbg() const { return gyro.n(); }
  int Kba() const { return accel.n(); }
  int gravity_const = 0, bias_const = 0;
  bool have_imu = false, have_gravity = false;
  double huber = 0.5, imu_scale = 1.6e-5, radius0 = 1e4;
  // ceres::Solver::Options termination tests (off: hb200_iterate runs exactly the requested number of iterations)
  bool term_enabled = false;
  double term_ftol = 1e-6, term_gtol = 1e-10, term_ptol = 1e-8, term_min_radius = 1e-32;

  // factor lists, on the device only (the setters write them in user order, hb200_bind sorts them into bound order):
  // the visual list holds pixel and bearing factors (kind flag in idx.w), which travel through the same kernels and the
  // same compact layout; inertial and manifold (pose) factors have their own lists.  A compaction writes a list's spare
  // copy and switches it in.  Spares grow as the live lists do, since the next append grows what was the spare, and
  // hold at least one factor, as every list.
  int Nv = 0, Ni = 0, Np = 0, Nb = 0, Nm = 0, P = 0;
  std::vector<double> h_sensors;
  VisualList visual, visual_spare;
  InertialList inertial, inertial_spare;
  ManifoldList manifold, manifold_spare;
  DevBuf<double> sensors;
  double huber_bearing = 1.6e-3;   // reference optimizer.cpp:204
  // list position -> user index (visual: pixel factors 0 .. Np-1, bearing factors Np .. Nv-1); appends and slides clear
  // them, ensure_perms rebuilds them
  std::vector<int> v_perm, i_perm;
  DevBuf<int> run_off, lm_off, lm_obs, d_invalid;
  // large windows: landmarks ordered by first knot base and cut into groups for schur_group_kernel
  DevBuf<int> lm_order, lm_group_off;
  int n_lm_groups = 0, schur_rt = 0;
  bool schur_groups = false;
  int nruns = 0, max_rows = 6;
  int imu_splits = 1, imu_splits_mma = 1;
  // beta = max(own, min_beta, agreed_beta): min_beta is the caller's floor (hb200_set_min_bandwidth), agreed_beta the
  // largest own value over the ranks at the latest agreement (hb200_bind with NCCL, or the last collective sliding-window
  // call) -- the packed layout must be identical on every rank, and it shrinks again when the longest track leaves
  int beta = 3, min_beta = 0, agreed_beta = 0;
  bool band_solver = true, band_smem = true, force_dense = false;
  DevBuf<double> band_ws;
  int band_chunk_cols = 0;       // !band_smem: block columns per shared-memory chunk view (per chain)
  size_t band_chunk_smem = 0;
  // long windows: multi-CTA block cyclic reduction instead of the single-CTA chain (hb200_bcr.cuh)
  bool use_bcr = false;
  BcrPlan bcr{};
  int bcr_ctas = 0;
  size_t bcr_smem = 0;
  DevBuf<double> bcr_ws;
  DevBuf<unsigned int> bcr_bar;
  DevBuf<long long> band_dbg;   // optional phase timings of band_solve_kernel (HB200_BAND_TIMING=1)
  bool bound = false;

  // device-side window bookkeeping (hb200_append_* / hb200_slide).  w_lkeep / w_lpos: landmark keep flags and new
  // positions of the last hb200_slide (slide_L landmarks before it; -1: none yet), kept until the next slide for
  // hb200_slide_landmark_map
  DevBuf<int> w_keep, w_pos, w_lkeep, w_lpos, w_cnt, w_scal;
  DevBuf<double> w_vote;   // sharded contexts: the agreement payload of a collective sliding-window call (agree_round)
  int slide_L = -1;
  // hb200_append_stereo_tracks inputs: [stamp | pixel0 | pixel1] and [camera0 | camera1 | landmark | new flag | rank]
  DevBuf<double> trk_d;
  DevBuf<int> trk_i;
  DevBuf<unsigned long long> w_last;
  // outputs, in list order (derive_window sizes them), and their host mirror in user order (hb200_factor_evaluate)
  VisualOut v_out;
  InertialOut i_out;
  ManifoldOut m_out;
  DevBuf<double> cp_pix[2], cp_imu[2];
  int n_pix_blocks = 0, n_imu_blocks = 0, n_man_blocks = 0;   // manifold cost partials follow the inertial ones in cp_imu
  bool evaluated_J = false;
  OutputMirror mirror;
  int quirks = 0;   // the reference-quirk switches

  // system (band-only packed storage, see SysLayout)
  int n = 0;
  SysLayout lay{};
  DevBuf<double> sys, D, Lw, Ldiag, dp, dl, Vchol, gl, Dl, lm_part, scal;
  DevBuf<int> spd;
  DevBuf<SolverState> st, records;
  int max_records = 64;
  int n_lm_blocks = 0;
  bool system_built = false;

  // deterministic assembly (hb200_set_deterministic; DetOut, hb200_eval.cuh): the J^T J kernels' record regions, the
  // records, the entry -> records index and its ready flag.  det_ready: the regions fit the current window
  // (prepare_det, dropped by kernel_args_changed()).
  bool deterministic = false, det_ready = false;
  DetOut det_pix{}, det_imu{}, det_man{}, det_schur{};
  long long det_records = 0;
  DevBuf<double> det_val;
  DevBuf<int> det_key, det_cnt, det_off, det_perm, det_flag, det_seg_off;

  // marginal covariances (hb200_build_covariance / hb200_compute_covariance).  cov_st: the build's own solver state
  // (radius +inf: no damping inside the landmark elimination; st is never touched).  cov_at: launch count after the last
  // covariance call -- any other launch since (an evaluation, an iteration, a slide) rewrote what the compute reads.
  // cov_pt: two linearisation points.  The build freezes one into the slot that is not committed (cov_slot_built); a
  // successful compute commits it by index (cov_slot_committed, meaningful while cov_valid), so a failed compute or a
  // build not yet computed leaves every reader on the committed point.  cov_res: the committed results; a compute writes
  // cov_next and a successful one switches the two.  The results are not part of a point: a second compute with no build
  // in between writes results while the built point is the committed one.
  DevBuf<SolverState> cov_st;
  DevBuf<double> cov_ws;
  CovResults cov_res, cov_next;
  DevBuf<int> cov_counts;
  DevBuf<CovStatus> cov_status;
  bool cov_built = false, cov_valid = false;
  long long cov_at = -1;
  int cov_degenerate = 0, cov_unobserved = 0;
  CovPoint cov_pt[2];
  int cov_slot_built = 0, cov_slot_committed = 0;
  DevBuf<double> cov_t, cov_o;   // hb200_interpolate_covariance / hb200_interpolate_state_covariance staging
  DevBuf<int> cov_bad;
  // requested blocks (hb200_set_covariance_blocks): the registered list, its device copy, the landmark spans and the
  // far-column plan and scratch of a compute
  std::vector<int4> cov_req;
  DevBuf<int4> cov_req_d;
  DevBuf<int2> cov_span;
  DevBuf<int> cov_plan;
  DevBuf<double> cov_far;
  // stamp pairs (hb200_set_covariance_stamp_pairs): the registered [t_a, t_b] per pair and their device copy (their
  // control-point spans follow the requests' landmark spans in cov_span)
  std::vector<double> cov_pairs;
  DevBuf<double> cov_pairs_d;

  hb200_allreduce_fn allreduce = nullptr;
  void* allreduce_user = nullptr;
  // multi-GPU: one NCCL all-reduce of the packed system per iteration, enqueued from C on the context's stream
  // (graph-capturable); the step-acceptance scalars travel through peer memory inside accept_kernel
  void* nccl = nullptr;
  bool own_nccl = false;
  long long nccl_calls = 0, nccl_calls_per_iteration = 0;
  int nranks = 1, rank = 0;
  bool comm_warm = false;        // one eager all-reduce has run (NCCL's lazy setup is done: safe to capture)
  DevBuf<double> mbox;           // the peer arena: [mailbox | flags | partial system A | partial system B] (hb200_solve.cuh)
  long long arena_cap = 0;       // doubles per partial
  int peer_par = 0;              // arena half the NEXT iteration assembles into
  bool peer_reduce_wanted = true;
  DevBuf<unsigned long long> red_round;
  DevBuf<unsigned int> red_arrive;
  bool peer_reduce() const { return nccl && peers_open && peer_reduce_wanted && lay.total <= arena_cap; }
  double* assembly() { return peer_reduce() ? mbox.p + kArenaParts + static_cast<long long>(peer_par) * arena_cap : sys.p; }
  DevBuf<unsigned long long> mbox_seq;
  DevBuf<double*> d_peers;
  std::vector<void*> peer_ptrs;  // cudaIpcOpenMemHandle mappings (own entry = mbox.p)
  bool peers_open = false;
  bool multi() const { return nccl != nullptr || allreduce != nullptr; }

  // profiling (hb200_profile_iteration)
  bool profiling = false;
  std::vector<cudaEvent_t> prof_events;
  std::vector<std::string> prof_names;
  size_t prof_used = 0;
  // snapshot (the variable blocks in the order of state_blocks)
  DevBuf<double> snap[5];
  DevBuf<SolverState> snap_st;
  bool have_snapshot = false;

  // the captured iteration, by the arena half it assembles into (peer_par; without the peer-memory reduction only half A)
  IterationGraph graphs[2];

  // family weight matrices (hb200_set_weights): which families have one, the device table the WT kernel instantiations
  // read (kWtSize doubles, identity where a family has none) and its host copy
  bool wt_set[4] = {false, false, false, false};
  DevBuf<double> wt;
  std::array<double, kWtSize> h_wt = [] {
    std::array<double, kWtSize> t{};
    const int sides[4] = {2, 6, 1, 6}, offs[4] = {kWtPixel, kWtInertial, kWtBearing, kWtManifold};   // indexed by HB200_PIXEL ...
    for (int f = 0; f < 4; ++f) for (int i = 0; i < sides[f]; ++i) t[offs[f] + (sides[f] + 1) * i] = 1.0;
    return t;
  }();
  bool wt_visual() const { return wt_set[HB200_PIXEL] || wt_set[HB200_BEARING]; }

  int o_bg() const { return 6 * K(); }
  int o_ba() const { return 6 * K() + 3 * Kbg(); }
  int o_g() const { return 6 * K() + 3 * Kbg() + 3 * Kba(); }

  // What a change makes stale, from the narrowest to the widest.  The calibration and output mirrors are only read
  // while evaluated_J holds, so dropping them with it never refuses a valid call.  `bound` and `have_snapshot` are
  // cleared by the callers that need it: appends keep the window bound but drop the snapshot, a new camera count
  // unbinds the window but keeps the snapshot.
  // constants or the state changed: the built system and the covariance build no longer match them
  void system_changed() { system_built = false; cov_built = false; }
  // the factor outputs changed or no longer match the state
  void outputs_changed() { system_changed(); evaluated_J = false; mirror.valid = false; mirror.calib_valid = false; }
  // something the captured iterations were recorded with changed (a kernel argument, the communicator, the peers)
  void iterations_changed() { for (IterationGraph& g : graphs) g.valid = false; }
  // shapes or buffers the captured iteration was recorded with changed
  void kernel_args_changed() { outputs_changed(); iterations_changed(); det_ready = false; }

  // The variable blocks in their canonical order (knots, gyroscope bias, accelerometer bias, gravity, landmarks): the
  // current state, the trial state, the snapshot and the block's length in doubles.  Every LM step rewrites the whole
  // trial state before reading it, so hb200_slide compacts the current state into the trial copy and switches the two.
  struct StateBlock { DevBuf<double>* cur; DevBuf<double>* trial; DevBuf<double>* snap; size_t count; };
  std::array<StateBlock, 5> state_blocks() {
    auto spline = [&](Spline& s, int i) { return StateBlock{&s.val[0], &s.val[1], &snap[i], s.doubles()}; };
    return {{spline(pose, 0), spline(gyro, 1), spline(accel, 2),
             {&grav[0], &grav[1], &snap[3], 3},
             {&lms[0], &lms[1], &snap[4], 3 * static_cast<size_t>(L)}}};
  }
};

namespace {

void prof_mark(hb200_ctx* c, const char* what) {
  if (!c->profiling) return;
  if (c->prof_used == c->prof_events.size()) { cudaEvent_t e; cudaEventCreate(&e); c->prof_events.push_back(e); c->prof_names.emplace_back(); }
  cudaEventRecord(c->prof_events[c->prof_used], c->stream);
  c->prof_names[c->prof_used] = what;
  c->prof_used += 1;
}

int check_launch(hb200_ctx* c, const char* what) {
  c->launches += 1;
  prof_mark(c, what);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(100 + static_cast<int>(e), "launch %s: %s", what, cudaGetErrorString(e));
  return 0;
}

#define HB_LAUNCH(ctx, what)                       \
  do {                                             \
    int rc__ = check_launch(ctx, what);            \
    if (rc__) return rc__;                         \
  } while (0)

int Spline::append(hb200_ctx* c, int count) {
  if (const int rc = reserve(count, c->stream)) return rc;
  append_knots_kernel<<<1, 32, 0, c->stream>>>(n(), count, stride, stride - 1, val[0].p);
  HB_LAUNCH(c, "append_knots_kernel");
  std::vector<double> tail(static_cast<size_t>(stride) * count);
  HB_CUDA(cudaMemcpyAsync(tail.data(), val[0].p + doubles(), sizeof(double) * tail.size(), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  for (int i = 0; i < count; ++i) stamp.push_back(stamp_of(tail.data(), i));
  return 0;
}
int Spline::shift(hb200_ctx* c, int count) {
  dropped = count;
  if (!count) return 0;
  shift_knots_kernel<<<(stride * (n() - count) + 255) / 256, 256, 0, c->stream>>>(n() - count, count, stride, val[0].p, val[1].p);
  HB_LAUNCH(c, "shift_knots_kernel");
  val[0].swap(val[1]);
  stamp.erase(stamp.begin(), stamp.begin() + count);
  return 0;
}

// The kernels are instantiated per spline order: f(std::integral_constant<int, K>) for K = k.
template <typename F>
int with_order(int k, F&& f) {
  if (k == 4) return f(std::integral_constant<int, 4>{});
  if (k == 6) return f(std::integral_constant<int, 6>{});
  return fail(-4, "spline order %d not supported (4 or 6)", k);
}
// f(std::true_type) or f(std::false_type), for the kernels' bool template flags
template <typename F>
int with_flag(bool b, F&& f) {
  return b ? f(std::true_type{}) : f(std::false_type{});
}
// f(K, DET) for both spline orders and both assembly modes: kernel attributes are set for every instantiation at once
template <typename F>
int for_each_order_mode(F&& f) {
  for (const int k : {4, 6})
    for (const bool det : {false, true})
      if (const int rc = with_order(k, [&](auto K) { return with_flag(det, [&](auto D) { return f(K, D); }); })) return rc;
  return 0;
}

// Launch configuration of the resident band solver: a grid of one 2-CTA cluster (chain r in CTA r) on the context's
// stream, each chain's workspace in its CTA's shared memory.  at: storage for the cluster-dimension attribute.
void band_cluster_config(hb200_ctx* c, cudaLaunchConfig_t* cfg, cudaLaunchAttribute* at) {
  cfg->gridDim = dim3(2); cfg->blockDim = dim3(kBandThreads); cfg->stream = c->stream;
  cfg->dynamicSmemBytes = band_cluster_doubles(c->K(), c->beta, c->n - 6 * c->K()) * sizeof(double);
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = 2; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg->attrs = at; cfg->numAttrs = 1;
}

cudaStream_t side(hb200_ctx* c) { return c->forked ? c->stream2 : c->stream; }
int fork_side(hb200_ctx* c) {
  if (c->profiling || c->forked || !c->stream2) return 0;   // the per-launch profile wants a serial timeline
  HB_CUDA(cudaEventRecord(c->ev_fork, c->stream));
  HB_CUDA(cudaStreamWaitEvent(c->stream2, c->ev_fork, 0));
  c->forked = true;
  return 0;
}
int join_side(hb200_ctx* c) {
  if (!c->forked) return 0;
  HB_CUDA(cudaEventRecord(c->ev_join, c->stream2));
  HB_CUDA(cudaStreamWaitEvent(c->stream, c->ev_join, 0));
  c->forked = false;
  return 0;
}

int update_fixed(hb200_ctx* c) {
  c->n = 6 * c->K() + 3 * c->Kbg() + 3 * c->Kba() + 2;
  std::vector<unsigned char> f(c->n, 0);
  for (int j = 0; j < c->K() && j < static_cast<int>(c->h_knot_const.size()); ++j)
    if (c->h_knot_const[j]) for (int a = 0; a < 6; ++a) f[6 * j + a] = 1;
  if (c->bias_const) for (int a = c->o_bg(); a < c->o_g(); ++a) f[a] = 1;
  if (c->gravity_const) { f[c->o_g()] = 1; f[c->o_g() + 1] = 1; }
  HB_CUDA(c->fixed.ensure(c->n));
  HB_CUDA(cudaMemcpyAsync(c->fixed.p, f.data(), c->n, cudaMemcpyHostToDevice, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

// dense work copy of the reduced system: only the dense fallback solver and hb200_get_system need it
int ensure_dense(hb200_ctx* c) {
  const size_t n = c->n;
  const size_t T = (n + kCholNB - 1) / kCholNB;
  HB_CUDA(c->Lw.ensure((T * kCholNB + 1) * n));
  HB_CUDA(c->Ldiag.ensure(T * kCholNB * kCholNB));
  return 0;
}

int ensure_system(hb200_ctx* c) {
  const size_t n = c->n;
  // block half-bandwidth of the reduced pose system = longest landmark track in control points (>= k - 1)
  c->beta = std::max(std::max(c->k() - 1, c->max_rows / 6 - 1), std::max(c->min_beta, c->agreed_beta));
  c->beta = std::min(c->beta, std::max(c->K() - 1, 0));
  c->lay = sys_layout(c->K(), c->beta, c->n - 6 * c->K());
  HB_CUDA(c->sys.ensure(static_cast<size_t>(c->lay.total)));
  HB_CUDA(c->D.ensure(n));
  HB_CUDA(c->dp.ensure(n));
  HB_CUDA(c->dl.ensure(3 * static_cast<size_t>(std::max(c->L, 1))));
  HB_CUDA(c->Vchol.ensure(9 * static_cast<size_t>(std::max(c->L, 1))));
  HB_CUDA(c->gl.ensure(3 * static_cast<size_t>(std::max(c->L, 1))));
  HB_CUDA(c->Dl.ensure(3 * static_cast<size_t>(std::max(c->L, 1))));
  c->n_lm_blocks = (c->L + kLmWarps - 1) / kLmWarps;
  HB_CUDA(c->lm_part.ensure(5 * static_cast<size_t>(std::max(c->n_lm_blocks, 1))));
  HB_CUDA(c->scal.ensure(8));
  HB_CUDA(c->spd.ensure(1));
  HB_CUDA(c->records.ensure(c->max_records));
  // solver selection: block-banded + arrowhead unless the band is wide on a large system
  const size_t ws = band_workspace_doubles(c->K(), c->beta, c->n - 6 * c->K()) * sizeof(double);
  c->band_solver = !c->force_dense && ((c->n <= 512) || (12 * (c->beta + 1) <= 6 * c->K()));
  c->band_smem = ws <= kBandSmemBytes;
  c->use_bcr = false;
  if (c->band_solver && !c->band_smem && 6 * c->beta <= kBcrMaxNb && c->n - 6 * c->K() <= 54) {
    // the band does not fit one CTA's shared memory: cyclic reduction over super-blocks of beta control points
    const int m = c->n - 6 * c->K();
    const int nsb = (c->K() + c->beta - 1) / c->beta;
    const int nctas = std::max(1, std::min(c->num_sms, (nsb + 1) / 2));
    const BcrPlan pl = bcr_plan(c->K(), c->beta, m, nctas);
    const size_t nb = pl.nb;
    const size_t p1 = nb * (nb | 1) + nb + 1 + nb * (((2 * nb + m + 1 + 11) / 16) * 16 + 4) + static_cast<size_t>(m + 1) * m;
    const size_t p2 = 3 * nb * nb + 2 * nb * m + 2 * nb;
    const size_t mp = static_cast<size_t>((m + 5) / 6) * 6;
    const size_t p3 = mp * (mp | 1) + 3 * (mp + 1) + 8;                       // corner: padded matrix, reciprocal diagonal, rhs, solution
    const size_t p4 = nb * static_cast<size_t>(m + 1);                         // corner partials: staged Y_f | y
    const size_t p5 = 2 * (nb + 1) + 2 * nb + m + 2 + nb * (nb | 1);           // way back: rv, x, staged neighbours, L
    const size_t smem = std::max(std::max(p1, p2), std::max(p3, std::max(p4, p5))) * sizeof(double);
    if (smem <= 220 * 1024) {
      if (nctas != c->bcr_ctas || pl.total != c->bcr.total) {
        HB_CUDA(c->bcr_ws.ensure(static_cast<size_t>(pl.total)));
        HB_CUDA(c->bcr_bar.ensure(1));
        HB_CUDA(cudaMemsetAsync(c->bcr_bar.p, 0, sizeof(unsigned int), c->stream));   // the grid-barrier counter stays a multiple of the grid size
      }
      c->bcr = pl; c->bcr_ctas = nctas; c->bcr_smem = smem; c->use_bcr = true;
      HB_CUDA(cudaFuncSetAttribute(bcr_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    }
  }
  if (c->band_solver && !c->use_bcr) {
    if (c->band_smem) {
      // resident workspace: one chain per CTA of a 2-CTA cluster, each CTA with its own chain's workspace
      cudaLaunchConfig_t cfg{};
      cudaLaunchAttribute at[1];
      band_cluster_config(c, &cfg, at);
      HB_CUDA(cudaFuncSetAttribute(band_solve_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(cfg.dynamicSmemBytes)));
      int nclusters = 0;
      HB_CUDA(cudaOccupancyMaxActiveClusters(&nclusters, band_solve_kernel<true>, &cfg));
      if (nclusters < 1) return fail(-6, "band solver: a cluster of 2 CTAs x %d threads with %zu B of shared memory each cannot be resident", kBandThreads, cfg.dynamicSmemBytes);
    } else {
      HB_CUDA(c->band_ws.ensure(ws / sizeof(double)));
      // chunked factorisation: two shared-memory views of band_chunk_cols block columns (band + arrow + LI)
      const size_t colbytes = (static_cast<size_t>(6 + 6 * c->beta) * 6 + 6 * static_cast<size_t>(c->n - 6 * c->K() + 1) + 48) * sizeof(double);
      const int fit = static_cast<int>((200 * 1024) / (2 * colbytes));
      c->band_chunk_cols = std::max(c->beta + 2, std::min(fit, c->K() + c->beta));
      // after the factorisation the corner system [m + 1][m | 1], its solution and factor diagonal (2m) and the
      // 6-double block scratch behind them move into the same shared memory (band_solve_kernel<false>): a wide
      // arrowhead needs more than the two chunk views
      const int m = c->n - 6 * c->K();
      const size_t corner = (static_cast<size_t>(m + 1) * (m | 1) + 2 * static_cast<size_t>(m) + 6) * sizeof(double);
      c->band_chunk_smem = std::max(2 * colbytes * c->band_chunk_cols, corner);
      if (c->band_chunk_smem > 220 * 1024) return fail(-6, "band solver: a chunk of %d block columns or the %d x %d corner does not fit shared memory (arrow too wide)", c->band_chunk_cols, m, m);
      HB_CUDA(cudaFuncSetAttribute(band_solve_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(c->band_chunk_smem)));
    }
  }
  HB_CUDA(c->band_ws.ensure(1));
  if (!c->band_solver) { int rc = ensure_dense(c); if (rc) return rc; }
  if (getenv("HB200_BAND_TIMING")) HB_CUDA(c->band_dbg.ensure(144));   // 72 per CTA of the cluster kernel
  // parallelism of the inertial J^T J kernels.  Scalar kernel: ~2 CTAs per SM, at least kImuMinChunk factors per CTA
  constexpr int kImuMinChunk = 8;
  c->imu_splits = std::max(1, std::min((2 * c->num_sms + std::max(c->nruns, 1) - 1) / std::max(c->nruns, 1), std::max(1, c->Ni / (kImuMinChunk * std::max(c->nruns, 1)))));
  // tensor-core kernel (large windows): ~kImuCtasPerSm CTAs per SM, at least two 8-factor chunks per CTA
  constexpr int kImuCtasPerSm = 6;
  c->imu_splits_mma = std::max(1, std::min((kImuCtasPerSm * c->num_sms + std::max(c->nruns, 1) - 1) / std::max(c->nruns, 1), std::max(1, c->Ni / (16 * std::max(c->nruns, 1)))));
  return 0;
}

int reset_solver_state(hb200_ctx* c) {
  SolverState s{};
  s.radius = c->radius0; s.decrease_factor = 2.0; s.spd = 1;
  HB_CUDA(c->st.ensure(1));
  HB_CUDA(cudaMemcpyAsync(c->st.p, &s, sizeof(s), cudaMemcpyHostToDevice, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  c->iter_total = 0;
  return 0;
}

// ---- kernel dispatch on (order, bias order) -------------------------------------------------
template <bool J>
PixelArgs pixel_args(hb200_ctx* c, int sel, double* sys) {
  PixelArgs a{};
  a.sys = sys; a.lay = c->lay; a.tiles_per_cta = 1;
  a.n = c->Nv; a.stamp = c->visual.stamp.p; a.pixel = c->visual.pixel.p; a.meas_z = c->visual.z.p; a.idx = c->visual.idx.p;
  a.tab = c->tab[sel].p; a.cam_tab = c->cam_tab.p; a.landmarks = c->lms[sel].p;
  a.r = J ? c->v_out.r.p : nullptr; a.Jp = c->v_out.Jp.p; a.Jl = c->v_out.Jl.p; a.w = c->v_out.w.p; a.cost_partial = c->cp_pix[J ? 0 : 1].p; a.huber = c->huber; a.huber_bearing = c->huber_bearing; a.K_knots = c->K();
  return a;
}
template <bool J>
InertialArgs inertial_args(hb200_ctx* c, int sel) {
  InertialArgs a{};
  a.n = c->Ni; a.stamp = c->inertial.stamp.p; a.meas = c->inertial.meas.p; a.idx = c->inertial.idx.p; a.tab = c->tab[sel].p; a.imu_tab = c->imu_tab.p;
  a.bg = c->gyro.val[sel].p; a.ba = c->accel.val[sel].p; a.gravity = c->grav[sel].p;
  a.r = J ? c->i_out.r.p : nullptr; a.Jp = c->i_out.Jp.p; a.wg = c->i_out.wg.p; a.wa = c->i_out.wa.p; a.Jg = c->i_out.Jg.p;
  a.cost_partial = c->cp_imu[J ? 0 : 1].p; a.loss_scale = c->imu_scale;
  return a;
}
// f(FUSE, DET) with the pixel body's flags: a Jacobian sweep with a system to accumulate into fuses the pixel J^T J,
// into the records of the deterministic assembly when the context asks for it
template <bool J, typename F>
int with_pixel_pass(const hb200_ctx* c, const PixelArgs& a, F&& f) {
  if constexpr (J) {
    if (a.sys) return with_flag(c->deterministic, [&](auto D) { return f(std::true_type{}, D); });
  }
  return f(std::false_type{}, std::false_type{});
}
template <int K, bool J>
int launch_pixel(hb200_ctx* c, int sel, double* sys) {
  if (c->Nv == 0) return 0;
  const PixelArgs a = pixel_args<J>(c, sel, sys);
  return with_pixel_pass<J>(c, a, [&](auto FUSE, auto DET) {
    return with_flag(c->wt_visual(), [&](auto WT) {
      pixel_eval_kernel<K, J, FUSE, DET, WT><<<c->n_pix_blocks, kEvalThreads, 0, c->stream>>>(a, c->pose.basis, DET ? c->det_pix : DetOut{}, DET ? c->det_seg_off.p : nullptr,
                                                                                            c->wt.p);
      return check_launch(c, DET ? "pixel_eval_det_kernel" : "pixel_eval_kernel");
    });
  });
}
template <int K, bool J>
int launch_inertial(hb200_ctx* c, int sel) {
  if (c->Ni == 0) return 0;
  const InertialArgs a = inertial_args<J>(c, sel);
  return with_flag(c->wt_set[HB200_INERTIAL], [&](auto WT) {
    inertial_eval_kernel<K, 4, J, WT><<<c->n_imu_blocks, kEvalThreads, J ? inertial_stash_bytes(K) : 0, side(c)>>>(a, c->pose.basis, c->gyro.basis, c->wt.p);
    return check_launch(c, "inertial_eval_kernel");
  });
}
// visual + inertial factors in one launch (both lists non-empty)
template <int K, bool J>
int launch_factors_merged(hb200_ctx* c, int sel, double* sys) {
  const PixelArgs pa = pixel_args<J>(c, sel, sys);
  const InertialArgs ia = inertial_args<J>(c, sel);
  const int blocks = c->n_pix_blocks + c->n_imu_blocks;
  return with_pixel_pass<J>(c, pa, [&](auto FUSE, auto DET) {
    return with_flag(c->wt_visual() || c->wt_set[HB200_INERTIAL], [&](auto WT) {
      factor_eval_kernel<K, 4, J, FUSE, DET, WT><<<blocks, kEvalThreads * factor_lanes(K), 0, c->stream>>>(pa, ia, c->pose.basis, c->gyro.basis, c->n_pix_blocks,
                                                                                           DET ? c->det_pix : DetOut{}, DET ? c->det_seg_off.p : nullptr, c->wt.p);
      return check_launch(c, DET ? "factor_eval_det_kernel" : "factor_eval_kernel");
    });
  });
}
template <int K, bool J>
int launch_manifold(hb200_ctx* c, int sel) {
  if (c->Nm == 0) return 0;
  ManifoldArgs a{};
  a.n = c->Nm; a.stamp = c->manifold.stamp.p; a.meas = c->manifold.meas.p; a.idx = c->manifold.idx.p; a.tab = c->tab[sel].p; a.sensors = c->sensors.p;
  a.r = J ? c->m_out.r.p : nullptr; a.Jp = c->m_out.Jp.p; a.cost_partial = c->cp_imu[J ? 0 : 1].p + c->n_imu_blocks;
  return with_flag(c->wt_set[HB200_MANIFOLD], [&](auto WT) {
    manifold_eval_kernel<K, J, WT><<<c->n_man_blocks, kEvalThreads, 0, side(c)>>>(a, c->pose.basis, c->wt.p);
    return check_launch(c, "manifold_eval_kernel");
  });
}

// The factor kernels of state `sel` (0: current, 1: trial) on its up-to-date knot table: residuals and cost partials,
// Jacobians with want_J.  sys (enqueue_assembly): Jacobians, the pixel J^T J fused into this packed system, and the
// side stream left forked for enqueue_build.
int enqueue_factors(hb200_ctx* c, bool want_J, int sel, double* sys = nullptr) {
  int rc = 0;
  const bool J_any = want_J || sys;
  // Small windows are latency-bound: one launch for both factor families, each factor on a lane group.  Large windows
  // are throughput-bound: one factor per thread, the families in separate kernels (a lane group repeats the work that
  // does not depend on the spline step on every lane, which costs issue slots there).
  if (c->Nv && c->Ni && c->n_pix_blocks + c->n_imu_blocks <= 4 * c->num_sms) {   // (also while profiling: same kernels as the graph)
    // visual and inertial factors side by side in one launch; pose factors (if any) on the side stream
    if (c->Nm && (rc = fork_side(c))) return rc;
    rc = with_order(c->k(), [&](auto K) {
      return with_flag(J_any, [&](auto J) {
        const int r = launch_factors_merged<K, J>(c, sel, sys);
        return r ? r : launch_manifold<K, J>(c, sel);
      });
    });
    // always join here: the inertial Jacobians were produced on the MAIN stream, so the J^T J kernels that follow
    // (enqueue_build) must not run on a still-forked side stream
    { const int rj = join_side(c); if (!rc) rc = rj; }
    return rc;
  }
  // visual factors on the main stream, inertial + manifold factors concurrently on the side stream
  if (c->Nv && (c->Ni || c->Nm) && (rc = fork_side(c))) return rc;
  // sys (fused path): the pixel J^T J is accumulated by the factor kernel itself
  rc = with_order(c->k(), [&](auto K) {
    return with_flag(J_any, [&](auto J) {
      int r = launch_pixel<K, J>(c, sel, sys);
      if (!r) r = launch_inertial<K, J>(c, sel);
      return r ? r : launch_manifold<K, J>(c, sel);
    });
  });
  if (rc || !sys) { const int rj = join_side(c); if (!rc) rc = rj; }
  return rc;
}

// Knot table of state `sel`, then its factor sweep
int enqueue_evaluate(hb200_ctx* c, bool want_J, int sel) {
  prep_kernel<<<(c->K() + 255) / 256, 256, 0, c->stream>>>(c->K(), c->pose.val[sel].p, c->tab[sel].p, nullptr, 0);
  HB_LAUNCH(c, "prep_kernel");
  return enqueue_factors(c, want_J, sel);
}

// The rest of the normal equations, after the factor kernels have cleared the packed system and accumulated the pixel
// J^T J into it: J^T J of the inertial / manifold factors and the cost sum on the side stream, the landmark Schur
// complement on the main stream.  Both accumulate into S with atomics (commutative), diag(J^T J) is kept apart from S,
// so nothing orders them.  The side stream is forked here, not before the evaluation, when the factor Jacobians were
// produced on the MAIN stream (merged factor kernel).
// st: the solver state whose radius damps the landmark blocks (the LM's c->st, or the covariance build's radius +inf).
// Inertial J^T J: large windows (>= 16 384 inertial factors) take the augmented product on the FP64 tensor cores, ~6 CTAs
// per SM of 8-factor chunks; small windows the scalar block-by-block kernel on short runs (cfg1, ~9 factors per CTA), which
// is faster there.  (Order 6 keeps 12-factor chunks at ~2 CTAs per SM, which beat 8-factor chunks at ~6 CTAs per SM on the
// order-6 window.)  A set inertial weight matrix makes the bias columns dense, which only the augmented product covers: it
// selects the tensor-core kernel at every size.  Returns the CTAs per run.
int inertial_splits(const hb200_ctx* c, bool* scalar_hess) {
  *scalar_hess = c->Ni < 16384 && !c->wt_set[HB200_INERTIAL];
  return (*scalar_hess || c->k() != 4) ? c->imu_splits : c->imu_splits_mma;
}

// DET instantiations (deterministic assembly) write the records of their region of the context's DetOut instead of
// adding into the packed system; their profile labels keep the _det_kernel names.
int enqueue_build(hb200_ctx* c, const SolverState* st) {
  const bool det = c->deterministic;
  if (det && !c->det_ready) return fail(-2, "deterministic assembly: record slots not laid out for this window");
  { const int rf = fork_side(c); if (rf) return rf; }   // (no-op when already forked or while profiling)
  if (c->Ni) {
    bool scalar_hess = false;
    const int splits = inertial_splits(c, &scalar_hess);
    const int grid = c->nruns * splits;
    const int rc = with_order(c->k(), [&](auto K) {
      return with_flag(det, [&](auto DET) {
        const DetOut d = DET ? c->det_imu : DetOut{};
        if (scalar_hess)
          inertial_hessian_kernel<K, 4, DET><<<grid, kHessThreads, 0, side(c)>>>(c->run_off.p, c->inertial.idx.p, c->i_out.r.p, c->i_out.Jp.p, c->i_out.wg.p, c->i_out.wa.p, c->i_out.Jg.p,
                                                                                 c->imu_scale, c->assembly(), c->lay, c->o_bg(), c->o_ba(), c->o_g(), splits, d);
        else if (c->wt_set[HB200_INERTIAL])
          inertial_hessian_mma_kernel<K, 4, K == 4 ? 8 : 12, DET, true><<<grid, kHessThreads, 0, side(c)>>>(c->run_off.p, c->inertial.idx.p, c->i_out.r.p, c->i_out.Jp.p, c->i_out.wg.p,
                                                                                                           c->i_out.wa.p, c->i_out.Jg.p, c->imu_scale, c->assembly(), c->lay,
                                                                                                           c->o_bg(), c->o_ba(), c->o_g(), splits, d, c->wt.p);
        else
          inertial_hessian_mma_kernel<K, 4, K == 4 ? 8 : 12, DET, false><<<grid, kHessThreads, 0, side(c)>>>(c->run_off.p, c->inertial.idx.p, c->i_out.r.p, c->i_out.Jp.p, c->i_out.wg.p, c->i_out.wa.p,
                                                                                                            c->i_out.Jg.p, c->imu_scale, c->assembly(), c->lay, c->o_bg(), c->o_ba(),
                                                                                                            c->o_g(), splits, d, nullptr);
        return check_launch(c, scalar_hess ? (DET ? "inertial_hessian_det_kernel" : "inertial_hessian_kernel")
                                           : (DET ? "inertial_hessian_mma_det_kernel" : "inertial_hessian_mma_kernel"));
      });
    });
    if (rc) return rc;
  }
  if (c->Nm) {
    const int blocks = (c->Nm + kManWarps - 1) / kManWarps;
    const int rc = with_order(c->k(), [&](auto K) {
      return with_flag(det, [&](auto DET) {
        manifold_hessian_kernel<K, DET><<<blocks, kManWarps * 32, 0, side(c)>>>(c->Nm, c->manifold.idx.p, c->m_out.r.p, c->m_out.Jp.p, c->assembly(), c->lay,
                                                                               DET ? c->det_man : DetOut{});
        return check_launch(c, DET ? "manifold_hessian_det_kernel" : "manifold_hessian_kernel");
      });
    });
    if (rc) return rc;
  }
  if (c->forked) {   // the cost partials of the visual factors come from the main stream
    HB_CUDA(cudaEventRecord(c->ev_mid, c->stream));
    HB_CUDA(cudaStreamWaitEvent(c->stream2, c->ev_mid, 0));
  }
  cost_kernel<<<1, 256, 0, side(c)>>>(c->assembly(), c->lay, c->cp_pix[0].p, c->Nv ? c->n_pix_blocks : 0, c->cp_imu[0].p, c->n_imu_blocks + c->n_man_blocks);
  HB_LAUNCH(c, "cost_kernel");
  if (c->Nv && c->L && c->schur_groups) {
    const size_t smem = (3 * static_cast<size_t>(kSchurGroup) * (c->schur_rt + 1) + 3 * kSchurGroup + 4 * 3 * static_cast<size_t>(c->schur_rt)) * sizeof(double);
    const int rc = with_order(c->k(), [&](auto K) {
      return with_flag(det, [&](auto DET) {
        schur_group_kernel<K, DET><<<c->n_lm_groups, kSchurGThreads, smem, c->stream>>>(c->lm_group_off.p, c->lm_order.p, c->lm_off.p, c->lm_obs.p, c->visual.idx.p, c->v_out.r.p,
                                                                                        c->v_out.Jp.p, c->v_out.Jl.p, c->v_out.w.p, st, c->assembly(), c->lay, c->Vchol.p, c->gl.p,
                                                                                        c->Dl.p, c->schur_rt, DET ? c->det_schur : DetOut{});
        return check_launch(c, DET ? "schur_group_det_kernel" : "schur_group_kernel");
      });
    });
    if (rc) return rc;
  } else if (c->Nv && c->L) {
    const size_t smem = 2 * 3 * static_cast<size_t>(c->max_rows) * sizeof(double);
    const int rc = with_order(c->k(), [&](auto K) {
      return with_flag(det, [&](auto DET) {
        schur_kernel<K, DET><<<c->L, kSchurThreads, smem, c->stream>>>(c->lm_off.p, c->lm_obs.p, c->visual.idx.p, c->v_out.r.p, c->v_out.Jp.p, c->v_out.Jl.p, c->v_out.w.p, st,
                                                                       c->assembly(), c->lay, c->Vchol.p, c->gl.p, c->Dl.p, c->max_rows, DET ? c->det_schur : DetOut{});
        return check_launch(c, DET ? "schur_det_kernel" : "schur_kernel");
      });
    });
    if (rc) return rc;
  }
  { const int rj = join_side(c); if (rj) return rj; }
  if (!det) return 0;
  // the fixed-order sums: the entry index (built by the first build after the slots were laid out), then every entry
  long long nrec = c->det_records;
  const int* key = c->det_key.p;
  int nent = static_cast<int>(c->lay.total);
  int *cnt = c->det_cnt.p, *off = c->det_off.p, *perm = c->det_perm.p, *flag = c->det_flag.p;
  void* args[] = {&nrec, &key, &nent, &cnt, &off, &perm, &flag};
  HB_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(det_index_kernel), dim3(c->num_sms), dim3(kDetThreads), args, 0, c->stream));
  HB_LAUNCH(c, "det_index_kernel");
  const int blocks = static_cast<int>(std::min<long long>((nent + kDetThreads - 1) / kDetThreads, 8LL * c->num_sms));
  det_reduce_kernel<<<std::max(blocks, 1), kDetThreads, 0, c->stream>>>(nent, c->det_off.p, c->det_perm.p, c->det_val.p, c->assembly());
  HB_LAUNCH(c, "det_reduce_kernel");
  return 0;
}

// The normal equations at the current state: the knot-table launch also zeroes the packed system, the Jacobian sweep
// accumulates the pixel J^T J into it (rewriting the same residuals and Jacobians), enqueue_build does the rest.
// st: as for enqueue_build.  The deterministic record slots must be laid out (prepare_det) before this is enqueued.
int enqueue_assembly(hb200_ctx* c, const SolverState* st) {
  const size_t nclear = static_cast<size_t>(c->lay.total);
  const int blocks = static_cast<int>(std::min<size_t>((nclear / 4 + 255) / 256, static_cast<size_t>(c->num_sms) * 4));
  prep_kernel<<<std::max(blocks, (c->K() + 255) / 256), 256, 0, c->stream>>>(c->K(), c->pose.val[0].p, c->tab[0].p, c->assembly(), nclear);
  HB_LAUNCH(c, "prep_kernel");
  const int rc = enqueue_factors(c, true, 0, c->assembly());
  return rc ? rc : enqueue_build(c, st);
}

// Lays out the deterministic assembly's record regions for the bound window and clears the keys and the entry index,
// which the next build rebuilds.  Eager (it reads the pixel segment count back), so it runs before a build is enqueued or
// captured; once per window shape (kernel_args_changed() drops det_ready).
int prepare_det(hb200_ctx* c) {
  if (!c->deterministic || c->det_ready) return 0;
  long long off = 0;
  auto region = [&](DetOut& d, long long slots, long long per_slot) { d.off = off; d.per_slot = per_slot; off += slots * per_slot; };
  c->det_pix = c->det_imu = c->det_man = c->det_schur = DetOut{};
  const int rc = with_order(c->k(), [&](auto K) {
    if (c->Nv) {   // pixel: one slot per (64-factor tile, knot-base segment)
      const int tiles = c->n_pix_blocks;
      HB_CUDA(c->det_seg_off.ensure(2 * (static_cast<size_t>(tiles) + 1)));   // offsets | counts
      int* counts = c->det_seg_off.p + tiles + 1;
      HB_CUDA(cudaMemsetAsync(counts, 0, sizeof(int) * (static_cast<size_t>(tiles) + 1), c->stream));
      det_pixel_segments_kernel<<<(tiles + 127) / 128, 128, 0, c->stream>>>(c->Nv, c->visual.idx.p, counts);
      HB_LAUNCH(c, "det_pixel_segments_kernel");
      HB_CUDA(c->w_scal.ensure(8));
      scan_kernel<<<1, 1024, 0, c->stream>>>(counts, tiles + 1, c->det_seg_off.p, c->w_scal.p);
      HB_LAUNCH(c, "scan_kernel");
      int segs = 0;
      HB_CUDA(cudaMemcpyAsync(&segs, c->w_scal.p, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
      HB_CUDA(cudaStreamSynchronize(c->stream));
      region(c->det_pix, segs, kEvalThreads * pixel_det_writes<K>());
    }
    if (c->Ni) {   // inertial: one slot per CTA
      bool scalar_hess = false;
      const int splits = inertial_splits(c, &scalar_hess);
      region(c->det_imu, static_cast<long long>(c->nruns) * splits, kHessThreads * (scalar_hess ? ImuHessScalar<K, 4>::DET_WRITES : imu_hess_mma_det_writes<K, 4>()));
    }
    if (c->Nm) region(c->det_man, c->Nm, 32 * manifold_det_writes<K>());   // one slot per factor
    if (c->Nv && c->L) {   // one slot per landmark group / landmark
      if (c->schur_groups) region(c->det_schur, c->n_lm_groups, kSchurGThreads * schur_group_det_writes(c->schur_rt));
      else region(c->det_schur, c->L, kSchurThreads * schur_det_writes(c->max_rows));
    }
    return 0;
  });
  if (rc) return rc;
  if (off >= (1LL << 31) - 1 || c->lay.total >= (1LL << 31) - 1)
    return fail(-6, "deterministic assembly: %lld records for a system of %lld entries exceed 32-bit indexing", off, c->lay.total);
  c->det_records = off;
  HB_CUDA(c->det_val.ensure(std::max<long long>(off, 1))); HB_CUDA(c->det_key.ensure(std::max<long long>(off, 1)));
  HB_CUDA(c->det_perm.ensure(std::max<long long>(off, 1)));
  HB_CUDA(c->det_cnt.ensure(static_cast<size_t>(c->lay.total))); HB_CUDA(c->det_off.ensure(static_cast<size_t>(c->lay.total) + 1));
  HB_CUDA(c->det_flag.ensure(1));
  HB_CUDA(cudaMemsetAsync(c->det_key.p, 0xff, sizeof(int) * std::max<long long>(off, 1), c->stream));
  HB_CUDA(cudaMemsetAsync(c->det_flag.p, 0, sizeof(int), c->stream));
  for (DetOut* d : {&c->det_pix, &c->det_imu, &c->det_man, &c->det_schur}) { d->val = c->det_val.p; d->key = c->det_key.p; }
  HB_CUDA(cudaStreamSynchronize(c->stream));
  c->det_ready = true;
  return 0;
}

// band-only raw system -> dense damped work copy Lw (dense fallback solver, hb200_get_system)
int enqueue_densify(hb200_ctx* c) {
  int rc = ensure_dense(c);
  if (rc) return rc;
  const size_t total = static_cast<size_t>(c->n + 1) * c->n;
  const int blocks = static_cast<int>(std::min<size_t>((total + 255) / 256, static_cast<size_t>(c->num_sms) * 8));
  densify_kernel<<<blocks, 256, 0, c->stream>>>(c->sys.p, c->lay, c->st.p, c->fixed.p, c->D.p, c->Lw.p, c->spd.p);
  HB_LAUNCH(c, "densify_kernel");
  return 0;
}

RetractArgs retract_args(hb200_ctx* c);
// Both solvers read the raw band-only system and apply LM damping + the constant-dof mask themselves (the band
// solver while it gathers, the dense fallback in densify_kernel);
// fuse_retract: the landmark back-substitution launch also retracts knots / biases / gravity (returns *fused)
int enqueue_solve(hb200_ctx* c, bool fuse_retract = false, bool* fused = nullptr) {
  if (c->use_bcr) {
    const double* sys = c->sys.p; SysLayout lay = c->lay; BcrPlan pl = c->bcr; double* ws = c->bcr_ws.p; unsigned int* bar = c->bcr_bar.p;
    double* x = c->dp.p; int* spd = c->spd.p; const SolverState* st = c->st.p; const unsigned char* fx = c->fixed.p; double* Dout = c->D.p;
    long long* dbg = c->band_dbg.p;
    void* args[] = {&sys, &lay, &pl, &ws, &bar, &x, &spd, &st, &fx, &Dout, &dbg};
    HB_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(bcr_solve_kernel), dim3(c->bcr_ctas), dim3(kBcrThreads), args, c->bcr_smem, c->stream));
    c->launches += 1;
    prof_mark(c, "bcr_solve_kernel");
  } else if (c->band_solver) {
    const SolverState* st = c->st.p;
    const unsigned char* fx = c->fixed.p;
    double* Dout = c->D.p;
    if (c->band_smem) {
      cudaLaunchConfig_t cfg{};
      cudaLaunchAttribute at[1];
      band_cluster_config(c, &cfg, at);
      HB_CUDA(cudaLaunchKernelEx(&cfg, band_solve_kernel<true>, static_cast<const double*>(c->sys.p), c->lay, c->band_ws.p, c->dp.p, c->spd.p, c->band_dbg.p, st, fx, Dout, 0));
    } else band_solve_kernel<false><<<1, kBandThreads, c->band_chunk_smem, c->stream>>>(c->sys.p, c->lay, c->band_ws.p, c->dp.p, c->spd.p, c->band_dbg.p, st, fx, Dout, c->band_chunk_cols);
    HB_LAUNCH(c, c->band_smem ? "band_solve_kernel" : "band_solve_kernel<false>");   // (the chunked path gets its own profile label)
  } else {
    { const int rd = enqueue_densify(c); if (rd) return rd; }
    int n = c->n;
    double* Lw = c->Lw.p; double* Ld = c->Ldiag.p; int* spd = c->spd.p;
    void* args[] = {&Lw, &Ld, &n, &spd};
    const int T = (n + kCholNB - 1) / kCholNB;
    const long long tiles = static_cast<long long>(T) * (T + 1) / 2 + T;
    int blocks = static_cast<int>(std::min<long long>(c->num_sms, std::max<long long>(1, (tiles + kCholWarps - 1) / kCholWarps)));
    HB_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(cholesky_kernel), dim3(blocks), dim3(kCholThreads), args, kCholSmem, c->stream));
    c->launches += 1;
    prof_mark(c, "cholesky_kernel");
    backsolve_kernel<<<1, 1024, 0, c->stream>>>(c->Lw.p, c->Ldiag.p, c->n, c->dp.p);
    HB_LAUNCH(c, "backsolve_kernel");
  }
  if (c->L) {
    if (c->Nv) {
      RetractArgs ra{};
      int extra = 0;
      if (fuse_retract) {
        ra = retract_args(c);
        extra = (std::max(std::max(c->K(), 1), std::max(c->Kbg(), c->Kba())) + kLmWarps * 32 - 1) / (kLmWarps * 32);
        if (fused) *fused = true;
      }
      const int rc = with_order(c->k(), [&](auto K) {
        lm_backsub_kernel<K><<<c->n_lm_blocks + extra, kLmWarps * 32, 0, c->stream>>>(c->L, c->lm_off.p, c->lm_obs.p, c->visual.idx.p, c->v_out.r.p, c->v_out.Jp.p, c->v_out.Jl.p, c->v_out.w.p,
                                                                                 c->Vchol.p, c->gl.p, c->Dl.p, c->dp.p, c->dl.p, c->lm_part.p, c->lms[0].p, c->lms[1].p, c->n_lm_blocks, ra);
        return check_launch(c, "lm_backsub_kernel");
      });
      if (rc) return rc;
    } else {
      HB_CUDA(cudaMemsetAsync(c->dl.p, 0, 3 * static_cast<size_t>(c->L) * sizeof(double), c->stream));
      HB_CUDA(cudaMemsetAsync(c->lm_part.p, 0, 5 * static_cast<size_t>(c->n_lm_blocks) * sizeof(double), c->stream));
    }
  }
  return 0;
}

RetractArgs retract_args(hb200_ctx* c) {
  RetractArgs ra{};
  ra.K = c->K(); ra.Kbg = c->Kbg(); ra.Kba = c->Kba(); ra.L = c->L;
  ra.dp = c->dp.p; ra.dl = c->dl.p; ra.knots = c->pose.val[0].p; ra.bg = c->gyro.val[0].p; ra.ba = c->accel.val[0].p; ra.grav = c->grav[0].p; ra.lms = c->lms[0].p;
  ra.knots_t = c->pose.val[1].p; ra.bg_t = c->gyro.val[1].p; ra.ba_t = c->accel.val[1].p; ra.grav_t = c->grav[1].p; ra.lms_t = c->lms[1].p; ra.tab_t = c->tab[1].p;
  ra.retract_landmarks = (c->L && !c->Nv) ? 1 : 0;
  return ra;
}
int enqueue_retract(hb200_ctx* c) {
  const int m = std::max(std::max(c->K(), c->L), std::max(std::max(c->Kbg(), c->Kba()), 1));
  retract_kernel<<<(m + 127) / 128, 128, 0, c->stream>>>(retract_args(c));
  HB_LAUNCH(c, "retract_kernel");
  return 0;
}

int enqueue_scalars(hb200_ctx* c) {
  scalars_kernel<<<1, 256, 0, c->stream>>>(c->cp_pix[1].p, c->Nv ? c->n_pix_blocks : 0, c->cp_imu[1].p, c->n_imu_blocks + c->n_man_blocks, c->lm_part.p,
                                          (c->L && c->Nv) ? c->n_lm_blocks : 0, c->scal.p);
  HB_LAUNCH(c, "scalars_kernel");
  return 0;
}

TermArgs term_args(hb200_ctx* c) {
  TermArgs t{};
  t.enabled = c->term_enabled ? 1 : 0;
  t.function_tolerance = c->term_ftol; t.gradient_tolerance = c->term_gtol; t.parameter_tolerance = c->term_ptol; t.min_radius = c->term_min_radius;
  t.K = c->K(); t.Kbg = c->Kbg(); t.Kba = c->Kba();
  t.knots = c->pose.val[0].p; t.knots_t = c->pose.val[1].p; t.bg = c->gyro.val[0].p; t.bg_t = c->gyro.val[1].p; t.ba = c->accel.val[0].p; t.ba_t = c->accel.val[1].p;
  t.grav = c->grav[0].p; t.grav_t = c->grav[1].p;
  return t;
}

int enqueue_accept(hb200_ctx* c) {
  ScalarArgs sa{c->cp_pix[1].p, c->Nv ? c->n_pix_blocks : 0, c->cp_imu[1].p, c->n_imu_blocks + c->n_man_blocks, c->lm_part.p, (c->L && c->Nv) ? c->n_lm_blocks : 0};
  CommitArgs a{};
  const auto blocks = c->state_blocks();
  size_t mx = 1, total = 0;
  for (int i = 0; i < 5; ++i) {
    a.count[i] = blocks[i].count; a.src[i] = blocks[i].trial->p; a.dst[i] = blocks[i].cur->p;
    mx = std::max(mx, blocks[i].count); total += blocks[i].count;
  }
  const bool fuse_commit = total <= 65536;   // small windows: one CTA commits the accepted state right away
  // scalars: summed inside this kernel on one GPU and, across GPUs, exchanged by it through peer memory; only the
  // fallbacks (callback hook, no peer mapping) run scalars_kernel + a second reduction before it
  const bool mailbox = c->nccl && c->peers_open;
  MailboxArgs mb{};
  mb.nranks = mailbox ? c->nranks : 1; mb.rank = c->rank; mb.peers = c->d_peers.p; mb.local = c->mbox.p; mb.seq = c->mbox_seq.p;
  accept_kernel<<<1, kAcceptThreads, 0, c->stream>>>(c->sys.p, c->lay, c->scal.p, c->dp.p, c->D.p, c->fixed.p, c->st.p, c->spd.p, c->records.p, c->max_records,
                                                    (!c->multi() || mailbox) ? 1 : 0, sa, fuse_commit ? 1 : 0, a, mb, term_args(c));
  HB_LAUNCH(c, "accept_kernel");
  if (!fuse_commit) {
    const int blocks = static_cast<int>(std::min<size_t>((mx + 255) / 256, static_cast<size_t>(c->num_sms) * 4));
    commit_kernel<<<blocks, 256, 0, c->stream>>>(c->st.p, a);
    HB_LAUNCH(c, "commit_kernel");
  }
  return 0;
}

// Sum of the packed partial systems over the ranks: ONE ncclAllReduce on the context's stream (capturable).
// err_st: the solver state whose comm_error a peer-memory timeout sets (the LM's c->st unless given).
int enqueue_reduce_system(hb200_ctx* c, SolverState* err_st = nullptr) {
  if (c->peer_reduce()) {
    // fused barrier + reduction over peer memory (peer_reduce_kernel); the next iteration assembles into the other half
    PeerReduceArgs a{};
    a.nranks = c->nranks; a.rank = c->rank; a.peers = c->d_peers.p; a.local = c->mbox.p;
    a.part_offset = kArenaParts + static_cast<long long>(c->peer_par) * c->arena_cap; a.total = c->lay.total;
    a.out = c->sys.p; a.round = c->red_round.p; a.arrive = c->red_arrive.p; a.st = err_st ? err_st : c->st.p;
    const long long pairs = c->lay.total / 2;
    const int grid = static_cast<int>(std::max<long long>(1, std::min<long long>(4LL * c->num_sms, (pairs + kReduceThreads - 1) / kReduceThreads)));
    peer_reduce_kernel<<<grid, kReduceThreads, 0, c->stream>>>(a);
    HB_LAUNCH(c, "peer_reduce_kernel");
    c->peer_par ^= 1;
    return 0;
  }
  if (c->nccl) {
    HB_NCCL(g_nccl.AllReduce(c->sys.p, c->sys.p, static_cast<size_t>(c->lay.total), /*ncclDouble*/ 8, /*ncclSum*/ 0, c->nccl, c->stream));
    c->nccl_calls += 1;
    prof_mark(c, "ncclAllReduce(system)");
  } else if (c->allreduce) {
    const int rc = c->allreduce(c->allreduce_user, c->sys.p, c->lay.total, c->stream);
    if (rc) return fail(200 + rc, "all-reduce callback failed (%d)", rc);
    prof_mark(c, "allreduce_callback(system)");
  }
  return 0;
}

// Trial-cost / model-decrease partials: fused into accept_kernel (one GPU: plain sums; NCCL + peer mapping: the
// mailbox exchange).  Fallbacks only: scalars_kernel + a 4-double reduction.
int enqueue_reduce_scalars(hb200_ctx* c) {
  if (!c->multi() || (c->nccl && c->peers_open)) return 0;
  int rc = enqueue_scalars(c);
  if (rc) return rc;
  if (c->nccl) {
    HB_NCCL(g_nccl.AllReduce(c->scal.p, c->scal.p, 8, 8, 0, c->nccl, c->stream));
    c->nccl_calls += 1;
    prof_mark(c, "ncclAllReduce(scalars)");
  } else {
    rc = c->allreduce(c->allreduce_user, c->scal.p, 8, c->stream);
    if (rc) return fail(200 + rc, "all-reduce callback failed (%d)", rc);
    prof_mark(c, "allreduce_callback(scalars)");
  }
  return 0;
}

// One LM iteration enqueued on the stream (graph-capturable unless the callback hook is in use).
int enqueue_iteration(hb200_ctx* c) {
  int rc = 0;
  if ((rc = enqueue_assembly(c, c->st.p))) return rc;
  if ((rc = enqueue_reduce_system(c))) return rc;
  bool retracted = false;
  if ((rc = enqueue_solve(c, /*fuse_retract=*/true, &retracted))) return rc;
  if (!retracted && (rc = enqueue_retract(c))) return rc;   // (also builds the trial knot table)
  if ((rc = enqueue_factors(c, false, 1))) return rc;   // the trial state's cost (its knot table is built)
  if ((rc = enqueue_reduce_scalars(c))) return rc;
  return enqueue_accept(c);
}

// The band layout depends on the longest landmark track of the LOCAL shard; the ranks agree on the maximum
// (one 4-byte ncclAllReduce(max) at bind / attach time, never on the iteration path).  The collective sliding-window
// calls agree on it again through agree_round.
int sync_layout(hb200_ctx* c) {
  if (!c->nccl || !c->bound) return 0;
  DevBuf<int> d;
  HB_CUDA(d.ensure(1));
  int v = c->beta;
  HB_CUDA(cudaMemcpyAsync(d.p, &v, sizeof(int), cudaMemcpyHostToDevice, c->stream));
  HB_NCCL(g_nccl.AllReduce(d.p, d.p, 1, /*ncclInt32*/ 2, /*ncclMax*/ 2, c->nccl, c->stream));
  HB_CUDA(cudaMemcpyAsync(&v, d.p, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  c->comm_warm = true;
  c->agreed_beta = v;
  if (v != c->beta) {
    const int rc = ensure_system(c);
    if (rc) return rc;
    c->kernel_args_changed();
  }
  return 0;
}

// ---- agreement of the collective sliding-window calls on a sharded context (hb200_window.cuh) ----
enum { kCallPixel = 1, kCallBearing = 2, kCallStereo = 3, kCallSlide = 4 };

VoteHeader vote_header(const hb200_ctx* c, int kind, int flags = 0, int ub = 0, int ubg = 0, int uba = 0) {
  return VoteHeader{{1.0, double(c->K()), double(c->Kbg()), double(c->Kba()), double(kind), double(flags), double(ub), double(ubg), double(uba)}};
}

// One agreement round: this rank's payload (window_vote_kernel), its sum over the ranks through the channel the context
// already has (NCCL -- peer-memory contexts have the communicator too -- or the callback hook), and the agreed values
// written to out[kAgreeOut] on the device (window_agree_kernel).  Enqueued on the context's stream: the caller's
// existing read-back brings the result home, so a round adds no host synchronisation.
int agree_round(hb200_ctx* c, const VoteHeader& h, const VoteSrc& src, int* out) {
  const int len = vote_payload_len(c->K(), c->Kbg(), c->Kba());
  if (static_cast<size_t>(len) > c->w_vote.cap) HB_CUDA(c->w_vote.ensure(2 * static_cast<size_t>(len)));   // (the window grows by a knot a frame)
  window_vote_kernel<<<1, 256, 0, c->stream>>>(c->w_vote.p, c->K(), c->Kbg(), c->Kba(), c->k(), h, src);
  HB_LAUNCH(c, "window_vote_kernel");
  if (c->nccl) {
    HB_NCCL(g_nccl.AllReduce(c->w_vote.p, c->w_vote.p, static_cast<size_t>(len), /*ncclDouble*/ 8, /*ncclSum*/ 0, c->nccl, c->stream));
    c->nccl_calls += 1;
    c->comm_warm = true;
    prof_mark(c, "ncclAllReduce(window)");
  } else {
    const int rc = c->allreduce(c->allreduce_user, c->w_vote.p, len, c->stream);
    if (rc) return fail(200 + rc, "all-reduce callback failed (%d)", rc);
    prof_mark(c, "allreduce_callback(window)");
  }
  window_agree_kernel<<<1, 256, 0, c->stream>>>(c->w_vote.p, c->K(), c->Kbg(), c->Kba(), h, out);
  HB_LAUNCH(c, "window_agree_kernel");
  return 0;
}

// A context that leaves (or changes) its communicator or hook: the band no longer follows the other ranks' tracks.
int forget_agreement(hb200_ctx* c) {
  if (!c->agreed_beta) return 0;
  c->agreed_beta = 0;
  if (!c->bound) return 0;
  HB_CUDA(cudaSetDevice(c->device));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  const int rc = ensure_system(c);
  if (rc) return rc;
  c->kernel_args_changed();
  return 0;
}

// What every rank returns after round A.  own: this rank's status code, its message already in the error string (0:
// its own checks passed); agreed: the read-back of agree_round's out (ignored on one context).  -2 when the ranks' calls
// differ, else the window-wide code: 0 lets the call go on, on every rank or on none.
int window_outcome(hb200_ctx* c, const int* agreed, int own) {
  if (!c->multi()) return own;
  if (agreed[kAgreeMismatch])
    return fail(-2, "sharded window calls out of step: the ranks made different calls or hold different knot / bias knot counts; no rank changed its window");
  const int code = agreed[kAgreeStatus];
  if (!code) return 0;
  if (own) return fail(code, "this rank failed its checks, so no rank changed its window: %s", std::string(g_error).c_str());
  return fail(code, "another rank failed its checks (code %d), so no rank changed its window", code);
}

int check_ready(hb200_ctx* c) {
  if (!c) return fail(-1, "null context");
  if (c->K() == 0) return fail(-2, "spline not set");
  if (!c->bound) return fail(-2, "factors not bound (call hb200_bind)");
  if (c->Ni && (!c->have_imu || !c->have_gravity || c->Kbg() == 0 || c->Kba() == 0)) return fail(-2, "inertial factors need IMU calibration, bias splines and gravity");
  if (c->Nv && (c->C == 0 || c->L == 0)) return fail(-2, "pixel / bearing factors need cameras and landmarks");
  if (c->Nm && c->P == 0) return fail(-2, "manifold factors need pose sensors");
  return 0;
}

int ensure_placeholders(hb200_ctx* c) {
  // Kernels take these pointers even when a factor family is absent.
  for (int s = 0; s < 2; ++s) {
    HB_CUDA(c->gyro.val[s].ensure(4)); HB_CUDA(c->accel.val[s].ensure(4)); HB_CUDA(c->grav[s].ensure(4)); HB_CUDA(c->lms[s].ensure(3));
    HB_CUDA(c->cp_pix[s].ensure(1)); HB_CUDA(c->cp_imu[s].ensure(1));
  }
  HB_CUDA(c->imu_tab.ensure(kImuStride)); HB_CUDA(c->cam_tab.ensure(kCamStride));
  HB_CUDA(c->v_out.w.ensure(1)); HB_CUDA(c->sensors.ensure(7));
  HB_CUDA(c->visual.grow(1, 0, c->stream)); HB_CUDA(c->inertial.grow(1, 0, c->stream)); HB_CUDA(c->manifold.grow(1, 0, c->stream));
  HB_CUDA(c->visual_spare.grow(1, 0, c->stream)); HB_CUDA(c->inertial_spare.grow(1, 0, c->stream)); HB_CUDA(c->manifold_spare.grow(1, 0, c->stream));
  return 0;
}

}  // namespace

extern "C" {

const char* hb200_last_error_string(void) { return g_error.c_str(); }

namespace {
int create_impl(const hb200_options* options, hb200_ctx* c) {
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) return fail(100 + static_cast<int>(e), "no CUDA device: %s (libhyperb200 has no CPU fallback)", cudaGetErrorString(e));
  c->device = options ? options->device : 0;
  if (c->device < 0 || c->device >= count) return fail(-1, "invalid device %d", c->device);
  HB_CUDA(cudaSetDevice(c->device));
  cudaDeviceProp prop{};
  HB_CUDA(cudaGetDeviceProperties(&prop, c->device));
  if (prop.major != 9 || prop.minor != 0) return fail(-5, "device sm_%d%d is not Hopper (built for sm_90a only)", prop.major, prop.minor);
  c->num_sms = prop.multiProcessorCount;
  c->use_graph = options ? options->use_graph != 0 : true;
  c->force_dense = options ? (options->reserved & 1) != 0 : false;
  if (options && options->stream) { c->stream = static_cast<cudaStream_t>(options->stream); c->own_stream = false; }
  else { HB_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking)); c->own_stream = true; }
  HB_CUDA(cudaStreamCreateWithFlags(&c->stream2, cudaStreamNonBlocking));
  HB_CUDA(cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming));
  HB_CUDA(cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming));
  HB_CUDA(cudaEventCreateWithFlags(&c->ev_mid, cudaEventDisableTiming));
  int rc = ensure_placeholders(c);
  if (rc) return rc;
  if (options && options->nccl_comm && (rc = hb200_set_nccl_comm(c, options->nccl_comm, options->nranks, options->rank))) return rc;
  HB_CUDA(cudaFuncSetAttribute(cholesky_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kCholSmem)));
  // the Jacobian pass of the large-window inertial kernel parks its forward-sweep state in dynamic shared memory (41.5 KB
  // at order 4, 69 KB at order 6: above the 48 KB default)
  rc = for_each_order_mode([&](auto K, auto DET) {
    if constexpr (!DET) {
      HB_CUDA(cudaFuncSetAttribute(inertial_eval_kernel<K, 4, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(inertial_stash_bytes(K))));
      HB_CUDA(cudaFuncSetAttribute(inertial_eval_kernel<K, 4, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(inertial_stash_bytes(K))));
    }
    return 0;
  });
  return rc ? rc : reset_solver_state(c);
}
}  // namespace

int hb200_create(const hb200_options* options, hb200_ctx** out) {
  if (!out) return fail(-1, "null output pointer");
  *out = nullptr;
  hb200_ctx* c = new hb200_ctx();
  const int rc = create_impl(options, c);
  if (rc) {
    const std::string keep = g_error;   // hb200_destroy must not clobber the message
    hb200_destroy(c);
    g_error = keep;
    return rc;
  }
  *out = c;
  return 0;
}

void hb200_destroy(hb200_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  if (c->stream2) cudaStreamSynchronize(c->stream2);
  for (size_t p = 0; p < c->peer_ptrs.size(); ++p)
    if (c->peer_ptrs[p] && c->peer_ptrs[p] != c->mbox.p) cudaIpcCloseMemHandle(c->peer_ptrs[p]);
  c->peer_ptrs.clear();
  // the captured iteration references the communicator: NCCL waits in ncclCommDestroy until such graphs are gone
  for (IterationGraph& g : c->graphs) g.release();
  if (c->nccl && c->own_nccl && g_nccl.CommDestroy) g_nccl.CommDestroy(c->nccl);
  c->nccl = nullptr;
  for (cudaEvent_t e : c->prof_events) cudaEventDestroy(e);
  if (c->h_stage) cudaFreeHost(c->h_stage);
  c->d_stage.release();
  if (c->ev_fork) cudaEventDestroy(c->ev_fork);
  if (c->ev_join) cudaEventDestroy(c->ev_join);
  if (c->ev_mid) cudaEventDestroy(c->ev_mid);
  if (c->stream2) cudaStreamDestroy(c->stream2);
  if (c->own_stream && c->stream) cudaStreamDestroy(c->stream);
  delete c;
}

int hb200_synchronize(hb200_ctx* c) {
  if (!c) return fail(-1, "null context");
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

void* hb200_stream(hb200_ctx* c) { return c ? c->stream : nullptr; }
long long hb200_launch_count(hb200_ctx* c) { return c ? c->launches : 0; }

int hb200_set_spline(hb200_ctx* c, int order, int K, const double* knots) {
  if (!c || !knots) return fail(-1, "null argument");
  if (order != 4 && order != 6) return fail(-4, "spline order %d not supported (4 or 6)", order);
  int rc = c->pose.check(order, K, knots, "knot");
  if (rc) return rc;
  HB_CUDA(cudaSetDevice(c->device));
  bool reshape = false;
  if ((rc = c->pose.set(order, K, knots, c->stream, &reshape))) return rc;
  for (DevBuf<double>& t : c->tab) HB_CUDA(t.ensure(static_cast<size_t>(K) * kTabStride));
  // the index maps of hb200_bind follow from the stamps: a window shifted by one knot keeps K but needs a re-bind
  if (reshape) { c->h_knot_const.assign(K, 0); c->bound = false; c->kernel_args_changed(); c->have_snapshot = false; if ((rc = update_fixed(c))) return rc; }
  c->outputs_changed();
  return 0;
}

int hb200_set_bias_splines(hb200_ctx* c, int order, int Kg, const double* gyro, int Ka, const double* accel) {
  if (!c || !gyro || !accel) return fail(-1, "null argument");
  if (order != 4) return fail(-4, "bias spline order %d not supported (4)", order);
  int rc = 0;
  if ((rc = c->gyro.check(order, Kg, gyro, "gyroscope bias knot")) || (rc = c->accel.check(order, Ka, accel, "accelerometer bias knot"))) return rc;
  HB_CUDA(cudaSetDevice(c->device));
  bool reshape[2] = {false, false};
  if ((rc = c->gyro.set(order, Kg, gyro, c->stream, &reshape[0])) || (rc = c->accel.set(order, Ka, accel, c->stream, &reshape[1]))) return rc;
  if (reshape[0] || reshape[1]) { c->bound = false; c->kernel_args_changed(); c->have_snapshot = false; if ((rc = update_fixed(c))) return rc; }
  c->outputs_changed();
  return 0;
}

int hb200_set_gravity(hb200_ctx* c, const double* g) {
  if (!c || !g) return fail(-1, "null argument");
  HB_CUDA(cudaSetDevice(c->device));
  HB_CUDA(cudaMemcpyAsync(c->grav[0].p, g, 3 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  c->have_gravity = true;
  c->outputs_changed();
  return 0;
}

int hb200_set_cameras(hb200_ctx* c, int C, const double* cams) {
  if (!c || !cams || C <= 0) return fail(-1, "invalid cameras");
  HB_CUDA(cudaSetDevice(c->device));
  if (C != c->C) { c->bound = false; c->kernel_args_changed(); }
  c->C = C;
  HB_CUDA(c->cams.ensure(15 * static_cast<size_t>(C)));
  HB_CUDA(c->cam_tab.ensure(kCamStride * static_cast<size_t>(C)));
  HB_CUDA(cudaMemcpyAsync(c->cams.p, cams, 15 * sizeof(double) * C, cudaMemcpyHostToDevice, c->stream));
  calib_kernel<<<(C + 63) / 64, 64, 0, c->stream>>>(C, c->cams.p, c->cam_tab.p, nullptr, nullptr, 0);
  HB_LAUNCH(c, "calib_kernel");
  HB_CUDA(cudaStreamSynchronize(c->stream));
  c->outputs_changed();
  return 0;
}

int hb200_set_imu(hb200_ctx* c, const double* imu) {
  if (!c || !imu) return fail(-1, "null argument");
  HB_CUDA(cudaSetDevice(c->device));
  HB_CUDA(c->imu.ensure(37));
  HB_CUDA(cudaMemcpyAsync(c->imu.p, imu, 37 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  calib_kernel<<<1, 64, 0, c->stream>>>(0, nullptr, nullptr, c->imu.p, c->imu_tab.p, c->quirks);
  HB_LAUNCH(c, "calib_kernel");
  HB_CUDA(cudaStreamSynchronize(c->stream));
  c->have_imu = true;
  c->outputs_changed();
  return 0;
}

int hb200_set_landmarks(hb200_ctx* c, int L, const double* xyz) {
  if (!c || (L > 0 && !xyz) || L < 0) return fail(-1, "invalid landmarks");
  HB_CUDA(cudaSetDevice(c->device));
  if (L != c->L) { c->bound = false; c->kernel_args_changed(); c->have_snapshot = false; }
  c->L = L;
  for (int s = 0; s < 2; ++s) HB_CUDA(c->lms[s].ensure(3 * static_cast<size_t>(std::max(L, 1))));
  if (L) HB_CUDA(cudaMemcpyAsync(c->lms[0].p, xyz, 3 * sizeof(double) * L, cudaMemcpyHostToDevice, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  c->outputs_changed();
  return 0;
}

int hb200_set_constant(hb200_ctx* c, const unsigned char* knot_constant, int gravity_constant, int bias_constant) {
  if (!c) return fail(-1, "null context");
  if (c->K() == 0) return fail(-2, "spline not set");
  HB_CUDA(cudaSetDevice(c->device));
  if (knot_constant) c->h_knot_const.assign(knot_constant, knot_constant + c->K());
  else c->h_knot_const.assign(c->K(), 0);
  c->gravity_const = gravity_constant; c->bias_const = bias_constant;
  c->system_changed();
  return update_fixed(c);
}

int hb200_set_reference_quirks(hb200_ctx* c, int quirks) {
  if (!c) return fail(-1, "null context");
  if (quirks < 0 || quirks > 15) return fail(-1, "quirks is a bit mask in [0, 15]");
  HB_CUDA(cudaSetDevice(c->device));
  c->quirks = quirks;
  if (c->have_imu) {   // rebuild the derived IMU table with the Jacobian-side matrices of this variant
    calib_kernel<<<1, 64, 0, c->stream>>>(0, nullptr, nullptr, c->imu.p, c->imu_tab.p, c->quirks);
    HB_LAUNCH(c, "calib_kernel");
    HB_CUDA(cudaStreamSynchronize(c->stream));
  }
  c->outputs_changed();
  return 0;
}

int hb200_set_options(hb200_ctx* c, double huber_pixel, double imu_loss_scale, double radius) {
  if (!c) return fail(-1, "null context");
  if (!(huber_pixel > 0) || !(imu_loss_scale > 0) || !(radius > 0)) return fail(-1, "options must be positive");
  HB_CUDA(cudaSetDevice(c->device));
  if (huber_pixel != c->huber || imu_loss_scale != c->imu_scale) c->iterations_changed();  // baked into kernel arguments
  c->huber = huber_pixel; c->imu_scale = imu_loss_scale; c->radius0 = radius;
  c->outputs_changed();
  return reset_solver_state(c);
}

namespace {
// The user index of every list position, when appends or slides cleared it: each family of the visual list in list
// order (pixel factors 0 .. Np-1, bearing factors Np .. Nv-1), the inertial list as it stands.
int ensure_perms(hb200_ctx* c) {
  const size_t Nv = c->Nv, Ni = c->Ni;
  if (c->v_perm.size() != Nv) {
    std::vector<int4> id(Nv);
    HB_CUDA(cudaSetDevice(c->device));
    HB_CUDA(cudaMemcpyAsync(id.data(), c->visual.idx.p, sizeof(int4) * Nv, cudaMemcpyDeviceToHost, c->stream));
    HB_CUDA(cudaStreamSynchronize(c->stream));
    c->v_perm.resize(Nv);
    for (size_t f = 0, p = 0, b = c->Np; f < Nv; ++f) c->v_perm[f] = static_cast<int>(id[f].w == 0 ? p++ : b++);
  }
  if (c->i_perm.size() != Ni) { c->i_perm.resize(Ni); std::iota(c->i_perm.begin(), c->i_perm.end(), 0); }
  return 0;
}

// Writes n visual factors of one kind to list positions [at, at + n): meas = pixel [n][2] (kind 0) or bearing [n][3]
// (kind 1: x, y in the pixel pair, z apart), and landmark, camera and kind into the index map, whose knot base
// bind_pixel_kernel fills in.
int upload_visual(hb200_ctx* c, int at, int n, const double* stamp, const int* camera, const int* landmark, const double* meas, int kind) {
  std::vector<double> xy(kind ? 2 * static_cast<size_t>(n) : 0), z(kind ? n : 0);
  for (int f = 0; f < static_cast<int>(z.size()); ++f) { xy[2 * f] = meas[3 * f]; xy[2 * f + 1] = meas[3 * f + 1]; z[f] = meas[3 * f + 2]; }
  std::vector<int4> id(n);
  for (int f = 0; f < n; ++f) id[f] = make_int4(0, landmark[f], camera[f], kind);
  HB_CUDA(cudaMemcpyAsync(c->visual.stamp.p + at, stamp, sizeof(double) * n, cudaMemcpyHostToDevice, c->stream));
  HB_CUDA(cudaMemcpyAsync(c->visual.pixel.p + at, kind ? xy.data() : meas, sizeof(double2) * n, cudaMemcpyHostToDevice, c->stream));
  if (kind) HB_CUDA(cudaMemcpyAsync(c->visual.z.p + at, z.data(), sizeof(double) * n, cudaMemcpyHostToDevice, c->stream));
  HB_CUDA(cudaMemcpyAsync(c->visual.idx.p + at, id.data(), sizeof(int4) * n, cudaMemcpyHostToDevice, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

// The compactions of the factor lists: the factors with keep[f] (nullptr: all n) move to positions pos[f] of the spare
// list, which then replaces the live one and holds `count` factors.  Knot bases drop by the shifts, landmarks go
// through lm_pos (nullptr: unchanged).  The switch moves the buffers the captured iteration points at.
int compact_visual(hb200_ctx* c, int n, const int* keep, const int* pos, const int* lm_pos, int knot_shift, int count) {
  HB_CUDA(c->visual_spare.grow(std::max(count, 1), 0, c->stream));
  compact_visual_kernel<<<(n + 255) / 256, 256, 0, c->stream>>>(n, keep, pos, lm_pos, knot_shift, c->visual.stamp.p, c->visual.pixel.p, c->visual.z.p, c->visual.idx.p,
                                                                c->visual_spare.stamp.p, c->visual_spare.pixel.p, c->visual_spare.z.p, c->visual_spare.idx.p);
  HB_LAUNCH(c, "compact_visual_kernel");
  c->visual.swap(c->visual_spare);
  c->kernel_args_changed();
  return 0;
}

int compact_inertial(hb200_ctx* c, int n, const int* keep, const int* pos, int knot_shift, int gyro_shift, int accel_shift, int count) {
  HB_CUDA(c->inertial_spare.grow(std::max(count, 1), 0, c->stream));
  compact_inertial_kernel<<<(n + 255) / 256, 256, 0, c->stream>>>(n, keep, pos, knot_shift, gyro_shift, accel_shift, c->inertial.stamp.p, c->inertial.meas.p, c->inertial.idx.p,
                                                                  c->inertial_spare.stamp.p, c->inertial_spare.meas.p, c->inertial_spare.idx.p);
  HB_LAUNCH(c, "compact_inertial_kernel");
  c->inertial.swap(c->inertial_spare);
  c->kernel_args_changed();
  return 0;
}

int compact_manifold(hb200_ctx* c, int n, const int* keep, const int* pos, int knot_shift, int count) {
  HB_CUDA(c->manifold_spare.grow(std::max(count, 1), 0, c->stream));
  compact_manifold_kernel<<<(n + 255) / 256, 256, 0, c->stream>>>(n, keep, pos, knot_shift, c->manifold.stamp.p, c->manifold.meas.p, c->manifold.sensor.p, c->manifold.idx.p,
                                                                  c->manifold_spare.stamp.p, c->manifold_spare.meas.p, c->manifold_spare.sensor.p, c->manifold_spare.idx.p);
  HB_LAUNCH(c, "compact_manifold_kernel");
  c->manifold.swap(c->manifold_spare);
  c->kernel_args_changed();
  return 0;
}

// Replaces the visual family of one kind (0 pixel, 1 bearing) by n factors in user order.  The list becomes [pixel
// family | bearing family], each in user order: the other family is moved there by one compaction.
int set_visual_family(hb200_ctx* c, int kind, int n, const double* stamp, const int* camera, const int* landmark, const double* meas) {
  HB_CUDA(cudaSetDevice(c->device));
  int rc = ensure_perms(c);
  if (rc) return rc;
  const int Nv = c->Nv, Np = kind ? c->Np : n, Nb = kind ? n : c->Nb;
  const int kept = kind ? Np : Nb, kept_at = kind ? 0 : n, kept_from = kind ? 0 : c->Np;   // the other family: count, new position, old user index
  if (!kept) HB_CUDA(c->visual.grow(n, 0, c->stream));
  if (kept) {
    std::vector<int> keep(Nv), pos(Nv);
    for (int f = 0; f < Nv; ++f) { const int u = c->v_perm[f]; keep[f] = (u < c->Np) == (kind == 1); pos[f] = kept_at + u - kept_from; }
    HB_CUDA(c->w_keep.ensure(Nv)); HB_CUDA(c->w_pos.ensure(Nv));
    HB_CUDA(cudaMemcpyAsync(c->w_keep.p, keep.data(), sizeof(int) * Nv, cudaMemcpyHostToDevice, c->stream));
    HB_CUDA(cudaMemcpyAsync(c->w_pos.p, pos.data(), sizeof(int) * Nv, cudaMemcpyHostToDevice, c->stream));
    if ((rc = compact_visual(c, Nv, c->w_keep.p, c->w_pos.p, nullptr, 0, Np + Nb))) return rc;
  }
  if (n && (rc = upload_visual(c, kind ? Np : 0, n, stamp, camera, landmark, meas, kind))) return rc;
  HB_CUDA(cudaStreamSynchronize(c->stream));
  c->Np = Np; c->Nb = Nb; c->Nv = Np + Nb;
  c->v_perm.resize(c->Nv); std::iota(c->v_perm.begin(), c->v_perm.end(), 0);
  c->bound = false; c->kernel_args_changed();
  return 0;
}
}  // namespace

int hb200_set_pixel_factors(hb200_ctx* c, int n, const double* stamp, const int* camera, const int* landmark, const double* pixel) {
  if (!c || n < 0 || (n > 0 && (!stamp || !camera || !landmark || !pixel))) return fail(-1, "invalid pixel factors");
  return set_visual_family(c, 0, n, stamp, camera, landmark, pixel);
}

int hb200_set_bearing_factors(hb200_ctx* c, int n, const double* stamp, const int* camera, const int* landmark, const double* bearing) {
  if (!c || n < 0 || (n > 0 && (!stamp || !camera || !landmark || !bearing))) return fail(-1, "invalid bearing factors");
  return set_visual_family(c, 1, n, stamp, camera, landmark, bearing);
}

int hb200_set_weights(hb200_ctx* c, int kind, const double* W) {
  if (!c) return fail(-1, "null context");
  if (kind < HB200_PIXEL || kind > HB200_MANIFOLD) return fail(-1, "unknown factor kind %d", kind);
  const int sides[4] = {2, 6, 1, 6}, offs[4] = {kWtPixel, kWtInertial, kWtBearing, kWtManifold};
  const int d = sides[kind], o = offs[kind];
  if (W) for (int i = 0; i < d * d; ++i) if (!std::isfinite(W[i])) return fail(-1, "weight matrix entry %d is not finite", i);
  std::array<double, kWtSize> next = c->h_wt;
  for (int i = 0; i < d * d; ++i) next[o + i] = W ? W[i] : (i % (d + 1) == 0 ? 1.0 : 0.0);
  const bool set = W != nullptr;
  if (set == c->wt_set[kind] && (!set || next == c->h_wt)) return 0;   // the current value: nothing changes
  HB_CUDA(cudaSetDevice(c->device));
  HB_CUDA(cudaStreamSynchronize(c->stream));   // no launch still reading the table
  HB_CUDA(c->wt.ensure(kWtSize));
  HB_CUDA(cudaMemcpy(c->wt.p, next.data(), sizeof(double) * kWtSize, cudaMemcpyHostToDevice));
  c->h_wt = next;
  c->wt_set[kind] = set;
  // the kernel instantiations (and the inertial J^T J kernel with its deterministic record regions) follow the flags
  c->kernel_args_changed();
  return 0;
}

int hb200_set_bearing_loss(hb200_ctx* c, double huber_bearing) {
  if (!c) return fail(-1, "null context");
  if (!(huber_bearing > 0)) return fail(-1, "options must be positive");
  if (huber_bearing != c->huber_bearing) c->iterations_changed();
  c->huber_bearing = huber_bearing;
  c->outputs_changed();
  return 0;
}

int hb200_set_pose_sensors(hb200_ctx* c, int n, const double* T_bs) {
  if (!c || n < 0 || (n > 0 && !T_bs)) return fail(-1, "invalid pose sensors");
  HB_CUDA(cudaSetDevice(c->device));
  if (n != c->P) c->bound = false;
  c->P = n;
  c->h_sensors.assign(T_bs, T_bs + 7 * static_cast<size_t>(n));
  HB_CUDA(c->sensors.ensure(7 * static_cast<size_t>(std::max(n, 1))));
  if (n) HB_CUDA(cudaMemcpyAsync(c->sensors.p, c->h_sensors.data(), sizeof(double) * 7 * n, cudaMemcpyHostToDevice, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  c->kernel_args_changed();
  return 0;
}

int hb200_set_manifold_factors(hb200_ctx* c, int n, const double* stamp, const int* sensor, const double* pose) {
  if (!c || n < 0 || (n > 0 && (!stamp || !sensor || !pose))) return fail(-1, "invalid manifold factors");
  HB_CUDA(cudaSetDevice(c->device));
  const size_t N = n;
  HB_CUDA(c->manifold.grow(N, 0, c->stream));
  if (N) {
    HB_CUDA(cudaMemcpyAsync(c->manifold.stamp.p, stamp, sizeof(double) * N, cudaMemcpyHostToDevice, c->stream));
    HB_CUDA(cudaMemcpyAsync(c->manifold.meas.p, pose, sizeof(double) * 7 * N, cudaMemcpyHostToDevice, c->stream));
    HB_CUDA(cudaMemcpyAsync(c->manifold.sensor.p, sensor, sizeof(int) * N, cudaMemcpyHostToDevice, c->stream));
  }
  HB_CUDA(cudaStreamSynchronize(c->stream));
  c->Nm = n;
  c->bound = false; c->kernel_args_changed();
  return 0;
}

int hb200_set_inertial_factors(hb200_ctx* c, int n, const double* stamp, const double* meas) {
  if (!c || n < 0 || (n > 0 && (!stamp || !meas))) return fail(-1, "invalid inertial factors");
  HB_CUDA(cudaSetDevice(c->device));
  const size_t N = n;
  HB_CUDA(c->inertial.grow(N, 0, c->stream));
  if (N) {
    HB_CUDA(cudaMemcpyAsync(c->inertial.stamp.p, stamp, sizeof(double) * N, cudaMemcpyHostToDevice, c->stream));
    HB_CUDA(cudaMemcpyAsync(c->inertial.meas.p, meas, sizeof(double) * 6 * N, cudaMemcpyHostToDevice, c->stream));
  }
  HB_CUDA(cudaStreamSynchronize(c->stream));
  c->Ni = n;
  c->i_perm.resize(N); std::iota(c->i_perm.begin(), c->i_perm.end(), 0);
  c->bound = false; c->kernel_args_changed();
  return 0;
}

}  // extern "C"

namespace {
// Everything the iteration runs on that follows from the bound factor lists on the device: the incidence lists
// (landmark CSR, inertial runs, longest track) by counting + scan kernels with one small read-back, then the output
// buffers and launch shapes of every factor family and the reduced system.  hb200_bind, hb200_append_* and
// hb200_slide all end here; the ones that change the lists on the device clear the user-index maps and drop the
// snapshot themselves.  kind > 0: a collective sliding-window call (kCall*), which on a sharded context ends with
// round B of the agreement -- the ranks' largest band half-width becomes agreed_beta.
int derive_window(hb200_ctx* c, int kind = 0) {
  const int Nv = c->Nv, Ni = c->Ni, Nm = c->Nm, L = c->L;
  // [L total, longest track rows, -, inertial runs, -, -, -, - | agreement (kAgreeOut)]
  HB_CUDA(c->w_scal.ensure(8 + kAgreeOut));
  HB_CUDA(cudaMemsetAsync(c->w_scal.p, 0, (8 + kAgreeOut) * sizeof(int), c->stream));
  HB_CUDA(c->lm_off.ensure(static_cast<size_t>(L) + 2)); HB_CUDA(c->lm_obs.ensure(std::max(Nv, 1)));
  HB_CUDA(c->run_off.ensure(static_cast<size_t>(Ni) + 2));
  HB_CUDA(c->w_cnt.ensure(static_cast<size_t>(std::max(L, 1)) + 1));
  HB_CUDA(c->w_keep.ensure(std::max(std::max(Nv, Ni), 1))); HB_CUDA(c->w_pos.ensure(std::max(std::max(Nv, Ni), 1)));
  // landmark CSR
  HB_CUDA(cudaMemsetAsync(c->w_cnt.p, 0, sizeof(int) * (static_cast<size_t>(L) + 1), c->stream));
  if (Nv) { count_kernel<<<(Nv + 255) / 256, 256, 0, c->stream>>>(Nv, c->visual.idx.p, c->w_cnt.p); HB_LAUNCH(c, "count_kernel"); }
  scan_kernel<<<1, 1024, 0, c->stream>>>(c->w_cnt.p, L + 1, c->lm_off.p, c->w_scal.p + 0);
  HB_LAUNCH(c, "scan_kernel");
  HB_CUDA(cudaMemsetAsync(c->w_cnt.p, 0, sizeof(int) * (static_cast<size_t>(L) + 1), c->stream));
  if (Nv) {
    csr_fill_kernel<<<(Nv + 255) / 256, 256, 0, c->stream>>>(Nv, c->visual.idx.p, c->lm_off.p, c->w_cnt.p, c->lm_obs.p);
    HB_LAUNCH(c, "csr_fill_kernel");
    csr_sort_kernel<<<(L + 127) / 128, 128, 0, c->stream>>>(L, c->lm_off.p, c->lm_obs.p, c->visual.idx.p, c->k(), c->w_scal.p + 1);
    HB_LAUNCH(c, "csr_sort_kernel");
  }
  // inertial runs
  if (Ni) {
    run_flag_kernel<<<(Ni + 255) / 256, 256, 0, c->stream>>>(Ni, c->inertial.idx.p, c->w_keep.p);
    HB_LAUNCH(c, "run_flag_kernel");
    scan_kernel<<<1, 1024, 0, c->stream>>>(c->w_keep.p, Ni, c->w_pos.p, c->w_scal.p + 3);
    HB_LAUNCH(c, "scan_kernel");
  }
  const bool agree = kind && c->multi();
  if (agree) {
    int rc = agree_round(c, vote_header(c, kind), VoteSrc{nullptr, {nullptr, nullptr, nullptr}, nullptr, c->w_scal.p + 1}, c->w_scal.p + 8);
    if (rc) return rc;
  }
  int h[8 + kAgreeOut];
  HB_CUDA(cudaMemcpyAsync(h, c->w_scal.p, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  if (agree) {
    if (h[8 + kAgreeMismatch]) return fail(-2, "sharded window calls out of step at the band agreement: the ranks made different calls or hold different knot / bias knot counts");
    c->agreed_beta = h[8 + kAgreeBeta];
  }
  c->max_rows = std::max(6 * c->k(), h[1]);
  c->schur_groups = false;   // the landmark groups are cut by hb200_bind, after this
  c->nruns = Ni ? h[3] : 0;
  if (Ni) { run_fill_kernel<<<(Ni + 255) / 256, 256, 0, c->stream>>>(Ni, c->w_keep.p, c->w_pos.p, c->nruns, c->run_off.p); HB_LAUNCH(c, "run_fill_kernel"); }
  else { const int z = 0; HB_CUDA(cudaMemcpyAsync(c->run_off.p, &z, sizeof(int), cudaMemcpyHostToDevice, c->stream)); }
  // sharded: the longest track over the ranks (6 (agreed beta + 1) rows), so that every rank refuses the window together
  const int rows = agree ? std::max(c->max_rows, 6 * (c->agreed_beta + 1)) : c->max_rows;
  if (2 * 3 * static_cast<size_t>(rows) * sizeof(double) > 200 * 1024) return fail(-6, "landmark track spans %d control-point dofs; exceeds the Schur kernel's shared-memory tile", rows);
  // outputs and launch shapes
  HB_CUDA(c->visual.grow(std::max(Nv, 1), Nv, c->stream));
  HB_CUDA(c->v_out.ensure(Nv, c->k())); HB_CUDA(c->i_out.ensure(Ni, c->k())); HB_CUDA(c->m_out.ensure(Nm, c->k()));
  c->n_pix_blocks = (Nv + kEvalThreads - 1) / kEvalThreads;
  c->n_imu_blocks = (Ni + kEvalThreads - 1) / kEvalThreads;
  c->n_man_blocks = (Nm + kEvalThreads - 1) / kEvalThreads;
  for (int s = 0; s < 2; ++s) { HB_CUDA(c->cp_pix[s].ensure(std::max(c->n_pix_blocks, 1))); HB_CUDA(c->cp_imu[s].ensure(std::max(c->n_imu_blocks + c->n_man_blocks, 1))); }
  if (c->max_rows * 6 * sizeof(double) > 48 * 1024) {
    const int smem = static_cast<int>(2 * 3 * static_cast<size_t>(c->max_rows) * sizeof(double));
    const int rs = for_each_order_mode([&](auto K, auto DET) {
      HB_CUDA(cudaFuncSetAttribute(schur_kernel<K, DET>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      return 0;
    });
    if (rs) return rs;
  }
  int rc = update_fixed(c);
  if (rc) return rc;
  if ((rc = ensure_system(c))) return rc;
  HB_CUDA(cudaStreamSynchronize(c->stream));
  c->bound = true;
  c->kernel_args_changed();
  return 0;
}

// Binds the visual factors at list positions [at, at + n) in place; factors that fail to bind are counted in d_invalid[0].
int bind_pixel_range(hb200_ctx* c, int at, int n) {
  bind_pixel_kernel<<<(n + 127) / 128, 128, 0, c->stream>>>(n, c->visual.stamp.p + at, c->pose.val[0].p, c->K(), c->k(), c->C, c->L, c->visual.idx.p + at, c->d_invalid.p);
  HB_LAUNCH(c, "bind_pixel_kernel");
  return 0;
}

// Binds the inertial factors at list positions [at, at + n) in place; factors that fail to bind are counted in d_invalid[0].
int bind_inertial_range(hb200_ctx* c, int at, int n) {
  bind_inertial_kernel<<<(n + 127) / 128, 128, 0, c->stream>>>(n, c->inertial.stamp.p + at, c->pose.val[0].p, c->K(), c->k(), c->gyro.val[0].p, c->Kbg(), c->accel.val[0].p, c->Kba(), c->gyro.order,
                                                             c->inertial.idx.p + at, c->d_invalid.p);
  HB_LAUNCH(c, "bind_inertial_kernel");
  return 0;
}

// Bound order of a list whose index maps id (host read-back) are not yet sorted by `less`: the stable sort's inverse
// permutation (old position -> new), with id and the user-index map perm permuted alongside.
template <typename Less>
std::vector<int> bound_order(std::vector<int4>& id, std::vector<int>& perm, Less less) {
  const size_t n = id.size();
  std::vector<int> s(n), inv(n), perm_s(n);
  std::vector<int4> id_s(n);
  std::iota(s.begin(), s.end(), 0);
  std::stable_sort(s.begin(), s.end(), [&](int a, int b) { return less(id[a], id[b]); });
  for (size_t p = 0; p < n; ++p) { inv[s[p]] = static_cast<int>(p); id_s[p] = id[s[p]]; perm_s[p] = perm[s[p]]; }
  id.swap(id_s); perm.swap(perm_s);
  return inv;
}
}  // namespace

extern "C" {

int hb200_bind(hb200_ctx* c, int* num_invalid) {
  if (!c) return fail(-1, "null context");
  if (c->K() == 0) return fail(-2, "spline not set");
  if (c->Ni && (c->Kbg() == 0 || c->Kba() == 0)) return fail(-2, "bias splines not set");
  if (c->Nv && (c->C == 0 || c->L == 0)) return fail(-2, "cameras / landmarks not set");
  if (c->Nm && c->P == 0) return fail(-2, "pose sensors not set");
  HB_CUDA(cudaSetDevice(c->device));
  int rc = ensure_perms(c);
  if (rc) return rc;
  const int Nv = c->Nv, Ni = c->Ni, Nm = c->Nm;
  HB_CUDA(c->d_invalid.ensure(1));
  HB_CUDA(cudaMemsetAsync(c->d_invalid.p, 0, sizeof(int), c->stream));
  // pass 1: index maps of the lists where they stand (a2/a4), one read-back of the invalid count and the keys
  if (Nv && (rc = bind_pixel_range(c, 0, Nv))) return rc;
  if (Ni && (rc = bind_inertial_range(c, 0, Ni))) return rc;
  if (Nm) {
    bind_manifold_kernel<<<(Nm + 127) / 128, 128, 0, c->stream>>>(Nm, c->manifold.stamp.p, c->manifold.sensor.p, c->pose.val[0].p, c->K(), c->k(), c->P, c->manifold.idx.p, c->d_invalid.p);
    HB_LAUNCH(c, "bind_manifold_kernel");
  }
  std::vector<int4> vi(Nv), ii(Ni);
  int invalid = 0;
  if (Nv) HB_CUDA(cudaMemcpyAsync(vi.data(), c->visual.idx.p, sizeof(int4) * Nv, cudaMemcpyDeviceToHost, c->stream));
  if (Ni) HB_CUDA(cudaMemcpyAsync(ii.data(), c->inertial.idx.p, sizeof(int4) * Ni, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaMemcpyAsync(&invalid, c->d_invalid.p, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  if (num_invalid) *num_invalid = invalid;
  if (invalid) return fail(2, "%d factor(s) reference a stamp outside the spline's valid range or an invalid camera / landmark / sensor", invalid);

  // pass 2: bound order = stable sort by knot base index (visual) / (base, gyro base, accel base) (inertial), applied on
  // the device by the compaction kernels with pos = the inverse permutation; the manifold list stays as it is
  auto by_base = [](const int4& a, const int4& b) { return a.x < b.x; };
  auto by_bases = [](const int4& a, const int4& b) { return a.x != b.x ? a.x < b.x : (a.y != b.y ? a.y < b.y : a.z < b.z); };
  std::vector<int> v_inv, i_inv;   // (host sources of the uploads below, alive until the synchronize)
  HB_CUDA(c->w_pos.ensure(std::max(std::max(Nv, Ni), 1)));
  if (!std::is_sorted(vi.begin(), vi.end(), by_base)) {
    v_inv = bound_order(vi, c->v_perm, by_base);
    HB_CUDA(cudaMemcpyAsync(c->w_pos.p, v_inv.data(), sizeof(int) * Nv, cudaMemcpyHostToDevice, c->stream));
    if ((rc = compact_visual(c, Nv, nullptr, c->w_pos.p, nullptr, 0, Nv))) return rc;
  }
  if (!std::is_sorted(ii.begin(), ii.end(), by_bases)) {
    i_inv = bound_order(ii, c->i_perm, by_bases);
    HB_CUDA(cudaMemcpyAsync(c->w_pos.p, i_inv.data(), sizeof(int) * Ni, cudaMemcpyHostToDevice, c->stream));
    if ((rc = compact_inertial(c, Ni, nullptr, c->w_pos.p, 0, 0, 0, Ni))) return rc;
  }
  HB_CUDA(cudaStreamSynchronize(c->stream));
  // a new window: the band starts from this rank's own tracks and the caller's floor; with a communicator attached the
  // ranks agree on the widest one here (collective), through the callback hook the host sets the floor
  c->agreed_beta = 0;
  if ((rc = derive_window(c))) return rc;
  if ((rc = sync_layout(c))) return rc;
  {
    // landmark groups for the large-window Schur kernel: observed landmarks ordered by their first knot base, cut so that
    // a group has at most kSchurGroup members and its control-point rows fit one window of RT rows
    constexpr int kSchurGroupMin = 8192;   // landmarks from which schur_group_kernel replaces schur_kernel
    c->schur_rt = ((c->max_rows + 12 + 7) / 8) * 8;
    if (c->L >= kSchurGroupMin && Nv) {
      // first / last knot base of every observed landmark (-1: unobserved); bound order is ascending knot base
      std::vector<int> first(c->L, -1), last(c->L, -1);
      for (const int4& id : vi) { if (first[id.y] < 0) first[id.y] = id.x; last[id.y] = id.x; }
      std::vector<int> order;
      order.reserve(c->L);
      for (int l = 0; l < c->L; ++l) if (first[l] >= 0) order.push_back(l);
      std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return first[a] < first[b]; });
      std::vector<int> goff;
      const int win = c->schur_rt / 6;   // control points per window
      int glo = 0;
      for (size_t i = 0; i < order.size(); ++i) {
        const int l = order[i];
        const int lo = first[l], hi = last[l] + c->k();
        if (goff.empty() || static_cast<int>(i) - goff.back() >= kSchurGroup || hi - glo > win) { goff.push_back(static_cast<int>(i)); glo = lo; }
      }
      c->n_lm_groups = static_cast<int>(goff.size());
      goff.push_back(static_cast<int>(order.size()));
      HB_CUDA(c->lm_order.ensure(std::max<size_t>(order.size(), 1))); HB_CUDA(c->lm_group_off.ensure(goff.size()));
      HB_CUDA(cudaMemcpyAsync(c->lm_order.p, order.data(), sizeof(int) * order.size(), cudaMemcpyHostToDevice, c->stream));
      HB_CUDA(cudaMemcpyAsync(c->lm_group_off.p, goff.data(), sizeof(int) * goff.size(), cudaMemcpyHostToDevice, c->stream));
      c->schur_groups = c->n_lm_groups > 0;
      const size_t smem = (3 * static_cast<size_t>(kSchurGroup) * (c->schur_rt + 1) + 3 * kSchurGroup + 4 * 3 * static_cast<size_t>(c->schur_rt)) * sizeof(double);
      if (smem > 200 * 1024) c->schur_groups = false;
      else {
        rc = for_each_order_mode([&](auto K, auto DET) {
          HB_CUDA(cudaFuncSetAttribute(schur_group_kernel<K, DET>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
          return 0;
        });
        if (rc) return rc;
      }
    }
  }
  if (c->schur_groups) {   // unobserved landmarks are not in any group: their blocks stay zero (no step)
    HB_CUDA(cudaMemsetAsync(c->Vchol.p, 0, sizeof(double) * 9 * static_cast<size_t>(std::max(c->L, 1)), c->stream));
    HB_CUDA(cudaMemsetAsync(c->gl.p, 0, sizeof(double) * 3 * static_cast<size_t>(std::max(c->L, 1)), c->stream));
    HB_CUDA(cudaMemsetAsync(c->Dl.p, 0, sizeof(double) * 3 * static_cast<size_t>(std::max(c->L, 1)), c->stream));
  }
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

int hb200_get_index_maps(hb200_ctx* c, int* pixel_base, int* inertial_base, int* gyro_bias_base, int* accel_bias_base) {
  if (!c || !c->bound) return fail(-2, "not bound");
  int rc = ensure_perms(c);
  if (rc) return rc;
  const int Nv = pixel_base ? c->Nv : 0, Ni = (inertial_base || gyro_bias_base || accel_bias_base) ? c->Ni : 0;
  std::vector<int4> vi(Nv), ii(Ni);
  if (Nv) HB_CUDA(cudaMemcpyAsync(vi.data(), c->visual.idx.p, sizeof(int4) * Nv, cudaMemcpyDeviceToHost, c->stream));
  if (Ni) HB_CUDA(cudaMemcpyAsync(ii.data(), c->inertial.idx.p, sizeof(int4) * Ni, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  for (int p = 0; p < Nv; ++p) if (c->v_perm[p] < c->Np) pixel_base[c->v_perm[p]] = vi[p].x;
  for (int p = 0; p < Ni; ++p) {
    const int u = c->i_perm[p];
    if (inertial_base) inertial_base[u] = ii[p].x;
    if (gyro_bias_base) gyro_bias_base[u] = ii[p].y;
    if (accel_bias_base) accel_bias_base[u] = ii[p].z;
  }
  return 0;
}

int hb200_evaluate(hb200_ctx* c, int flags) {
  int rc = check_ready(c);
  if (rc) return rc;
  HB_CUDA(cudaSetDevice(c->device));
  const bool J = flags & HB200_EVAL_JACOBIANS;
  const int sel = (flags & HB200_EVAL_TRIAL) ? 1 : 0;
  rc = enqueue_evaluate(c, J, sel);
  if (rc) return rc;
  c->outputs_changed();
  c->evaluated_J = J && sel == 0;   // a trial-state sweep overwrites the residual / Jacobian buffers
  return 0;
}

namespace {
// Where read_visual_outputs writes one visual kind's outputs in user order (null: not wanted).
struct VisualDest { double *r, *Jp, *Jl; };
// The outputs of the pixel factors (dst[0]) and the bearing factors (dst[1]) from one read-back of the visual list.  A
// bearing factor fills the first row of its 2-row slot.
int read_visual_outputs(hb200_ctx* c, const VisualDest (&dst)[2]) {
  if (!c || !c->bound) return fail(-2, "not bound");
  { const int rs = ensure_perms(c); if (rs) return rs; }
  HB_CUDA(cudaSetDevice(c->device));
  const size_t N = c->Nv, w = 6 * static_cast<size_t>(c->k());   // w: one row of a state Jacobian
  if (N == 0) return 0;
  const bool Jp = dst[0].Jp || dst[1].Jp, Jl = dst[0].Jl || dst[1].Jl;
  std::vector<double> tr(2 * N), tJ(Jp ? 2 * w * N : 0), tl(Jl ? 6 * N : 0);
  HB_CUDA(cudaMemcpyAsync(tr.data(), c->v_out.r.p, sizeof(double) * 2 * N, cudaMemcpyDeviceToHost, c->stream));
  if (Jp) HB_CUDA(cudaMemcpyAsync(tJ.data(), c->v_out.Jp.p, sizeof(double) * 2 * w * N, cudaMemcpyDeviceToHost, c->stream));
  if (Jl) HB_CUDA(cudaMemcpyAsync(tl.data(), c->v_out.Jl.p, sizeof(double) * 6 * N, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  for (size_t p = 0; p < N; ++p) {
    const int b = c->v_perm[p] >= c->Np ? 1 : 0;   // pixel factors 0 .. Np-1, bearing factors after
    const size_t u = c->v_perm[p] - b * c->Np, rows = 2 - b;
    const VisualDest& d = dst[b];
    if (d.r) std::memcpy(d.r + rows * u, tr.data() + 2 * p, sizeof(double) * rows);
    if (d.Jp) std::memcpy(d.Jp + rows * w * u, tJ.data() + 2 * w * p, sizeof(double) * rows * w);
    if (d.Jl) std::memcpy(d.Jl + 3 * rows * u, tl.data() + 6 * p, sizeof(double) * 3 * rows);
  }
  return 0;
}
}  // namespace

int hb200_get_pixel_outputs(hb200_ctx* c, double* r, double* Jp, double* Jl) { return read_visual_outputs(c, {{r, Jp, Jl}, {}}); }

int hb200_get_bearing_outputs(hb200_ctx* c, double* r, double* Jp, double* Jl) { return read_visual_outputs(c, {{}, {r, Jp, Jl}}); }

int hb200_get_manifold_outputs(hb200_ctx* c, double* r, double* Jp) {
  if (!c || !c->bound) return fail(-2, "not bound");
  HB_CUDA(cudaSetDevice(c->device));
  const size_t N = c->Nm, w = 36 * static_cast<size_t>(c->k());
  if (N == 0) return 0;
  if (r) HB_CUDA(cudaMemcpyAsync(r, c->m_out.r.p, sizeof(double) * 6 * N, cudaMemcpyDeviceToHost, c->stream));
  if (Jp) HB_CUDA(cudaMemcpyAsync(Jp, c->m_out.Jp.p, sizeof(double) * w * N, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

int hb200_get_inertial_outputs(hb200_ctx* c, double* r, double* Jp, double* wg, double* wa, double* Jg) {
  if (!c || !c->bound) return fail(-2, "not bound");
  { const int rs = ensure_perms(c); if (rs) return rs; }
  HB_CUDA(cudaSetDevice(c->device));
  const size_t N = c->Ni, w = 36 * static_cast<size_t>(c->k());
  if (N == 0) return 0;
  std::vector<double> tr(6 * N), tJ(Jp ? w * N : 0), tg(wg ? 4 * N : 0), ta(wa ? 4 * N : 0), tG(Jg ? 12 * N : 0);
  HB_CUDA(cudaMemcpyAsync(tr.data(), c->i_out.r.p, sizeof(double) * 6 * N, cudaMemcpyDeviceToHost, c->stream));
  if (Jp) HB_CUDA(cudaMemcpyAsync(tJ.data(), c->i_out.Jp.p, sizeof(double) * w * N, cudaMemcpyDeviceToHost, c->stream));
  if (wg) HB_CUDA(cudaMemcpyAsync(tg.data(), c->i_out.wg.p, sizeof(double) * 4 * N, cudaMemcpyDeviceToHost, c->stream));
  if (wa) HB_CUDA(cudaMemcpyAsync(ta.data(), c->i_out.wa.p, sizeof(double) * 4 * N, cudaMemcpyDeviceToHost, c->stream));
  if (Jg) HB_CUDA(cudaMemcpyAsync(tG.data(), c->i_out.Jg.p, sizeof(double) * 12 * N, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  for (size_t p = 0; p < N; ++p) {
    const size_t u = c->i_perm[p];
    if (r) std::memcpy(r + 6 * u, tr.data() + 6 * p, sizeof(double) * 6);
    if (Jp) std::memcpy(Jp + w * u, tJ.data() + w * p, sizeof(double) * w);
    if (wg) std::memcpy(wg + 4 * u, tg.data() + 4 * p, sizeof(double) * 4);
    if (wa) std::memcpy(wa + 4 * u, ta.data() + 4 * p, sizeof(double) * 4);
    if (Jg) std::memcpy(Jg + 12 * u, tG.data() + 12 * p, sizeof(double) * 12);
  }
  return 0;
}

}  // extern "C"

namespace {
// rows of a tangent-space SE3 Jacobian [d/dtheta | d/drho] -> ambient [q(4) | p(3)] through the SE3JacobianAdapter
// (reference pixel.cpp:141, inertial.cpp:161): J_theta A_q(q) | J_rho, in output rows of ld_out >= 7 doubles (zero after
// the seventh)
void tangent_to_ambient_se3(const double* Jt, int ld, int rows, const double* T, double* out, int ld_out = 7) {
  const double* q = T;
  const double Aq[12] = {2 * q[3], -2 * q[2], 2 * q[1], -2 * q[0], 2 * q[2], 2 * q[3], -2 * q[0], -2 * q[1], -2 * q[1], 2 * q[0], 2 * q[3], -2 * q[2]};
  for (int row = 0; row < rows; ++row) {
    const double* jt = Jt + static_cast<size_t>(ld) * row;
    double* o = out + static_cast<size_t>(ld_out) * row;
    for (int col = 0; col < 4; ++col) o[col] = jt[0] * Aq[col] + jt[1] * Aq[4 + col] + jt[2] * Aq[8 + col];
    o[4] = jt[3]; o[5] = jt[4]; o[6] = jt[5];
    std::fill(o + 7, o + ld_out, 0.0);
  }
}

// calibration-block Jacobians of every factor at the current state, mirrored to the host in user order
int ensure_calib_mirror(hb200_ctx* c) {
  HB_CUDA(cudaSetDevice(c->device));
  const size_t Nv = c->Nv, Ni = c->Ni, Nm = c->Nm;
  DevBuf<double> dv, di, dm;
  std::vector<double> tv(28 * Nv), ti(216 * Ni);
  std::vector<double>* Jc = c->mirror.Jc;   // user order: [Np], [Nb] ([2][14] each), [Ni][6][36], [Nm][6][6]
  Jc[HB200_PIXEL].assign(28 * static_cast<size_t>(c->Np), 0.0); Jc[HB200_BEARING].assign(28 * static_cast<size_t>(c->Nb), 0.0);
  Jc[HB200_INERTIAL].assign(216 * Ni, 0.0); Jc[HB200_MANIFOLD].assign(36 * Nm, 0.0);
  if (Nv) {
    HB_CUDA(dv.ensure(28 * Nv));
    const int blocks = static_cast<int>((Nv + kEvalThreads - 1) / kEvalThreads);
    const int rc = with_order(c->k(), [&](auto K) {
      return with_flag(c->wt_visual(), [&](auto WT) {
        pixel_calib_kernel<K, WT><<<blocks, kEvalThreads, 0, c->stream>>>(c->Nv, c->visual.stamp.p, c->visual.pixel.p, c->visual.z.p, c->visual.idx.p, c->tab[0].p,
                                                                          c->cam_tab.p, c->lms[0].p, c->pose.basis, dv.p, c->wt.p);
        return check_launch(c, "pixel_calib_kernel");
      });
    });
    if (rc) return rc;
    HB_CUDA(cudaMemcpyAsync(tv.data(), dv.p, sizeof(double) * 28 * Nv, cudaMemcpyDeviceToHost, c->stream));
  }
  if (Ni) {
    HB_CUDA(di.ensure(216 * Ni));
    const int blocks = static_cast<int>((Ni + kEvalThreads - 1) / kEvalThreads);
    const int rc = with_order(c->k(), [&](auto K) {
      return with_flag(c->wt_set[HB200_INERTIAL], [&](auto WT) {
        inertial_calib_kernel<K, WT><<<blocks, kEvalThreads, 0, c->stream>>>(c->Ni, c->inertial.stamp.p, c->inertial.idx.p, c->tab[0].p, c->imu.p, c->grav[0].p, c->pose.basis, c->quirks, di.p,
                                                                             c->wt.p);
        return check_launch(c, "inertial_calib_kernel");
      });
    });
    if (rc) return rc;
    HB_CUDA(cudaMemcpyAsync(ti.data(), di.p, sizeof(double) * 216 * Ni, cudaMemcpyDeviceToHost, c->stream));
  }
  if (Nm) {
    HB_CUDA(dm.ensure(36 * Nm));
    const int blocks = static_cast<int>((Nm + kEvalThreads - 1) / kEvalThreads);
    const int rc = with_order(c->k(), [&](auto K) {
      return with_flag(c->wt_set[HB200_MANIFOLD], [&](auto WT) {
        manifold_calib_kernel<K, WT><<<blocks, kEvalThreads, 0, c->stream>>>(c->Nm, c->manifold.stamp.p, c->manifold.meas.p, c->manifold.idx.p, c->tab[0].p, c->sensors.p, c->pose.basis, dm.p, c->wt.p);
        return check_launch(c, "manifold_calib_kernel");
      });
    });
    if (rc) return rc;
    HB_CUDA(cudaMemcpyAsync(Jc[HB200_MANIFOLD].data(), dm.p, sizeof(double) * 36 * Nm, cudaMemcpyDeviceToHost, c->stream));
  }
  HB_CUDA(cudaStreamSynchronize(c->stream));
  for (size_t p = 0; p < Nv; ++p)   // pixel factors 0 .. Np-1, bearing factors after
    std::memcpy(c->v_perm[p] < c->Np ? &Jc[HB200_PIXEL][28 * c->v_perm[p]] : &Jc[HB200_BEARING][28 * (c->v_perm[p] - c->Np)], &tv[28 * p], 28 * sizeof(double));
  for (size_t p = 0; p < Ni; ++p) std::memcpy(&Jc[HB200_INERTIAL][216 * static_cast<size_t>(c->i_perm[p])], &ti[216 * p], 216 * sizeof(double));
  c->mirror.calib_valid = true;
  return 0;
}
}  // namespace

extern "C" {

int hb200_factor_evaluate(hb200_ctx* c, int kind, int index, const double* const* parameters, double* residuals, double** jacobians) {
  if (!c || !c->bound) return fail(-2, "not bound");
  if (!c->evaluated_J) return fail(-2, "call hb200_evaluate(HB200_EVAL_JACOBIANS) first");
  if (!parameters || !residuals) return fail(-1, "null argument");
  { const int rs = ensure_perms(c); if (rs) return rs; }
  OutputMirror& mir = c->mirror;
  const int nrs[4] = {2, 6, 1, 6};
  const int Ns[4] = {c->Np, c->Ni, c->Nb, c->Nm};
  if (!mir.valid) {
    const size_t k = c->k(), Ni = c->Ni;
    for (int f = HB200_PIXEL; f <= HB200_MANIFOLD; ++f) {
      mir.r[f].resize(static_cast<size_t>(nrs[f]) * Ns[f]);
      mir.Jp[f].resize(6 * k * nrs[f] * Ns[f]);
    }
    for (int f : {HB200_PIXEL, HB200_BEARING}) mir.Jl[f].resize(3 * static_cast<size_t>(nrs[f]) * Ns[f]);
    mir.wg.resize(4 * Ni); mir.wa.resize(4 * Ni); mir.Jg.resize(12 * Ni);
    auto visual = [&](int f) { return VisualDest{mir.r[f].data(), mir.Jp[f].data(), mir.Jl[f].data()}; };
    int rc = read_visual_outputs(c, {visual(HB200_PIXEL), visual(HB200_BEARING)});
    if (!rc) rc = hb200_get_inertial_outputs(c, mir.r[HB200_INERTIAL].data(), mir.Jp[HB200_INERTIAL].data(), mir.wg.data(), mir.wa.data(), mir.Jg.data());
    if (!rc) rc = hb200_get_manifold_outputs(c, mir.r[HB200_MANIFOLD].data(), mir.Jp[HB200_MANIFOLD].data());
    if (rc) return rc;
    mir.valid = true;
  }
  const int k = c->k(), kb = c->gyro.order;
  if (kind < HB200_PIXEL || kind > HB200_MANIFOLD) return fail(-1, "unknown factor kind %d", kind);
  if (jacobians && !mir.calib_valid) {
    // calibration blocks requested?  (constant in the live configuration, so they are produced on demand only)
    const int first = k, count = (kind == HB200_INERTIAL) ? 5 : (kind == HB200_MANIFOLD ? 1 : 3);
    bool want = false;
    for (int b = 0; b < count; ++b) want = want || jacobians[first + b] != nullptr;
    if (want) { const int rc = ensure_calib_mirror(c); if (rc) return rc; }
  }
  const int nr = nrs[kind], N = Ns[kind];
  if (index < 0 || index >= N) return fail(-1, "factor index %d out of range", index);
  const double* r = mir.r[kind].data() + static_cast<size_t>(nr) * index;
  for (int i = 0; i < nr; ++i) residuals[i] = r[i];
  if (!jacobians) return 0;
  const double* Jp = mir.Jp[kind].data() + static_cast<size_t>(nr) * 6 * k * index;
  // state blocks: [J_theta * A_q(q_m) | J_rho | 0]  (ambient 8, row-major nr x 8)
  for (int m = 0; m < k; ++m)
    if (jacobians[m]) tangent_to_ambient_se3(Jp + 6 * m, 6 * k, nr, parameters[m], jacobians[m], 8);
  if (kind == HB200_PIXEL || kind == HB200_BEARING) {
    const int sizes[4] = {7, 4, 4, 3};
    const double* Jl = mir.Jl[kind].data() + 3 * static_cast<size_t>(nr) * index;
    // calibration blocks (reference pixel.cpp:91-135,141; bearing.cpp:76): rows of [T_bs tangent 6 | intrinsics 4 | distortion 4]
    const double* Jc = mir.Jc[kind].data() + 28 * static_cast<size_t>(index);
    const int coff[3] = {0, 6, 10};
    for (int b = 0; b < 4; ++b) {
      double* o = jacobians[k + b];
      if (!o) continue;
      if (b == 0) tangent_to_ambient_se3(Jc, 14, nr, parameters[k], o);
      else if (b < 3) { for (int row = 0; row < nr; ++row) for (int col = 0; col < sizes[b]; ++col) o[sizes[b] * row + col] = Jc[14 * row + coff[b] + col]; }
      else std::memcpy(o, Jl, 3 * nr * sizeof(double));
    }
  } else if (kind == HB200_MANIFOLD) {
    if (jacobians[k]) tangent_to_ambient_se3(mir.Jc[kind].data() + 36 * static_cast<size_t>(index), 6, 6, parameters[k], jacobians[k]);   // reference manifold.cpp:57
  } else {
    // reference inertial.cpp:155-194: rows of [T_bs tangent 6 | i_g 6 | i_a 6 | S_g 9 | X_a 9]
    const int sizes[5] = {7, 6, 6, 9, 9};
    const int coff[5] = {0, 6, 12, 18, 27};
    const double* Jc = mir.Jc[kind].data() + 216 * static_cast<size_t>(index);
    for (int b = 0; b < 5; ++b) {
      double* o = jacobians[k + b];
      if (!o) continue;
      if (b == 0) tangent_to_ambient_se3(Jc, 36, 6, parameters[k], o);
      else for (int row = 0; row < 6; ++row) for (int col = 0; col < sizes[b]; ++col) o[sizes[b] * row + col] = Jc[36 * row + coff[b] + col];
    }
    // bias knot m: w_g[m] [I3 ; 0] / w_a[m] [0 ; I3], times the inertial weight matrix when one is set
    const double* W = &c->h_wt[kWtInertial];
    for (int m = 0; m < kb; ++m) {
      if (double* o = jacobians[k + 5 + m]) {
        std::fill(o, o + 24, 0.0);
        const double wv = mir.wg[4 * static_cast<size_t>(index) + m];
        if (c->wt_set[HB200_INERTIAL]) { for (int row = 0; row < 6; ++row) for (int a = 0; a < 3; ++a) o[4 * row + a] = wv * W[6 * row + a]; }
        else for (int a = 0; a < 3; ++a) o[4 * a + a] = wv;
      }
      if (double* o = jacobians[k + 5 + kb + m]) {
        std::fill(o, o + 24, 0.0);
        const double wv = mir.wa[4 * static_cast<size_t>(index) + m];
        if (c->wt_set[HB200_INERTIAL]) { for (int row = 0; row < 6; ++row) for (int a = 0; a < 3; ++a) o[4 * row + a] = wv * W[6 * row + 3 + a]; }
        else for (int a = 0; a < 3; ++a) o[4 * (3 + a) + a] = wv;
      }
    }
    if (double* o = jacobians[k + 5 + 2 * kb]) {
      // minimal-norm ambient Jacobian: J_tangent * PlusJacobian^T / |g|^2  (PlusJacobian^T PlusJacobian = |g|^2 I)
      const double* x = parameters[k + 5 + 2 * kb];
      const double sigma = x[0] * x[0] + x[1] * x[1];
      double v[3] = {x[0], x[1], 1.0}, beta = 0.0;
      if (sigma <= 2.220446049250313e-16) { if (x[2] < 0.0) beta = 2.0; }
      else {
        const double mu = std::sqrt(x[2] * x[2] + sigma);
        const double vp = (x[2] <= 0.0) ? (x[2] - mu) : (-sigma / (x[2] + mu));
        beta = 2.0 * vp * vp / (sigma + vp * vp);
        v[0] /= vp; v[1] /= vp;
      }
      const double nx = std::sqrt(sigma + x[2] * x[2]);
      double PJ[6];
      for (int cc = 0; cc < 2; ++cc) for (int rr = 0; rr < 3; ++rr) PJ[2 * rr + cc] = nx * ((rr == cc ? 1.0 : 0.0) - beta * v[cc] * v[rr]);
      const double* Jg = &mir.Jg[12 * static_cast<size_t>(index)];
      for (int row = 0; row < 6; ++row)
        for (int col = 0; col < 3; ++col) o[3 * row + col] = (Jg[2 * row] * PJ[2 * col] + Jg[2 * row + 1] * PJ[2 * col + 1]) / (nx * nx);
    }
  }
  return 0;
}

int hb200_reduced_size(hb200_ctx* c) { return c ? 6 * c->K() + 3 * c->Kbg() + 3 * c->Kba() + 2 : -1; }

int hb200_build_system(hb200_ctx* c) {
  int rc = check_ready(c);
  if (rc) return rc;
  if (!c->evaluated_J) return fail(-2, "call hb200_evaluate(HB200_EVAL_JACOBIANS) first");
  HB_CUDA(cudaSetDevice(c->device));
  if ((rc = prepare_det(c))) return rc;
  if ((rc = enqueue_assembly(c, c->st.p))) return rc;   // as enqueue_iteration assembles
  if ((rc = enqueue_reduce_system(c))) return rc;
  c->system_built = true;
  return 0;
}

int hb200_get_system(hb200_ctx* c, double* S, double* b) {
  if (!c || !c->system_built) return fail(-2, "system not built");
  HB_CUDA(cudaSetDevice(c->device));
  const size_t n = c->n;
  { const int rc = enqueue_densify(c); if (rc) return rc; }   // dense, damped, masked -- what the solvers factor
  if (S) HB_CUDA(cudaMemcpyAsync(S, c->Lw.p, sizeof(double) * n * n, cudaMemcpyDeviceToHost, c->stream));
  if (b) HB_CUDA(cudaMemcpyAsync(b, c->Lw.p + static_cast<size_t>((n + 31) / 32) * 32 * n, sizeof(double) * n, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

int hb200_solve(hb200_ctx* c) {
  if (!c || !c->system_built) return fail(-2, "system not built");
  HB_CUDA(cudaSetDevice(c->device));
  return enqueue_solve(c);
}

int hb200_get_delta(hb200_ctx* c, double* dp, double* dl) {
  if (!c || !c->bound) return fail(-2, "not bound");
  HB_CUDA(cudaSetDevice(c->device));
  if (dp) HB_CUDA(cudaMemcpyAsync(dp, c->dp.p, sizeof(double) * c->n, cudaMemcpyDeviceToHost, c->stream));
  if (dl && c->L) HB_CUDA(cudaMemcpyAsync(dl, c->dl.p, sizeof(double) * 3 * c->L, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

}  // extern "C"

// ---- marginal covariances (hb200_cov.cuh) ------------------------------------------------------------------------
namespace {
void cov_info(hb200_ctx* c, hb200_covariance_info* info) {
  const CovPoint& pt = c->cov_pt[c->cov_slot_committed];
  info->degenerate_landmarks = c->cov_degenerate; info->unobserved_landmarks = c->cov_unobserved;
  info->K = c->cov_valid ? pt.lay.K : 0; info->beta = c->cov_valid ? pt.lay.beta : 0;
  info->m = c->cov_valid ? pt.lay.m : 0; info->L = c->cov_valid ? pt.L : 0;
}

// the current state as the linearisation point of a build
int freeze_point(hb200_ctx* c, CovPoint& pt) {
  pt.lay = c->lay; pt.L = c->L; pt.Nv = c->Nv; pt.max_rows = c->max_rows;
  int rc = 0;
  if ((rc = pt.pose.freeze(c->pose, c->stream)) || (rc = pt.gyro.freeze(c->gyro, c->stream)) || (rc = pt.accel.freeze(c->accel, c->stream))) return rc;
  HB_CUDA(pt.tab.ensure(static_cast<size_t>(kTabStride) * c->K()));
  HB_CUDA(cudaMemcpyAsync(pt.tab.p, c->tab[0].p, sizeof(double) * kTabStride * c->K(), cudaMemcpyDeviceToDevice, c->stream));
  return 0;
}

// Both interpolation entry points: `launch(K, pt)` enqueues one kernel over the committed point that reads the stamps
// in cov_t and writes `block` doubles per stamp to cov_o and an invalid flag to cov_bad.
template <typename F>
int cov_interpolate(hb200_ctx* c, int n, const double* stamps, double* cov, int* num_invalid, size_t block, F&& launch) {
  if (!c) return fail(-1, "null context");
  if (n < 0 || (n > 0 && (!stamps || !cov))) return fail(-1, "invalid argument");
  if (!c->cov_valid) return fail(-2, "no covariance computed (hb200_compute_covariance has not succeeded)");
  HB_CUDA(cudaSetDevice(c->device));
  if (num_invalid) *num_invalid = 0;
  if (n == 0) return 0;
  const bool stamp = c->cov_built && c->cov_at == c->launches;   // (reads nothing a compute needs)
  HB_CUDA(c->cov_t.ensure(n)); HB_CUDA(c->cov_o.ensure(block * n)); HB_CUDA(c->cov_bad.ensure(n));
  HB_CUDA(cudaMemcpyAsync(c->cov_t.p, stamps, sizeof(double) * n, cudaMemcpyHostToDevice, c->stream));
  const CovPoint& pt = c->cov_pt[c->cov_slot_committed];
  const int rc = with_order(pt.pose.order, [&](auto K) { return launch(K, pt); });
  if (rc) return rc;
  std::vector<int> bad(n);
  HB_CUDA(cudaMemcpyAsync(cov, c->cov_o.p, sizeof(double) * block * n, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaMemcpyAsync(bad.data(), c->cov_bad.p, sizeof(int) * n, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  if (num_invalid) *num_invalid = std::accumulate(bad.begin(), bad.end(), 0);
  if (stamp) c->cov_at = c->launches;
  return 0;
}

// A registered request against the build's shapes.
bool cov_request_ok(const int4& r, const CovPoint& pt) {
  auto ok = [&](int kind, int i) {
    switch (kind) {
      case kCovKnot: return i >= 0 && i < pt.lay.K;
      case kCovGyroBias: return i >= 0 && i < pt.gyro.n();
      case kCovAccelBias: return i >= 0 && i < pt.accel.n();
      case kCovGravity: return i == 0;
      case kCovLandmark: return i >= 0 && i < pt.L;
      default: return false;
    }
  };
  return ok(r.x, r.y) && ok(r.z, r.w);
}

// The requested blocks and stamp pairs of a compute, after cov_landmark_kernel: the control-point spans of the requests'
// landmarks and of the pairs' stamps (one read-back, only when a request has a landmark or a pair is registered), the
// far-column plan -- for every knot pair more than beta blocks apart that a request or a pair reads, directly or through
// a span, its column (the larger block) and the lowest row the march must reach -- then cov_far_column_kernel over the
// planned columns, cov_cross_landmark_kernel over the requests and cov_pose_pair_kernel over the pairs, into cov_next.
// A column's values do not depend on its lowest row, so the requests' blocks are the same with or without pairs.
int cov_blocks_enqueue(hb200_ctx* c, const CovPoint& pt) {
  const SysLayout& lay = pt.lay;
  const int n = static_cast<int>(c->cov_req.size()), npair = static_cast<int>(c->cov_pairs.size() / 2), K = lay.K, beta = lay.beta;
  if (n) {
    HB_CUDA(c->cov_req_d.ensure(n));
    HB_CUDA(cudaMemcpyAsync(c->cov_req_d.p, c->cov_req.data(), sizeof(int4) * n, cudaMemcpyHostToDevice, c->stream));
  }
  // cov_span: [2n] landmark spans of the requests' sides, then [npair] (base_a, base_b) of the pairs
  std::vector<int2> span(2 * static_cast<size_t>(n) + npair, make_int2(-1, -1));
  const bool landmarks = pt.Nv && std::any_of(c->cov_req.begin(), c->cov_req.end(), [](const int4& r) { return r.x == kCovLandmark || r.z == kCovLandmark; });
  HB_CUDA(c->cov_span.ensure(span.size()));
  if (landmarks) {
    cov_landmark_span_kernel<<<(n + 127) / 128, 128, 0, c->stream>>>(n, c->cov_req_d.p, c->lm_off.p, c->lm_obs.p, c->visual.idx.p, pt.pose.order, c->cov_span.p);
    HB_LAUNCH(c, "cov_landmark_span_kernel");
  }
  if (npair) {
    HB_CUDA(c->cov_pairs_d.ensure(2 * static_cast<size_t>(npair)));
    HB_CUDA(cudaMemcpyAsync(c->cov_pairs_d.p, c->cov_pairs.data(), sizeof(double) * 2 * npair, cudaMemcpyHostToDevice, c->stream));
    cov_stamp_span_kernel<<<(npair + 127) / 128, 128, 0, c->stream>>>(npair, c->cov_pairs_d.p, pt.pose.val[0].p, K, pt.pose.order, c->cov_span.p + 2 * n);
    HB_LAUNCH(c, "cov_stamp_span_kernel");
  }
  if (landmarks || npair) {
    const size_t first = landmarks ? 0 : 2 * static_cast<size_t>(n);
    HB_CUDA(cudaMemcpyAsync(span.data() + first, c->cov_span.p + first, sizeof(int2) * (span.size() - first), cudaMemcpyDeviceToHost, c->stream));
    HB_CUDA(cudaStreamSynchronize(c->stream));
  }
  std::vector<int> need(K, K);   // lowest row block per column block (K: none)
  auto far = [&](int r, int s) {
    if (std::abs(r - s) > beta) need[std::max(r, s)] = std::min(need[std::max(r, s)], std::min(r, s));
  };
  for (int q = 0; q < n; ++q) {
    const int4& r = c->cov_req[q];
    // each side as a knot range [first, end): a knot, a landmark's span; nothing for bias / gravity / unobserved
    int lo[2] = {0, 0}, hi[2] = {0, 0};
    const int kind[2] = {r.x, r.z}, index[2] = {r.y, r.w};
    for (int s = 0; s < 2; ++s) {
      if (kind[s] == kCovKnot) { lo[s] = index[s]; hi[s] = index[s] + 1; }
      else if (kind[s] == kCovLandmark && span[2 * q + s].x >= 0) { lo[s] = span[2 * q + s].x; hi[s] = span[2 * q + s].y; }
    }
    if (kind[0] == kCovLandmark && kind[1] == kCovLandmark && index[0] == index[1]) continue;   // the marginal
    for (int a = lo[0]; a < hi[0]; ++a)
      for (int b = lo[1]; b < hi[1]; ++b) far(a, b);
  }
  for (int q = 0; q < npair; ++q) {
    const int2 s = span[2 * static_cast<size_t>(n) + q];
    if (s.x < 0 || s.y < 0) continue;
    for (int a = s.x; a < s.x + pt.pose.order; ++a)
      for (int b = s.y; b < s.y + pt.pose.order; ++b) far(a, b);
  }
  std::vector<int> plan(K, -1);
  int nc = 0, blocks = 0;
  for (int j = 0; j < K; ++j)
    if (need[j] < K) { plan[j] = nc++; }
  plan.resize(K + 3 * static_cast<size_t>(nc));
  for (int j = 0; j < K; ++j)
    if (need[j] < K) {
      const int s = plan[j];
      plan[K + s] = j; plan[K + nc + s] = need[j]; plan[K + 2 * nc + s] = blocks;
      blocks += j - beta - need[j];
    }
  HB_CUDA(c->cov_plan.ensure(plan.size()));
  HB_CUDA(cudaMemcpyAsync(c->cov_plan.p, plan.data(), sizeof(int) * plan.size(), cudaMemcpyHostToDevice, c->stream));
  HB_CUDA(c->cov_far.ensure(36 * static_cast<size_t>(blocks)));
  CovResults& next = c->cov_next;
  HB_CUDA(next.blk.ensure(36 * static_cast<size_t>(n)));
  HB_CUDA(next.blk_st.ensure(n));
  const CovFarPlan fp{c->cov_plan.p, nc};
  if (nc) {
    const size_t smem = (36 * static_cast<size_t>(beta) + 6 * lay.m + 36) * sizeof(double);
    cov_far_column_kernel<<<nc, kFarThreads, smem, c->stream>>>(c->cov_ws.p, next.packed.p, lay, c->fixed.p, fp, c->cov_status.p, c->cov_far.p);
    HB_LAUNCH(c, "cov_far_column_kernel");
  }
  HB_CUDA(next.pair_joint.ensure(144 * static_cast<size_t>(npair)));
  HB_CUDA(next.pair_rel.ensure(36 * static_cast<size_t>(npair)));
  HB_CUDA(next.pair_st.ensure(npair));
  const size_t smem = static_cast<size_t>(kLmWarps) * 6 * pt.max_rows * sizeof(double);
  return with_order(pt.pose.order, [&](auto Kc) {
    if (n) {
      HB_CUDA(cudaFuncSetAttribute(cov_cross_landmark_kernel<Kc>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
      cov_cross_landmark_kernel<Kc><<<(n + kLmWarps - 1) / kLmWarps, kLmWarps * 32, smem, c->stream>>>(
          n, c->cov_req_d.p, c->lm_off.p, c->lm_obs.p, c->visual.idx.p, c->v_out.Jp.p, c->v_out.Jl.p, c->v_out.w.p, c->Vchol.p, next.packed.p, next.lm.p,
          c->cov_far.p, fp, lay, pt.gyro.n(), c->multi() ? 1 : 0, c->cov_status.p, pt.max_rows, next.blk.p, next.blk_st.p);
      if (const int rc = check_launch(c, "cov_cross_landmark_kernel")) return rc;
    }
    if (npair) {
      cov_pose_pair_kernel<Kc><<<(npair + kPairWarps - 1) / kPairWarps, kPairWarps * 32, 0, c->stream>>>(
          npair, c->cov_pairs_d.p, c->cov_span.p + 2 * n, pt.tab.p, pt.pose.basis, next.packed.p, c->cov_far.p, fp, lay, c->cov_status.p,
          next.pair_joint.p, next.pair_rel.p, next.pair_st.p);
      if (const int rc = check_launch(c, "cov_pose_pair_kernel")) return rc;
    }
    return 0;
  });
}
}  // namespace

extern "C" {

// Sharded contexts (a communicator or the all-reduce callback): collective.  Each rank assembles its undamped partial
// system and writes its degenerate-landmark count into the tail slot kCovDegenerateSlot; ONE system reduction (as
// hb200_build_system) then leaves the same reduced system and the window-wide count on every rank.  The -6 refusal
// depends only on the agreed layout, so every rank refuses before the reduction.
int hb200_build_covariance(hb200_ctx* c) {
  if (!c) return fail(-1, "null context");
  int rc = check_ready(c);
  if (rc) return rc;
  HB_CUDA(cudaSetDevice(c->device));
  const bool sharded = c->multi();
  const size_t smem = cov_smem_doubles(c->beta, c->lay.m) * sizeof(double);
  if (smem > 220 * 1024)
    return fail(-6, "covariance: a window of %d block columns and %d arrow rows needs %zu B of shared memory", c->beta + 1, c->lay.m, smem);
  c->cov_built = false;
  if ((rc = prepare_det(c))) return rc;
  SolverState s{};
  s.radius = INFINITY;   // mu = 1 / radius = 0 in the Schur kernels
  HB_CUDA(c->cov_st.ensure(1));
  HB_CUDA(cudaMemcpyAsync(c->cov_st.p, &s, sizeof(s), cudaMemcpyHostToDevice, c->stream));
  if ((rc = enqueue_assembly(c, c->cov_st.p))) return rc;   // undamped
  c->cov_slot_built = 1 - c->cov_slot_committed;
  if ((rc = freeze_point(c, c->cov_pt[c->cov_slot_built]))) return rc;
  int counts[2] = {0, c->L};
  if (c->Nv && c->L) {
    HB_CUDA(c->cov_counts.ensure(2));
    cov_landmark_flags_kernel<<<1, kCovFlagThreads, 0, c->stream>>>(c->L, c->lm_off.p, c->Vchol.p, c->Dl.p, c->cov_counts.p);
    HB_LAUNCH(c, "cov_landmark_flags_kernel");
    if (sharded) {
      cov_degenerate_slot_kernel<<<1, 1, 0, c->stream>>>(c->cov_counts.p, c->assembly(), c->lay);
      HB_LAUNCH(c, "cov_degenerate_slot_kernel");
    }
    HB_CUDA(cudaMemcpyAsync(counts, c->cov_counts.p, sizeof(counts), cudaMemcpyDeviceToHost, c->stream));
  }
  double window_degenerate = 0.0;
  SolverState red_st{};
  if (sharded) {
    // the peer reduction reports a timed-out peer in cov_st, not in the LM's state; it flips peer_par like any eager
    // reduction, so the next hb200_iterate assembles into (and launches the graph of) the other arena half
    if ((rc = enqueue_reduce_system(c, c->cov_st.p))) { c->outputs_changed(); return rc; }
    HB_CUDA(cudaMemcpyAsync(&window_degenerate, c->sys.p + c->lay.os + kCovDegenerateSlot, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    HB_CUDA(cudaMemcpyAsync(&red_st, c->cov_st.p, sizeof(red_st), cudaMemcpyDeviceToHost, c->stream));
  }
  HB_CUDA(cudaStreamSynchronize(c->stream));
  if (red_st.comm_error) {
    c->outputs_changed();
    return fail(-7, "covariance: a peer did not reach the system reduction in time (every rank must call hb200_build_covariance)");
  }
  c->cov_degenerate = sharded ? static_cast<int>(window_degenerate) : counts[0];
  c->cov_unobserved = counts[1];
  // the factor outputs are those of an evaluation at the current state; the packed buffer is not what hb200_solve expects
  c->outputs_changed();
  c->evaluated_J = true; c->cov_built = true;
  c->cov_at = c->launches;
  return 0;
}

// No collective step: on a sharded context every rank inverts the same reduced system with the same atomic-free kernel
// (Sigma, the status, bad_dof and the pivot are bit-identical across ranks; the degenerate count is the window's), and
// the landmark kernel runs over the rank's own landmarks and their factors.
int hb200_compute_covariance(hb200_ctx* c, hb200_covariance_info* info) {
  if (!c) return fail(-1, "null context");
  if (!info) return fail(-1, "null info");
  // every setter that changes shapes, constants or the state clears cov_built; any other launch since the build (an
  // evaluation, an iteration, a slide) rewrote the factor outputs or the packed buffer the compute reads
  const CovPoint& pt = c->cov_pt[c->cov_slot_built];
  if (!c->cov_built || c->cov_at != c->launches || c->L != pt.L || c->k() != pt.pose.order || c->Nv != pt.Nv ||
      c->max_rows != pt.max_rows || c->lay.total != pt.lay.total || c->lay.beta != pt.lay.beta)
    return fail(-2, "call hb200_build_covariance first (the window was evaluated, iterated or changed since)");
  HB_CUDA(cudaSetDevice(c->device));
  info->status = 0; info->bad_dof = -1; info->min_pivot_ratio = 0.0;
  if (c->cov_degenerate) {
    cov_info(c, info);
    info->status = 2;
    return fail(HB200_COV_DEGENERATE_LANDMARKS, "covariance: %d landmark(s) with a rank-deficient V_l (observed by too few factors)", c->cov_degenerate);
  }
  for (size_t q = 0; q < c->cov_req.size(); ++q)
    if (!cov_request_ok(c->cov_req[q], pt))
      return fail(-1, "covariance block %zu: (kind %d, index %d) x (kind %d, index %d) is not a block of the built window", q, c->cov_req[q].x,
                  c->cov_req[q].y, c->cov_req[q].z, c->cov_req[q].w);
  const SysLayout& lay = pt.lay;
  const size_t smem = cov_smem_doubles(lay.beta, lay.m) * sizeof(double);
  HB_CUDA(c->cov_ws.ensure(static_cast<size_t>(cov_workspace_doubles(lay))));
  const int L = pt.L, k = pt.pose.order, max_rows = pt.max_rows;   // (the build's shapes)
  CovResults& next = c->cov_next;
  HB_CUDA(next.packed.ensure(static_cast<size_t>(cov_packed_doubles(lay))));
  HB_CUDA(next.lm.ensure(9 * static_cast<size_t>(std::max(L, 1))));
  next.blk_n = static_cast<int>(c->cov_req.size());
  next.pair_n = static_cast<int>(c->cov_pairs.size() / 2);
  HB_CUDA(c->cov_status.ensure(1));
  HB_CUDA(cudaFuncSetAttribute(cov_selinv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  cov_selinv_kernel<<<1, kCovThreads, smem, c->stream>>>(c->sys.p, lay, c->fixed.p, c->cov_ws.p, next.packed.p, c->cov_status.p);
  HB_LAUNCH(c, "cov_selinv_kernel");
  if (L && pt.Nv) {
    const int blocks = (L + kLmWarps - 1) / kLmWarps;
    const size_t lsmem = static_cast<size_t>(kLmWarps) * 3 * max_rows * sizeof(double);
    const int rc = with_order(k, [&](auto K) {
      cov_landmark_kernel<K><<<blocks, kLmWarps * 32, lsmem, c->stream>>>(L, c->lm_off.p, c->lm_obs.p, c->visual.idx.p, c->v_out.Jp.p, c->v_out.Jl.p, c->v_out.w.p, c->Vchol.p,
                                                                         next.packed.p, lay, c->cov_status.p, next.lm.p, max_rows);
      return check_launch(c, "cov_landmark_kernel");
    });
    if (rc) return rc;
  } else if (L) {
    HB_CUDA(cudaMemsetAsync(next.lm.p, 0, sizeof(double) * 9 * L, c->stream));
  }
  // requested blocks and stamp pairs: the landmark blocks need the build's factor outputs and the far columns the factor
  // in cov_ws, both valid only until the next launch, so they are computed here (nothing runs without a request or pair)
  if (!c->cov_req.empty() || !c->cov_pairs.empty())
    if (const int rc = cov_blocks_enqueue(c, pt)) return rc;
  CovStatus st{};
  HB_CUDA(cudaMemcpyAsync(&st, c->cov_status.p, sizeof(st), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  c->cov_at = c->launches;
  info->bad_dof = st.bad_dof;
  info->min_pivot_ratio = std::isfinite(st.min_pivot) ? st.min_pivot : 0.0;
  if (st.status) {
    cov_info(c, info);
    info->status = 1;
    return fail(HB200_COV_NOT_POSITIVE_DEFINITE, "covariance: the reduced system is not positive definite (pivot %.3e of dof %d, threshold %.0e)",
                st.min_pivot, st.bad_dof, kCovMinPivot);
  }
  // commit: results, and the linearisation point they belong to
  c->cov_res.swap(next);
  c->cov_slot_committed = c->cov_slot_built;
  c->cov_valid = true;
  cov_info(c, info);
  return 0;
}

int hb200_set_covariance_blocks(hb200_ctx* c, int n, const int* pairs) {
  if (!c) return fail(-1, "null context");
  static_assert(+HB200_COV_KNOT == +kCovKnot && +HB200_COV_GYRO_BIAS == +kCovGyroBias && +HB200_COV_ACCEL_BIAS == +kCovAccelBias &&
                    +HB200_COV_GRAVITY == +kCovGravity && +HB200_COV_LANDMARK == +kCovLandmark,
                "covariance block kinds");
  if (n < 0 || (n > 0 && !pairs)) return fail(-1, "invalid argument");
  c->cov_req.resize(n);
  for (int q = 0; q < n; ++q) c->cov_req[q] = make_int4(pairs[4 * q], pairs[4 * q + 1], pairs[4 * q + 2], pairs[4 * q + 3]);
  return 0;
}

int hb200_get_covariance_blocks(hb200_ctx* c, int n, double* out, int* status) {
  if (!c) return fail(-1, "null context");
  if (n < 0 || (n > 0 && !out)) return fail(-1, "invalid argument");
  if (!c->cov_valid) return fail(-2, "no covariance computed (hb200_compute_covariance has not succeeded)");
  if (n != c->cov_res.blk_n) return fail(-2, "the last successful compute had %d covariance blocks, not %d", c->cov_res.blk_n, n);
  if (n == 0) return 0;
  HB_CUDA(cudaSetDevice(c->device));
  HB_CUDA(cudaMemcpyAsync(out, c->cov_res.blk.p, sizeof(double) * 36 * n, cudaMemcpyDeviceToHost, c->stream));
  if (status) HB_CUDA(cudaMemcpyAsync(status, c->cov_res.blk_st.p, sizeof(int) * n, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

int hb200_set_covariance_stamp_pairs(hb200_ctx* c, int n, const double* stamps) {
  if (!c) return fail(-1, "null context");
  if (n < 0 || (n > 0 && !stamps)) return fail(-1, "invalid argument");
  for (size_t i = 0; i < 2 * static_cast<size_t>(n); ++i)
    if (!std::isfinite(stamps[i])) return fail(-1, "stamp pair %zu: stamp %zu is not finite", i / 2, i % 2);
  c->cov_pairs.assign(stamps, stamps + 2 * static_cast<size_t>(n));
  return 0;
}

int hb200_get_pose_pair_covariance(hb200_ctx* c, int n, double* joint, double* relative, int* status) {
  if (!c) return fail(-1, "null context");
  if (n < 0) return fail(-1, "invalid argument");
  if (!c->cov_valid) return fail(-2, "no covariance computed (hb200_compute_covariance has not succeeded)");
  if (n != c->cov_res.pair_n) return fail(-2, "the last successful compute had %d stamp pairs, not %d", c->cov_res.pair_n, n);
  if (n == 0) return 0;
  HB_CUDA(cudaSetDevice(c->device));
  if (joint) HB_CUDA(cudaMemcpyAsync(joint, c->cov_res.pair_joint.p, sizeof(double) * 144 * n, cudaMemcpyDeviceToHost, c->stream));
  if (relative) HB_CUDA(cudaMemcpyAsync(relative, c->cov_res.pair_rel.p, sizeof(double) * 36 * n, cudaMemcpyDeviceToHost, c->stream));
  if (status) HB_CUDA(cudaMemcpyAsync(status, c->cov_res.pair_st.p, sizeof(int) * n, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

int hb200_get_covariance(hb200_ctx* c, double* packed, double* landmark) {
  if (!c) return fail(-1, "null context");
  if (!c->cov_valid) return fail(-2, "no covariance computed (hb200_compute_covariance has not succeeded)");
  HB_CUDA(cudaSetDevice(c->device));
  const CovPoint& pt = c->cov_pt[c->cov_slot_committed];
  if (packed) HB_CUDA(cudaMemcpyAsync(packed, c->cov_res.packed.p, sizeof(double) * cov_packed_doubles(pt.lay), cudaMemcpyDeviceToHost, c->stream));
  if (landmark && pt.L) HB_CUDA(cudaMemcpyAsync(landmark, c->cov_res.lm.p, sizeof(double) * 9 * pt.L, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

int hb200_interpolate_covariance(hb200_ctx* c, int n, const double* stamps, double* cov, int* num_invalid) {
  return cov_interpolate(c, n, stamps, cov, num_invalid, 36, [&](auto K, const CovPoint& pt) {
    cov_stamp_kernel<K, 6><<<(n + kStateWarps - 1) / kStateWarps, kStateWarps * 32, 0, c->stream>>>(
        n, c->cov_t.p, pt.pose.val[0].p, pt.tab.p, pt.lay.K, pt.pose.basis, nullptr, 0, nullptr, 0, pt.gyro.basis, c->cov_res.packed.p, pt.lay, c->cov_o.p, c->cov_bad.p);
    return check_launch(c, "cov_stamp_kernel");
  });
}

int hb200_interpolate_state_covariance(hb200_ctx* c, int n, const double* stamps, double* cov, int* num_invalid) {
  static_assert(HB200_STATE_COV_DIM == kStateDim, "state covariance dimension");
  return cov_interpolate(c, n, stamps, cov, num_invalid, HB200_STATE_COV_DIM * HB200_STATE_COV_DIM, [&](auto K, const CovPoint& pt) {
    cov_stamp_kernel<K, kStateDim><<<(n + kStateWarps - 1) / kStateWarps, kStateWarps * 32, 0, c->stream>>>(
        n, c->cov_t.p, pt.pose.val[0].p, pt.tab.p, pt.lay.K, pt.pose.basis, pt.gyro.val[0].p, pt.gyro.n(), pt.accel.val[0].p, pt.accel.n(), pt.gyro.basis, c->cov_res.packed.p, pt.lay, c->cov_o.p, c->cov_bad.p);
    return check_launch(c, "cov_stamp_kernel");
  });
}

}  // extern "C"

namespace {

int iterate_enqueue(hb200_ctx* c, int iterations) {
  int rc = prepare_det(c);
  if (rc) return rc;
  for (int it = 0; it < iterations; ++it) {
    // the callback hook cannot be captured; with NCCL the first iteration runs eagerly (NCCL finishes its lazy
    // channel / buffer setup outside of a capture), every later one is a graph launch.  With the peer-memory
    // reduction the iteration exists twice: it assembles into arena half A or B by parity.
    const bool graph_ok = c->use_graph && !c->allreduce && (!c->nccl || c->comm_warm || c->peer_reduce());
    if (graph_ok) {
      const bool slot_b = c->peer_reduce() && c->peer_par == 1;
      IterationGraph& g = c->graphs[slot_b];
      if (!g.valid) {
        g.release();
        const int par_before = c->peer_par;
        HB_CUDA(cudaStreamBeginCapture(c->stream, c->nccl ? cudaStreamCaptureModeRelaxed : cudaStreamCaptureModeThreadLocal));
        const long long before = c->launches, nccl_before = c->nccl_calls;
        rc = enqueue_iteration(c);
        cudaError_t e = cudaStreamEndCapture(c->stream, &g.graph);
        c->launches = before;  // capture does not execute
        c->nccl_calls_per_iteration = c->nccl_calls - nccl_before;
        c->nccl_calls = nccl_before;
        c->peer_par = par_before;   // (enqueue_iteration toggled it: the toggle happens again at the launch below)
        if (rc) return rc;
        if (e != cudaSuccess) {
          if (!c->nccl) return fail(100 + static_cast<int>(e), "graph capture: %s", cudaGetErrorString(e));
          // a communicator that cannot be captured: fall back to direct launches for this context
          cudaGetLastError();
          c->use_graph = false; g.graph = nullptr;
          --it;
          continue;
        }
        HB_CUDA(cudaGraphInstantiate(&g.exec, g.graph, 0));
        g.valid = true;
        c->launches_per_iteration = 0;
        size_t nodes = 0;
        HB_CUDA(cudaGraphGetNodes(g.graph, nullptr, &nodes));
        cudaGraphNode_t* nd = new cudaGraphNode_t[nodes];
        HB_CUDA(cudaGraphGetNodes(g.graph, nd, &nodes));
        for (size_t i = 0; i < nodes; ++i) { cudaGraphNodeType t; if (cudaGraphNodeGetType(nd[i], &t) == cudaSuccess && t == cudaGraphNodeTypeKernel) c->launches_per_iteration += 1; }
        delete[] nd;
        c->launches_per_iteration -= c->nccl_calls_per_iteration;   // NCCL's kernel nodes are not this library's launches
        if (getenv("HB200_GRAPH_DEBUG")) {
          size_t edges = 0;
          cudaGraphGetEdges(g.graph, nullptr, nullptr, &edges);
          std::fprintf(stderr, "[hb200] iteration graph%s: %zu nodes (%lld own kernels, %lld NCCL), %zu edges\n", slot_b ? " (arena half B)" : "", nodes,
                       c->launches_per_iteration, c->nccl_calls_per_iteration, edges);
        }
      }
      HB_CUDA(cudaGraphLaunch(g.exec, c->stream));
      if (c->peer_reduce()) c->peer_par ^= 1;
      c->launches += c->launches_per_iteration;
      c->nccl_calls += c->nccl_calls_per_iteration;
    } else {
      if ((rc = enqueue_iteration(c))) return rc;
      if (c->nccl) c->comm_warm = true;
    }
  }
  c->outputs_changed();
  if (!c->term_enabled) c->iter_total += iterations;   // (with the termination tests on, the device counter is authoritative: pick_records)
  return 0;
}

// The device ring buffer of iteration records and the solver state, fetched in one batch (asynchronously); the
// records of the iterations PERFORMED since `it_before` are picked out after the synchronisation (with the
// termination tests on, fewer iterations than requested may have been performed).
struct RecordFetch {
  std::vector<SolverState> ring;
  SolverState st{};
};
int fetch_records(hb200_ctx* c, RecordFetch* f, SolverState* pinned = nullptr) {
  f->ring.resize(c->max_records);
  SolverState* dst = pinned ? pinned : f->ring.data();
  HB_CUDA(cudaMemcpyAsync(dst, c->records.p, sizeof(SolverState) * c->max_records, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaMemcpyAsync(pinned ? pinned + c->max_records : &f->st, c->st.p, sizeof(SolverState), cudaMemcpyDeviceToHost, c->stream));
  return 0;
}
// after the stream synchronisation: records of iterations it_before+1 .. st.iteration in order; returns their number
int pick_records(hb200_ctx* c, RecordFetch* f, long long it_before, int requested, std::vector<SolverState>* rec, const SolverState* pinned = nullptr) {
  if (pinned) { std::copy(pinned, pinned + c->max_records, f->ring.begin()); f->st = pinned[c->max_records]; }
  const long long it_after = f->st.iteration;
  const int performed = static_cast<int>(std::max<long long>(0, std::min<long long>(it_after - it_before, requested)));
  rec->resize(performed);
  for (int i = 0; i < performed; ++i) (*rec)[i] = f->ring[(it_before + i) % c->max_records];
  c->iter_total = it_after;
  c->last_terminated = f->st.terminated; c->last_performed = performed;
  c->last_gmax = f->st.gradient_max_norm; c->last_step_norm = f->st.step_norm; c->last_x_norm = f->st.x_norm;
  return performed;
}

// The reductions that can only sum (callback hook, NCCL without a peer mapping) cannot form the maximum of the landmark
// gradient over the ranks (scalars_kernel), so the gradient-tolerance test would see only the replicated blocks.  Checked
// when the iterations run, so that the order of hb200_set_termination and attaching the reduction does not matter.
int check_gradient_test(hb200_ctx* c) {
  const bool sum_only = c->multi() && !(c->nccl && c->peers_open);
  if (sum_only && c->term_enabled && c->term_gtol > 0.0)
    return fail(-2, "the gradient tolerance needs the peer mailbox across ranks (NCCL + hb200_peer_connect); set it to 0 with the "
                    "all-reduce callback or NCCL without a peer mapping");
  return 0;
}

void convert_records(const std::vector<SolverState>& rec, hb200_iteration* records) {
  for (size_t i = 0; i < rec.size(); ++i) {
    records[i].cost = rec[i].cost; records[i].cost_new = rec[i].cost_new; records[i].model_change = rec[i].model_change; records[i].rho = rec[i].rho;
    records[i].radius = rec[i].radius; records[i].accepted = rec[i].accepted; records[i].spd = rec[i].spd;
  }
}
}  // namespace

extern "C" {

int hb200_iterate(hb200_ctx* c, int iterations, hb200_iteration* records) {
  int rc = check_ready(c);
  if (rc) return rc;
  if (iterations < 0 || iterations > c->max_records) return fail(-1, "iterations must be in [0, %d]", c->max_records);
  if ((rc = check_gradient_test(c))) return rc;
  HB_CUDA(cudaSetDevice(c->device));
  if (c->term_enabled) {   // a new call continues the trust region but starts with a clean termination state
    new_solve_kernel<<<1, 1, 0, c->stream>>>(c->st.p, c->radius0, 0);
    HB_LAUNCH(c, "new_solve_kernel");
  }
  const long long it_before = c->iter_total;
  if ((rc = iterate_enqueue(c, iterations))) return rc;
  if (iterations && (records || c->term_enabled)) {
    RecordFetch f;
    std::vector<SolverState> rec;
    if ((rc = fetch_records(c, &f))) return rc;
    HB_CUDA(cudaStreamSynchronize(c->stream));
    const int performed = pick_records(c, &f, it_before, iterations, &rec);
    if (records) {
      convert_records(rec, records);
      for (int i = performed; i < iterations; ++i) records[i] = hb200_iteration{};   // not performed: the solve terminated earlier
    }
  }
  return 0;
}

int hb200_optimize(hb200_ctx* c, int iterations, double* knots, double* gyro, double* accel, double* gravity, double* landmarks,
                   hb200_iteration* records) {
  int rc = check_ready(c);
  if (rc) return rc;
  if (iterations < 0 || iterations > c->max_records) return fail(-1, "iterations must be in [0, %d]", c->max_records);
  if ((rc = check_gradient_test(c))) return rc;
  HB_CUDA(cudaSetDevice(c->device));
  // the blocks alias the caller's variables, stamps included: the bound index maps are only valid for the stamps
  // they were computed from (a slid window needs hb200_set_spline / hb200_slide + hb200_bind first)
  int j = -1;
  if (knots && (j = c->pose.mismatch(knots)) >= 0) return fail(-2, "knot %d: stamp differs from the bound window (re-bind after changing stamps)", j);
  if (gyro && (j = c->gyro.mismatch(gyro)) >= 0) return fail(-2, "gyroscope bias knot %d: stamp differs from the bound window", j);
  if (accel && (j = c->accel.mismatch(accel)) >= 0) return fail(-2, "accelerometer bias knot %d: stamp differs from the bound window", j);
  const auto blocks = c->state_blocks();
  double* host[5] = {knots, gyro, accel, gravity, landmarks};
  double* dev[5];
  size_t cnt[5], off[5], total = 0;
  for (int i = 0; i < 5; ++i) {
    dev[i] = blocks[i].cur->p; cnt[i] = blocks[i].count;
    if (!cnt[i]) host[i] = nullptr;   // (an empty block is never copied)
    off[i] = total; if (host[i]) total += cnt[i];
  }
  if (gravity) c->have_gravity = true;
  // Small windows: 11 small copies cost more than the iteration's kernels save; pack the blocks into one pinned
  // staging buffer (host memcpy, a few KB), one H2D, one segmented device copy -- and the mirror image back.
  const bool staged = total > 0 && total <= 8192;
  CommitArgs in{}, out{};
  if (staged) {
    if (c->h_stage_cap < total) {
      if (c->h_stage) cudaFreeHost(c->h_stage);
      c->h_stage = nullptr; c->h_stage_cap = 0;
      HB_CUDA(cudaMallocHost(&c->h_stage, sizeof(double) * 8192 + sizeof(SolverState) * (c->max_records + 1)));
      c->h_stage_cap = 8192;
    }
    HB_CUDA(c->d_stage.ensure(8192));
    for (int i = 0; i < 5; ++i) {
      const size_t n_i = host[i] ? cnt[i] : 0;
      if (n_i) std::memcpy(c->h_stage + off[i], host[i], sizeof(double) * n_i);
      in.count[i] = n_i; in.src[i] = c->d_stage.p + off[i]; in.dst[i] = dev[i];
      out.count[i] = n_i; out.src[i] = dev[i]; out.dst[i] = c->d_stage.p + off[i];
    }
    HB_CUDA(cudaMemcpyAsync(c->d_stage.p, c->h_stage, sizeof(double) * total, cudaMemcpyHostToDevice, c->stream));
    copy_segments_kernel<<<4, 256, 0, c->stream>>>(in);
    HB_LAUNCH(c, "copy_segments_kernel");
  } else {
    for (int i = 0; i < 5; ++i)
      if (host[i]) HB_CUDA(cudaMemcpyAsync(dev[i], host[i], sizeof(double) * cnt[i], cudaMemcpyHostToDevice, c->stream));
  }
  // every ceres::Solve starts from the initial trust-region radius and a clean termination state
  new_solve_kernel<<<1, 1, 0, c->stream>>>(c->st.p, c->radius0, 1);
  HB_LAUNCH(c, "new_solve_kernel");
  const long long it_before = c->iter_total;
  if ((rc = iterate_enqueue(c, iterations))) return rc;
  if (staged) {
    copy_segments_kernel<<<4, 256, 0, c->stream>>>(out);
    HB_LAUNCH(c, "copy_segments_kernel");
    HB_CUDA(cudaMemcpyAsync(c->h_stage, c->d_stage.p, sizeof(double) * total, cudaMemcpyDeviceToHost, c->stream));
  } else {
    for (int i = 0; i < 5; ++i)
      if (host[i]) HB_CUDA(cudaMemcpyAsync(host[i], dev[i], sizeof(double) * cnt[i], cudaMemcpyDeviceToHost, c->stream));
  }
  std::vector<SolverState> rec;
  RecordFetch fetch;
  SolverState* rec_pinned = staged ? reinterpret_cast<SolverState*>(c->h_stage + 8192) : nullptr;
  const bool want_records = (records && iterations) || c->term_enabled;
  if (want_records && (rc = fetch_records(c, &fetch, rec_pinned))) return rc;
  HB_CUDA(cudaStreamSynchronize(c->stream));
  if (staged) {
    for (int i = 0; i < 5; ++i)
      if (host[i]) std::memcpy(host[i], c->h_stage + off[i], sizeof(double) * cnt[i]);
  }
  if (want_records) {
    const int performed = pick_records(c, &fetch, it_before, iterations, &rec, rec_pinned);
    if (records) {
      convert_records(rec, records);
      for (int i = performed; i < iterations; ++i) records[i] = hb200_iteration{};
    }
  }
  return 0;
}

int hb200_set_termination(hb200_ctx* c, double function_tolerance, double gradient_tolerance, double parameter_tolerance, double min_trust_region_radius) {
  if (!c) return fail(-1, "null context");
  c->term_ftol = function_tolerance; c->term_gtol = gradient_tolerance; c->term_ptol = parameter_tolerance; c->term_min_radius = min_trust_region_radius;
  c->term_enabled = function_tolerance > 0 || gradient_tolerance > 0 || parameter_tolerance > 0 || min_trust_region_radius > 0;
  c->iterations_changed();   // baked into kernel arguments
  return 0;
}

int hb200_get_termination(hb200_ctx* c, int* type, int* iterations_performed, double* gradient_max_norm, double* step_norm, double* x_norm) {
  if (!c) return fail(-1, "null context");
  if (type) *type = c->last_terminated;
  if (iterations_performed) *iterations_performed = c->last_performed;
  if (gradient_max_norm) *gradient_max_norm = c->last_gmax;
  if (step_norm) *step_norm = c->last_step_norm;
  if (x_norm) *x_norm = c->last_x_norm;
  return 0;
}

int hb200_cost(hb200_ctx* c, double* cost) {
  int rc = check_ready(c);
  if (rc) return rc;
  if (!cost) return fail(-1, "null argument");
  HB_CUDA(cudaSetDevice(c->device));
  if ((rc = enqueue_evaluate(c, false, 0))) return rc;
  if ((rc = enqueue_scalars(c))) return rc;
  double s[4];
  HB_CUDA(cudaMemcpyAsync(s, c->scal.p, sizeof(s), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  *cost = s[0];
  return 0;
}

// FP64 throughput ceiling of the device (SURVEY.md 8d: "FP64 peak not in MEASURED_PEAKS.json -- measure"):
// 8 independent DFMA chains per thread, enough warps to hide the 8-cycle dependent latency.
__global__ void __launch_bounds__(256) hb200_fp64_peak_kernel(double* out, int iters, double a, double b) {
  double x0 = threadIdx.x, x1 = x0 + 1, x2 = x0 + 2, x3 = x0 + 3, x4 = x0 + 4, x5 = x0 + 5, x6 = x0 + 6, x7 = x0 + 7;
#pragma unroll 1
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      x0 = fma(x0, a, b); x1 = fma(x1, a, b); x2 = fma(x2, a, b); x3 = fma(x3, a, b);
      x4 = fma(x4, a, b); x5 = fma(x5, a, b); x6 = fma(x6, a, b); x7 = fma(x7, a, b);
    }
  }
  const double s = x0 + x1 + x2 + x3 + x4 + x5 + x6 + x7;
  if (s == 1.2345e300) out[0] = s;   // never true: keeps the chains alive
}

int hb200_measure_fp64_peak(hb200_ctx* c, double* tflops) {
  if (!c || !tflops) return fail(-1, "null argument");
  HB_CUDA(cudaSetDevice(c->device));
  DevBuf<double> d;
  HB_CUDA(d.ensure(1));
  cudaEvent_t e0, e1;
  HB_CUDA(cudaEventCreate(&e0)); HB_CUDA(cudaEventCreate(&e1));
  const int blocks = c->num_sms * 8, iters = 4096;
  double best = 0.0;
  for (int rep = 0; rep < 4; ++rep) {
    HB_CUDA(cudaEventRecord(e0, c->stream));
    hb200_fp64_peak_kernel<<<blocks, 256, 0, c->stream>>>(d.p, iters, 0.999999, 1e-7);
    HB_CUDA(cudaEventRecord(e1, c->stream));
    HB_CUDA(cudaStreamSynchronize(c->stream));
    float ms = 0;
    HB_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    const double flops = 2.0 * 64.0 * iters * 256.0 * blocks;
    if (rep > 0) best = std::max(best, flops / (ms * 1e-3) / 1e12);
  }
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  *tflops = best;
  return 0;
}

__global__ void hb200_spin_kernel(long long cycles) {
  const long long t0 = clock64();
  while (clock64() - t0 < cycles) {}
}

int hb200_profile_iteration(hb200_ctx* c, int reps, int max_entries, char* names, double* ms, int* count) {
  int rc = check_ready(c);
  if (rc) return rc;
  if (reps == 0 || !names || !ms || !count) return fail(-1, "invalid argument");
  const bool reps_mode_evaluate = reps < 0;   // negative reps: profile the Evaluate sweep only
  if (reps < 0) reps = -reps;
  HB_CUDA(cudaSetDevice(c->device));
  if ((rc = prepare_det(c))) return rc;
  std::vector<double> acc;
  std::vector<std::string> nm;
  for (int rep = 0; rep < reps; ++rep) {
    c->prof_used = 0;
    // keep the GPU busy while the host enqueues the whole iteration, so kernels run back to back
    hb200_spin_kernel<<<1, 1, 0, c->stream>>>(600000);
    c->profiling = true;
    prof_mark(c, "start");
    if (reps_mode_evaluate) rc = enqueue_evaluate(c, true, 0);   // the plain Evaluate sweep (hb200_evaluate), Jacobians materialised
    else rc = enqueue_iteration(c);
    c->profiling = false;
    if (rc) return rc;
    if (!reps_mode_evaluate) c->iter_total += 1;
    HB_CUDA(cudaStreamSynchronize(c->stream));
    if (rep == 0) { acc.assign(c->prof_used, 0.0); nm.assign(c->prof_names.begin(), c->prof_names.begin() + c->prof_used); }
    for (size_t i = 1; i < c->prof_used && i < acc.size(); ++i) {
      float t = 0;
      HB_CUDA(cudaEventElapsedTime(&t, c->prof_events[i - 1], c->prof_events[i]));
      acc[i] += t;
    }
  }
  int n_out = 0;
  for (size_t i = 1; i < acc.size() && n_out < max_entries; ++i, ++n_out) {
    std::snprintf(names + 32 * n_out, 32, "%s", nm[i].c_str());
    ms[n_out] = acc[i] / reps;
  }
  *count = n_out;
  c->outputs_changed();
  return 0;
}

int hb200_interpolate(hb200_ctx* c, int n, const double* stamps, double* pose, double* velocity, double* acceleration, int* num_invalid) {
  if (!c || n < 0 || (n > 0 && (!stamps || !pose))) return fail(-1, "invalid argument");
  if (c->K() == 0) return fail(-2, "spline not set");
  HB_CUDA(cudaSetDevice(c->device));
  if (num_invalid) *num_invalid = 0;
  if (n == 0) return 0;
  DevBuf<double> d_t, d_p, d_v, d_a;
  HB_CUDA(d_t.ensure(n)); HB_CUDA(d_p.ensure(7 * static_cast<size_t>(n)));
  if (velocity) HB_CUDA(d_v.ensure(6 * static_cast<size_t>(n)));
  if (acceleration) HB_CUDA(d_a.ensure(6 * static_cast<size_t>(n)));
  HB_CUDA(c->d_invalid.ensure(1));
  HB_CUDA(cudaMemsetAsync(c->d_invalid.p, 0, sizeof(int), c->stream));
  HB_CUDA(cudaMemcpyAsync(d_t.p, stamps, sizeof(double) * n, cudaMemcpyHostToDevice, c->stream));
  prep_kernel<<<(c->K() + 63) / 64, 64, 0, c->stream>>>(c->K(), c->pose.val[0].p, c->tab[0].p, nullptr, 0);
  HB_LAUNCH(c, "prep_kernel");
  const int rc = with_order(c->k(), [&](auto K) {
    interpolate_kernel<K><<<(n + 127) / 128, 128, 0, c->stream>>>(n, d_t.p, c->pose.val[0].p, c->tab[0].p, c->K(), c->pose.basis, d_p.p, d_v.p, d_a.p, c->d_invalid.p);
    return check_launch(c, "interpolate_kernel");
  });
  if (rc) return rc;
  int bad = 0;
  HB_CUDA(cudaMemcpyAsync(pose, d_p.p, sizeof(double) * 7 * n, cudaMemcpyDeviceToHost, c->stream));
  if (velocity) HB_CUDA(cudaMemcpyAsync(velocity, d_v.p, sizeof(double) * 6 * n, cudaMemcpyDeviceToHost, c->stream));
  if (acceleration) HB_CUDA(cudaMemcpyAsync(acceleration, d_a.p, sizeof(double) * 6 * n, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaMemcpyAsync(&bad, c->d_invalid.p, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  cudaError_t e = cudaStreamSynchronize(c->stream);
  d_t.release(); d_p.release(); d_v.release(); d_a.release();
  if (e != cudaSuccess) return fail(100 + static_cast<int>(e), "interpolate: %s", cudaGetErrorString(e));
  if (num_invalid) *num_invalid = bad;
  return 0;
}

int hb200_debug_band_timing(hb200_ctx* c, long long* cycles /*[144]: per CTA, 8 phase totals + 8 steps x 8 raw stamps; [70]: SPD flag of the solve*/) {
  if (!c || !c->band_dbg.p) return fail(-2, "set HB200_BAND_TIMING=1 before hb200_bind");
  HB_CUDA(cudaMemcpy(cycles, c->band_dbg.p, 144 * sizeof(long long), cudaMemcpyDeviceToHost));
  return 0;
}

int hb200_snapshot(hb200_ctx* c) {
  if (!c || c->K() == 0) return fail(-2, "spline not set");
  HB_CUDA(cudaSetDevice(c->device));
  const auto blocks = c->state_blocks();
  for (const auto& b : blocks) HB_CUDA(b.snap->ensure(std::max<size_t>(b.count, 1)));
  HB_CUDA(c->snap_st.ensure(1));
  for (const auto& b : blocks)
    if (b.count) HB_CUDA(cudaMemcpyAsync(b.snap->p, b.cur->p, sizeof(double) * b.count, cudaMemcpyDeviceToDevice, c->stream));
  HB_CUDA(cudaMemcpyAsync(c->snap_st.p, c->st.p, sizeof(SolverState), cudaMemcpyDeviceToDevice, c->stream));
  c->have_snapshot = true;
  c->snap_iter_total = c->iter_total;
  return 0;
}

int hb200_restore(hb200_ctx* c) {
  if (!c || !c->have_snapshot) return fail(-2, "no snapshot");
  HB_CUDA(cudaSetDevice(c->device));
  for (const auto& b : c->state_blocks())
    if (b.count) HB_CUDA(cudaMemcpyAsync(b.cur->p, b.snap->p, sizeof(double) * b.count, cudaMemcpyDeviceToDevice, c->stream));
  HB_CUDA(cudaMemcpyAsync(c->st.p, c->snap_st.p, sizeof(SolverState), cudaMemcpyDeviceToDevice, c->stream));
  c->iter_total = c->snap_iter_total;
  c->outputs_changed();
  return 0;
}

int hb200_ingest_stereo(hb200_ctx* c, int n, const double* stamp, const int* camera0, const int* camera1, const double* pixel0,
                        const double* pixel1, double* bearing0, double* bearing1, double* landmark, int* num_invalid) {
  if (!c || n < 0) return fail(-1, "invalid arguments");
  if (c->K() == 0 || c->C == 0) return fail(-2, "spline / cameras not set");
  if (n > 0 && (!stamp || !camera0 || !camera1 || !pixel0 || !pixel1 || !bearing0 || !bearing1 || !landmark)) return fail(-1, "null argument");
  if (num_invalid) *num_invalid = 0;
  if (n == 0) return 0;
  HB_CUDA(cudaSetDevice(c->device));
  DevBuf<double> d_t, d_p0, d_p1, d_b0, d_b1, d_lm;
  DevBuf<int> d_c0, d_c1;
  const size_t N = static_cast<size_t>(n);
  HB_CUDA(d_t.ensure(N)); HB_CUDA(d_p0.ensure(2 * N)); HB_CUDA(d_p1.ensure(2 * N)); HB_CUDA(d_b0.ensure(3 * N)); HB_CUDA(d_b1.ensure(3 * N));
  HB_CUDA(d_lm.ensure(3 * N)); HB_CUDA(d_c0.ensure(N)); HB_CUDA(d_c1.ensure(N));
  HB_CUDA(c->d_invalid.ensure(1));
  HB_CUDA(cudaMemsetAsync(c->d_invalid.p, 0, sizeof(int), c->stream));
  HB_CUDA(cudaMemcpyAsync(d_t.p, stamp, sizeof(double) * N, cudaMemcpyHostToDevice, c->stream));
  HB_CUDA(cudaMemcpyAsync(d_c0.p, camera0, sizeof(int) * N, cudaMemcpyHostToDevice, c->stream));
  HB_CUDA(cudaMemcpyAsync(d_c1.p, camera1, sizeof(int) * N, cudaMemcpyHostToDevice, c->stream));
  HB_CUDA(cudaMemcpyAsync(d_p0.p, pixel0, sizeof(double) * 2 * N, cudaMemcpyHostToDevice, c->stream));
  HB_CUDA(cudaMemcpyAsync(d_p1.p, pixel1, sizeof(double) * 2 * N, cudaMemcpyHostToDevice, c->stream));
  prep_kernel<<<(c->K() + 63) / 64, 64, 0, c->stream>>>(c->K(), c->pose.val[0].p, c->tab[0].p, nullptr, 0);
  HB_LAUNCH(c, "prep_kernel");
  const int rc = with_order(c->k(), [&](auto K) {
    ingest_stereo_kernel<K><<<(n + 127) / 128, 128, 0, c->stream>>>(n, d_t.p, d_c0.p, d_c1.p, d_p0.p, d_p1.p, c->pose.val[0].p, c->tab[0].p, c->K(), c->pose.basis, c->cams.p, c->C, d_b0.p, d_b1.p, d_lm.p, c->d_invalid.p);
    return check_launch(c, "ingest_stereo_kernel");
  });
  if (rc) return rc;
  int bad = 0;
  HB_CUDA(cudaMemcpyAsync(bearing0, d_b0.p, sizeof(double) * 3 * N, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaMemcpyAsync(bearing1, d_b1.p, sizeof(double) * 3 * N, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaMemcpyAsync(landmark, d_lm.p, sizeof(double) * 3 * N, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaMemcpyAsync(&bad, c->d_invalid.p, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  d_t.release(); d_p0.release(); d_p1.release(); d_b0.release(); d_b1.release(); d_lm.release(); d_c0.release(); d_c1.release();
  if (num_invalid) *num_invalid = bad;
  return 0;
}

int hb200_get_state(hb200_ctx* c, double* knots, double* gyro, double* accel, double* gravity, double* landmarks) {
  if (!c) return fail(-1, "null context");
  HB_CUDA(cudaSetDevice(c->device));
  double* host[5] = {knots, gyro, accel, gravity, landmarks};
  const auto blocks = c->state_blocks();
  for (int i = 0; i < 5; ++i)
    if (host[i] && blocks[i].count) HB_CUDA(cudaMemcpyAsync(host[i], blocks[i].cur->p, sizeof(double) * blocks[i].count, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

// ---- device-side sliding-window bookkeeping (hb200_window.cuh) -----------------------------------------------
namespace {
int check_device_window(hb200_ctx* c) {
  if (!c) return fail(-1, "null context");
  if (!c->bound) return fail(-2, "bind the window first (hb200_bind)");
  return 0;
}

// Appends n visual factors of one kind to the tail of the visual list and binds them there: meas = pixel [n][2] (kind 0)
// or bearing [n][3] (kind 1).  The counts advance only when every new factor binds and the tail keeps the bound order --
// on a sharded context on every rank or on none (round A of the agreement; n = 0 takes part).
int append_visual(hb200_ctx* c, int n, const double* stamp, const int* camera, const int* landmark, const double* meas, int kind) {
  HB_CUDA(cudaSetDevice(c->device));
  const size_t Nv = c->Nv;
  HB_CUDA(c->visual.grow(Nv + n, Nv, c->stream));
  HB_CUDA(c->d_invalid.ensure(2 + kAgreeOut));   // [bad index, arrival order | agreement]
  HB_CUDA(cudaMemsetAsync(c->d_invalid.p, 0, (2 + kAgreeOut) * sizeof(int), c->stream));
  int rc = 0;
  if (n) {
    if ((rc = upload_visual(c, static_cast<int>(Nv), n, stamp, camera, landmark, meas, kind))) return rc;
    if ((rc = bind_pixel_range(c, static_cast<int>(Nv), n))) return rc;
    tail_sorted_kernel<<<(n + 127) / 128, 128, 0, c->stream>>>(static_cast<int>(Nv), n, c->visual.idx.p, c->d_invalid.p + 1);
    HB_LAUNCH(c, "tail_sorted_kernel");
  }
  const int call = kind ? kCallBearing : kCallPixel;
  if (c->multi() && (rc = agree_round(c, vote_header(c, call), VoteSrc{c->d_invalid.p, {nullptr, nullptr, nullptr}, nullptr, nullptr}, c->d_invalid.p + 2))) return rc;
  int bad[2 + kAgreeOut] = {};
  HB_CUDA(cudaMemcpyAsync(bad, c->d_invalid.p, sizeof(bad), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  int own = 0;
  if (bad[0]) own = fail(2, "%d appended factor(s) reference a stamp outside the spline's valid range or an invalid camera / landmark", bad[0]);
  else if (bad[1]) own = fail(3, "appended factors must arrive in stamp order (%d fall before the end of the visual list): use hb200_set_%s_factors + hb200_bind", bad[1],
                              kind ? "bearing" : "pixel");
  if ((rc = window_outcome(c, bad + 2, own))) return rc;
  c->Nv = static_cast<int>(Nv) + n;
  (kind ? c->Nb : c->Np) += n;
  c->v_perm.clear(); c->i_perm.clear(); c->have_snapshot = false;
  return derive_window(c, call);
}

// n = 0 (with any pointers) is a valid collective call on a sharded context: the rank has nothing of its own this time
bool empty_collective(const hb200_ctx* c, int n) { return n == 0 && c->multi(); }
}  // namespace

int hb200_append_knots(hb200_ctx* c, int count) {
  int rc = check_device_window(c);
  if (rc) return rc;
  if (count <= 0) return fail(-1, "count must be positive");
  HB_CUDA(cudaSetDevice(c->device));
  for (DevBuf<double>& t : c->tab) HB_CUDA(t.ensure(static_cast<size_t>(c->K() + count) * kTabStride));
  if ((rc = c->pose.append(c, count))) return rc;
  c->h_knot_const.insert(c->h_knot_const.end(), count, 0);
  if ((rc = update_fixed(c))) return rc;
  if ((rc = ensure_system(c))) return rc;
  HB_CUDA(cudaStreamSynchronize(c->stream));
  c->kernel_args_changed(); c->have_snapshot = false;
  return 0;   // replicated: every rank appends the same knots, the agreed band half-width stays what it was
}

int hb200_append_bias_knots(hb200_ctx* c, double stamp, int* gyro_added, int* accel_added) {
  if (gyro_added) *gyro_added = 0;
  if (accel_added) *accel_added = 0;
  if (!c) return fail(-1, "null context");
  if (c->Kbg() == 0 || c->Kba() == 0) return fail(-2, "bias splines not set");
  int rc = check_device_window(c);
  if (rc) return rc;
  if (!std::isfinite(stamp)) return fail(-1, "stamp is not finite");
  int add[2] = {0, 0};
  Spline* bias[2] = {&c->gyro, &c->accel};
  for (int w = 0; w < 2; ++w) {
    rc = bias_append_count(*bias[w], stamp, &add[w]);
    if (rc == 2) return fail(2, "stamp %.17g lies before the %s bias spline's valid span (bias knots are never prepended)", stamp, w ? "accelerometer" : "gyroscope");
    if (rc) return fail(-1, "stamp %.17g needs more than %d new %s bias knots", stamp, HB200_BIAS_APPEND_MAX, w ? "accelerometer" : "gyroscope");
  }
  if (add[0] == 0 && add[1] == 0) return 0;
  HB_CUDA(cudaSetDevice(c->device));
  for (int w = 0; w < 2; ++w)   // both splines' copies, contents kept, before anything changes
    if ((rc = bias[w]->reserve(add[w], c->stream))) return rc;
  for (int w = 0; w < 2; ++w)
    if (add[w] && (rc = bias[w]->append(c, add[w]))) return rc;
  if (gyro_added) *gyro_added = add[0];
  if (accel_added) *accel_added = add[1];
  if ((rc = update_fixed(c))) return rc;
  if ((rc = ensure_system(c))) return rc;
  HB_CUDA(cudaStreamSynchronize(c->stream));
  c->kernel_args_changed(); c->have_snapshot = false;
  return 0;   // replicated, as hb200_append_knots
}

int hb200_bias_knots(hb200_ctx* c, int* num_gyro, int* num_accel, int* gyro_dropped, int* accel_dropped) {
  if (!c) return fail(-1, "null context");
  if (num_gyro) *num_gyro = c->Kbg();
  if (num_accel) *num_accel = c->Kba();
  if (gyro_dropped) *gyro_dropped = c->gyro.dropped;
  if (accel_dropped) *accel_dropped = c->accel.dropped;
  return 0;
}

int hb200_append_landmarks(hb200_ctx* c, int n, const double* xyz) {
  int rc = check_device_window(c);
  if (rc) return rc;
  if (n <= 0 || !xyz) return fail(-1, "invalid landmarks");
  HB_CUDA(cudaSetDevice(c->device));
  const size_t L = c->L;
  for (int s2 = 0; s2 < 2; ++s2) HB_CUDA(c->lms[s2].grow(3 * (L + n), s2 == 0 ? 3 * L : 0, c->stream));
  HB_CUDA(cudaMemcpyAsync(c->lms[0].p + 3 * L, xyz, sizeof(double) * 3 * n, cudaMemcpyHostToDevice, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  c->L = static_cast<int>(L) + n;
  c->v_perm.clear(); c->i_perm.clear(); c->have_snapshot = false;
  return derive_window(c);
}

int hb200_append_pixel_factors(hb200_ctx* c, int n, const double* stamp, const int* camera, const int* landmark, const double* pixel) {
  int rc = check_device_window(c);
  if (rc) return rc;
  if (!empty_collective(c, n) && (n <= 0 || !stamp || !camera || !landmark || !pixel)) return fail(-1, "invalid pixel factors");
  return append_visual(c, n, stamp, camera, landmark, pixel, 0);
}

int hb200_append_bearing_factors(hb200_ctx* c, int n, const double* stamp, const int* camera, const int* landmark, const double* bearing) {
  int rc = check_device_window(c);
  if (rc) return rc;
  if (!empty_collective(c, n) && (n <= 0 || !stamp || !camera || !landmark || !bearing)) return fail(-1, "invalid bearing factors");
  return append_visual(c, n, stamp, camera, landmark, bearing, 1);
}

int hb200_append_manifold_factors(hb200_ctx* c, int n, const double* stamp, const int* sensor, const double* pose) {
  int rc = check_device_window(c);
  if (rc) return rc;
  if (n <= 0 || !stamp || !sensor || !pose) return fail(-1, "invalid manifold factors");
  if (c->P == 0) return fail(-2, "pose sensors not set");
  HB_CUDA(cudaSetDevice(c->device));
  const size_t Nm = c->Nm;
  HB_CUDA(c->manifold.grow(Nm + n, Nm, c->stream));
  HB_CUDA(c->d_invalid.ensure(1));
  HB_CUDA(cudaMemsetAsync(c->d_invalid.p, 0, sizeof(int), c->stream));
  HB_CUDA(cudaMemcpyAsync(c->manifold.stamp.p + Nm, stamp, sizeof(double) * n, cudaMemcpyHostToDevice, c->stream));
  HB_CUDA(cudaMemcpyAsync(c->manifold.meas.p + 7 * Nm, pose, sizeof(double) * 7 * n, cudaMemcpyHostToDevice, c->stream));
  HB_CUDA(cudaMemcpyAsync(c->manifold.sensor.p + Nm, sensor, sizeof(int) * n, cudaMemcpyHostToDevice, c->stream));
  bind_manifold_kernel<<<(n + 127) / 128, 128, 0, c->stream>>>(n, c->manifold.stamp.p + Nm, c->manifold.sensor.p + Nm, c->pose.val[0].p, c->K(), c->k(), c->P, c->manifold.idx.p + Nm, c->d_invalid.p);
  HB_LAUNCH(c, "bind_manifold_kernel");
  int bad = 0;
  HB_CUDA(cudaMemcpyAsync(&bad, c->d_invalid.p, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  if (bad) return fail(2, "%d appended factor(s) reference a stamp outside the spline's valid range or an invalid pose sensor", bad);
  c->Nm = static_cast<int>(Nm) + n;
  c->v_perm.clear(); c->i_perm.clear(); c->have_snapshot = false;
  return derive_window(c);
}

int hb200_append_stereo_tracks(hb200_ctx* c, int n, const double* stamp, const int* camera0, const int* camera1, const double* pixel0,
                               const double* pixel1, const int* landmark, int* landmark_out, int* num_new) {
  int rc = check_device_window(c);
  if (rc) return rc;
  if (!empty_collective(c, n) && (n <= 0 || !stamp || !camera0 || !camera1 || !pixel0 || !pixel1 || !landmark)) return fail(-1, "invalid stereo tracks");
  if (c->C == 0) return fail(-2, "cameras not set");
  HB_CUDA(cudaSetDevice(c->device));
  const size_t N = n, Nv = c->Nv, L = c->L;
  // one upload each way: doubles [stamp | pixel0 | pixel1], ints [camera0 | camera1 | landmark | new flag]
  std::vector<double> hd(5 * N);
  std::vector<int> hi(4 * N);
  size_t fresh = 0;
  for (size_t f = 0; f < N; ++f) {
    hd[f] = stamp[f];
    hd[N + 2 * f] = pixel0[2 * f]; hd[N + 2 * f + 1] = pixel0[2 * f + 1];
    hd[3 * N + 2 * f] = pixel1[2 * f]; hd[3 * N + 2 * f + 1] = pixel1[2 * f + 1];
    hi[f] = camera0[f]; hi[N + f] = camera1[f]; hi[2 * N + f] = landmark[f]; hi[3 * N + f] = landmark[f] < 0;
    fresh += landmark[f] < 0;
  }
  HB_CUDA(c->visual.grow(Nv + 2 * N, Nv, c->stream));
  for (int s2 = 0; s2 < 2; ++s2) HB_CUDA(c->lms[s2].grow(3 * (L + fresh), s2 == 0 ? 3 * L : 0, c->stream));
  HB_CUDA(c->d_invalid.ensure(3 + kAgreeOut));   // [bad tracks, order violations, new landmarks | agreement]
  HB_CUDA(cudaMemsetAsync(c->d_invalid.p, 0, (3 + kAgreeOut) * sizeof(int), c->stream));
  if (n) {
    HB_CUDA(c->trk_d.ensure(5 * N)); HB_CUDA(c->trk_i.ensure(5 * N));
    HB_CUDA(cudaMemcpyAsync(c->trk_d.p, hd.data(), sizeof(double) * 5 * N, cudaMemcpyHostToDevice, c->stream));
    HB_CUDA(cudaMemcpyAsync(c->trk_i.p, hi.data(), sizeof(int) * 4 * N, cudaMemcpyHostToDevice, c->stream));
    const double* d_t = c->trk_d.p;
    const int* d_lm = c->trk_i.p + 2 * N;
    int* d_rank = c->trk_i.p + 4 * N;
    scan_kernel<<<1, 1024, 0, c->stream>>>(c->trk_i.p + 3 * N, n, d_rank, c->d_invalid.p + 2);
    HB_LAUNCH(c, "scan_kernel");
    prep_kernel<<<(c->K() + 63) / 64, 64, 0, c->stream>>>(c->K(), c->pose.val[0].p, c->tab[0].p, nullptr, 0);   // knot table of the current state
    HB_LAUNCH(c, "prep_kernel");
    rc = with_order(c->k(), [&](auto K) {
      stereo_track_kernel<K><<<(n + 127) / 128, 128, 0, c->stream>>>(n, d_t, c->trk_i.p, c->trk_i.p + N, d_t + N, d_t + 3 * N, d_lm, d_rank, c->pose.val[0].p, c->tab[0].p, c->K(),
                                                                    c->pose.basis, c->cams.p, c->C, static_cast<int>(L), static_cast<int>(Nv), c->visual.stamp.p, c->visual.pixel.p, c->visual.z.p,
                                                                    c->visual.idx.p, c->lms[0].p, c->d_invalid.p);
      return check_launch(c, "stereo_track_kernel");
    });
    if (rc) return rc;
    tail_sorted_kernel<<<(2 * n + 127) / 128, 128, 0, c->stream>>>(static_cast<int>(Nv), 2 * n, c->visual.idx.p, c->d_invalid.p + 1);
    HB_LAUNCH(c, "tail_sorted_kernel");
  }
  if (c->multi() && (rc = agree_round(c, vote_header(c, kCallStereo), VoteSrc{c->d_invalid.p, {nullptr, nullptr, nullptr}, nullptr, nullptr}, c->d_invalid.p + 3))) return rc;
  int h[3 + kAgreeOut] = {};   // bad tracks, order violations, new landmarks | agreement
  HB_CUDA(cudaMemcpyAsync(h, c->d_invalid.p, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  int own = 0;
  if (h[0]) own = fail(2, "%d stereo track(s) have a stamp outside the spline's valid range, an invalid camera / landmark or a non-finite triangulation", h[0]);
  else if (h[1]) own = fail(3, "stereo tracks must arrive in stamp order (%d fall before the end of the visual list)", h[1]);
  if ((rc = window_outcome(c, h + 3, own))) return rc;
  if (landmark_out)
    for (size_t f = 0, r = 0; f < N; ++f) landmark_out[f] = landmark[f] < 0 ? static_cast<int>(L + r++) : landmark[f];
  if (num_new) *num_new = h[2];
  c->Nv = static_cast<int>(Nv + 2 * N); c->Nb += 2 * n; c->L = static_cast<int>(L) + h[2];
  c->v_perm.clear(); c->i_perm.clear(); c->have_snapshot = false;
  return derive_window(c, kCallStereo);
}

int hb200_append_inertial_factors(hb200_ctx* c, int n, const double* stamp, const double* meas) {
  int rc = check_device_window(c);
  if (rc) return rc;
  if (n <= 0 || !stamp || !meas) return fail(-1, "invalid inertial factors");
  if (!c->have_imu || c->Kbg() == 0 || c->Kba() == 0) return fail(-2, "inertial factors need IMU calibration and bias splines");
  HB_CUDA(cudaSetDevice(c->device));
  const size_t Ni = c->Ni;
  HB_CUDA(c->inertial.grow(Ni + n, Ni, c->stream));
  HB_CUDA(c->d_invalid.ensure(2));
  HB_CUDA(cudaMemsetAsync(c->d_invalid.p, 0, 2 * sizeof(int), c->stream));
  HB_CUDA(cudaMemcpyAsync(c->inertial.stamp.p + Ni, stamp, sizeof(double) * n, cudaMemcpyHostToDevice, c->stream));
  HB_CUDA(cudaMemcpyAsync(c->inertial.meas.p + 6 * Ni, meas, sizeof(double) * 6 * n, cudaMemcpyHostToDevice, c->stream));
  if ((rc = bind_inertial_range(c, static_cast<int>(Ni), n))) return rc;
  tail_sorted_kernel<<<(n + 127) / 128, 128, 0, c->stream>>>(static_cast<int>(Ni), n, c->inertial.idx.p, c->d_invalid.p + 1);
  HB_LAUNCH(c, "tail_sorted_kernel");
  int bad[2] = {0, 0};
  HB_CUDA(cudaMemcpyAsync(bad, c->d_invalid.p, 2 * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  if (bad[0]) return fail(2, "%d appended factor(s) reference a stamp outside the state or bias splines' valid range", bad[0]);
  if (bad[1]) return fail(3, "appended factors must arrive in stamp order (%d fall before the end of the list): use hb200_set_inertial_factors + hb200_bind", bad[1]);
  c->Ni = static_cast<int>(Ni) + n;
  c->v_perm.clear(); c->i_perm.clear(); c->have_snapshot = false;
  return derive_window(c);
}

int hb200_slide(hb200_ctx* c, double lower_bound, int flags, hb200_slide_stats* stats) {
  int rc = check_device_window(c);
  if (rc) return rc;
  HB_CUDA(cudaSetDevice(c->device));
  const int Nv = c->Nv, Ni = c->Ni, Nm = c->Nm, L = c->L;
  const int ub = c->pose.upper(lower_bound);
  const int last_const = ub - 1;   // knots 0 .. last_const have stamp <= lower bound
  // leading bias knots go only with the inertial factors that reached them: without DROP_INERTIAL nothing is dropped
  const bool drop_bias = (flags & HB200_SLIDE_DROP_BIAS) && (flags & HB200_SLIDE_DROP_INERTIAL) && c->Kbg() && c->Kba();
  HB_CUDA(c->w_scal.ensure(10 + kAgreeOut));
  // [L_new, Nv_new, Ni_new, min base visual, min base inertial, Nm_new, min base manifold, kept bearing factors,
  //  min gyro bias base, min accel bias base (kept inertial factors) | agreement (sharded contexts)]
  int init[10 + kAgreeOut] = {0, 0, 0, 0x7fffffff, 0x7fffffff, 0, 0x7fffffff, 0, 0x7fffffff, 0x7fffffff};
  HB_CUDA(cudaMemcpyAsync(c->w_scal.p, init, sizeof(init), cudaMemcpyHostToDevice, c->stream));
  HB_CUDA(c->w_last.ensure(std::max(L, 1))); HB_CUDA(c->w_lkeep.ensure(std::max(L, 1) + 1)); HB_CUDA(c->w_lpos.ensure(std::max(L, 1) + 1));
  HB_CUDA(c->w_keep.ensure(std::max(std::max(Nv, Ni), 1))); HB_CUDA(c->w_pos.ensure(std::max(std::max(Nv, Ni), 1)));
  DevBuf<int> f_keep, f_pos;   // inertial [0, Ni), manifold [Ni, Ni + Nm)
  HB_CUDA(f_keep.ensure(std::max(Ni + Nm, 1))); HB_CUDA(f_pos.ensure(std::max(Ni + Nm, 1)));
  int* i_keep = f_keep.p; int* i_pos = f_pos.p; int* m_keep = f_keep.p + Ni; int* m_pos = f_pos.p + Ni;
  HB_CUDA(cudaMemsetAsync(c->w_last.p, 0, sizeof(unsigned long long) * std::max(L, 1), c->stream));
  if (Nv) { landmark_last_stamp_kernel<<<(Nv + 255) / 256, 256, 0, c->stream>>>(Nv, c->visual.stamp.p, c->visual.idx.p, c->w_last.p); HB_LAUNCH(c, "landmark_last_stamp_kernel"); }
  if (L) {
    landmark_keep_kernel<<<(L + 255) / 256, 256, 0, c->stream>>>(L, c->w_last.p, lower_bound, c->w_lkeep.p);
    HB_LAUNCH(c, "landmark_keep_kernel");
    scan_kernel<<<1, 1024, 0, c->stream>>>(c->w_lkeep.p, L, c->w_lpos.p, c->w_scal.p + 0);
    HB_LAUNCH(c, "scan_kernel");
  }
  if (Nv) {
    visual_keep_kernel<<<(Nv + 255) / 256, 256, 0, c->stream>>>(Nv, c->visual.idx.p, c->w_lkeep.p, c->w_keep.p, c->w_scal.p + 3, c->w_scal.p + 7);
    HB_LAUNCH(c, "visual_keep_kernel");
    scan_kernel<<<1, 1024, 0, c->stream>>>(c->w_keep.p, Nv, c->w_pos.p, c->w_scal.p + 1);
    HB_LAUNCH(c, "scan_kernel");
  }
  if (Ni) {
    inertial_keep_kernel<<<(Ni + 255) / 256, 256, 0, c->stream>>>(Ni, c->inertial.idx.p, c->k(), (flags & HB200_SLIDE_DROP_INERTIAL) ? last_const : -1, i_keep, c->w_scal.p + 4,
                                                                  drop_bias ? c->w_scal.p + 8 : nullptr);
    HB_LAUNCH(c, "inertial_keep_kernel");
    scan_kernel<<<1, 1024, 0, c->stream>>>(i_keep, Ni, i_pos, c->w_scal.p + 2);
    HB_LAUNCH(c, "scan_kernel");
  }
  if (Nm) {   // the reference never removes pose residuals either: same rule as the inertial ones, its own flag
    inertial_keep_kernel<<<(Nm + 255) / 256, 256, 0, c->stream>>>(Nm, c->manifold.idx.p, c->k(), (flags & HB200_SLIDE_DROP_MANIFOLD) ? last_const : -1, m_keep, c->w_scal.p + 6);
    HB_LAUNCH(c, "manifold_keep_kernel");
    scan_kernel<<<1, 1024, 0, c->stream>>>(m_keep, Nm, m_pos, c->w_scal.p + 5);
    HB_LAUNCH(c, "scan_kernel");
  }
  // sharded: round A of the agreement -- the smallest kept knot and bias bases over the ranks, before anything moves
  if (c->multi()) {
    int* w = c->w_scal.p;
    rc = agree_round(c, vote_header(c, kCallSlide, flags, ub, c->gyro.upper(lower_bound), c->accel.upper(lower_bound)),
                     VoteSrc{nullptr, {w + 3, w + 4, w + 6}, drop_bias ? w + 8 : nullptr, nullptr}, w + 10);
    if (rc) return rc;
  }
  int h[10 + kAgreeOut];
  HB_CUDA(cudaMemcpyAsync(h, c->w_scal.p, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  if ((rc = window_outcome(c, h + 10, 0))) {
    c->slide_L = -1;   // (the keep flags of this attempt replaced the last slide's landmark map)
    return rc;
  }
  const int L_new = L ? h[0] : 0, Nv_new = Nv ? h[1] : 0, Ni_new = Ni ? h[2] : 0, Nm_new = Nm ? h[5] : 0, Nb_new = Nv ? h[7] : 0;
  const int knot_min = c->multi() ? h[10 + kAgreeKnotMin] : std::min(h[6], std::min(h[3], h[4]));
  const int gyro_min = c->multi() ? h[10 + kAgreeGyroMin] : h[8], accel_min = c->multi() ? h[10 + kAgreeAccelMin] : h[9];
  // leading knots go once no kept factor touches them (the smallest bases of the kept factors)
  const int shift = c->pose.drop_count(lower_bound, knot_min);
  const int g_shift = drop_bias ? c->gyro.drop_count(lower_bound, gyro_min) : 0, a_shift = drop_bias ? c->accel.drop_count(lower_bound, accel_min) : 0;
  // compaction of the factor lists into their spare copies and of the state into its trial copy, each then switched in
  if (Nv && (rc = compact_visual(c, Nv, c->w_keep.p, c->w_pos.p, c->w_lpos.p, shift, Nv_new))) return rc;
  if (Ni && (rc = compact_inertial(c, Ni, i_keep, i_pos, shift, g_shift, a_shift, Ni_new))) return rc;
  if (Nm && (rc = compact_manifold(c, Nm, m_keep, m_pos, shift, Nm_new))) return rc;
  c->kernel_args_changed();   // (the state switches below move buffers the captured iteration points at)
  if (L) {
    compact_landmarks_kernel<<<(L + 255) / 256, 256, 0, c->stream>>>(L, c->w_lkeep.p, c->w_lpos.p, c->lms[0].p, c->lms[1].p);
    HB_LAUNCH(c, "compact_landmarks_kernel");
    c->lms[0].swap(c->lms[1]);
  }
  if ((rc = c->pose.shift(c, shift)) || (rc = c->gyro.shift(c, g_shift)) || (rc = c->accel.shift(c, a_shift))) return rc;
  HB_CUDA(cudaStreamSynchronize(c->stream));
  // host bookkeeping: constancy (elements at or before the lower bound: reference optimizer.cpp:322-328; gravity once
  // the window no longer covers the whole state range: reference abstract.cpp:57-61) and sizes
  c->h_knot_const.assign(c->K(), 0);
  for (int j = 0; j < c->K(); ++j) c->h_knot_const[j] = c->pose.stamp[j] <= lower_bound ? 1 : 0;
  if (ub > 0) c->gravity_const = 1;
  c->L = L_new; c->Nv = Nv_new; c->Np = Nv_new - Nb_new; c->Nb = Nb_new; c->Ni = Ni_new; c->Nm = Nm_new;
  c->slide_L = L;
  if (stats) {
    stats->knots_dropped = shift; stats->knots_constant = std::max(0, ub - shift); stats->landmarks_dropped = L - L_new;
    stats->visual_factors_dropped = Nv - Nv_new; stats->inertial_factors_dropped = Ni - Ni_new;
    stats->knots = c->K(); stats->landmarks = L_new; stats->visual_factors = Nv_new; stats->inertial_factors = Ni_new;
  }
  c->v_perm.clear(); c->i_perm.clear(); c->have_snapshot = false;
  return derive_window(c, kCallSlide);
}

int hb200_window_sizes(hb200_ctx* c, int* knots, int* landmarks, int* visual_factors, int* inertial_factors) {
  if (!c) return fail(-1, "null context");
  if (knots) *knots = c->K();
  if (landmarks) *landmarks = c->L;
  if (visual_factors) *visual_factors = c->Nv;
  if (inertial_factors) *inertial_factors = c->Ni;
  return 0;
}

int hb200_factor_counts(hb200_ctx* c, int* counts) {
  if (!c || !counts) return fail(-1, "null argument");
  counts[HB200_PIXEL] = c->Np; counts[HB200_INERTIAL] = c->Ni; counts[HB200_BEARING] = c->Nb; counts[HB200_MANIFOLD] = c->Nm;
  return 0;
}

int hb200_slide_landmark_map(hb200_ctx* c, int n, int* new_index) {
  if (!c) return fail(-1, "null context");
  if (c->slide_L < 0) return fail(-2, "no hb200_slide yet");
  if (n != c->slide_L || (n > 0 && !new_index)) return fail(-1, "the last hb200_slide started from %d landmarks, not %d", c->slide_L, n);
  if (n == 0) return 0;
  HB_CUDA(cudaSetDevice(c->device));
  std::vector<int> keep(n);
  HB_CUDA(cudaMemcpyAsync(keep.data(), c->w_lkeep.p, sizeof(int) * n, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaMemcpyAsync(new_index, c->w_lpos.p, sizeof(int) * n, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  for (int l = 0; l < n; ++l) if (!keep[l]) new_index[l] = -1;
  return 0;
}

int hb200_set_allreduce(hb200_ctx* c, hb200_allreduce_fn fn, void* user) {
  if (!c) return fail(-1, "null context");
  if (fn && c->nccl) return fail(-2, "a NCCL communicator is attached; the callback hook is its replacement, not an addition");
  const bool detach = !fn && c->allreduce;
  c->allreduce = fn; c->allreduce_user = user;
  c->iterations_changed();
  return detach ? forget_agreement(c) : 0;
}

int hb200_comm_unique_id(char* id) {
  if (!id) return fail(-1, "null argument");
  int rc = load_nccl();
  if (rc) return rc;
  NcclUid u;
  HB_NCCL(g_nccl.GetUniqueId(&u));
  std::memcpy(id, u.internal, sizeof(u.internal));
  return 0;
}

int hb200_set_nccl_comm(hb200_ctx* c, void* comm, int nranks, int rank) {
  if (!c) return fail(-1, "null context");
  if (comm && (nranks < 1 || nranks > kMaxRanks || rank < 0 || rank >= nranks)) return fail(-1, "invalid rank %d of %d (at most %d ranks)", rank, nranks, kMaxRanks);
  if (comm && c->allreduce) return fail(-2, "the all-reduce callback hook is set; clear it first");
  if (comm) { int rc = load_nccl(); if (rc) return rc; }
  HB_CUDA(cudaSetDevice(c->device));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  for (IterationGraph& g : c->graphs) g.release();   // they reference the old communicator
  if (c->nccl && c->own_nccl) g_nccl.CommDestroy(c->nccl);
  c->nccl = comm; c->own_nccl = false;
  c->nranks = comm ? nranks : 1; c->rank = comm ? rank : 0;
  c->comm_warm = false;
  const int rc = forget_agreement(c);   // a new communicator agrees afresh; none leaves a single context
  return rc ? rc : sync_layout(c);
}

int hb200_comm_init_rank(hb200_ctx* c, int nranks, int rank, const char* id) {
  if (!c || !id) return fail(-1, "null argument");
  if (nranks < 1 || nranks > kMaxRanks || rank < 0 || rank >= nranks) return fail(-1, "invalid rank %d of %d (at most %d ranks)", rank, nranks, kMaxRanks);
  int rc = load_nccl();
  if (rc) return rc;
  HB_CUDA(cudaSetDevice(c->device));
  NcclUid u;
  std::memcpy(u.internal, id, sizeof(u.internal));
  void* comm = nullptr;
  HB_NCCL(g_nccl.CommInitRank(&comm, nranks, u, rank));
  rc = hb200_set_nccl_comm(c, comm, nranks, rank);
  if (rc) { g_nccl.CommDestroy(comm); return rc; }
  c->own_nccl = true;
  return 0;
}

int hb200_peer_handle(hb200_ctx* c, char* handle) {
  if (!c || !handle) return fail(-1, "null argument");
  HB_CUDA(cudaSetDevice(c->device));
  // the arena: mailbox + flag row + two partial-system halves (capacity HB200_PEER_ARENA_DOUBLES each, default 600 k doubles =
  // 4.8 MB: a K = 1000 window; larger systems fall back to ncclAllReduce)
  const long long cap = getenv("HB200_PEER_ARENA_DOUBLES") ? std::max(0LL, atoll(getenv("HB200_PEER_ARENA_DOUBLES"))) & ~1LL : 600000LL;
  const size_t arena = static_cast<size_t>(kArenaParts) + 2 * static_cast<size_t>(cap);
  HB_CUDA(c->mbox.ensure(arena));
  c->arena_cap = cap;
  HB_CUDA(c->mbox_seq.ensure(1)); HB_CUDA(c->red_round.ensure(1)); HB_CUDA(c->red_arrive.ensure(1));
  HB_CUDA(cudaMemsetAsync(c->mbox.p, 0, sizeof(double) * kArenaParts, c->stream));
  HB_CUDA(cudaMemsetAsync(c->mbox_seq.p, 0, sizeof(unsigned long long), c->stream));
  HB_CUDA(cudaMemsetAsync(c->red_round.p, 0, sizeof(unsigned long long), c->stream));
  HB_CUDA(cudaMemsetAsync(c->red_arrive.p, 0, sizeof(unsigned int), c->stream));
  c->peer_par = 0;
  c->peer_reduce_wanted = !(getenv("HB200_PEER_REDUCE") && atoi(getenv("HB200_PEER_REDUCE")) == 0);
  HB_CUDA(cudaStreamSynchronize(c->stream));
  cudaIpcMemHandle_t h;
  HB_CUDA(cudaIpcGetMemHandle(&h, c->mbox.p));
  static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
  std::memcpy(handle, &h, sizeof(h));
  return 0;
}

namespace {
void close_peers(hb200_ctx* c) {
  for (size_t p = 0; p < c->peer_ptrs.size(); ++p)
    if (c->peer_ptrs[p] && c->peer_ptrs[p] != c->mbox.p) cudaIpcCloseMemHandle(c->peer_ptrs[p]);
  c->peer_ptrs.clear();
  c->peers_open = false;
}
}  // namespace

int hb200_peer_connect(hb200_ctx* c, int nranks, int rank, const char* handles) {
  if (!c || !handles) return fail(-1, "null argument");
  if (!c->nccl || nranks != c->nranks || rank != c->rank) return fail(-2, "attach the communicator first (same nranks / rank)");
  if (!c->mbox.p) return fail(-2, "call hb200_peer_handle first");
  HB_CUDA(cudaSetDevice(c->device));
  close_peers(c);
  c->peer_ptrs.assign(nranks, nullptr);
  for (int p = 0; p < nranks; ++p) {
    if (p == rank) { c->peer_ptrs[p] = c->mbox.p; continue; }
    cudaIpcMemHandle_t h;
    std::memcpy(&h, handles + 64 * static_cast<size_t>(p), sizeof(h));
    void* ptr = nullptr;
    const cudaError_t e = cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      cudaGetLastError();
      close_peers(c);
      return fail(100 + static_cast<int>(e), "cudaIpcOpenMemHandle(rank %d): %s (the scalar exchange falls back to a second ncclAllReduce)", p, cudaGetErrorString(e));
    }
    c->peer_ptrs[p] = ptr;
  }
  HB_CUDA(c->d_peers.ensure(kMaxRanks));
  std::vector<double*> host(kMaxRanks, nullptr);
  for (int p = 0; p < nranks; ++p) host[p] = static_cast<double*>(c->peer_ptrs[p]);
  HB_CUDA(cudaMemcpyAsync(c->d_peers.p, host.data(), sizeof(double*) * kMaxRanks, cudaMemcpyHostToDevice, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  c->peers_open = true;
  c->iterations_changed();
  return 0;
}

int hb200_set_min_bandwidth(hb200_ctx* c, int beta) {
  if (!c || beta < 0) return fail(-1, "invalid argument");
  HB_CUDA(cudaSetDevice(c->device));
  c->min_beta = beta;
  if (c->bound) {
    HB_CUDA(cudaStreamSynchronize(c->stream));
    const int rc = ensure_system(c);
    if (rc) return rc;
    c->kernel_args_changed();
  }
  return 0;
}

int hb200_set_deterministic(hb200_ctx* c, int enable) {
  if (!c) return fail(-1, "null context");
  const bool on = enable != 0;
  if (on == c->deterministic) return 0;
  c->deterministic = on;
  c->kernel_args_changed();
  return 0;
}

int hb200_get_deterministic(hb200_ctx* c, int* enable) {
  if (!c || !enable) return fail(-1, "invalid argument");
  *enable = c->deterministic ? 1 : 0;
  return 0;
}

int hb200_get_bandwidth(hb200_ctx* c, int* beta) {
  if (!c || !beta) return fail(-1, "null argument");
  if (!c->bound) return fail(-2, "not bound");
  *beta = c->beta;
  return 0;
}

int hb200_peer_disconnect(hb200_ctx* c) {
  if (!c) return fail(-1, "null context");
  HB_CUDA(cudaSetDevice(c->device));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  close_peers(c);
  c->iterations_changed();
  return 0;
}

int hb200_comm_info(hb200_ctx* c, int* nranks, int* rank, int* nccl, int* peer_mailbox, int* graph, long long* payload_doubles) {
  if (!c) return fail(-1, "null context");
  if (nranks) *nranks = c->nranks;
  if (rank) *rank = c->rank;
  if (nccl) *nccl = c->nccl ? 1 : 0;
  if (peer_mailbox) *peer_mailbox = (c->nccl && c->peers_open) ? (c->peer_reduce() ? 2 : 1) : 0;   // 2: the system reduction runs over peer memory too
  if (graph) *graph = (c->use_graph && !c->allreduce && c->graphs[0].valid) ? 1 : 0;
  if (payload_doubles) *payload_doubles = c->bound ? c->lay.total : 0;
  return 0;
}

void* hb200_system_device_ptr(hb200_ctx* c, long long* count) {
  if (!c) return nullptr;
  if (count) *count = c->lay.total;
  return c->sys.p;
}

}  // extern "C"
