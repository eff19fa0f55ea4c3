/* hyperb200.h -- C-ABI of the H100-native HyperSLAM hot path (libhyperb200.so).
 *
 * Drop-in boundary (SURVEY.md section 8b): one context owns the flattened sliding window that the
 * reference's optimizer holds as a pointer graph, and runs what ceres::Solve runs per iteration --
 * every residual block's Evaluate(), the normal equations and the linear solve -- as batched sm_90a
 * kernels.  All pointers are plain host pointers unless a name says "device"; buffers are copied in
 * or out, never aliased across calls.  Every function returns 0 on success, <0 for an invalid
 * argument, >0 for a CUDA / numerical failure; hb200_last_error_string() describes the last one.
 * (The reference aborts through glog CHECKs and Evaluate() always returns true,
 * reference internal/hyper/optimizers/ceres/costs/exteroceptive.cpp:159,162-178.)
 * A context is not thread-safe (the reference runs everything optimiser-side on one backend thread,
 * reference internal/hyper/system/components/backend.cpp:124-158).
 */
#ifndef HYPERB200_H_
#define HYPERB200_H_

#ifdef __cplusplus
extern "C" {
#endif

typedef struct hb200_ctx hb200_ctx;

typedef struct hb200_options {
  int device;        /* CUDA device ordinal */
  void* stream;      /* cudaStream_t to run on; NULL => the context creates its own */
  int use_graph;     /* capture hb200_iterate() in a CUDA graph (1) or launch kernels directly (0) */
  int reserved;      /* bit 0: force the dense cooperative Cholesky instead of the banded-arrow solver */
  void* nccl_comm;   /* ncclComm_t spanning the ranks that share this window, or NULL (single GPU); not owned */
  int nranks, rank;  /* size of / position in that communicator (ignored when nccl_comm is NULL) */
} hb200_options;

/* Per-iteration record, the analogue of ceres::IterationSummary printed through
 * summary.BriefReport() (reference internal/hyper/optimizers/ceres/optimizer.cpp:279). */
typedef struct hb200_iteration {
  double cost;          /* 1/2 sum rho(|r|^2) at the linearisation point */
  double cost_new;      /* cost at the trial point */
  double model_change;  /* predicted decrease of the quadratic model */
  double rho;           /* (cost - cost_new) / model_change */
  double radius;        /* trust-region radius after the update */
  int accepted;         /* step accepted */
  int spd;              /* reduced system was positive definite */
} hb200_iteration;

enum { HB200_PIXEL = 0, HB200_INERTIAL = 1, HB200_BEARING = 2, HB200_MANIFOLD = 3 };
enum { HB200_EVAL_JACOBIANS = 1, HB200_EVAL_TRIAL = 2 };

int hb200_create(const hb200_options* options, hb200_ctx** out);
void hb200_destroy(hb200_ctx* ctx);
const char* hb200_last_error_string(void);
int hb200_synchronize(hb200_ctx* ctx);

/* ---- window state: replaces the parameter blocks Ceres aliases ------------------------------
 * knots  [K][8] = Stamped<SE3> blocks [qx qy qz qw px py pz | stamp] ordered by stamp
 *         (reference optimizer.cpp:287-305 AddParameterBlock per state element; storage order
 *         reference settings.yaml:34-36, stamped.hpp:35-36).  order = layout().outer.size.      */
/* Knots must be UNIFORMLY spaced (relative tolerance 1e-6; the reference only creates uniform knots,
 * abstract.cpp:89,128), likewise the bias knots.  RE-BIND RULE: the index maps of hb200_bind follow from the
 * stamps, so changing the order, the number of knots OR ANY STAMP (a window slid by one knot keeps K) unbinds the
 * factor lists -- call hb200_bind again; hb200_optimize rejects blocks whose stamps differ from the bound window. */
int hb200_set_spline(hb200_ctx* ctx, int order, int num_knots, const double* knots);
/* bias control points [Kb][4] = Stamped<R3> [bx by bz | stamp] (reference imu.cpp:64-80). */
int hb200_set_bias_splines(hb200_ctx* ctx, int order, int num_gyro, const double* gyro, int num_accel, const double* accel);
/* gravity parameter block, 3 doubles on the sphere (reference optimizer.cpp:104). */
int hb200_set_gravity(hb200_ctx* ctx, const double* gravity);
/* cameras [C][15] = T_bs(7) | intrinsics cx cy fx fy | radtan k1 k2 p1 p2
 * (Sensor::parameters order, reference pixel.cpp:43-45). */
int hb200_set_cameras(hb200_ctx* ctx, int num_cameras, const double* cameras);
/* IMU static blocks (37) = T_bs(7) | i_g(6) | i_a(6) | S_g(9) | X_a(9) (reference inertial.cpp:35-39,45-49). */
int hb200_set_imu(hb200_ctx* ctx, const double* imu);
/* landmark position blocks [L][3] (reference optimizer.cpp:347-358). */
int hb200_set_landmarks(hb200_ctx* ctx, int num_landmarks, const double* xyz);
/* constancy: SetParameterBlockConstant on state elements (reference optimizer.cpp:322-328),
 * setGravityConstant (reference abstract.cpp:57-61), bias manifolds (reference optimizer.cpp:62-63). */
int hb200_set_constant(hb200_ctx* ctx, const unsigned char* knot_constant, int gravity_constant, int bias_constant);
/* losses: HuberLoss(huber_pixel) (reference optimizer.cpp:226), ScaledLoss(NULL, imu_loss_scale)
 * (:267-268); radius = initial trust-region radius (Ceres default 1e4). */
int hb200_set_options(hb200_ctx* ctx, double huber_pixel, double imu_loss_scale, double radius);
/* Family weight matrix: the weights branch of ExteroceptiveCost::Evaluate (reference exteroceptive.cpp:101-160), set in
 * place of CostConfiguration::weights (:162-178), one matrix per family as the reference's per-family configuration
 * (optimizer.cpp:191,214,236,255).  Wf is row-major d x d: d = 2 for HB200_PIXEL, 1 for HB200_BEARING (the one angular
 * row), 6 for HB200_INERTIAL (rows gyro | accel) and HB200_MANIFOLD (rows [theta | p]); any finite matrix is accepted (it
 * need not be triangular or positive definite; a singular one shows up as a failed covariance or a damped LM step).
 * NULL clears the family's matrix, which is the default (the reference's weights = nullptr): without a matrix every
 * output is what it is without this call, bit for bit.  With one, each factor of the family has residual Wf r and every
 * Jacobian block Wf J; the loss sees the weighted residual (Huber on |Wf r|^2, ScaledLoss times |Wf r|^2), and the cost,
 * J^T J, the Schur complement, the LM step and the covariances all follow from the weighted r and J.  So the copy-outs
 * (hb200_get_*_outputs, hb200_factor_evaluate, calibration blocks included) return weighted residuals and Jacobians --
 * except the inertial wg / wa outputs, which stay the bias splines' basis weights: with a matrix set the bias Jacobian
 * of gyro knot m is wg[m] Wf[:, 0:3] and that of accel knot m is wa[m] Wf[:, 3:6] (without one, wg[m] [I3 ; 0] and
 * wa[m] [0 ; I3]).  Returns -1 for an unknown kind or a non-finite entry (nothing changes).  Setting the value a family
 * already has changes nothing; a change drops a built system and a pending covariance build (-2 until rebuilt), like
 * every setter, and the next iteration is captured again with the new matrix. */
int hb200_set_weights(hb200_ctx* ctx, int kind, const double* Wf);

/* HYPER_REFERENCE_QUIRKS (SURVEY.md section 8a): 0 (default) = the mathematically consistent inertial Jacobians;
 * bits switch on the in-tree formulas verbatim -- 1: gyroscope intrinsics in the accelerometer rows (reference
 * inertial.cpp:136,142,148,158), 2: no Jacobian of the S_g a_b_m term (:135,147), 4: extrinsics block without R_sb
 * (:157-158), 8: X_a ignored in the rate / acceleration coefficients (:142,148); 15 = the reference as written.
 * All variants coincide on the calibration every reference fixture uses (I_g = I_a = I, S_g = X_a = 0, R_bs = I). */
int hb200_set_reference_quirks(hb200_ctx* ctx, int quirks);

/* ---- factor lists: replace problem_.AddResidualBlock (reference optimizer.cpp:212-232,253-274).  The lists live on
 * the device only.  Each setter writes its family there in the given (user) order, replacing that family whatever
 * appends or slides did to it, keeps the other families as they stand and unbinds the window; the copy-out calls and
 * hb200_get_index_maps number each family's factors in user order. */
int hb200_set_pixel_factors(hb200_ctx* ctx, int n, const double* stamp, const int* camera, const int* landmark, const double* pixel);
int hb200_set_inertial_factors(hb200_ctx* ctx, int n, const double* stamp, const double* measurement /* [n][6] gyro|accel */);
/* VisualBearingObservation -> AngularMetric residual behind HuberLoss(1.6e-3) (reference
 * optimizer.cpp:189-210, evaluators/bearing.cpp:14-79); bearing = [n][3] direction in the sensor frame
 * (any positive length).  Same parameter blocks as a pixel factor. */
int hb200_set_bearing_factors(hb200_ctx* ctx, int n, const double* stamp, const int* camera, const int* landmark, const double* bearing);
int hb200_set_bearing_loss(hb200_ctx* ctx, double huber_bearing);
/* ManifoldObservation<SE3> -> ManifoldMetric residual, no loss (reference optimizer.cpp:234-251,
 * evaluators/manifold.cpp:12-61).  Pose sensors carry only T_bs [q(4) p(3)] (plain Sensor, reference
 * manifold.cpp:30); pose = [n][7] measured T_ws. */
int hb200_set_pose_sensors(hb200_ctx* ctx, int num_sensors, const double* T_bs /* [P][7] */);
int hb200_set_manifold_factors(hb200_ctx* ctx, int n, const double* stamp, const int* sensor, const double* pose /* [n][7] */);
/* ExteroceptiveCost::update() for every factor (reference exteroceptive.cpp:25-99): resolves the
 * knot base index of each stamp and the segment / landmark incidence lists.  num_invalid receives
 * the number of factors whose stamp or indices fall outside the window (they are an error).  The lists are
 * bound where they stand and put into bound order on the device by a stable sort: visual factors by knot base, inertial
 * factors by knot, gyro and accel bias base; manifold factors keep their order. */
int hb200_bind(hb200_ctx* ctx, int* num_invalid);
int hb200_get_index_maps(hb200_ctx* ctx, int* pixel_base, int* inertial_base, int* gyro_bias_base, int* accel_bias_base);

/* ---- sliding-window bookkeeping on the device (SURVEY.md section 8f rank 3) ---------------------------------
 * What the reference does per message on its pointer graph, applied to the flattened window that already lives in
 * HBM -- no host re-sort, no re-upload of the factor lists (all four families).  After any of these calls the user
 * order of each family is its bound order on the device: the visual list holds pixel and bearing factors together in
 * bound order, and the copy-out calls number the pixel factors 0 .. Np-1 and the bearing factors 0 .. Nb-1 in that order.
 * A later hb200_bind without a setter in between keeps that numbering and the list order of factors with equal keys.
 *   hb200_append_knots:    `count` state elements appended by the reference's extrapolation -- the new elements AND
 *                          the current last one take the variable of the second to last, stamps continue at the knot
 *                          separation (reference internal/hyper/optimizers/abstract.cpp:126-136).
 *   hb200_append_*:        a frame's residual blocks / new landmarks (reference optimizer.cpp:189-274,347-358).
 *                          Pixel, bearing and stereo-track stamps must not precede the end of the visual list, inertial
 *                          stamps the end of the inertial list (arrival order; else 3); manifold factors have no order
 *                          rule (their list is not sorted, hb200_bind keeps it as given).  The new factors are bound on
 *                          the device (index maps of the tail only); a bad stamp / camera / landmark / sensor index
 *                          returns 2.  A failed call leaves sizes, landmarks and factor lists as they were.
 *   hb200_append_stereo_tracks: process(VisualTracks) on the device (reference abstract.cpp:243-260).  Track i ->
 *                          bearings b0, b1 (convertPixelsToBearings); landmark[i] >= 0: an existing window landmark,
 *                          < 0: a new landmark triangulated at the current state (Camera::Triangulate + T_w0.vectorPlus,
 *                          as hb200_ingest_stereo, bit for bit) and appended in track order; then bearing factors
 *                          (stamp[i], camera0[i]) and (stamp[i], camera1[i]) at visual list positions Nv + 2i and
 *                          Nv + 2i + 1 (add(observation_0); add(observation_1)).  A new track whose triangulation is not
 *                          finite (parallel rays) is a bad track (2).  landmark_out [n] (may be NULL): each track's
 *                          landmark index after the call; num_new (may be NULL): landmarks added.
 *   hb200_slide:           new window lower bound -- landmarks whose observation range left the window are removed
 *                          with their pixel and bearing residuals (optimizer.cpp:360-382), state elements at or before
 *                          the bound become constant (:322-328), the ones in front of the window that no residual
 *                          touches are removed (:331-341), gravity becomes constant (abstract.cpp:57-61).  The reference
 *                          never removes inertial or pose residuals; HB200_SLIDE_DROP_INERTIAL / _MANIFOLD additionally
 *                          drop the inertial / manifold factors whose control points are all at or before the bound, so
 *                          that the window stays bounded.  visual_factors in the stats counts pixel + bearing factors.
 *                          HB200_SLIDE_DROP_BIAS applies the removal rule (:331-341) to each bias spline as well: with
 *                          ub = number of bias stamps <= lower_bound, the leading min(max(0, ub - 1 - (kb-1)/2), smallest
 *                          gyro (accel) bias base of the inertial factors this slide keeps) knots go, at least kb stay,
 *                          and the kept factors' bias bases are remapped.  It only acts together with
 *                          HB200_SLIDE_DROP_INERTIAL (the inertial factors are what holds the leading bias knots).
 *   hb200_append_bias_knots: the reference's updateSensor (abstract.cpp:272-292) for a stamp past the bias splines:
 *                          each spline independently gets the fewest knots that put `stamp` inside its valid span (the
 *                          span hb200_bind and hb200_append_inertial_factors accept), by the hb200_append_knots rule --
 *                          the new knots AND the current last one take the value of the second to last, stamps continue
 *                          at the spline's own separation (new stamp i = fma(i + 1, dt, last stamp)).  A convention of
 *                          this library: the reference leaves updateSensor unimplemented.  A stamp already inside
 *                          appends nothing.  gyro_added / accel_added (may be NULL): knots appended.  Returns -1 for a
 *                          non-finite stamp or one that needs more than HB200_BIAS_APPEND_MAX knots on a spline, -2
 *                          without bias splines or a bound window, 2 for a stamp before a spline's valid span (knots
 *                          are never prepended); a failed call changes nothing.
 *   hb200_bias_knots:      current gyro / accel bias knot counts and the leading knots the last hb200_slide removed
 *                          from each (a caller drops as many leading elements from its own copy); any may be NULL.
 *   hb200_slide_landmark_map: old -> new landmark index across the last hb200_slide (-1: dropped); n = number of
 *                          landmarks before that slide.  With landmark_out it keeps a caller's id -> slot map.
 *   hb200_factor_counts:   factor counts per family, indexed by HB200_PIXEL / _INERTIAL / _BEARING / _MANIFOLD.
 * On a sharded context (a communicator or the all-reduce hook attached) these calls fall into three classes, see the
 * SHARDING CONTRACT below: hb200_append_pixel_factors / _bearing_factors / _stereo_tracks and hb200_slide are
 * collective (n = 0 accepted), hb200_append_knots / hb200_append_bias_knots replicated, hb200_append_landmarks /
 * _inertial_factors / _manifold_factors rank-local. */
typedef struct hb200_slide_stats {
  int knots_dropped, knots_constant, landmarks_dropped, visual_factors_dropped, inertial_factors_dropped;
  int knots, landmarks, visual_factors, inertial_factors;   /* sizes after the call */
} hb200_slide_stats;
enum { HB200_SLIDE_DROP_INERTIAL = 1, HB200_SLIDE_DROP_MANIFOLD = 2, HB200_SLIDE_DROP_BIAS = 4 };
enum { HB200_BIAS_APPEND_MAX = 1024 };   /* knots one hb200_append_bias_knots call may add to one spline */
int hb200_append_knots(hb200_ctx* ctx, int count);
int hb200_append_bias_knots(hb200_ctx* ctx, double stamp, int* gyro_added, int* accel_added);
int hb200_bias_knots(hb200_ctx* ctx, int* num_gyro, int* num_accel, int* gyro_dropped, int* accel_dropped);
int hb200_append_landmarks(hb200_ctx* ctx, int n, const double* xyz);
int hb200_append_pixel_factors(hb200_ctx* ctx, int n, const double* stamp, const int* camera, const int* landmark, const double* pixel);
int hb200_append_inertial_factors(hb200_ctx* ctx, int n, const double* stamp, const double* measurement);
int hb200_append_bearing_factors(hb200_ctx* ctx, int n, const double* stamp, const int* camera, const int* landmark, const double* bearing /* [n][3] */);
int hb200_append_manifold_factors(hb200_ctx* ctx, int n, const double* stamp, const int* sensor, const double* pose /* [n][7] */);
int hb200_append_stereo_tracks(hb200_ctx* ctx, int n, const double* stamp, const int* camera0, const int* camera1, const double* pixel0 /* [n][2] */,
                               const double* pixel1 /* [n][2] */, const int* landmark, int* landmark_out, int* num_new);
int hb200_slide(hb200_ctx* ctx, double lower_bound, int flags, hb200_slide_stats* stats /* may be NULL */);
int hb200_slide_landmark_map(hb200_ctx* ctx, int n, int* new_index);
int hb200_window_sizes(hb200_ctx* ctx, int* knots, int* landmarks, int* visual_factors, int* inertial_factors);
int hb200_factor_counts(hb200_ctx* ctx, int* counts /* [4] */);

/* ---- the hot path --------------------------------------------------------------------------
 * hb200_evaluate: residual (+ Jacobian) of every factor at the current state (flags 0 / JACOBIANS)
 * or at the trial state (TRIAL).  Compact outputs (DESIGN.md "HBM layout"):
 *   pixel   : r[n][2], Jp[n][2][6k], Jl[n][2][3]
 *   inertial: r[n][6], Jp[n][6][6k], wg[n][kb], wa[n][kb], Jg[n][6][2]                       */
int hb200_evaluate(hb200_ctx* ctx, int flags);
int hb200_get_pixel_outputs(hb200_ctx* ctx, double* r, double* Jp, double* Jl);
int hb200_get_inertial_outputs(hb200_ctx* ctx, double* r, double* Jp, double* wg, double* wa, double* Jg);
/*   bearing : r[n], Jp[n][6k], Jl[n][3]            manifold: r[n][6], Jp[n][6][6k]             */
int hb200_get_bearing_outputs(hb200_ctx* ctx, double* r, double* Jp, double* Jl);
int hb200_get_manifold_outputs(hb200_ctx* ctx, double* r, double* Jp);
/* Ceres-shaped copy-out of one factor after hb200_evaluate(JACOBIANS): same signature, block order
 * and row-major ambient Jacobians as ExteroceptiveCost::Evaluate (reference exteroceptive.hpp:31,
 * exteroceptive.cpp:149-156), weighted by the family's matrix when one is set (hb200_set_weights).  parameters must be the blocks the window was uploaded from.  Every block is served,
 * the calibration blocks too (extrinsics, intrinsics, distortion; i_g, i_a, S_g, X_a -- reference pixel.cpp:91-135,141,
 * inertial.cpp:155-194): they are constant in the live configuration (optimizer.cpp:59-63), so their Jacobians are
 * computed by separate kernels the first time one is requested after an evaluation, not on the iteration path. */
int hb200_factor_evaluate(hb200_ctx* ctx, int kind, int index, const double* const* parameters, double* residuals, double** jacobians);

/* normal equations + landmark Schur complement at the current linearisation point;
 * requires hb200_evaluate(JACOBIANS).  System layout: [6K pose | 3Kbg | 3Kba | 2 gravity]. */
int hb200_reduced_size(hb200_ctx* ctx);
int hb200_build_system(hb200_ctx* ctx);
/* dense copy of what the solver factors: damped (mu * clamp(diag H)), constant dofs masked to identity. */
int hb200_get_system(hb200_ctx* ctx, double* S /* n x n */, double* b /* n */);
/* dense Cholesky of the reduced system, back-substitution, landmark back-substitution. */
int hb200_solve(hb200_ctx* ctx);
int hb200_get_delta(hb200_ctx* ctx, double* delta_pose /* n */, double* delta_landmark /* 3L */);
/* ---- marginal covariances: the replacement of ceres::Covariance (default options: apply_loss_function, constant
 * blocks get zero covariance) -----------------------------------------------------------------------------------------
 * Sigma = (J^T W J)^-1 over the non-constant dofs at the current state, J the Jacobian of the (family-matrix weighted,
 * hb200_set_weights) residuals, W the loss weights of the LM build (Huber rho' of
 * pixel / bearing factors, the inertial ScaledLoss, none for pose factors), no damping anywhere (mu = 0, also inside the
 * landmark elimination).  Constant knots, bias_const and gravity_const dofs get exact zeros.  Tangent convention of the
 * device: rotation global (R <- Exp(theta) R), SE3 split [theta | rho] with p <- p + rho, gravity the 2-dof sphere tangent.
 *   hb200_build_covariance:   evaluates at the current state and assembles the UNDAMPED reduced system into the packed
 *                             buffer (hb200_system_device_ptr) with the factor, J^T J and Schur kernels of hb200_build_system;
 *                             flags degenerate / unobserved landmarks; one read-back.  The LM's trust-region state is not
 *                             touched, but the packed buffer is no longer a damped-solve input: hb200_get_system / hb200_solve
 *                             return -2 until the next hb200_build_system.  Copies the knots it linearised at.
 *   hb200_compute_covariance: band + arrow Cholesky of the (equilibrated, masked) packed buffer and its selected inverse --
 *                             every entry of Sigma on the block band of half-width beta, the arrow and the corner -- then the
 *                             3 x 3 marginal of every landmark.  Only valid right after hb200_build_covariance (-2 when a
 *                             setter changed the window or any other call launched work since).  status 1 (returns HB200_COV_NOT_POSITIVE_DEFINITE): a pivot
 *                             of the equilibrated reduced factor is <= 1e-10 (gauge not fixed, a bias / gravity dof without a
 *                             factor); bad_dof = the first such dof.  status 2 (returns HB200_COV_DEGENERATE_LANDMARKS): a
 *                             landmark's undamped V_l is rank-deficient (seen by one pixel factor only).  An unobserved
 *                             landmark is no failure: zero block, counted.  On failure the previous results stay in place.
 *   hb200_get_covariance:     packed = Sigma in the P | A | C part of the packed layout (doubles [0, oC + m*m): diagonal blocks
 *                             and corner full, padding rows 0), landmark = [L][3][3] (may be NULL).  Shape: info K, beta, m, L.
 *   hb200_interpolate_covariance: the 6 x 6 covariance of the pose [theta | p] interpolated at each stamp, at the knots of
 *                             the last successful compute; stamps outside the valid span give zero blocks, counted.
 *   hb200_interpolate_state_covariance: the 18 x 18 joint covariance of x(t) = [theta p | omega v | b_g b_a] at each stamp:
 *                             the pose as above, the body velocity of hb200_interpolate (omega the body rate, v = R^T pdot)
 *                             and both bias splines evaluated at t, J(t) Sigma J(t)^T over the stamp's k control points
 *                             and the 4 knots of each bias spline (all within the band, the arrow and the corner), exactly
 *                             symmetric.  Knots, knot table and bias splines are those of the last successful compute:
 *                             later iterations, appends and slides change nothing until the next one.  A stamp outside the
 *                             pose spline's valid span, or outside that of a bias spline with knots, gives a zero block,
 *                             counted; a window without bias splines gives zero bias rows and columns.  Gravity cross terms
 *                             are in the corner of hb200_get_covariance.  -2 before a compute succeeded, -1 for n < 0 or a
 *                             NULL stamps / cov with n > 0.
 * Sharded contexts (a communicator or the all-reduce callback): hb200_build_covariance and hb200_compute_covariance are
 * collective, see the SHARDING CONTRACT below.  The build assembles each rank's undamped partial system (its factors, the
 * Schur complement of the landmarks it owns) and sums it over the ranks with ONE system reduction, as hb200_build_system
 * does; the compute then inverts the same reduced system on every rank (band, arrow, corner, status, bad_dof and
 * min_pivot_ratio bit-identical across ranks) and the marginals of the rank's own landmarks: read a landmark's block from
 * its owner (a landmark a rank holds but does not observe gets a zero block there).  hb200_get_covariance and
 * hb200_interpolate_covariance / hb200_interpolate_state_covariance are local calls; the interpolated covariances are
 * identical on every rank.  A peer that does not reach the reduction makes the build fail (-7 after the peer-memory
 * reduction's timeout, the callback's error + 200) instead of hanging the others.
 * A window whose band + arrow (6 (beta+1) + m rows, square) does not fit one CTA's shared memory gets -6 (on a sharded
 * context from every rank, before the reduction: it depends only on the agreed layout).  Ceres-tangent and ambient
 * blocks: hyper::Covariance (host, one GPU). */
typedef struct hb200_covariance_info {
  int status;                 /* 0 ok, 1 reduced system not positive definite, 2 degenerate landmarks */
  int bad_dof;                /* status 1: first reduced-system dof whose pivot failed, else -1 */
  /* degenerate_landmarks (and so status 2) counts the whole window on a sharded context and is the same on every rank;
   * unobserved_landmarks and L are rank-local: the landmarks this context holds, and those of them it does not observe. */
  int degenerate_landmarks, unobserved_landmarks;
  double min_pivot_ratio;     /* smallest pivot of the equilibrated reduced factor (status 1: the failing one) */
  int K, beta, m, L;          /* shape of what hb200_get_covariance returns */
} hb200_covariance_info;
enum { HB200_COV_NOT_POSITIVE_DEFINITE = 40, HB200_COV_DEGENERATE_LANDMARKS = 41 };
int hb200_build_covariance(hb200_ctx* ctx);
int hb200_compute_covariance(hb200_ctx* ctx, hb200_covariance_info* info);
int hb200_get_covariance(hb200_ctx* ctx, double* packed /* P | A | C of SysLayout */, double* landmark /* [L][3][3], may be NULL */);
int hb200_interpolate_covariance(hb200_ctx* ctx, int n, const double* stamps, double* cov /* [n][6][6] */, int* num_invalid);
enum { HB200_STATE_COV_DIM = 18 };
int hb200_interpolate_state_covariance(hb200_ctx* ctx, int n, const double* stamps, double* cov /* [n][18][18] */, int* num_invalid);
/* Blocks outside the selected inverse's pattern, the list of ceres::Covariance::Compute(covariance_blocks): knot pairs
 * more than beta apart, landmark x knot / bias / gravity and landmark x landmark (any pair is accepted; pairs in the
 * pattern are copied from Sigma and the landmark marginals bit for bit).
 *   hb200_set_covariance_blocks: registers n pairs (kind_a, index_a, kind_b, index_b) that every later
 *                             hb200_compute_covariance computes with Sigma (n = 0 clears the list; with no list the compute
 *                             runs exactly as without this call).  Host-only: touches neither the build nor committed results.
 *                             The compute checks the indices against the build's shapes (knots < K, bias knots < Kbg / Kba,
 *                             gravity 0, landmarks < L of this context) and returns -1 without computing anything on a bad one.
 *   hb200_get_covariance_blocks: Sigma_ab of the last successful compute, t_a x t_b row-major in the top-left of a 6 x 6
 *                             slot (device tangents: knot 6, bias knot 3, gravity 2, landmark 3), the rest 0; (b, a) is the
 *                             exact transpose of (a, b); constant dofs 0.  status[i] (may be NULL): 0 computed, 1 a landmark
 *                             without observations on a sharded context (its owner computes the pair), 2 a landmark without
 *                             observations (as its marginal); both with a zero block.  -2 before a successful compute and
 *                             when n differs from the number of pairs that compute was given.  Like Sigma, the blocks are
 *                             a snapshot: a failed compute, later iterations, appends and slides leave them as they are.
 * Sharded contexts: no collective step is added.  Knot, bias and gravity pairs are bit-identical on every rank; a pair
 * with landmarks is computed by the rank that observes them (status 1 elsewhere); two landmarks owned by different ranks
 * are not supported (status 1 on both). */
enum { HB200_COV_KNOT = 0, HB200_COV_GYRO_BIAS = 1, HB200_COV_ACCEL_BIAS = 2, HB200_COV_GRAVITY = 3, HB200_COV_LANDMARK = 4 };
int hb200_set_covariance_blocks(hb200_ctx* ctx, int n, const int* pairs /* [n][4] */);
int hb200_get_covariance_blocks(hb200_ctx* ctx, int n, double* out /* [n][6][6] */, int* status /* [n], may be NULL */);
/* Poses at two stamps: their joint covariance and the covariance of the relative pose between them (loop-closure gates,
 * increment uncertainty).
 *   hb200_set_covariance_stamp_pairs: registers n pairs (t_a, t_b) that every later hb200_compute_covariance computes with
 *                             Sigma (n = 0 clears the list; with no list the compute runs exactly as without this call).
 *                             Host-only: touches neither the build nor committed results.  -1 for n < 0, NULL stamps with
 *                             n > 0 or a non-finite stamp (the previous list stays).
 *   hb200_get_pose_pair_covariance: per pair, at the knots of the last successful compute --
 *                             joint    [12][12]: covariance of [theta_a p_a | theta_b p_b] in the device tangent (R <- Exp(theta) R,
 *                                      p <- p + rho).  Its diagonal blocks are hb200_interpolate_covariance at t_a and t_b, its
 *                                      off-diagonal block J(t_a) Sigma_{span(a), span(b)} J(t_b)^T (knot pairs beyond the band
 *                                      included); exactly symmetric, and (t_b, t_a) is exactly the permutation of (t_a, t_b).
 *                             relative [6][6]: covariance of T_ab = T_a^-1 T_b (R_ab = R_a^T R_b, p_ab = R_a^T (p_b - p_a)) in
 *                                      the same split tangent in frame a (R_ab <- Exp(dtheta) R_ab, p_ab <- p_ab + dp):
 *                                      A joint A^T with A = [[-R_a^T, 0, R_a^T, 0], [R_a^T hat(p_b - p_a), -R_a^T, 0, R_a^T]],
 *                                      R_a, p_a, p_b the interpolated poses; exactly symmetric.
 *                             status [n]: 0 computed, 1 a stamp outside the pose spline's valid span (both blocks zero).
 *                             joint, relative and status may each be NULL.  -2 before a successful compute and when n differs
 *                             from the number of pairs that compute was given.  A snapshot like Sigma: a failed compute, a
 *                             registration without a compute, later iterations, appends and slides leave the results as
 *                             they are.
 * Sharded contexts: no collective step is added; the pairs involve knots only, so the results are bit-identical on every
 * rank. */
int hb200_set_covariance_stamp_pairs(hb200_ctx* ctx, int n, const double* stamps /* [n][2]: t_a, t_b */);
int hb200_get_pose_pair_covariance(hb200_ctx* ctx, int n, double* joint /* [n][12][12], may be NULL */, double* relative /* [n][6][6], may be NULL */,
                                   int* status /* [n], may be NULL */);

/* full LM iterations: evaluate -> build -> [allreduce] -> solve -> retract -> cost at trial ->
 * accept/reject, all on the device.  records may be NULL. */
int hb200_iterate(hb200_ctx* ctx, int iterations, hb200_iteration* records);
int hb200_cost(hb200_ctx* ctx, double* cost);
/* ceres::Solver::Options termination tests (the reference leaves them at Ceres' defaults, optimizer.cpp:38-54:
 * function_tolerance 1e-6, gradient_tolerance 1e-10, parameter_tolerance 1e-8, min_trust_region_radius 1e-32), evaluated
 * on the device in the step-acceptance kernel exactly where ceres::TrustRegionMinimizer evaluates them; a value <= 0
 * switches a test off, all four off (the default of this library) makes hb200_iterate / hb200_optimize run exactly the
 * requested number of iterations.  Once a test fires the remaining iterations of the call are no-ops and their records
 * are zero.  hb200_get_termination: 0 none (iteration limit), 1 function, 2 parameter, 3 gradient tolerance, 4 minimum
 * trust-region radius, 5 five consecutive invalid steps; plus the number of iterations performed by the last call
 * that fetched records and the last |x - Plus(x, -g)|_inf, |step|, |x| the tests saw.
 * hb200_optimize starts every call at the initial radius of hb200_set_options (as ceres::Solve does); hb200_iterate
 * continues the trust region of the previous call.  At N > 1 the gradient test needs the peer mailbox: with the
 * all-reduce callback or NCCL without a peer mapping the ranks can only sum, gradient_max_norm then covers the replicated
 * blocks (knots, biases, gravity) and not the landmarks, and hb200_iterate / hb200_optimize refuse a gradient tolerance > 0. */
int hb200_set_termination(hb200_ctx* ctx, double function_tolerance, double gradient_tolerance, double parameter_tolerance, double min_trust_region_radius);
int hb200_get_termination(hb200_ctx* ctx, int* type, int* iterations_performed, double* gradient_max_norm, double* step_norm, double* x_norm);
/* Deterministic assembly (off by default).  By default the normal-equation kernels add into the packed system with FP64
 * atomics, so the order of the additions -- and the last bits of S, b and g -- depends on how the GPU schedules them,
 * and two runs of the same window can take different LM steps.  With it on, every kernel stores its contributions
 * with plain stores into slots of its own and one reduction kernel sums each packed entry over its slots in an order
 * fixed by the bound window.  Same build of this library, same GPU model, same window and the same call sequence then
 * give bit-identical results for:
 *   - the packed buffer hb200_build_system leaves (hb200_system_device_ptr), hb200_get_system, hb200_solve / hb200_get_delta
 *   - hb200_iterate / hb200_optimize: records, termination and state
 *   - hb200_build_covariance + hb200_compute_covariance (hb200_get_covariance) and hb200_interpolate_covariance
 *   - hb200_get_pose_pair_covariance (the stamp pairs of hb200_set_covariance_stamp_pairs)
 *   - sharded contexts: each rank's partial system; the peer-memory reduction sums the ranks in rank order.
 * Not covered: other GPU models or builds, the dense fallback solver (hb200_options.reserved bit 0) and the NCCL
 * all-reduce (as deterministic as NCCL's reduction).  It costs extra device memory for the slots and time for the
 * reduction (DESIGN.md §5.4).  May be set before or after hb200_bind; a change drops a built system and a pending
 * covariance build (as any change of the kernels' arguments does) and takes effect at the next build or iteration,
 * which then lays out the slots for the window.  Setting the current value changes nothing. */
int hb200_set_deterministic(hb200_ctx* ctx, int enable);
int hb200_get_deterministic(hb200_ctx* ctx, int* enable);
/* The drop-in for CeresOptimizer::optimize() (reference optimizer.cpp:276-280) with the parameter
 * blocks in HOST memory, as Ceres aliases them: uploads the five variable families, runs
 * `iterations` LM iterations on the device, downloads the updated blocks into the same buffers and
 * synchronises once.  Factor lists stay bound.  Buffers should be pinned for asynchronous copies. */
int hb200_optimize(hb200_ctx* ctx, int iterations, double* knots, double* gyro, double* accel, double* gravity, double* landmarks,
                   hb200_iteration* records);
/* device-side snapshot / restore of the variable blocks and the trust-region state (benchmarks,
 * step rejection experiments). */
int hb200_snapshot(hb200_ctx* ctx);
int hb200_restore(hb200_ctx* ctx);
/* Runs `reps` LM iterations with a CUDA event after every kernel and returns the average duration of
 * each launch in issue order (names are kernel names, 32 chars each).  Not for timing the step --
 * for attributing it (bench.py roofline / kernel shares).  A negative `reps` profiles |reps| plain
 * Evaluate sweeps (what hb200_evaluate(HB200_EVAL_JACOBIANS) launches) instead of full iterations. */
int hb200_profile_iteration(hb200_ctx* ctx, int reps, int max_entries, char* names /* [max_entries][32] */, double* ms, int* count);
/* Spline interpolation of the current state at `n` stamps (device kernel): pose [n][7] = [q|p], and
 * optionally (may be NULL) body velocity [n][6] = [omega | R^T pdot] and acceleration [n][6]. Stamps
 * outside the valid span give identity/zero rows and are counted in num_invalid.  Replaces
 * state->evaluate(StateQuery{stamp, derivative}) for trajectory dumps (reference apps/hyperslam/main.cpp:69-80). */
int hb200_interpolate(hb200_ctx* ctx, int n, const double* stamps, double* pose, double* velocity, double* acceleration, int* num_invalid);
int hb200_get_state(hb200_ctx* ctx, double* knots, double* gyro, double* accel, double* gravity, double* landmarks);
/* Ingest of stereo tracks in front of the factor lists (reference internal/hyper/optimizers/abstract.cpp:186-264):
 * per track i the unit bearings of both views (C.convertPixelsToBearings, :221-223) and the landmark
 * triangulated from them and moved to the world frame with the CURRENT state's pose at stamp[i]
 * (Camera::Triangulate(T_01, b0, b1) :252, T_w0.vectorPlus :253).  Outputs may not be NULL.  Tracks whose stamp
 * or camera index is invalid are zero-filled and counted. */
int hb200_ingest_stereo(hb200_ctx* ctx, int n, const double* stamp, const int* camera0, const int* camera1, const double* pixel0 /* [n][2] */,
                        const double* pixel1 /* [n][2] */, double* bearing0 /* [n][3] */, double* bearing1 /* [n][3] */,
                        double* landmark /* [n][3] */, int* num_invalid);

/* ---- multi-GPU (SURVEY.md section 8e) ---------------------------------------------------------
 * Factors shard over ranks, the window state is replicated.  Per iteration every rank builds its partial
 * reduced system, ONE ncclAllReduce sums it on the context's stream (enqueued from C, so the iteration stays
 * one CUDA graph), every rank solves redundantly and retracts its replica; the three step-acceptance scalars
 * (trial cost, landmark parts of the model decrease) are exchanged through peer memory inside accept_kernel
 * (hb200_peer_*), with a second 4-double ncclAllReduce as the fallback when no peer mapping exists.
 *
 * SHARDING CONTRACT (the caller's responsibility; violating it gives silently wrong steps):
 *   - every observation (pixel / bearing factor) of a landmark must live on ONE rank -- the landmark's owner.
 *     The landmark block is eliminated rank-locally (Schur complement of a sum is not the sum of Schur
 *     complements) and only the owner updates the landmark, so non-owned landmarks of a replica are stale;
 *     read each landmark back from its owner.
 *   - inertial and manifold factors may be split arbitrarily; every factor lives on exactly one rank.
 *   - knots, bias splines, gravity, calibration, constancy flags, options and family weight matrices
 *     (hb200_set_weights: replicated configuration, no collective step) must be identical on all ranks,
 *     and every rank must make the same sequence of hb200_iterate / hb200_optimize / hb200_build_system /
 *     hb200_build_covariance / hb200_compute_covariance calls.  The covariance build takes one system reduction
 *     (like hb200_build_system) and leaves the LM's trust-region state alone; the compute has no collective step.
 *     Registered stamp pairs (hb200_set_covariance_stamp_pairs) need not be the same on every rank; a pair's results
 *     are bit-identical on every rank that registered it.
 *     A rank that fails a call for a reason of its own (an invalid argument, a stale build) breaks the contract as
 *     in hb200_iterate; the peer reduction's timeout and the callback's error return keep the others from waiting
 *     forever.
 *   - a sharded window slides.  The sliding-window calls come in three classes:
 *       collective  hb200_append_pixel_factors, _bearing_factors, _stereo_tracks, hb200_slide: every rank makes the
 *                   same sequence of these calls, each with its own shard's data (n = 0, with any pointers, when it
 *                   has nothing of its own).  Each ends with agreement rounds on one small payload of doubles that a
 *                   SUM over the ranks answers, through the context's channel (ncclAllReduce, or the hook): round A
 *                   before anything moves (the header -- K, Kbg, Kba, call kind, slide flags, knots and bias knots at
 *                   or before the lower bound --, every rank's validation status and, for hb200_slide, the smallest
 *                   kept knot and bias bases), round B after the incidence lists (the band half-width).  Ranks whose
 *                   calls differ all return -2 and change nothing (the header and its squares are summed, so a
 *                   difference is seen on every rank); when any rank's own checks fail, every rank
 *                   returns the same window-wide code (2 before 3) and changes nothing (the error string tells this
 *                   rank's failure from another's).  The knot and bias shifts are the whole window's; slide stats
 *                   knots* are identical on every rank, landmark and factor counts and hb200_slide_landmark_map are
 *                   rank-local.  A slide refused with -2 leaves no landmark map (-2 from hb200_slide_landmark_map).
 *                   The payload has 20 + 2K + Kbg + Kba doubles: ranks whose K, Kbg or Kba already differ (replicated
 *                   calls out of step) reduce payloads of different lengths, which the hook can see but NCCL does not
 *                   check -- the header catches differing calls, not replicated state that already diverged.  A track
 *                   too long for the Schur tile (-6) is refused on every rank, after the call has taken effect, as
 *                   on one context.  Detaching the hook or the communicator drops the agreed half-width.
 *       replicated  hb200_append_knots, hb200_append_bias_knots: every rank calls with the same arguments; no
 *                   communication, the result follows from replicated state.
 *       rank-local  hb200_append_landmarks, _inertial_factors, _manifold_factors: no collective call -- they change
 *                   neither the band nor replicated state.
 *     Routing is the caller's: tracks of a known landmark go to its owner, a new landmark's owner is the caller's
 *     choice, inertial and pose factors may go to any rank.  Owners never change (no landmark moves between ranks).
 *     beta = max(own, the hb200_set_min_bandwidth floor, the agreed value of the latest agreement): hb200_bind with a
 *     communicator takes the maximum over the ranks as the agreed value (collective); through the hook hb200_bind
 *     agrees on nothing and the host sets the floor.  So a sharded band narrows again, as one context's does, when
 *     the longest track leaves the window -- down to the floor.
 *
 * Reduced buffer (what is summed): the band-only packed system, hb200_system_device_ptr(), in doubles
 *   [ P K*h*6 | A m*6K | C m*m | b n | diagH n | g n | scal 8 ],  h = 6 + 6*beta, m = n - 6K
 * (block-banded pose part of half-bandwidth beta = longest landmark track in control points, arrowhead of
 * the bias / gravity dofs; scal[0] = cost at the linearisation point).  K = 50: 20 k doubles (0.16 MB). */
/* ncclGetUniqueId / ncclCommInitRank through the library (libnccl.so.2 is bound with dlopen at the first call):
 * rank 0 creates the 128-byte id, the host program ships it to the other ranks (MPI, torch.distributed, ...). */
int hb200_comm_unique_id(char* id /* [128] */);
int hb200_comm_init_rank(hb200_ctx* ctx, int nranks, int rank, const char* id /* [128] */);
/* or attach an existing ncclComm_t (not owned; NULL detaches).  Same as hb200_options.nccl_comm at creation. */
int hb200_set_nccl_comm(hb200_ctx* ctx, void* nccl_comm, int nranks, int rank);
/* peer-memory mailbox for the step-acceptance scalars: every rank exports a 64-byte cudaIpcMemHandle_t, the
 * host program all-gathers them, every rank maps its peers' mailboxes.  Ranks must be processes on one node
 * with NVLink / PCIe peer access.  Optional: without it the scalars take a second ncclAllReduce. */
int hb200_peer_handle(hb200_ctx* ctx, char* handle /* [64] */);
int hb200_peer_connect(hb200_ctx* ctx, int nranks, int rank, const char* handles /* [nranks][64] */);
/* all ranks or none: when the mapping failed on any rank, every rank drops it (collective protocol). */
int hb200_peer_disconnect(hb200_ctx* ctx);
int hb200_comm_info(hb200_ctx* ctx, int* nranks, int* rank, int* nccl, int* peer_mailbox, int* graph, long long* payload_doubles);
/* Block half-bandwidth beta of the packed layout.  It follows from the longest landmark track of the local factor
 * shard; with a communicator attached hb200_bind / hb200_set_nccl_comm agree on the maximum over the ranks
 * themselves (collective), and the collective sliding-window calls agree on it again.  Hosts using the callback hook
 * below must do that after hb200_bind: read it, take the maximum over ranks, set it as the lower bound everywhere
 * (a floor the band then never goes below; hb200_set_min_bandwidth(0) after the first collective call lifts it). */
int hb200_get_bandwidth(hb200_ctx* ctx, int* beta);
int hb200_set_min_bandwidth(hb200_ctx* ctx, int beta);
/* Escape hatch for hosts without NCCL: the caller sums `count_doubles` doubles at `device_buffer` across ranks
 * on `stream` (called twice per iteration: packed system, then 8 scalars; once per hb200_build_system and
 * hb200_build_covariance: packed system; once per agreement round of a collective sliding-window call -- two per
 * call, one when a rank's checks failed or the calls differ).  Disables CUDA-graph capture. */
typedef int (*hb200_allreduce_fn)(void* user, void* device_buffer, long long count_doubles, void* stream);
int hb200_set_allreduce(hb200_ctx* ctx, hb200_allreduce_fn fn, void* user);
void* hb200_system_device_ptr(hb200_ctx* ctx, long long* count_doubles);
void* hb200_stream(hb200_ctx* ctx);

/* Measured FP64 FMA throughput of the device in TFLOP/s (DFMA chains, all SMs): the second roofline ceiling of the
 * FP64 factor kernels next to the HBM copy bandwidth (bench.py reports both). */
int hb200_measure_fp64_peak(hb200_ctx* ctx, double* tflops);

/* kernel-launch counter (number of this library's kernels launched since creation). */
long long hb200_launch_count(hb200_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* HYPERB200_H_ */
