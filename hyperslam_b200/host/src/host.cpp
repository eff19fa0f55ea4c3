// Host-side plugin surface over libhyperb200 (C-ABI).  No arithmetic of the hot path happens here:
// spline interpolation, factor evaluation and the solve are device kernels; this file flattens the
// object graph, forwards, and implements the (host-side) manifold hooks Ceres would call.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <stdexcept>
#include <string>

#include "hyper/covariance.hpp"
#include "hyper/optimizer.hpp"
#include "../../../include/hyperb200.h"

namespace hyper {

namespace {
void check(int rc, const char* what) {
  if (rc != 0) throw std::runtime_error(std::string(what) + ": hb200 error " + std::to_string(rc) + ": " + hb200_last_error_string());
}
void quat_mul(const double* a, const double* b, double* c) {
  const double x = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  const double y = a[3] * b[1] - a[0] * b[2] + a[1] * b[3] + a[2] * b[0];
  const double z = a[3] * b[2] + a[0] * b[1] - a[1] * b[0] + a[2] * b[3];
  const double w = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
  c[0] = x; c[1] = y; c[2] = z; c[3] = w;
}
// Householder vector of Ceres' sphere manifold.
void householder(const double* x, int n, double* v, double* beta) {
  double sigma = 0;
  for (int i = 0; i < n - 1; ++i) sigma += x[i] * x[i];
  for (int i = 0; i < n; ++i) v[i] = x[i];
  v[n - 1] = 1.0; *beta = 0.0;
  const double xp = x[n - 1];
  if (sigma <= 2.220446049250313e-16) { if (xp < 0.0) *beta = 2.0; return; }
  const double mu = std::sqrt(xp * xp + sigma);
  const double vp = (xp <= 0.0) ? xp - mu : -sigma / (xp + mu);
  *beta = 2.0 * vp * vp / (sigma + vp * vp);
  for (int i = 0; i < n - 1; ++i) v[i] /= vp;
}
}  // namespace

// ---------------------------------------------------------------------------------------------
// Manifold hooks
// ---------------------------------------------------------------------------------------------
bool Manifold::Plus(const Scalar* x, const Scalar* delta, Scalar* out) const {
  int a = 0, t = 0;
  for (const Part& p : parts_) {
    const int n = p.ambient;
    switch (p.kind) {
      case kEuclidean: for (int i = 0; i < n; ++i) out[a + i] = x[a + i] + delta[t + i]; break;
      case kConstant: for (int i = 0; i < n; ++i) out[a + i] = x[a + i]; break;
      case kQuaternion: {
        const double* d = delta + t;
        const double nd = std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
        double q[4] = {0, 0, 0, 1};
        if (nd > 0.0) { const double s = std::sin(nd) / nd; q[0] = s * d[0]; q[1] = s * d[1]; q[2] = s * d[2]; q[3] = std::cos(nd); }
        quat_mul(q, x + a, out + a);
      } break;
      case kSphere: {
        const double* d = delta + t;
        double nd = 0;
        for (int i = 0; i < n - 1; ++i) nd += d[i] * d[i];
        nd = std::sqrt(nd);
        if (nd == 0.0) { for (int i = 0; i < n; ++i) out[a + i] = x[a + i]; break; }
        double v[8], beta, y[8], nx = 0, vy = 0;
        householder(x + a, n, v, &beta);
        for (int i = 0; i < n; ++i) nx += x[a + i] * x[a + i];
        nx = std::sqrt(nx);
        const double s = std::sin(nd) / nd;
        for (int i = 0; i < n - 1; ++i) y[i] = s * d[i];
        y[n - 1] = std::cos(nd);
        for (int i = 0; i < n; ++i) vy += v[i] * y[i];
        for (int i = 0; i < n; ++i) out[a + i] = nx * (y[i] - v[i] * beta * vy);
      } break;
    }
    a += n; t += tangent(p);
  }
  return true;
}

bool Manifold::PlusJacobian(const Scalar* x, Scalar* J) const {
  const int na = AmbientSize(), nt = TangentSize();
  std::fill(J, J + static_cast<size_t>(na) * nt, 0.0);
  int a = 0, t = 0;
  for (const Part& p : parts_) {
    const int n = p.ambient;
    switch (p.kind) {
      case kEuclidean: for (int i = 0; i < n; ++i) J[(a + i) * nt + t + i] = 1.0; break;
      case kConstant: break;
      case kQuaternion: {
        const double qx = x[a], qy = x[a + 1], qz = x[a + 2], qw = x[a + 3];
        const double M[12] = {qw, qz, -qy, -qz, qw, qx, qy, -qx, qw, -qx, -qy, -qz};
        for (int i = 0; i < 4; ++i) for (int j = 0; j < 3; ++j) J[(a + i) * nt + t + j] = M[3 * i + j];
      } break;
      case kSphere: {
        double v[8], beta, nx = 0;
        householder(x + a, n, v, &beta);
        for (int i = 0; i < n; ++i) nx += x[a + i] * x[a + i];
        nx = std::sqrt(nx);
        for (int c = 0; c < n - 1; ++c) for (int r = 0; r < n; ++r) J[(a + r) * nt + t + c] = nx * ((r == c ? 1.0 : 0.0) - beta * v[c] * v[r]);
      } break;
    }
    a += n; t += tangent(p);
  }
  return true;
}

bool Manifold::RightMultiplyByPlusJacobian(const Scalar* x, int num_rows, const Scalar* A, Scalar* T) const {
  const int na = AmbientSize(), nt = TangentSize();
  std::vector<double> J(static_cast<size_t>(na) * std::max(nt, 1));
  PlusJacobian(x, J.data());
  for (int r = 0; r < num_rows; ++r)
    for (int c = 0; c < nt; ++c) {
      double s = 0;
      for (int i = 0; i < na; ++i) s += A[r * na + i] * J[i * nt + c];
      T[r * nt + c] = s;
    }
  return true;
}

bool Manifold::Minus(const Scalar* y, const Scalar* x, Scalar* out) const {
  int a = 0, t = 0;
  for (const Part& p : parts_) {
    const int n = p.ambient;
    switch (p.kind) {
      case kEuclidean: for (int i = 0; i < n; ++i) out[t + i] = y[a + i] - x[a + i]; break;
      case kConstant: break;
      case kQuaternion: {
        const double xc[4] = {-x[a], -x[a + 1], -x[a + 2], x[a + 3]};
        double q[4];
        quat_mul(y + a, xc, q);
        const double u = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
        if (u > 0.0) { const double th = std::atan2(u, q[3]); for (int i = 0; i < 3; ++i) out[t + i] = th * q[i] / u; }
        else { out[t] = out[t + 1] = out[t + 2] = 0.0; }
      } break;
      case kSphere: {
        double v[8], beta, hy[8], vy = 0, nh = 0;
        householder(x + a, n, v, &beta);
        for (int i = 0; i < n; ++i) vy += v[i] * y[a + i];
        for (int i = 0; i < n; ++i) hy[i] = y[a + i] - v[i] * beta * vy;
        for (int i = 0; i < n - 1; ++i) nh += hy[i] * hy[i];
        nh = std::sqrt(nh);
        if (nh == 0.0) { for (int i = 0; i < n - 1; ++i) out[t + i] = 0.0; }
        else { const double th = std::atan2(nh, hy[n - 1]); for (int i = 0; i < n - 1; ++i) out[t + i] = th * hy[i] / nh; }
      } break;
    }
    a += n; t += tangent(p);
  }
  return true;
}

bool Manifold::MinusJacobian(const Scalar* x, Scalar* J) const {
  // d Minus(y, x) / dy at y = x: left inverse of PlusJacobian (tangent x ambient).
  const int na = AmbientSize(), nt = TangentSize();
  std::fill(J, J + static_cast<size_t>(nt) * na, 0.0);
  int a = 0, t = 0;
  for (const Part& p : parts_) {
    const int n = p.ambient;
    switch (p.kind) {
      case kEuclidean: for (int i = 0; i < n; ++i) J[(t + i) * na + a + i] = 1.0; break;
      case kConstant: break;
      case kQuaternion: {
        const double qx = x[a], qy = x[a + 1], qz = x[a + 2], qw = x[a + 3];
        const double M[12] = {qw, qz, -qy, -qx, -qz, qw, qx, -qy, qy, -qx, qw, -qz};   // transpose of the Plus Jacobian (|q| = 1)
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 4; ++j) J[(t + i) * na + a + j] = M[4 * i + j];
      } break;
      case kSphere: {
        double v[8], beta, nx = 0;
        householder(x + a, n, v, &beta);
        for (int i = 0; i < n; ++i) nx += x[a + i] * x[a + i];
        nx = std::sqrt(nx);
        for (int c = 0; c < n - 1; ++c) for (int r = 0; r < n; ++r) J[(t + c) * na + a + r] = ((r == c ? 1.0 : 0.0) - beta * v[c] * v[r]) / nx;
      } break;
    }
    a += n; t += tangent(p);
  }
  return true;
}

// ---------------------------------------------------------------------------------------------
// ContinuousState
// ---------------------------------------------------------------------------------------------
std::vector<StateResult> ContinuousState::evaluate(hb200_ctx* ctx, const std::vector<Stamp>& stamps, Index derivative) const {
  const int n = static_cast<int>(stamps.size());
  std::vector<double> pose(7 * static_cast<size_t>(n)), vel(6 * static_cast<size_t>(n)), acc(6 * static_cast<size_t>(n));
  int bad = 0;
  check(hb200_interpolate(ctx, n, stamps.data(), pose.data(), derivative >= 1 ? vel.data() : nullptr, derivative >= 2 ? acc.data() : nullptr, &bad),
        "hb200_interpolate");
  if (bad) throw std::out_of_range("ContinuousState::evaluate: stamp outside range()");
  std::vector<StateResult> out(n);
  for (int i = 0; i < n; ++i) {
    std::copy(pose.begin() + 7 * i, pose.begin() + 7 * i + 7, out[i].value.v.begin());
    if (derivative >= 1) std::copy(vel.begin() + 6 * i, vel.begin() + 6 * i + 6, out[i].velocity.v.begin());
    if (derivative >= 2) std::copy(acc.begin() + 6 * i, acc.begin() + 6 * i + 6, out[i].acceleration.v.begin());
  }
  return out;
}

// ---------------------------------------------------------------------------------------------
// Optimizer
// ---------------------------------------------------------------------------------------------
Optimizer::Optimizer(int device) {
  hb200_options o{device, nullptr, 1, 0, nullptr, 1, 0};
  check(hb200_create(&o, &ctx_), "hb200_create");
}
Optimizer::~Optimizer() { hb200_destroy(ctx_); }

void Optimizer::setSolverTolerances(double function_tolerance, double gradient_tolerance, double parameter_tolerance, double min_trust_region_radius) {
  check(hb200_set_termination(ctx_, function_tolerance, gradient_tolerance, parameter_tolerance, min_trust_region_radius), "hb200_set_termination");
}
void Optimizer::setDeterministic(bool deterministic) { check(hb200_set_deterministic(ctx_, deterministic ? 1 : 0), "hb200_set_deterministic"); }
void Optimizer::setWeights(ExteroceptiveCost::Kind kind, const std::vector<double>& weights) {
  static constexpr size_t kSide[] = {2, 6, 1, 6};   // indexed by ExteroceptiveCost::Kind (== HB200_PIXEL ...)
  const int k = static_cast<int>(kind);
  if (k < 0 || k > 3) throw std::invalid_argument("setWeights: unknown factor kind " + std::to_string(k));
  const size_t d = kSide[k];
  if (!weights.empty() && weights.size() != d * d) throw std::invalid_argument("setWeights: the matrix of this family is " + std::to_string(d) + " x " + std::to_string(d));
  check(hb200_set_weights(ctx_, static_cast<int>(kind), weights.empty() ? nullptr : weights.data()), "hb200_set_weights");
}
int Optimizer::terminationType() const {
  int type = 0;
  hb200_get_termination(ctx_, &type, nullptr, nullptr, nullptr, nullptr);
  return type;
}

Index Optimizer::cameraIndex(const Camera* camera) const {
  for (size_t i = 0; i < cameras_.size(); ++i) if (cameras_[i] == camera) return static_cast<Index>(i);
  throw std::invalid_argument("observation refers to an unknown camera");
}
Index Optimizer::landmarkIndex(const Landmark* landmark) const {
  for (size_t i = 0; i < landmarks_.size(); ++i) if (landmarks_[i] == landmark) return static_cast<Index>(i);
  throw std::invalid_argument("observation refers to an unknown landmark");
}

ExteroceptiveCost* Optimizer::add(VisualPixelObservation& obs) {
  pixel_obs_.push_back(&obs);
  costs_.emplace_back(new ExteroceptiveCost(this, ExteroceptiveCost::kPixel, static_cast<Index>(pixel_obs_.size() - 1)));
  dirty_ = true;
  return costs_.back().get();
}
ExteroceptiveCost* Optimizer::add(InertialObservation& obs) {
  inertial_obs_.push_back(&obs);
  costs_.emplace_back(new ExteroceptiveCost(this, ExteroceptiveCost::kInertial, static_cast<Index>(inertial_obs_.size() - 1)));
  dirty_ = true;
  return costs_.back().get();
}

ExteroceptiveCost* Optimizer::add(VisualBearingObservation& obs) {
  bearing_obs_.push_back(&obs);
  costs_.emplace_back(new ExteroceptiveCost(this, ExteroceptiveCost::kBearing, static_cast<Index>(bearing_obs_.size() - 1)));
  dirty_ = true;
  return costs_.back().get();
}
ExteroceptiveCost* Optimizer::add(ManifoldObservation& obs) {
  manifold_obs_.push_back(&obs);
  if (std::find(pose_sensors_.begin(), pose_sensors_.end(), obs.sensor) == pose_sensors_.end()) pose_sensors_.push_back(obs.sensor);
  costs_.emplace_back(new ExteroceptiveCost(this, ExteroceptiveCost::kManifold, static_cast<Index>(manifold_obs_.size() - 1)));
  dirty_ = true;
  return costs_.back().get();
}

void Optimizer::upload(bool factors) {
  if (!state_) throw std::logic_error("Optimizer: state not set");
  const auto& el = state_->elements();
  const int K = static_cast<int>(el.size()), order = state_->interpolator()->layout().outer.size;
  knots_.resize(8 * static_cast<size_t>(K));
  for (int j = 0; j < K; ++j) std::copy(el[j].v.begin(), el[j].v.end(), knots_.begin() + 8 * j);
  check(hb200_set_spline(ctx_, order, K, knots_.data()), "hb200_set_spline");
  if (imu_) {
    auto flat = [](std::vector<IMU::Bias>& b, std::vector<double>& out) { out.resize(4 * b.size()); for (size_t j = 0; j < b.size(); ++j) std::copy(b[j].v.begin(), b[j].v.end(), out.begin() + 4 * j); };
    flat(imu_->gyroscopeBias(), bg_); flat(imu_->accelerometerBias(), ba_);
    check(hb200_set_bias_splines(ctx_, 4, static_cast<int>(bg_.size() / 4), bg_.data(), static_cast<int>(ba_.size() / 4), ba_.data()), "hb200_set_bias_splines");
    double blk[37];
    auto v = imu_->variables();
    const int sizes[5] = {7, 6, 6, 9, 9};
    int o = 0;
    for (int b = 0; b < 5; ++b) { std::copy(v[b], v[b] + sizes[b], blk + o); o += sizes[b]; }
    check(hb200_set_imu(ctx_, blk), "hb200_set_imu");
  }
  if (gravity_) check(hb200_set_gravity(ctx_, gravity_->data()), "hb200_set_gravity");
  if (!cameras_.empty()) {
    std::vector<double> cams(15 * cameras_.size());
    for (size_t c = 0; c < cameras_.size(); ++c) {
      auto v = cameras_[c]->variables();
      std::copy(v[0], v[0] + 7, cams.begin() + 15 * c); std::copy(v[1], v[1] + 4, cams.begin() + 15 * c + 7); std::copy(v[2], v[2] + 4, cams.begin() + 15 * c + 11);
    }
    check(hb200_set_cameras(ctx_, static_cast<int>(cameras_.size()), cams.data()), "hb200_set_cameras");
  }
  lms_.resize(3 * landmarks_.size());
  for (size_t l = 0; l < landmarks_.size(); ++l) std::copy(landmarks_[l]->variable.v.begin(), landmarks_[l]->variable.v.end(), lms_.begin() + 3 * l);
  check(hb200_set_landmarks(ctx_, static_cast<int>(landmarks_.size()), lms_.data()), "hb200_set_landmarks");
  if (!pose_sensors_.empty()) {
    std::vector<double> T(7 * pose_sensors_.size());
    for (size_t i = 0; i < pose_sensors_.size(); ++i) std::copy(pose_sensors_[i]->transformation().v.begin(), pose_sensors_[i]->transformation().v.end(), T.begin() + 7 * i);
    check(hb200_set_pose_sensors(ctx_, static_cast<int>(pose_sensors_.size()), T.data()), "hb200_set_pose_sensors");
  }
  if (factors) {
    std::vector<double> vs, vp, is, im;
    std::vector<int> vc, vl;
    for (auto* o : pixel_obs_) { vs.push_back(o->stamp); vc.push_back(cameraIndex(o->camera)); vl.push_back(landmarkIndex(o->landmark)); vp.push_back(o->measurement[0]); vp.push_back(o->measurement[1]); }
    for (auto* o : inertial_obs_) { is.push_back(o->stamp); for (int i = 0; i < 6; ++i) im.push_back(o->measurement[i]); }
    check(hb200_set_pixel_factors(ctx_, static_cast<int>(vs.size()), vs.data(), vc.data(), vl.data(), vp.data()), "hb200_set_pixel_factors");
    check(hb200_set_inertial_factors(ctx_, static_cast<int>(is.size()), is.data(), im.data()), "hb200_set_inertial_factors");
    std::vector<double> bs, bm, ms, mm;
    std::vector<int> bc, bl, msens;
    for (auto* o : bearing_obs_) { bs.push_back(o->stamp); bc.push_back(cameraIndex(o->camera)); bl.push_back(landmarkIndex(o->landmark)); for (int i = 0; i < 3; ++i) bm.push_back(o->measurement[i]); }
    for (auto* o : manifold_obs_) {
      ms.push_back(o->stamp);
      msens.push_back(static_cast<int>(std::find(pose_sensors_.begin(), pose_sensors_.end(), o->sensor) - pose_sensors_.begin()));
      for (int i = 0; i < 7; ++i) mm.push_back(o->measurement.v[i]);
    }
    check(hb200_set_bearing_factors(ctx_, static_cast<int>(bs.size()), bs.data(), bc.data(), bl.data(), bm.data()), "hb200_set_bearing_factors");
    check(hb200_set_manifold_factors(ctx_, static_cast<int>(ms.size()), ms.data(), msens.data(), mm.data()), "hb200_set_manifold_factors");
    int bad = 0;
    check(hb200_bind(ctx_, &bad), "hb200_bind");                       // == cost->update() for every cost
    std::vector<unsigned char> kc(K, 0);
    for (int j = 0; j < K && j < static_cast<int>(constant_.size()); ++j) kc[j] = constant_[j];
    check(hb200_set_constant(ctx_, kc.data(), gravity_constant_ ? 1 : 0, 0), "hb200_set_constant");
    dirty_ = false;
  }
}

void Optimizer::download() {
  const int K = static_cast<int>(state_->elements().size());
  bg_.resize(imu_ ? 4 * imu_->gyroscopeBias().size() : 0); ba_.resize(imu_ ? 4 * imu_->accelerometerBias().size() : 0);
  grav_.assign(3, 0.0);
  check(hb200_get_state(ctx_, knots_.data(), bg_.empty() ? nullptr : bg_.data(), ba_.empty() ? nullptr : ba_.data(), grav_.data(), lms_.empty() ? nullptr : lms_.data()), "hb200_get_state");
  for (int j = 0; j < K; ++j) std::copy(knots_.begin() + 8 * j, knots_.begin() + 8 * j + 8, state_->elements()[j].v.begin());
  if (imu_) {
    for (size_t j = 0; j < imu_->gyroscopeBias().size(); ++j) std::copy(bg_.begin() + 4 * j, bg_.begin() + 4 * j + 4, imu_->gyroscopeBias()[j].v.begin());
    for (size_t j = 0; j < imu_->accelerometerBias().size(); ++j) std::copy(ba_.begin() + 4 * j, ba_.begin() + 4 * j + 4, imu_->accelerometerBias()[j].v.begin());
  }
  if (gravity_) std::copy(grav_.begin(), grav_.end(), gravity_->v.begin());
  for (size_t l = 0; l < landmarks_.size(); ++l) std::copy(lms_.begin() + 3 * l, lms_.begin() + 3 * l + 3, landmarks_[l]->variable.v.begin());
}

void Optimizer::prepareForEvaluation(bool evaluate_jacobians) {
  upload(dirty_);
  check(hb200_evaluate(ctx_, evaluate_jacobians ? HB200_EVAL_JACOBIANS : 0), "hb200_evaluate");
}

std::vector<IterationSummary> Optimizer::optimize(int max_num_iterations) {
  upload(dirty_);
  std::vector<hb200_iteration> rec(max_num_iterations);
  check(hb200_iterate(ctx_, max_num_iterations, rec.data()), "hb200_iterate");
  download();
  int performed = max_num_iterations, type = 0;
  hb200_get_termination(ctx_, &type, &performed, nullptr, nullptr, nullptr);   // fewer when a termination test fired
  std::vector<IterationSummary> out;
  for (int i = 0; i < std::min(performed, max_num_iterations); ++i) {
    const auto& r = rec[i];
    out.push_back({r.cost, r.cost_new, r.rho, r.radius, r.accepted != 0, r.spd != 0});
  }
  return out;
}

// ---------------------------------------------------------------------------------------------
// ExteroceptiveCost
// ---------------------------------------------------------------------------------------------
Pointers<Scalar> ExteroceptiveCost::update() {
  Optimizer& o = *optimizer_;
  Pointers<Scalar> p;
  layout_ = EvaluatorLayout{};
  const Stamp stamp = (kind_ == kPixel) ? o.pixel_obs_[index_]->stamp : (kind_ == kInertial) ? o.inertial_obs_[index_]->stamp
                    : (kind_ == kBearing) ? o.bearing_obs_[index_]->stamp : o.manifold_obs_[index_]->stamp;
  auto state_blocks = o.state_->parameters(stamp);
  if (state_blocks.empty()) throw std::out_of_range("ExteroceptiveCost::update: stamp outside the state's range");
  for (auto* b : state_blocks) { p.push_back(b); layout_.sizes.push_back(8); }
  layout_.indices.static_state_idx = 0;
  layout_.indices.static_sensor_idx = static_cast<Index>(p.size());
  if (kind_ == kPixel || kind_ == kBearing) {
    const Camera* camera = (kind_ == kPixel) ? o.pixel_obs_[index_]->camera : o.bearing_obs_[index_]->camera;
    Landmark* landmark = (kind_ == kPixel) ? o.pixel_obs_[index_]->landmark : o.bearing_obs_[index_]->landmark;
    auto v = const_cast<Camera*>(camera)->variables();
    const int sizes[3] = {7, 4, 4};
    for (int b = 0; b < 3; ++b) { p.push_back(v[b]); layout_.sizes.push_back(sizes[b]); }
    layout_.indices.dynamic_sensor_idx = static_cast<Index>(p.size());
    layout_.indices.static_observation_idx = static_cast<Index>(p.size());
    p.push_back(landmark->variable.data()); layout_.sizes.push_back(3);
    num_residuals_ = (kind_ == kPixel) ? 2 : 1;   // CartesianMetric<Pixel> / AngularMetric<Bearing>
  } else if (kind_ == kManifold) {
    auto* obs = o.manifold_obs_[index_];
    p.push_back(const_cast<Sensor*>(obs->sensor)->transformation().data()); layout_.sizes.push_back(7);
    layout_.indices.dynamic_sensor_idx = static_cast<Index>(p.size());
    layout_.indices.static_observation_idx = static_cast<Index>(p.size());   // no observation variables
    num_residuals_ = 6;                           // ManifoldMetric<SE3>
  } else {
    auto* obs = o.inertial_obs_[index_];
    IMU* imu = const_cast<IMU*>(obs->imu);
    auto v = imu->variables();
    const int sizes[5] = {7, 6, 6, 9, 9};
    for (int b = 0; b < 5; ++b) { p.push_back(v[b]); layout_.sizes.push_back(sizes[b]); }
    layout_.indices.dynamic_sensor_idx = static_cast<Index>(p.size());
    auto bias_blocks = [&](std::vector<IMU::Bias>& knots) {
      auto it = std::upper_bound(knots.begin(), knots.end(), stamp, [](Stamp s, const IMU::Bias& e) { return s < e.stamp(); });
      const int base = static_cast<int>(it - knots.begin()) - 1 - 1;   // order 4: left padding 1
      if (base < 0 || base + 3 >= static_cast<int>(knots.size())) throw std::out_of_range("inertial stamp outside the bias spline's valid range");
      for (int m = 0; m < 4; ++m) { p.push_back(knots[base + m].data()); layout_.sizes.push_back(4); }
    };
    bias_blocks(imu->gyroscopeBias());
    bias_blocks(imu->accelerometerBias());
    layout_.indices.static_observation_idx = static_cast<Index>(p.size());
    p.push_back(obs->gravity->data()); layout_.sizes.push_back(3);
    num_residuals_ = 6;
  }
  layout_.offsets.assign(layout_.sizes.size(), 0);
  for (size_t i = 1; i < layout_.sizes.size(); ++i) layout_.offsets[i] = layout_.offsets[i - 1] + layout_.sizes[i - 1];
  layout_.num_parameters = layout_.offsets.back() + layout_.sizes.back();
  return p;
}

bool ExteroceptiveCost::Evaluate(const double* const* parameters, double* residuals, double** jacobians) const {
  return hb200_factor_evaluate(optimizer_->ctx_, static_cast<int>(kind_), index_, parameters, residuals, jacobians) == 0;
}

// ---------------------------------------------------------------------------------------------
// Covariance
// ---------------------------------------------------------------------------------------------
bool Covariance::locate(const double* p, Block* b) const {
  const Optimizer& o = optimizer_;
  const int K = static_cast<int>(o.state_->elements().size());
  const int Kbg = o.imu_ ? static_cast<int>(o.imu_->gyroscopeBias().size()) : 0;
  const int Kba = o.imu_ ? static_cast<int>(o.imu_->accelerometerBias().size()) : 0;
  for (int j = 0; j < K; ++j)
    if (o.state_->elements()[j].data() == p) { *b = {kState, j, 6 * j, 6, 8}; return true; }
  for (int j = 0; j < Kbg; ++j)
    if (o.imu_->gyroscopeBias()[j].data() == p) { *b = {kGyroBias, j, 6 * K + 3 * j, 3, 4}; return true; }
  for (int j = 0; j < Kba; ++j)
    if (o.imu_->accelerometerBias()[j].data() == p) { *b = {kAccelBias, j, 6 * K + 3 * Kbg + 3 * j, 3, 4}; return true; }
  if (o.gravity_ && o.gravity_->data() == p) { *b = {kGravity, 0, 6 * K + 3 * (Kbg + Kba), 2, 3}; return true; }
  for (size_t l = 0; l < o.landmarks_.size(); ++l)
    if (o.landmarks_[l]->variable.data() == p) { *b = {kLandmark, static_cast<int>(l), -1, 3, 3}; return true; }
  return false;
}

bool Covariance::inPattern(const Block& a, const Block& b, int beta) const {
  if (a.kind == kLandmark || b.kind == kLandmark) return a.kind == b.kind && a.index == b.index;
  if (a.kind == kState && b.kind == kState) return std::abs(a.index - b.index) <= beta;
  return true;   // arrow and corner
}

Manifold Covariance::manifold(const Block& b) const {
  switch (b.kind) {
    case kState: return Manifold::StampedSE3(true, false, false);
    case kGyroBias:
    case kAccelBias: return Manifold::StampedEuclidean(3, true, false);
    case kGravity: return Manifold::Sphere(3);
    default: return Manifold::Euclidean(3);
  }
}

bool Covariance::Compute(const std::vector<std::pair<const double*, const double*>>& blocks) {
  Optimizer& o = optimizer_;
  if (!o.state_) return false;
  o.upload(o.dirty_);   // the device window == the host variables (as Ceres evaluates at the values it aliases)
  int beta = 0;
  check(hb200_get_bandwidth(o.ctx_, &beta), "hb200_get_bandwidth");
  // pairs outside the pattern as hb200_set_covariance_blocks requests (kind, index, kind, index)
  static constexpr int kKind[] = {HB200_COV_KNOT, HB200_COV_GYRO_BIAS, HB200_COV_ACCEL_BIAS, HB200_COV_GRAVITY, HB200_COV_LANDMARK};
  std::vector<int> requests;
  std::vector<std::pair<const double*, const double*>> outside;
  for (const auto& [pa, pb] : blocks) {
    Block a, b;
    if (!locate(pa, &a) || !locate(pb, &b)) return false;
    if (inPattern(a, b, beta)) continue;
    if (!options_.full_pattern) return false;
    requests.insert(requests.end(), {kKind[a.kind], a.index, kKind[b.kind], b.index});
    outside.emplace_back(pa, pb);
  }
  const int nreq = static_cast<int>(outside.size());
  check(hb200_set_covariance_blocks(o.ctx_, nreq, requests.data()), "hb200_set_covariance_blocks");
  check(hb200_build_covariance(o.ctx_), "hb200_build_covariance");
  hb200_covariance_info info{};
  const int rc = hb200_compute_covariance(o.ctx_, &info);
  info_ = info;
  if (rc == HB200_COV_NOT_POSITIVE_DEFINITE || rc == HB200_COV_DEGENERATE_LANDMARKS) return false;
  check(rc, "hb200_compute_covariance");
  packed_.assign(static_cast<size_t>(info.K) * (6 + 6 * info.beta) * 6 + static_cast<size_t>(info.m) * 6 * info.K + static_cast<size_t>(info.m) * info.m, 0.0);
  landmarks_.assign(9 * static_cast<size_t>(info.L), 0.0);
  check(hb200_get_covariance(o.ctx_, packed_.data(), landmarks_.empty() ? nullptr : landmarks_.data()), "hb200_get_covariance");
  std::vector<double> slots(36 * static_cast<size_t>(nreq));
  check(hb200_get_covariance_blocks(o.ctx_, nreq, slots.data(), nullptr), "hb200_get_covariance_blocks");
  outside_.clear();
  for (int q = 0; q < nreq; ++q) {   // (status 1, a landmark on another rank, cannot occur on one GPU; status 2 is a zero block)
    Block a, b;
    locate(outside[q].first, &a);
    locate(outside[q].second, &b);
    std::vector<double>& t = outside_[outside[q]];
    t.resize(static_cast<size_t>(a.tangent) * b.tangent);
    for (int i = 0; i < a.tangent; ++i)
      for (int j = 0; j < b.tangent; ++j) t[static_cast<size_t>(i) * b.tangent + j] = slots[36 * static_cast<size_t>(q) + 6 * i + j];
  }
  beta_ = info.beta; K_ = info.K; n_ = 6 * info.K + info.m;
  computed_ = blocks;
  values_.clear();
  for (const auto& [pa, pb] : blocks)
    for (const double* p : {pa, pb}) {
      Block b;
      locate(p, &b);
      values_[p] = std::vector<double>(p, p + b.ambient);
    }
  return true;
}

bool Covariance::tangentBlock(const double* pa, const double* pb, std::vector<double>* out, Block* a, Block* b) const {
  bool found = false;
  for (const auto& [x, y] : computed_) found = found || (x == pa && y == pb) || (x == pb && y == pa);
  if (!found || !locate(pa, a) || !locate(pb, b)) return false;
  out->assign(static_cast<size_t>(a->tangent) * b->tangent, 0.0);
  // Ceres' quaternion tangent: delta = theta / 2
  auto scale = [](const Block& bl, int i) { return (bl.kind == kState && i < 3) ? 0.5 : 1.0; };
  const auto ab = outside_.find({pa, pb}), ba = outside_.find({pb, pa});
  if (ab != outside_.end() || ba != outside_.end()) {   // outside the pattern: (b, a) is the transpose of (a, b)
    for (int i = 0; i < a->tangent; ++i)
      for (int j = 0; j < b->tangent; ++j) {
        const double v = ab != outside_.end() ? ab->second[static_cast<size_t>(i) * b->tangent + j] : ba->second[static_cast<size_t>(j) * a->tangent + i];
        (*out)[static_cast<size_t>(i) * b->tangent + j] = scale(*a, i) * v * scale(*b, j);
      }
    return true;
  }
  if (a->kind == kLandmark) {   // (same landmark: the only landmark pair in the pattern)
    for (int i = 0; i < 9; ++i) (*out)[i] = landmarks_[9 * static_cast<size_t>(a->index) + i];
    return true;
  }
  // entry (r, c), r >= c, of the packed P | A | C layout (diagonal blocks and corner stored in full)
  const int np = 6 * K_, h = 6 + 6 * beta_, m = n_ - np;
  auto at = [&](int r, int c) {
    if (r < c) std::swap(r, c);
    if (r < np) { const int cb = c / 6; return packed_[(static_cast<size_t>(cb) * h + (r - 6 * cb)) * 6 + (c - 6 * cb)]; }
    if (c < np) return packed_[static_cast<size_t>(K_) * h * 6 + static_cast<size_t>(r - np) * np + c];
    return packed_[static_cast<size_t>(K_) * h * 6 + static_cast<size_t>(m) * np + static_cast<size_t>(r - np) * m + (c - np)];
  };
  for (int i = 0; i < a->tangent; ++i)
    for (int j = 0; j < b->tangent; ++j) (*out)[static_cast<size_t>(i) * b->tangent + j] = scale(*a, i) * at(a->dof + i, b->dof + j) * scale(*b, j);
  return true;
}

bool Covariance::GetCovarianceBlockInTangentSpace(const double* pa, const double* pb, double* cov) const {
  std::vector<double> T;
  Block a, b;
  if (!tangentBlock(pa, pb, &T, &a, &b)) return false;
  std::copy(T.begin(), T.end(), cov);
  return true;
}

bool Covariance::GetCovarianceBlock(const double* pa, const double* pb, double* cov) const {
  std::vector<double> T;
  Block a, b;
  if (!tangentBlock(pa, pb, &T, &a, &b)) return false;
  const Manifold ma = manifold(a), mb = manifold(b);
  const int ta = ma.TangentSize(), tb = mb.TangentSize();
  std::vector<double> Pa(static_cast<size_t>(a.ambient) * ta), Pb(static_cast<size_t>(b.ambient) * tb);
  ma.PlusJacobian(values_.at(pa).data(), Pa.data());
  mb.PlusJacobian(values_.at(pb).data(), Pb.data());
  // P_a T P_b^T
  for (int r = 0; r < a.ambient; ++r)
    for (int c = 0; c < b.ambient; ++c) {
      double s = 0.0;
      for (int i = 0; i < ta; ++i)
        for (int j = 0; j < tb; ++j) s += Pa[static_cast<size_t>(r) * ta + i] * T[static_cast<size_t>(i) * tb + j] * Pb[static_cast<size_t>(c) * tb + j];
      cov[static_cast<size_t>(r) * b.ambient + c] = s;
    }
  return true;
}

}  // namespace hyper
