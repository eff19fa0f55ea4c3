// hyper::Optimizer<H100> and the Ceres-shaped cost functor over libhyperb200
// (mirrors reference include/hyper/optimizers/{abstract,ceres/optimizer}.hpp and
//  include/hyper/optimizers/ceres/costs/exteroceptive.hpp; see INTEGRATION.md).
#pragma once
#include <memory>
#include <string>
#include <vector>

#include "hyper/manifolds.hpp"
#include "hyper/sensors.hpp"
#include "hyper/state.hpp"

struct hb200_ctx;

namespace hyper {

struct Landmark { Position variable; };

struct VisualPixelObservation { Stamp stamp; const Camera* camera; Landmark* landmark; Pixel measurement; };
struct InertialObservation { Stamp stamp; const IMU* imu; Gravity* gravity; Tangent6 measurement; };
// Bearing = direction of the landmark in the sensor frame (reference optimizers/evaluators/bearing.cpp:14-79).
struct VisualBearingObservation { Stamp stamp; const Camera* camera; Landmark* landmark; Position measurement; };
// ManifoldObservation<SE3>: a measured T_ws of a plain Sensor (reference optimizers/evaluators/manifold.cpp:12-61).
struct ManifoldObservation { Stamp stamp; const Sensor* sensor; SE3 measurement; };

// Evaluator layout of one cost (reference include/hyper/optimizers/evaluators/forward.hpp:19-39).
struct EvaluatorLayout {
  Index num_parameters = 0;
  struct Indices { Index static_state_idx, static_sensor_idx, dynamic_sensor_idx, static_observation_idx; } indices{};
  std::vector<Index> offsets;
  std::vector<int> sizes;
};

class CostFunction {   // the slice of ceres::CostFunction the reference relies on
 public:
  virtual ~CostFunction() = default;
  virtual bool Evaluate(const double* const* parameters, double* residuals, double** jacobians) const = 0;
  int num_residuals() const { return num_residuals_; }
  const std::vector<int>& parameter_block_sizes() const { return layout_.sizes; }
 protected:
  int num_residuals_ = 0;
  EvaluatorLayout layout_;
};

class Optimizer;

// One per observation; Evaluate() is a copy-out of the batched device evaluation
// (reference internal/hyper/optimizers/ceres/costs/exteroceptive.cpp:101-160).
class ExteroceptiveCost final : public CostFunction {
 public:
  enum Kind { kPixel = 0, kInertial = 1, kBearing = 2, kManifold = 3 };
  // Collects the parameter-block pointers in reference order and fills the layout (exteroceptive.cpp:25-99).
  Pointers<Scalar> update();
  bool Evaluate(const double* const* parameters, double* residuals, double** jacobians) const override;
  const EvaluatorLayout& layout() const { return layout_; }
  Kind kind() const { return kind_; }
  Index index() const { return index_; }
 private:
  friend class Optimizer;
  ExteroceptiveCost(Optimizer* optimizer, Kind kind, Index index) : optimizer_{optimizer}, kind_{kind}, index_{index} {}
  Optimizer* optimizer_;
  Kind kind_;
  Index index_;
};

struct IterationSummary { double cost, cost_new, rho, radius; bool accepted, spd; };

class Optimizer {   // OptimizerSuite::H100
 public:
  explicit Optimizer(int device = 0);
  ~Optimizer();
  Optimizer(const Optimizer&) = delete;
  Optimizer& operator=(const Optimizer&) = delete;

  void setState(ContinuousState* state) { state_ = state; dirty_ = true; }
  void setCameras(std::vector<Camera*> cameras) { cameras_ = std::move(cameras); dirty_ = true; }
  void setIMU(IMU* imu) { imu_ = imu; dirty_ = true; }
  void setGravity(Gravity* gravity) { gravity_ = gravity; }
  void addLandmark(Landmark& landmark) { landmarks_.push_back(&landmark); dirty_ = true; }       // reference optimizer.cpp:347-358
  ExteroceptiveCost* add(VisualPixelObservation& observation);                                   // reference optimizer.cpp:212-232
  ExteroceptiveCost* add(InertialObservation& observation);                                      // reference optimizer.cpp:253-274
  ExteroceptiveCost* add(VisualBearingObservation& observation);                                 // reference optimizer.cpp:189-210
  ExteroceptiveCost* add(ManifoldObservation& observation);                                      // reference optimizer.cpp:234-251
  void setStateConstant(const std::vector<bool>& constant) { constant_ = constant; dirty_ = true; }
  void setGravityConstant(bool constant) { gravity_constant_ = constant; dirty_ = true; }          // reference abstract.cpp:57-61

  // ceres::EvaluationCallback::PrepareForEvaluation: one batched device evaluation of every cost.
  void prepareForEvaluation(bool evaluate_jacobians = true);
  // CeresOptimizer::optimize (reference optimizer.cpp:276-280): <= max_num_iterations LM iterations,
  // variables updated in place.
  std::vector<IterationSummary> optimize(int max_num_iterations = 5);
  // ceres::Solver::Options termination tests, evaluated on the device (hb200_set_termination); the reference keeps Ceres'
  // defaults (reference optimizer.cpp:38-54): setSolverTolerances() with no arguments switches exactly those on.
  void setSolverTolerances(double function_tolerance = 1e-6, double gradient_tolerance = 1e-10, double parameter_tolerance = 1e-8,
                           double min_trust_region_radius = 1e-32);
  // summary.termination_type of the last optimize(): 0 iteration limit, 1 function, 2 parameter, 3 gradient tolerance, 4 radius, 5 invalid steps
  int terminationType() const;

  hb200_ctx* context() { return ctx_; }
  const ContinuousState& state() const { return *state_; }

 private:
  friend class ExteroceptiveCost;
  void upload(bool factors);
  void download();
  Index cameraIndex(const Camera* camera) const;
  Index landmarkIndex(const Landmark* landmark) const;

  hb200_ctx* ctx_ = nullptr;
  ContinuousState* state_ = nullptr;
  std::vector<Camera*> cameras_;
  IMU* imu_ = nullptr;
  Gravity* gravity_ = nullptr;
  std::vector<Landmark*> landmarks_;
  std::vector<VisualPixelObservation*> pixel_obs_;
  std::vector<InertialObservation*> inertial_obs_;
  std::vector<VisualBearingObservation*> bearing_obs_;
  std::vector<ManifoldObservation*> manifold_obs_;
  std::vector<const Sensor*> pose_sensors_;   // distinct sensors of the manifold observations, in order of first use
  std::vector<std::unique_ptr<ExteroceptiveCost>> costs_;
  std::vector<bool> constant_;
  bool gravity_constant_ = false;
  bool dirty_ = true;
  // flat mirrors handed to the C-ABI
  std::vector<double> knots_, bg_, ba_, lms_, grav_;
};

}  // namespace hyper
