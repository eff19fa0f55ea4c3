// hyper::Covariance -- ceres::Covariance (default options: loss applied, constant blocks get zero covariance) over the
// device's selected inverse (hb200_build_covariance / hb200_compute_covariance, include/hyperb200.h).
//
// Parameter blocks are the optimizer's own variables, named by their data pointers as in Ceres: state elements
// (Stamped<SE3>, 8 doubles), gyroscope / accelerometer bias knots (Stamped<R3>, 4), gravity (3, on the sphere) and
// landmarks (3).  The selected inverse covers every pair of state elements at most beta control points apart (beta =
// the window's block half-bandwidth, hb200_get_bandwidth), every pair involving a bias knot or gravity, and each
// landmark with itself.  By default those are the pairs Compute accepts: for landmark cross-covariances and state pairs
// further apart it returns false, as Ceres does for a pair it cannot compute.  With Options::full_pattern, Compute
// accepts any pair, as ceres::Covariance::Compute(covariance_blocks) does, and has the device compute the pairs outside
// the pattern with the same compute (hb200_set_covariance_blocks); a landmark without observations gets a zero block.
//
// Tangent spaces are Ceres': a state element's quaternion tangent is delta = theta / 2 of the device's global rotation
// tangent, so its tangent-space block is T S T^T with T = diag(1/2 I3, I3) (the stamp is constant, no tangent); biases,
// gravity (SphereManifold<3>) and landmarks share the device's tangent.  GetCovarianceBlock returns ambient blocks
// P_a (T S T^T) P_b^T with P the block's Manifold::PlusJacobian at the values Compute saw.
#pragma once
#include <map>
#include <utility>
#include <vector>

#include "../../../../include/hyperb200.h"
#include "hyper/optimizer.hpp"

namespace hyper {

class Covariance {
 public:
  // The counterpart of ceres::Covariance::Options.
  struct Options {
    // Compute accepts every pair of parameter blocks, not only those inside the selected inverse's pattern.
    bool full_pattern = false;
  };
  explicit Covariance(Optimizer& optimizer) : Covariance(optimizer, Options{}) {}
  Covariance(Optimizer& optimizer, const Options& options) : optimizer_{optimizer}, options_{options} {}
  // Evaluates the undamped Gauss-Newton matrix at the optimizer's current state and computes the covariance.  false: a
  // pair outside the computed pattern (without Options::full_pattern) or an unknown block (nothing is computed), or the
  // system is not positive definite / has a degenerate landmark (info() says which; results of an earlier Compute stay
  // readable).
  bool Compute(const std::vector<std::pair<const double*, const double*>>& covariance_blocks);
  // Row-major, ambient a x ambient b.  false for a pair that was not part of the last successful Compute.
  bool GetCovarianceBlock(const double* a, const double* b, double* covariance_block) const;
  // Row-major, tangent a x tangent b (Ceres' tangent spaces).
  bool GetCovarianceBlockInTangentSpace(const double* a, const double* b, double* covariance_block) const;
  const hb200_covariance_info& info() const { return info_; }

 private:
  enum Kind { kState, kGyroBias, kAccelBias, kGravity, kLandmark };
  struct Block {
    Kind kind = kState;
    int index = -1;     // element / knot / landmark index
    int dof = -1;       // first device dof (reduced-system order), -1 for landmarks
    int tangent = 0;    // device tangent size
    int ambient = 0;
  };
  bool locate(const double* p, Block* b) const;
  bool inPattern(const Block& a, const Block& b, int beta) const;
  Manifold manifold(const Block& b) const;
  bool tangentBlock(const double* a, const double* b, std::vector<double>* out, Block* ba, Block* bb) const;

  Optimizer& optimizer_;
  Options options_;
  hb200_covariance_info info_{};
  int beta_ = 0, n_ = 0, K_ = 0;
  std::vector<double> packed_, landmarks_;
  std::vector<std::pair<const double*, const double*>> computed_;
  // pairs outside the pattern (Options::full_pattern): their device-tangent blocks, t_a x t_b row-major
  std::map<std::pair<const double*, const double*>, std::vector<double>> outside_;
  std::map<const double*, std::vector<double>> values_;   // block values at Compute (PlusJacobian point)
};

}  // namespace hyper
