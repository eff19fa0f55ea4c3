// GPU test of Optimizer::setWeights (CostConfiguration::weights): reads a flat window dump and one row-major matrix per
// family (tests/test_gpu_host_weights.py), and checks through ExteroceptiveCost::Evaluate that
//  (1) a weighted cost returns W r and W J for every parameter block, calibration blocks included, against the same cost
//      evaluated without a matrix (row-scale bound), the inertial bias blocks exactly wg[m] W[:, 0:3] / wa[m] W[:, 3:6];
//  (2) the reference's Probe protocol passes on the weighted costs with every block non-constant
//      (reference tests/include/tests/optimizers/evaluators/evaluator.hpp:26-65);
//  (3) clearing the matrices gives the unweighted outputs back bit for bit.
#include <cmath>
#include <cstdio>
#include <fstream>
#include <iostream>
#include <memory>

#include "hyper/optimizer.hpp"

using namespace hyper;

static std::vector<double> readv(std::istream& in, size_t n) { std::vector<double> v(n); for (auto& x : v) in >> x; return v; }

struct Eval { std::vector<double> r; std::vector<std::vector<double>> J; };

int main(int argc, char** argv) {
  if (argc < 3) { std::fprintf(stderr, "usage: weights_test <window.txt> <weights.txt>\n"); return 2; }
  std::ifstream in(argv[1]);
  if (!in) { std::fprintf(stderr, "cannot open %s\n", argv[1]); return 2; }
  int order, K, Kb, C, L, Nv, Ni, nconst, Nb, Nm, P;
  in >> order >> K >> Kb >> C >> L >> Nv >> Ni >> nconst >> Nb >> Nm >> P;
  ContinuousState state(std::make_unique<BasisInterpolator>(order - 1, true));
  for (int j = 0; j < K; ++j) { ContinuousState::Element e; for (int i = 0; i < 8; ++i) in >> e.v[i]; state.elements().push_back(e); }
  IMU imu;
  for (int j = 0; j < Kb; ++j) { IMU::Bias b; for (int i = 0; i < 4; ++i) in >> b.v[i]; imu.gyroscopeBias().push_back(b); }
  for (int j = 0; j < Kb; ++j) { IMU::Bias b; for (int i = 0; i < 4; ++i) in >> b.v[i]; imu.accelerometerBias().push_back(b); }
  Gravity gravity; for (int i = 0; i < 3; ++i) in >> gravity[i];
  std::vector<std::unique_ptr<Camera>> cams;
  for (int c = 0; c < C; ++c) {
    cams.emplace_back(new Camera());
    for (int i = 0; i < 7; ++i) in >> cams[c]->transformation().v[i];
    for (int i = 0; i < 4; ++i) in >> cams[c]->intrinsics()[i];
    for (int i = 0; i < 4; ++i) in >> cams[c]->distortion()[i];
  }
  { auto v = readv(in, 37); auto p = imu.variables(); const int s[5] = {7, 6, 6, 9, 9}; int o = 0; for (int b = 0; b < 5; ++b) { std::copy(v.begin() + o, v.begin() + o + s[b], p[b]); o += s[b]; } }
  std::vector<Landmark> lms(L);
  for (int l = 0; l < L; ++l) for (int i = 0; i < 3; ++i) in >> lms[l].variable[i];
  std::vector<VisualPixelObservation> vobs(Nv);
  for (int f = 0; f < Nv; ++f) { int c, l; in >> vobs[f].stamp >> c >> l >> vobs[f].measurement[0] >> vobs[f].measurement[1]; if (!in || c < 0 || c >= C || l < 0 || l >= L) { std::fprintf(stderr, "malformed pixel factor %d\n", f); return 2; } vobs[f].camera = cams[c].get(); vobs[f].landmark = &lms[l]; }
  std::vector<InertialObservation> iobs(Ni);
  for (int f = 0; f < Ni; ++f) { in >> iobs[f].stamp; for (int i = 0; i < 6; ++i) in >> iobs[f].measurement[i]; iobs[f].imu = &imu; iobs[f].gravity = &gravity; }
  std::vector<VisualBearingObservation> bobs(Nb);
  for (int f = 0; f < Nb; ++f) { int c, l; in >> bobs[f].stamp >> c >> l; for (int i = 0; i < 3; ++i) in >> bobs[f].measurement[i]; bobs[f].camera = cams[c].get(); bobs[f].landmark = &lms[l]; }
  std::vector<Sensor> pose_sensors(P);
  for (int p = 0; p < P; ++p) for (int i = 0; i < 7; ++i) in >> pose_sensors[p].transformation().v[i];
  std::vector<ManifoldObservation> mobs(Nm);
  for (int f = 0; f < Nm; ++f) { int sidx; in >> mobs[f].stamp >> sidx; for (int i = 0; i < 7; ++i) in >> mobs[f].measurement.v[i]; mobs[f].sensor = &pose_sensors[sidx]; }
  if (!in) { std::fprintf(stderr, "window file is truncated\n"); return 2; }
  Optimizer optimizer(0);
  optimizer.setState(&state);
  std::vector<Camera*> cam_ptrs; for (auto& c : cams) cam_ptrs.push_back(c.get());
  optimizer.setCameras(cam_ptrs);
  optimizer.setIMU(&imu);
  optimizer.setGravity(&gravity);
  for (auto& l : lms) optimizer.addLandmark(l);
  std::vector<ExteroceptiveCost*> vcosts, icosts, bcosts, mcosts;
  for (auto& o : vobs) vcosts.push_back(optimizer.add(o));
  for (auto& o : iobs) icosts.push_back(optimizer.add(o));
  for (auto& o : bobs) bcosts.push_back(optimizer.add(o));
  for (auto& o : mobs) mcosts.push_back(optimizer.add(o));
  std::vector<bool> constant(K, false); for (int j = 0; j < nconst; ++j) constant[j] = true;
  optimizer.setStateConstant(constant);

  std::ifstream win(argv[2]);
  const size_t sides[4] = {2, 6, 1, 6};   // ExteroceptiveCost::Kind order
  std::vector<double> W[4];
  for (int f = 0; f < 4; ++f) W[f] = readv(win, sides[f] * sides[f]);
  if (!win) { std::fprintf(stderr, "malformed weights file\n"); return 2; }

  auto eval = [&](ExteroceptiveCost* cost) {
    auto params = cost->update();
    const int nr = cost->num_residuals();
    const auto& sizes = cost->parameter_block_sizes();
    Eval e{std::vector<double>(nr), std::vector<std::vector<double>>(params.size())};
    std::vector<double*> jp(params.size());
    for (size_t b = 0; b < params.size(); ++b) { e.J[b].assign(static_cast<size_t>(nr) * sizes[b], 0.0); jp[b] = e.J[b].data(); }
    cost->Evaluate(params.data(), e.r.data(), jp.data());
    return e;
  };
  std::vector<ExteroceptiveCost*> picked;
  for (auto* v : {&vcosts, &icosts, &bcosts, &mcosts}) if (!v->empty()) { picked.push_back(v->front()); picked.push_back(v->back()); }
  optimizer.prepareForEvaluation(true);
  std::vector<Eval> plain;
  for (auto* c : picked) plain.push_back(eval(c));

  for (int f = 0; f < 4; ++f) optimizer.setWeights(static_cast<ExteroceptiveCost::Kind>(f), W[f]);
  optimizer.prepareForEvaluation(true);
  int failures = 0;
  const double u = std::ldexp(1.0, -53);
  const int k = order, kb = 4;
  for (size_t i = 0; i < picked.size(); ++i) {
    const Eval got = eval(picked[i]);
    const Eval& p = plain[i];
    const int kind = picked[i]->kind(), nr = static_cast<int>(p.r.size()), d = static_cast<int>(sides[kind]);
    const double* w = W[kind].data();
    // row i of W x for x with nr rows and n columns (the bearing's one row: d = 1 = nr)
    auto wx = [&](const std::vector<double>& x, int n, int row, int col) { double s = 0; for (int j = 0; j < d; ++j) s += w[d * row + j] * x[static_cast<size_t>(j) * n + col]; return s; };
    std::vector<double> rowmax(nr, 0.0);
    for (auto& Jb : p.J) { const int n = static_cast<int>(Jb.size()) / nr; for (int r = 0; r < nr; ++r) for (int c = 0; c < n; ++c) rowmax[r] = std::max(rowmax[r], std::fabs(Jb[static_cast<size_t>(r) * n + c])); }
    for (int r = 0; r < nr; ++r) rowmax[r] = std::max(rowmax[r], std::fabs(p.r[r]));
    auto bound = [&](int row) { double s = 0; for (int j = 0; j < d; ++j) s += std::fabs(w[d * row + j]) * rowmax[j]; return 64 * u * s; };
    for (int r = 0; r < nr; ++r)
      if (std::fabs(got.r[r] - wx(p.r, 1, r, 0)) > bound(r)) { ++failures; std::fprintf(stderr, "residual: kind %d row %d\n", kind, r); }
    for (size_t b = 0; b < p.J.size(); ++b) {
      const int n = static_cast<int>(p.J[b].size()) / nr;
      const bool bias = kind == ExteroceptiveCost::kInertial && static_cast<int>(b) >= k + 5 && static_cast<int>(b) < k + 5 + 2 * kb;
      for (int r = 0; r < nr; ++r)
        for (int c = 0; c < n; ++c) {
          const double g = got.J[b][static_cast<size_t>(r) * n + c];
          if (bias) {   // wg[m] W[:, 0:3] (gyro knots) / wa[m] W[:, 3:6] (accel knots); stamp column zero
            const bool gyro = static_cast<int>(b) < k + 5 + kb;
            const double wv = gyro ? p.J[b][0] : p.J[b][static_cast<size_t>(3) * n];
            const double want = c < 3 ? wv * w[d * r + (gyro ? 0 : 3) + c] : 0.0;
            if (g != want) { ++failures; std::fprintf(stderr, "bias block %zu row %d col %d: %.17g != %.17g\n", b, r, c, g, want); }
          } else if (std::fabs(g - wx(p.J[b], n, r, c)) > bound(r)) {
            ++failures; std::fprintf(stderr, "jacobian: kind %d block %zu row %d col %d\n", kind, b, r, c);
          }
        }
    }
  }
  const Manifold state_manifold = Manifold::StampedSE3(true, false, false);   // reference pixel.cpp(test):52
  const Manifold landmark_manifold = Manifold::Euclidean(3);
  const Manifold bias_manifold = Manifold::StampedEuclidean(3, true, false);   // reference imu.cpp:64-66
  const Manifold gravity_manifold = Manifold::Sphere(3);

  // ---- (2) Probe through the plugin surface, on the variable blocks of a few weighted costs ----
  int probe_failures = 0, probe_blocks = 0;
  auto probe = [&](ExteroceptiveCost* cost, const std::vector<std::pair<int, const Manifold*>>& blocks) {
    auto params = cost->update();
    const int nr = cost->num_residuals();
    const auto& sizes = cost->parameter_block_sizes();
    std::vector<std::vector<double>> J(params.size());
    std::vector<double*> jp(params.size());
    for (size_t b = 0; b < params.size(); ++b) { J[b].assign(static_cast<size_t>(nr) * sizes[b], 0.0); jp[b] = J[b].data(); }
    std::vector<double> r0(nr), rp(nr), rm(nr);
    optimizer.prepareForEvaluation(true);
    cost->Evaluate(params.data(), r0.data(), jp.data());
    for (auto [b, m] : blocks) {
      const int na = m->AmbientSize(), nt = m->TangentSize();
      std::vector<double> Ja(static_cast<size_t>(nr) * nt), Jn(static_cast<size_t>(nr) * nt), save(params[b], params[b] + na), delta(nt), xp(na);
      m->RightMultiplyByPlusJacobian(params[b], nr, J[b].data(), Ja.data());
      const double h = 1e-6;
      for (int c = 0; c < nt; ++c) {
        for (int s = 0; s < 2; ++s) {
          std::fill(delta.begin(), delta.end(), 0.0); delta[c] = s ? -h : h;
          m->Plus(save.data(), delta.data(), xp.data());
          std::copy(xp.begin(), xp.end(), params[b]);
          optimizer.prepareForEvaluation(false);                      // new evaluation point -> one device batch
          cost->Evaluate(params.data(), s ? rm.data() : rp.data(), nullptr);
        }
        std::copy(save.begin(), save.end(), params[b]);
        for (int r = 0; r < nr; ++r) Jn[r * nt + c] = (rp[r] - rm[r]) / (2 * h);
      }
      double na2 = 0, nn2 = 0, worst_rel = 0, worst_abs = 0;
      for (size_t i = 0; i < Ja.size(); ++i) { na2 += Ja[i] * Ja[i]; nn2 += Jn[i] * Jn[i]; }
      for (size_t i = 0; i < Ja.size(); ++i) {
        const double ae = std::fabs(Ja[i] - Jn[i]);
        double re = ae / std::max(std::fabs(Ja[i]), std::fabs(Jn[i]));
        if (Ja[i] == 0.0 || Jn[i] == 0.0) re = ae;
        worst_rel = std::max(worst_rel, re);
        worst_abs = std::max(worst_abs, std::fabs(Ja[i] / std::sqrt(na2) - Jn[i] / std::sqrt(nn2)));
      }
      ++probe_blocks;
      if (worst_rel > 1e-5 && worst_abs > 1e-5) { ++probe_failures; std::fprintf(stderr, "probe: cost kind %d index %d block %d rel %.3e abs %.3e\n", cost->kind(), cost->index(), b, worst_rel, worst_abs); }
    }
  };
  if (Nv) { std::vector<std::pair<int, const Manifold*>> blk; for (int m = 1; m + 1 < k; ++m) blk.push_back({m, &state_manifold}); blk.push_back({k + 3, &landmark_manifold}); probe(vcosts[Nv / 2], blk); }
  if (Ni) { std::vector<std::pair<int, const Manifold*>> blk; for (int m = 1; m + 1 < k; ++m) blk.push_back({m, &state_manifold}); blk.push_back({k + 5 + 1, &bias_manifold}); blk.push_back({k + 5 + 4 + 2, &bias_manifold}); blk.push_back({k + 13, &gravity_manifold}); probe(icosts[Ni / 3], blk); }
  if (Nb) { std::vector<std::pair<int, const Manifold*>> blk; for (int m = 1; m + 1 < k; ++m) blk.push_back({m, &state_manifold}); blk.push_back({k + 3, &landmark_manifold}); probe(bcosts[Nb - 1], blk); }
  if (Nm) { std::vector<std::pair<int, const Manifold*>> blk; for (int m = 1; m + 1 < k; ++m) blk.push_back({m, &state_manifold}); probe(mcosts[0], blk); }

  for (int f = 0; f < 4; ++f) optimizer.setWeights(static_cast<ExteroceptiveCost::Kind>(f), {});
  optimizer.prepareForEvaluation(true);
  int cleared_mismatch = 0;
  for (size_t i = 0; i < picked.size(); ++i) {
    const Eval e = eval(picked[i]);
    if (e.r != plain[i].r || e.J != plain[i].J) ++cleared_mismatch;
  }
  std::printf("weights_test: costs %zu failures %d probe blocks %d failures %d cleared mismatches %d\n", picked.size(), failures, probe_blocks, probe_failures,
              cleared_mismatch);
  return (failures || probe_failures || cleared_mismatch || probe_blocks == 0) ? 1 : 0;
}
