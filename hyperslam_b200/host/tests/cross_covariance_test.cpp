// GPU test of hyper::Covariance with Options::full_pattern: reads the window dump of covariance_test (written by
// tests/test_gpu_host_cross_covariance.py), checks that the default options refuse pairs outside the selected inverse's
// pattern and that full_pattern accepts them, and writes the ambient and tangent-space blocks of a set of pairs inside
// and outside the pattern for the Python side to compare with hb200_get_covariance_blocks.
#include <cstdio>
#include <fstream>
#include <memory>
#include <string>

#include "hyper/covariance.hpp"
#include "hyper/optimizer.hpp"

using namespace hyper;

int main(int argc, char** argv) {
  if (argc < 3) { std::fprintf(stderr, "usage: cross_covariance_test <window.txt> <out.txt>\n"); return 2; }
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
  { std::vector<double> v(37); for (auto& x : v) in >> x; auto p = imu.variables(); const int s[5] = {7, 6, 6, 9, 9}; int o = 0; for (int b = 0; b < 5; ++b) { std::copy(v.begin() + o, v.begin() + o + s[b], p[b]); o += s[b]; } }
  std::vector<Landmark> lms(L);
  for (int l = 0; l < L; ++l) for (int i = 0; i < 3; ++i) in >> lms[l].variable[i];
  std::vector<VisualPixelObservation> vobs(Nv);
  for (int f = 0; f < Nv; ++f) { int c, l; in >> vobs[f].stamp >> c >> l >> vobs[f].measurement[0] >> vobs[f].measurement[1]; vobs[f].camera = cams[c].get(); vobs[f].landmark = &lms[l]; }
  std::vector<InertialObservation> iobs(Ni);
  for (int f = 0; f < Ni; ++f) { in >> iobs[f].stamp; for (int i = 0; i < 6; ++i) in >> iobs[f].measurement[i]; iobs[f].imu = &imu; iobs[f].gravity = &gravity; }
  std::vector<VisualBearingObservation> bobs(Nb);
  for (int f = 0; f < Nb; ++f) { int c, l; in >> bobs[f].stamp >> c >> l; for (int i = 0; i < 3; ++i) in >> bobs[f].measurement[i]; bobs[f].camera = cams[c].get(); bobs[f].landmark = &lms[l]; }
  std::vector<Sensor> pose_sensors(P);
  for (int p = 0; p < P; ++p) for (int i = 0; i < 7; ++i) in >> pose_sensors[p].transformation().v[i];
  std::vector<ManifoldObservation> mobs(Nm);
  for (int f = 0; f < Nm; ++f) { int sidx; in >> mobs[f].stamp >> sidx; for (int i = 0; i < 7; ++i) in >> mobs[f].measurement.v[i]; mobs[f].sensor = &pose_sensors[sidx]; }
  std::vector<bool> constant(K, false);
  for (int j = 0; j < K; ++j) { int f; in >> f; constant[j] = f != 0; }
  if (!in) { std::fprintf(stderr, "window file is truncated\n"); return 2; }
  (void)nconst;

  Optimizer optimizer(0);
  optimizer.setState(&state);
  std::vector<Camera*> cam_ptrs; for (auto& c : cams) cam_ptrs.push_back(c.get());
  optimizer.setCameras(cam_ptrs);
  optimizer.setIMU(&imu);
  optimizer.setGravity(&gravity);
  for (auto& l : lms) optimizer.addLandmark(l);
  for (auto& o : vobs) optimizer.add(o);
  for (auto& o : iobs) optimizer.add(o);
  for (auto& o : bobs) optimizer.add(o);
  for (auto& o : mobs) optimizer.add(o);
  optimizer.setStateConstant(constant);
  optimizer.prepareForEvaluation(true);   // uploads and binds the window
  int beta = 0;
  hb200_get_bandwidth(optimizer.context(), &beta);

  auto S = [&](int j) { return static_cast<const double*>(state.elements()[j].data()); };
  auto M = [&](int l) { return static_cast<const double*>(lms[l].variable.data()); };
  const double* G = gravity.data();
  const double* BG = imu.gyroscopeBias()[1].data();
  const double* BA = imu.accelerometerBias()[2].data();
  std::ofstream out(argv[2]);
  out.precision(17);
  // the pairs covariance_test shows refused by the default options: state elements beta + 1 apart, a landmark with a
  // state element, two landmarks
  const std::vector<std::vector<std::pair<const double*, const double*>>> outside = {{{S(4), S(4 + beta + 1)}}, {{M(0), S(5)}}, {{M(0), M(1)}}};
  Covariance plain(optimizer);
  int refused = 0;
  for (const auto& pairs : outside) refused += plain.Compute(pairs) ? 0 : 1;
  Covariance::Options options;
  options.full_pattern = true;
  Covariance full(optimizer, options);
  int accepted = 0;
  for (const auto& pairs : outside) accepted += full.Compute(pairs) ? 1 : 0;
  out << "refused " << outside.size() << " " << refused << " accepted " << accepted << " beta " << beta << "\n";
  // pairs outside the pattern (either order), and inside it
  const std::vector<std::pair<const double*, const double*>> pairs = {
      {S(4), S(4 + beta + 1)}, {S(K - 2), S(2)}, {M(0), S(5)}, {S(9), M(3)}, {M(0), M(1)}, {M(4), M(2)}, {BG, M(2)}, {M(3), BA}, {G, M(1)},
      {S(6), S(7)}, {S(8), BG}, {M(2), M(2)}};
  const bool ok = full.Compute(pairs);
  const auto& info = full.info();
  out << "compute " << ok << " " << info.status << " " << info.K << " " << info.beta << " " << info.m << " " << info.L << "\n";
  auto name = [&](const double* p) -> std::string {
    for (int j = 0; j < K; ++j) if (p == S(j)) return "state " + std::to_string(j);
    for (int j = 0; j < Kb; ++j) if (p == imu.gyroscopeBias()[j].data()) return "gyro " + std::to_string(j);
    for (int j = 0; j < Kb; ++j) if (p == imu.accelerometerBias()[j].data()) return "accel " + std::to_string(j);
    if (p == G) return "gravity 0";
    for (int l = 0; l < L; ++l) if (p == M(l)) return "landmark " + std::to_string(l);
    return "unknown -1";
  };
  auto sizes = [&](const std::string& n, int* amb, int* tan) {
    if (n.rfind("state", 0) == 0) { *amb = 8; *tan = 6; }
    else if (n.rfind("gravity", 0) == 0) { *amb = 3; *tan = 2; }
    else if (n.rfind("landmark", 0) == 0) { *amb = 3; *tan = 3; }
    else { *amb = 4; *tan = 3; }
  };
  int failures = 0;
  for (const auto& [a, b] : pairs) {
    int aa, ta, ab, tb;
    sizes(name(a), &aa, &ta);
    sizes(name(b), &ab, &tb);
    std::vector<double> amb(static_cast<size_t>(aa) * ab), tan(static_cast<size_t>(ta) * tb), back(static_cast<size_t>(tb) * ta);
    failures += full.GetCovarianceBlock(a, b, amb.data()) ? 0 : 1;
    failures += full.GetCovarianceBlockInTangentSpace(a, b, tan.data()) ? 0 : 1;
    // the reversed pair is the exact transpose
    failures += full.GetCovarianceBlockInTangentSpace(b, a, back.data()) ? 0 : 1;
    for (int i = 0; i < ta; ++i)
      for (int j = 0; j < tb; ++j) failures += back[static_cast<size_t>(j) * ta + i] == tan[static_cast<size_t>(i) * tb + j] ? 0 : 1;
    out << "pair " << name(a) << " " << name(b) << "\n";
    for (double x : tan) out << x << " ";
    out << "\n";
    for (double x : amb) out << x << " ";
    out << "\n";
  }
  std::vector<double> dummy(64);
  failures += full.GetCovarianceBlock(S(6), S(9), dummy.data()) ? 1 : 0;   // not requested: not served
  out << "failures " << failures << "\n";
  std::printf("cross_covariance_test: beta %d, refused %d / accepted %d of %zu, compute %d, failures %d\n", beta, refused, accepted, outside.size(), ok ? 1 : 0,
              failures);
  const int n = static_cast<int>(outside.size());
  return (ok && failures == 0 && refused == n && accepted == n) ? 0 : 1;
}
