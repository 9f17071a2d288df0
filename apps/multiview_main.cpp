// apps/multiview_main.cpp -- headless drop-in for the reference's `multiview` executable (src/main_multiview.cpp:130-173)
// on top of compat/mvicp_compat.hpp: same flags (gflags syntax --name=value, defaults of main_multiview.cpp:30-51), same
// loop (20 rounds of closest points + global optimisation), same timing lines (CPUTimer.cpp:17-27).  --g2o runs the g2o
// backend (ICP_G2O::g2oOptimizer, main_multiview.cpp:158-164) and prints its `round: … chi2: … impr: …` lines
// (icp-g2o.cpp:264-300).  Not reproduced: the viewer, and the random pose noise of loadFrames (common.h:38-67 uses a
// default-seeded std::mt19937 with an unspecified argument evaluation order): initial poses come from pose files, noise
// from --sigma uses a fixed LCG.
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <iomanip>
#include <iostream>
#include <map>
#include <string>
#include "../compat/mvicp_compat.hpp"
#include "io.hpp"

struct Flags {
  std::map<std::string, std::string> kv;
  Flags(int argc, char** argv) {
    for (int i = 1; i < argc; ++i) {
      std::string a(argv[i]);
      if (a.compare(0, 2, "--") != 0) continue;
      a = a.substr(2);
      const size_t eq = a.find('=');
      if (eq == std::string::npos) { if (a.compare(0, 2, "no") == 0) kv[a.substr(2)] = "false"; else kv[a] = "true"; }
      else kv[a.substr(0, eq)] = a.substr(eq + 1);
    }
  }
  std::string s(const char* k, const char* d) const { auto it = kv.find(k); return it == kv.end() ? d : it->second; }
  double f(const char* k, double d) const { auto it = kv.find(k); return it == kv.end() ? d : atof(it->second.c_str()); }
  int i(const char* k, int d) const { auto it = kv.find(k); return it == kv.end() ? d : atoi(it->second.c_str()); }
  bool b(const char* k, bool d) const { auto it = kv.find(k); return it == kv.end() ? d : (it->second == "true" || it->second == "1"); }
};

struct CPUTimer {   // CPUTimer.cpp:12-27
  std::chrono::steady_clock::time_point t0;
  void tic() { t0 = std::chrono::steady_clock::now(); }
  double toc(const std::string& name) {
    const double s = std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - t0).count() * 1e-6;
    std::cout << std::endl << "=====  TIMING[" << name << "] is " << s << " s" << std::endl << std::endl;
    return s;
  }
};

static void add_noise(Eigen::Isometry3d& P, double sigma, double sigmat, unsigned long long& state) {   // cf. common.h:38-67
  auto gauss = [&]() { double s = 0; for (int i = 0; i < 12; ++i) { state = state * 6364136223846793005ULL + 1442695040888963407ULL; s += (double)(state >> 11) / 9007199254740992.0; } return s - 6.0; };
  const double w[3] = {gauss() * sigma, gauss() * sigma, gauss() * sigma};
  const double th = std::sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  if (th > 0) {
    const double k[3] = {w[0] / th, w[1] / th, w[2] / th}, c = std::cos(th), s = std::sin(th), oc = 1 - c;
    const double Q[9] = {c + k[0] * k[0] * oc, k[0] * k[1] * oc - k[2] * s, k[0] * k[2] * oc + k[1] * s,
                         k[1] * k[0] * oc + k[2] * s, c + k[1] * k[1] * oc, k[1] * k[2] * oc - k[0] * s,
                         k[2] * k[0] * oc - k[1] * s, k[2] * k[1] * oc + k[0] * s, c + k[2] * k[2] * oc};
    std::memcpy(R, Q, sizeof R);
  }
  double M[9];
  for (int r = 0; r < 3; ++r) for (int c2 = 0; c2 < 3; ++c2) M[3 * r + c2] = P(r, 0) * R[c2] + P(r, 1) * R[3 + c2] + P(r, 2) * R[6 + c2];   // pose * q(w)
  for (int r = 0; r < 3; ++r) { for (int c2 = 0; c2 < 3; ++c2) P(r, c2) = M[3 * r + c2]; P(r, 3) += gauss() * sigmat; }
}

int main(int argc, char** argv) {
  const Flags F(argc, argv);
  const std::string dir = F.s("dir", "../samples/Bunny_RealData");
  const bool pointToPlane = F.b("pointToPlane", true), sophusSE3 = F.b("sophusSE3", true), angleAxis = F.b("angleAxis", false);
  const bool robust = F.b("robust", true), recomputeNormals = F.b("recomputeNormals", true), eof_quirk = F.b("ref_eof_quirk", false);
  const bool g2o = F.b("g2o", false);   // main_multiview.cpp:35
  const double cutoff = F.f("cutoff", 0.05), sigma = F.f("sigma", 0.02), sigmat = F.f("sigmat", 0.01);
  const int knn = F.i("knn", 2), limit = F.i("limit", 40), step = F.i("step", 2), rounds = F.i("rounds", 20);
  const std::string out = F.s("out", "");

  // loadFrames (main_multiview.cpp:53-100)
  std::vector<std::shared_ptr<Frame>> frames;
  const auto clouds = io::files_with_prefix(dir, "cloud"), poses = io::files_with_prefix(dir, "pose"), gts = io::files_with_prefix(dir, "groundtruth");
  if (clouds.size() != poses.size()) std::cout << "unequal size" << std::endl;
  unsigned long long rng = 0x9E3779B97F4A7C15ULL;
  for (size_t i = 0; i < clouds.size() && i < poses.size() && (int)i < limit * step; i += step) {
    auto f = std::make_shared<Frame>();
    if (!io::load_xyz(clouds[i], f->pts, f->nor, eof_quirk)) return 1;
    if (gts.size() == clouds.size()) { io::load_pose(poses[i], f->pose); io::load_pose(gts[i], f->poseGroundTruth); }
    else {
      io::load_pose(poses[i], f->poseGroundTruth);
      f->pose = f->poseGroundTruth;
      if (i != 0 && (sigma > 0 || sigmat > 0)) add_noise(f->pose, sigma, sigmat, rng);
    }
    frames.push_back(f);
  }
  if (frames.size() < 2) { std::cerr << "need at least two frames in " << dir << std::endl; return 1; }
  std::cout << "loaded " << frames.size() << " frames" << std::endl;

  CPUTimer timer;
  mvicp_compat::Session<Frame> session;
  try {
    if (recomputeNormals) { timer.tic(); mvicp_compat::recomputeNormals(session, frames, 10); timer.toc("recompute normals"); }
    frames[0]->fixed = true;                                      // main_multiview.cpp:141
    // ApproachComponents::computePoseNeighbours (main_multiview.cpp:104-117)
    session.bind(frames); session.push_poses();
    mvicp_compat::check(mvicp_pose_graph_knn(session.ctx, knn));
    int32_t E = 0; mvicp_compat::check(mvicp_get_graph(session.ctx, &E, nullptr, nullptr));
    std::vector<int32_t> es(E), ed(E); mvicp_compat::check(mvicp_get_graph(session.ctx, &E, es.data(), ed.data()));
    for (int e = 0; e < E; ++e) frames[es[e]]->neighbours.push_back(OutgoingEdge{ed[e], 0.f, {}});
    const int param = sophusSE3 ? MVICP_PARAM_SE3 : (angleAxis ? MVICP_PARAM_AA : MVICP_PARAM_QUAT);   // main_multiview.cpp:158-164
    for (int i = 0; i < rounds; ++i) {
      timer.tic();
      mvicp_compat::computeClosestPoints(session, frames, (float)cutoff, /*materialize=*/false);
      timer.toc(std::string("closest pts ") + std::to_string(i));
      timer.tic();
      if (g2o) {   // main_multiview.cpp:158-160
        std::vector<double> chi;
        const mvicp_g2o_summary s = mvicp_compat::g2oOptimizer(session, frames, pointToPlane, &chi);
        // icp-g2o.cpp:264,283-298; FIXED(x) = std::fixed << x << resetiosflags(fixed)
        std::cout << "round: " << "s" << " chi2: " << std::fixed << chi[0] << std::resetiosflags(std::ios_base::fixed) << std::endl;
        for (size_t k = 1; k < chi.size(); ++k) {
          const double impr = (chi[k - 1] - chi[k]) / chi[k - 1];
          std::cout << "round: " << k - 1 << " chi2: " << std::fixed << chi[k] << std::resetiosflags(std::ios_base::fixed) << " impr: " << impr << std::endl;
          if (impr > 0.0) std::cout << "impr > 0%" << std::endl;
        }
        if (s.ended == MVICP_G2O_END_NO_IMPROVEMENT) std::cout << "100 times no impr, break";
        timer.toc(std::string("global ") + std::to_string(i));
        std::cout << "round: " << i << "  g2o calls " << s.calls << " iterations " << s.iterations << " trials " << s.trials
                  << "  chi2 " << s.chi2_initial << " -> " << s.chi2_final << std::endl;
        continue;
      }
      const mvicp_lm_summary s = mvicp_compat::optimize(session, frames, param, pointToPlane, robust);
      timer.toc(std::string("global ") + std::to_string(i));
      std::cout << "round: " << i << "  LM iterations " << s.num_iterations << "  cost " << s.initial_cost << " -> " << s.final_cost << std::endl;
    }
  } catch (const std::exception& e) { std::cerr << e.what() << std::endl; return 2; }
  if (!out.empty())
    for (size_t i = 0; i < frames.size(); ++i) io::save_pose(out + "/pose_out_" + std::to_string(i) + ".txt", frames[i]->pose);
  return 0;
}
