// apps/pairwise_main.cpp -- headless drop-in for the reference's `pairwise` executable (src/main_pairwise.cpp:29-134): a
// cloud is moved by a known transform P and every pairwise solver has to recover P from the 1:1 correspondences; prints
// the CPUTimer lines and the "Accurracy" block (translation / rotation error, common.h:259-282).  Reproduced: the three
// Ceres-backed solvers (angle-axis, Eigen quaternion, Sophus SE3), point-to-point or --pointToPlane, and the closed-form
// comparison row (mvicp_pairwise_closed), and with --g2o the g2o row (ICP_G2O::pointToPoint / pointToPlane,
// main_pairwise.cpp:26,76-80,98-102,123-127).  Not reproduced: addNoise's RNG stream -- the perturbation of P comes from a
// fixed LCG with the same sigmas (0.1 rad, 0.1 m; main_pairwise.cpp:56).
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <iomanip>
#include <iostream>
#include <map>
#include <string>
#include "../compat/mvicp_compat.hpp"
#include "io.hpp"

typedef Eigen::Isometry3d Iso;
static void mat_mul(const Iso& A, const Iso& B, Iso& C) { for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c) { double s = 0; for (int k = 0; k < 4; ++k) s += A(r, k) * B(k, c); C(r, c) = s; } }
static Iso axis_rot(int axis, double a) {
  Iso R; const double c = std::cos(a), s = std::sin(a); const int i = (axis + 1) % 3, j = (axis + 2) % 3;
  R(i, i) = c; R(i, j) = -s; R(j, i) = s; R(j, j) = c; return R;
}
static void quat_of(const Iso& P, double q[4]) {   // w x y z of the rotation block (trace branch as Eigen's Quaterniond(Matrix3d))
  const double t = P(0, 0) + P(1, 1) + P(2, 2);
  if (t > 0) { double s = std::sqrt(t + 1.0); q[0] = 0.5 * s; s = 0.5 / s; q[1] = (P(2, 1) - P(1, 2)) * s; q[2] = (P(0, 2) - P(2, 0)) * s; q[3] = (P(1, 0) - P(0, 1)) * s; }
  else {
    int i = 0; if (P(1, 1) > P(0, 0)) i = 1; if (P(2, 2) > P(i, i)) i = 2; const int j = (i + 1) % 3, k = (j + 1) % 3;
    double s = std::sqrt(P(i, i) - P(j, j) - P(k, k) + 1.0); q[1 + i] = 0.5 * s; s = 0.5 / s;
    q[0] = (P(k, j) - P(j, k)) * s; q[1 + j] = (P(j, i) + P(i, j)) * s; q[1 + k] = (P(k, i) + P(i, k)) * s;
  }
}
static std::string pose_diff(const Iso& A, const Iso& B) {   // common.h:259-282
  const double dt = std::sqrt((A(0, 3) - B(0, 3)) * (A(0, 3) - B(0, 3)) + (A(1, 3) - B(1, 3)) * (A(1, 3) - B(1, 3)) + (A(2, 3) - B(2, 3)) * (A(2, 3) - B(2, 3)));
  double qa[4], qb[4]; quat_of(A, qa); quat_of(B, qb);
  const double d = qa[0] * qb[0] + qa[1] * qb[1] + qa[2] * qb[2] + qa[3] * qb[3];
  double v = 2 * d * d - 1; if (v < -1) v = -1; if (v > 1) v = 1;
  char buf[128]; std::snprintf(buf, sizeof buf, "\t diff_tra:%g\t diff_rot_degrees:%g\n", dt, std::acos(v) * 180.0 / M_PI);
  return buf;
}

int main(int argc, char** argv) {
  bool pointToPlane = false, g2o = false; std::string cloud = "../samples/Bunny_RealData/cloudXYZ_0.xyz", out;
  for (int i = 1; i < argc; ++i) {
    const std::string a(argv[i]);
    if (a == "--pointToPlane" || a == "--pointToPlane=true") pointToPlane = true;
    else if (a == "--nopointToPlane" || a == "--pointToPlane=false") pointToPlane = false;
    else if (a == "--g2o" || a == "--g2o=true") g2o = true;   // main_pairwise.cpp:26
    else if (a == "--nog2o" || a == "--g2o=false") g2o = false;
    else if (a.compare(0, 8, "--cloud=") == 0) cloud = a.substr(8);
    else if (a.compare(0, 6, "--out=") == 0) out = a.substr(6);
  }
  std::vector<Eigen::Vector3d> pts, nor;
  if (!io::load_xyz(cloud, pts, nor, false) || pts.empty()) return 1;
  for (size_t i = 0; i < 10 && i < pts.size(); ++i) std::cout << pts[i][0] << " " << pts[i][1] << " " << pts[i][2] << "\t" << nor[i][0] << " " << nor[i][1] << " " << nor[i][2] << std::endl;

  // P = Translation(.01,-.01,-.005) * Rx(pi/4) Ry(1) Rz(-0.2), perturbed (main_pairwise.cpp:44-56)
  Iso P, T1, T2; mat_mul(axis_rot(0, M_PI_4), axis_rot(1, 1.0), T1); mat_mul(T1, axis_rot(2, -0.2), T2);
  T2(0, 3) = .01; T2(1, 3) = -.01; T2(2, 3) = -.005;
  unsigned long long st = 0x853C49E6748FEA9BULL;
  auto gauss = [&]() { double s = 0; for (int i = 0; i < 12; ++i) { st = st * 6364136223846793005ULL + 1442695040888963407ULL; s += (double)(st >> 11) / 9007199254740992.0; } return s - 6.0; };
  Iso N; { const double w[3] = {gauss() * 0.1, gauss() * 0.1, gauss() * 0.1}; Iso a, b; mat_mul(axis_rot(0, w[0]), axis_rot(1, w[1]), a); mat_mul(a, axis_rot(2, w[2]), b); N = b; }
  mat_mul(T2, N, P); for (int r = 0; r < 3; ++r) P(r, 3) += gauss() * 0.1;

  std::vector<Eigen::Vector3d> dst(pts.size()), dnor(pts.size());
  for (size_t i = 0; i < pts.size(); ++i)
    for (int r = 0; r < 3; ++r) {
      dst[i][r] = P(r, 0) * pts[i][0] + P(r, 1) * pts[i][1] + P(r, 2) * pts[i][2] + P(r, 3);
      dnor[i][r] = P(r, 0) * nor[i][0] + P(r, 1) * nor[i][1] + P(r, 2) * nor[i][2];
    }

  std::map<std::string, float> timings;
  Iso closed; bool have_closed = true;
  try {
    const auto t0 = std::chrono::steady_clock::now();
    mvicp_compat::closedForm(pointToPlane, pts, dst, pointToPlane ? &dnor : nullptr, closed.data());   // main_pairwise.cpp:73,95
    const double s = std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - t0).count() * 1e-6;
    std::cout << std::endl << "=====  TIMING[closed] is " << s << " s" << std::endl << std::endl;
    timings["closed"] = (float)s;
  } catch (const std::exception& e) { std::cerr << "closed form: " << e.what() << std::endl; have_closed = false; }   // the comparison row is optional
  const char* names[3] = {"ceres CeresAngleAxis", "ceres EigenQuaternion", "ceres SophusSE3"};
  const int params[3] = {MVICP_PARAM_AA, MVICP_PARAM_QUAT, MVICP_PARAM_SE3};
  Iso est[3], est_g2o;
  try {
    if (g2o) {   // main_pairwise.cpp:76-80,98-102
      const auto t0 = std::chrono::steady_clock::now();
      mvicp_compat::pairwiseG2O(pointToPlane, pts, dst, pointToPlane ? &dnor : nullptr, est_g2o.data());
      const double s = std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - t0).count() * 1e-6;
      std::cout << std::endl << "=====  TIMING[g2o] is " << s << " s" << std::endl << std::endl;
      timings["g2o"] = (float)s;
    }
    for (int k = 0; k < 3; ++k) {
      const auto t0 = std::chrono::steady_clock::now();
      mvicp_compat::pairwise(params[k], pointToPlane, pts, dst, pointToPlane ? &dnor : nullptr, est[k].data());
      const double s = std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - t0).count() * 1e-6;
      std::cout << std::endl << "=====  TIMING[" << names[k] << "] is " << s << " s" << std::endl << std::endl;   // CPUTimer.cpp:17-27
      timings[names[k]] = (float)s;
    }
  } catch (const std::exception& e) { std::cerr << e.what() << std::endl; return 2; }
  std::cout << "=====  TIMINGS ====" << std::endl;                                                               // CPUTimer.cpp:28-36
  for (auto& kv : timings) { std::cout << std::left << std::setw(20) << kv.first << ":\t"; std::printf("%0.3f\n", kv.second); std::fflush(stdout); }
  std::cout << std::endl << "=====  Accurracy ====" << std::endl;
  if (have_closed) std::cout << "closed form      " << pose_diff(P, closed) << std::endl;
  if (g2o) std::cout << "g2o              " << pose_diff(P, est_g2o) << std::endl;   // main_pairwise.cpp:123-127
  std::cout << "ceres CeresAngleAxis" << pose_diff(P, est[0]) << std::endl;
  std::cout << "ceres EigenQuaternion" << pose_diff(P, est[1]) << std::endl;
  std::cout << "ceres SophusSE3    " << pose_diff(P, est[2]) << std::endl;
  if (!out.empty()) { io::save_pose(out + "/P_true.txt", P); if (have_closed) io::save_pose(out + "/P_closed.txt", closed); for (int k = 0; k < 3; ++k) io::save_pose(out + "/P_est_" + std::to_string(k) + ".txt", est[k]);
                     if (g2o) io::save_pose(out + "/P_g2o.txt", est_g2o); }
  return 0;
}
