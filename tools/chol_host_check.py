"""Run the TEXT of csrc/lm_step.cuh:chol_solve on the host: 512 std::threads, __syncthreads()/__syncwarp() as std::barrier,
on a ring-graph normal matrix whose entries outside the row profiles are NaN (so any read outside the envelope poisons the
result).  With --tsan the harness is built with ThreadSanitizer: a missing barrier shows up as a data race.
usage: python tools/chol_host_check.py [--tsan]      (development aid; g++ >= 11)"""
import os, subprocess, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
src = open(os.path.join(ROOT, "mv_lm_icp_b200", "csrc", "lm_step.cuh")).read()
fn = src[src.index("__device__ __forceinline__ void chol_factor_diag("):src.index("// ---- the LM trust-region state machine")]
harness = r'''
#include <barrier>
#include <thread>
#include <vector>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
using std::min; using std::isfinite;
#define __device__
#define __forceinline__ inline
static double rsqrt(double x) { return 1.0 / std::sqrt(x); }
static long long clock64() { return 0; }
#define __restrict__
struct Dim { int x; };
static Dim blockDim{512};
static thread_local Dim threadIdx{0};
static std::barrier<>* g_bar; static std::vector<std::barrier<>*> g_wbar;
static void __syncthreads() { g_bar->arrive_and_wait(); }
static void __syncwarp() { g_wbar[threadIdx.x >> 5]->arrive_and_wait(); }
''' + fn + r'''
int main() {
  const int M = 20, n = 6 * (M - 1), ld = n | 1;   // ring of 20 frames, frame 0 fixed
  std::vector<double> H((size_t)n * n, 0.0), g(n);
  std::vector<int> rfirst(n), rlast(n);
  for (int r = 0; r < n; ++r) rfirst[r] = (r / 6) * 6;
  srand(1);
  auto rnd = []() { return rand() / (double)RAND_MAX - 0.5; };
  for (int s = 0; s < M; ++s) for (int k = 1; k <= 2; ++k) {
    const int d = (s + k) % M; std::vector<int> idx;
    for (int f : {s, d}) if (f > 0) for (int i = 0; i < 6; ++i) idx.push_back(6 * (f - 1) + i);
    for (int rep = 0; rep < 20; ++rep) { std::vector<double> J(idx.size()); for (auto& v : J) v = rnd();
      for (size_t a = 0; a < idx.size(); ++a) for (size_t b = 0; b < idx.size(); ++b) H[(size_t)idx[a] * n + idx[b]] += J[a] * J[b]; }
    if (s > 0 && d > 0) { const int br = 6 * (std::max(s, d) - 1), bc = 6 * (std::min(s, d) - 1); for (int i = 0; i < 6; ++i) rfirst[br + i] = std::min(rfirst[br + i], bc); }
  }
  for (int i = 0; i < n; ++i) { H[(size_t)i * n + i] += 1e-3; g[i] = rnd(); }
  for (int j = 0; j < n; ++j) rlast[j] = j;
  for (int r = 0; r < n; ++r) for (int j = rfirst[r]; j <= r; ++j) rlast[j] = std::max(rlast[j], r);
  for (int j = 1; j < n; ++j) rlast[j] = std::max(rlast[j], rlast[j - 1]);
  std::vector<double> L((size_t)(n + 1) * ld, NAN), scratch(2 * (n + 1)), dinv(n + 1), y(n);
  std::vector<int> rowbase(n + 1); for (int r = 0; r <= n; ++r) rowbase[r] = r * ld;   // dense rows here; the engine packs the profiles
  for (int i = 0; i < n; ++i) for (int j = rfirst[i]; j <= i; ++j) L[(size_t)i * ld + j] = H[(size_t)i * n + j];
  for (int j = 0; j < n; ++j) L[(size_t)n * ld + j] = g[j];
  std::barrier<> bar(512); g_bar = &bar; for (int w = 0; w < 16; ++w) g_wbar.push_back(new std::barrier<>(32));
  std::vector<std::thread> th; std::vector<int> oks(512);
  for (int t = 0; t < 512; ++t) th.emplace_back([&, t]() { threadIdx.x = t; oks[t] = chol_solve(L.data(), rowbase.data(), n, scratch.data(), dinv.data(), y.data(), rlast.data(), rfirst.data()); });
  for (auto& t : th) t.join();
  double maxr = 0, maxg = 0;
  for (int i = 0; i < n; ++i) { double s = 0; for (int j = 0; j < n; ++j) s += H[(size_t)i * n + j] * y[j]; maxr = std::max(maxr, std::fabs(s - g[i])); maxg = std::max(maxg, std::fabs(g[i])); }
  printf("ok %d  max residual %.3e (|g| max %.3e)\n", oks[0], maxr, maxg);
  return (oks[0] && maxr < 1e-12) ? 0 : 1;
}
'''
with tempfile.TemporaryDirectory() as d:
    open(os.path.join(d, "h.cpp"), "w").write(harness)
    flags = ["-O1", "-g", "-std=c++20", "-pthread"] + (["-fsanitize=thread"] if "--tsan" in sys.argv else [])
    subprocess.run(["/usr/bin/g++", *flags, "-o", os.path.join(d, "h"), os.path.join(d, "h.cpp")], check=True)
    r = subprocess.run([os.path.join(d, "h")], capture_output=True, text=True)
    print(r.stdout, r.stderr[-2000:])
    sys.exit(1 if (r.returncode or "ThreadSanitizer" in r.stderr) else 0)
