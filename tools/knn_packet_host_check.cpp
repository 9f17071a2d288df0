// tools/knn_packet_host_check.cpp -- compiles the engine's own csrc/knn.cuh + tree_build.h with g++ against the host CUDA model
// (tools/hostemu: warp votes, reductions and shuffles) and runs the seeded rounds' PACKET search (nn_search_packet: per-lane prologue,
// then nn_packet_walk) one warp at a time against a brute force in the reference's operation order: exact index (lowest on ties) and
// bit-exact d^2, with and without the per-leaf neighbour lists, and the certificate of the same search (Q = NNQueryT): its margin
// never exceeds the true gap to the runner-up.  The 32 queries of a warp lie around one spot of the surface, as neighbours in the src
// tree order do, and mix seed kinds (none, the right leaf, a stale leaf) and query kinds (near, far, on a point), so that settled and
// walking lanes share a warp; the last warp is partial.
// Usage: knn_packet_host_check <n_points> <n_warps> <seed> <mode>   mode 0: fp32-exact coordinates, 1: arbitrary doubles.
// HOSTEMU_ORDER=random runs the lanes in a fresh random order between any two warp operations.  Exit code 0 = all exact.
#include <cstdio>
#include <cstdlib>
#include <random>
#include <string>
#include <vector>
#include "../mv_lm_icp_b200/csrc/knn.cuh"
#include "../mv_lm_icp_b200/csrc/tree_build.h"

template <bool F32> static int run(int n, int n_warps, unsigned seed) {
  std::mt19937_64 rng(seed);
  std::uniform_real_distribution<double> U(-1.0, 1.0); std::normal_distribution<double> G(0.0, 1.0);
  // a wavy surface patch with a few exact duplicates (distance ties), as tools/knn_host_check.cpp
  std::vector<double> pts(3 * (size_t)n);
  for (int i = 0; i < n; ++i) {
    double x = 0.1 * U(rng), y = 0.1 * U(rng), z = 0.45 + 0.02 * std::sin(40 * x) * std::cos(25 * y) + 1e-4 * G(rng);
    if (!F32) { x += 1e-9 * G(rng); y += 1e-9 * G(rng); }
    else { x = (float)x; y = (float)y; z = (float)z; }
    pts[3 * i] = x; pts[3 * i + 1] = y; pts[3 * i + 2] = z;
  }
  for (int d = 0; d < n / 50; ++d) { const int a = rng() % n, b = rng() % n; for (int k = 0; k < 3; ++k) pts[3 * a + k] = pts[3 * b + k]; }
  HostFrameBuild hb; build_frame(pts.data(), n, hb);
  const int64_t npad = ((n + LEAF - 1) / LEAF) * LEAF;
  std::vector<float4> sf(npad); std::vector<double4a> sd(npad);
  for (int64_t i = 0; i < npad; ++i) {
    const int32_t w = i < n ? hb.order[i] : INT32_MAX; const int64_t j = i < n ? hb.order[i] : 0;
    float4 r; double4a q;
    if (i < n) { r.x = (float)pts[3 * j]; r.y = (float)pts[3 * j + 1]; r.z = (float)pts[3 * j + 2]; q.x = pts[3 * j]; q.y = pts[3 * j + 1]; q.z = pts[3 * j + 2]; }
    else { r.x = r.y = r.z = INFINITY; q.x = q.y = q.z = INFINITY; }
    std::memcpy(&r.w, &w, 4); const long long wl = w; std::memcpy(&q.w, &wl, 8);
    sf[i] = r; sd[i] = q;
  }
  FrameDev fd{};
  fd.pts_s = F32 ? (const void*)sf.data() : (const void*)sd.data(); fd.pts_sf = sf.data(); fd.boxes = hb.boxes.data(); fd.faces = hb.faces.data();
  fd.pos_of = hb.pos_of.data(); fd.n = n; fd.n_leaf_pad = hb.n_leaf_pad; fd.depth = hb.depth; fd.absmax = hb.absmax;

  // queries, 32 per warp around one base point; the last warp holds 32 - 7 of them
  const int nq = 32 * n_warps - 7;
  std::vector<double> q(3 * (size_t)nq), want_d(nq), want_gap(nq);
  std::vector<int> want_i(nq), start(nq), kind(nq);
  for (int w = 0; w < n_warps; ++w) {
    const int base = rng() % n;
    const double spread = w % 3 == 0 ? 2e-3 : (w % 3 == 1 ? 1e-2 : 3e-2);
    for (int l = 0; l < 32 && 32 * w + l < nq; ++l) {
      const int qi = 32 * w + l;
      kind[qi] = (l + w) % 4;
      const double s = kind[qi] == 0 ? 1e-4 : (kind[qi] == 1 ? 2e-2 : (kind[qi] == 2 ? 0.0 : 5e-3));
      for (int k = 0; k < 3; ++k) q[3 * qi + k] = pts[3 * base + k] + spread * G(rng) * (k < 2) + s * G(rng);
      double best = INFINITY, second = INFINITY; int bi = INT32_MAX;   // frame.h:70-76 operation order, lowest index on ties
      for (int i = 0; i < n; ++i) {
        const double d0 = q[3 * qi] - pts[3 * i], d1 = q[3 * qi + 1] - pts[3 * i + 1], d2 = q[3 * qi + 2] - pts[3 * i + 2];
        const double d = (d0 * d0 + d1 * d1) + d2 * d2;
        if (d < best) { second = best; best = d; bi = i; } else if (d < second) second = d;
      }
      want_i[qi] = bi; want_d[qi] = best; want_gap[qi] = std::sqrt(second) - std::sqrt(best);
      const int sk = (l * 7 + w) % 3;   // seeds: none, the right leaf, a random (stale) leaf
      start[qi] = sk == 0 ? -1 : (sk == 1 ? hb.pos_of[bi] / LEAF : (int)(rng() % ((n + LEAF - 1) / LEAF)));
    }
  }
  int bad = 0; long n_cert = 0, n_pos = 0;
  for (int sched = 0; sched < 2; ++sched) {
    FrameDev fdx = fd; fdx.adj = sched == 0 ? hb.adj.data() : nullptr;   // with / without the neighbour lists
    std::vector<int> got_i(nq), got_ti(nq); std::vector<double> got_d(nq), got_td(nq); std::vector<float> margin(nq);
    hostemu::launch(dim3(n_warps), dim3(32), 0, [&]() {
      const int qi = 32 * (int)blockIdx.x + (int)threadIdx.x;
      const bool has = qi < nq;
      const double* p = has ? &q[3 * qi] : nullptr;
      NNQuery s; nn_query_init(s, has ? p[0] : 0.0, has ? p[1] : 0.0, has ? p[2] : 0.0, fdx.absmax);
      nn_search_packet<F32, NNQuery>(fdx, s, has, has ? start[qi] : -1);
      NNQueryT st; nn_query_init(st, has ? p[0] : 0.0, has ? p[1] : 0.0, has ? p[2] : 0.0, fdx.absmax); nn_track_init(st);
      nn_search_packet<F32, NNQueryT>(fdx, st, has, has ? start[qi] : -1);
      if (has) { got_i[qi] = s.bi; got_d[qi] = s.best; got_ti[qi] = st.bi; got_td[qi] = st.best; margin[qi] = nn_margin(st); }
    });
    for (int qi = 0; qi < nq; ++qi) {
      if (got_i[qi] != want_i[qi] || got_d[qi] != want_d[qi] || got_ti[qi] != want_i[qi] || got_td[qi] != want_d[qi] || (double)margin[qi] > want_gap[qi]) {
        if (++bad < 10) std::printf("MISMATCH q %d kind %d sched %d: got (%d, %.17g) tracked (%d, %.17g, margin %.9g) want (%d, %.17g, gap %.9g)\n", qi, kind[qi],
                                    sched, got_i[qi], got_d[qi], got_ti[qi], got_td[qi], margin[qi], want_i[qi], want_d[qi], want_gap[qi]);
      }
      if (kind[qi] == 0) { ++n_cert; if (margin[qi] > 0.f) ++n_pos; }
    }
  }
  std::printf("n %d warps %d storage %s: %d mismatches; certificates of near-surface queries: %ld, margin > 0: %ld\n",
              n, n_warps, F32 ? "fp32" : "fp64", bad, n_cert, n_pos);
  return bad;
}

int main(int argc, char** argv) {
  const int n = argc > 1 ? atoi(argv[1]) : 5000, n_warps = argc > 2 ? atoi(argv[2]) : 40;
  const unsigned seed = argc > 3 ? (unsigned)atoi(argv[3]) : 1u; const int mode = argc > 4 ? atoi(argv[4]) : 0;
  return (mode == 0 ? run<true>(n, n_warps, seed) : run<false>(n, n_warps, seed)) ? 1 : 0;
}
