// tree_build.h -- host-side, one-time construction of the per-frame search tree (replaces the lazily built nanoflann
// index, src/internal/frame.cpp:188-193).  Included by mvicp.cu and by tools/sim_search.cpp (CPU step-count model).
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <numeric>
#include <vector>
#include "adjacency.h"
#include "types.cuh"

using namespace mv;

static inline float f_down(double v) { float f = (float)v; if ((double)f > v) f = std::nextafterf(f, -INFINITY); return f; }
static inline float f_up(double v) { float f = (float)v; if ((double)f < v) f = std::nextafterf(f, INFINITY); return f; }

struct HostFrameBuild {
  std::vector<int32_t> order;      // tree order -> original index
  std::vector<int32_t> pos_of;     // original index -> tree position
  std::vector<Box> boxes;
  std::vector<float> faces;        // split-plane bound per node (axis in the low 2 mantissa bits)
  std::vector<int32_t> adj;        // per leaf slot ADJ_SLOTS ints: reach, count, neighbouring leaves (adjacency.h)
  int n_leaf_pad = 1, depth = 0;
  float absmax = 0.f;
};

// Left-balanced KD ordering: the node that covers leaf slots [a, b) of the implicit tree holds the points at sorted
// positions [LEAF a, min(LEAF b, n)); each internal node splits its points at the capacity of its left half along
// the widest axis of their bounding box (nth_element), so sibling boxes never overlap and leaves are compact.
static void kd_order(const double* pts, int32_t* idx, int64_t begin, int64_t count, int64_t leaf_slots, int node, uint8_t* axis_of) {
  if (leaf_slots <= 1) return;
  axis_of[node] = 0;
  if (count <= LEAF) { kd_order(pts, idx, begin, count, leaf_slots / 2, 2 * node, axis_of); return; }
  const int64_t cap_left = (leaf_slots / 2) * LEAF;
  if (count > cap_left) {
    double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int64_t i = begin; i < begin + count; ++i)
      for (int a = 0; a < 3; ++a) { const double v = pts[3 * (int64_t)idx[i] + a]; lo[a] = std::min(lo[a], v); hi[a] = std::max(hi[a], v); }
    int ax = 0; for (int a = 1; a < 3; ++a) if (hi[a] - lo[a] > hi[ax] - lo[ax]) ax = a;
    axis_of[node] = (uint8_t)ax;
    std::nth_element(idx + begin, idx + begin + cap_left, idx + begin + count, [&](int32_t x, int32_t y) {
      const double vx = pts[3 * (int64_t)x + ax], vy = pts[3 * (int64_t)y + ax];
      return vx < vy || (vx == vy && x < y);
    });
    kd_order(pts, idx, begin, cap_left, leaf_slots / 2, 2 * node, axis_of);
    kd_order(pts, idx, begin + cap_left, count - cap_left, leaf_slots / 2, 2 * node + 1, axis_of);
  } else {
    kd_order(pts, idx, begin, count, leaf_slots / 2, 2 * node, axis_of);
  }
}

static void build_frame(const double* pts, int64_t n, HostFrameBuild& out) {
  double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int64_t i = 0; i < n; ++i)
    for (int a = 0; a < 3; ++a) { lo[a] = std::min(lo[a], pts[3 * i + a]); hi[a] = std::max(hi[a], pts[3 * i + a]); }
  const int64_t n_leaf = std::max<int64_t>(1, (n + LEAF - 1) / LEAF);
  int L = 1; while (L < n_leaf) L <<= 1;
  out.order.resize(n); out.pos_of.resize(n);
  std::iota(out.order.begin(), out.order.end(), 0);
  std::vector<uint8_t> axis_of((size_t)2 * L, 0);
  kd_order(pts, out.order.data(), 0, n, L, 1, axis_of.data());
  for (int64_t i = 0; i < n; ++i) out.pos_of[out.order[i]] = (int32_t)i;
  double am = 0; for (int a = 0; a < 3; ++a) am = std::max(am, std::max(std::fabs(lo[a]), std::fabs(hi[a])));
  out.absmax = f_up(am);
  out.n_leaf_pad = L;
  out.depth = 0; while ((1 << out.depth) < L) ++out.depth;
  // axis-aligned boxes, rounded outward, bottom-up; and per node a one-sided bound along its parent's split axis:
  // every point of a right (odd) node has coordinate >= face, of a left (even) node <= face (rounded conservatively,
  // the axis rides in the two low mantissa bits) -- the cheap split-plane test of the upward sweep.
  out.boxes.assign((size_t)2 * L, Box{{INFINITY, INFINITY, INFINITY}, {-INFINITY, -INFINITY, -INFINITY}, {0, 0}});
  std::vector<double> dlo((size_t)2 * L * 3, INFINITY), dhi((size_t)2 * L * 3, -INFINITY);
  for (int64_t l = 0; l < n_leaf; ++l)
    for (int64_t i = l * LEAF; i < std::min<int64_t>(n, (l + 1) * LEAF); ++i)
      for (int a = 0; a < 3; ++a) {
        const double v = pts[3 * (int64_t)out.order[i] + a];
        dlo[(L + l) * 3 + a] = std::min(dlo[(L + l) * 3 + a], v); dhi[(L + l) * 3 + a] = std::max(dhi[(L + l) * 3 + a], v);
      }
  for (int i = L - 1; i >= 1; --i)
    for (int a = 0; a < 3; ++a) {
      dlo[(size_t)i * 3 + a] = std::min(dlo[(size_t)2 * i * 3 + a], dlo[(size_t)(2 * i + 1) * 3 + a]);
      dhi[(size_t)i * 3 + a] = std::max(dhi[(size_t)2 * i * 3 + a], dhi[(size_t)(2 * i + 1) * 3 + a]);
    }
  out.faces.assign((size_t)2 * L, 0.f);
  for (int i = 1; i < 2 * L; ++i) {
    for (int a = 0; a < 3; ++a) { out.boxes[i].lo[a] = f_down(dlo[(size_t)i * 3 + a]); out.boxes[i].hi[a] = f_up(dhi[(size_t)i * 3 + a]); }
    if (i >= 2) {
      const int axp = axis_of[i / 2]; const bool right = (i & 1) != 0;
      float ff = right ? f_down(dlo[(size_t)i * 3 + axp]) : f_up(dhi[(size_t)i * 3 + axp]);   // +inf / -inf for empty nodes
      for (int guard = 0; guard < 8 && std::isfinite(ff); ++guard) {
        uint32_t bits; std::memcpy(&bits, &ff, 4);
        if ((bits & 3u) == (uint32_t)axp) break;
        ff = std::nextafterf(ff, right ? -INFINITY : INFINITY);
      }
      if (!std::isfinite(ff)) { uint32_t bits; std::memcpy(&bits, &ff, 4); bits = (bits & ~3u); std::memcpy(&ff, &bits, 4); }   // inf: low bits 0 = axis 0, any axis prunes
      out.faces[i] = ff;
    }
  }
  out.adj.assign((size_t)ADJ_SLOTS * L, 0);
  for (int l = 0; l < L; ++l) adj_build_leaf(out.boxes.data(), L, (int)n_leaf, l, out.adj.data() + (size_t)ADJ_SLOTS * l);
}



// ---- hybrid oriented boxes for the far-round search (far.cuh, MVICP_FLAG_OBB_FAR) ---------------------------------------
// Per node either the box of the coordinate axes or -- for nodes of at most OBB_PCA_LEAVES leaves whose principal-axes
// box is clearly smaller -- the box of the principal axes of its points.  The extents are taken in fp64 against the STORED
// fp32 centre and axes, so the containment the kernel relies on is exact for them; (1 + 1e-6) covers |A x| <= (1 + 1e-6)|x|
// for axes that are orthonormal to 2e-7 (else the node keeps the coordinate axes).
struct ObbHost { float c[3]; float e0; float a0[3]; float e1; float a1[3]; float e2; float a2[3]; float pad; };
static const double OBB_PCA_RATIO = 0.5;

static void build_obb(const double* pts, int64_t n, const HostFrameBuild& hb, std::vector<ObbHost>& out) {
  const int L = hb.n_leaf_pad;
  const int64_t n_leaf = std::max<int64_t>(1, (n + LEAF - 1) / LEAF);
  struct Mom { double n = 0, s[3] = {0, 0, 0}, ss[6] = {0, 0, 0, 0, 0, 0}; };
  std::vector<Mom> mom((size_t)2 * L);
  for (int64_t l = 0; l < n_leaf; ++l) {
    Mom& mm = mom[L + l];
    for (int64_t i = l * LEAF; i < std::min<int64_t>(n, (l + 1) * LEAF); ++i) {
      const double* p = pts + 3 * (int64_t)hb.order[i];
      mm.n += 1; for (int a = 0; a < 3; ++a) mm.s[a] += p[a];
      mm.ss[0] += p[0] * p[0]; mm.ss[1] += p[0] * p[1]; mm.ss[2] += p[0] * p[2]; mm.ss[3] += p[1] * p[1]; mm.ss[4] += p[1] * p[2]; mm.ss[5] += p[2] * p[2];
    }
  }
  for (int i = L - 1; i >= 1; --i) {
    Mom& mm = mom[i]; const Mom &x = mom[2 * i], &y = mom[2 * i + 1];
    mm.n = x.n + y.n; for (int a = 0; a < 3; ++a) mm.s[a] = x.s[a] + y.s[a]; for (int a = 0; a < 6; ++a) mm.ss[a] = x.ss[a] + y.ss[a];
  }
  ObbHost empty; std::memset(&empty, 0, sizeof empty);
  empty.a0[0] = empty.a1[1] = empty.a2[2] = 1.f; empty.e0 = empty.e1 = empty.e2 = -INFINITY;
  out.assign((size_t)2 * L, empty);
  for (int lev = 0; (1 << lev) <= L; ++lev) {
    const int first = 1 << lev, per = L >> lev;   // nodes of this level, leaves under each
    for (int i = first; i < 2 * first; ++i) {
      const Mom& mm = mom[i];
      if (mm.n < 1) continue;
      ObbHost& b = out[i];
      const double mean[3] = {mm.s[0] / mm.n, mm.s[1] / mm.n, mm.s[2] / mm.n};
      double C[3][3] = {{mm.ss[0] / mm.n - mean[0] * mean[0], mm.ss[1] / mm.n - mean[0] * mean[1], mm.ss[2] / mm.n - mean[0] * mean[2]},
                        {0, mm.ss[3] / mm.n - mean[1] * mean[1], mm.ss[4] / mm.n - mean[1] * mean[2]},
                        {0, 0, mm.ss[5] / mm.n - mean[2] * mean[2]}};
      C[1][0] = C[0][1]; C[2][0] = C[0][2]; C[2][1] = C[1][2];
      double V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
      if (mm.n >= 3 && per <= OBB_PCA_LEAVES) {   // cyclic Jacobi, symmetric 3x3
        for (int sweep = 0; sweep < 12; ++sweep) {
          if (std::fabs(C[0][1]) + std::fabs(C[0][2]) + std::fabs(C[1][2]) < 1e-30) break;
          for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
              if (std::fabs(C[p][q]) < 1e-300) continue;
              const double th = (C[q][q] - C[p][p]) / (2.0 * C[p][q]);
              const double tt = (th >= 0 ? 1.0 : -1.0) / (std::fabs(th) + std::sqrt(th * th + 1.0));
              const double cs = 1.0 / std::sqrt(tt * tt + 1.0), sn = tt * cs;
              for (int k = 0; k < 3; ++k) { const double ckp = C[k][p], ckq = C[k][q]; C[k][p] = cs * ckp - sn * ckq; C[k][q] = sn * ckp + cs * ckq; }
              for (int k = 0; k < 3; ++k) { const double cpk = C[p][k], cqk = C[q][k]; C[p][k] = cs * cpk - sn * cqk; C[q][k] = sn * cpk + cs * cqk; }
              for (int k = 0; k < 3; ++k) { const double vkp = V[k][p], vkq = V[k][q]; V[k][p] = cs * vkp - sn * vkq; V[k][q] = sn * vkp + cs * vkq; }
            }
        }
      }
      float* ax[3] = {b.a0, b.a1, b.a2};
      const int64_t lo_leaf = (int64_t)(i - first) * per;
      const int64_t t0 = lo_leaf * LEAF, t1 = std::min<int64_t>(n, (lo_leaf + per) * LEAF);
      double best_vol = INFINITY;
      for (int cand = 0; cand < 2; ++cand) {
        float A[3][3];
        for (int a = 0; a < 3; ++a) for (int k = 0; k < 3; ++k) A[a][k] = cand == 0 ? (a == k ? 1.f : 0.f) : (float)V[k][a];
        if (cand == 1) {
          if (per > OBB_PCA_LEAVES) break;
          bool ortho = true;
          for (int a = 0; a < 3; ++a)
            for (int k = a; k < 3; ++k) {
              const double dp = (double)A[a][0] * A[k][0] + (double)A[a][1] * A[k][1] + (double)A[a][2] * A[k][2];
              if (!(std::fabs(dp - (a == k ? 1.0 : 0.0)) < 2e-7)) ortho = false;
            }
          if (!ortho) break;
        }
        double mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
        for (int64_t t = t0; t < t1; ++t) {
          const double* p = pts + 3 * (int64_t)hb.order[t];
          const double d[3] = {p[0] - mean[0], p[1] - mean[1], p[2] - mean[2]};
          for (int a = 0; a < 3; ++a) {
            const double pr = (double)A[a][0] * d[0] + (double)A[a][1] * d[1] + (double)A[a][2] * d[2];
            mn[a] = std::min(mn[a], pr); mx[a] = std::max(mx[a], pr);
          }
        }
        float cf[3];
        for (int k = 0; k < 3; ++k) {
          double ck = mean[k];
          for (int a = 0; a < 3; ++a) ck += (double)A[a][k] * 0.5 * (mn[a] + mx[a]);
          cf[k] = (float)ck;
        }
        double ext[3] = {0, 0, 0};
        for (int64_t t = t0; t < t1; ++t) {
          const double* p = pts + 3 * (int64_t)hb.order[t];
          const double d[3] = {p[0] - (double)cf[0], p[1] - (double)cf[1], p[2] - (double)cf[2]};
          for (int a = 0; a < 3; ++a) ext[a] = std::max(ext[a], std::fabs((double)A[a][0] * d[0] + (double)A[a][1] * d[1] + (double)A[a][2] * d[2]));
        }
        const double floor_e = 1e-7 * (std::fabs(mean[0]) + std::fabs(mean[1]) + std::fabs(mean[2]) + 1e-3);
        const double vol = (ext[0] + floor_e) * (ext[1] + floor_e) * (ext[2] + floor_e);
        if (cand == 0 || vol < OBB_PCA_RATIO * best_vol) {
          best_vol = vol;
          for (int a = 0; a < 3; ++a) { b.c[a] = cf[a]; for (int k = 0; k < 3; ++k) ax[a][k] = A[a][k]; }
          b.e0 = f_up(ext[0] * (1.0 + 1e-6)); b.e1 = f_up(ext[1] * (1.0 + 1e-6)); b.e2 = f_up(ext[2] * (1.0 + 1e-6));
        }
      }
    }
  }
}
