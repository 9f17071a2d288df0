// knn.cuh -- exact nearest-neighbour correspondence kernel (replaces nanoflann on the hot path).
//
// Reference semantics reproduced (SURVEY 8(a) A2/A3/A5):
//   * query transform  g = R_s p + t_s ; q = Rinv_d (g - t_d)   src/internal/frame.cpp:117-118,131,136
//     in fp64, round-to-nearest after every multiply and add (no FMA contraction), left-fold sums;
//   * distance         (d0*d0 + d1*d1) + d2*d2 with d = q - p   include/frame.h:70-76, fp64, no FMA;
//   * result           the dst point minimising that value      nanoflann.hpp:1200-1247 (exact search, eps = 0);
//     ties (equal fp64 distance) resolve to the LOWEST ORIGINAL INDEX here, whereas nanoflann keeps the first
//     point its traversal meets (nanoflann.hpp:1210) -- documented deviation, counted by the tests;
//   * cutoff           sqrt(d2) < (double)thresh                 frame.cpp:142,156 -- evaluated as d2 <= d2max, the largest double
//                      whose correctly rounded square root is still below the threshold (cutoff_d2max; sqrt is monotone)
//
// Search structure: implicit binary AABB tree over leaves in left-balanced KD order (types.cuh), walked in fp32 with a
// conservative screen and re-ranked in fp64 (see "fp32 screening" below): the answer is the exact fp64 arg-min.
//
// Shortcuts, all exact (same index, same fp64 distance as the plain search; each with a flag that switches it off, mvicp.h):
//   * seeds            the previous round's match names the leaf the search starts in (nn_search);
//   * neighbour lists  a seeded query inside its start leaf's reach looks at that leaf and its listed neighbours only (nn_adj_fast);
//   * certificates     a search also reports the margin by which its match wins (nn_margin); in converged rounds a query that stayed
//                      within half that margin keeps its match without a search (knn_cert_kernel), the rest is searched densely
//                      (knn_todo_kernel);
//   * select epilogue  in converged rounds the kernels also count the inliers below / collect the keys inside a window around the
//                      previous median, which replaces the passes of the median select (knn_sel_account, select.cuh).
#pragma once
#include <cuda_runtime.h>
#include <limits.h>
#include <type_traits>
#include "adjacency.h"
#include "types.cuh"

namespace mv {

template <bool F32> struct Rec;
template <> struct Rec<true> {
  typedef float4 type;
  static __device__ __forceinline__ void load(const void* base, int64_t i, double& x, double& y, double& z, int& w) {
    const float4 r = __ldg(reinterpret_cast<const float4*>(base) + i);
    x = (double)r.x; y = (double)r.y; z = (double)r.z; w = __float_as_int(r.w);
  }
};
template <> struct Rec<false> {
  typedef double4a type;
  static __device__ __forceinline__ void load(const void* base, int64_t i, double& x, double& y, double& z, int& w) {
    const double2* p = reinterpret_cast<const double2*>(reinterpret_cast<const double4a*>(base) + i);
    const double2 a = __ldg(p), b = __ldg(p + 1);
    x = a.x; y = a.y; z = b.x; w = (int)__double_as_longlong(b.y);
  }
};

__device__ __forceinline__ double d2_rn(double qx, double qy, double qz, double px, double py, double pz) {
  const double d0 = __dsub_rn(qx, px), d1 = __dsub_rn(qy, py), d2 = __dsub_rn(qz, pz);
  return __dadd_rn(__dadd_rn(__dmul_rn(d0, d0), __dmul_rn(d1, d1)), __dmul_rn(d2, d2));
}

// ---- fp32 screening + fp64 exact re-rank ------------------------------------------------------------------------
// The tree is walked in fp32.  A candidate (or a box) is looked at exactly only if its fp32 distance does not exceed
// bound32, an upper bound -- rounded up, with the fp32 error budget added -- of the current exact best:
//   per-axis error of an fp32 difference (query rounded to fp32, rounded subtraction; stored coordinates exact in the
//   fp32 storage mode, rounded in the fp64 mode)  <= delta = 2^-23 (|q|_inf + absmax)
//   => computed d32 <= (D + sqrt(3) delta)^2 (1 + 2^-24)^3 for a point at true distance D (same for a box lower bound or
//   a split-plane distance), so every point with D^2 <= best satisfies
//   d32 <= bound32 := ru[(sqrt(best) + ea)^2 (1 + 1e-6)], ea = 6 sqrt(3) delta
//   (bound32 itself is evaluated in fp32 with every operation rounded up).
// Whatever passes the screen is re-evaluated with the reference's fp64 operation sequence (d2_rn) on the exact
// coordinates, and only that value decides: the result is the exact arg-min with the lowest-index tie rule.
struct NNQuery {
  double qx, qy, qz;     // exact query (dst-local)
  float fx, fy, fz;      // fp32 rounding of it
  float eaf;             // absolute error allowance on a distance (rounded up)
  double best; int bi;   // exact best so far
  float bound32;
};

// r >= sqrt(b): the hardware's approximate square root (2 ulp, one MUFU) scaled up by 1 + 2^-20 instead of the correctly rounded
// software sequence -- the bound only has to be an upper bound, and it is re-evaluated at every improvement of the best
__device__ __forceinline__ float sqrt_upper(float b) {
#ifdef __CUDA_ARCH__
  float r; asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(b));
  return __fmul_ru(r, 1.00000095367431640625f);
#else
  return __fsqrt_ru(b);
#endif
}

__device__ __forceinline__ void nn_tighten(NNQuery& s) {
  // (sqrt(best) + ea)^2 (1 + 1e-6), evaluated upward in fp32: b >= best, r >= sqrt(b)
  const float b = __double2float_ru(s.best);
  const float r = sqrt_upper(b);
  s.bound32 = __fmul_ru(__fmaf_ru(s.eaf, __fmaf_ru(2.0f, r, s.eaf), b), 1.000001f);
}

// ---- certificates (temporal coherence) ----------------------------------------------------------------------------------
// A search can also report how far the runner-up is: the smallest fp32 screen value of any point other than the winner that it
// looked at, and the smallest lower bound of anything it pruned (a box, a split plane, "outside the start leaf's reach").  With
// the error model above, everything except the winner lies at a true distance >= sqrt(other)(1 - 2^-22) - ea, the winner at
// sqrt(best): the difference is a MARGIN m.  If the query is later found within m/2 of where it was then (in the dst frame), the
// winner is still the strictly nearest point: |q'-p_j| <= d1 + D < d2 - D <= |q'-p_k| for D < m/2 -- no search needed, only its
// distance (knn_kernel, CERT).  A certificate is {where the query was (fp32), m}, 16 bytes per query, stored in the kernel's own
// (tile) order: read and written coalesced, renewed whenever the query has to be searched again.
struct NNQueryT : NNQuery {
  float m1, m2;     // the two smallest screen values over all scanned points
  float v1;         // screen value of the current winner
  float lbmin;      // smallest lower bound among everything pruned
};
template <class Q> struct nn_track { static constexpr bool value = false; };
template <> struct nn_track<NNQueryT> { static constexpr bool value = true; };

__device__ __forceinline__ void nn_track_init(NNQueryT& s) {
  const float inf = __int_as_float(0x7f800000);
  s.m1 = inf; s.m2 = inf; s.v1 = inf; s.lbmin = inf;
}
template <class Q> __device__ __forceinline__ void nn_pruned(Q& s, float lb) {
  if constexpr (nn_track<Q>::value) s.lbmin = fminf(s.lbmin, lb);
}
// (Pruning boxes and planes against a slightly larger bound while a certificate is written -- so that a box just outside the exact
// bound does not leave a margin of nothing -- keeps a few more queries but makes every search dearer.)
// r <= sqrt(b)
__device__ __forceinline__ float sqrt_lower(float b) {
#ifdef __CUDA_ARCH__
  float r; asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(b));
  return __fmul_rd(r, 0.99999904632568359375f);
#else
  return __fmul_rd(sqrtf(b), 0.99999904632568359375f);
#endif
}
// margin, rounded down (<= 0: no certificate).  The winner has to hold the smallest screen value itself; if another point does
// (fp32 reordering of near-equal distances, or the winner scanned twice) that point counts as the runner-up.
__device__ __forceinline__ float nn_margin(const NNQueryT& s) {
  const float other = fminf(s.v1 == s.m1 ? s.m2 : s.m1, s.lbmin);
  const float lo = __fsub_rd(__fmul_rd(sqrt_lower(other), 0.999999f), s.eaf);
  const float hi = sqrt_upper(__double2float_ru(s.best));
  return __fsub_rd(lo, __fmul_ru(hi, 1.000001f));
}

template <class Q>
__device__ __forceinline__ float box_lb32(const Box* __restrict__ boxes, int node, const Q& s) {
  const float4* b = reinterpret_cast<const float4*>(boxes + node);
  const float4 u = __ldg(b), v = __ldg(b + 1);   // u = lo.xyz, hi.x ; v = hi.yz
  const float dx = fmaxf(fmaxf(u.x - s.fx, s.fx - u.w), 0.f);
  const float dy = fmaxf(fmaxf(u.y - s.fy, s.fy - v.x), 0.f);
  const float dz = fmaxf(fmaxf(u.z - s.fz, s.fz - v.y), 0.f);
  return fmaf(dz, dz, fmaf(dy, dy, dx * dx));
}

// one candidate that passed the fp32 screen: exact fp64 distance in the reference's operation order
template <bool F32>
__device__ __forceinline__ void nn_exact(const FrameDev& fd, int64_t pos, const float4& r, NNQuery& s) {
  double px, py, pz; int pi;
  if (F32) { px = (double)r.x; py = (double)r.y; pz = (double)r.z; pi = __float_as_int(r.w); }
  else Rec<false>::load(fd.pts_s, pos, px, py, pz, pi);
  const double d = d2_rn(s.qx, s.qy, s.qz, px, py, pz);
  if (d < s.best || (d == s.best && pi < s.bi)) { s.best = d; s.bi = pi; nn_tighten(s); }
}

template <class Q>
__device__ __forceinline__ float pt_d32(const float4& r, const Q& s) {
  const float dx = s.fx - r.x, dy = s.fy - r.y, dz = s.fz - r.z;
  return fmaf(dz, dz, fmaf(dy, dy, dx * dx));
}

// two points of a leaf per step (the point arrays are padded with +inf up to a multiple of LEAF)
// track = false (certificates only): the screen values do not enter m1 / m2 -- the lane has scanned these points before, or is not
// searching; a data select rather than a branch, so that a warp walking together stays converged
template <bool F32, class Q>
__device__ __forceinline__ void nn_leaf_step(const FrameDev& fd, int leaf, int sub, Q& s, bool track = true) {
  const int64_t pos = (int64_t)leaf * LEAF + 2 * sub;
  if (pos >= fd.n) return;   // padding leaf of the implicit tree (reachable only while the bound is still infinite)
  const float4 r0 = __ldg(fd.pts_sf + pos), r1 = __ldg(fd.pts_sf + pos + 1);
  const float d0 = pt_d32(r0, s), d1 = pt_d32(r1, s);
  if constexpr (nn_track<Q>::value) {
    const float inf = __int_as_float(0x7f800000);
    const float t0 = track ? d0 : inf, t1 = track ? d1 : inf;
    s.m2 = fminf(s.m2, fmaxf(s.m1, t0)); s.m1 = fminf(s.m1, t0);
    s.m2 = fminf(s.m2, fmaxf(s.m1, t1)); s.m1 = fminf(s.m1, t1);
    int before = s.bi;
    if (d0 <= s.bound32) { nn_exact<F32>(fd, pos, r0, s); if (s.bi != before) { s.v1 = d0; before = s.bi; } }
    if (d1 <= s.bound32) { nn_exact<F32>(fd, pos + 1, r1, s); if (s.bi != before) s.v1 = d1; }
  } else {
    if (d0 <= s.bound32) nn_exact<F32>(fd, pos, r0, s);
    if (d1 <= s.bound32) nn_exact<F32>(fd, pos + 1, r1, s);
  }
}

// Exact 1-NN.  start_leaf >= 0: the leaf holding a good guess (previous round's match); < 0: greedy descent.
// Equivalent to a full depth-first search whose first root-to-leaf path is given: the start leaf is scanned, then the
// sibling subtree of every ancestor, bottom-up (nearest first), is searched if its box can still hold a closer point.
// The search loop is made of uniform steps -- "test two things": the two child boxes of an internal node, or two
// points of a leaf (a leaf takes LEAF/2 steps) -- so that the lanes of a warp, which sit at different nodes, still
// execute the same instructions; only the trip count differs between lanes.
constexpr int NN_STACK = 64;   // >= 2 * depth: flagged siblings + far children of one descent
// The rest of the search after the first root-to-leaf path: the stacked sibling subtrees, depth-first, nearest child first.
// WW = false: every trip of ONE loop does one uniform step -- "test the two child boxes of the current node" or "test two points of
//             the current leaf" -- whichever the lane needs (round 1's schedule);
// WW = true:  "while-while" (Aila & Laine): an inner loop runs node steps only until the lane holds the next leaf that can matter,
//             then all such lanes scan their leaves together -- a warp executes one kind of step at a time.
// lb_of(node) is the fp32 lower bound of a node's box (axis-aligned in knn.cuh, hybrid oriented in far.cuh).
template <bool F32, bool WW, class Q, class LBF>
__device__ __forceinline__ void nn_drain(const FrameDev& fd, Q& s, int* stk_n, float* stk_lb, int sp, LBF lb_of) {
  const int L = fd.n_leaf_pad;
  if (WW) {
    while (true) {
      int leaf = -1;
      while (sp > 0) {
        --sp;
        if (stk_lb[sp] > s.bound32) { nn_pruned(s, stk_lb[sp]); continue; }
        int node = stk_n[sp];
        while (node < L) {   // descend: nearer child first, the other one onto the stack
          const int c0 = 2 * node;
          const float l0 = lb_of(c0), l1 = lb_of(c0 + 1);
          const bool first0 = l0 <= l1;
          const float ln = first0 ? l0 : l1, lf = first0 ? l1 : l0;
          if (ln > s.bound32) { nn_pruned(s, ln); node = -1; break; }
          if (lf <= s.bound32) { stk_n[sp] = first0 ? c0 + 1 : c0; stk_lb[sp] = lf; ++sp; } else nn_pruned(s, lf);
          node = first0 ? c0 : c0 + 1;
        }
        if (node >= L) { leaf = node - L; break; }
      }
      if (leaf < 0) break;
#pragma unroll
      for (int sub = 0; sub < LEAF / 2; ++sub) nn_leaf_step<F32, Q>(fd, leaf, sub, s);
    }
  } else {
    int node = -1, sub = 0;
    while (true) {
      if (node < 0) {
        if (sp == 0) break;
        --sp;
        if (stk_lb[sp] > s.bound32) { nn_pruned(s, stk_lb[sp]); continue; }
        node = stk_n[sp]; sub = 0;
      }
      if (node >= L) {
        nn_leaf_step<F32, Q>(fd, node - L, sub, s);
        if (++sub == LEAF / 2) node = -1;
      } else {
        const int c0 = 2 * node;
        const float l0 = lb_of(c0), l1 = lb_of(c0 + 1);
        const bool first0 = l0 <= l1;
        const float ln = first0 ? l0 : l1, lf = first0 ? l1 : l0;
        if (ln <= s.bound32) {
          if (lf <= s.bound32) { stk_n[sp] = first0 ? c0 + 1 : c0; stk_lb[sp] = lf; ++sp; } else nn_pruned(s, lf);
          node = first0 ? c0 : c0 + 1; sub = 0;
        } else { nn_pruned(s, ln); node = -1; }
      }
    }
  }
}

// Inside the start leaf's reach (adjacency.h) the answer lies in this leaf -- already scanned by the caller, (u, v) its box -- or
// in one of its listed neighbours: test their boxes, scan the ones that can still hold a closer point; no walk up the ancestors,
// no descents.  Returns false, having done nothing, when the query is not inside the reach.
template <bool F32, class Q>
__device__ __forceinline__ bool nn_adj_fast(const FrameDev& fd, Q& s, int start_leaf, const float4 u, const float4 v) {
  if (!fd.adj) return false;
  const int L = fd.n_leaf_pad;
  const int32_t* ap = fd.adj + (size_t)ADJ_SLOTS * start_leaf;
  const int2 hd = __ldg(reinterpret_cast<const int2*>(ap));
  const float ex0 = fmaxf(fmaxf(u.x - s.fx, s.fx - u.w), 0.f), ey0 = fmaxf(fmaxf(u.y - s.fy, s.fy - v.x), 0.f), ez0 = fmaxf(fmaxf(u.z - s.fz, s.fz - v.y), 0.f);
  const float e2 = fmaf(ez0, ez0, fmaf(ey0, ey0, ex0 * ex0));
  // e + r <= R_S, every operation rounded up; the error of e (query and box in fp32) is inside the allowance that bound32 carries
  if (!(__fadd_ru(sqrt_upper(e2), sqrt_upper(s.bound32)) <= __int_as_float(hd.x))) return false;
  if constexpr (nn_track<Q>::value) {   // every leaf outside the list is further than R_S - e
    const float t = __fsub_rd(__int_as_float(hd.x), sqrt_upper(e2));
    nn_pruned(s, t > 0.f ? __fmul_rd(t, t) : 0.f);
  }
  unsigned todo = 0u;
  for (int i = 0; i < hd.y; ++i) {
    const int t = __ldg(ap + 2 + i);
    const float lb = box_lb32(fd.boxes, L + t, s);
    if (lb <= s.bound32) todo |= 1u << i; else nn_pruned(s, lb);
  }
  while (todo) {
    const int i = __ffs(todo) - 1; todo &= todo - 1u;
    const int t = __ldg(ap + 2 + i);
#pragma unroll
    for (int sub = 0; sub < LEAF / 2; ++sub) nn_leaf_step<F32, Q>(fd, t, sub, s);
  }
  return true;
}

template <bool F32, class Q, bool WW = false>
__device__ __forceinline__ void nn_search(const FrameDev& fd, Q& s, int start_leaf) {
  const int L = fd.n_leaf_pad;
  int leaf_node = -1;
  if (start_leaf >= 0) {
    leaf_node = L + start_leaf;
#pragma unroll
    for (int sub = 0; sub < LEAF / 2; ++sub) nn_leaf_step<F32, Q>(fd, start_leaf, sub, s);
    const float4* b = reinterpret_cast<const float4*>(fd.boxes + leaf_node);
    const float4 u = __ldg(b), v = __ldg(b + 1);
    if (nn_adj_fast<F32, Q>(fd, s, start_leaf, u, v)) return;
    // a stale guess (the poses moved a lot since it was made) leaves a loose bound, and everything inside that ball
    // would be visited on the way up: if the guess is further than a few leaf sizes, descend greedily instead
    const float ex = u.w - u.x, ey = v.x - u.y, ez = v.y - u.z;                 // extents of the leaf
    if (s.bound32 > 16.0f * fmaf(ez, ez, fmaf(ey, ey, ex * ex))) start_leaf = -1;
  }
  if (start_leaf < 0) {
    int node = 1;
    while (node < L) {
      const int c0 = 2 * node;
      const float l0 = box_lb32(fd.boxes, c0, s), l1 = box_lb32(fd.boxes, c0 + 1, s);
      node = (l1 < l0) ? c0 + 1 : c0;
    }
    if (node != leaf_node) {
#pragma unroll
      for (int sub = 0; sub < LEAF / 2; ++sub) nn_leaf_step<F32, Q>(fd, node - L, sub, s);
    }
    leaf_node = node;
  }

  int stk_n[NN_STACK]; float stk_lb[NN_STACK]; int sp = 0;
  // sibling subtrees that can matter at all, pushed top-down so that the nearest (lowest) one is popped first
  for (int l = fd.depth - 1; l >= 0; --l) {
    const int sib = (leaf_node >> l) ^ 1;
    // cheap pre-filter (what nanoflann prunes with, nanoflann.hpp:1237-1243): the split plane between the two siblings
    const float face = __ldg(fd.faces + sib);
    const int axis = __float_as_int(face) & 3;
    const float qa = axis == 0 ? s.fx : (axis == 1 ? s.fy : s.fz);
    const float dpl = (sib & 1) ? face - qa : qa - face;
    if (dpl > 0.f && dpl * dpl > s.bound32) { nn_pruned(s, dpl * dpl); continue; }
    const float lb = box_lb32(fd.boxes, sib, s);
    if (lb <= s.bound32) { stk_n[sp] = sib; stk_lb[sp] = lb; ++sp; } else nn_pruned(s, lb);
  }
  nn_drain<F32, WW, Q>(fd, s, stk_n, stk_lb, sp, [&](int nd) { return box_lb32(fd.boxes, nd, s); });
}

__device__ __forceinline__ void nn_query_init(NNQuery& s, double qx, double qy, double qz, float absmax) {
  s.qx = qx; s.qy = qy; s.qz = qz;
  s.fx = (float)qx; s.fy = (float)qy; s.fz = (float)qz;
  const double m = fmax(fmax(fabs(qx), fabs(qy)), fabs(qz)) + (double)absmax;
  s.eaf = __double2float_ru(6.0 * 1.7320508075688774 * 1.1920928955078125e-7 * m);
  s.best = __longlong_as_double(0x7ff0000000000000LL); s.bi = INT_MAX;
  s.bound32 = __int_as_float(0x7f800000);
}

// query transform, the operation sequence of knn_one (frame.cpp:117-118,131,136): g = R_s p + t_s ; q = Rinv_d (g - t_d)
__device__ __forceinline__ void edge_query(const EdgeXf& sx, double px, double py, double pz, double& qx, double& qy, double& qz) {
  const double gx = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(sx.Rs[0], px), __dmul_rn(sx.Rs[1], py)), __dmul_rn(sx.Rs[2], pz)), sx.ts[0]);
  const double gy = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(sx.Rs[3], px), __dmul_rn(sx.Rs[4], py)), __dmul_rn(sx.Rs[5], pz)), sx.ts[1]);
  const double gz = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(sx.Rs[6], px), __dmul_rn(sx.Rs[7], py)), __dmul_rn(sx.Rs[8], pz)), sx.ts[2]);
  const double ex = __dsub_rn(gx, sx.td[0]), ey = __dsub_rn(gy, sx.td[1]), ez = __dsub_rn(gz, sx.td[2]);
  qx = __dadd_rn(__dadd_rn(__dmul_rn(sx.Rinv[0], ex), __dmul_rn(sx.Rinv[1], ey)), __dmul_rn(sx.Rinv[2], ez));
  qy = __dadd_rn(__dadd_rn(__dmul_rn(sx.Rinv[3], ex), __dmul_rn(sx.Rinv[4], ey)), __dmul_rn(sx.Rinv[5], ez));
  qz = __dadd_rn(__dadd_rn(__dmul_rn(sx.Rinv[6], ex), __dmul_rn(sx.Rinv[7], ey)), __dmul_rn(sx.Rinv[8], ez));
}

// ---- packet walk: the 32 queries of a warp share one depth-first walk of the dst tree -----------------------------------------------
// Each lane has run its own prologue (a start-leaf scan, the greedy descent) for a first bound.  Then at every step all lanes look
// at the same node or leaf -- one broadcast load per warp.  A child is kept if any lane's bound admits it and the one with the
// smaller lower bound (over those lanes) is visited first; a popped entry is skipped when its lower bound exceeds every lane's bound,
// a popped leaf is first re-tested per lane.  Every node that can hold a point within a lane's bound is visited for that lane, and the
// arg-min with the lowest-index tie rule does not depend on the order in which candidates are met: same results as nn_search, bit
// for bit.  The stack holds at most one entry per level of the current path (<= depth < 32): entry i lives in a register of lane i.
// live = false: the lane has no query or its prologue settled it; it votes with a bound that admits nothing and records nothing --
//   only its bound32 is overwritten, its result and certificate terms stay as they are.
// skip0, skip1: leaf nodes the lane's prologue already scanned (or -1).  The lane does not vote for them, and when the warp visits
//   one anyway its screen values do not enter the lane's m1 / m2: a second scan would make the winner its own runner-up in the
//   certificate (nn_margin).  (Every lane runs every leaf scan: a lane that is not live admits nothing, and a lane re-scanning its own
//   points cannot change its best.  A lane-dependent branch around the scan left the warp unconverged at the pop, whose node index
//   and stack pointer sm_90a code keeps in uniform registers -- DESIGN 4.1.)
// Certificates (Q = NNQueryT): a live lane records its own lower bound for every child and every popped entry it does not visit
//   (nn_pruned), except for its skipped leaves, whose points its m1 / m2 already hold; a leaf the warp visits is scanned by every live
//   lane whose bound it exceeds as well, which only adds screen values of real points.
// lb_of(node) is the fp32 lower bound of a node's box (axis-aligned in knn.cuh, hybrid oriented in far.cuh).
template <bool F32, class Q, class LBF>
__device__ __forceinline__ void nn_packet_walk(const FrameDev& fd, Q& s, bool live, int skip0, int skip1, LBF lb_of) {
  const unsigned full = 0xffffffffu, inf_bits = 0x7f800000u;
  const float inf = __uint_as_float(inf_bits);
  const int L = fd.n_leaf_pad;
  const int lane = threadIdx.x & 31;
  if (!live) s.bound32 = -1.0f;
  int my_n = 0; float my_lb = 0.f;   // stack entry `lane`
  int sp = 0, node = 1;
  while (true) {
    if (node < L) {
      const int c0 = 2 * node;
      const float l0 = lb_of(c0), l1 = lb_of(c0 + 1);
      const bool i0 = l0 <= s.bound32, i1 = l1 <= s.bound32;
      const bool k0 = i0 && c0 != skip0 && c0 != skip1, k1 = i1 && c0 + 1 != skip0 && c0 + 1 != skip1;
      if constexpr (nn_track<Q>::value) { nn_pruned(s, live && !i0 ? l0 : inf); nn_pruned(s, live && !i1 ? l1 : inf); }
      const unsigned b0 = __ballot_sync(full, k0), b1 = __ballot_sync(full, k1);
      if (b0 && b1) {
        // non-negative floats order like their bit patterns: one integer min per child
        const unsigned m0 = __reduce_min_sync(full, k0 ? __float_as_uint(l0) : inf_bits);
        const unsigned m1 = __reduce_min_sync(full, k1 ? __float_as_uint(l1) : inf_bits);
        const bool f0 = m0 <= m1;
        if (lane == sp) { my_n = f0 ? c0 + 1 : c0; my_lb = __uint_as_float(f0 ? m1 : m0); }
        ++sp;
        node = f0 ? c0 : c0 + 1;
        continue;
      }
      if (b0 | b1) { node = b0 ? c0 : c0 + 1; continue; }
    } else {
      const bool first = live && node != skip0 && node != skip1;
#pragma unroll
      for (int sub = 0; sub < LEAF / 2; ++sub) nn_leaf_step<F32, Q>(fd, node - L, sub, s, first);
    }
    node = -1;
    while (sp > 0) {
      --sp;
      const int nd = __shfl_sync(full, my_n, sp);
      const float m = __shfl_sync(full, my_lb, sp);
      if (m > __uint_as_float(__reduce_max_sync(full, __float_as_uint(fmaxf(s.bound32, 0.f))))) {
        if constexpr (nn_track<Q>::value) {   // beyond every lane's bound, so beyond this lane's (unless it skips the leaf)
          const float l = lb_of(nd);
          nn_pruned(s, live && !(l <= s.bound32) ? l : inf);
        }
        continue;
      }
      if (nd >= L) {
        const float l = lb_of(nd);
        const bool i = l <= s.bound32;
        if (!__ballot_sync(full, i && nd != skip0 && nd != skip1)) {
          if constexpr (nn_track<Q>::value) nn_pruned(s, live && !i ? l : inf);
          continue;
        }
      }
      node = nd;
      break;
    }
    if (node < 0) break;
  }
}

// One (edge, src point) query: transform, seed, [certificate test], search, results.  MODE 0: always search; 1: keep the match if
// the certificate allows it (returns 1), otherwise do nothing and return 0 -- the caller searches it later; 2: search (no test).
template <bool F32, bool WW, int CERT, int MODE>
__device__ __forceinline__ int knn_one(const FrameDev& fs, const FrameDev& fd, const EdgeXf& sx, const EdgeDev& e, int ks,
                                       int32_t* corr, double* __restrict__ d2out, const int32_t* seed, double thresh /* cutoff_d2max */,
                                       float4* __restrict__ certs, bool& inlier, double& best) {
  double px, py, pz; int orig;
  Rec<F32>::load(fs.pts_s, ks, px, py, pz, orig);
  // g = R_s p + t_s
  const double gx = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(sx.Rs[0], px), __dmul_rn(sx.Rs[1], py)), __dmul_rn(sx.Rs[2], pz)), sx.ts[0]);
  const double gy = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(sx.Rs[3], px), __dmul_rn(sx.Rs[4], py)), __dmul_rn(sx.Rs[5], pz)), sx.ts[1]);
  const double gz = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(sx.Rs[6], px), __dmul_rn(sx.Rs[7], py)), __dmul_rn(sx.Rs[8], pz)), sx.ts[2]);
  const double ex = __dsub_rn(gx, sx.td[0]), ey = __dsub_rn(gy, sx.td[1]), ez = __dsub_rn(gz, sx.td[2]);
  const double qx = __dadd_rn(__dadd_rn(__dmul_rn(sx.Rinv[0], ex), __dmul_rn(sx.Rinv[1], ey)), __dmul_rn(sx.Rinv[2], ez));
  const double qy = __dadd_rn(__dadd_rn(__dmul_rn(sx.Rinv[3], ex), __dmul_rn(sx.Rinv[4], ey)), __dmul_rn(sx.Rinv[5], ez));
  const double qz = __dadd_rn(__dadd_rn(__dmul_rn(sx.Rinv[6], ex), __dmul_rn(sx.Rinv[7], ey)), __dmul_rn(sx.Rinv[8], ez));

  typedef typename std::conditional<CERT != 0, NNQueryT, NNQuery>::type QT;
  QT nq; nn_query_init(nq, qx, qy, qz, fd.absmax);
  int start_leaf = -1, si = -1;
  if (seed) {   // previous round's match: a valid first guess, the search stays exact
    const int sd = seed[e.off + orig];
    si = sd >= 0 ? sd : ~sd;
    if (!(si >= 0 && si < fd.n)) si = -1;
    else if (MODE != 1) start_leaf = __ldg(fd.pos_of + si) / LEAF;
  }
  if constexpr (MODE == 1) {
    // displacement since the certificate, rounded up, + the fp32 rounding of both positions (eaf covers it many times over)
    const float4 ct = certs[e.off + ks];
    const float dx = nq.fx - ct.x, dy = nq.fy - ct.y, dz = nq.fz - ct.z;
    const float disp = __fadd_ru(__fmul_ru(sqrt_upper(__fmaf_ru(dz, dz, __fmaf_ru(dy, dy, __fmul_ru(dx, dx)))), 1.000001f), nq.eaf);
    if (!(si >= 0 && __fmul_ru(2.0f, disp) < ct.w)) return 0;
    // the previous match is still strictly nearer than anything else; its distance in the reference's operations
    double mx, my, mz; int dummy;
    Rec<F32>::load(fd.pts_o, si, mx, my, mz, dummy);
    nq.best = d2_rn(qx, qy, qz, mx, my, mz); nq.bi = si;
  } else {
    if constexpr (CERT != 0) nn_track_init(nq);
    nn_search<F32, QT, WW>(fd, nq, start_leaf);
    if constexpr (CERT != 0) certs[e.off + ks] = make_float4(nq.fx, nq.fy, nq.fz, nn_margin(nq));
  }
  best = nq.best; const int bi = nq.bi;
  inlier = best <= thresh;
  corr[e.off + orig] = inlier ? bi : ~bi;
  d2out[e.off + orig] = best;
  return 1;
}

// Exact 1-NN for the 32 queries of a warp, every lane calls it (has = the lane holds a query, initialised in s).  Each lane runs
// nn_search's prologue on its own: the start-leaf scan, the neighbour lists (nn_adj_fast), then the stale-seed rule or the greedy
// descent.  A lane the neighbour lists settle is done; the others share one packet walk (nn_packet_walk) instead of each walking the
// ancestors with a local-memory stack in a diverged warp, and a warp with no such lane skips the walk.  Same result as nn_search.
template <bool F32, class Q>
__device__ __forceinline__ void nn_search_packet(const FrameDev& fd, Q& s, bool has, int start_leaf) {
  const int L = fd.n_leaf_pad;
  int skip0 = -1, skip1 = -1;
  bool live = has;
  if (has) {
    if (start_leaf >= 0) {
      skip0 = L + start_leaf;
#pragma unroll
      for (int sub = 0; sub < LEAF / 2; ++sub) nn_leaf_step<F32, Q>(fd, start_leaf, sub, s);
      const float4* b = reinterpret_cast<const float4*>(fd.boxes + skip0);
      const float4 u = __ldg(b), v = __ldg(b + 1);
      if (nn_adj_fast<F32, Q>(fd, s, start_leaf, u, v)) live = false;
      else {   // the stale-seed rule of nn_search
        const float bx = u.w - u.x, by = v.x - u.y, bz = v.y - u.z;
        if (s.bound32 > 16.0f * fmaf(bz, bz, fmaf(by, by, bx * bx))) start_leaf = -1;
      }
    }
    if (live && start_leaf < 0) {
      int node = 1;
      while (node < L) {
        const int c0 = 2 * node;
        const float l0 = box_lb32(fd.boxes, c0, s), l1 = box_lb32(fd.boxes, c0 + 1, s);
        node = (l1 < l0) ? c0 + 1 : c0;
      }
      if (node != skip0) {
#pragma unroll
        for (int sub = 0; sub < LEAF / 2; ++sub) nn_leaf_step<F32, Q>(fd, node - L, sub, s);
      }
      skip1 = node;
    }
  }
  if (__ballot_sync(0xffffffffu, live))
    nn_packet_walk<F32, Q>(fd, s, live, skip0, skip1, [&](int nd) { return box_lb32(fd.boxes, nd, s); });
}

// knn_one (MODE 0) with the packet fall-through (nn_search_packet); every lane of the warp calls it (has = the lane holds a query)
template <bool F32, int CERT>
__device__ __forceinline__ void knn_one_packet(const FrameDev& fs, const FrameDev& fd, const EdgeXf& sx, const EdgeDev& e, int ks, bool has,
                                               int32_t* corr, double* __restrict__ d2out, const int32_t* seed, double thresh,
                                               float4* __restrict__ certs, bool& inlier, double& best) {
  typedef typename std::conditional<CERT != 0, NNQueryT, NNQuery>::type QT;
  QT nq;
  int orig = 0, start_leaf = -1;
  if (has) {
    double px, py, pz, qx, qy, qz;
    Rec<F32>::load(fs.pts_s, ks, px, py, pz, orig);
    edge_query(sx, px, py, pz, qx, qy, qz);
    nn_query_init(nq, qx, qy, qz, fd.absmax);
    if constexpr (CERT != 0) nn_track_init(nq);
    if (seed) {   // previous round's match: a valid first guess, the search stays exact
      const int sd = seed[e.off + orig];
      const int si = sd >= 0 ? sd : ~sd;
      if (si >= 0 && si < fd.n) start_leaf = __ldg(fd.pos_of + si) / LEAF;
    }
  } else {
    nn_query_init(nq, 0.0, 0.0, 0.0, fd.absmax);
  }
  nn_search_packet<F32, QT>(fd, nq, has, start_leaf);
  if (!has) return;
  if constexpr (CERT != 0) certs[e.off + ks] = make_float4(nq.fx, nq.fy, nq.fz, nn_margin(nq));
  best = nq.best; const int bi = nq.bi;
  inlier = best <= thresh;
  corr[e.off + orig] = inlier ? bi : ~bi;
  d2out[e.off + orig] = best;
}

// what a finished query contributes to the guessed median select; every lane of the warp calls it (`done` = has a result)
__device__ __forceinline__ void knn_sel_account(const SelGuess& sg, int edge, int n_edges, bool done, bool inlier, double best, unsigned int* s_cnt) {
  const unsigned long long key = (unsigned long long)__double_as_longlong(best);
  const unsigned long long lo = sg.win[edge], hi = sg.win[(size_t)n_edges + edge];
  const bool in = done && inlier;
  const unsigned int m_in = __ballot_sync(0xffffffffu, in), m_lo = __ballot_sync(0xffffffffu, in && key < lo);
  if ((threadIdx.x & 31) == 0) { if (m_in) atomicAdd(&s_cnt[0], (unsigned int)__popc(m_in)); if (m_lo) atomicAdd(&s_cnt[1], (unsigned int)__popc(m_lo)); }
  if (in && key >= lo && key < hi) {
    const unsigned int slot = atomicAdd(&sg.cand_n[edge], 1u);
    if (slot < (unsigned int)SEL_CAP) sg.cand[(size_t)edge * SEL_CAP + slot] = key;
  }
}

// One thread per (edge, src point) query; src points are walked in the src frame's tree order so that the
// lanes of a warp descend the dst tree together.
// WW = true: the queries the neighbour lists do not settle share one packet walk per warp (knn_one_packet); WW = false
// (MVICP_FLAG_STEP_LOOP): every lane runs nn_search with the one-step loop of nn_drain -- the per-lane reference.
// SEL: the epilogue also feeds the guessed median select (select.cuh): per edge, the number of inliers, the number of inliers
// below the guessed window of keys, and the keys inside the window.
// CERT = 1 (needs seeds): every query also leaves a certificate {its position, the margin by which its match beats everything
// else (nn_margin)} for the certified rounds that follow (knn_cert_kernel).
template <bool F32, bool WW, bool SEL = false, int CERT = 0>
__global__ void __launch_bounds__(KNN_TILE, 5)   // 5 CTAs per SM = 48 registers: the SEL epilogue must not cost a CTA of occupancy
knn_kernel(const FrameDev* __restrict__ frames, const EdgeDev* __restrict__ edges, const EdgeXf* __restrict__ xfs,
           const Tile* __restrict__ tiles, int32_t* corr /* aliases seed */, double* __restrict__ d2out,
           const int32_t* seed, double thresh, SelGuess sg, int n_edges /* stride of sg.win */, float4* __restrict__ certs) {
  const Tile t = tiles[blockIdx.x];
  const EdgeDev e = edges[t.edge];
  __shared__ EdgeXf sx;
  __shared__ unsigned int s_cnt[2];            // inliers | inliers below the window
  if (SEL && threadIdx.x < 2) s_cnt[threadIdx.x] = 0u;
  {
    const double* g = reinterpret_cast<const double*>(xfs + t.edge);
    double* s = reinterpret_cast<double*>(&sx);
    for (int i = threadIdx.x; i < (int)(sizeof(EdgeXf) / sizeof(double)); i += blockDim.x) s[i] = g[i];
  }
  __syncthreads();
  const FrameDev fs = frames[e.src];
  const FrameDev fd = frames[e.dst];
  const int ks = t.start + threadIdx.x;
  // the packet walk needs the whole warp: only a warp wholly past the edge's end leaves early
  if (!SEL && (WW ? t.start + (int)(threadIdx.x & ~31u) : ks) >= e.n_src) return;
  bool inlier = false; double best = 0.0;
  const bool has = ks < e.n_src;
  if (WW) knn_one_packet<F32, CERT>(fs, fd, sx, e, ks, has, corr, d2out, seed, thresh, certs, inlier, best);
  else if (has) knn_one<F32, false, CERT, 0>(fs, fd, sx, e, ks, corr, d2out, seed, thresh, certs, inlier, best);
  if (SEL) {   // every thread of the CTA arrives here
    knn_sel_account(sg, t.edge, n_edges, has, inlier, best, s_cnt);
    __syncthreads();
    if (threadIdx.x == 0) {
      if (s_cnt[0]) atomicAdd(&sg.total[t.edge], s_cnt[0]);
      if (s_cnt[1]) atomicAdd(&sg.below[t.edge], s_cnt[1]);
    }
  }
}

// ---- certified rounds: two launches instead of knn_kernel -------------------------------------------------------------------------
// knn_cert_kernel streams over all queries: a query that is still within half its margin of the certified position keeps its match
// and only recomputes the distance (knn_one, MODE 1); the others are appended to a device-wide list.  knn_todo_kernel then searches
// and re-certifies the listed queries with every lane busy.  (Searching them inside the first kernel, even compacted per CTA, is
// slower than searching everything: a CTA's finished warps hold their slots while one warp walks the tree.)
struct CertTodo { int2* list; unsigned int* n; };     // {edge, position in the src frame's tree order}

template <bool F32>
__global__ void __launch_bounds__(KNN_TILE)
knn_cert_kernel(const FrameDev* __restrict__ frames, const EdgeDev* __restrict__ edges, const EdgeXf* __restrict__ xfs,
                const Tile* __restrict__ tiles, int32_t* corr /* aliases seed */, double* __restrict__ d2out,
                const int32_t* seed, double thresh, SelGuess sg, int n_edges, float4* __restrict__ certs,
                unsigned long long* __restrict__ reused /* per edge */, CertTodo todo) {
  const Tile t = tiles[blockIdx.x];
  const EdgeDev e = edges[t.edge];
  __shared__ EdgeXf sx;
  __shared__ unsigned int s_cnt[4];            // inliers | inliers below the window | kept by certificate | to be searched
  __shared__ unsigned int s_base;
  __shared__ unsigned short s_list[KNN_TILE];
  if (threadIdx.x < 4) s_cnt[threadIdx.x] = 0u;
  {
    const double* g = reinterpret_cast<const double*>(xfs + t.edge);
    double* s = reinterpret_cast<double*>(&sx);
    for (int i = threadIdx.x; i < (int)(sizeof(EdgeXf) / sizeof(double)); i += blockDim.x) s[i] = g[i];
  }
  __syncthreads();
  const FrameDev fs = frames[e.src];
  const FrameDev fd = frames[e.dst];
  const int ks = t.start + threadIdx.x;
  bool inlier = false; double best = 0.0;
  int kept = 0;
  if (ks < e.n_src) {
    kept = knn_one<F32, true, 1, 1>(fs, fd, sx, e, ks, corr, d2out, seed, thresh, certs, inlier, best);
    if (!kept) s_list[atomicAdd(&s_cnt[3], 1u)] = (unsigned short)threadIdx.x;
  }
  knn_sel_account(sg, t.edge, n_edges, kept != 0, inlier, best, s_cnt);
  const unsigned int mk = __ballot_sync(0xffffffffu, kept != 0);
  if ((threadIdx.x & 31) == 0 && mk) atomicAdd(&s_cnt[2], (unsigned int)__popc(mk));
  __syncthreads();
  if (threadIdx.x == 0) {
    if (s_cnt[0]) atomicAdd(&sg.total[t.edge], s_cnt[0]);
    if (s_cnt[1]) atomicAdd(&sg.below[t.edge], s_cnt[1]);
    if (s_cnt[2]) atomicAdd(&reused[t.edge], (unsigned long long)s_cnt[2]);
    s_base = s_cnt[3] ? atomicAdd(todo.n, s_cnt[3]) : 0u;
  }
  __syncthreads();
  for (unsigned int i = threadIdx.x; i < s_cnt[3]; i += blockDim.x) todo.list[s_base + i] = make_int2(t.edge, t.start + (int)s_list[i]);
}

template <bool F32>
__global__ void __launch_bounds__(KNN_TILE, 5)
knn_todo_kernel(const FrameDev* __restrict__ frames, const EdgeDev* __restrict__ edges, const EdgeXf* __restrict__ xfs,
                int32_t* corr /* aliases seed */, double* __restrict__ d2out, const int32_t* seed, double thresh,
                SelGuess sg, int n_edges, float4* __restrict__ certs, CertTodo todo) {
  const unsigned int n = *todo.n, lane = threadIdx.x & 31u;
  for (unsigned int base = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < n; base += gridDim.x * blockDim.x) {   // warp-uniform
    const unsigned int i = base + lane;
    const bool has = i < n;
    int edge = 0; bool inlier = false; double best = 0.0;
    if (has) {
      const int2 it = todo.list[i];
      edge = it.x;
      const EdgeDev e = edges[edge];
      const FrameDev fs = frames[e.src];
      const FrameDev fd = frames[e.dst];
      knn_one<F32, true, 1, 2>(fs, fd, xfs[edge], e, it.y, corr, d2out, seed, thresh, certs, inlier, best);
    }
    // what the searched queries contribute to the guessed select, summed over the lanes of equal edge first
    const bool in = has && inlier;
    const unsigned long long key = (unsigned long long)__double_as_longlong(best);
    const unsigned long long lo = sg.win[edge], hi = sg.win[(size_t)n_edges + edge];
    const unsigned int grp = __match_any_sync(0xffffffffu, in ? edge : (int)(0x40000000u | lane));
    const unsigned int m_lo = __ballot_sync(0xffffffffu, in && key < lo) & grp;
    if (in && lane == (unsigned int)(__ffs(grp) - 1)) {
      atomicAdd(&sg.total[edge], (unsigned int)__popc(grp));
      if (m_lo) atomicAdd(&sg.below[edge], (unsigned int)__popc(m_lo));
    }
    if (in && key >= lo && key < hi) {
      const unsigned int slot = atomicAdd(&sg.cand_n[edge], 1u);
      if (slot < (unsigned int)SEL_CAP) sg.cand[(size_t)edge * SEL_CAP + slot] = key;
    }
  }
}

template <bool F32>
__global__ void knn_single_kernel(const FrameDev* __restrict__ frames, int frame, double qx, double qy, double qz,
                                  long long* out_idx, double* out_d2) {
  const FrameDev fd = frames[frame];
  NNQuery nq; nn_query_init(nq, qx, qy, qz, fd.absmax);
  nn_search<F32, NNQuery>(fd, nq, -1);
  *out_idx = nq.bi; *out_d2 = nq.best;
}

// Per-edge constants from the current poses (poses16: column-major 4x4 per frame), with the reference's
// arithmetic: general 3x3 inverse by cofactors (frame.cpp:118; Eigen's size-3 inverse).
__global__ void edge_xf_kernel(const double* __restrict__ poses16, const EdgeDev* __restrict__ edges, int n_edges,
                               EdgeXf* __restrict__ out) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const double* Ps = poses16 + 16 * edges[e].src;
  const double* Pd = poses16 + 16 * edges[e].dst;
  EdgeXf x;
  double M[9];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) { x.Rs[3 * i + j] = Ps[4 * j + i]; M[3 * i + j] = Pd[4 * j + i]; }
    x.ts[i] = Ps[12 + i]; x.td[i] = Pd[12 + i];
  }
  auto cof = [&](int i, int j) {
    const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
    return __dsub_rn(__dmul_rn(M[3 * i1 + j1], M[3 * i2 + j2]), __dmul_rn(M[3 * i1 + j2], M[3 * i2 + j1]));
  };
  const double c00 = cof(0, 0), c10 = cof(1, 0), c20 = cof(2, 0);
  const double det = __dadd_rn(__dadd_rn(__dmul_rn(c00, M[0]), __dmul_rn(c10, M[3])), __dmul_rn(c20, M[6]));
  const double invdet = __ddiv_rn(1.0, det);
  x.Rinv[0] = __dmul_rn(c00, invdet); x.Rinv[1] = __dmul_rn(c10, invdet); x.Rinv[2] = __dmul_rn(c20, invdet);
  x.Rinv[3] = __dmul_rn(cof(0, 1), invdet); x.Rinv[4] = __dmul_rn(cof(1, 1), invdet); x.Rinv[5] = __dmul_rn(cof(2, 1), invdet);
  x.Rinv[6] = __dmul_rn(cof(0, 2), invdet); x.Rinv[7] = __dmul_rn(cof(1, 2), invdet); x.Rinv[8] = __dmul_rn(cof(2, 2), invdet);
  out[e] = x;
}

}  // namespace mv
