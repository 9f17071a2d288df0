// adjacency.h -- per-leaf neighbour lists of the search tree, and the reach within which they are complete.
//
// For leaf S:  adj(S) = every other leaf T whose box lies within R_S of S's box (at most ADJ_MAX of them; R_S is at most
// ADJ_REACH leaf diagonals and is shrunk until the list fits).  Why it is exact: let q be a query, s* the point of box(S) nearest
// to q, e = |q - s*|.  A point p of leaf T with |p - q| <= r satisfies boxdist(S, T) <= |s* - p| <= e + r.  So if e + r <= R_S
// every point within r of q lies in S or in a leaf of adj(S): a seeded query whose start leaf gives it a reach e + r <= R_S
// needs no tree walk at all -- it tests the listed leaves' boxes and scans those that can still hold a closer point (knn.cuh).
// Motivation (config 3, converged round): the walk up 15 ancestor levels and the divergent descents that follow find on
// average 0.6 neighbouring leaves per query; with R_S = 0.6 diagonals 95 % of the queries are inside their leaf's reach and
// the lists hold 9-10 leaves (host model, tools/sim_search.cpp).
// Boxes are the stored fp32 boxes (rounded outward): distances between them can only be SMALLER than between the true boxes,
// so a list can only gain members by rounding, never lose one.
#pragma once
#include <math.h>
#include <stdint.h>
#include "types.cuh"

#if defined(__CUDACC__)
#define MV_ADJ_HD __host__ __device__
#else
#define MV_ADJ_HD
#endif

namespace mv {

constexpr int ADJ_SLOTS = 16;              // ints per leaf: [0] R_S as float bits, [1] count, [2..15] neighbouring leaf indices
constexpr int ADJ_MAX = ADJ_SLOTS - 2;
constexpr double ADJ_REACH = 0.6;          // x leaf diagonal
constexpr int ADJ_CAND = 48;               // candidates gathered per attempt before the reach is halved

MV_ADJ_HD inline double adj_boxdist2(const Box& a, const Box& b) {
  double s = 0.0;
  for (int k = 0; k < 3; ++k) {
    const double d1 = (double)a.lo[k] - (double)b.hi[k], d2 = (double)b.lo[k] - (double)a.hi[k];
    const double d = d1 > d2 ? d1 : d2;
    if (d > 0.0) s += d * d;
  }
  return s;
}

// boxes: heap order, 2L entries; n_leaf: leaves that hold points; out: ADJ_SLOTS ints of leaf `leaf`
MV_ADJ_HD inline void adj_build_leaf(const Box* boxes, int L, int n_leaf, int leaf, int32_t* out) {
  for (int i = 0; i < ADJ_SLOTS; ++i) out[i] = 0;
  if (leaf >= n_leaf || L < 2) return;                 // empty slot / single-leaf tree: reach 0, no list
  const Box me = boxes[L + leaf];
  double diag2 = 0.0;
  for (int k = 0; k < 3; ++k) { const double d = (double)me.hi[k] - (double)me.lo[k]; diag2 += d * d; }
  if (!(diag2 > 0.0) || !(diag2 < 1e300)) return;
  double R2 = ADJ_REACH * ADJ_REACH * diag2;
  double cd[ADJ_CAND]; int32_t ci[ADJ_CAND]; int nc = 0; bool complete = false;
  for (int attempt = 0; attempt < 6 && !complete; ++attempt, R2 *= 0.25) {
    nc = 0; complete = true;
    int stack[64]; int sp = 0; stack[sp++] = 1;
    while (sp > 0 && complete) {
      const int node = stack[--sp];
      const double d2 = adj_boxdist2(me, boxes[node]);
      if (!(d2 <= R2)) continue;
      if (node >= L) {
        if (node - L == leaf) continue;
        if (nc == ADJ_CAND) { complete = false; break; }
        cd[nc] = d2; ci[nc] = node - L; ++nc;
      } else { stack[sp++] = 2 * node; stack[sp++] = 2 * node + 1; }
    }
    if (complete) break;
  }
  if (!complete) return;                               // a leaf with masses of neighbours even at 1/1000 of its reach: no list
  // ascending distance (insertion sort: nc <= 48)
  for (int i = 1; i < nc; ++i) { const double d = cd[i]; const int32_t id = ci[i]; int j = i - 1; while (j >= 0 && cd[j] > d) { cd[j + 1] = cd[j]; ci[j + 1] = ci[j]; --j; } cd[j + 1] = d; ci[j + 1] = id; }
  double Rd = sqrt(R2); int keep = nc;
  if (nc > ADJ_MAX) {   // keep the leaves strictly nearer than the first one that does not fit; the reach ends below that one
    const double dcut = cd[ADJ_MAX];
    keep = 0; while (keep < nc && cd[keep] < dcut) ++keep;
    Rd = sqrt(dcut);
    if (keep > ADJ_MAX) keep = ADJ_MAX;                // (cannot happen: cd[keep] < dcut holds for at most ADJ_MAX entries)
  }
  float Rf = (float)Rd;
  while (Rf > 0.f && ((double)Rf >= Rd || (nc > ADJ_MAX && (double)Rf * (double)Rf >= cd[ADJ_MAX]))) Rf = nextafterf(Rf, 0.f);   // stored reach: strictly inside
  if (!(Rf > 0.f)) return;
  union { float f; int32_t i; } u; u.f = Rf;
  out[0] = u.i; out[1] = keep;
  for (int i = 0; i < keep; ++i) out[2 + i] = ci[i];
}

}  // namespace mv
