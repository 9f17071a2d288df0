// tools/sim_search.cpp -- CPU model of csrc/knn.cuh's search loop that COUNTS steps (box tests, point tests) per query.
// Development aid only (lets tree/bound variants be compared without a GPU); not part of the product or the oracle.
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <vector>
#include "../mv_lm_icp_b200/csrc/tree_build.h"

struct Sim { HostFrameBuild b; std::vector<float> px, py, pz; std::vector<int> pi; int64_t n; const double* pts; std::vector<ObbHost> ob; };

static inline float lb32(const Box& b, float fx, float fy, float fz) {
  const float dx = std::fmax(std::fmax(b.lo[0] - fx, fx - b.hi[0]), 0.f), dy = std::fmax(std::fmax(b.lo[1] - fy, fy - b.hi[1]), 0.f),
              dz = std::fmax(std::fmax(b.lo[2] - fz, fz - b.hi[2]), 0.f);
  return dx * dx + dy * dy + dz * dz;
}

// far.cuh:obb_lb32, the hybrid bound of the far rounds: oriented boxes at and below the PCA level (sim_set_obb)
static inline float obb_lb(const ObbHost& b, float fx, float fy, float fz) {
  const float dx = fx - b.c[0], dy = fy - b.c[1], dz = fz - b.c[2];
  const float p0 = std::fma(b.a0[2], dz, std::fma(b.a0[1], dy, b.a0[0] * dx));
  const float p1 = std::fma(b.a1[2], dz, std::fma(b.a1[1], dy, b.a1[0] * dx));
  const float p2 = std::fma(b.a2[2], dz, std::fma(b.a2[1], dy, b.a2[0] * dx));
  const float g0 = std::fmax(std::fabs(p0) - b.e0, 0.f), g1 = std::fmax(std::fabs(p1) - b.e1, 0.f), g2 = std::fmax(std::fabs(p2) - b.e2, 0.f);
  return std::fma(g2, g2, std::fma(g1, g1, g0 * g0));
}
static int g_obb = 0;
static inline float lbn(const Sim& s, int nd, float fx, float fy, float fz) {
  if (g_obb && nd >= s.b.n_leaf_pad / OBB_PCA_LEAVES) return obb_lb(s.ob[nd], fx, fy, fz);
  return lb32(s.b.boxes[nd], fx, fy, fz);
}

extern "C" {
static unsigned char* g_trace = nullptr; static int g_trace_cap = 0, g_trace_n = 0;
extern "C" void sim_set_trace(unsigned char* t, int cap) { g_trace = t; g_trace_cap = cap; }
extern "C" int sim_trace_len() { return g_trace_n; }
static double g_cap = INFINITY; static int g_coarse = 0;
extern "C" void sim_set_coarse(int c) { g_coarse = c; }
void sim_config(int, double) {}
void sim_set_cap(double c) { g_cap = c; }
void* sim_build(const double* pts, int64_t n) {
  Sim* s = new Sim(); s->n = n; s->pts = pts;
  build_frame(pts, n, s->b);
  const int64_t npad = ((n + LEAF - 1) / LEAF) * LEAF;
  s->px.assign(npad, INFINITY); s->py.assign(npad, INFINITY); s->pz.assign(npad, INFINITY); s->pi.assign(npad, INT32_MAX);
  for (int64_t i = 0; i < n; ++i) { const int o = s->b.order[i]; s->px[i] = (float)pts[3 * o]; s->py[i] = (float)pts[3 * o + 1]; s->pz[i] = (float)pts[3 * o + 2]; s->pi[i] = o; }
  return s;
}
// 1: every lower bound of sim_query / sim_packet is far.cuh's hybrid one (the oriented boxes are built on first use)
void sim_set_obb(void* h, int on) { Sim& s = *(Sim*)h; g_obb = on; if (on && s.ob.empty()) build_obb(s.pts, s.n, s.b, s.ob); }
void sim_free(void* h) { delete (Sim*)h; }
void sim_order(void* h, int* out) { Sim& s = *(Sim*)h; for (int64_t i = 0; i < s.n; ++i) out[i] = s.b.order[i]; }
int sim_leaf_of(void* h, int orig) { return ((Sim*)h)->b.pos_of[orig] / LEAF; }
// returns NN original index; counts[0] = box tests, counts[1] = point tests, counts[2] = loop steps
int sim_query(void* h, const double* q, int start_leaf, int reseed, int64_t* counts) {
  Sim& s = *(Sim*)h; const HostFrameBuild& t = s.b; const int L = t.n_leaf_pad;
  const float fx = (float)q[0], fy = (float)q[1], fz = (float)q[2];
  double best = g_cap; int bi = INT32_MAX; float bound = std::isinf(g_cap) ? INFINITY : (float)((std::sqrt(best) + 1e-6) * (std::sqrt(best) + 1e-6) * 1.000001);
  int64_t nb = 0, np = 0, ns = 0; g_trace_n = 0;
  auto tr = [&](unsigned char c) { if (g_trace && g_trace_n < g_trace_cap) g_trace[g_trace_n++] = c; };
  auto scan2 = [&](int leaf, int sub) {
    for (int j = 0; j < 2; ++j) {
      const int64_t pos = (int64_t)leaf * LEAF + 2 * sub + j; ++np;
      const float dx = fx - s.px[pos], dy = fy - s.py[pos], dz = fz - s.pz[pos];
      const float d32 = dx * dx + dy * dy + dz * dz;
      if (d32 <= bound) {
        const double ex = q[0] - (double)s.px[pos], ey = q[1] - (double)s.py[pos], ez = q[2] - (double)s.pz[pos];
        const double d = ex * ex + ey * ey + ez * ez;
        if (d < best || (d == best && s.pi[pos] < bi)) { best = d; bi = s.pi[pos]; const double r = std::sqrt(best) + 1e-6; bound = (float)(r * r * 1.000001); }
      }
    }
  };
  int leaf_node = -1; bool coarse_on = false;
  if (start_leaf >= 0) {
    leaf_node = L + start_leaf;
    for (int sub = 0; sub < LEAF / 2; ++sub) { scan2(start_leaf, sub); ++ns; tr(3); }
    const Box& b = t.boxes[leaf_node];
    const float ex = b.hi[0] - b.lo[0], ey = b.hi[1] - b.lo[1], ez = b.hi[2] - b.lo[2];
    if (reseed && bound > 16.f * (ex * ex + ey * ey + ez * ez)) start_leaf = -1;
  }
  if (start_leaf < 0) {
    int node = 1;
    while (node < (L >> g_coarse)) { const float l0 = lbn(s, 2 * node, fx, fy, fz), l1 = lbn(s, 2 * node + 1, fx, fy, fz); nb += 2; ++ns; tr(4); node = (l1 < l0) ? 2 * node + 1 : 2 * node; }
    if (g_coarse) { const int first = (node << g_coarse) - L; for (int lf = first; lf < first + (1 << g_coarse); ++lf) for (int sub = 0; sub < LEAF / 2; ++sub) { scan2(lf, sub); ++ns; } coarse_on = true; }
    else if (node != leaf_node) for (int sub = 0; sub < LEAF / 2; ++sub) { scan2(node - L, sub); ++ns; tr(5); }
    leaf_node = node;
  }
  std::vector<int> sn; std::vector<float> sl;
  const int cz = coarse_on ? g_coarse : 0; const int Lc = L >> cz;
  for (int l = t.depth - 1 - cz; l >= 0; --l) {
    const int sib = (leaf_node >> l) ^ 1;
    const float face = t.faces[sib]; uint32_t bits; std::memcpy(&bits, &face, 4); const int axis = bits & 3;
    const float qa = axis == 0 ? fx : (axis == 1 ? fy : fz);
    const float dpl = (sib & 1) ? face - qa : qa - face; ++counts[3];
    if (dpl > 0.f && dpl * dpl > bound) continue;
    const float lb = lbn(s, sib, fx, fy, fz); ++nb; if (lb <= bound) { sn.push_back(sib); sl.push_back(lb); } }
  ns += t.depth;
  int node = -1, sub = 0;
  while (true) {
    if (node < 0) { if (sn.empty()) break; const int nn = sn.back(); const float ll = sl.back(); sn.pop_back(); sl.pop_back(); if (ll > bound) continue; node = nn; sub = 0; }
    ++ns; tr(node >= Lc ? 2 : 1);
    if (node >= Lc) { const int first = (node << cz) - L; scan2(first + sub / (LEAF / 2), sub % (LEAF / 2)); if (++sub == (LEAF / 2) << cz) node = -1; }
    else {
      const int c0 = 2 * node; const float l0 = lbn(s, c0, fx, fy, fz), l1 = lbn(s, c0 + 1, fx, fy, fz); nb += 2;
      const bool f0 = l0 <= l1; const float ln = f0 ? l0 : l1, lf = f0 ? l1 : l0;
      if (ln <= bound) { if (lf <= bound) { sn.push_back(f0 ? c0 + 1 : c0); sl.push_back(lf); } node = f0 ? c0 : c0 + 1; sub = 0; } else node = -1;
    }
  }
  counts[0] += nb; counts[1] += np; counts[2] += ns;
  return bi;
}

// Packet walk of far.cuh (knn_far_kernel) for the nl <= 32 queries of one warp: each lane runs sim_query's prologue (start-leaf
// scan + stale-seed rule, or the greedy descent), then ONE depth-first walk from the root is shared by all lanes -- at an internal
// node every lane tests both children, a child is kept if any lane needs it, the one with the smaller lane minimum is visited
// first; a leaf is scanned by every lane; a popped entry is skipped when its smallest lane bound exceeds every lane's bound, a
// popped leaf is re-tested per lane first.  out[k] = NN of lane k.  counts (warp-steps, added): [0] prologue (slowest lane),
// [1] node steps of the walk (child pairs and popped-leaf re-tests), [2] leaf steps of the walk (LEAF/2 per leaf),
// [3] lane-steps of the walk in which the lane needed the node or leaf (its own bound admits it).
int sim_packet(void* h, const double* q, const int* start_leaf, int nl, int* out, int64_t* counts) {
  Sim& s = *(Sim*)h; const HostFrameBuild& t = s.b; const int L = t.n_leaf_pad;
  struct Lane { double q[3]; float f[3]; double best; int bi; float bound; };
  std::vector<Lane> ln(nl);
  auto scan2 = [&](Lane& a, int leaf, int sub) {
    for (int j = 0; j < 2; ++j) {
      const int64_t pos = (int64_t)leaf * LEAF + 2 * sub + j;
      const float dx = a.f[0] - s.px[pos], dy = a.f[1] - s.py[pos], dz = a.f[2] - s.pz[pos];
      if (dx * dx + dy * dy + dz * dz <= a.bound) {
        const double ex = a.q[0] - (double)s.px[pos], ey = a.q[1] - (double)s.py[pos], ez = a.q[2] - (double)s.pz[pos];
        const double d = ex * ex + ey * ey + ez * ez;
        if (d < a.best || (d == a.best && s.pi[pos] < a.bi)) { a.best = d; a.bi = s.pi[pos]; const double r = std::sqrt(a.best) + 1e-6; a.bound = (float)(r * r * 1.000001); }
      }
    }
  };
  auto lb = [&](const Lane& a, int nd) { return lbn(s, nd, a.f[0], a.f[1], a.f[2]); };
  int64_t pro = 0;
  for (int k = 0; k < nl; ++k) {
    Lane& a = ln[k];
    for (int c = 0; c < 3; ++c) { a.q[c] = q[3 * k + c]; a.f[c] = (float)a.q[c]; }
    a.best = INFINITY; a.bi = INT32_MAX; a.bound = INFINITY;
    int64_t st = 0; int sl = start_leaf[k], leaf_node = -1;
    if (sl >= 0) {
      leaf_node = L + sl;
      for (int sub = 0; sub < LEAF / 2; ++sub) scan2(a, sl, sub);
      st += LEAF / 2;
      const Box& b = t.boxes[leaf_node];
      const float ex = b.hi[0] - b.lo[0], ey = b.hi[1] - b.lo[1], ez = b.hi[2] - b.lo[2];
      if (a.bound > 16.f * (ex * ex + ey * ey + ez * ez)) sl = -1;
    }
    if (sl < 0) {
      int node = 1;
      while (node < L) { const float l0 = lb(a, 2 * node), l1 = lb(a, 2 * node + 1); node = (l1 < l0) ? 2 * node + 1 : 2 * node; ++st; }
      if (node != leaf_node) { for (int sub = 0; sub < LEAF / 2; ++sub) scan2(a, node - L, sub); st += LEAF / 2; }
    }
    pro = std::max(pro, st);
  }
  int64_t wn = 0, wl = 0, busy = 0;
  std::vector<std::pair<int, float>> stk;
  int node = 1;
  while (true) {
    if (node < 0) {
      while (!stk.empty()) {
        const int nd = stk.back().first; const float m = stk.back().second; stk.pop_back();
        float bmax = 0.f; for (const Lane& a : ln) bmax = std::fmax(bmax, a.bound);
        if (m > bmax) continue;
        if (nd >= L) { ++wn; bool any = false; for (const Lane& a : ln) any |= lb(a, nd) <= a.bound; if (!any) continue; }
        node = nd; break;
      }
      if (node < 0) break;
    }
    if (node >= L) {
      for (const Lane& a : ln) busy += (lb(a, node) <= a.bound) ? LEAF / 2 : 0;
      for (int sub = 0; sub < LEAF / 2; ++sub) for (Lane& a : ln) scan2(a, node - L, sub);
      wl += LEAF / 2; node = -1; continue;
    }
    ++wn;
    const int c0 = 2 * node;
    bool k0 = false, k1 = false; float m0 = INFINITY, m1 = INFINITY; int nb = 0;
    for (const Lane& a : ln) {
      const float l0 = lb(a, c0), l1 = lb(a, c0 + 1);
      if (l0 <= a.bound) { k0 = true; m0 = std::fmin(m0, l0); }
      if (l1 <= a.bound) { k1 = true; m1 = std::fmin(m1, l1); }
      nb += (l0 <= a.bound || l1 <= a.bound) ? 1 : 0;
    }
    busy += nb;
    if (k0 && k1) { const bool f0 = m0 <= m1; stk.push_back({f0 ? c0 + 1 : c0, f0 ? m1 : m0}); node = f0 ? c0 : c0 + 1; }
    else if (k0) node = c0;
    else if (k1) node = c0 + 1;
    else node = -1;
  }
  for (int k = 0; k < nl; ++k) out[k] = ln[k].bi;
  counts[0] += pro; counts[1] += wn; counts[2] += wl; counts[3] += busy;
  return 0;
}
}

// steady-state anatomy of one seeded query (development aid): after the start leaf's scan, which ancestor levels survive the
// split-plane pre-filter (bit l of *plane_mask), which of those also survive the box test (*box_mask), and the per-leaf
// "reach" table idea: the smallest level L* such that every level >= L* is pruned by the distance from the LEAF'S BOX to the
// split planes alone (no per-query work) given the query's reach r + e (returned in *lstar).
extern "C" int sim_anatomy(void* h, const double* q, int start_leaf, unsigned* plane_mask, unsigned* box_mask, int* lstar) {
  Sim& s = *(Sim*)h; const HostFrameBuild& t = s.b; const int L = t.n_leaf_pad;
  const float fx = (float)q[0], fy = (float)q[1], fz = (float)q[2];
  double best = INFINITY; int bi = -1;
  for (int j = 0; j < LEAF; ++j) {
    const int64_t pos = (int64_t)start_leaf * LEAF + j; if (pos >= s.n) break;
    const double ex = q[0] - (double)s.px[pos], ey = q[1] - (double)s.py[pos], ez = q[2] - (double)s.pz[pos];
    const double d = ex * ex + ey * ey + ez * ez; if (d < best) { best = d; bi = s.pi[pos]; }
  }
  const float bound = (float)((std::sqrt(best) + 1e-6) * (std::sqrt(best) + 1e-6) * 1.000001);
  const int leaf_node = L + start_leaf;
  const Box& lb = t.boxes[leaf_node];
  const float qa3[3] = {fx, fy, fz};
  float emax = 0.f; for (int a = 0; a < 3; ++a) emax = std::fmax(emax, std::fmax(lb.lo[a] - qa3[a], qa3[a] - lb.hi[a]));
  emax = std::fmax(emax, 0.f);
  *plane_mask = 0; *box_mask = 0; *lstar = 0;
  float mmin = INFINITY;   // running min over levels >= l of the leaf-box-to-plane gap, scanned from the top level down
  int ls = t.depth;
  for (int l = t.depth - 1; l >= 0; --l) {
    const int sib = (leaf_node >> l) ^ 1;
    const float face = t.faces[sib]; uint32_t bits; std::memcpy(&bits, &face, 4); const int axis = bits & 3;
    const float g = (sib & 1) ? face - lb.hi[axis] : lb.lo[axis] - face;   // gap between the leaf's box and the plane
    mmin = std::fmin(mmin, g);
    const float reach = mmin - emax;
    if (reach > 0.f && reach * reach > bound) ls = l;   // every level >= l is out of reach
    const float dpl = (sib & 1) ? face - qa3[axis] : qa3[axis] - face;
    if (dpl > 0.f && dpl * dpl > bound) continue;
    *plane_mask |= 1u << l;
    if (lb32(t.boxes[sib], fx, fy, fz) <= bound) *box_mask |= 1u << l;
  }
  // ls as computed is the smallest l for which the suffix [l, depth) is prunable by the table (suffix minima are monotone)
  *lstar = ls;
  return bi;
}
extern "C" void sim_leaf_boxes(void* h, float* out /*[L][6]*/) {
  Sim& s = *(Sim*)h; const int L = s.b.n_leaf_pad;
  for (int l = 0; l < L; ++l) for (int a = 0; a < 3; ++a) { out[6 * l + a] = s.b.boxes[L + l].lo[a]; out[6 * l + 3 + a] = s.b.boxes[L + l].hi[a]; }
}
extern "C" int sim_nleafpad(void* h) { return ((Sim*)h)->b.n_leaf_pad; }
