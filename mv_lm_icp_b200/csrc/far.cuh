// far.cuh -- the NN search of knn.cuh with HYBRID ORIENTED node boxes, for the rounds in which the clouds are still far
// apart (a round without seeds and the first round that has them).  Same results as knn_kernel, bit for bit.
//
// A depth scan is a tilted, locally flat sheet: its axis-aligned boxes are as thick as the tilt makes them, and a query
// that is still millimetres off the surface has to open every box within sqrt(height x thickness) of its foot point.  Nodes
// of up to 64 points therefore get the box of their principal axes when that is clearly smaller (volume ratio < 0.5), all
// others keep the coordinate axes (KD siblings stay disjoint near the root).  From the second seeded round on the 32-byte
// AABB nodes of knn.cuh win (64-byte nodes cost more than the tighter boxes save once the seeds are good), hence a second
// node array and the switch in mvicp_correspond.  MVICP_FLAG_NO_OBB builds no such array: every round then runs knn_kernel.
// Above the PCA level (nodes of more than OBB_PCA_LEAVES leaves) an oriented box is always the box of the coordinate axes, and
// the 32-byte fp32 AABB of knn.cuh bounds the same points as tightly (up to rounding) in half the bytes: the search reads it there.
#pragma once
#include "knn.cuh"

namespace mv {

// every point p of the node satisfies |a_i . (p - c)| <= e_i (i = 0..2) for the stored fp32 a_i, c (checked in fp64 at
// build time, tree_build.h:build_obb); empty nodes carry e = -inf => lower bound +inf
struct ObbNode { float c[3]; float e0; float a0[3]; float e1; float a1[3]; float e2; float a2[3]; float pad; };
struct ObbDev { const ObbNode* nodes; };   // per frame, heap order like FrameDev::boxes

__device__ __forceinline__ float obb_lb32(const ObbNode* __restrict__ nodes, int node, const NNQuery& s) {
  const float4* b = reinterpret_cast<const float4*>(nodes + node);
  const float4 q0 = __ldg(b), q1 = __ldg(b + 1), q2 = __ldg(b + 2), q3 = __ldg(b + 3);   // (c, e0) (a0, e1) (a1, e2) (a2, -)
  const float dx = s.fx - q0.x, dy = s.fy - q0.y, dz = s.fz - q0.z;
  const float p0 = fmaf(q1.z, dz, fmaf(q1.y, dy, q1.x * dx));
  const float p1 = fmaf(q2.z, dz, fmaf(q2.y, dy, q2.x * dx));
  const float p2 = fmaf(q3.z, dz, fmaf(q3.y, dy, q3.x * dx));
  const float g0 = fmaxf(fabsf(p0) - q0.w, 0.f), g1 = fmaxf(fabsf(p1) - q1.w, 0.f), g2 = fmaxf(fabsf(p2) - q2.w, 0.f);
  return fmaf(g2, g2, fmaf(g1, g1, g0 * g0));
}

// Far rounds as a PACKET walk: the 32 queries of a warp (neighbours in the src tree order) share one depth-first walk of the dst
// tree.  Each lane first runs its own prologue (start-leaf scan + stale-seed rule, or the greedy descent) for a first bound; then at
// every step all lanes look at the same node or leaf -- one broadcast load per warp.  A child is kept if any lane's bound admits it
// and the one with the smaller lower bound (over those lanes) is visited first; a popped entry is skipped when its lower bound
// exceeds every lane's bound, a popped leaf is first re-tested per lane.  Every node that can hold a point within a lane's bound is
// visited for that lane, and the arg-min with the lowest-index tie rule does not depend on the order in which candidates are met:
// same results as nn_search, bit for bit.  The stack holds at most one entry per level of the current path (<= depth < 32): entry i
// lives in a register of lane i.
template <bool F32>
__global__ void __launch_bounds__(KNN_TILE)
knn_far_kernel(const FrameDev* __restrict__ frames, const EdgeDev* __restrict__ edges, const EdgeXf* __restrict__ xfs,
               const Tile* __restrict__ tiles, int32_t* corr /* aliases seed */, double* __restrict__ d2out,
               const int32_t* seed, double thresh, const ObbDev* __restrict__ obbs) {
  const Tile t = tiles[blockIdx.x];
  const EdgeDev e = edges[t.edge];
  __shared__ EdgeXf sx;
  {
    const double* g = reinterpret_cast<const double*>(xfs + t.edge);
    double* s = reinterpret_cast<double*>(&sx);
    for (int i = threadIdx.x; i < (int)(sizeof(EdgeXf) / sizeof(double)); i += blockDim.x) s[i] = g[i];
  }
  __syncthreads();
  if (t.start + (int)(threadIdx.x & ~31u) >= e.n_src) return;   // whole warp past the edge's end; a partial warp stays whole for the votes
  const FrameDev fs = frames[e.src];
  const FrameDev fd = frames[e.dst];
  const ObbNode* ob = obbs[e.dst].nodes;
  const int L = fd.n_leaf_pad;
  const int pca_first = L / OBB_PCA_LEAVES;   // first node that may hold principal axes
  const int ks = t.start + threadIdx.x;
  const bool act = ks < e.n_src;
  NNQuery nq;
  const auto lb_of = [&](int nd) { return nd < pca_first ? box_lb32(fd.boxes, nd, nq) : obb_lb32(ob, nd, nq); };
  int orig = 0;
  if (act) {
    double px, py, pz;
    Rec<F32>::load(fs.pts_s, ks, px, py, pz, orig);
    // query transform, the operation sequence of knn_kernel (frame.cpp:117-118,131,136)
    const double gx = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(sx.Rs[0], px), __dmul_rn(sx.Rs[1], py)), __dmul_rn(sx.Rs[2], pz)), sx.ts[0]);
    const double gy = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(sx.Rs[3], px), __dmul_rn(sx.Rs[4], py)), __dmul_rn(sx.Rs[5], pz)), sx.ts[1]);
    const double gz = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(sx.Rs[6], px), __dmul_rn(sx.Rs[7], py)), __dmul_rn(sx.Rs[8], pz)), sx.ts[2]);
    const double ex = __dsub_rn(gx, sx.td[0]), ey = __dsub_rn(gy, sx.td[1]), ez = __dsub_rn(gz, sx.td[2]);
    const double qx = __dadd_rn(__dadd_rn(__dmul_rn(sx.Rinv[0], ex), __dmul_rn(sx.Rinv[1], ey)), __dmul_rn(sx.Rinv[2], ez));
    const double qy = __dadd_rn(__dadd_rn(__dmul_rn(sx.Rinv[3], ex), __dmul_rn(sx.Rinv[4], ey)), __dmul_rn(sx.Rinv[5], ez));
    const double qz = __dadd_rn(__dadd_rn(__dmul_rn(sx.Rinv[6], ex), __dmul_rn(sx.Rinv[7], ey)), __dmul_rn(sx.Rinv[8], ez));
    nn_query_init(nq, qx, qy, qz, fd.absmax);
    int start_leaf = -1, leaf_node = -1;
    if (seed) {
      const int sd = seed[e.off + orig];
      const int si = sd >= 0 ? sd : ~sd;
      if (si >= 0 && si < fd.n) start_leaf = __ldg(fd.pos_of + si) / LEAF;
    }
    if (start_leaf >= 0) {
      leaf_node = L + start_leaf;
#pragma unroll
      for (int sub = 0; sub < LEAF / 2; ++sub) nn_leaf_step<F32, NNQuery>(fd, start_leaf, sub, nq);
      const float4* b = reinterpret_cast<const float4*>(fd.boxes + leaf_node);
      const float4 u = __ldg(b), v = __ldg(b + 1);
      const float bx = u.w - u.x, by = v.x - u.y, bz = v.y - u.z;
      if (nq.bound32 > 16.0f * fmaf(bz, bz, fmaf(by, by, bx * bx))) start_leaf = -1;
    }
    if (start_leaf < 0) {
      int node = 1;
      while (node < L) {
        const int c0 = 2 * node;
        const float l0 = lb_of(c0), l1 = lb_of(c0 + 1);
        node = (l1 < l0) ? c0 + 1 : c0;
      }
      if (node != leaf_node) {
#pragma unroll
        for (int sub = 0; sub < LEAF / 2; ++sub) nn_leaf_step<F32, NNQuery>(fd, node - L, sub, nq);
      }
    }
  } else {
    nn_query_init(nq, 0.0, 0.0, 0.0, fd.absmax);
    nq.bound32 = -1.0f;   // admits nothing: the lane only takes part in the votes
  }
  const unsigned full = 0xffffffffu, inf_bits = 0x7f800000u;
  const int lane = threadIdx.x & 31;
  int my_n = 0; float my_lb = 0.f;   // stack entry `lane`
  int sp = 0, node = 1;
  while (true) {
    if (node < L) {
      const int c0 = 2 * node;
      const float l0 = lb_of(c0), l1 = lb_of(c0 + 1);
      const bool k0 = l0 <= nq.bound32, k1 = l1 <= nq.bound32;
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
#pragma unroll
      for (int sub = 0; sub < LEAF / 2; ++sub) nn_leaf_step<F32, NNQuery>(fd, node - L, sub, nq);
    }
    node = -1;
    while (sp > 0) {
      --sp;
      const int nd = __shfl_sync(full, my_n, sp);
      const float m = __shfl_sync(full, my_lb, sp);
      if (m > __uint_as_float(__reduce_max_sync(full, __float_as_uint(fmaxf(nq.bound32, 0.f))))) continue;
      if (nd >= L && !__ballot_sync(full, lb_of(nd) <= nq.bound32)) continue;
      node = nd;
      break;
    }
    if (node < 0) break;
  }
  if (!act) return;
  const double best = nq.best; const int bi = nq.bi;
  const bool inlier = best <= thresh;   // thresh = cutoff_d2max (knn.cuh)
  corr[e.off + orig] = inlier ? bi : ~bi;
  d2out[e.off + orig] = best;
}

}  // namespace mv
