// far.cuh -- the NN search of knn.cuh with HYBRID ORIENTED node boxes, for the rounds in which the clouds are still far
// apart (a round without seeds and the first round that has them).  Same results as knn_kernel, bit for bit.
//
// A depth scan is a tilted, locally flat sheet: its axis-aligned boxes are as thick as the tilt makes them, and a query
// that is still millimetres off the surface has to open every box within sqrt(height x thickness) of its foot point.  Nodes
// of up to 64 points therefore get the box of their principal axes when that is clearly smaller (volume ratio < 0.5), all
// others keep the coordinate axes (KD siblings stay disjoint near the root).  From the second seeded round on the 32-byte
// AABB nodes of knn.cuh win (64-byte nodes cost more than the tighter boxes save once the seeds are good), hence a second
// node array and the switch in mvicp_correspond.  MVICP_FLAG_NO_OBB builds no such array: every round then runs knn_kernel.
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

// nn_search of knn.cuh with the oriented lower bound (the split-plane pre-filter and the stale-seed rule are unchanged)
template <bool F32, bool WW>
__device__ __forceinline__ void nn_search_obb(const FrameDev& fd, const ObbNode* __restrict__ ob, NNQuery& s, int start_leaf) {
  const int L = fd.n_leaf_pad;
  int leaf_node = -1;
  if (start_leaf >= 0) {
    leaf_node = L + start_leaf;
#pragma unroll
    for (int sub = 0; sub < LEAF / 2; ++sub) nn_leaf_step<F32, NNQuery>(fd, start_leaf, sub, s);
    const float4* b = reinterpret_cast<const float4*>(fd.boxes + leaf_node);
    const float4 u = __ldg(b), v = __ldg(b + 1);
    const float ex = u.w - u.x, ey = v.x - u.y, ez = v.y - u.z;
    if (s.bound32 > 16.0f * fmaf(ez, ez, fmaf(ey, ey, ex * ex))) start_leaf = -1;
  }
  if (start_leaf < 0) {
    int node = 1;
    while (node < L) {
      const int c0 = 2 * node;
      const float l0 = obb_lb32(ob, c0, s), l1 = obb_lb32(ob, c0 + 1, s);
      node = (l1 < l0) ? c0 + 1 : c0;
    }
    if (node != leaf_node) {
#pragma unroll
      for (int sub = 0; sub < LEAF / 2; ++sub) nn_leaf_step<F32, NNQuery>(fd, node - L, sub, s);
    }
    leaf_node = node;
  }
  int stk_n[NN_STACK]; float stk_lb[NN_STACK]; int sp = 0;
  for (int l = fd.depth - 1; l >= 0; --l) {
    const int sib = (leaf_node >> l) ^ 1;
    const float face = __ldg(fd.faces + sib);
    const int axis = __float_as_int(face) & 3;
    const float qa = axis == 0 ? s.fx : (axis == 1 ? s.fy : s.fz);
    const float dpl = (sib & 1) ? face - qa : qa - face;
    if (dpl > 0.f && dpl * dpl > s.bound32) continue;
    const float lb = obb_lb32(ob, sib, s);
    if (lb <= s.bound32) { stk_n[sp] = sib; stk_lb[sp] = lb; ++sp; }
  }
  nn_drain<F32, WW, NNQuery>(fd, s, stk_n, stk_lb, sp, [&](int nd) { return obb_lb32(ob, nd, s); });
}

template <bool F32, bool WW>
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
  const FrameDev fs = frames[e.src];
  const FrameDev fd = frames[e.dst];
  const ObbNode* ob = obbs[e.dst].nodes;
  const int ks = t.start + threadIdx.x;
  if (ks >= e.n_src) return;
  double px, py, pz; int orig;
  Rec<F32>::load(fs.pts_s, ks, px, py, pz, orig);
  // query transform, the operation sequence of knn_kernel (frame.cpp:117-118,131,136)
  const double gx = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(sx.Rs[0], px), __dmul_rn(sx.Rs[1], py)), __dmul_rn(sx.Rs[2], pz)), sx.ts[0]);
  const double gy = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(sx.Rs[3], px), __dmul_rn(sx.Rs[4], py)), __dmul_rn(sx.Rs[5], pz)), sx.ts[1]);
  const double gz = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(sx.Rs[6], px), __dmul_rn(sx.Rs[7], py)), __dmul_rn(sx.Rs[8], pz)), sx.ts[2]);
  const double ex = __dsub_rn(gx, sx.td[0]), ey = __dsub_rn(gy, sx.td[1]), ez = __dsub_rn(gz, sx.td[2]);
  const double qx = __dadd_rn(__dadd_rn(__dmul_rn(sx.Rinv[0], ex), __dmul_rn(sx.Rinv[1], ey)), __dmul_rn(sx.Rinv[2], ez));
  const double qy = __dadd_rn(__dadd_rn(__dmul_rn(sx.Rinv[3], ex), __dmul_rn(sx.Rinv[4], ey)), __dmul_rn(sx.Rinv[5], ez));
  const double qz = __dadd_rn(__dadd_rn(__dmul_rn(sx.Rinv[6], ex), __dmul_rn(sx.Rinv[7], ey)), __dmul_rn(sx.Rinv[8], ez));
  NNQuery nq; nn_query_init(nq, qx, qy, qz, fd.absmax);
  int start_leaf = -1;
  if (seed) {
    const int sd = seed[e.off + orig];
    const int si = sd >= 0 ? sd : ~sd;
    if (si >= 0 && si < fd.n) start_leaf = __ldg(fd.pos_of + si) / LEAF;
  }
  nn_search_obb<F32, WW>(fd, ob, nq, start_leaf);
  const double best = nq.best; const int bi = nq.bi;
  const bool inlier = best <= thresh;   // thresh = cutoff_d2max (knn.cuh)
  corr[e.off + orig] = inlier ? bi : ~bi;
  d2out[e.off + orig] = best;
}

}  // namespace mv
