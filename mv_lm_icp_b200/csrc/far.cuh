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

// Far rounds as a PACKET walk (nn_packet_walk, knn.cuh): the 32 queries of a warp (neighbours in the src tree order) share one
// depth-first walk of the dst tree.  Each lane first runs its own prologue (start-leaf scan + stale-seed rule, or the greedy
// descent) for a first bound; the walk then tests the hybrid boxes below the PCA level and the AABBs above it.
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
  int orig = 0, skip0 = -1, skip1 = -1;
  if (act) {
    double px, py, pz, qx, qy, qz;
    Rec<F32>::load(fs.pts_s, ks, px, py, pz, orig);
    edge_query(sx, px, py, pz, qx, qy, qz);
    nn_query_init(nq, qx, qy, qz, fd.absmax);
    int start_leaf = -1;
    if (seed) {
      const int sd = seed[e.off + orig];
      const int si = sd >= 0 ? sd : ~sd;
      if (si >= 0 && si < fd.n) start_leaf = __ldg(fd.pos_of + si) / LEAF;
    }
    if (start_leaf >= 0) {
      skip0 = L + start_leaf;
#pragma unroll
      for (int sub = 0; sub < LEAF / 2; ++sub) nn_leaf_step<F32, NNQuery>(fd, start_leaf, sub, nq);
      const float4* b = reinterpret_cast<const float4*>(fd.boxes + skip0);
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
      if (node != skip0) {
#pragma unroll
        for (int sub = 0; sub < LEAF / 2; ++sub) nn_leaf_step<F32, NNQuery>(fd, node - L, sub, nq);
      }
      skip1 = node;
    }
  } else {
    nn_query_init(nq, 0.0, 0.0, 0.0, fd.absmax);
  }
  nn_packet_walk<F32, NNQuery>(fd, nq, act, skip0, skip1, lb_of);
  if (!act) return;
  const double best = nq.best; const int bi = nq.bi;
  const bool inlier = best <= thresh;   // thresh = cutoff_d2max (knn.cuh)
  corr[e.off + orig] = inlier ? bi : ~bi;
  d2out[e.off + orig] = best;
}

}  // namespace mv
