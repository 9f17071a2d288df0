// types.cuh -- device-visible data layout of the engine.
//
// HBM layout (DESIGN.md section 3).  Every frame keeps, resident for the life of the context:
//   pts_o / nor_o : points / normals in the caller's order, one 16-byte (float4) or 32-byte (double4)
//                   record each -> the LM kernel's coalesced src stream and its dst gathers;
//   pts_s         : the same points in left-balanced KD order ("tree order"), record.w = original index;
//   boxes         : implicit binary AABB tree over leaves of LEAF consecutive tree-order points,
//                   heap order (root = 1, children 2i, 2i+1, leaves at [n_leaf_pad, 2 n_leaf_pad)).
// float storage is used iff every coordinate of every frame is exactly fp32-representable
// (checked at upload); arithmetic is fp64 either way, so results do not depend on the choice.
#pragma once
#include <stdint.h>
#include <vector_types.h>

namespace mv {

constexpr int LEAF = 8;          // points per BVH leaf
constexpr int NUM_SMS = 132;     // H100 SXM: sizes the grid-stride launches and the LM streaming tile (mvicp.cu)
constexpr int KNN_TILE = 256;    // queries per CTA of the NN kernel
constexpr int EVAL_TILE = 2048;  // correspondence slots per CTA of the LM streaming kernel
constexpr int EVAL_THREADS = 256;
// per-edge block (doubles):  A = upper 6x6 of the point-to-plane normal matrix in the src frame's canonical tangent,
// b = rhs (both costs), cost, then the point-to-point moments sum w, sum w p, sum w q, sum w pp^T, sum w qq^T, sum w pq^T
constexpr int BLK_A = 0, BLK_B = 21, BLK_COST = 27, BLK_SW = 28, BLK_SWP = 29, BLK_SWQ = 32, BLK_SWPP = 35, BLK_SWQQ = 41,
              BLK_SWPQ = 47;
constexpr int NBLK_PLANE = 28;   // entries used by a point-to-plane-only solve
constexpr int NBLK = 56;         // stride of a block

struct Box { float lo[3]; float hi[3]; float pad[2]; };   // 32 B fp32 AABB; child pairs are 64-B contiguous

struct double4a { double x, y, z, w; };   // 32-byte record for the fp64 storage mode

struct FrameDev {
  const void* pts_o;     // float4* or double4a*: exact coordinates, caller's order
  const void* nor_o;     // may be null
  const float4* pn_o;    // fp32 storage with normals: {x y z -, nx ny nz -} per point, 32 B = one sector per LM gather (else null)
  const void* pts_s;     // exact coordinates in tree order, .w = original index (int bits / int64 bits)
  const float4* pts_sf;  // fp32 screening copy in tree order, .w = original index; == pts_s in the fp32 storage mode
  const Box* boxes;      // 2 * n_leaf_pad entries (entry 0 unused), fp32 AABBs rounded outward
  const float* faces;    // per node: one-sided bound along the parent's split axis, axis in the low 2 mantissa bits
  const int32_t* pos_of; // original index -> position in tree order (seed -> leaf)
  const int32_t* adj;    // per leaf 16 ints: reach, count, neighbouring leaves (adjacency.h); may be null
  int32_t n;             // points
  int32_t n_leaf_pad;    // power of two >= ceil(n / LEAF)
  int32_t depth;         // log2(n_leaf_pad)
  float absmax;          // max |coordinate| of the cloud (bounds the fp32 rounding of a difference)
};

struct EdgeDev {
  int32_t src, dst;
  int64_t off;           // offset of this edge's slot 0 in the flat per-query arrays
  int32_t n_src;
  int32_t owned;         // 1 if this rank processes the edge
};

// Per-edge constants of the query transform (frame.cpp:117-118,131,136), recomputed from the poses.
struct EdgeXf { double Rs[9], ts[3], Rinv[9], td[3]; };

struct Tile { int32_t edge; int32_t start; };   // work item: `count` slots of one edge from `start`

// ---- median select (select.cuh); the NN kernel's epilogue feeds its guessed variant (knn.cuh) ----
struct SelState {            // one per edge
  unsigned long long prefix; // bits decided so far (high part)
  unsigned long long rank;   // remaining rank inside the current prefix bucket
  unsigned long long count;  // inliers of the edge
};

constexpr int SEL_CAP = 4096;   // collected candidates per edge

// what the NN kernel's epilogue needs for the guessed select (all per edge)
struct SelGuess {
  const unsigned long long* win;  // [3E]: window [lo, hi) of keys around the previous median | log2 of its half-width
  unsigned int* total;            // += inliers
  unsigned int* below;            // += inliers whose key lies below the window
  unsigned long long* cand;       // [SEL_CAP] keys inside the window
  unsigned int* cand_n;
};

}  // namespace mv
