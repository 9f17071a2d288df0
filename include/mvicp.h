/* mvicp.h -- C ABI of the H100-native multiview LM-ICP engine (libmvicp.so).
 *
 * The reference (adrelino/mv-lm-icp) has no FFI layer: its hot path is a set of C++ signatures on
 * Eigen types called from two drivers.  Each entry point below names the reference interface it
 * replaces (paths relative to the reference tree).  Plain pointers and sizes only; every call
 * returns 0 on success or an MVICP_ERR_* code, with text in mvicp_last_error().
 *
 * Data conventions (bit-compatible with the reference containers, include/frame.h:18-46):
 *   points / normals : N x 3 doubles, 24-byte stride  == std::vector<Eigen::Vector3d>::data()
 *   pose             : double[16], 4x4 column-major   == Eigen::Isometry3d::data()
 *   correspondence   : (int32 first = src index, int32 second = dst index, double dist)
 *   edge weight      : float (OutgoingEdge::weight)
 * Threading: one context = one host thread at a time (the reference is single-threaded).
 * One process per GPU; multi-GPU runs shard the edges (frame -> neighbour query sets) across processes (mvicp_comm_init).
 */
#ifndef MVICP_H
#define MVICP_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct mvicp_ctx mvicp_ctx;

enum { MVICP_OK = 0, MVICP_ERR_INVALID = 1, MVICP_ERR_CUDA = 2, MVICP_ERR_NCCL = 3, MVICP_ERR_STATE = 4,
       MVICP_ERR_NONRIGID = 5 /* internal guard only: non-rigid poses are supported */, MVICP_ERR_NOT_OWNER = 6, MVICP_ERR_EMPTY = 7 };

/* SE(3) parameterisations (main_multiview.cpp:158-164 dispatch; layouts SURVEY 8(b)) */
enum { MVICP_PARAM_AA = 0,   /* ceresOptimizer_ceresAngleAxis : [wx wy wz tx ty tz]            */
       MVICP_PARAM_QUAT = 1, /* ceresOptimizer (Eigen quaternion): [qx qy qz qw] + [tx ty tz]  */
       MVICP_PARAM_SE3 = 2   /* ceresOptimizer_sophusSE3      : [qx qy qz qw tx ty tz]         */ };
/* cost: FLAGS_pointToPlane (main_multiview.cpp:39); MIXED = both blocks per correspondence   */
enum { MVICP_COST_P2P = 0, MVICP_COST_P2PLANE = 1, MVICP_COST_MIXED = 2 };

typedef struct {
  int32_t device;       /* CUDA device ordinal                                                */
  int32_t flags;        /* MVICP_FLAG_*                                                       */
  void*   stream;       /* cudaStream_t to run on (NULL: the context creates its own)         */
} mvicp_config;
enum { MVICP_FLAG_NO_CERT = 128,         /* NN search: never keep a match on the strength of the previous round's certificate (csrc/knn.cuh,
                                        CERT): every query of every round is searched */
       MVICP_FLAG_NO_SELECT_GUESS = 64, /* median select: always the three histogram passes, never the guess checked by the NN kernel's epilogue
                                        (csrc/select.cuh) in rounds that follow a one-iteration solve */
       MVICP_FLAG_STEP_LOOP = 32, /* NN search: round 1's single loop of uniform steps instead of the while-while loop (csrc/knn.cuh
                                      nn_drain); same matches, for A/B measurements */
       MVICP_FLAG_NO_ADJ = 8,     /* NN search: do not use the per-leaf neighbour lists (csrc/adjacency.h) that let a seeded query inside its
                                      start leaf's reach skip the tree walk; same matches, for A/B measurements */
       MVICP_FLAG_HOST_BUILD = 4,  /* build the per-frame search trees on the host (csrc/tree_build.h) instead of on the device
                                      (csrc/tree_gpu.cuh); same matches, for A/B measurements */
       MVICP_FLAG_NO_SEED = 1,     /* do not seed the NN search with the previous round's match */
       MVICP_FLAG_NCCL_ONLY = 2,   /* sharded LM: exchange pair matrices with ncclAllReduce instead of peer-memory stores */
       MVICP_FLAG_NO_OBB = 16      /* do not build the second node array of hybrid oriented boxes that the far rounds (no seeds yet /
                                      first seeded round) search (csrc/far.cuh); same results, for A/B measurements */ };

/* Ceres options that the reference sets (icp-ceres.cpp:66-89) or leaves at Ceres defaults. */
typedef struct {
  int32_t max_num_iterations;               /* 50  icp-ceres.cpp:81 */
  int32_t max_num_consecutive_invalid_steps;/* 5   */
  int32_t jacobi_scaling;                   /* 1   */
  int32_t reserved;
  double initial_trust_region_radius;       /* 1e4 */
  double max_trust_region_radius;           /* 1e16 */
  double min_trust_region_radius;           /* 1e-32 */
  double min_relative_decrease;             /* 1e-3 */
  double min_lm_diagonal;                   /* 1e-6 */
  double max_lm_diagonal;                   /* 1e32 */
  double function_tolerance;                /* 1e-6 */
  double gradient_tolerance;                /* 1e-10 */
  double parameter_tolerance;               /* 1e-8 */
} mvicp_lm_options;

enum { MVICP_TERM_FUNCTION_TOLERANCE = 0, MVICP_TERM_GRADIENT_TOLERANCE = 1, MVICP_TERM_PARAMETER_TOLERANCE = 2,
       MVICP_TERM_MAX_ITERATIONS = 3, MVICP_TERM_MIN_RADIUS = 4, MVICP_TERM_INVALID_STEPS = 5, MVICP_TERM_EVAL_FAILURE = 6 };

typedef struct {                  /* what ceres::Solver::Summary::FullReport() would tell (icp-ceres.cpp:94) */
  int32_t termination;            /* MVICP_TERM_* */
  int32_t num_iterations;         /* step attempts */
  int32_t num_successful_steps;
  int32_t num_evaluations;        /* streaming passes over the correspondences (residual + Jacobian blocks) */
  int32_t num_linear_solves;
  int32_t reserved;
  double initial_cost, final_cost;
} mvicp_lm_summary;

typedef struct {                  /* device-side timings of the last mvicp_correspond / mvicp_optimize call */
  float  knn_ms;                  /* nearest-neighbour kernel(s)                     */
  float  select_ms;               /* inlier count + exact median (radix select)      */
  float  lm_eval_ms;              /* sum over residual/Jacobian streaming kernels    */
  float  lm_other_ms;             /* reductions, collectives, Cholesky / LM step     */
  float  correspond_ms, optimize_ms;
  int64_t kernel_launches;        /* kernels of this library launched since mvicp_create */
  int64_t queries;                /* NN queries answered by the last correspond      */
  int64_t correspondences;        /* inliers after the cutoff, all local edges       */
  int64_t select_guess_rounds;    /* mvicp_correspond calls whose median select was the guess checked by the NN kernel (csrc/select.cuh) */
  int64_t select_guess_misses;    /* (edge, round) pairs in which that guess missed and the edge was redone from scratch */
  int64_t cert_rounds;            /* mvicp_correspond calls that kept certified matches (csrc/knn.cuh, CERT) */
  int64_t cert_reused;            /* queries answered that way, all local edges, since mvicp_create */
} mvicp_stats;

void mvicp_default_lm_options(mvicp_lm_options* o);
const char* mvicp_last_error(void);

int  mvicp_create(const mvicp_config* cfg, mvicp_ctx** out);
void mvicp_destroy(mvicp_ctx* ctx);

/* Frame::pts / Frame::nor of every frame (include/frame.h:38-39). Uploaded once; clouds are immutable
 * in the reference after load.  Builds the per-frame search structure that replaces the lazily built
 * nanoflann index (src/internal/frame.cpp:188-193).  nor_xyz[i] may be NULL (point-to-point only). */
int mvicp_set_frames(mvicp_ctx* ctx, int32_t n_frames, const double* const* pts_xyz, const double* const* nor_xyz,
                     const int64_t* n_pts);

/* Frame::pose and Frame::fixed (include/frame.h:41,43). fixed may be NULL; frame 0 is always treated as
 * fixed by mvicp_optimize, as every ceresOptimizer* does (icp-ceres.cpp:242-244,342-344,417-419). */
int mvicp_set_poses(mvicp_ctx* ctx, const double* poses16, const uint8_t* fixed);
int mvicp_get_poses(mvicp_ctx* ctx, double* poses16);

/* Frame::neighbours[*].neighbourIdx for all frames: E directed edges src -> dst, in the order
 * (src ascending, then the frame's neighbour order) that the reference iterates (frame.cpp:107). */
int mvicp_set_graph(mvicp_ctx* ctx, int32_t n_edges, const int32_t* src, const int32_t* dst);
/* Frame::computePoseNeighboursKnn for every frame (frame.cpp:67-89, main_multiview.cpp:104-117): builds the
 * graph from the current poses, then behaves as if mvicp_set_graph had been called. */
int mvicp_pose_graph_knn(mvicp_ctx* ctx, int32_t knn);
int mvicp_get_graph(mvicp_ctx* ctx, int32_t* n_edges, int32_t* src /*nullable*/, int32_t* dst /*nullable*/);

/* ApproachComponents::computeClosestPoints == Frame::computeClosestPointsToNeighbours for every frame
 * (main_multiview.cpp:119-127, frame.cpp:91-185): all edges in one launch. thresh as the reference's float. */
int mvicp_correspond(mvicp_ctx* ctx, float thresh);

/* OutgoingEdge::{correspondances, weight} of edge e (include/frame.h:24-29), ordered by ascending src index.
 * Pass NULL arrays to query only count/weight. Arrays must hold n_pts[src] entries. */
int mvicp_get_edge(mvicp_ctx* ctx, int32_t e, int32_t* first, int32_t* second, double* dist, int64_t* count,
                   float* weight);
/* Every edge at once, for a caller that materialises OutgoingEdge::correspondances (the viewer draws them, Visualize.cpp:470-479):
 * edge e's inliers are out_records[offsets[e] .. offsets[e+1]) as the reference's own 16-byte records
 * struct Correspondance {int first; int second; double dist;} (include/frame.h:18-22), ascending src index (frame.cpp:156-160);
 * weights[e] = OutgoingEdge::weight.  offsets has n_edges + 1 entries; out_records may be NULL (counts and weights only) and
 * otherwise holds `capacity` records (sum of the src cloud sizes always suffices).  Built on the device, one copy back. */
int mvicp_get_all_edges(mvicp_ctx* ctx, void* out_records, int64_t capacity, int64_t* offsets, float* weights /*nullable*/);
/* Page-locked host memory for the arrays a caller hands to mvicp_get_all_edges / mvicp_get_edge / mvicp_get_nn: copies into it run at
 * the link's speed instead of through the driver's staging buffer (config 3: 121 MB of records per round).  Any host pointer works;
 * this is an allocation helper, not a requirement. */
int mvicp_host_alloc(size_t bytes, void** out);
int mvicp_host_free(void* p);
/* Raw nearest neighbour of every src point of edge e (before the cutoff): index + squared distance, i.e. what
 * Frame::getClosestPoint returns per query (frame.cpp:187-206). */
int mvicp_get_nn(mvicp_ctx* ctx, int32_t e, int32_t* nn_idx, double* nn_d2);
/* Overwrite edge e's correspondences / weight (lets a caller run the LM step on its own matches, and is how
 * the pairwise solvers feed identity correspondences). */
int mvicp_set_edge(mvicp_ctx* ctx, int32_t e, const int32_t* first, const int32_t* second, int64_t count,
                   float weight);

/* Frame::getClosestPoint (frame.cpp:187-206): query in the frame's local coordinates; returns index and d^2. */
int mvicp_closest_point(mvicp_ctx* ctx, int32_t frame, const double query[3], int64_t* idx, double* d2);

/* ICP_Ceres::ceresOptimizer / _ceresAngleAxis / _sophusSE3 (include/icp-ceres.h:40-42, icp-ceres.cpp:220-475):
 * LM over all absolute poses with the current correspondences; writes every frame's pose back. */
int mvicp_optimize(mvicp_ctx* ctx, int32_t param, int32_t cost, int32_t robust, const mvicp_lm_options* opt,
                   mvicp_lm_summary* summary);

/* One pass of the loop body main_multiview.cpp:150-169 (correspond + optimize). */
int mvicp_icp_round(mvicp_ctx* ctx, float thresh, int32_t param, int32_t cost, int32_t robust,
                    const mvicp_lm_options* opt, mvicp_lm_summary* summary);

/* ICP_Ceres::pointToPoint_* / pointToPlane_* (include/icp-ceres.h:30-36, icp-ceres.cpp:137-218,525-565): one pose
 * from identity with 1:1 correspondences src[i] <-> dst[i]; nor = dst normals (NULL for point-to-point). */
int mvicp_pairwise(const mvicp_config* cfg, int32_t param, int32_t cost, const double* src_xyz, const double* dst_xyz,
                   const double* nor_xyz, int64_t n, const mvicp_lm_options* opt, double* pose16_out,
                   mvicp_lm_summary* summary);

/* ICP_Closedform::pointToPoint (cost = MVICP_COST_P2P: SVD of the centred cross-covariance, with the reference's
 * `R.col(2) *= -1` for det < 0) / pointToPlane (MVICP_COST_P2PLANE: small-angle 6x6 normal equations, LDL^T, Rx Ry Rz)
 * (src/internal/icp-closedform.cpp:9-54): the comparison baseline of main_pairwise.cpp:73,95 and a one-shot initialiser. */
int mvicp_pairwise_closed(const mvicp_config* cfg, int32_t cost, const double* src_xyz, const double* dst_xyz, const double* nor_xyz,
                          int64_t n, double* pose16_out);

/* Frame::recomputeNormals for every frame (frame.cpp:244-255; default-on in main_multiview.cpp:49,68): k nearest
 * neighbours of each point in its own cloud (the point included; the reference uses k = 10) + pointSetPCA
 * (common.h:331-346).  The new normals replace the uploaded ones for mvicp_optimize; mvicp_get_normals copies them back
 * (N x 3 doubles) so that the caller can store them in Frame::nor. */
int mvicp_recompute_normals(mvicp_ctx* ctx, int32_t k);
int mvicp_get_normals(mvicp_ctx* ctx, int32_t frame, double* nor_xyz, float* elapsed_ms /*nullable: device time of the recompute*/);
/* Frame::getNeighbours(i, k) for every point i of one frame (frame.cpp:208-242): nn_idx[i*k + j], ascending distance. */
int mvicp_knn_self(mvicp_ctx* ctx, int32_t frame, int32_t k, int32_t* nn_idx);

/* ---- multi-GPU: one process per GPU; the edges with a free src frame, in graph order, are cut into world_size
 * contiguous runs of equal query count (every rank holds all clouds and ends every call with identical poses) ---- */
int mvicp_nccl_unique_id(void* out128);   /* rank 0 creates, the launcher broadcasts the 128 bytes */
int mvicp_comm_init(mvicp_ctx* ctx, const void* id128, int32_t rank, int32_t world_size);

/* ---- introspection ------------------------------------------------------------------------------------- */
int mvicp_get_stats(mvicp_ctx* ctx, mvicp_stats* out);
int mvicp_get_stream(mvicp_ctx* ctx, void** stream);
int mvicp_sync(mvicp_ctx* ctx);
int mvicp_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* MVICP_H */
