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
       MVICP_FLAG_STEP_LOOP = 32, /* NN search, rounds after the far ones: every query searched by its own lane (csrc/knn.cuh nn_search, the
                                      single loop of uniform steps of nn_drain) instead of the warp's shared packet walk for the queries the
                                      neighbour lists do not settle (nn_search_packet); no certificates, no guessed select; same matches, the
                                      reference for tests and A/B measurements */
       MVICP_FLAG_NO_ADJ = 8,     /* NN search: do not use the per-leaf neighbour lists (csrc/adjacency.h) that let a seeded query inside its
                                      start leaf's reach skip the tree walk; same matches, for A/B measurements */
       MVICP_FLAG_HOST_BUILD = 4,  /* build the per-frame search trees on the host (csrc/tree_build.h) instead of on the device
                                      (csrc/tree_gpu.cuh); same matches, for A/B measurements */
       MVICP_FLAG_NO_SEED = 1,     /* do not seed the NN search with the previous round's match */
       MVICP_FLAG_NCCL_ONLY = 2,   /* sharded LM: exchange pair matrices with ncclAllReduce instead of peer-memory stores */
       MVICP_FLAG_NO_OBB = 16      /* do not build the second node array of hybrid oriented boxes that the far rounds (no seeds yet /
                                      first seeded round) search (csrc/far.cuh); same results, for A/B measurements */ };

/* Ceres options that the reference sets (icp-ceres.cpp:66-89) or leaves at Ceres defaults.
 * Valid options (the rules Ceres' Solver::Options::IsValid applies to a trust-region LM solve); mvicp_optimize,
 * mvicp_optimize_components, mvicp_icp_round and mvicp_pairwise return MVICP_ERR_INVALID for anything else, before they
 * change any state (poses, fixed flags, correspondences).  A NaN breaks every rule it takes part in.
 *   max_num_iterations >= 0, max_num_consecutive_invalid_steps >= 0  (0 iterations: evaluate the start point only)
 *   function_tolerance, gradient_tolerance, parameter_tolerance >= 0
 *   initial_, max_ and min_trust_region_radius > 0, min <= initial <= max
 *   min_relative_decrease >= 0
 *   min_lm_diagonal >= 0, max_lm_diagonal >= 0, min_lm_diagonal <= max_lm_diagonal
 * jacobi_scaling is a flag (0: no column scaling). */
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

/* Connected components of the current graph: the undirected graph the edges induce over all frames (a frame without edges is
 * a component of its own), numbered in ascending order of their lowest frame.  *n_components, and component_of_frame[M]
 * (nullable). */
int mvicp_get_components(mvicp_ctx* ctx, int32_t* n_components, int32_t* component_of_frame);
/* One independent LM solve per component, all in one pipelined loop: a batch of unrelated registrations in one context.  The
 * lowest frame of every component is fixed (and stays fixed, as frame 0 does after mvicp_optimize; user-set flags are kept).
 * Each component is solved exactly as mvicp_optimize would solve it in a fresh context holding only that component (its frames
 * in ascending order, its edges in graph order, the same fixed flags and options): its own trust region, counters,
 * termination and costs; on a connected graph the result equals mvicp_optimize's bit for bit.  Shared by the batch: the
 * streaming tile length (from all active correspondence slots), the unit / general eval path (general if any pose is not
 * rigid) and the storage mode.  Every frame's pose is written back.  summaries (nullable): n_components entries; a component
 * without a free frame gets mvicp_optimize's summary for a problem without unknowns.  Sharded context: MVICP_ERR_STATE. */
int mvicp_optimize_components(mvicp_ctx* ctx, int32_t param, int32_t cost, int32_t robust, const mvicp_lm_options* opt,
                              mvicp_lm_summary* summaries);

/* Pose covariances of the LM problem (ceres::Covariance, DESIGN.md section 6j): C = (J^T J)^-1 at the CURRENT poses, for the
 * problem mvicp_optimize(param, cost, robust) would solve now -- the current correspondences and edge weights, frame 0 and every
 * flagged frame fixed, the edges of fixed src frames inactive, the unit or general eval path chosen as the solve chooses it.
 * J^T J is the matrix of the solve's first evaluation, with the loss applied as Ceres applies it (apply_loss_function = true;
 * SoftL1: rows scaled by sqrt(rho')).  After mvicp_optimize_components the lowest frame of every component is flagged, so the
 * call covers such a batch as it stands.
 *   cov36[36 k .. 36 k + 36): Cov(x_a, x_b), a = frame_a[k], b = frame_b[k], 6x6 row-major, in the local tangent of the solve
 * (and of mvicp_debug_edge_blocks), what Ceres >= 1.14's GetCovarianceBlockInTangentSpace returns for the reference's blocks:
 *   MVICP_PARAM_SE3   (upsilon, omega) of x exp(delta), Sophus order;
 *   MVICP_PARAM_QUAT  (dq, dt): EigenQuaternionParameterization's dq (x, y, z), then the translation;
 *   MVICP_PARAM_AA    (dw, dt): angle-axis, then the translation.
 *   status[k] (nullable), in this order of precedence:
 *     MVICP_COV_FIXED        a or b is fixed: zeros (Ceres gives constant blocks zero covariance);
 *     MVICP_COV_INDEPENDENT  a and b lie in different connected components (mvicp_get_components): zeros, since J^T J is
 *                            block-diagonal over the components;
 *     MVICP_COV_SINGULAR     their component is rank-deficient: NaN.  A component without a fixed frame always is (its gauge
 *                            is free); otherwise the rank rule [ext, not Ceres' QR rule]: with S = diag(1 / sqrt(H_jj)) and the
 *                            Cholesky factor L~ of S H S, singular if some H_jj is zero or not finite, a pivot is not positive
 *                            or not finite, or L~_jj^2 <= 64 n 2^-53 (n unknowns of the component);
 *     MVICP_COV_OK           the block of C = S (S H S)^-1 S, each component factored as a problem of its own.
 * A block's bits depend only on the problem: not on which other pairs are requested, their order or duplicates; (b, a) is
 * the exact transpose of (a, b), so a diagonal block is exactly symmetric; two calls give the same bytes.  The call changes no
 * pose, fixed flag, correspondence, certificate, cached LM / g2o layout or statistic other than kernel_launches.
 * MVICP_ERR_INVALID before any work: bad param / cost, n_pairs < 0, a null array with n_pairs > 0, a frame outside [0, M),
 * point-to-plane without normals.  MVICP_ERR_STATE: no frames or graph, or a sharded context (the call runs on one GPU). */
enum { MVICP_COV_OK = 0, MVICP_COV_FIXED = 1, MVICP_COV_INDEPENDENT = 2, MVICP_COV_SINGULAR = 3 };
int mvicp_covariance(mvicp_ctx* ctx, int32_t param, int32_t cost, int32_t robust, int32_t n_pairs, const int32_t* frame_a,
                     const int32_t* frame_b, double* cov36, int32_t* status);

/* ICP_G2O::g2oOptimizer (include/icp-g2o.h:14, icp-g2o.cpp:149-303), the --g2o path of main_multiview.cpp:158-164: one g2o
 * Edge_V_V_GICP per stored correspondence of every edge with a free end (vertex 0 = dst, vertex 1 = src), VertexSE3 poses,
 * Levenberg-Marquardt over H + lambda I (no Jacobi scaling), and the reference's outer loop of optimize(iterations_per_call)
 * calls that stops after more than no_improvement_limit calls without a relative chi2 improvement.  Frame 0 is fixed.  A free
 * frame without any correspondence is not part of the problem and keeps its pose bit for bit.  DESIGN.md section 2 states
 * the g2o semantics that are restated here. */
typedef struct {
  int32_t iterations_per_call;      /* 100: optimizer.optimize(100), icp-g2o.cpp:271 (the pairwise solvers use 300)  */
  int32_t max_calls;                /* 100: icp-g2o.cpp:267                                                           */
  int32_t no_improvement_limit;     /* 5: stop once more than this many calls did not improve chi2, icp-g2o.cpp:297   */
  int32_t max_trials;               /* 10: g2o's maxTrialsAfterFailure                                                */
  int32_t orthonormalize_after;     /* 1000: VertexSE3::orthogonalizeAfter                                            */
  int32_t reserved;
  double tau;                       /* 1e-5: g2o's initial lambda = tau * max |H_jj|                                  */
  double information_eps;           /* 0.01: point-to-plane information prec0(eps), icp-g2o.cpp:248                   */
} mvicp_g2o_options;

enum { MVICP_G2O_END_NO_IMPROVEMENT = 0, /* the outer loop's noImpr counter passed its limit                   */
       MVICP_G2O_END_MAX_CALLS = 1,      /* max_calls calls of optimize() ran                                   */
       MVICP_G2O_END_NO_VERTICES = 2     /* no free frame has a correspondence: nothing was optimised           */ };
enum { MVICP_G2O_CALL_TERMINATE = 0,     /* the last call stopped on g2o's Terminate (trials exhausted or rho == 0) */
       MVICP_G2O_CALL_ITERATIONS = 1     /* the last call ran all of its iterations                                */ };

typedef struct {
  int32_t calls;                    /* optimize() calls                                          */
  int32_t iterations;               /* LM iterations over all calls                              */
  int32_t trials;                   /* trial steps = linear solves                               */
  int32_t accepted;                 /* trials kept                                               */
  int32_t evaluations;              /* streaming passes over the correspondences                 */
  int32_t ended;                    /* MVICP_G2O_END_*                                           */
  int32_t last_call_end;            /* MVICP_G2O_CALL_*                                          */
  int32_t reserved;
  double chi2_initial, chi2_final;  /* sum e^T Omega e before the first call / after the last    */
} mvicp_g2o_summary;

void mvicp_default_g2o_options(mvicp_g2o_options* o);
/* cost: MVICP_COST_P2P or MVICP_COST_P2PLANE (MIXED: MVICP_ERR_INVALID).  Not available in a sharded context (world > 1:
 * MVICP_ERR_STATE).  chi2_per_call (nullable, >= max_calls + 1 doubles): chi2 before the first call, then after each call. */
int mvicp_optimize_g2o(mvicp_ctx* ctx, int32_t cost, const mvicp_g2o_options* opt, mvicp_g2o_summary* summary,
                       double* chi2_per_call);
/* ICP_G2O::pointToPoint / pointToPlane (include/icp-g2o.h:10-11, icp-g2o.cpp:26-147): dst fixed at the identity, src from the
 * identity, 1:1 correspondences, one optimize() call of opt->iterations_per_call (opt NULL: 300) iterations, no outer loop.
 * pose16_out = the src vertex's pose (src -> dst).  nor = dst normals (NULL for point-to-point). */
int mvicp_pairwise_g2o(const mvicp_config* cfg, int32_t cost, const double* src_xyz, const double* dst_xyz, const double* nor_xyz,
                       int64_t n, const mvicp_g2o_options* opt, double* pose16_out, mvicp_g2o_summary* summary);
/* The trial trace of the last mvicp_optimize_g2o: 5 doubles per trial (lambda, chi, tchi, rho, accepted), in order.  Copies
 * min(capacity, recorded) rows; *n_trials = trials run (the first 65536 are recorded).  After mvicp_optimize_g2o_components:
 * MVICP_ERR_STATE (use mvicp_g2o_trace_component). */
int mvicp_g2o_trace(mvicp_ctx* ctx, double* out5, int64_t capacity, int64_t* n_trials);
/* One independent g2o solve per connected component (mvicp_get_components numbering), all in one pipelined loop: a batch of
 * unrelated registrations in one context.  The lowest frame of every component is fixed (as frame 0 is by mvicp_optimize_g2o,
 * icp-g2o.cpp:182-186); user-set flags are kept.  Each component is solved exactly as mvicp_optimize_g2o solves it in a fresh
 * context holding only that component (frames ascending, edges in graph order, same fixed flags, correspondences and options):
 * its own lambda, trials, calls, noImpr counter, ended / last_call_end and chi2; on a connected graph the result equals
 * mvicp_optimize_g2o's bit for bit.  Shared by the batch: the streaming tile length (from all active correspondence slots) and
 * the storage mode.  Argument checks are mvicp_optimize_g2o's, made before any state changes.  summaries (nullable):
 * n_components entries; a component without a vertex gets mvicp_optimize_g2o's MVICP_G2O_END_NO_VERTICES summary and keeps its
 * poses bit for bit.  chi2_per_call (nullable): n_components rows of (max_calls + 1) doubles, row k as mvicp_optimize_g2o fills
 * it for component k (entries past calls + 1 unspecified).  Each problem of a batch of P records the first
 * max(1024, 65536 / P) trials of its trace.  Sharded context: MVICP_ERR_STATE. */
int mvicp_optimize_g2o_components(mvicp_ctx* ctx, int32_t cost, const mvicp_g2o_options* opt, mvicp_g2o_summary* summaries,
                                  double* chi2_per_call);
/* The trial trace of component k of the last g2o solve, as mvicp_g2o_trace returns a trace (k = 0 after mvicp_optimize_g2o,
 * where it equals mvicp_g2o_trace).  k outside the last solve's components: MVICP_ERR_INVALID. */
int mvicp_g2o_trace_component(mvicp_ctx* ctx, int32_t component, double* out5, int64_t capacity, int64_t* n_trials);

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

/* Frame::getClosestPoint for n queries at once (q_xyz: n x 3 doubles in the frame's local coordinates): idx[i] / d2[i] are
 * bit for bit what mvicp_closest_point returns for query i (same fp32 screen, fp64 re-rank, lowest index on ties).  A query
 * with a non-finite coordinate gets idx -1 and d2 NaN; n = 0 does nothing; idx and d2 are nullable.  Host memory: the queries
 * go through the context's buffers and the call returns with the results in place. */
int mvicp_closest_points(mvicp_ctx* ctx, int32_t frame, const double* q_xyz, int64_t n, int64_t* idx, double* d2);

/* ---- device twins: the calls above whose per-point arrays are in device memory ---------------------------------------
 * Each one returns the same bytes as its host-memory twin, with the same argument checks, state errors (MVICP_ERR_STATE) and
 * sharding rules (a rank sees the edges it processes; the others' lists are empty).  Every array argument must be device or
 * managed memory of the context's device (cudaPointerGetAttributes); anything else, a host pointer included, gives
 * MVICP_ERR_INVALID before any work is done.  Reads and writes are ordered on the context's stream (mvicp_get_stream): a caller
 * that produces inputs or consumes outputs on another stream orders it against that one.  mvicp_set_frames_device and
 * mvicp_set_edge_device return only after the caller's arrays have been read; the others are stream-ordered only and do not
 * wait for the device. */
/* mvicp_set_frames with pts_xyz[f] / nor_xyz[f] in device memory (the pointer arrays and n_pts stay on the host).  The frames
 * are copied device to device and built there; under MVICP_FLAG_HOST_BUILD they are staged to the host and built there. */
int mvicp_set_frames_device(mvicp_ctx* ctx, int32_t n_frames, const double* const* pts_xyz, const double* const* nor_xyz,
                            const int64_t* n_pts);
/* mvicp_set_edge with first / second in device memory: the same range check (a bad index leaves the edge as it was), the
 * whole edge reset to "no match", the last occurrence of a duplicated src index wins, count stored as given. */
int mvicp_set_edge_device(mvicp_ctx* ctx, int32_t e, const int32_t* first, const int32_t* second, int64_t count, float weight);
/* mvicp_get_all_edges into device memory: out_records (16-byte Correspondance records, nullable), offsets (int64, n_edges + 1)
 * and weights (nullable).  No host synchronisation; for that reason, when out_records is given, capacity must be at least the
 * sum of the src cloud sizes over the edges this context processes (MVICP_ERR_INVALID otherwise, before any launch).  Records
 * past offsets[n_edges] are unspecified. */
int mvicp_get_all_edges_device(mvicp_ctx* ctx, void* out_records, int64_t capacity, int64_t* offsets, float* weights);
/* mvicp_closest_points with q_xyz, idx and d2 in device memory. */
int mvicp_closest_points_device(mvicp_ctx* ctx, int32_t frame, const double* q_xyz, int64_t n, int64_t* idx, double* d2);
/* mvicp_get_normals into device memory (N x 3 doubles). */
int mvicp_get_normals_device(mvicp_ctx* ctx, int32_t frame, double* nor_xyz);
/* mvicp_knn_self into device memory (N x k int32); scratch comes from the context's reusable buffers. */
int mvicp_knn_self_device(mvicp_ctx* ctx, int32_t frame, int32_t k, int32_t* nn_idx);

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
