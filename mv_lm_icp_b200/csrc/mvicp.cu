// mvicp.cu -- context, host orchestration and the C ABI of libmvicp.so (include/mvicp.h).
//
// Host side stays thin C++: it owns device buffers, builds the per-frame search structure once, enqueues the
// kernels of knn.cuh / select.cuh / lm_eval.cuh / lm_step.cuh on one stream, and (multi-GPU) calls NCCL between
// them.  No CPU fallback exists: every compute entry point fails with MVICP_ERR_CUDA when no device is usable.
#include <cuda_runtime.h>
#include <nccl.h>
#ifdef __linux__
#include <sched.h>
#endif
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <numeric>
#include <string>
#include <thread>
#include <vector>

#include "../../include/mvicp.h"
#include "closed.cuh"
#include "compact.cuh"
#include "covariance.cuh"
#include "device_io.cuh"
#include "far.cuh"
#include "g2o.cuh"
#include "knn.cuh"
#include "lm_eval.cuh"
#include "lm_step.cuh"
#include "normals.cuh"
#include "se3_math.cuh"
#include "select.cuh"
#include "types.cuh"

using namespace mv;

static thread_local std::string g_err;
static int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
  g_err = buf;
  return code;
}
#define CU(call)                                                                                              \
  do {                                                                                                        \
    cudaError_t e_ = (call);                                                                                  \
    if (e_ != cudaSuccess) return fail(MVICP_ERR_CUDA, "%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
  } while (0)
#define NC(call)                                                                                              \
  do {                                                                                                        \
    ncclResult_t r_ = (call);                                                                                 \
    if (r_ != ncclSuccess) return fail(MVICP_ERR_NCCL, "%s:%d %s: %s", __FILE__, __LINE__, #call, ncclGetErrorString(r_)); \
  } while (0)
#define RET(call) do { int r__ = (call); if (r__ != MVICP_OK) return r__; } while (0)

// A device allocation that only grows; freed with its owner (the context's device must be current then, as in mvicp_destroy)
struct DevBuf {
  void* p = nullptr; size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
  int reserve(size_t bytes) {
    if (bytes <= cap) return MVICP_OK;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    CU(cudaMalloc(&p, bytes ? bytes : 16));
    cap = bytes ? bytes : 16;
    return MVICP_OK;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
  template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
};

// LM problems as upload_problems lays them out: one int32 buffer (frame and edge lists, gather lists, envelopes, skylines, the
// edge -> problem map), one fp64 buffer, the LmProblem views (device, and a host copy), room for P + 1 states
struct ProblemBufs {
  DevBuf i32, f64, prob, state;
  std::vector<LmProblem> h_prob;           // host copy of the views
  const int32_t* edge_prob = nullptr;      // [E] edge -> problem, or -1 (in i32)
  size_t dyn = 0;                          // dynamic shared memory of the step kernels: the maximum over the problems
  std::vector<uint8_t> key;                // kind of solve, fixed flags and graph generation the problems were uploaded for
};

struct mvicp_ctx {
  int device = 0, flags = 0;
  cudaStream_t stream = nullptr; bool own_stream = false;
  int rank = 0, world = 1; ncclComm_t comm = nullptr;
  // peer-memory exchange of the LM pair matrices (sharded runs): own buffer + IPC mappings of every peer's
  void* xbuf = nullptr; void* peer_x[MAX_PEERS] = {}; bool p2p_ok = false; int32_t xseq = 0;
  static constexpr int X_ECAP = 4096;   // edges the exchange buffer is sized for (2 halves x X_ECAP x EOUT doubles + flags)
  // frames
  int M = 0; bool f32 = true; bool nor_f32 = true; bool have_normals = true;
  std::vector<void*> nor_dbl;   // per frame: fp64 normals [n][3] after mvicp_recompute_normals (device)
  float normals_ms = 0.f;
  std::vector<int64_t> n_pts;
  std::vector<FrameDev> h_frames;
  std::vector<void*> frame_allocs;
  DevBuf d_obb;                // ObbDev per frame (unless MVICP_FLAG_NO_OBB)
  int seeded_rounds = 0;       // consecutive mvicp_correspond calls that started from the previous call's matches
  DevBuf d_single;             // result slot of mvicp_closest_point
  DevBuf d_prof;               // lm_step_kernel's clock stamps (MVICP_STEP_PROFILE=1, one-problem solves)
  DevBuf d_tile_count, d_tile_off, d_edge_off, d_recs;   // mvicp_get_all_edges
  bool obb_ready = false;
  int last_lm_iters = 1 << 20; // LM iterations of the previous mvicp_optimize: large = the clouds are still far apart
  DevBuf d_frames, d_poses;
  std::vector<uint8_t> fixed;
  std::vector<double> h_poses;   // mirror of the last set/get (pose graph construction is host side)
  // graph
  int E = 0;
  std::vector<EdgeDev> h_edges;
  std::vector<int32_t> edge_owner;   // rank that processes edge e (-1: src frame fixed, nobody)
  DevBuf d_edges, d_xf, d_corr, d_d2, d_count, d_sel, d_hist, d_weight, d_median, d_selcand, d_selcand_n;
  DevBuf d_sel_cnt;            // guessed select: [E] inliers | [E] inliers below the guessed window | [1] guesses that missed
  DevBuf d_sel_win;            // [3E] window lo | hi | log2 half-width (select.cuh)
  DevBuf d_certs, d_cert_cnt;  // certificates (knn.cuh, CERT): {position, margin} per slot in tile order; reused queries per edge
  DevBuf d_todo, d_todo_n;     // certified rounds: the queries that have to be searched after all ({edge, position}), and their number
  bool cert_valid = false;     // every slot's margin belongs to the match in d_corr (the last mvicp_correspond ran with certificates)
  int64_t cert_rounds = 0;
  bool sel_valid = false;      // d_sel holds the previous round's medians (a select ran since the buffers were laid out)
  int64_t sel_guess_rounds = 0;
  DevBuf d_knn_tiles, d_eval_tiles, d_edge_tile_begin, d_partial;
  int n_knn_tiles = 0, n_eval_tiles = 0, eval_tile_len = EVAL_TILE;
  int64_t total_slots = 0;
  bool have_corr = false;      // corr[] holds a previous round (usable as seeds)
  bool nonrigid = false;       // some uploaded pose does not yield a unit quaternion (general LM path for QUAT / SE3)
  std::vector<float> h_weight; std::vector<unsigned long long> h_count;
  // LM
  DevBuf d_x, d_cand, d_Rt, d_K, d_eout, d_posegather, d_gen;
  int lm_blocks_E = 0;         // edges of the evaluation d_eout holds; 0: none since the graph was set, or the last solve failed
  bool blocks_g2o = false;     // that evaluation is a g2o solve's (g2o_edge_kernel's records), not an LM solve's
  std::vector<uint8_t> lm_blocks_fixed;   // LM: the fixed flags of that solve: the edges of a fixed src read as zeros
  std::vector<uint8_t> g2o_blocks_unwritten;   // g2o: the edges no evaluation of that solve wrote (they read as zeros)
  std::vector<int32_t> h_col;
  volatile int32_t* h_flag = nullptr; volatile int32_t* d_flag = nullptr;   // mapped pinned ring written by the step kernels
  uint32_t graph_gen = 0;
  // the LM problems last uploaded for a solve (upload_problems), and the step kernel's ticket
  ProblemBufs lm;
  DevBuf d_lm_ticket;
  // mvicp_covariance: its own problems (cached like lm), evaluation point, tiles, pair matrices and outputs, so that nothing a
  // solve or mvicp_debug_edge_blocks reads is touched
  ProblemBufs cov;
  DevBuf d_cov_x, d_cov_cand, d_cov_Rt, d_cov_K, d_cov_gen, d_cov_partial, d_cov_eout, d_cov_tiles, d_cov_etb, d_cov_status,
         d_cov_jobs, d_cov_out;
  void* h_state = nullptr; size_t h_state_cap = 0;   // pinned staging of the P + 1 LmStates
  // g2o solve (g2o.cuh); the normal equations of its problems are uploaded LM problems
  DevBuf d_g2o_state, d_g2o_prob, d_g2o_x, d_g2o_ev, d_g2o_nop, d_g2o_chi, d_g2o_trace, d_g2o_tiles, d_g2o_tile_begin, d_g2o_cnt;
  // trace of the last g2o solve, per component (one entry after mvicp_optimize_g2o): trials run, first row in d_g2o_trace
  // (-1: no problem), and the rows recorded per problem
  std::vector<int64_t> g2o_trials{0}, g2o_trace_row{-1};
  int64_t g2o_trace_cap = 0;
  bool g2o_per_component = false;
  // stats
  mvicp_stats stats{};
  cudaEvent_t ev[8]{};
  std::vector<cudaEvent_t> eval_ev;   // pairs around every lm_eval launch of the last optimize
  int eval_ev_used = 0;
  bool ev_knn = false, ev_lm = false;
  float lm_eval_acc = 0.f;
  // scratch of the device twins (mvicp_closest_points, mvicp_set_edge_device, mvicp_knn_self_device)
  DevBuf d_cpq, d_cpr;         // queries, then results (int64 index | fp64 d2)
  DevBuf d_set_win, d_set_bad; // winning position + 1 per src slot, lowest bad position
  DevBuf d_knn_nor;            // the normals the k-NN kernel also writes
};

static inline int owner_of(const mvicp_ctx* c, int frame) { return (int)(((int64_t)frame * c->world) / std::max(1, c->M)); }
// Sharding rule (mirrored in mv_lm_icp_b200/dist.py:edge_owners): the edges whose src frame is not fixed, in graph order,
// are cut into `world` contiguous runs of (nearly) equal query count -- an edge goes to the rank that the midpoint of its
// query range falls to.  Contiguous runs keep a rank on few src frames; cutting by queries rather than by frames keeps the
// ranks within one edge of each other (20 frames over 8 ranks would be 3 frames against 2).
static void assign_edge_owners(mvicp_ctx* c) {
  const int E = c->E;
  c->edge_owner.assign(E, -1);
  int64_t total = 0;
  for (int e = 0; e < E; ++e) if (!c->fixed[c->h_edges[e].src]) total += c->n_pts[c->h_edges[e].src];
  int64_t before = 0;
  for (int e = 0; e < E; ++e) {
    const int s = c->h_edges[e].src;
    if (c->fixed[s]) continue;
    const int64_t n = c->n_pts[s];
    c->edge_owner[e] = total > 0 ? (int)std::min<int64_t>(c->world - 1, ((2 * before + n) * c->world) / (2 * total)) : 0;
    before += n;
  }
}

// =================================================================================================
// one-time per-frame search structure (replaces the lazily built nanoflann index, frame.cpp:188-193)
// =================================================================================================
#include "tree_build.h"
#include "tree_gpu.cuh"

extern "C" { static int refresh_after_fixed_change(mvicp_ctx* c); }

// Does some pose's rotation part yield a quaternion that is not unit (to 1e-9)?  Then the reference's quaternion / SE3 functors run
// on non-unit quaternions (no normalisation anywhere, so3.hpp:666-668) and the LM step takes the general frame model.  True for
// non-rigid input (the Bunny_RealData sample poses), and it can BECOME true: every solve writes q -> matrix back without
// normalising (eigenQuaternionToIso / sophusToIso, icp-ceres.cpp:117-134), so the quaternion parameterisation drifts.
static bool poses_nonrigid(const double* poses16, int M) {
  for (int f = 0; f < M; ++f) {
    Rt a; pose16_to_Rt(poses16 + 16 * f, &a);
    double q[4]; quat_of_matrix(a.R, q);
    const double n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
    if (!(std::fabs(n2 - 1.0) <= 1e-9)) return true;
  }
  return false;
}

// worker threads for the one-time host work: the CPUs this process may use (affinity mask, cgroup v2 quota), not the machine's
static unsigned host_workers() {
  unsigned n = std::max(1u, std::thread::hardware_concurrency());
#ifdef __linux__
  cpu_set_t set; CPU_ZERO(&set);
  if (sched_getaffinity(0, sizeof set, &set) == 0) { const int k = CPU_COUNT(&set); if (k > 0) n = std::min<unsigned>(n, (unsigned)k); }
  if (FILE* f = std::fopen("/sys/fs/cgroup/cpu.max", "r")) {
    char q[32]; long long period = 0;
    if (std::fscanf(f, "%31s %lld", q, &period) == 2 && std::strcmp(q, "max") != 0 && period > 0) {
      const long long quota = std::atoll(q);
      if (quota > 0) n = std::min<unsigned>(n, (unsigned)std::max<long long>(1, quota / period));
    }
    std::fclose(f);
  }
#endif
  return std::max(1u, n);
}

// common tail of mvicp_set_frames: frame table and identity poses on the device, graph and solver state reset
static int finish_set_frames(mvicp_ctx* c, int M) {
  if (c->f32 && c->nor_f32)   // packed point+normal records for the LM gathers (fp32 storage only)
    for (int f = 0; f < M; ++f) {
      FrameDev& fr = c->h_frames[f];
      if (!fr.nor_o) continue;
      void* d_pn = nullptr;
      CU(cudaMalloc(&d_pn, sizeof(float4) * 2 * (size_t)fr.n)); c->frame_allocs.push_back(d_pn);
      pack_pn_kernel<<<(fr.n + 255) / 256, 256, 0, c->stream>>>((const float4*)fr.pts_o, (const float4*)fr.nor_o, fr.n, (float4*)d_pn);
      c->stats.kernel_launches += 1;
      fr.pn_o = (const float4*)d_pn;
    }
  RET(c->d_frames.reserve(sizeof(FrameDev) * M));
  CU(cudaMemcpy(c->d_frames.p, c->h_frames.data(), sizeof(FrameDev) * M, cudaMemcpyHostToDevice));
  RET(c->d_poses.reserve(sizeof(double) * 16 * M));
  c->h_poses.assign((size_t)16 * M, 0.0);
  for (int f = 0; f < M; ++f) for (int i = 0; i < 4; ++i) c->h_poses[16 * f + 5 * i] = 1.0;
  CU(cudaMemcpy(c->d_poses.p, c->h_poses.data(), sizeof(double) * 16 * M, cudaMemcpyHostToDevice));
  c->fixed.assign(M, 0); c->fixed[0] = 1;
  c->E = 0; c->h_edges.clear(); c->have_corr = false; c->lm_blocks_E = 0;
  c->last_lm_iters = 1 << 20;
  return MVICP_OK;
}

#ifdef __CUDACC__
// Device construction of every frame's search structure (tree_gpu.cuh): raw coordinates go up once, everything else -- the
// fp32-representability scan that picks the storage mode, the KD ordering, records, boxes, faces, oriented boxes -- is built there.
template <bool F32>
static int build_frames_on_device(mvicp_ctx* c, int M, const std::vector<double*>& d_xyz, const std::vector<double*>& d_nor,
                                  const int64_t* n_pts, const std::vector<float>& absmax) {
  const size_t rec = F32 ? sizeof(float4) : sizeof(double4a);
  const bool want_obb = !(c->flags & MVICP_FLAG_NO_OBB);
  KdScratch S;
  std::vector<ObbDev> ho(M);
  cudaError_t err = cudaSuccess;
  for (int f = 0; f < M && err == cudaSuccess; ++f) {
    const int n = (int)n_pts[f];
    const int64_t n_leaf = std::max<int64_t>(1, ((int64_t)n + LEAF - 1) / LEAF);
    int L = 1; while (L < n_leaf) L <<= 1;
    int depth = 0; while ((1 << depth) < L) ++depth;
    const int n_pad = (int)(n_leaf * LEAF);
    void *d_o = nullptr, *d_n = nullptr, *d_s = nullptr, *d_b = nullptr, *d_sf = nullptr, *d_pos = nullptr, *d_fc = nullptr, *d_ob = nullptr, *d_adj = nullptr;
    auto grab = [&](void** p, size_t bytes) { if (err == cudaSuccess) { err = cudaMalloc(p, bytes); if (err == cudaSuccess) c->frame_allocs.push_back(*p); } };
    grab(&d_o, rec * (size_t)n); grab(&d_s, rec * (size_t)n_pad); grab(&d_b, sizeof(Box) * 2 * (size_t)L); grab(&d_fc, sizeof(float) * 2 * (size_t)L);
    grab(&d_pos, sizeof(int32_t) * (size_t)n); grab(&d_adj, sizeof(int32_t) * ADJ_SLOTS * (size_t)L);
    if (F32) d_sf = d_s; else grab(&d_sf, sizeof(float4) * (size_t)n_pad);
    if (d_nor[f]) grab(&d_n, rec * (size_t)n);
    if (want_obb) grab(&d_ob, sizeof(ObbNode) * 2 * (size_t)L);
    if (err != cudaSuccess) break;
    const KdGeom g{n, L, depth};
    err = kd_build_device<F32>(c->stream, S, d_xyz[f], g, d_s, (float4*)d_sf, (int32_t*)d_pos, (Box*)d_b, (float*)d_fc, (int32_t*)d_adj, (ObbNode*)d_ob,
                               &c->stats.kernel_launches);
    kd_pack_orig_kernel<F32><<<(n + 255) / 256, 256, 0, c->stream>>>(d_xyz[f], n, d_o);
    if (d_nor[f]) kd_pack_orig_kernel<F32><<<(n + 255) / 256, 256, 0, c->stream>>>(d_nor[f], n, d_n);
    c->stats.kernel_launches += d_nor[f] ? 2 : 1;
    c->h_frames[f] = FrameDev{d_o, d_n, nullptr, d_s, (const float4*)d_sf, (const Box*)d_b, (const float*)d_fc, (const int32_t*)d_pos,
                              (c->flags & MVICP_FLAG_NO_ADJ) ? nullptr : (const int32_t*)d_adj, (int32_t)n, L, depth, absmax[f]};
    ho[f] = ObbDev{(const ObbNode*)d_ob};
  }
  if (err == cudaSuccess) err = cudaStreamSynchronize(c->stream);
  S.release();
  if (err != cudaSuccess) return fail(MVICP_ERR_CUDA, "device tree build: %s", cudaGetErrorString(err));
  if (want_obb) {
    RET(c->d_obb.reserve(sizeof(ObbDev) * M));
    CU(cudaMemcpy(c->d_obb.p, ho.data(), sizeof(ObbDev) * M, cudaMemcpyHostToDevice));
    c->obb_ready = true;
  }
  return MVICP_OK;
}

// kind: cudaMemcpyHostToDevice (mvicp_set_frames) or cudaMemcpyDeviceToDevice (mvicp_set_frames_device)
static int set_frames_device(mvicp_ctx* c, int M, const double* const* pts, const double* const* nor, const int64_t* n_pts,
                             cudaMemcpyKind kind) {
  std::vector<double*> d_xyz(M, nullptr), d_nor(M, nullptr);
  int* d_flags = nullptr;
  auto cleanup = [&]() { for (double* p : d_xyz) cudaFree(p); for (double* p : d_nor) cudaFree(p); cudaFree(d_flags); };
  std::vector<int> h_flags(4 * (size_t)M);
  for (int f = 0; f < M; ++f) { h_flags[4 * f] = 1; h_flags[4 * f + 1] = 0; h_flags[4 * f + 2] = 1; h_flags[4 * f + 3] = 0; }
  cudaError_t err = cudaMalloc(&d_flags, sizeof(int) * 4 * (size_t)M);
  if (err == cudaSuccess) err = cudaMemcpy(d_flags, h_flags.data(), sizeof(int) * 4 * (size_t)M, cudaMemcpyHostToDevice);
  for (int f = 0; f < M && err == cudaSuccess; ++f) {
    const size_t bytes = sizeof(double) * 3 * (size_t)n_pts[f];
    err = cudaMalloc(&d_xyz[f], bytes);
    if (err == cudaSuccess) err = cudaMemcpyAsync(d_xyz[f], pts[f], bytes, kind, c->stream);
    if (err == cudaSuccess) kd_scan_kernel<<<2 * NUM_SMS, 256, 0, c->stream>>>(d_xyz[f], 3ll * n_pts[f], d_flags + 4 * f);
    if (err == cudaSuccess && nor && nor[f]) {
      err = cudaMalloc(&d_nor[f], bytes);
      if (err == cudaSuccess) err = cudaMemcpyAsync(d_nor[f], nor[f], bytes, kind, c->stream);
      if (err == cudaSuccess) kd_scan_kernel<<<2 * NUM_SMS, 256, 0, c->stream>>>(d_nor[f], 3ll * n_pts[f], d_flags + 4 * f + 2);
    }
    c->stats.kernel_launches += (nor && nor[f]) ? 2 : 1;
  }
  if (err == cudaSuccess) err = cudaMemcpyAsync(h_flags.data(), d_flags, sizeof(int) * 4 * (size_t)M, cudaMemcpyDeviceToHost, c->stream);
  if (err == cudaSuccess) err = cudaStreamSynchronize(c->stream);
  if (err != cudaSuccess) { cleanup(); return fail(MVICP_ERR_CUDA, "mvicp_set_frames (upload): %s", cudaGetErrorString(err)); }
  bool f32 = true; std::vector<float> absmax(M);
  for (int f = 0; f < M; ++f) {
    f32 = f32 && h_flags[4 * f] != 0 && h_flags[4 * f + 2] != 0;
    std::memcpy(&absmax[f], &h_flags[4 * f + 1], 4);
    if (!std::isfinite(absmax[f])) { cleanup(); return fail(MVICP_ERR_INVALID, "frame %d has a non-finite coordinate", f); }
  }
  c->f32 = f32; c->nor_f32 = f32;
  c->h_frames.assign(M, FrameDev{});
  const int rc = f32 ? build_frames_on_device<true>(c, M, d_xyz, d_nor, n_pts, absmax) : build_frames_on_device<false>(c, M, d_xyz, d_nor, n_pts, absmax);
  cleanup();
  return rc;
}
#endif

static bool all_fp32(const double* v, int64_t n) {
  for (int64_t i = 0; i < n; ++i) if ((double)(float)v[i] != v[i]) return false;
  return true;
}

static void pack_records(bool f32, const double* xyz, const int32_t* order, const int32_t* wfield, int64_t n, void* out) {
  // record i <- point order[i] (or i when order == null); .w <- wfield[i] bits (or 0)
  for (int64_t i = 0; i < n; ++i) {
    const int64_t j = order ? order[i] : i;
    const int32_t w = wfield ? wfield[i] : 0;
    if (f32) {
      float4 r; r.x = (float)xyz[3 * j]; r.y = (float)xyz[3 * j + 1]; r.z = (float)xyz[3 * j + 2];
      std::memcpy(&r.w, &w, 4);
      reinterpret_cast<float4*>(out)[i] = r;
    } else {
      double4a r; r.x = xyz[3 * j]; r.y = xyz[3 * j + 1]; r.z = xyz[3 * j + 2];
      const long long wl = w; std::memcpy(&r.w, &wl, 8);
      reinterpret_cast<double4a*>(out)[i] = r;
    }
  }
}

static void pad_records(bool f32, void* recs, int64_t n, int64_t n_pad) {
  const int32_t w = INT32_MAX;
  for (int64_t i = n; i < n_pad; ++i) {
    if (f32) { float4 r; r.x = r.y = r.z = INFINITY; std::memcpy(&r.w, &w, 4); reinterpret_cast<float4*>(recs)[i] = r; }
    else { double4a r; r.x = r.y = r.z = INFINITY; const long long wl = w; std::memcpy(&r.w, &wl, 8); reinterpret_cast<double4a*>(recs)[i] = r; }
  }
}

// Arguments of the `_device` entry points: device (or managed) memory of the context's device, nothing else -- a host pointer
// is refused before any work is done.
static int check_device_ptr(const mvicp_ctx* c, const void* p, const char* fn, const char* what) {
  if (!p) return fail(MVICP_ERR_INVALID, "%s: %s is null", fn, what);
  cudaPointerAttributes a; std::memset(&a, 0, sizeof a);
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return fail(MVICP_ERR_INVALID, "%s: %s is not device memory", fn, what); }
  if ((a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) || a.device != c->device)
    return fail(MVICP_ERR_INVALID, "%s: %s is not device memory of device %d", fn, what, c->device);
  return MVICP_OK;
}

// =================================================================================================
// C ABI
// =================================================================================================
extern "C" {

int mvicp_abi_version(void) { return 1; }
const char* mvicp_last_error(void) { return g_err.c_str(); }

void mvicp_default_lm_options(mvicp_lm_options* o) {
  o->max_num_iterations = 50; o->max_num_consecutive_invalid_steps = 5; o->jacobi_scaling = 1; o->reserved = 0;
  o->initial_trust_region_radius = 1e4; o->max_trust_region_radius = 1e16; o->min_trust_region_radius = 1e-32;
  o->min_relative_decrease = 1e-3; o->min_lm_diagonal = 1e-6; o->max_lm_diagonal = 1e32;
  o->function_tolerance = 1e-6; o->gradient_tolerance = 1e-10; o->parameter_tolerance = 1e-8;
}

}  // extern "C"
// The rules of mvicp_lm_options (include/mvicp.h): what Ceres' Solver::Options::IsValid rejects for a trust-region LM solve.
// Every test is written as "the valid case holds", so a NaN fails it.  Called before an entry point changes any state; a null
// pointer stands for the defaults.
static int check_lm_options(const mvicp_lm_options* o, const char* fn) {
  if (!o) return MVICP_OK;
  const char* bad = nullptr;
  if (!(o->max_num_iterations >= 0)) bad = "max_num_iterations < 0";
  else if (!(o->max_num_consecutive_invalid_steps >= 0)) bad = "max_num_consecutive_invalid_steps < 0";
  else if (!(o->function_tolerance >= 0.0)) bad = "function_tolerance < 0";
  else if (!(o->gradient_tolerance >= 0.0)) bad = "gradient_tolerance < 0";
  else if (!(o->parameter_tolerance >= 0.0)) bad = "parameter_tolerance < 0";
  else if (!(o->initial_trust_region_radius > 0.0)) bad = "initial_trust_region_radius <= 0";
  else if (!(o->max_trust_region_radius > 0.0)) bad = "max_trust_region_radius <= 0";
  else if (!(o->min_trust_region_radius > 0.0)) bad = "min_trust_region_radius <= 0";
  else if (!(o->min_trust_region_radius <= o->initial_trust_region_radius)) bad = "min_trust_region_radius > initial_trust_region_radius";
  else if (!(o->initial_trust_region_radius <= o->max_trust_region_radius)) bad = "initial_trust_region_radius > max_trust_region_radius";
  else if (!(o->min_relative_decrease >= 0.0)) bad = "min_relative_decrease < 0";
  else if (!(o->min_lm_diagonal >= 0.0)) bad = "min_lm_diagonal < 0";
  else if (!(o->max_lm_diagonal >= 0.0)) bad = "max_lm_diagonal < 0";
  else if (!(o->min_lm_diagonal <= o->max_lm_diagonal)) bad = "min_lm_diagonal > max_lm_diagonal";
  return bad ? fail(MVICP_ERR_INVALID, "%s: invalid LM options: %s (or NaN)", fn, bad) : MVICP_OK;
}
extern "C" {

int mvicp_create(const mvicp_config* cfg, mvicp_ctx** out) {
  if (!out) return fail(MVICP_ERR_INVALID, "mvicp_create: out is null");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(MVICP_ERR_CUDA, "mvicp_create: no CUDA device (%s); this engine has no CPU path", cudaGetErrorString(e));
  mvicp_ctx* c = new mvicp_ctx();
  c->device = cfg ? cfg->device : 0;
  c->flags = cfg ? cfg->flags : 0;
  if (c->device < 0 || c->device >= ndev) { const int d = c->device; delete c; return fail(MVICP_ERR_INVALID, "device %d out of range", d); }
  auto init = [&]() -> int {
    CU(cudaSetDevice(c->device));
    if (cfg && cfg->stream) c->stream = (cudaStream_t)cfg->stream;
    else { CU(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking)); c->own_stream = true; }
    for (auto& ev : c->ev) CU(cudaEventCreate(&ev));
    CU(cudaHostAlloc((void**)&c->h_flag, sizeof(int32_t) * 8, cudaHostAllocMapped));
    CU(cudaHostGetDevicePointer((void**)&c->d_flag, (void*)c->h_flag, 0));
    RET(c->d_single.reserve(16));
    return MVICP_OK;
  };
  const int rc = init();
  if (rc != MVICP_OK) { const std::string keep = g_err; mvicp_destroy(c); g_err = keep; return rc; }   // frees whatever was created
  *out = c;
  return MVICP_OK;
}

void mvicp_destroy(mvicp_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  for (int p = 0; p < MAX_PEERS; ++p) if (c->peer_x[p] && c->peer_x[p] != c->xbuf) cudaIpcCloseMemHandle(c->peer_x[p]);
  if (c->xbuf) cudaFree(c->xbuf);
  if (c->comm) ncclCommDestroy(c->comm);
  for (void* p : c->frame_allocs) cudaFree(p);
  for (auto& ev : c->ev) if (ev) cudaEventDestroy(ev);
  for (auto& ev : c->eval_ev) cudaEventDestroy(ev);
  if (c->h_state) cudaFreeHost(c->h_state);
  if (c->h_flag) cudaFreeHost((void*)c->h_flag);

  if (c->own_stream && c->stream) cudaStreamDestroy(c->stream);
  delete c;   // frees every DevBuf, on the device set above
}

}  // extern "C"
// mvicp_set_frames and its device twin: dev_src = the coordinate arrays are device memory (checked by the caller)
static int set_frames_impl(mvicp_ctx* c, int32_t M, const double* const* pts, const double* const* nor, const int64_t* n_pts, bool dev_src) {
  if (!c || M <= 0 || !pts || !n_pts) return fail(MVICP_ERR_INVALID, "mvicp_set_frames: bad arguments");
  CU(cudaSetDevice(c->device));
  CU(cudaStreamSynchronize(c->stream));
  for (void* p : c->frame_allocs) cudaFree(p);
  c->frame_allocs.clear();
  c->M = M; c->n_pts.assign(n_pts, n_pts + M);
  c->have_normals = true;
  bool f32 = true;
  for (int f = 0; f < M; ++f) {
    if (n_pts[f] <= 0) return fail(MVICP_ERR_EMPTY, "frame %d has no points (nanoflann would throw, nanoflann.hpp:904)", f);
    if (n_pts[f] > (int64_t)INT32_MAX / 2) return fail(MVICP_ERR_INVALID, "frame %d too large", f);
    if (!pts[f]) return fail(MVICP_ERR_INVALID, "frame %d: null points", f);
    if (!nor || !nor[f]) c->have_normals = false;
  }
  c->nor_dbl.clear();
  c->obb_ready = false;
#ifdef __CUDACC__
  if (!(c->flags & MVICP_FLAG_HOST_BUILD)) {
    RET(set_frames_device(c, M, pts, nor, n_pts, dev_src ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
    return finish_set_frames(c, M);
  }
#endif
  // the host build of device-resident frames: stage them to the host first (the A/B flag and the host model take this path)
  std::vector<std::vector<double>> staged;
  std::vector<const double*> hp, hn;
  if (dev_src) {
    staged.resize(2 * (size_t)M); hp.assign(M, nullptr); hn.assign(M, nullptr);
    for (int f = 0; f < M; ++f) {
      const size_t cnt = 3 * (size_t)n_pts[f];
      staged[2 * f].resize(cnt);
      CU(cudaMemcpyAsync(staged[2 * f].data(), pts[f], sizeof(double) * cnt, cudaMemcpyDeviceToHost, c->stream));
      hp[f] = staged[2 * f].data();
      if (nor && nor[f]) {
        staged[2 * f + 1].resize(cnt);
        CU(cudaMemcpyAsync(staged[2 * f + 1].data(), nor[f], sizeof(double) * cnt, cudaMemcpyDeviceToHost, c->stream));
        hn[f] = staged[2 * f + 1].data();
      }
    }
    CU(cudaStreamSynchronize(c->stream));
    pts = hp.data();
    if (nor) nor = hn.data();
  }
  for (int f = 0; f < M; ++f) f32 = f32 && all_fp32(pts[f], 3 * n_pts[f]) && (!nor || !nor[f] || all_fp32(nor[f], 3 * n_pts[f]));
  c->f32 = f32; c->nor_f32 = f32;
  const size_t rec = f32 ? sizeof(float4) : sizeof(double4a);
  std::vector<HostFrameBuild> builds(M);
  {
    const unsigned hw = host_workers();
    std::vector<std::thread> pool;
    std::atomic<int> next{0};
    for (unsigned t = 0; t < std::min<unsigned>(hw, (unsigned)M); ++t)
      pool.emplace_back([&]() { for (int f; (f = next.fetch_add(1)) < M;) build_frame(pts[f], n_pts[f], builds[f]); });
    for (auto& th : pool) th.join();
  }
  c->h_frames.assign(M, FrameDev{});
  std::vector<char> stage;
  for (int f = 0; f < M; ++f) {
    const int64_t n = n_pts[f];
    void *d_o = nullptr, *d_n = nullptr, *d_s = nullptr, *d_b = nullptr, *d_sf = nullptr, *d_pos = nullptr, *d_fc = nullptr, *d_adj = nullptr;
    CU(cudaMalloc(&d_o, rec * n)); c->frame_allocs.push_back(d_o);
    const int64_t n_pad = ((n + LEAF - 1) / LEAF) * LEAF;   // tree-order arrays are padded to whole leaves with +inf points
    CU(cudaMalloc(&d_s, rec * n_pad)); c->frame_allocs.push_back(d_s);
    CU(cudaMalloc(&d_b, sizeof(Box) * builds[f].boxes.size())); c->frame_allocs.push_back(d_b);
    stage.resize(rec * n);
    pack_records(f32, pts[f], nullptr, nullptr, n, stage.data());
    CU(cudaMemcpy(d_o, stage.data(), rec * n, cudaMemcpyHostToDevice));
    stage.resize(rec * n_pad);
    pack_records(f32, pts[f], builds[f].order.data(), builds[f].order.data(), n, stage.data());
    pad_records(f32, stage.data(), n, n_pad);
    CU(cudaMemcpy(d_s, stage.data(), rec * n_pad, cudaMemcpyHostToDevice));
    if (nor && nor[f]) {
      CU(cudaMalloc(&d_n, rec * n)); c->frame_allocs.push_back(d_n);
      pack_records(f32, nor[f], nullptr, nullptr, n, stage.data());
      CU(cudaMemcpy(d_n, stage.data(), rec * n, cudaMemcpyHostToDevice));
    }
    CU(cudaMemcpy(d_b, builds[f].boxes.data(), sizeof(Box) * builds[f].boxes.size(), cudaMemcpyHostToDevice));
    if (f32) d_sf = d_s;
    else {   // rounded fp32 copy used only to screen candidates; exact arithmetic reads pts_s
      CU(cudaMalloc(&d_sf, sizeof(float4) * n_pad)); c->frame_allocs.push_back(d_sf);
      stage.resize(sizeof(float4) * n_pad);
      pack_records(true, pts[f], builds[f].order.data(), builds[f].order.data(), n, stage.data());
      pad_records(true, stage.data(), n, n_pad);
      CU(cudaMemcpy(d_sf, stage.data(), sizeof(float4) * n_pad, cudaMemcpyHostToDevice));
    }
    CU(cudaMalloc(&d_fc, sizeof(float) * builds[f].faces.size())); c->frame_allocs.push_back(d_fc);
    CU(cudaMemcpy(d_fc, builds[f].faces.data(), sizeof(float) * builds[f].faces.size(), cudaMemcpyHostToDevice));
    CU(cudaMalloc(&d_pos, sizeof(int32_t) * n)); c->frame_allocs.push_back(d_pos);
    CU(cudaMemcpy(d_pos, builds[f].pos_of.data(), sizeof(int32_t) * n, cudaMemcpyHostToDevice));
    CU(cudaMalloc(&d_adj, sizeof(int32_t) * builds[f].adj.size())); c->frame_allocs.push_back(d_adj);
    CU(cudaMemcpy(d_adj, builds[f].adj.data(), sizeof(int32_t) * builds[f].adj.size(), cudaMemcpyHostToDevice));
    c->h_frames[f] = FrameDev{d_o, d_n, nullptr, d_s, (const float4*)d_sf, (const Box*)d_b, (const float*)d_fc, (const int32_t*)d_pos,
                              (c->flags & MVICP_FLAG_NO_ADJ) ? nullptr : (const int32_t*)d_adj, (int32_t)n, builds[f].n_leaf_pad, builds[f].depth, builds[f].absmax};
  }
  c->last_lm_iters = 1 << 20;
  if (!(c->flags & MVICP_FLAG_NO_OBB)) {    // hybrid oriented boxes: a second node array for the far rounds (far.cuh)
    std::vector<ObbDev> ho(M);
    std::vector<std::vector<ObbHost>> obbs(M);
    {
      const unsigned hw = host_workers();
      std::vector<std::thread> pool; std::atomic<int> next{0};
      for (unsigned t = 0; t < std::min<unsigned>(hw, (unsigned)M); ++t)
        pool.emplace_back([&]() { for (int f; (f = next.fetch_add(1)) < M;) build_obb(pts[f], n_pts[f], builds[f], obbs[f]); });
      for (auto& th : pool) th.join();
    }
    static_assert(sizeof(ObbHost) == sizeof(ObbNode) && sizeof(ObbNode) == 64, "oriented node = 64 bytes");
    for (int f = 0; f < M; ++f) {
      void* d = nullptr;
      CU(cudaMalloc(&d, sizeof(ObbNode) * obbs[f].size())); c->frame_allocs.push_back(d);
      CU(cudaMemcpy(d, obbs[f].data(), sizeof(ObbNode) * obbs[f].size(), cudaMemcpyHostToDevice));
      ho[f] = ObbDev{(const ObbNode*)d};
    }
    RET(c->d_obb.reserve(sizeof(ObbDev) * M));
    CU(cudaMemcpy(c->d_obb.p, ho.data(), sizeof(ObbDev) * M, cudaMemcpyHostToDevice));
    c->obb_ready = true;
  }
  return finish_set_frames(c, M);
}
extern "C" {

int mvicp_set_frames(mvicp_ctx* c, int32_t M, const double* const* pts, const double* const* nor, const int64_t* n_pts) {
  return set_frames_impl(c, M, pts, nor, n_pts, false);
}

int mvicp_set_frames_device(mvicp_ctx* c, int32_t M, const double* const* pts, const double* const* nor, const int64_t* n_pts) {
  if (!c || M <= 0 || !pts || !n_pts) return fail(MVICP_ERR_INVALID, "mvicp_set_frames_device: bad arguments");
  CU(cudaSetDevice(c->device));
  for (int f = 0; f < M; ++f) {
    if (n_pts[f] <= 0 || !pts[f]) continue;   // the twin's own checks report these
    RET(check_device_ptr(c, pts[f], "mvicp_set_frames_device", "pts_xyz[f]"));
    if (nor && nor[f]) RET(check_device_ptr(c, nor[f], "mvicp_set_frames_device", "nor_xyz[f]"));
  }
  return set_frames_impl(c, M, pts, nor, n_pts, true);
}

int mvicp_set_poses(mvicp_ctx* c, const double* poses16, const uint8_t* fixed) {
  if (!c || !c->M || !poses16) return fail(MVICP_ERR_INVALID, "mvicp_set_poses: bad arguments / no frames");
  CU(cudaSetDevice(c->device));
  // poses other than the ones this context last handed out: what the previous LM solve said about convergence is void
  if (std::memcmp(c->h_poses.data(), poses16, sizeof(double) * 16 * c->M) != 0) c->last_lm_iters = 1 << 20;
  std::memcpy(c->h_poses.data(), poses16, sizeof(double) * 16 * c->M);
  CU(cudaMemcpyAsync(c->d_poses.p, c->h_poses.data(), sizeof(double) * 16 * c->M, cudaMemcpyHostToDevice, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  if (fixed && !std::equal(fixed, fixed + c->M, c->fixed.begin())) { c->fixed.assign(fixed, fixed + c->M); RET(refresh_after_fixed_change(c)); }
  // Non-rigid "isometries" (e.g. the reference's Bunny_RealData sample poses) give non-unit quaternions, on which the
  // reference's quaternion / SE3 functors keep running (no normalisation, so3.hpp:666-668): remember it, the LM step
  // then uses the general frame model.  Sticky until the next upload: a fixed frame keeps its non-unit quaternion.
  c->nonrigid = poses_nonrigid(poses16, c->M);
  return MVICP_OK;
}

int mvicp_get_poses(mvicp_ctx* c, double* poses16) {
  if (!c || !c->M || !poses16) return fail(MVICP_ERR_INVALID, "mvicp_get_poses: bad arguments / no frames");
  CU(cudaSetDevice(c->device));
  CU(cudaMemcpyAsync(c->h_poses.data(), c->d_poses.p, sizeof(double) * 16 * c->M, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  std::memcpy(poses16, c->h_poses.data(), sizeof(double) * 16 * c->M);
  return MVICP_OK;
}

// LM streaming tile length for this many active correspondence slots (edges of free src frames, over all ranks)
static int eval_tile_len_of(int64_t active_slots) {
  int tl = 8192;
  while (tl > 1024 && active_slots / tl < 8 * NUM_SMS) tl >>= 1;
  return tl;
}

// edge ownership, slot offsets and the tile lists of the NN / LM streaming kernels: depends on the graph, the cloud sizes, the
// fixed flags and the rank layout -- not on the correspondences, which keep their slots
static int layout_work(mvicp_ctx* c) {
  const int E = c->E;
  if (!E) return MVICP_OK;
  int64_t off = 0, owned_slots = 0;
  assign_edge_owners(c);
  for (int e = 0; e < E; ++e) {
    EdgeDev& ed = c->h_edges[e];
    ed.off = off; ed.n_src = (int32_t)c->n_pts[ed.src];
    ed.owned = c->edge_owner[e] == c->rank ? 1 : 0;   // fixed src: nobody (`if(this->fixed) return;` frame.cpp:93)
    off += ed.n_src;
    if (ed.owned) owned_slots += ed.n_src;
  }
  c->total_slots = off;
  // LM streaming tile: long enough to amortise the 28-value block reduction, short enough to fill the SMs.  Its length fixes how
  // an edge's sum is associated (per-tile partials, added in tile order), so it must not depend on how many ranks share the
  // work: it is chosen from ALL active slots, and a sharded run's poses stay bit-identical to the single-GPU run's
  // (bench.py checks that in every multi-GPU run; round 1 chose it from the rank's own share and was not).
  int64_t active_slots = 0;
  for (int e = 0; e < E; ++e) if (c->edge_owner[e] >= 0) active_slots += c->h_edges[e].n_src;
  const int tl = eval_tile_len_of(active_slots);
  c->eval_tile_len = tl;
  (void)owned_slots;
  std::vector<Tile> kt, et; std::vector<int32_t> etb(E + 1, 0);
  for (int e = 0; e < E; ++e) {
    const EdgeDev& ed = c->h_edges[e];
    etb[e] = (int32_t)et.size();
    if (!ed.owned) continue;
    for (int s = 0; s < ed.n_src; s += KNN_TILE) kt.push_back(Tile{e, s});
    for (int s = 0; s < ed.n_src; s += tl) et.push_back(Tile{e, s});
  }
  etb[E] = (int32_t)et.size();
  c->n_knn_tiles = (int)kt.size(); c->n_eval_tiles = (int)et.size();
  RET(c->d_edges.reserve(sizeof(EdgeDev) * E));
  RET(c->d_knn_tiles.reserve(sizeof(Tile) * std::max<size_t>(1, kt.size())));
  RET(c->d_eval_tiles.reserve(sizeof(Tile) * std::max<size_t>(1, et.size())));
  RET(c->d_edge_tile_begin.reserve(sizeof(int32_t) * (E + 1)));
  RET(c->d_partial.reserve(sizeof(double) * NBLK * std::max<size_t>(1, et.size())));
  CU(cudaMemcpy(c->d_edges.p, c->h_edges.data(), sizeof(EdgeDev) * E, cudaMemcpyHostToDevice));
  if (!kt.empty()) CU(cudaMemcpy(c->d_knn_tiles.p, kt.data(), sizeof(Tile) * kt.size(), cudaMemcpyHostToDevice));
  if (!et.empty()) CU(cudaMemcpy(c->d_eval_tiles.p, et.data(), sizeof(Tile) * et.size(), cudaMemcpyHostToDevice));
  CU(cudaMemcpy(c->d_edge_tile_begin.p, etb.data(), sizeof(int32_t) * (E + 1), cudaMemcpyHostToDevice));
  ++c->graph_gen;
  return MVICP_OK;
}

// (re)build tile lists and per-edge buffers, forgetting every correspondence; called by set_graph and comm_init
static int rebuild_work(mvicp_ctx* c) {
  const int E = c->E;
  if (!E) return MVICP_OK;
  RET(layout_work(c));
  const int64_t off = c->total_slots;
  RET(c->d_xf.reserve(sizeof(EdgeXf) * E));
  RET(c->d_corr.reserve(sizeof(int32_t) * off));
  RET(c->d_d2.reserve(sizeof(double) * off));
  RET(c->d_count.reserve(sizeof(unsigned long long) * E));
  RET(c->d_sel.reserve(sizeof(SelState) * E));
  RET(c->d_hist.reserve(sizeof(unsigned int) * SEL_BINS * (size_t)E));
  RET(c->d_weight.reserve(sizeof(float) * E));
  RET(c->d_median.reserve(sizeof(double) * E));
  RET(c->d_selcand.reserve(sizeof(unsigned long long) * SEL_CAP * (size_t)E));
  RET(c->d_selcand_n.reserve(sizeof(unsigned int) * E));
  RET(c->d_sel_cnt.reserve(sizeof(unsigned int) * (2 * (size_t)E + 1)));
  CU(cudaMemset(c->d_sel_cnt.p, 0, sizeof(unsigned int) * (2 * (size_t)E + 1)));
  RET(c->d_sel_win.reserve(sizeof(unsigned long long) * 3 * (size_t)E));
  RET(c->d_certs.reserve(sizeof(float4) * off));
  RET(c->d_todo.reserve(sizeof(int2) * off));
  RET(c->d_todo_n.reserve(sizeof(unsigned int)));
  CU(cudaMemset(c->d_todo_n.p, 0, sizeof(unsigned int)));
  RET(c->d_cert_cnt.reserve(sizeof(unsigned long long) * E));
  CU(cudaMemset(c->d_cert_cnt.p, 0, sizeof(unsigned long long) * E));
  c->cert_valid = false;
  c->sel_valid = false;
  CU(cudaMemset(c->d_hist.p, 0, sizeof(unsigned int) * SEL_BINS * (size_t)E));
  CU(cudaMemset(c->d_weight.p, 0, sizeof(float) * E));
  CU(cudaMemset(c->d_selcand_n.p, 0, sizeof(unsigned int) * E));
  CU(cudaMemset(c->d_count.p, 0, sizeof(unsigned long long) * E));
  CU(cudaMemset(c->d_corr.p, 0xff, sizeof(int32_t) * off));   // ~0 = "no inlier, candidate 0"
  c->h_weight.assign(E, 0.f); c->h_count.assign(E, 0ull);
  c->have_corr = false;
  return MVICP_OK;
}

// The fixed flags changed after the graph was laid out (mvicp_set_poses, or mvicp_optimize fixing frame 0 as every
// ceresOptimizer* does, icp-ceres.cpp:242-244): the reference keeps working with whatever correspondences exist and only skips
// the edges of fixed src frames (`if(srcCloud.fixed) continue;` icp-ceres.cpp:255,353,426).  On one GPU ownership is exactly
// "src is free", so the layout is refreshed and the correspondences stay; sharded, edges would change ranks: everything is
// laid out again and the next mvicp_correspond refills it.
static int refresh_after_fixed_change(mvicp_ctx* c) {
  if (!c->E) return MVICP_OK;
  CU(cudaStreamSynchronize(c->stream));
  return c->world > 1 ? rebuild_work(c) : layout_work(c);
}

int mvicp_set_graph(mvicp_ctx* c, int32_t E, const int32_t* src, const int32_t* dst) {
  if (!c || !c->M || E < 0 || (E && (!src || !dst))) return fail(MVICP_ERR_INVALID, "mvicp_set_graph: bad arguments / no frames");
  CU(cudaSetDevice(c->device));
  CU(cudaStreamSynchronize(c->stream));
  for (int e = 0; e < E; ++e)
    if (src[e] < 0 || src[e] >= c->M || dst[e] < 0 || dst[e] >= c->M || src[e] == dst[e])
      return fail(MVICP_ERR_INVALID, "edge %d: (%d -> %d) invalid", e, src[e], dst[e]);
  c->E = E; c->h_edges.assign(E, EdgeDev{}); c->lm_blocks_E = 0;
  for (int e = 0; e < E; ++e) { c->h_edges[e].src = src[e]; c->h_edges[e].dst = dst[e]; }
  return rebuild_work(c);
}

int mvicp_pose_graph_knn(mvicp_ctx* c, int32_t knn) {
  if (!c || !c->M || knn < 0) return fail(MVICP_ERR_INVALID, "mvicp_pose_graph_knn: bad arguments / no frames");
  // Frame::computePoseNeighboursKnn (frame.cpp:67-89): k frames with the smallest float |t_i - t_j|
  std::vector<int32_t> src, dst;
  for (int i = 0; i < c->M; ++i) {
    std::vector<std::pair<float, int>> nb;
    for (int j = 0; j < c->M; ++j) {
      if (i == j) continue;
      const double* a = &c->h_poses[16 * i + 12]; const double* b = &c->h_poses[16 * j + 12];
      const double d0 = a[0] - b[0], d1 = a[1] - b[1], d2 = a[2] - b[2];
      nb.push_back({(float)std::sqrt(d0 * d0 + d1 * d1 + d2 * d2), j});
    }
    std::stable_sort(nb.begin(), nb.end(), [](const std::pair<float, int>& x, const std::pair<float, int>& y) { return x.first < y.first; });
    for (int q = 0; q < knn && q < (int)nb.size(); ++q) { src.push_back(i); dst.push_back(nb[q].second); }
  }
  return mvicp_set_graph(c, (int32_t)src.size(), src.data(), dst.data());
}

int mvicp_get_graph(mvicp_ctx* c, int32_t* E, int32_t* src, int32_t* dst) {
  if (!c || !E) return fail(MVICP_ERR_INVALID, "mvicp_get_graph: bad arguments");
  *E = c->E;
  for (int e = 0; e < c->E; ++e) { if (src) src[e] = c->h_edges[e].src; if (dst) dst[e] = c->h_edges[e].dst; }
  return MVICP_OK;
}

}  // extern "C"
// sqrt(d2) < t  <=>  d2 <= the largest double whose correctly rounded square root is below t (sqrt is monotone, IEEE on both sides)
static double cutoff_d2max(float thresh) {
  const double t = (double)thresh;
  if (!(t > 0.0)) return -1.0;                  // nothing is an inlier (also for a NaN threshold)
  if (std::isinf(t)) return std::numeric_limits<double>::max();
  double x = t * t;
  while (x > 0.0 && !(std::sqrt(x) < t)) x = std::nextafter(x, 0.0);
  while (std::sqrt(std::nextafter(x, std::numeric_limits<double>::infinity())) < t) x = std::nextafter(x, std::numeric_limits<double>::infinity());
  return std::sqrt(x) < t ? x : -1.0;
}
template <bool F32> static int launch_correspond(mvicp_ctx* c, float thresh) {
  const int E = c->E;
  const double d2max = cutoff_d2max(thresh);
  const bool seed = c->have_corr && !(c->flags & MVICP_FLAG_NO_SEED);
  bool guess = false, far = false;
  int cert = 0;
  const bool ww = !(c->flags & MVICP_FLAG_STEP_LOOP);
  if (c->n_knn_tiles) {
    // Far rounds search the oriented-box node array (far.cuh): a round without seeds, and the first round that has them (its
    // seeds were found before the first LM solve moved the clouds by centimetres); from the second seeded round on the 64-byte
    // oriented boxes cost more than their tighter fit saves.  Poses set from outside since the last solve count as a fresh start.
    if (!seed || c->last_lm_iters == (1 << 20)) c->seeded_rounds = 0;
    far = c->obb_ready && (!seed || c->seeded_rounds < 1);
    if (seed) ++c->seeded_rounds;
    // A round that follows a one-iteration solve hardly moves anything: a window of keys around the previous median is a guess that
    // the NN kernel's epilogue can check on the fly, which replaces the three passes of the select (select.cuh) ...
    const bool steady = seed && !far && ww, converged = steady && c->last_lm_iters <= 1;
    guess = converged && c->sel_valid && !(c->flags & MVICP_FLAG_NO_SELECT_GUESS);
    // ... and most queries need no search at all: the previous search left a margin by which its match beats every other point,
    // and the query is still within half of it of where it was (knn.cuh, CERT).  Certificates are written by the rounds that lead up to that
    // (the previous solve took <= 3 iterations) and stay valid only while every round keeps them current.
    if (steady && !(c->flags & MVICP_FLAG_NO_CERT)) cert = (guess && c->cert_valid) ? 2 : (c->last_lm_iters <= 3 ? 1 : 0);
  }
  edge_xf_kernel<<<(E + 127) / 128, 128, 0, c->stream>>>(c->d_poses.as<double>(), c->d_edges.as<EdgeDev>(), E, c->d_xf.as<EdgeXf>());
  CU(cudaEventRecord(c->ev[0], c->stream));
  if (c->n_knn_tiles) {
    unsigned int* cnt = c->d_sel_cnt.as<unsigned int>();
    const SelGuess sg = {c->d_sel_win.as<unsigned long long>(), cnt, cnt + E, c->d_selcand.as<unsigned long long>(), c->d_selcand_n.as<unsigned int>()};
#define MV_KNN_ARGS c->d_frames.as<FrameDev>(), c->d_edges.as<EdgeDev>(), c->d_xf.as<EdgeXf>(), c->d_knn_tiles.as<Tile>(), \
                    c->d_corr.as<int32_t>(), c->d_d2.as<double>(), seed ? c->d_corr.as<int32_t>() : nullptr, d2max
#define MV_KNN_TAIL sg, E, c->d_certs.as<float4>()
    if (far) knn_far_kernel<F32><<<c->n_knn_tiles, KNN_TILE, 0, c->stream>>>(MV_KNN_ARGS, c->d_obb.as<ObbDev>());
    else if (cert == 2) {
      const CertTodo todo = {c->d_todo.as<int2>(), c->d_todo_n.as<unsigned int>()};
      knn_cert_kernel<F32><<<c->n_knn_tiles, KNN_TILE, 0, c->stream>>>(MV_KNN_ARGS, MV_KNN_TAIL, c->d_cert_cnt.as<unsigned long long>(), todo);
      knn_todo_kernel<F32><<<NUM_SMS * 5, KNN_TILE, 0, c->stream>>>(c->d_frames.as<FrameDev>(), c->d_edges.as<EdgeDev>(), c->d_xf.as<EdgeXf>(),
          c->d_corr.as<int32_t>(), c->d_d2.as<double>(), c->d_corr.as<int32_t>(), d2max, MV_KNN_TAIL, todo);
      c->stats.kernel_launches += 1;
    }
    else if (guess && cert == 1) knn_kernel<F32, true, true, 1><<<c->n_knn_tiles, KNN_TILE, 0, c->stream>>>(MV_KNN_ARGS, MV_KNN_TAIL);
    else if (guess) knn_kernel<F32, true, true, 0><<<c->n_knn_tiles, KNN_TILE, 0, c->stream>>>(MV_KNN_ARGS, MV_KNN_TAIL);
    else if (cert == 1) knn_kernel<F32, true, false, 1><<<c->n_knn_tiles, KNN_TILE, 0, c->stream>>>(MV_KNN_ARGS, MV_KNN_TAIL);
    else if (ww) knn_kernel<F32, true, false, 0><<<c->n_knn_tiles, KNN_TILE, 0, c->stream>>>(MV_KNN_ARGS, MV_KNN_TAIL);
    else knn_kernel<F32, false, false, 0><<<c->n_knn_tiles, KNN_TILE, 0, c->stream>>>(MV_KNN_ARGS, MV_KNN_TAIL);
    c->cert_valid = cert != 0;
    if (cert == 2) ++c->cert_rounds;
#undef MV_KNN_TAIL
#undef MV_KNN_ARGS
  }
  CU(cudaEventRecord(c->ev[1], c->stream));
  c->stats.kernel_launches += 1 + (c->n_knn_tiles ? 1 : 0);
  // exact median -> weight
  if (guess) {
    unsigned int* cnt = c->d_sel_cnt.as<unsigned int>();
    select_guess_finish_kernel<<<E, SEL_THREADS, 0, c->stream>>>(c->d_edges.as<EdgeDev>(), c->d_corr.as<int32_t>(), c->d_d2.as<double>(),
        c->d_sel.as<SelState>(), cnt, cnt + E, c->d_selcand.as<unsigned long long>(), c->d_selcand_n.as<unsigned int>(),
        c->d_weight.as<float>(), c->d_median.as<double>(), c->d_count.as<unsigned long long>(), c->d_sel_win.as<unsigned long long>(), cnt + 2 * (size_t)E,
        c->d_todo_n.as<unsigned int>());
    c->stats.kernel_launches += 1;
    ++c->sel_guess_rounds;
  } else {
  select_init_kernel<<<(E + 127) / 128, 128, 0, c->stream>>>(c->d_sel.as<SelState>(), E);
  c->stats.kernel_launches += 1;
  const int shifts[2] = {53, 42};
  for (int p = 0; p < 2; ++p) {
    if (c->n_eval_tiles)
      select_hist_kernel<<<c->n_eval_tiles, SEL_THREADS, 0, c->stream>>>(
          c->d_edges.as<EdgeDev>(), c->d_eval_tiles.as<Tile>(), c->eval_tile_len, c->d_corr.as<int32_t>(), c->d_d2.as<double>(),
          c->d_sel.as<SelState>(), shifts[p], 11, c->d_hist.as<unsigned int>());
    select_pick_kernel<<<E, SEL_THREADS, 0, c->stream>>>(c->d_sel.as<SelState>(), c->d_hist.as<unsigned int>(), shifts[p], p == 0, 0,
                                                         c->d_weight.as<float>(), c->d_median.as<double>(),
                                                         c->d_count.as<unsigned long long>());
    c->stats.kernel_launches += 1 + (c->n_eval_tiles ? 1 : 0);
  }
  if (c->n_eval_tiles)
    select_collect_kernel<<<c->n_eval_tiles, SEL_THREADS, 0, c->stream>>>(
        c->d_edges.as<EdgeDev>(), c->d_eval_tiles.as<Tile>(), c->eval_tile_len, c->d_corr.as<int32_t>(), c->d_d2.as<double>(),
        c->d_sel.as<SelState>(), c->d_selcand.as<unsigned long long>(), c->d_selcand_n.as<unsigned int>());
  select_finish_kernel<<<E, SEL_THREADS, 0, c->stream>>>(c->d_edges.as<EdgeDev>(), c->d_corr.as<int32_t>(), c->d_d2.as<double>(),
                                                         c->d_sel.as<SelState>(), c->d_selcand.as<unsigned long long>(),
                                                         c->d_selcand_n.as<unsigned int>(), c->d_weight.as<float>(), c->d_median.as<double>(),
                                                         c->d_sel_win.as<unsigned long long>());
  c->stats.kernel_launches += 1 + (c->n_eval_tiles ? 1 : 0);
  }
  c->sel_valid = true;
  CU(cudaEventRecord(c->ev[2], c->stream));
  CU(cudaGetLastError());
  return MVICP_OK;
}

extern "C" {
int mvicp_correspond(mvicp_ctx* c, float thresh) {
  if (!c || !c->M || !c->E) return fail(MVICP_ERR_STATE, "mvicp_correspond: frames and graph must be set first");
  CU(cudaSetDevice(c->device));
  RET(c->f32 ? launch_correspond<true>(c, thresh) : launch_correspond<false>(c, thresh));
  c->have_corr = true; c->ev_knn = true;
  int64_t q = 0; for (const EdgeDev& e : c->h_edges) if (e.owned) q += e.n_src;
  c->stats.queries = q;
  return MVICP_OK;
}

static int fetch_edge_meta(mvicp_ctx* c) {
  CU(cudaMemcpyAsync(c->h_weight.data(), c->d_weight.p, sizeof(float) * c->E, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaMemcpyAsync(c->h_count.data(), c->d_count.p, sizeof(unsigned long long) * c->E, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return MVICP_OK;
}

int mvicp_get_edge(mvicp_ctx* c, int32_t e, int32_t* first, int32_t* second, double* dist, int64_t* count, float* weight) {
  if (!c || e < 0 || e >= c->E) return fail(MVICP_ERR_INVALID, "mvicp_get_edge: bad edge");
  CU(cudaSetDevice(c->device));
  const EdgeDev& ed = c->h_edges[e];
  if (!ed.owned && !c->fixed[ed.src]) return fail(MVICP_ERR_NOT_OWNER, "edge %d is processed by rank %d", e, c->edge_owner[e]);
  RET(fetch_edge_meta(c));
  if (weight) *weight = c->h_weight[e];
  if (count) *count = (int64_t)c->h_count[e];
  if (first || second || dist) {
    std::vector<int32_t> corr(ed.n_src); std::vector<double> d2(ed.n_src);
    CU(cudaMemcpy(corr.data(), c->d_corr.as<int32_t>() + ed.off, sizeof(int32_t) * ed.n_src, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(d2.data(), c->d_d2.as<double>() + ed.off, sizeof(double) * ed.n_src, cudaMemcpyDeviceToHost));
    int64_t n = 0;
    for (int k = 0; k < ed.n_src; ++k)
      if (corr[k] >= 0) {
        if (first) first[n] = k;
        if (second) second[n] = corr[k];
        if (dist) dist[n] = std::sqrt(d2[k]);
        ++n;
      }
    if (count) *count = n;
  }
  return MVICP_OK;
}

// inliers per tile and their exclusive scan: d_tile_off (first record of every tile), d_edge_off (of every edge, [E] = total)
static int compact_count_scan(mvicp_ctx* c) {
  const int E = c->E, nt = c->n_knn_tiles;
  RET(c->d_tile_count.reserve(sizeof(unsigned int) * std::max(1, nt)));
  RET(c->d_tile_off.reserve(sizeof(unsigned long long) * std::max(1, nt)));
  RET(c->d_edge_off.reserve(sizeof(unsigned long long) * (E + 1)));
  if (nt) compact_count_kernel<<<nt, KNN_TILE, 0, c->stream>>>(c->d_edges.as<EdgeDev>(), c->d_knn_tiles.as<Tile>(), c->d_corr.as<int32_t>(), c->d_tile_count.as<unsigned int>());
  compact_scan_kernel<<<1, 1024, 0, c->stream>>>(c->d_tile_count.as<unsigned int>(), nt, c->d_knn_tiles.as<Tile>(), E,
                                                 c->d_tile_off.as<unsigned long long>(), c->d_edge_off.as<unsigned long long>());
  c->stats.kernel_launches += nt ? 2 : 1;
  return MVICP_OK;
}

int mvicp_get_all_edges(mvicp_ctx* c, void* out_records, int64_t capacity, int64_t* offsets, float* weights) {
  if (!c || !c->E || !offsets) return fail(MVICP_ERR_INVALID, "mvicp_get_all_edges: bad arguments / no graph");
  if (!c->have_corr) return fail(MVICP_ERR_STATE, "mvicp_get_all_edges: call mvicp_correspond first");
  CU(cudaSetDevice(c->device));
  const int E = c->E, nt = c->n_knn_tiles;
  RET(compact_count_scan(c));
  std::vector<unsigned long long> eo(E + 1);
  CU(cudaMemcpyAsync(eo.data(), c->d_edge_off.p, sizeof(unsigned long long) * (E + 1), cudaMemcpyDeviceToHost, c->stream));
  if (weights) CU(cudaMemcpyAsync(weights, c->d_weight.p, sizeof(float) * E, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  for (int e = 0; e <= E; ++e) offsets[e] = (int64_t)eo[e];
  if (out_records) {
    const int64_t total = (int64_t)eo[E];
    if (total > capacity) return fail(MVICP_ERR_INVALID, "mvicp_get_all_edges: %lld records, capacity %lld", (long long)total, (long long)capacity);
    if (total) {
      RET(c->d_recs.reserve(sizeof(CorrRec) * (size_t)total));
      compact_scatter_kernel<<<nt, KNN_TILE, 0, c->stream>>>(c->d_edges.as<EdgeDev>(), c->d_knn_tiles.as<Tile>(), c->d_corr.as<int32_t>(), c->d_d2.as<double>(),
                                                             c->d_tile_off.as<unsigned long long>(), c->d_recs.as<CorrRec>());
      c->stats.kernel_launches += 1;
      CU(cudaMemcpyAsync(out_records, c->d_recs.p, sizeof(CorrRec) * (size_t)total, cudaMemcpyDeviceToHost, c->stream));
      CU(cudaStreamSynchronize(c->stream));
    }
  }
  CU(cudaGetLastError());
  return MVICP_OK;
}

// The same three compaction kernels, writing straight into the caller's device buffer; offsets and weights are device-to-device
// copies.  Nothing waits for the device: the capacity is checked up front against what the kernels may write at most.
int mvicp_get_all_edges_device(mvicp_ctx* c, void* out_records, int64_t capacity, int64_t* offsets, float* weights) {
  if (!c || !c->E || !offsets) return fail(MVICP_ERR_INVALID, "mvicp_get_all_edges_device: bad arguments / no graph");
  if (!c->have_corr) return fail(MVICP_ERR_STATE, "mvicp_get_all_edges_device: call mvicp_correspond first");
  CU(cudaSetDevice(c->device));
  RET(check_device_ptr(c, offsets, "mvicp_get_all_edges_device", "offsets"));
  if (out_records) RET(check_device_ptr(c, out_records, "mvicp_get_all_edges_device", "out_records"));
  if (weights) RET(check_device_ptr(c, weights, "mvicp_get_all_edges_device", "weights"));
  const int E = c->E, nt = c->n_knn_tiles;
  if (out_records) {
    int64_t bound = 0;
    for (const EdgeDev& ed : c->h_edges) if (ed.owned) bound += ed.n_src;
    if (capacity < bound)
      return fail(MVICP_ERR_INVALID, "mvicp_get_all_edges_device: up to %lld records, capacity %lld", (long long)bound, (long long)capacity);
  }
  RET(compact_count_scan(c));
  static_assert(sizeof(unsigned long long) == sizeof(int64_t), "offsets are copied as they are");
  CU(cudaMemcpyAsync(offsets, c->d_edge_off.p, sizeof(int64_t) * (E + 1), cudaMemcpyDeviceToDevice, c->stream));
  if (weights) CU(cudaMemcpyAsync(weights, c->d_weight.p, sizeof(float) * E, cudaMemcpyDeviceToDevice, c->stream));
  if (out_records && nt) {
    compact_scatter_kernel<<<nt, KNN_TILE, 0, c->stream>>>(c->d_edges.as<EdgeDev>(), c->d_knn_tiles.as<Tile>(), c->d_corr.as<int32_t>(), c->d_d2.as<double>(),
                                                           c->d_tile_off.as<unsigned long long>(), reinterpret_cast<CorrRec*>(out_records));
    c->stats.kernel_launches += 1;
  }
  CU(cudaGetLastError());
  return MVICP_OK;
}

int mvicp_host_alloc(size_t bytes, void** out) {
  if (!out) return fail(MVICP_ERR_INVALID, "mvicp_host_alloc: bad arguments");
  *out = nullptr;
  if (!bytes) return MVICP_OK;
  CU(cudaHostAlloc(out, bytes, cudaHostAllocPortable));
  return MVICP_OK;
}
int mvicp_host_free(void* p) {
  if (p) CU(cudaFreeHost(p));
  return MVICP_OK;
}

int mvicp_get_nn(mvicp_ctx* c, int32_t e, int32_t* nn_idx, double* nn_d2) {
  if (!c || e < 0 || e >= c->E) return fail(MVICP_ERR_INVALID, "mvicp_get_nn: bad edge");
  CU(cudaSetDevice(c->device));
  const EdgeDev& ed = c->h_edges[e];
  if (!ed.owned) return fail(MVICP_ERR_NOT_OWNER, "edge %d is not processed by this rank", e);
  CU(cudaStreamSynchronize(c->stream));
  if (nn_idx) {
    CU(cudaMemcpy(nn_idx, c->d_corr.as<int32_t>() + ed.off, sizeof(int32_t) * ed.n_src, cudaMemcpyDeviceToHost));
    for (int k = 0; k < ed.n_src; ++k) if (nn_idx[k] < 0) nn_idx[k] = ~nn_idx[k];
  }
  if (nn_d2) CU(cudaMemcpy(nn_d2, c->d_d2.as<double>() + ed.off, sizeof(double) * ed.n_src, cudaMemcpyDeviceToHost));
  return MVICP_OK;
}

int mvicp_set_edge(mvicp_ctx* c, int32_t e, const int32_t* first, const int32_t* second, int64_t count, float weight) {
  if (!c || e < 0 || e >= c->E || count < 0 || (count && (!first || !second))) return fail(MVICP_ERR_INVALID, "mvicp_set_edge: bad arguments");
  CU(cudaSetDevice(c->device));
  const EdgeDev& ed = c->h_edges[e];
  std::vector<int32_t> corr(ed.n_src, ~0);
  const int n_dst = (int)c->n_pts[ed.dst];
  for (int64_t i = 0; i < count; ++i) {
    if (first[i] < 0 || first[i] >= ed.n_src || second[i] < 0 || second[i] >= n_dst) return fail(MVICP_ERR_INVALID, "mvicp_set_edge: index out of range at %lld", (long long)i);
    corr[first[i]] = second[i];
  }
  CU(cudaStreamSynchronize(c->stream));
  CU(cudaMemcpy(c->d_corr.as<int32_t>() + ed.off, corr.data(), sizeof(int32_t) * ed.n_src, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(c->d_weight.as<float>() + e, &weight, sizeof(float), cudaMemcpyHostToDevice));
  const unsigned long long cnt = (unsigned long long)count;
  CU(cudaMemcpy(c->d_count.as<unsigned long long>() + e, &cnt, sizeof cnt, cudaMemcpyHostToDevice));
  c->cert_valid = false;   // the matches in d_corr are no longer the ones the certificates were written for
  return MVICP_OK;
}

// mvicp_set_edge with first / second in device memory: range check + last-occurrence winner per slot, then the write, which the
// device skips when the check failed; one readback of the check, after which the caller's arrays have been read
int mvicp_set_edge_device(mvicp_ctx* c, int32_t e, const int32_t* first, const int32_t* second, int64_t count, float weight) {
  if (!c || e < 0 || e >= c->E || count < 0 || (count && (!first || !second))) return fail(MVICP_ERR_INVALID, "mvicp_set_edge_device: bad arguments");
  CU(cudaSetDevice(c->device));
  if (count) {
    RET(check_device_ptr(c, first, "mvicp_set_edge_device", "first"));
    RET(check_device_ptr(c, second, "mvicp_set_edge_device", "second"));
  }
  const EdgeDev& ed = c->h_edges[e];
  const int n_dst = (int)c->n_pts[ed.dst];
  RET(c->d_set_win.reserve(sizeof(unsigned long long) * (size_t)std::max(1, ed.n_src)));
  RET(c->d_set_bad.reserve(sizeof(unsigned long long)));
  unsigned long long* win = c->d_set_win.as<unsigned long long>();
  unsigned long long* bad = c->d_set_bad.as<unsigned long long>();
  CU(cudaMemsetAsync(win, 0, sizeof(unsigned long long) * (size_t)ed.n_src, c->stream));
  CU(cudaMemsetAsync(bad, 0xff, sizeof(unsigned long long), c->stream));
  if (count) {
    const int grid = (int)std::min<int64_t>((count + 255) / 256, 8 * NUM_SMS);
    set_edge_scan_kernel<<<grid, 256, 0, c->stream>>>(first, second, (long long)count, ed.n_src, n_dst, win, bad);
    c->stats.kernel_launches += 1;
  }
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((ed.n_src + 255) / 256, 8 * NUM_SMS));
  set_edge_write_kernel<<<grid, 256, 0, c->stream>>>(second, win, ed.n_src, bad, c->d_corr.as<int32_t>() + ed.off, c->d_weight.as<float>() + e,
                                                     c->d_count.as<unsigned long long>() + e, weight, (unsigned long long)count);
  c->stats.kernel_launches += 1;
  unsigned long long h_bad = 0;
  CU(cudaMemcpyAsync(&h_bad, bad, sizeof h_bad, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  CU(cudaGetLastError());
  if (h_bad != ~0ull) return fail(MVICP_ERR_INVALID, "mvicp_set_edge_device: index out of range at %lld", (long long)h_bad);
  c->cert_valid = false;   // as mvicp_set_edge
  return MVICP_OK;
}

int mvicp_closest_point(mvicp_ctx* c, int32_t frame, const double q[3], int64_t* idx, double* d2) {
  if (!c || frame < 0 || frame >= c->M || !q) return fail(MVICP_ERR_INVALID, "mvicp_closest_point: bad arguments");
  CU(cudaSetDevice(c->device));
  long long* d_i = c->d_single.as<long long>(); double* d_d = c->d_single.as<double>() + 1;
  if (c->f32) knn_single_kernel<true><<<1, 1, 0, c->stream>>>(c->d_frames.as<FrameDev>(), frame, q[0], q[1], q[2], d_i, d_d);
  else knn_single_kernel<false><<<1, 1, 0, c->stream>>>(c->d_frames.as<FrameDev>(), frame, q[0], q[1], q[2], d_i, d_d);
  c->stats.kernel_launches += 1;
  long long hi = 0; double hd = 0;
  CU(cudaMemcpyAsync(&hi, d_i, 8, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaMemcpyAsync(&hd, d_d, 8, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  if (idx) *idx = hi;
  if (d2) *d2 = hd;
  return MVICP_OK;
}

}  // extern "C"
static int launch_closest_points(mvicp_ctx* c, int frame, const double* q, int64_t n, long long* idx, double* d2) {
  const int grid = (int)std::min<int64_t>((n + 127) / 128, 64 * NUM_SMS);
  if (c->f32) closest_points_kernel<true><<<grid, 128, 0, c->stream>>>(c->d_frames.as<FrameDev>(), frame, q, (long long)n, idx, d2);
  else closest_points_kernel<false><<<grid, 128, 0, c->stream>>>(c->d_frames.as<FrameDev>(), frame, q, (long long)n, idx, d2);
  c->stats.kernel_launches += 1;
  CU(cudaGetLastError());
  return MVICP_OK;
}
extern "C" {

// mvicp_closest_point for n queries at once: the queries go up through the context's buffers, the results come back
int mvicp_closest_points(mvicp_ctx* c, int32_t frame, const double* q, int64_t n, int64_t* idx, double* d2) {
  if (!c || frame < 0 || frame >= c->M || n < 0 || (n && !q)) return fail(MVICP_ERR_INVALID, "mvicp_closest_points: bad arguments");
  if (!n) return MVICP_OK;
  CU(cudaSetDevice(c->device));
  RET(c->d_cpq.reserve(sizeof(double) * 3 * (size_t)n));
  RET(c->d_cpr.reserve(16 * (size_t)n));
  long long* d_i = c->d_cpr.as<long long>(); double* d_d = c->d_cpr.as<double>() + n;
  CU(cudaMemcpyAsync(c->d_cpq.p, q, sizeof(double) * 3 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
  RET(launch_closest_points(c, frame, c->d_cpq.as<double>(), n, d_i, d_d));
  if (idx) CU(cudaMemcpyAsync(idx, d_i, sizeof(int64_t) * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
  if (d2) CU(cudaMemcpyAsync(d2, d_d, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return MVICP_OK;
}

int mvicp_closest_points_device(mvicp_ctx* c, int32_t frame, const double* q, int64_t n, int64_t* idx, double* d2) {
  if (!c || frame < 0 || frame >= c->M || n < 0 || (n && !q)) return fail(MVICP_ERR_INVALID, "mvicp_closest_points_device: bad arguments");
  if (!n) return MVICP_OK;
  CU(cudaSetDevice(c->device));
  RET(check_device_ptr(c, q, "mvicp_closest_points_device", "q_xyz"));
  if (idx) RET(check_device_ptr(c, idx, "mvicp_closest_points_device", "idx"));
  if (d2) RET(check_device_ptr(c, d2, "mvicp_closest_points_device", "d2"));
  return launch_closest_points(c, frame, q, n, reinterpret_cast<long long*>(idx), d2);
}

// ---- the normal-equation layout and the host loop shared by both solvers (lm_step.cuh NormalLayout) -----------------
// Block structure of the normal matrix over the local columns c->h_col (n of them): edge e, when active[e], puts its pair
// matrix's ss / sk / ks / kk sub-blocks into blocks (s, s) / (s, k) / (k, s) / (k, k) and its (e, side) pair gradient into frame
// s's / k's gradient, wherever those ends have a column.  Uploads the gather lists, the envelope and the skyline layout of the
// factor, and zeroes the dense normal matrix.
//
// plan_normal_layout is the host half for one problem: `frames` (ascending) are its frames, local frame i being frames[i], and
// `edges` its edges in graph order; hcol holds the local columns (n of them).  The gather lists name graph edges.
struct LayoutPlan {
  std::vector<int32_t> col, hb_ptr{0}, hb_row, hb_col, hc_edge, hc_sub, gb_ptr{0}, gc_edge, gc_side, rlast, rfirst, rowbase;
  int64_t l_size = 0;        // doubles of the factor's skyline storage (row profiles + rhs row)
};
static int plan_normal_layout(const mvicp_ctx* c, const std::vector<int32_t>& hcol, const std::vector<int32_t>& frames,
                              const std::vector<int32_t>& edges, int n, const std::vector<uint8_t>& active, LayoutPlan& p) {
  const int M = (int)frames.size();
  std::vector<int32_t> loc(c->M, -1);
  for (int i = 0; i < M; ++i) loc[frames[i]] = i;
  std::vector<std::vector<std::pair<int, int>>> blk((size_t)M * M), gl(M);
  for (const int e : edges) {
    if (!active[e]) continue;
    const int s = loc[c->h_edges[e].src], k = loc[c->h_edges[e].dst];
    const bool fs = hcol[frames[s]] >= 0, fk = hcol[frames[k]] >= 0;
    if (fs) { blk[(size_t)s * M + s].push_back({e, 0}); gl[s].push_back({e, 0}); }
    if (fs && fk) { blk[(size_t)s * M + k].push_back({e, 1}); blk[(size_t)k * M + s].push_back({e, 2}); }
    if (fk) { blk[(size_t)k * M + k].push_back({e, 3}); gl[k].push_back({e, 1}); }
  }
  p.col.resize(M);
  for (int i = 0; i < M; ++i) p.col[i] = hcol[frames[i]];
  for (int r = 0; r < M; ++r)
    for (int q = 0; q < M; ++q) {
      const auto& l = blk[(size_t)r * M + q];
      if (l.empty()) continue;
      p.hb_row.push_back(p.col[r]); p.hb_col.push_back(p.col[q]);
      for (auto& pr : l) { p.hc_edge.push_back(pr.first); p.hc_sub.push_back(pr.second); }
      p.hb_ptr.push_back((int32_t)p.hc_edge.size());
    }
  for (int f = 0; f < M; ++f) { for (auto& pr : gl[f]) { p.gc_edge.push_back(pr.first); p.gc_side.push_back(pr.second); } p.gb_ptr.push_back((int32_t)p.gc_edge.size()); }
  const int n_hblocks = (int)p.hb_row.size();
  // envelope: first structurally non-zero column of every row, and the last row that reaches column j
  std::vector<int32_t>& rfirst = p.rfirst; std::vector<int32_t>& rlast = p.rlast;
  rfirst.resize(n); rlast.resize(n);
  for (int r = 0; r < n; ++r) rfirst[r] = (r / 6) * 6;
  for (int b = 0; b < n_hblocks; ++b)
    if (p.hb_col[b] < p.hb_row[b]) for (int i = 0; i < 6; ++i) rfirst[p.hb_row[b] + i] = std::min(rfirst[p.hb_row[b] + i], p.hb_col[b]);
  for (int j = 0; j < n; ++j) { rlast[j] = j; }
  for (int r = 0; r < n; ++r) for (int j = rfirst[r]; j <= r; ++j) rlast[j] = std::max(rlast[j], r);
  for (int j = 1; j < n; ++j) rlast[j] = std::max(rlast[j], rlast[j - 1]);   // monotone (fill-in stays inside)
  // skyline storage of the Cholesky factor: row r keeps columns rfirst[r]..r, the rhs row all n
  p.rowbase.resize(n + 1); int64_t at = 0;
  for (int r = 0; r < n; ++r) { p.rowbase[r] = (int32_t)(at - rfirst[r]); at += r - rfirst[r] + 1; }
  p.rowbase[n] = (int32_t)at; at += n;
  if (at > INT32_MAX) return fail(MVICP_ERR_INVALID, "normal matrix too large");
  p.l_size = at;
  return MVICP_OK;
}

// The LM problems, problem q over frames[q] and edges[q] with the local columns in hcol, laid out by plan_normal_layout and
// uploaded end to end into pb: one int32 buffer (frame and edge lists, gather lists, envelopes, skylines, then the edge -> problem
// map), one fp64 buffer (per problem H, Hc | g, gc, scale, diag, step, rhs | factor; Sigma n^2, not (Sigma n)^2), the LmProblem
// views, room for P + 1 states ([P]: the whole graph, for lm_init_kernel), the step kernel's ticket and the pair matrices' buffer
// d_eout.  `key` names what was uploaded.
static int upload_problems(mvicp_ctx* c, ProblemBufs& pb, const std::vector<int32_t>& hcol, const std::vector<std::vector<int32_t>>& frames,
                           const std::vector<std::vector<int32_t>>& edges, const std::vector<uint8_t>& active, const std::vector<uint8_t>& key) {
  const int P = (int)frames.size(), E = c->E;
  pb.key.clear();   // the buffers below change before the new views are complete
  std::vector<LayoutPlan> plans(P); std::vector<int> ns(P, 0);
  for (int q = 0; q < P; ++q) {
    for (int f : frames[q]) if (hcol[f] >= 0) ns[q] += 6;
    RET(plan_normal_layout(c, hcol, frames[q], edges[q], ns[q], active, plans[q]));
  }
  std::vector<int32_t> blob;
  auto put = [&](const std::vector<int32_t>& v) { const size_t o = blob.size(); blob.insert(blob.end(), v.begin(), v.end()); return o; };
  struct Off { size_t frame, edge, col, hb_ptr, hb_row, hb_col, hc_edge, hc_sub, gb_ptr, gc_edge, gc_side, rlast, rfirst, rowbase; };
  std::vector<Off> io(P);
  for (int q = 0; q < P; ++q) {
    const LayoutPlan& pl = plans[q];
    io[q] = Off{put(frames[q]), put(edges[q]), put(pl.col), put(pl.hb_ptr), put(pl.hb_row), put(pl.hb_col), put(pl.hc_edge), put(pl.hc_sub),
                put(pl.gb_ptr), put(pl.gc_edge), put(pl.gc_side), put(pl.rlast), put(pl.rfirst), put(pl.rowbase)};
  }
  std::vector<int32_t> prob_of_edge(E, -1);
  for (int q = 0; q < P; ++q) for (int e : edges[q]) prob_of_edge[e] = q;
  const size_t edge_map = put(prob_of_edge);
  std::vector<size_t> fo(P + 1, 0);
  for (int q = 0; q < P; ++q) { const size_t n = ns[q]; fo[q + 1] = fo[q] + 2 * n * n + 6 * n + (size_t)plans[q].l_size; }
  RET(pb.i32.reserve(sizeof(int32_t) * blob.size()));
  RET(pb.f64.reserve(sizeof(double) * fo[P]));
  RET(pb.prob.reserve(sizeof(LmProblem) * P));
  RET(pb.state.reserve(sizeof(LmState) * (P + 1)));
  RET(c->d_lm_ticket.reserve(sizeof(unsigned int)));
  RET(c->d_eout.reserve(sizeof(double) * EOUT * E));
  if (c->h_state_cap < (size_t)P + 1) {
    if (c->h_state) CU(cudaFreeHost(c->h_state));
    c->h_state = nullptr; c->h_state_cap = 0;
    CU(cudaMallocHost(&c->h_state, sizeof(LmState) * (P + 1)));
    c->h_state_cap = P + 1;
  }
  const int32_t* ib = pb.i32.as<int32_t>();
  std::vector<LmProblem> probs(P);
  size_t dyn = 0;
  for (int q = 0; q < P; ++q) {
    const int n = ns[q]; const Off& o = io[q];
    LmProblem& p = probs[q];
    std::memset(&p, 0, sizeof p);
    p.S = pb.state.as<LmState>() + q;
    p.frame = ib + o.frame; p.edge = ib + o.edge;
    NormalLayout& l = p.lay;
    l.col = ib + o.col;
    l.hb_ptr = ib + o.hb_ptr; l.hb_row = ib + o.hb_row; l.hb_col = ib + o.hb_col; l.hc_edge = ib + o.hc_edge; l.hc_sub = ib + o.hc_sub;
    l.n_hblocks = (int32_t)plans[q].hb_row.size();
    l.gb_ptr = ib + o.gb_ptr; l.gc_edge = ib + o.gc_edge; l.gc_side = ib + o.gc_side;
    l.rlast = ib + o.rlast; l.rfirst = ib + o.rfirst; l.rowbase = ib + o.rowbase;
    double* d = pb.f64.as<double>() + fo[q];
    p.H = d; d += (size_t)n * n; p.Hc = d; d += (size_t)n * n;
    p.g = d; d += n; p.gc = d; d += n; p.scale = d; d += n; p.diag = d; d += n; p.step = d; d += n; l.rhs = d; d += n;
    l.Lg = d;
    // the factor stays in shared memory when it fits with its vectors (colj, dg: 3 (n + 1) doubles); else this problem alone
    // factors in global memory
    const size_t vec = sizeof(double) * 3 * (size_t)(n + 1), lb = sizeof(double) * (size_t)plans[q].l_size;
    l.l_in_smem = lb + vec <= 220 * 1024 ? 1 : 0;
    dyn = std::max(dyn, vec + (l.l_in_smem ? lb : 0));
  }
  CU(cudaMemcpyAsync(pb.i32.p, blob.data(), sizeof(int32_t) * blob.size(), cudaMemcpyHostToDevice, c->stream));
  CU(cudaMemcpyAsync(pb.prob.p, probs.data(), sizeof(LmProblem) * P, cudaMemcpyHostToDevice, c->stream));
  // the step kernels write only the listed blocks of H and Hc; everything else stays zero from here
  CU(cudaMemsetAsync(pb.f64.p, 0, sizeof(double) * fo[P], c->stream));
  CU(cudaMemsetAsync(c->d_lm_ticket.p, 0, sizeof(unsigned int), c->stream));
  CU(cudaStreamSynchronize(c->stream));   // the host vectors above must outlive their copies
  pb.h_prob = std::move(probs); pb.edge_prob = ib + edge_map; pb.dyn = dyn; pb.key = key;
  return MVICP_OK;
}
}  // extern "C"
// What one streaming evaluation reads and writes besides the frames, edges and correspondences: the tiles, the evaluation point
// (per-frame Rt for the unit path, FrameGen for the general one) and the per-tile partials.  The solves use the context's own
// (lm_eval_args); mvicp_covariance brings its own.
struct EvalArgs { const Tile* tiles; int nt, tile_len; const Rt* Rt_; const FrameGen* gen; double* partial; };
static EvalArgs lm_eval_args(mvicp_ctx* c) {
  return EvalArgs{c->d_eval_tiles.as<Tile>(), c->n_eval_tiles, c->eval_tile_len, c->d_Rt.as<Rt>(), c->d_gen.as<FrameGen>(), c->d_partial.as<double>()};
}
template <bool F32> static void launch_eval(mvicp_ctx* c, const EvalArgs& a, int cost, int robust, DoneGate gate) {
  const int nt = a.nt;
  if (!nt) return;
#define MV_EVAL(NF, COSTK)                                                                                       \
  lm_eval_kernel<F32, NF, COSTK><<<nt, EVAL_THREADS, 0, c->stream>>>(                                            \
      c->d_frames.as<FrameDev>(), c->d_edges.as<EdgeDev>(), a.tiles, a.tile_len,                                \
      c->d_corr.as<int32_t>(), a.Rt_, c->d_weight.as<float>(), robust, a.partial, gate)
#define MV_EVALC(NF) { if (cost == COST_P2P) MV_EVAL(NF, COST_P2P); else if (cost == COST_P2PLANE) MV_EVAL(NF, COST_P2PLANE); else MV_EVAL(NF, COST_MIXED); }
  if (F32 && c->nor_f32) MV_EVALC(F32) else MV_EVALC(false)
#undef MV_EVALC
#undef MV_EVAL
}

template <bool F32> static void launch_eval_general(mvicp_ctx* c, const EvalArgs& a, int param, int cost, int robust, DoneGate gate) {
  const int rot0 = param == PARAM_QUAT ? 0 : 3;   // tangent order: quaternion (rotation, translation), SE3 (translation, rotation)
  const int nt = a.nt;
  if (!nt) return;
#define MV_EVALG(COSTK)                                                                                          \
  if (F32 && c->nor_f32) lm_eval_general_kernel<F32, F32, COSTK><<<nt, EVAL_THREADS, 0, c->stream>>>(        \
      c->d_frames.as<FrameDev>(), c->d_edges.as<EdgeDev>(), a.tiles, a.tile_len,                                \
      c->d_corr.as<int32_t>(), a.gen, c->d_weight.as<float>(), robust, rot0, a.partial, gate);                   \
  else lm_eval_general_kernel<F32, false, COSTK><<<nt, EVAL_THREADS, 0, c->stream>>>(                        \
      c->d_frames.as<FrameDev>(), c->d_edges.as<EdgeDev>(), a.tiles, a.tile_len,                                \
      c->d_corr.as<int32_t>(), a.gen, c->d_weight.as<float>(), robust, rot0, a.partial, gate)
  if (cost == COST_P2P) { MV_EVALG(COST_P2P); } else if (cost == COST_P2PLANE) { MV_EVALG(COST_P2PLANE); } else { MV_EVALG(COST_MIXED); }
#undef MV_EVALG
}

// The pipelined loop of both solvers: evaluation i+1 is enqueued before the host learns whether step i finished the solve,
// so the GPU never waits for the host; kernels issued after termination exit at once.  `eval()` enqueues the streaming
// evaluation (timed by a pair of events), `step(dyn)` the rest of the iteration, ending with the step kernel `kernel` (dynamic
// shared memory `dyn`, from upload_problems), which publishes (seq << 1) | done into the mapped ring.
template <typename Kernel, typename Eval, typename Step>
static int run_steps(mvicp_ctx* c, Kernel kernel, size_t dyn, int64_t max_evals, const char* what, int32_t& seq, Eval&& eval, Step&& step) {
  CU(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  for (int i = 0; i < 8; ++i) c->h_flag[i] = 0;
  c->eval_ev_used = 0;
  int64_t issued = 0, seen = 0;
  auto issue = [&]() -> int {
    if ((int)c->eval_ev.size() < c->eval_ev_used + 2) { cudaEvent_t a, b; CU(cudaEventCreate(&a)); CU(cudaEventCreate(&b)); c->eval_ev.push_back(a); c->eval_ev.push_back(b); }
    CU(cudaEventRecord(c->eval_ev[c->eval_ev_used], c->stream));
    eval();
    CU(cudaEventRecord(c->eval_ev[c->eval_ev_used + 1], c->stream));
    c->eval_ev_used += 2;
    seq = (int32_t)(issued + 1);
    RET(step(dyn));
    ++issued;
    return MVICP_OK;
  };
  RET(issue());
  while (true) {
    if (issued - seen < 2 && issued <= max_evals) RET(issue());
    // the step kernel publishes (sequence << 1 | done) into mapped pinned memory: spin on it, no stream round trip
    const int32_t want = (int32_t)(seen + 1);
    int32_t v;
    long spins = 0;
    while (((v = c->h_flag[want & 7]) >> 1) != want) {
      if ((++spins & 0xfffff) == 0 && cudaStreamQuery(c->stream) != cudaErrorNotReady) {   // kernels died or stream drained
        v = c->h_flag[want & 7];
        if ((v >> 1) != want) { CU(cudaGetLastError()); return fail(MVICP_ERR_CUDA, "%s step %d never reported", what, want); }
        break;
      }
    }
    ++seen;
    if ((v & 1) != 0 || seen > max_evals) break;
  }
  return MVICP_OK;
}

// End of a solve: the solver state and every pose back to the host.  The host pose mirror follows the device:
// mvicp_pose_graph_knn and mvicp_set_poses' "same poses as last handed out" test read it.
static int read_back_solve(mvicp_ctx* c, void* state, const void* d_state, size_t bytes) {
  CU(cudaEventRecord(c->ev[4], c->stream));
  CU(cudaMemcpyAsync(state, d_state, bytes, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaMemcpyAsync(c->h_poses.data(), c->d_poses.p, sizeof(double) * 16 * c->M, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  CU(cudaGetLastError());
  c->ev_lm = true;
  return MVICP_OK;
}

// Edge ownership follows the fixed flags (a fixed src frame's edges belong to nobody): refresh the layout when a solve has
// just fixed frame 0 (frames[0]->fixed = true, icp-ceres.cpp:242-244, icp-g2o.cpp:182-186) or mvicp_set_poses changed them.
static int refresh_if_fixed_changed(mvicp_ctx* c) {
  bool stale = false;
  for (int e = 0; e < c->E; ++e) if ((c->edge_owner[e] < 0) != (c->fixed[c->h_edges[e].src] != 0)) stale = true;
  if (!stale) return MVICP_OK;
  if (c->world > 1) return fail(MVICP_ERR_STATE, "sharded run: frame 0 was free when the edges were distributed; fix it (mvicp_set_poses) before mvicp_correspond");
  return refresh_after_fixed_change(c);
}

// The two-frame problem of mvicp_pairwise*: frame 0 = dst (fixed at the identity), frame 1 = src (from the identity), edge
// 1 -> 0 with identity matches.  Runs `solve(c)` on it, copies pose 1 out and destroys the context, keeping the error text.
template <typename Solve>
static int run_pairwise(const mvicp_config* cfg, const double* src, const double* dst, const double* nor, int64_t n, double* pose16_out,
                        Solve&& solve) {
  mvicp_ctx* c = nullptr;
  RET(mvicp_create(cfg, &c));
  const double* pts[2] = {dst, src}; const double* nrs[2] = {nor, nor};   // src normals are never read
  const int64_t np[2] = {n, n};
  int rc = mvicp_set_frames(c, 2, pts, nor ? nrs : nullptr, np);
  const int32_t es = 1, ed = 0;
  if (rc == MVICP_OK) rc = mvicp_set_graph(c, 1, &es, &ed);
  if (rc == MVICP_OK) {
    std::vector<int32_t> id(n); std::iota(id.begin(), id.end(), 0);
    rc = mvicp_set_edge(c, 0, id.data(), id.data(), n, 1.0f);
  }
  if (rc == MVICP_OK) rc = solve(c);
  std::vector<double> poses(32);
  if (rc == MVICP_OK) rc = mvicp_get_poses(c, poses.data());
  if (rc == MVICP_OK) std::memcpy(pose16_out, poses.data() + 16, sizeof(double) * 16);
  const std::string keep = g_err;
  mvicp_destroy(c);
  g_err = keep;
  return rc;
}

static void summary_of_state(const LmState& st, mvicp_lm_summary* s) {
  s->termination = st.termination; s->num_iterations = st.iteration; s->num_successful_steps = st.n_success;
  s->num_evaluations = st.n_evals; s->num_linear_solves = st.n_solves; s->reserved = 0;
  s->initial_cost = st.initial_cost; s->final_cost = st.x_cost;
}
// the summary of a solve without unknowns ("nothing to optimise")
static void summary_no_unknowns(mvicp_lm_summary* s) { std::memset(s, 0, sizeof *s); s->termination = MVICP_TERM_GRADIENT_TOLERANCE; }

// ---- the LM solves (mvicp_optimize, mvicp_optimize_components) ------------------------------------------------------
// Connected components of the undirected graph the edges induce over all frames, numbered in ascending order of their lowest
// frame: the root of every union-find tree is its lowest frame, so a frame's component is known once its root's is.
static int graph_components(const mvicp_ctx* c, std::vector<int32_t>& comp) {
  std::vector<int32_t> up(c->M);
  std::iota(up.begin(), up.end(), 0);
  auto root = [&](int f) { while (up[f] != f) f = up[f] = up[up[f]]; return f; };
  for (const EdgeDev& e : c->h_edges) {
    const int a = root(e.src), b = root(e.dst);
    if (a != b) up[std::max(a, b)] = std::min(a, b);
  }
  comp.assign(c->M, -1);
  int n = 0;
  for (int f = 0; f < c->M; ++f) { const int r = root(f); comp[f] = r == f ? n++ : comp[r]; }
  return n;
}

// One LM solve: the whole graph as one problem (frame 0 fixed), or every connected component as a problem of its own, solved as
// mvicp_optimize solves it in a context that holds only that component (its lowest frame fixed, its own trust region, counters
// and termination).  One pipelined loop for all problems: the streaming kernels skip the edges of the problems that are done,
// lm_step_kernel steps each of the others in its own CTA.  Only the whole-graph solve may run sharded.
static int solve_lm(mvicp_ctx* c, bool per_component, const char* fn, int32_t param, int32_t cost, int32_t robust,
                    const mvicp_lm_options* opt_in, mvicp_lm_summary* summaries) {
  if (!c || !c->M || !c->E) return fail(MVICP_ERR_STATE, "%s: frames and graph must be set first", fn);
  if (param < 0 || param > 2 || cost < 0 || cost > 2) return fail(MVICP_ERR_INVALID, "%s: bad param/cost", fn);
  if (cost != COST_P2P && !c->have_normals) return fail(MVICP_ERR_INVALID, "point-to-plane needs normals for every frame");
  if (per_component && c->world > 1) return fail(MVICP_ERR_STATE, "%s: the component solve runs on one GPU; this context is sharded", fn);
  RET(check_lm_options(opt_in, fn));
  CU(cudaSetDevice(c->device));
  c->lm_blocks_E = 0;   // until this solve's evaluations have run
  const int M = c->M, E = c->E;
  std::vector<int32_t> comp(M, 0);
  const int K = per_component ? graph_components(c, comp) : 1;
  // the lowest frame of every component is fixed: frames[0]->fixed = true (icp-ceres.cpp:242-244,342-344,417-419)
  std::vector<std::vector<int32_t>> fr(K), ed(K);
  for (int f = 0; f < M; ++f) { if (fr[comp[f]].empty()) c->fixed[f] = 1; fr[comp[f]].push_back(f); }
  for (int e = 0; e < E; ++e) ed[comp[c->h_edges[e].src]].push_back(e);
  // the problems: the components with a free frame, with local columns; edges of fixed src frames contribute nothing
  // (icp-ceres.cpp:255,353,426)
  c->h_col.assign(M, -1);
  std::vector<int32_t> prob_of(K, -1), ns;
  std::vector<std::vector<int32_t>> pf, pe;
  for (int k = 0; k < K; ++k) {
    int n = 0;
    for (int f : fr[k]) if (!c->fixed[f]) { c->h_col[f] = n; n += 6; }
    if (!n) continue;
    prob_of[k] = (int32_t)pf.size(); ns.push_back(n);
    pf.push_back(std::move(fr[k])); pe.push_back(std::move(ed[k]));
  }
  const int P = (int)pf.size();
  mvicp_lm_options opt; if (opt_in) opt = *opt_in; else mvicp_default_lm_options(&opt);
  if (!P) {   // nothing to optimise; still "writes the poses back"
    if (summaries) for (int k = 0; k < K; ++k) summary_no_unknowns(summaries + k);
    return MVICP_OK;
  }
  RET(refresh_if_fixed_changed(c));
  // the layout depends only on the kind of solve, the graph and the fixed flags: build and upload it when those change
  std::vector<uint8_t> key(c->fixed); key.push_back((uint8_t)(c->graph_gen & 0xff)); key.push_back((uint8_t)((c->graph_gen >> 8) & 0xff));
  key.push_back(per_component ? 1 : 0);
  if (key != c->lm.key) {
    std::vector<uint8_t> active(E);
    for (int e = 0; e < E; ++e) active[e] = !c->fixed[c->h_edges[e].src];
    RET(upload_problems(c, c->lm, c->h_col, pf, pe, active, key));
  }
  LmState* st = static_cast<LmState*>(c->h_state);   // pinned staging: no synchronisation needed before the kernels
  std::memset(st, 0, sizeof(LmState) * (P + 1));
  for (int q = 0; q <= P; ++q) {
    LmState& s = st[q];
    s.opt = opt; s.param = param; s.cost_kind = cost; s.robust = robust ? 1 : 0; s.G = ambient_size(param);
    if (q == P) { s.M = M; s.E = E; continue; }
    s.M = (int32_t)pf[q].size(); s.E = (int32_t)pe[q].size(); s.n = ns[q]; s.F = s.n / 6;
    s.radius = opt.initial_trust_region_radius; s.decrease_factor = 2.0;
  }
  LmState* dS = c->lm.state.as<LmState>();
  CU(cudaMemcpyAsync(dS, st, sizeof(LmState) * (P + 1), cudaMemcpyHostToDevice, c->stream));
  // the per-frame arrays of the evaluation point are shared by every problem (indexed by graph frame)
  RET(c->d_x.reserve(sizeof(double) * 7 * M)); RET(c->d_cand.reserve(sizeof(double) * 7 * M));
  RET(c->d_Rt.reserve(sizeof(Rt) * M)); RET(c->d_K.reserve(sizeof(double) * 36 * M));

  LmWork w{};
  w.S = dS + P; w.edges = c->d_edges.as<EdgeDev>(); w.eout = c->d_eout.as<double>();
  // one row of stamps per launch: only a one-problem solve, whose single CTA writes it
  if (P == 1 && std::getenv("MVICP_STEP_PROFILE")) { RET(c->d_prof.reserve(sizeof(long long) * 64)); w.prof = c->d_prof.as<long long>(); }
  c->nonrigid = poses_nonrigid(c->h_poses.data(), M);   // the mirror follows every solve and every mvicp_set_poses
  const bool general = c->nonrigid && param != PARAM_AA;   // one eval path for every problem
  if (general) { RET(c->d_gen.reserve(sizeof(FrameGen) * M)); RET(c->d_partial.reserve(sizeof(double) * GBLK * std::max<size_t>(1, c->n_eval_tiles))); }
  w.G_eval = general ? c->d_gen.as<FrameGen>() : nullptr;
  w.x = c->d_x.as<double>(); w.cand = c->d_cand.as<double>(); w.Rt_eval = c->d_Rt.as<Rt>(); w.K_eval = c->d_K.as<double>();
  w.poses16 = c->d_poses.as<double>(); w.host_flag = c->d_flag;
  const LmProblem* probs = c->lm.prob.as<LmProblem>();
  unsigned int* ticket = c->d_lm_ticket.as<unsigned int>();

  CU(cudaEventRecord(c->ev[3], c->stream));
  lm_init_kernel<<<(M + 63) / 64, 64, 0, c->stream>>>(w);
  c->stats.kernel_launches += 1;
  const int64_t max_evals = (int64_t)opt.max_num_iterations + 2;   // per problem, so for the loop as well (no int overflow at INT32_MAX)
  const bool use_p2p = c->comm && c->world > 1 && c->p2p_ok && E <= mvicp_ctx::X_ECAP;
  const DoneGate gate{&dS[0].done, c->lm.edge_prob, (int32_t)(sizeof(LmState) / sizeof(int))};
  const int rob = robust ? 1 : 0;
  const EvalArgs ea = lm_eval_args(c);
  auto eval = [&]() {
    if (general) { if (c->f32) launch_eval_general<true>(c, ea, param, cost, rob, gate); else launch_eval_general<false>(c, ea, param, cost, rob, gate); }
    else if (c->f32) launch_eval<true>(c, ea, cost, rob, gate); else launch_eval<false>(c, ea, cost, rob, gate);
  };
  auto step = [&](size_t dyn) -> int {
    // sharded: pair matrices go straight into every peer's exchange buffer (double-buffered by iteration parity)
    PeerTable pt; std::memset(&pt, 0, sizeof pt); pt.world = 1; pt.rank = 0;
    double* eout_local = c->d_eout.as<double>();
    unsigned int* xcounter = nullptr;
    int xs = 0;
    if (use_p2p) {
      xs = ++c->xseq;
      const size_t half = (size_t)mvicp_ctx::X_ECAP * EOUT;
      pt.world = c->world; pt.rank = c->rank;
      for (int p = 0; p < c->world; ++p) {
        pt.eout[p] = (double*)c->peer_x[p] + (size_t)(xs & 1) * half;
        pt.flags[p] = (volatile int*)((double*)c->peer_x[p] + 2 * half);
      }
      eout_local = pt.eout[c->rank];
      xcounter = (unsigned int*)((double*)c->xbuf + 2 * half) + 32;
    }
    if (general)
      lm_edge_general_kernel<<<E, EDGE_THREADS, 0, c->stream>>>(c->d_edges.as<EdgeDev>(), c->d_edge_tile_begin.as<int32_t>(),
                                                                c->d_partial.as<double>(), eout_local, gate, pt, xs, xcounter);
    else
      lm_edge_kernel<<<E, EDGE_THREADS, 0, c->stream>>>(c->d_edges.as<EdgeDev>(), c->d_edge_tile_begin.as<int32_t>(), c->d_partial.as<double>(),
                                                        cost == COST_P2PLANE ? NBLK_PLANE : NBLK, c->d_Rt.as<Rt>(), c->d_K.as<double>(),
                                                        eout_local, gate, pt, xs, xcounter);
    if (c->comm && c->world > 1 && !use_p2p)
      NC(ncclAllReduce(c->d_eout.p, c->d_eout.p, (size_t)EOUT * E, ncclDouble, ncclSum, c->comm, c->stream));
    w.eout = eout_local; w.peer_flags = use_p2p ? pt.flags[c->rank] : nullptr; w.world = c->world; w.xseq = xs;
    lm_step_kernel<<<P, STEP_THREADS, dyn, c->stream>>>(w, probs, ticket);
    c->stats.kernel_launches += (c->n_eval_tiles ? 1 : 0) + 2;
    return MVICP_OK;
  };
  RET(run_steps(c, lm_step_kernel, c->lm.dyn, max_evals, "LM", w.seq, eval, step));
  // sharded runs: every rank holds bit-identical poses (the same lm_step_kernel ran on bit-identical pair matrices), so
  // no pose exchange is needed; the NCCL-only mode still all-gathers the owners' copies (6-dof poses per outer iteration,
  // as the north-star words it) -- a few small copies that change nothing.
  if (c->comm && c->world > 1 && !use_p2p) {
    const int chunk = (M + c->world - 1) / c->world;
    RET(c->d_posegather.reserve(sizeof(double) * 16 * (size_t)chunk * c->world * 2));
    double* sendb = c->d_posegather.as<double>();
    double* recvb = sendb + (size_t)16 * chunk * c->world;
    CU(cudaMemsetAsync(sendb, 0, sizeof(double) * 16 * chunk, c->stream));
    int f0 = -1, f1 = -1;
    for (int f = 0; f < M; ++f) if (owner_of(c, f) == c->rank) { if (f0 < 0) f0 = f; f1 = f; }
    if (f0 >= 0) CU(cudaMemcpyAsync(sendb, c->d_poses.as<double>() + 16 * f0, sizeof(double) * 16 * (f1 - f0 + 1), cudaMemcpyDeviceToDevice, c->stream));
    NC(ncclAllGather(sendb, recvb, (size_t)16 * chunk, ncclDouble, c->comm, c->stream));
    for (int r = 0; r < c->world; ++r) {
      int a = -1, b = -1;
      for (int f = 0; f < M; ++f) if (owner_of(c, f) == r) { if (a < 0) a = f; b = f; }
      if (a >= 0) CU(cudaMemcpyAsync(c->d_poses.as<double>() + 16 * a, recvb + (size_t)16 * chunk * r, sizeof(double) * 16 * (b - a + 1), cudaMemcpyDeviceToDevice, c->stream));
    }
  }
  RET(read_back_solve(c, st, dS, sizeof(LmState) * (P + 1)));
  int max_iters = 0; bool all_done = true, timed_out = false;
  for (int q = 0; q < P; ++q) { max_iters = std::max(max_iters, (int)st[q].iteration); all_done = all_done && st[q].done; timed_out = timed_out || st[q].nonrigid == 2; }
  c->last_lm_iters = max_iters;   // the cross-round shortcuts of mvicp_correspond wait for the slowest problem
  if (summaries)
    for (int k = 0; k < K; ++k) {
      if (prob_of[k] < 0) summary_no_unknowns(summaries + k);
      else summary_of_state(st[prob_of[k]], summaries + k);
    }
  if (timed_out) return fail(MVICP_ERR_NCCL, "a peer rank never delivered its pair matrices (peer-memory exchange timed out)");
  if (st[P].nonrigid && !general)   // cannot happen after mvicp_set_poses; guards poses that reached the device another way
    return fail(MVICP_ERR_NONRIGID, "a pose's quaternion is not unit (non-rigid Isometry) but the unit-quaternion LM path was run");
  if (!all_done) return fail(MVICP_ERR_STATE, "LM loop did not terminate within %lld evaluations", (long long)max_evals);
  c->lm_blocks_E = E; c->blocks_g2o = false; c->lm_blocks_fixed = c->fixed;
  return MVICP_OK;
}

extern "C" {
int mvicp_optimize(mvicp_ctx* c, int32_t param, int32_t cost, int32_t robust, const mvicp_lm_options* opt_in, mvicp_lm_summary* summary) {
  return solve_lm(c, false, "mvicp_optimize", param, cost, robust, opt_in, summary);
}

int mvicp_get_components(mvicp_ctx* c, int32_t* n_components, int32_t* component_of_frame) {
  if (!c || !n_components) return fail(MVICP_ERR_INVALID, "mvicp_get_components: bad arguments");
  if (!c->M) return fail(MVICP_ERR_STATE, "mvicp_get_components: frames must be set first");
  std::vector<int32_t> comp;
  *n_components = graph_components(c, comp);
  if (component_of_frame) std::memcpy(component_of_frame, comp.data(), sizeof(int32_t) * c->M);
  return MVICP_OK;
}

int mvicp_optimize_components(mvicp_ctx* c, int32_t param, int32_t cost, int32_t robust, const mvicp_lm_options* opt_in,
                              mvicp_lm_summary* summaries) {
  return solve_lm(c, true, "mvicp_optimize_components", param, cost, robust, opt_in, summaries);
}

// ---- pose covariances (covariance.cuh, DESIGN.md section 6j) ---------------------------------------------------------------
// The problem of mvicp_optimize (frame 0 and the flagged frames fixed), split into its connected components as
// mvicp_optimize_components splits it, but without fixing anything: a component without a fixed frame is singular (its gauge is
// free) and is not factored.  One evaluation at the current poses with the solve's kernels, tile length and eval path, on
// buffers of this call's own; then cov_factor_kernel per problem and cov_solve_kernel per (problem, frame whose columns some pair
// needs); the pairs are read out on the host from one copy.  The block of (a, b) always comes from the columns of the one of the
// two frames with the higher local column, so (b, a) is its exact transpose and no block depends on the other pairs.
int mvicp_covariance(mvicp_ctx* c, int32_t param, int32_t cost, int32_t robust, int32_t n_pairs, const int32_t* frame_a,
                     const int32_t* frame_b, double* cov36, int32_t* status) {
  const char* fn = "mvicp_covariance";
  if (!c) return fail(MVICP_ERR_INVALID, "%s: null context", fn);
  if (param < 0 || param > 2 || cost < 0 || cost > 2) return fail(MVICP_ERR_INVALID, "%s: bad param/cost", fn);
  if (n_pairs < 0 || (n_pairs > 0 && (!frame_a || !frame_b || !cov36))) return fail(MVICP_ERR_INVALID, "%s: bad pair arrays", fn);
  if (!c->M || !c->E) return fail(MVICP_ERR_STATE, "%s: frames and graph must be set first", fn);
  if (c->world > 1) return fail(MVICP_ERR_STATE, "%s: the covariance runs on one GPU; this context is sharded", fn);
  const int M = c->M, E = c->E;
  for (int k = 0; k < n_pairs; ++k)
    if (frame_a[k] < 0 || frame_a[k] >= M || frame_b[k] < 0 || frame_b[k] >= M)
      return fail(MVICP_ERR_INVALID, "%s: pair %d (%d, %d): frame outside [0, %d)", fn, k, frame_a[k], frame_b[k], M);
  if (cost != COST_P2P && !c->have_normals) return fail(MVICP_ERR_INVALID, "point-to-plane needs normals for every frame");
  if (!n_pairs) return MVICP_OK;
  CU(cudaSetDevice(c->device));
  std::vector<uint8_t> fixed(c->fixed);
  fixed[0] = 1;   // as mvicp_optimize fixes it (icp-ceres.cpp:242-244)
  std::vector<int32_t> comp;
  const int K = graph_components(c, comp);
  std::vector<std::vector<int32_t>> fr(K), ed(K);
  std::vector<uint8_t> anchored(K, 0);
  for (int f = 0; f < M; ++f) { fr[comp[f]].push_back(f); if (fixed[f]) anchored[comp[f]] = 1; }
  for (int e = 0; e < E; ++e) ed[comp[c->h_edges[e].src]].push_back(e);
  std::vector<int32_t> col(M, -1), prob_of(K, -1), ns;
  std::vector<std::vector<int32_t>> pf, pe;
  for (int k = 0; k < K; ++k) {
    if (!anchored[k]) continue;
    int n = 0;
    for (int f : fr[k]) if (!fixed[f]) { col[f] = n; n += 6; }
    if (!n) continue;
    prob_of[k] = (int32_t)pf.size(); ns.push_back(n);
    pf.push_back(std::move(fr[k])); pe.push_back(std::move(ed[k]));
  }
  const int P = (int)pf.size();
  // classify the pairs; the ones that need C name the frame whose columns hold their block
  std::vector<int32_t> st(n_pairs), hi_of(n_pairs, -1), job_of(M, -1);
  std::vector<CovJob> jobs;
  int64_t out_len = 0;
  int n_max = 0;
  for (int k = 0; k < n_pairs; ++k) {
    const int a = frame_a[k], b = frame_b[k];
    if (fixed[a] || fixed[b]) { st[k] = MVICP_COV_FIXED; continue; }
    if (comp[a] != comp[b]) { st[k] = MVICP_COV_INDEPENDENT; continue; }
    const int q = prob_of[comp[a]];
    if (q < 0) { st[k] = MVICP_COV_SINGULAR; continue; }
    st[k] = MVICP_COV_OK;
    const int hi = col[a] >= col[b] ? a : b;
    hi_of[k] = hi;
    if (job_of[hi] < 0) {
      job_of[hi] = (int32_t)jobs.size();
      jobs.push_back(CovJob{q, col[hi], out_len});
      out_len += 6 * (int64_t)ns[q]; n_max = std::max(n_max, ns[q]);
    }
  }
  std::vector<int32_t> pstat(P, MVICP_COV_OK);
  std::vector<double> hout(out_len);
  if (!jobs.empty()) {
    // layout of the problems: cached, as the solves cache theirs
    std::vector<uint8_t> key(fixed); key.push_back((uint8_t)(c->graph_gen & 0xff)); key.push_back((uint8_t)((c->graph_gen >> 8) & 0xff));
    if (key != c->cov.key) {
      std::vector<uint8_t> active(E);
      for (int e = 0; e < E; ++e) active[e] = !fixed[c->h_edges[e].src];
      RET(upload_problems(c, c->cov, col, pf, pe, active, key));
    }
    // the streaming tiles mvicp_optimize lays out on one GPU once frame 0 is fixed (layout_work)
    int64_t active_slots = 0;
    for (int e = 0; e < E; ++e) if (!fixed[c->h_edges[e].src]) active_slots += c->h_edges[e].n_src;
    const int tl = eval_tile_len_of(active_slots);
    std::vector<Tile> et; std::vector<int32_t> etb(E + 1, 0);
    for (int e = 0; e < E; ++e) {
      etb[e] = (int32_t)et.size();
      if (fixed[c->h_edges[e].src]) continue;
      for (int s = 0; s < c->h_edges[e].n_src; s += tl) et.push_back(Tile{e, s});
    }
    etb[E] = (int32_t)et.size();
    const int nt = (int)et.size();
    std::vector<LmState> hs(P + 1);
    std::memset(hs.data(), 0, sizeof(LmState) * (P + 1));
    for (int q = 0; q <= P; ++q) {
      LmState& s = hs[q];
      mvicp_default_lm_options(&s.opt);
      s.param = param; s.cost_kind = cost; s.robust = robust ? 1 : 0; s.G = ambient_size(param);
      if (q == P) { s.M = M; s.E = E; continue; }
      s.M = (int32_t)pf[q].size(); s.E = (int32_t)pe[q].size(); s.n = ns[q]; s.F = s.n / 6;
    }
    const bool general = poses_nonrigid(c->h_poses.data(), M) && param != PARAM_AA;   // the solve's rule
    RET(c->d_cov_x.reserve(sizeof(double) * 7 * M)); RET(c->d_cov_cand.reserve(sizeof(double) * 7 * M));
    RET(c->d_cov_Rt.reserve(sizeof(Rt) * M)); RET(c->d_cov_K.reserve(sizeof(double) * 36 * M));
    if (general) RET(c->d_cov_gen.reserve(sizeof(FrameGen) * M));
    RET(c->d_cov_partial.reserve(sizeof(double) * (general ? GBLK : NBLK) * std::max(1, nt)));
    RET(c->d_cov_eout.reserve(sizeof(double) * EOUT * E));
    RET(c->d_cov_tiles.reserve(sizeof(Tile) * std::max(1, nt))); RET(c->d_cov_etb.reserve(sizeof(int32_t) * (E + 1)));
    RET(c->d_cov_status.reserve(sizeof(int32_t) * P)); RET(c->d_cov_jobs.reserve(sizeof(CovJob) * jobs.size()));
    RET(c->d_cov_out.reserve(sizeof(double) * out_len));
    LmState* dS = c->cov.state.as<LmState>();
    CU(cudaMemcpyAsync(dS, hs.data(), sizeof(LmState) * (P + 1), cudaMemcpyHostToDevice, c->stream));
    if (nt) CU(cudaMemcpyAsync(c->d_cov_tiles.p, et.data(), sizeof(Tile) * nt, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(c->d_cov_etb.p, etb.data(), sizeof(int32_t) * (E + 1), cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(c->d_cov_jobs.p, jobs.data(), sizeof(CovJob) * jobs.size(), cudaMemcpyHostToDevice, c->stream));
    LmWork w{};
    w.S = dS + P; w.x = c->d_cov_x.as<double>(); w.cand = c->d_cov_cand.as<double>(); w.Rt_eval = c->d_cov_Rt.as<Rt>();
    w.K_eval = c->d_cov_K.as<double>(); w.G_eval = general ? c->d_cov_gen.as<FrameGen>() : nullptr; w.poses16 = c->d_poses.as<double>();
    lm_init_kernel<<<(M + 63) / 64, 64, 0, c->stream>>>(w);
    const DoneGate gate{&dS[0].done, c->cov.edge_prob, (int32_t)(sizeof(LmState) / sizeof(int))};
    const EvalArgs ea{c->d_cov_tiles.as<Tile>(), nt, tl, c->d_cov_Rt.as<Rt>(), c->d_cov_gen.as<FrameGen>(), c->d_cov_partial.as<double>()};
    const int rob = robust ? 1 : 0;
    if (general) { if (c->f32) launch_eval_general<true>(c, ea, param, cost, rob, gate); else launch_eval_general<false>(c, ea, param, cost, rob, gate); }
    else if (c->f32) launch_eval<true>(c, ea, cost, rob, gate); else launch_eval<false>(c, ea, cost, rob, gate);
    PeerTable pt; std::memset(&pt, 0, sizeof pt); pt.world = 1; pt.rank = 0;
    double* eout = c->d_cov_eout.as<double>();
    if (general)
      lm_edge_general_kernel<<<E, EDGE_THREADS, 0, c->stream>>>(c->d_edges.as<EdgeDev>(), c->d_cov_etb.as<int32_t>(),
                                                                c->d_cov_partial.as<double>(), eout, gate, pt, 0, nullptr);
    else
      lm_edge_kernel<<<E, EDGE_THREADS, 0, c->stream>>>(c->d_edges.as<EdgeDev>(), c->d_cov_etb.as<int32_t>(), c->d_cov_partial.as<double>(),
                                                        cost == COST_P2PLANE ? NBLK_PLANE : NBLK, c->d_cov_Rt.as<Rt>(), c->d_cov_K.as<double>(),
                                                        eout, gate, pt, 0, nullptr);
    const LmProblem* probs = c->cov.prob.as<LmProblem>();
    int32_t* dstat = c->d_cov_status.as<int32_t>();
    CU(cudaFuncSetAttribute(cov_factor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    cov_factor_kernel<<<P, STEP_THREADS, c->cov.dyn, c->stream>>>(probs, eout, dstat);
    const size_t vec = sizeof(double) * 6 * (size_t)n_max;
    const int vec_in_smem = vec <= 220 * 1024 ? 1 : 0;
    if (vec_in_smem) CU(cudaFuncSetAttribute(cov_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    cov_solve_kernel<<<(int)jobs.size(), COV_SOLVE_THREADS, vec_in_smem ? vec : 0, c->stream>>>(probs, c->d_cov_jobs.as<CovJob>(), dstat,
                                                                                               c->d_cov_out.as<double>(), vec_in_smem);
    c->stats.kernel_launches += 4 + (nt ? 1 : 0);
    CU(cudaMemcpyAsync(pstat.data(), dstat, sizeof(int32_t) * P, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaMemcpyAsync(hout.data(), c->d_cov_out.p, sizeof(double) * out_len, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    CU(cudaGetLastError());
  }
  // the blocks: Cov(a, b)[i][j] = C[col a + i][col b + j], read from the columns of hi = the frame with the higher column
  const double nan = std::numeric_limits<double>::quiet_NaN();
  for (int k = 0; k < n_pairs; ++k) {
    double* o = cov36 + 36 * (size_t)k;
    const int a = frame_a[k], b = frame_b[k], hi = hi_of[k];
    if (st[k] == MVICP_COV_OK && pstat[prob_of[comp[a]]] != MVICP_COV_OK) st[k] = MVICP_COV_SINGULAR;
    if (status) status[k] = st[k];
    if (st[k] == MVICP_COV_FIXED || st[k] == MVICP_COV_INDEPENDENT) { for (int i = 0; i < 36; ++i) o[i] = 0.0; continue; }
    if (st[k] == MVICP_COV_SINGULAR) { for (int i = 0; i < 36; ++i) o[i] = nan; continue; }
    const CovJob& jb = jobs[job_of[hi]];
    const int n = ns[jb.prob];
    const double* base = hout.data() + jb.at;   // column col[hi] + j at base[j n ..]
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j < 6; ++j) {
        if (a == b) o[6 * i + j] = 0.5 * (base[(size_t)j * n + col[a] + i] + base[(size_t)i * n + col[a] + j]);   // exactly symmetric
        else if (b == hi) o[6 * i + j] = base[(size_t)j * n + col[a] + i];
        else o[6 * i + j] = base[(size_t)i * n + col[b] + j];
      }
  }
  return MVICP_OK;
}

int mvicp_icp_round(mvicp_ctx* c, float thresh, int32_t param, int32_t cost, int32_t robust, const mvicp_lm_options* opt, mvicp_lm_summary* summary) {
  RET(check_lm_options(opt, "mvicp_icp_round"));   // before the correspondence step changes anything
  RET(mvicp_correspond(c, thresh));
  return mvicp_optimize(c, param, cost, robust, opt, summary);
}

int mvicp_pairwise(const mvicp_config* cfg, int32_t param, int32_t cost, const double* src, const double* dst, const double* nor,
                   int64_t n, const mvicp_lm_options* opt, double* pose16_out, mvicp_lm_summary* summary) {
  if (!src || !dst || n <= 0 || !pose16_out) return fail(MVICP_ERR_INVALID, "mvicp_pairwise: bad arguments");
  if (cost != MVICP_COST_P2P && !nor) return fail(MVICP_ERR_INVALID, "mvicp_pairwise: point-to-plane needs dst normals");
  RET(check_lm_options(opt, "mvicp_pairwise"));
  return run_pairwise(cfg, src, dst, nor, n, pose16_out, [&](mvicp_ctx* c) { return mvicp_optimize(c, param, cost, 0, opt, summary); });
}

}  // extern "C"
// ---- g2o backend (g2o.cuh; icp-g2o.cpp) ---------------------------------------------------------------------
template <bool F32> static void launch_g2o_eval(mvicp_ctx* c, int cost, int nt, G2oGate gate, double eps) {
#define MV_G2O(NF, COSTK)                                                                                          \
  g2o_eval_kernel<F32, NF, COSTK><<<nt, EVAL_THREADS, 0, c->stream>>>(c->d_frames.as<FrameDev>(), c->d_edges.as<EdgeDev>(), \
      c->d_g2o_tiles.as<Tile>(), c->eval_tile_len, c->d_corr.as<int32_t>(), c->d_g2o_ev.as<Rt>(), gate, eps, c->d_partial.as<double>())
  if (cost == COST_P2P) MV_G2O(F32, COST_P2P);
  else if (F32 && c->nor_f32) MV_G2O(F32, COST_P2PLANE);
  else MV_G2O(false, COST_P2PLANE);
#undef MV_G2O
}
// trace rows per problem: a one-problem solve records its first G2O_TRACE_CAP trials, a batch of P problems the first
// max(G2O_TRACE_MIN, G2O_TRACE_CAP / P) of each, so the buffer stays bounded for hundreds of components
static constexpr int G2O_TRACE_CAP = 65536, G2O_TRACE_MIN = 1024;

extern "C" {
void mvicp_default_g2o_options(mvicp_g2o_options* o) {
  o->iterations_per_call = 100; o->max_calls = 100; o->no_improvement_limit = 5; o->max_trials = 10; o->orthonormalize_after = 1000;
  o->reserved = 0; o->tau = 1e-5; o->information_eps = 0.01;
}
}  // extern "C"

// One g2o solve: the whole graph as one problem (frame 0 fixed), or every connected component as a problem of its own, solved as
// mvicp_optimize_g2o solves it in a context that holds only that component (its lowest frame fixed; its own lambda, trials,
// calls, noImpr counter and chi2).  One pipelined loop for all problems: the streaming kernels skip the edges of the problems
// that are done (G2oGate), g2o_step_kernel steps each of the others in its own CTA.  The problems are laid out again on every
// call, since their vertices follow the correspondences.  summaries / chi2_per_call: one entry / row per component.
static int solve_g2o(mvicp_ctx* c, bool per_component, const char* fn, int32_t cost, const mvicp_g2o_options* opt_in,
                     mvicp_g2o_summary* summaries, double* chi2_per_call) {
  if (!c || !c->M || !c->E) return fail(MVICP_ERR_STATE, "%s: frames and graph must be set first", fn);
  if (cost != COST_P2P && cost != COST_P2PLANE) return fail(MVICP_ERR_INVALID, "%s: cost must be point-to-point or point-to-plane", fn);
  if (cost == COST_P2PLANE && !c->have_normals) return fail(MVICP_ERR_INVALID, "point-to-plane needs normals for every frame");
  if (c->world > 1) return fail(MVICP_ERR_STATE, "%s: the g2o solve runs on one GPU; this context is sharded", fn);
  mvicp_g2o_options opt; if (opt_in) opt = *opt_in; else mvicp_default_g2o_options(&opt);
  if (opt.iterations_per_call < 1 || opt.max_calls < 1 || opt.max_trials < 1 || opt.no_improvement_limit < 0 || opt.orthonormalize_after < 0)
    return fail(MVICP_ERR_INVALID, "%s: bad options", fn);
  c->lm_blocks_E = 0;   // until this solve has run: it writes its own edge blocks into d_eout
  CU(cudaSetDevice(c->device));
  const int M = c->M, E = c->E;
  std::vector<int32_t> comp(M, 0);
  const int K = per_component ? graph_components(c, comp) : 1;
  // the lowest frame of every component is fixed: frames[0]->fixed = true (icp-g2o.cpp:182-186)
  std::vector<std::vector<int32_t>> fr(K), ed(K);
  for (int f = 0; f < M; ++f) { if (fr[comp[f]].empty()) c->fixed[f] = 1; fr[comp[f]].push_back(f); }
  for (int e = 0; e < E; ++e) ed[comp[c->h_edges[e].src]].push_back(e);
  RET(refresh_if_fixed_changed(c));
  // every edge with a free end carries one GICP edge per stored correspondence (an edge between fixed vertices is not active)
  const int tl = c->eval_tile_len;
  std::vector<Tile> tiles; std::vector<int32_t> tb(E + 1, 0);
  for (int e = 0; e < E; ++e) {
    tb[e] = (int32_t)tiles.size();
    const EdgeDev& eg = c->h_edges[e];
    if (c->fixed[eg.src] && c->fixed[eg.dst]) continue;
    for (int s = 0; s < eg.n_src; s += tl) tiles.push_back(Tile{e, s});
  }
  tb[E] = (int32_t)tiles.size();
  const int nt = (int)tiles.size();
  RET(c->d_g2o_tiles.reserve(sizeof(Tile) * std::max(1, nt)));
  RET(c->d_g2o_tile_begin.reserve(sizeof(int32_t) * (E + 1)));
  RET(c->d_g2o_cnt.reserve(sizeof(unsigned long long) * E));
  RET(c->d_partial.reserve(sizeof(double) * GBLK * std::max(1, nt)));
  if (nt) CU(cudaMemcpyAsync(c->d_g2o_tiles.p, tiles.data(), sizeof(Tile) * nt, cudaMemcpyHostToDevice, c->stream));
  CU(cudaMemcpyAsync(c->d_g2o_tile_begin.p, tb.data(), sizeof(int32_t) * (E + 1), cudaMemcpyHostToDevice, c->stream));
  CU(cudaMemsetAsync(c->d_g2o_cnt.p, 0, sizeof(unsigned long long) * E, c->stream));
  if (nt) {
    g2o_count_kernel<<<nt, 256, 0, c->stream>>>(c->d_edges.as<EdgeDev>(), c->d_g2o_tiles.as<Tile>(), tl, c->d_corr.as<int32_t>(),
                                                c->d_g2o_cnt.as<unsigned long long>());
    c->stats.kernel_launches += 1;
  }
  std::vector<unsigned long long> cnt(E);
  CU(cudaMemcpyAsync(cnt.data(), c->d_g2o_cnt.p, sizeof(unsigned long long) * E, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  // the vertices: free frames with at least one correspondence (a vertex without edges is not optimised); the problems: the
  // components with a vertex, each with its own local columns
  std::vector<uint8_t> touched(M, 0);
  for (int e = 0; e < E; ++e) if (cnt[e]) { touched[c->h_edges[e].src] = 1; touched[c->h_edges[e].dst] = 1; }
  c->h_col.assign(M, -1);
  std::vector<int32_t> prob_of(K, -1), ns;
  std::vector<std::vector<int32_t>> pf, pe;
  for (int k = 0; k < K; ++k) {
    int n = 0;
    for (int f : fr[k]) if (touched[f] && !c->fixed[f]) { c->h_col[f] = n; n += 6; }
    if (!n) continue;
    prob_of[k] = (int32_t)pf.size(); ns.push_back(n);
    pf.push_back(std::move(fr[k])); pe.push_back(std::move(ed[k]));
  }
  const int P = (int)pf.size();
  const size_t row = (size_t)opt.max_calls + 1;   // doubles per chi2_per_call row
  if (summaries) std::memset(summaries, 0, sizeof(mvicp_g2o_summary) * K);
  c->g2o_per_component = per_component;
  c->g2o_trials.assign(K, 0); c->g2o_trace_row.assign(K, -1);
  // no active edge: chi2 = 0 (g2o's optimize() returns at once, "0 vertices to optimize"), nothing moves
  auto no_vertices = [&](int k) {
    if (summaries) summaries[k].ended = MVICP_G2O_END_NO_VERTICES;
    if (chi2_per_call) chi2_per_call[row * k] = 0.0;
  };
  // mvicp_debug_edge_blocks after this solve: the edges of a component without a problem are never evaluated
  auto readout_after = [&]() {
    c->g2o_blocks_unwritten.assign(E, 0);
    for (int e = 0; e < E; ++e) c->g2o_blocks_unwritten[e] = prob_of[comp[c->h_edges[e].src]] < 0;
    c->lm_blocks_E = E; c->blocks_g2o = true;
  };
  if (!P) {
    for (int k = 0; k < K; ++k) no_vertices(k);
    readout_after();
    return MVICP_OK;
  }
  std::vector<uint8_t> active(E);
  for (int e = 0; e < E; ++e) active[e] = cnt[e] != 0;
  std::vector<uint8_t> key(c->fixed); key.push_back((uint8_t)(c->graph_gen & 0xff)); key.push_back((uint8_t)((c->graph_gen >> 8) & 0xff));
  key.push_back(per_component ? 3 : 2);
  RET(upload_problems(c, c->lm, c->h_col, pf, pe, active, key));
  const int64_t cap = std::max<int64_t>(G2O_TRACE_MIN, G2O_TRACE_CAP / P);
  RET(c->d_g2o_state.reserve(sizeof(G2oState) * P)); RET(c->d_g2o_prob.reserve(sizeof(G2oProblem) * P));
  RET(c->d_g2o_x.reserve(sizeof(Rt) * M)); RET(c->d_g2o_ev.reserve(sizeof(Rt) * M)); RET(c->d_g2o_nop.reserve(sizeof(int32_t) * M));
  RET(c->d_g2o_chi.reserve(sizeof(double) * row * P));
  RET(c->d_g2o_trace.reserve(sizeof(double) * 5 * (size_t)cap * P));
  G2oState* dS = c->d_g2o_state.as<G2oState>();
  std::vector<G2oState> st(P);
  std::vector<G2oProblem> probs(P);
  for (int q = 0; q < P; ++q) {
    G2oState& s = st[q];
    std::memset(&s, 0, sizeof s);
    s.M = (int32_t)pf[q].size(); s.E = (int32_t)pe[q].size(); s.n = ns[q];
    s.max_iter = opt.iterations_per_call; s.max_calls = opt.max_calls;
    s.no_impr_limit = opt.no_improvement_limit; s.max_trials = opt.max_trials; s.ortho_after = opt.orthonormalize_after;
    s.phase = G2O_BUILD; s.trace_cap = (int32_t)cap; s.tau = opt.tau;
    const LmProblem& lp = c->lm.h_prob[q];
    probs[q] = G2oProblem{dS + q, lp.frame, lp.edge, lp.lay, lp.H, lp.g, c->d_g2o_chi.as<double>() + row * q,
                          c->d_g2o_trace.as<double>() + 5 * (size_t)cap * q};
  }
  CU(cudaMemcpyAsync(dS, st.data(), sizeof(G2oState) * P, cudaMemcpyHostToDevice, c->stream));
  CU(cudaMemcpyAsync(c->d_g2o_prob.p, probs.data(), sizeof(G2oProblem) * P, cudaMemcpyHostToDevice, c->stream));

  G2oWork w{};
  w.eout = c->d_eout.as<double>();
  w.x = c->d_g2o_x.as<Rt>(); w.ev = c->d_g2o_ev.as<Rt>(); w.n_oplus = c->d_g2o_nop.as<int32_t>();
  w.poses16 = c->d_poses.as<double>(); w.host_flag = c->d_flag;
  const G2oProblem* dprobs = c->d_g2o_prob.as<G2oProblem>();
  unsigned int* ticket = c->d_lm_ticket.as<unsigned int>();

  CU(cudaEventRecord(c->ev[3], c->stream));
  g2o_init_kernel<<<(M + 63) / 64, 64, 0, c->stream>>>(w, M);
  c->stats.kernel_launches += 1;
  // the kernels read what to evaluate (build or trial) from the state of the edge's problem
  const int64_t max_evals = (int64_t)opt.max_calls * opt.iterations_per_call * (opt.max_trials + 1) + 2;   // per problem, so for the loop
  const double eps = opt.information_eps;
  // the joint solve (every edge in problem 0) runs without the edge -> problem lookup and with its own step kernel
  const G2oGate gate{dS, per_component ? c->lm.edge_prob : nullptr};
  auto eval = [&]() { if (c->f32) launch_g2o_eval<true>(c, cost, nt, gate, eps); else launch_g2o_eval<false>(c, cost, nt, gate, eps); };
  auto step = [&](size_t dyn) -> int {
    g2o_edge_kernel<<<E, EDGE_THREADS, 0, c->stream>>>(c->d_g2o_tile_begin.as<int32_t>(), c->d_partial.as<double>(), gate, c->d_eout.as<double>());
    if (per_component) g2o_step_kernel<<<P, STEP_THREADS, dyn, c->stream>>>(w, dprobs, ticket);
    else g2o_step_one_kernel<<<1, STEP_THREADS, dyn, c->stream>>>(w, probs[0]);
    c->stats.kernel_launches += 3;
    return MVICP_OK;
  };
  if (per_component) RET(run_steps(c, g2o_step_kernel, c->lm.dyn, max_evals, "g2o", w.seq, eval, step));
  else RET(run_steps(c, g2o_step_one_kernel, c->lm.dyn, max_evals, "g2o", w.seq, eval, step));
  RET(read_back_solve(c, st.data(), dS, sizeof(G2oState) * P));
  std::vector<double> chis;
  if (chi2_per_call) {
    chis.resize(row * P);
    CU(cudaMemcpy(chis.data(), c->d_g2o_chi.p, sizeof(double) * row * P, cudaMemcpyDeviceToHost));
  }
  c->last_lm_iters = 1 << 20;
  c->g2o_trace_cap = cap;
  bool all_done = true;
  for (int k = 0; k < K; ++k) {
    const int q = prob_of[k];
    if (q < 0) { no_vertices(k); continue; }
    const G2oState& s = st[q];
    all_done = all_done && s.done;
    c->g2o_trials[k] = s.n_trace; c->g2o_trace_row[k] = cap * q;
    if (chi2_per_call) std::memcpy(chi2_per_call + row * k, chis.data() + row * q, sizeof(double) * (s.call + 1));
    if (summaries) {
      mvicp_g2o_summary* o = summaries + k;
      o->calls = s.call; o->iterations = s.n_iters; o->trials = s.n_trials; o->accepted = s.n_accepted;
      o->evaluations = s.n_evals; o->ended = s.ended; o->last_call_end = s.last_call_end;
      o->chi2_initial = s.chi_initial; o->chi2_final = s.last_chi;
    }
  }
  if (!all_done) return fail(MVICP_ERR_STATE, "g2o solve did not terminate within %lld evaluations", (long long)max_evals);
  readout_after();
  return MVICP_OK;
}

// rows of component k's trial trace of the last g2o solve
static int g2o_trace_rows(mvicp_ctx* c, int k, double* out5, int64_t capacity, int64_t* n_trials) {
  if (n_trials) *n_trials = c->g2o_trials[k];
  const int64_t rows = std::min<int64_t>(capacity, std::min<int64_t>(c->g2o_trials[k], c->g2o_trace_cap));
  if (rows <= 0) return MVICP_OK;
  CU(cudaSetDevice(c->device));
  CU(cudaStreamSynchronize(c->stream));
  CU(cudaMemcpy(out5, c->d_g2o_trace.as<double>() + 5 * (size_t)c->g2o_trace_row[k], sizeof(double) * 5 * (size_t)rows, cudaMemcpyDeviceToHost));
  return MVICP_OK;
}

extern "C" {
int mvicp_optimize_g2o(mvicp_ctx* c, int32_t cost, const mvicp_g2o_options* opt_in, mvicp_g2o_summary* summary, double* chi2_per_call) {
  return solve_g2o(c, false, "mvicp_optimize_g2o", cost, opt_in, summary, chi2_per_call);
}

int mvicp_optimize_g2o_components(mvicp_ctx* c, int32_t cost, const mvicp_g2o_options* opt_in, mvicp_g2o_summary* summaries,
                                  double* chi2_per_call) {
  return solve_g2o(c, true, "mvicp_optimize_g2o_components", cost, opt_in, summaries, chi2_per_call);
}

int mvicp_pairwise_g2o(const mvicp_config* cfg, int32_t cost, const double* src, const double* dst, const double* nor, int64_t n,
                       const mvicp_g2o_options* opt_in, double* pose16_out, mvicp_g2o_summary* summary) {
  if (!src || !dst || n <= 0 || !pose16_out) return fail(MVICP_ERR_INVALID, "mvicp_pairwise_g2o: bad arguments");
  if (cost != MVICP_COST_P2P && !nor) return fail(MVICP_ERR_INVALID, "mvicp_pairwise_g2o: point-to-plane needs dst normals");
  mvicp_g2o_options opt;
  if (opt_in) opt = *opt_in; else { mvicp_default_g2o_options(&opt); opt.iterations_per_call = 300; }   // optimize(300), icp-g2o.cpp:72,133
  opt.max_calls = 1;
  return run_pairwise(cfg, src, dst, nor, n, pose16_out, [&](mvicp_ctx* c) { return mvicp_optimize_g2o(c, cost, &opt, summary, nullptr); });
}

int mvicp_g2o_trace(mvicp_ctx* c, double* out5, int64_t capacity, int64_t* n_trials) {
  if (!c || capacity < 0 || (capacity && !out5)) return fail(MVICP_ERR_INVALID, "mvicp_g2o_trace: bad arguments");
  if (c->g2o_per_component)
    return fail(MVICP_ERR_STATE, "mvicp_g2o_trace: the last g2o solve ran per component; read its traces with mvicp_g2o_trace_component");
  return g2o_trace_rows(c, 0, out5, capacity, n_trials);
}

int mvicp_g2o_trace_component(mvicp_ctx* c, int32_t component, double* out5, int64_t capacity, int64_t* n_trials) {
  if (!c || capacity < 0 || (capacity && !out5)) return fail(MVICP_ERR_INVALID, "mvicp_g2o_trace_component: bad arguments");
  if (component < 0 || component >= (int64_t)c->g2o_trials.size())
    return fail(MVICP_ERR_INVALID, "mvicp_g2o_trace_component: component %d out of range (the last g2o solve had %d)", component,
                (int)c->g2o_trials.size());
  return g2o_trace_rows(c, component, out5, capacity, n_trials);
}

// ---- closed-form pairwise solvers (SURVEY 8(f) row 4; icp-closedform.cpp:9-54) ------------------------------
static void host_eig_sym3(double A[3][3], double w[3], double V[3][3]) {   // cyclic Jacobi: A = V diag(w) V^T
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) V[i][j] = (i == j);
  for (int sweep = 0; sweep < 60; ++sweep) {
    if (A[0][1] * A[0][1] + A[0][2] * A[0][2] + A[1][2] * A[1][2] < 1e-300) break;
    for (int p = 0; p < 2; ++p) for (int q = p + 1; q < 3; ++q) {
      if (A[p][q] == 0.0) continue;
      const double th = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
      const double t = (th >= 0 ? 1.0 : -1.0) / (std::fabs(th) + std::sqrt(th * th + 1.0)), cs = 1.0 / std::sqrt(t * t + 1.0), sn = t * cs;
      for (int k = 0; k < 3; ++k) { const double a = A[k][p], b = A[k][q]; A[k][p] = cs * a - sn * b; A[k][q] = sn * a + cs * b; }
      for (int k = 0; k < 3; ++k) { const double a = A[p][k], b = A[q][k]; A[p][k] = cs * a - sn * b; A[q][k] = sn * a + cs * b; }
      for (int k = 0; k < 3; ++k) { const double a = V[k][p], b = V[k][q]; V[k][p] = cs * a - sn * b; V[k][q] = sn * a + cs * b; }
    }
  }
  for (int i = 0; i < 3; ++i) w[i] = A[i][i];
}

int mvicp_pairwise_closed(const mvicp_config* cfg, int32_t cost, const double* src, const double* dst, const double* nor, int64_t n,
                          double* pose16_out) {
  if (!src || !dst || n <= 0 || !pose16_out) return fail(MVICP_ERR_INVALID, "mvicp_pairwise_closed: bad arguments");
  if (cost != MVICP_COST_P2P && cost != MVICP_COST_P2PLANE) return fail(MVICP_ERR_INVALID, "mvicp_pairwise_closed: cost must be P2P or P2PLANE");
  if (cost == MVICP_COST_P2PLANE && !nor) return fail(MVICP_ERR_INVALID, "mvicp_pairwise_closed: point-to-plane needs dst normals");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) return fail(MVICP_ERR_CUDA, "no CUDA device; this engine has no CPU path");
  const int dev = cfg ? cfg->device : 0;
  if (dev < 0 || dev >= ndev) return fail(MVICP_ERR_INVALID, "mvicp_pairwise_closed: bad device %d", dev);
  CU(cudaSetDevice(dev));
  cudaStream_t st = cfg && cfg->stream ? (cudaStream_t)cfg->stream : nullptr;
  const size_t bytes = sizeof(double) * 3 * (size_t)n;
  const int grid = (int)std::min<int64_t>(2 * NUM_SMS, (n + CLOSED_THREADS - 1) / CLOSED_THREADS);
  double *d_src = nullptr, *d_dst = nullptr, *d_nor = nullptr, *d_part = nullptr, *d_aux = nullptr;
  std::vector<double> part((size_t)grid * CLOSED_MAXV);
  auto cleanup = [&]() { cudaFree(d_src); cudaFree(d_dst); cudaFree(d_nor); cudaFree(d_part); cudaFree(d_aux); };
#define CUX(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { cleanup(); return fail(MVICP_ERR_CUDA, "%s: %s", #x, cudaGetErrorString(e_)); } } while (0)
  CUX(cudaMalloc(&d_src, bytes)); CUX(cudaMalloc(&d_dst, bytes)); CUX(cudaMalloc(&d_part, sizeof(double) * part.size())); CUX(cudaMalloc(&d_aux, sizeof(double) * 6));
  CUX(cudaMemcpyAsync(d_src, src, bytes, cudaMemcpyHostToDevice, st)); CUX(cudaMemcpyAsync(d_dst, dst, bytes, cudaMemcpyHostToDevice, st));
  if (cost == MVICP_COST_P2PLANE) { CUX(cudaMalloc(&d_nor, bytes)); CUX(cudaMemcpyAsync(d_nor, nor, bytes, cudaMemcpyHostToDevice, st)); }
  auto fetch = [&](int nv, double* out) -> int {   // per-CTA partials, summed in CTA order
    if (cudaMemcpyAsync(part.data(), d_part, sizeof(double) * part.size(), cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) return 1;
    for (int i = 0; i < nv; ++i) { double s = 0; for (int b = 0; b < grid; ++b) s += part[(size_t)b * CLOSED_MAXV + i]; out[i] = s; }
    return 0;
  };
  for (int i = 0; i < 16; ++i) pose16_out[i] = 0.0;
  pose16_out[15] = 1.0;
  if (cost == MVICP_COST_P2P) {
    double sums[6], K9[9];
    closed_reduce_kernel<0><<<grid, CLOSED_THREADS, 0, st>>>(d_src, d_dst, nullptr, (long long)n, nullptr, d_part);
    if (fetch(6, sums)) { cleanup(); return fail(MVICP_ERR_CUDA, "mvicp_pairwise_closed: reduction failed: %s", cudaGetErrorString(cudaGetLastError())); }
    for (int i = 0; i < 6; ++i) sums[i] /= (double)n;            // pbar, qbar
    CUX(cudaMemcpyAsync(d_aux, sums, sizeof sums, cudaMemcpyHostToDevice, st));
    closed_reduce_kernel<1><<<grid, CLOSED_THREADS, 0, st>>>(d_src, d_dst, nullptr, (long long)n, d_aux, d_part);
    if (fetch(9, K9)) { cleanup(); return fail(MVICP_ERR_CUDA, "mvicp_pairwise_closed: reduction failed: %s", cudaGetErrorString(cudaGetLastError())); }
    // R = U V^T with K = U S V^T (icp-closedform.cpp:18-19, JacobiSVD).  V and S^2 come from the symmetric eigen-decomposition of
    // K^T K; u_j = K v_j / s_j only for the two largest singular values, u_3 = +-(u_1 x u_2) with the sign that keeps s_3 >= 0:
    // a rank-deficient K (coplanar / collinear centred clouds, n < 3) then still yields an orthonormal U as the reference's SVD
    // does, and a thin cloud does not pay the squared condition number on its smallest singular value.  Then the reference's
    // `R.col(2) *= -1` when det R < 0 (icp-closedform.cpp:20-22); t = qbar - R pbar
    double S[3][3], w[3], V[3][3], R[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) { S[a][b] = 0; for (int k = 0; k < 3; ++k) S[a][b] += K9[3 * k + a] * K9[3 * k + b]; }
    host_eig_sym3(S, w, V);
    int ord[3] = {0, 1, 2};
    std::sort(ord, ord + 3, [&](int x, int y) { return w[x] > w[y]; });
    double U[3][3], Vs[3][3];   // columns j = singular triplets, descending
    for (int j = 0; j < 3; ++j) for (int a = 0; a < 3; ++a) Vs[a][j] = V[a][ord[j]];
    auto Kv = [&](int j, double out[3]) { for (int a = 0; a < 3; ++a) { out[a] = 0; for (int k = 0; k < 3; ++k) out[a] += K9[3 * a + k] * Vs[k][j]; } };
    auto nrm = [](const double v[3]) { return std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); };
    double u0[3], u1[3], u2[3];
    Kv(0, u0); const double s0 = nrm(u0);
    if (s0 > 0) { for (int a = 0; a < 3; ++a) u0[a] /= s0; } else { u0[0] = 1; u0[1] = u0[2] = 0; }
    Kv(1, u1);
    { const double d = u1[0] * u0[0] + u1[1] * u0[1] + u1[2] * u0[2]; for (int a = 0; a < 3; ++a) u1[a] -= d * u0[a]; }
    double s1 = nrm(u1);
    if (s1 > 1e-13 * s0 && s1 > 0) { for (int a = 0; a < 3; ++a) u1[a] /= s1; }
    else {   // rank <= 1: any unit vector orthogonal to u0
      const int m = std::fabs(u0[0]) <= std::fabs(u0[1]) ? (std::fabs(u0[0]) <= std::fabs(u0[2]) ? 0 : 2) : (std::fabs(u0[1]) <= std::fabs(u0[2]) ? 1 : 2);
      double e[3] = {0, 0, 0}; e[m] = 1;
      const double d = u0[m]; for (int a = 0; a < 3; ++a) u1[a] = e[a] - d * u0[a];
      s1 = nrm(u1); for (int a = 0; a < 3; ++a) u1[a] /= s1;
    }
    u2[0] = u0[1] * u1[2] - u0[2] * u1[1]; u2[1] = u0[2] * u1[0] - u0[0] * u1[2]; u2[2] = u0[0] * u1[1] - u0[1] * u1[0];
    {   // sign of u_3: s_3 = u_3 . K v_3 >= 0; when s_3 vanishes (rank-deficient K) either sign is an SVD -- take the proper rotation
      double k2[3]; Kv(2, k2);
      const double s2 = k2[0] * u2[0] + k2[1] * u2[1] + k2[2] * u2[2];
      const double detV = Vs[0][0] * (Vs[1][1] * Vs[2][2] - Vs[1][2] * Vs[2][1]) - Vs[0][1] * (Vs[1][0] * Vs[2][2] - Vs[1][2] * Vs[2][0]) +
                          Vs[0][2] * (Vs[1][0] * Vs[2][1] - Vs[1][1] * Vs[2][0]);
      const bool neg = std::fabs(s2) > 1e-13 * s0 ? s2 < 0 : detV < 0;
      if (neg) for (int a = 0; a < 3; ++a) u2[a] = -u2[a];
    }
    for (int a = 0; a < 3; ++a) { U[a][0] = u0[a]; U[a][1] = u1[a]; U[a][2] = u2[a]; }
    for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) for (int j = 0; j < 3; ++j) R[a][b] += U[a][j] * Vs[b][j];
    const double det = R[0][0] * (R[1][1] * R[2][2] - R[1][2] * R[2][1]) - R[0][1] * (R[1][0] * R[2][2] - R[1][2] * R[2][0]) + R[0][2] * (R[1][0] * R[2][1] - R[1][1] * R[2][0]);
    if (det < 0) for (int a = 0; a < 3; ++a) R[a][2] = -R[a][2];
    for (int a = 0; a < 3; ++a) {
      for (int b = 0; b < 3; ++b) pose16_out[4 * b + a] = R[a][b];
      pose16_out[12 + a] = sums[3 + a] - (R[a][0] * sums[0] + R[a][1] * sums[1] + R[a][2] * sums[2]);
    }
    for (int i = 0; i < 16; ++i) if (!std::isfinite(pose16_out[i])) { cleanup(); return fail(MVICP_ERR_INVALID, "mvicp_pairwise_closed: non-finite result (non-finite input?)"); }
  } else {
    double v[27];
    closed_reduce_kernel<2><<<grid, CLOSED_THREADS, 0, st>>>(d_src, d_dst, d_nor, (long long)n, nullptr, d_part);
    if (fetch(27, v)) { cleanup(); return fail(MVICP_ERR_CUDA, "mvicp_pairwise_closed: reduction failed: %s", cudaGetErrorString(cudaGetLastError())); }
    double Cm[6][6], L[6][6] = {{0}}, D[6], y[6], x[6];
    { int k = 0; for (int r = 0; r < 6; ++r) for (int c2 = r; c2 < 6; ++c2) { Cm[r][c2] = v[k]; Cm[c2][r] = v[k]; ++k; } }
    for (int j = 0; j < 6; ++j) {      // LDL^T (icp-closedform.cpp:46)
      double dj = Cm[j][j]; for (int k = 0; k < j; ++k) dj -= L[j][k] * L[j][k] * D[k];
      D[j] = dj; L[j][j] = 1;
      for (int i = j + 1; i < 6; ++i) { double u = Cm[i][j]; for (int k = 0; k < j; ++k) u -= L[i][k] * L[j][k] * D[k]; L[i][j] = u / dj; }
    }
    for (int i = 0; i < 6; ++i) { y[i] = v[21 + i]; for (int k = 0; k < i; ++k) y[i] -= L[i][k] * y[k]; }
    for (int i = 5; i >= 0; --i) { x[i] = y[i] / D[i]; for (int k = i + 1; k < 6; ++k) x[i] -= L[k][i] * x[k]; }
    const double ca = std::cos(x[0]), sa = std::sin(x[0]), cb = std::cos(x[1]), sb = std::sin(x[1]), cg = std::cos(x[2]), sg = std::sin(x[2]);
    const double R[3][3] = {{cb * cg, -cb * sg, sb}, {sa * sb * cg + ca * sg, -sa * sb * sg + ca * cg, -sa * cb}, {-ca * sb * cg + sa * sg, ca * sb * sg + sa * cg, ca * cb}};
    for (int a = 0; a < 3; ++a) { for (int b = 0; b < 3; ++b) pose16_out[4 * b + a] = R[a][b]; pose16_out[12 + a] = x[3 + a]; }   // Rx Ry Rz, t (:48-52)
    for (int i = 0; i < 16; ++i) if (!std::isfinite(pose16_out[i])) { cleanup(); return fail(MVICP_ERR_INVALID, "mvicp_pairwise_closed: singular point-to-plane system (degenerate surface)"); }
  }
#undef CUX
  cleanup();
  return MVICP_OK;
}

// ---- normal estimation (SURVEY 8(f) row 1) ---------------------------------------------------------------
int mvicp_recompute_normals(mvicp_ctx* c, int32_t k) {
  if (!c || !c->M) return fail(MVICP_ERR_STATE, "mvicp_recompute_normals: frames must be set first");
  if (k < 3 || k > KNN_MAXK) return fail(MVICP_ERR_INVALID, "mvicp_recompute_normals: k must be in [3, %d] (pointSetPCA asserts >= 3)", KNN_MAXK);
  CU(cudaSetDevice(c->device));
  CU(cudaStreamSynchronize(c->stream));
  c->nor_dbl.resize(c->M, nullptr);
  cudaEvent_t e0 = c->ev[5], e1 = c->ev[6];
  CU(cudaEventRecord(e0, c->stream));
  for (int f = 0; f < c->M; ++f) {
    const int n = (int)c->n_pts[f];
    if (!c->nor_dbl[f]) { CU(cudaMalloc(&c->nor_dbl[f], sizeof(double) * 3 * (size_t)n)); c->frame_allocs.push_back(c->nor_dbl[f]); }
    if (c->f32) normals_kernel<true><<<(n + 127) / 128, 128, 0, c->stream>>>(c->d_frames.as<FrameDev>(), f, k, (double*)c->nor_dbl[f], nullptr);
    else normals_kernel<false><<<(n + 127) / 128, 128, 0, c->stream>>>(c->d_frames.as<FrameDev>(), f, k, (double*)c->nor_dbl[f], nullptr);
    // the LM kernels gather normals as records: recomputed normals are not fp32-exact, so they become 32-byte fp64 records
    void* rec = nullptr;
    if (c->nor_f32 || !c->h_frames[f].nor_o) { CU(cudaMalloc(&rec, sizeof(double4a) * (size_t)n)); c->frame_allocs.push_back(rec); }
    else rec = const_cast<void*>(c->h_frames[f].nor_o);
    pack_normals_kernel<<<(n + 255) / 256, 256, 0, c->stream>>>((const double*)c->nor_dbl[f], n, (double4a*)rec);
    c->h_frames[f].nor_o = rec;
    c->stats.kernel_launches += 2;
  }
  CU(cudaEventRecord(e1, c->stream));
  CU(cudaMemcpyAsync(c->d_frames.p, c->h_frames.data(), sizeof(FrameDev) * c->M, cudaMemcpyHostToDevice, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  CU(cudaGetLastError());
  cudaEventElapsedTime(&c->normals_ms, e0, e1);
  c->nor_f32 = false; c->have_normals = true;
  return MVICP_OK;
}

int mvicp_get_normals(mvicp_ctx* c, int32_t frame, double* nor_xyz, float* elapsed_ms) {
  if (!c || frame < 0 || frame >= c->M || !nor_xyz) return fail(MVICP_ERR_INVALID, "mvicp_get_normals: bad arguments");
  if ((int)c->nor_dbl.size() <= frame || !c->nor_dbl[frame]) return fail(MVICP_ERR_STATE, "mvicp_get_normals: call mvicp_recompute_normals first");
  CU(cudaSetDevice(c->device));
  CU(cudaMemcpy(nor_xyz, c->nor_dbl[frame], sizeof(double) * 3 * (size_t)c->n_pts[frame], cudaMemcpyDeviceToHost));
  if (elapsed_ms) *elapsed_ms = c->normals_ms;
  return MVICP_OK;
}

// Frame::getNeighbours for every point of one frame (frame.cpp:208-242): the k nearest neighbours, knnSearch order.
int mvicp_knn_self(mvicp_ctx* c, int32_t frame, int32_t k, int32_t* nn_idx) {
  if (!c || frame < 0 || frame >= c->M || !nn_idx || k < 1 || k > KNN_MAXK) return fail(MVICP_ERR_INVALID, "mvicp_knn_self: bad arguments");
  CU(cudaSetDevice(c->device));
  const int n = (int)c->n_pts[frame];
  double* d_nor = nullptr; int32_t* d_nn = nullptr;
  CU(cudaMalloc(&d_nor, sizeof(double) * 3 * (size_t)n)); CU(cudaMalloc(&d_nn, sizeof(int32_t) * (size_t)k * n));
  if (c->f32) normals_kernel<true><<<(n + 127) / 128, 128, 0, c->stream>>>(c->d_frames.as<FrameDev>(), frame, k, d_nor, d_nn);
  else normals_kernel<false><<<(n + 127) / 128, 128, 0, c->stream>>>(c->d_frames.as<FrameDev>(), frame, k, d_nor, d_nn);
  c->stats.kernel_launches += 1;
  CU(cudaMemcpyAsync(nn_idx, d_nn, sizeof(int32_t) * (size_t)k * n, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  cudaFree(d_nor); cudaFree(d_nn);
  CU(cudaGetLastError());
  return MVICP_OK;
}

int mvicp_get_normals_device(mvicp_ctx* c, int32_t frame, double* nor_xyz) {
  if (!c || frame < 0 || frame >= c->M || !nor_xyz) return fail(MVICP_ERR_INVALID, "mvicp_get_normals_device: bad arguments");
  if ((int)c->nor_dbl.size() <= frame || !c->nor_dbl[frame]) return fail(MVICP_ERR_STATE, "mvicp_get_normals_device: call mvicp_recompute_normals first");
  CU(cudaSetDevice(c->device));
  RET(check_device_ptr(c, nor_xyz, "mvicp_get_normals_device", "nor_xyz"));
  CU(cudaMemcpyAsync(nor_xyz, c->nor_dbl[frame], sizeof(double) * 3 * (size_t)c->n_pts[frame], cudaMemcpyDeviceToDevice, c->stream));
  return MVICP_OK;
}

// mvicp_knn_self into the caller's device buffer; the normals the kernel computes on the way go to a reusable context buffer
int mvicp_knn_self_device(mvicp_ctx* c, int32_t frame, int32_t k, int32_t* nn_idx) {
  if (!c || frame < 0 || frame >= c->M || !nn_idx || k < 1 || k > KNN_MAXK) return fail(MVICP_ERR_INVALID, "mvicp_knn_self_device: bad arguments");
  CU(cudaSetDevice(c->device));
  RET(check_device_ptr(c, nn_idx, "mvicp_knn_self_device", "nn_idx"));
  const int n = (int)c->n_pts[frame];
  RET(c->d_knn_nor.reserve(sizeof(double) * 3 * (size_t)n));
  if (c->f32) normals_kernel<true><<<(n + 127) / 128, 128, 0, c->stream>>>(c->d_frames.as<FrameDev>(), frame, k, c->d_knn_nor.as<double>(), nn_idx);
  else normals_kernel<false><<<(n + 127) / 128, 128, 0, c->stream>>>(c->d_frames.as<FrameDev>(), frame, k, c->d_knn_nor.as<double>(), nn_idx);
  c->stats.kernel_launches += 1;
  CU(cudaGetLastError());
  return MVICP_OK;
}

// ---- multi-GPU ---------------------------------------------------------------------------------------
int mvicp_nccl_unique_id(void* out128) {
  if (!out128) return fail(MVICP_ERR_INVALID, "mvicp_nccl_unique_id: null");
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  ncclUniqueId id; NC(ncclGetUniqueId(&id));
  std::memcpy(out128, &id, 128);
  return MVICP_OK;
}

int mvicp_comm_init(mvicp_ctx* c, const void* id128, int32_t rank, int32_t world) {
  if (!c || !id128 || world < 1 || rank < 0 || rank >= world) return fail(MVICP_ERR_INVALID, "mvicp_comm_init: bad arguments");
  CU(cudaSetDevice(c->device));
  if (c->comm) { ncclCommDestroy(c->comm); c->comm = nullptr; }
  ncclUniqueId id; std::memcpy(&id, id128, 128);
  if (world > 1) NC(ncclCommInitRank(&c->comm, world, id, rank));
  c->rank = rank; c->world = world;
  c->p2p_ok = false;
  if (world > 1 && world <= MAX_PEERS && !(c->flags & MVICP_FLAG_NCCL_ONLY)) {
    // exchange buffer in this rank's memory, mapped into every peer through CUDA IPC (handles travel over NCCL)
    const size_t xbytes = sizeof(double) * 2 * (size_t)mvicp_ctx::X_ECAP * EOUT + 256;
    bool ok = true;
    if (!c->xbuf) ok = cudaMalloc(&c->xbuf, xbytes) == cudaSuccess;
    if (ok) ok = cudaMemset(c->xbuf, 0, xbytes) == cudaSuccess;
    cudaIpcMemHandle_t mine; std::memset(&mine, 0, sizeof mine);
    if (ok) ok = cudaIpcGetMemHandle(&mine, c->xbuf) == cudaSuccess;
    void* d_h = nullptr;
    std::vector<cudaIpcMemHandle_t> all(world);
    int32_t okflag = ok ? 1 : 0;
    if (cudaMalloc(&d_h, sizeof(cudaIpcMemHandle_t) * (world + 1) + 64) != cudaSuccess) return fail(MVICP_ERR_CUDA, "comm_init: cudaMalloc");
    char* dh = (char*)d_h;
    struct Guard { void* p; ~Guard() { cudaFree(p); } } guard{d_h};   // released on every return path below
    CU(cudaMemcpy(dh, &mine, sizeof mine, cudaMemcpyHostToDevice));
    NC(ncclAllGather(dh, dh + sizeof(cudaIpcMemHandle_t), sizeof(cudaIpcMemHandle_t), ncclUint8, c->comm, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    CU(cudaMemcpy(all.data(), dh + sizeof(cudaIpcMemHandle_t), sizeof(cudaIpcMemHandle_t) * world, cudaMemcpyDeviceToHost));
    for (int p = 0; p < world && ok; ++p) {
      if (p == rank) { c->peer_x[p] = c->xbuf; continue; }
      if (!c->peer_x[p]) ok = cudaIpcOpenMemHandle(&c->peer_x[p], all[p], cudaIpcMemLazyEnablePeerAccess) == cudaSuccess;
    }
    cudaGetLastError();
    // every rank must agree, or the flag protocol would wait for a rank that took the NCCL path
    okflag = ok ? 1 : 0;
    int32_t* d_ok = (int32_t*)(dh + sizeof(cudaIpcMemHandle_t) * (world + 1));
    CU(cudaMemcpy(d_ok, &okflag, sizeof okflag, cudaMemcpyHostToDevice));
    NC(ncclAllReduce(d_ok, d_ok, 1, ncclInt32, ncclMin, c->comm, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    CU(cudaMemcpy(&okflag, d_ok, sizeof okflag, cudaMemcpyDeviceToHost));
    c->p2p_ok = okflag == 1;
    c->xseq = 0;
  }
  return rebuild_work(c);
}

// ---- introspection -------------------------------------------------------------------------------------
int mvicp_get_stats(mvicp_ctx* c, mvicp_stats* out) {
  if (!c || !out) return fail(MVICP_ERR_INVALID, "mvicp_get_stats: bad arguments");
  CU(cudaSetDevice(c->device));
  CU(cudaStreamSynchronize(c->stream));
  if (c->ev_knn) {
    cudaEventElapsedTime(&c->stats.knn_ms, c->ev[0], c->ev[1]);
    cudaEventElapsedTime(&c->stats.select_ms, c->ev[1], c->ev[2]);
    c->stats.correspond_ms = c->stats.knn_ms + c->stats.select_ms;
  }
  if (c->ev_lm) {
    cudaEventElapsedTime(&c->stats.optimize_ms, c->ev[3], c->ev[4]);
    float acc = 0.f;
    for (int i = 0; i + 1 < c->eval_ev_used; i += 2) { float ms = 0.f; cudaEventElapsedTime(&ms, c->eval_ev[i], c->eval_ev[i + 1]); acc += ms; }
    c->stats.lm_eval_ms = acc; c->stats.lm_other_ms = c->stats.optimize_ms - acc;
  }
  if (c->E && fetch_edge_meta(c) == MVICP_OK) {
    int64_t s = 0; for (int e = 0; e < c->E; ++e) if (c->h_edges[e].owned) s += (int64_t)c->h_count[e];
    c->stats.correspondences = s;
  }
  c->stats.select_guess_rounds = c->sel_guess_rounds;
  c->stats.cert_rounds = c->cert_rounds;
  if (c->d_cert_cnt.p && c->E) {
    std::vector<unsigned long long> h(c->E);
    CU(cudaMemcpy(h.data(), c->d_cert_cnt.p, sizeof(unsigned long long) * c->E, cudaMemcpyDeviceToHost));
    int64_t s = 0; for (unsigned long long v : h) s += (int64_t)v;
    c->stats.cert_reused = s;
  }
  if (c->d_sel_cnt.p && c->E) {
    unsigned int miss = 0;
    CU(cudaMemcpy(&miss, c->d_sel_cnt.as<unsigned int>() + 2 * (size_t)c->E, sizeof miss, cudaMemcpyDeviceToHost));
    c->stats.select_guess_misses = miss;
  }
  *out = c->stats;
  return MVICP_OK;
}
// development aid: the 16 clock64() stamps lm_step_kernel left when MVICP_STEP_PROFILE=1 (0..7 phase boundaries, 8..10 Cholesky parts)
int mvicp_debug_step_profile(mvicp_ctx* c, long long* out64) {
  if (!c || !out64 || !c->d_prof.p) return fail(MVICP_ERR_STATE, "mvicp_debug_step_profile: run with MVICP_STEP_PROFILE=1");
  CU(cudaSetDevice(c->device));
  CU(cudaMemcpy(out64, c->d_prof.p, sizeof(long long) * 64, cudaMemcpyDeviceToHost));
  return MVICP_OK;
}
// development aid: the per-edge output of the last LM (or g2o, below) evaluation, E x 160 doubles (EOUT), as lm_edge_kernel /
// lm_edge_general_kernel wrote it and gather_blocks / gather_gradient / edge_cost_sum read it.  Edge e's record:
//   [0, 144)    the 12x12 pair matrix Hp, row-major; rows and columns 0-5 are the src frame's tangent, 6-11 the dst frame's
//               (lm_step's sub-blocks ss | sk over ks | kk)
//   [144, 156)  the pair gradient: 6 src entries, then 6 dst entries
//   156         the edge's cost, 1/2 sum rho(|r|^2) (1/2 sum |r|^2 without the loss);  157-159 zero
// Each 6-vector is in the parameterisation's own tangent order: angle-axis (dw, dt), quaternion (dq, dt), SE3 (upsilon,
// omega).  An edge whose src frame is fixed contributes nothing and reads as zeros: lm_edge_kernel writes zeros for it in a
// joint solve, but in a component solve the edges of a component without a free frame belong to no problem and are never
// written, so the readout zeroes every such record itself.  The blocks are those of the LAST evaluation: after
// mvicp_optimize with max_num_iterations = 0 the start point; after a rejected step the rejected candidate.  The evaluation
// enqueued behind a finished solve is skipped by its DoneGate and leaves them alone.  In a component solve each edge holds its
// own problem's last evaluation.
// After mvicp_optimize_g2o / mvicp_optimize_g2o_components the records are g2o_edge_kernel's, in the same layout: the pair
// matrix over [src | dst] and the gradient sum J^T Omega e (g2o's b is -g), both in g2o's increment order (tx ty tz qx qy
// qz); slot 156 the edge's chi2 sum e^T Omega e (no 1/2); 157-159 zero.  Slots 0-155 come from the last build of the edge's
// problem, slot 156 from its last evaluation, build or trial (a trial writes only slot 156).  An edge out of a fixed frame
// into a free one is active and reads as its full record; an edge between two fixed frames reads as zeros.  The edges of a
// component without a g2o problem, and every edge when no problem has a vertex, are never written and read as zeros.
// MVICP_ERR_STATE before any LM or g2o solve has evaluated since the graph was set, after a solve that failed once it had
// started, and in a sharded context.  A call refused for its arguments (state, cost, normals, options) touches nothing, so
// the previous solve's records stay readable after it.  Launches nothing and changes no state.
int mvicp_debug_edge_blocks(mvicp_ctx* c, double* out, int64_t capacity, int32_t* n_edges) {
  if (!c || !n_edges) return fail(MVICP_ERR_INVALID, "mvicp_debug_edge_blocks: bad arguments");
  if (c->world > 1) return fail(MVICP_ERR_STATE, "mvicp_debug_edge_blocks: the context is sharded");
  if (!c->lm_blocks_E || c->lm_blocks_E != c->E) return fail(MVICP_ERR_STATE, "mvicp_debug_edge_blocks: no completed LM or g2o solve since the graph was set");
  *n_edges = c->E;
  if (!out) return MVICP_OK;
  if (capacity < (int64_t)EOUT * c->E) return fail(MVICP_ERR_INVALID, "mvicp_debug_edge_blocks: capacity %lld < %lld", (long long)capacity, (long long)EOUT * c->E);
  CU(cudaSetDevice(c->device));
  CU(cudaStreamSynchronize(c->stream));
  const size_t rec = sizeof(double) * EOUT;
  if (!c->blocks_g2o) {
    CU(cudaMemcpy(out, c->d_eout.p, rec * c->E, cudaMemcpyDeviceToHost));
    for (int e = 0; e < c->E; ++e)
      if (c->lm_blocks_fixed[c->h_edges[e].src]) std::memset(out + (size_t)EOUT * e, 0, rec);
    return MVICP_OK;
  }
  bool any = false;   // a g2o solve without a vertex evaluated nothing (and may have found no d_eout)
  for (int e = 0; e < c->E; ++e) any = any || !c->g2o_blocks_unwritten[e];
  if (any) CU(cudaMemcpy(out, c->d_eout.p, rec * c->E, cudaMemcpyDeviceToHost));
  for (int e = 0; e < c->E; ++e) {
    double* o = out + (size_t)EOUT * e;
    if (c->g2o_blocks_unwritten[e]) std::memset(o, 0, rec);
    else o[157] = o[158] = o[159] = 0.0;   // g2o_edge_kernel writes slots 0-156 only
  }
  return MVICP_OK;
}
int mvicp_get_stream(mvicp_ctx* c, void** stream) { if (!c || !stream) return fail(MVICP_ERR_INVALID, "bad arguments"); *stream = (void*)c->stream; return MVICP_OK; }
int mvicp_sync(mvicp_ctx* c) { if (!c) return fail(MVICP_ERR_INVALID, "null ctx"); CU(cudaSetDevice(c->device)); CU(cudaStreamSynchronize(c->stream)); return MVICP_OK; }

}  // extern "C"
