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
#include "far.cuh"
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

struct DevBuf {
  void* p = nullptr; size_t cap = 0;
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
  DevBuf d_prof;               // lm_step_kernel's clock stamps (MVICP_STEP_PROFILE=1)
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
  DevBuf d_state, d_x, d_cand, d_Rt, d_K, d_col, d_H, d_g, d_Hc, d_gc, d_scale, d_diag, d_L, d_rhs, d_step,
      d_eout, d_hb_ptr, d_hb_row, d_hb_col, d_hc_edge, d_hc_sub, d_gb_ptr, d_gc_edge, d_gc_side, d_posegather, d_rlast, d_rfirst, d_rowbase, d_gen;
  int64_t l_size = 0;          // doubles of the factor's skyline storage (row profiles + rhs row)
  int n_free = 0, n_hblocks = 0;
  std::vector<int32_t> h_col;
  void* h_state = nullptr;     // pinned staging of LmState
  volatile int32_t* h_flag = nullptr; volatile int32_t* d_flag = nullptr;   // mapped pinned ring written by lm_step_kernel
  std::vector<uint8_t> lm_key; uint32_t graph_gen = 0;
  // stats
  mvicp_stats stats{};
  cudaEvent_t ev[8]{};
  std::vector<cudaEvent_t> eval_ev;   // pairs around every lm_eval launch of the last optimize
  int eval_ev_used = 0;
  bool ev_knn = false, ev_lm = false;
  float lm_eval_acc = 0.f;
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
  c->E = 0; c->h_edges.clear(); c->have_corr = false;
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

static int set_frames_device(mvicp_ctx* c, int M, const double* const* pts, const double* const* nor, const int64_t* n_pts) {
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
    if (err == cudaSuccess) err = cudaMemcpyAsync(d_xyz[f], pts[f], bytes, cudaMemcpyHostToDevice, c->stream);
    if (err == cudaSuccess) kd_scan_kernel<<<2 * NUM_SMS, 256, 0, c->stream>>>(d_xyz[f], 3ll * n_pts[f], d_flags + 4 * f);
    if (err == cudaSuccess && nor && nor[f]) {
      err = cudaMalloc(&d_nor[f], bytes);
      if (err == cudaSuccess) err = cudaMemcpyAsync(d_nor[f], nor[f], bytes, cudaMemcpyHostToDevice, c->stream);
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
    CU(cudaMallocHost(&c->h_state, sizeof(LmState)));
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
  DevBuf* bufs[] = {&c->d_frames, &c->d_poses, &c->d_edges, &c->d_xf, &c->d_corr, &c->d_d2, &c->d_count, &c->d_sel, &c->d_hist,
                    &c->d_weight, &c->d_median, &c->d_selcand, &c->d_selcand_n, &c->d_sel_cnt, &c->d_sel_win, &c->d_certs, &c->d_cert_cnt, &c->d_todo, &c->d_todo_n, &c->d_knn_tiles, &c->d_eval_tiles, &c->d_edge_tile_begin, &c->d_partial,
                    &c->d_state, &c->d_x, &c->d_cand, &c->d_Rt, &c->d_K, &c->d_col, &c->d_H, &c->d_g, &c->d_Hc,
                    &c->d_gc, &c->d_scale, &c->d_diag, &c->d_L, &c->d_rhs, &c->d_step, &c->d_eout,
                    &c->d_hb_ptr, &c->d_hb_row, &c->d_hb_col, &c->d_hc_edge, &c->d_hc_sub, &c->d_gb_ptr, &c->d_gc_edge,
                    &c->d_gc_side, &c->d_posegather, &c->d_rlast, &c->d_rfirst, &c->d_rowbase, &c->d_gen, &c->d_obb, &c->d_single, &c->d_prof, &c->d_tile_count, &c->d_tile_off, &c->d_edge_off, &c->d_recs};
  for (DevBuf* b : bufs) b->release();
  for (auto& ev : c->ev) if (ev) cudaEventDestroy(ev);
  for (auto& ev : c->eval_ev) cudaEventDestroy(ev);
  if (c->h_state) cudaFreeHost(c->h_state);
  if (c->h_flag) cudaFreeHost((void*)c->h_flag);

  if (c->own_stream && c->stream) cudaStreamDestroy(c->stream);
  delete c;
}

int mvicp_set_frames(mvicp_ctx* c, int32_t M, const double* const* pts, const double* const* nor, const int64_t* n_pts) {
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
  if (!(c->flags & MVICP_FLAG_HOST_BUILD)) { RET(set_frames_device(c, M, pts, nor, n_pts)); return finish_set_frames(c, M); }
#endif
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
  int tl = 8192;
  while (tl > 1024 && active_slots / tl < 8 * NUM_SMS) tl >>= 1;
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
  c->E = E; c->h_edges.assign(E, EdgeDev{});
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
    if (far && ww) knn_far_kernel<F32, true><<<c->n_knn_tiles, KNN_TILE, 0, c->stream>>>(MV_KNN_ARGS, c->d_obb.as<ObbDev>());
    else if (far) knn_far_kernel<F32, false><<<c->n_knn_tiles, KNN_TILE, 0, c->stream>>>(MV_KNN_ARGS, c->d_obb.as<ObbDev>());
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

int mvicp_get_all_edges(mvicp_ctx* c, void* out_records, int64_t capacity, int64_t* offsets, float* weights) {
  if (!c || !c->E || !offsets) return fail(MVICP_ERR_INVALID, "mvicp_get_all_edges: bad arguments / no graph");
  if (!c->have_corr) return fail(MVICP_ERR_STATE, "mvicp_get_all_edges: call mvicp_correspond first");
  CU(cudaSetDevice(c->device));
  const int E = c->E, nt = c->n_knn_tiles;
  RET(c->d_tile_count.reserve(sizeof(unsigned int) * std::max(1, nt)));
  RET(c->d_tile_off.reserve(sizeof(unsigned long long) * std::max(1, nt)));
  RET(c->d_edge_off.reserve(sizeof(unsigned long long) * (E + 1)));
  if (nt) compact_count_kernel<<<nt, KNN_TILE, 0, c->stream>>>(c->d_edges.as<EdgeDev>(), c->d_knn_tiles.as<Tile>(), c->d_corr.as<int32_t>(), c->d_tile_count.as<unsigned int>());
  compact_scan_kernel<<<1, 1024, 0, c->stream>>>(c->d_tile_count.as<unsigned int>(), nt, c->d_knn_tiles.as<Tile>(), E,
                                                 c->d_tile_off.as<unsigned long long>(), c->d_edge_off.as<unsigned long long>());
  c->stats.kernel_launches += nt ? 2 : 1;
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

// ---- LM ------------------------------------------------------------------------------------------
static int prepare_lm(mvicp_ctx* c, int n) {
  const int M = c->M, E = c->E;
  RET(c->d_state.reserve(sizeof(LmState)));
  RET(c->d_x.reserve(sizeof(double) * 7 * M)); RET(c->d_cand.reserve(sizeof(double) * 7 * M));
  RET(c->d_Rt.reserve(sizeof(Rt) * M)); RET(c->d_K.reserve(sizeof(double) * 36 * M));
  RET(c->d_col.reserve(sizeof(int32_t) * M));
  RET(c->d_H.reserve(sizeof(double) * n * n)); RET(c->d_Hc.reserve(sizeof(double) * n * n));
  RET(c->d_g.reserve(sizeof(double) * n)); RET(c->d_gc.reserve(sizeof(double) * n)); RET(c->d_scale.reserve(sizeof(double) * n));
  RET(c->d_diag.reserve(sizeof(double) * n)); RET(c->d_rhs.reserve(sizeof(double) * n)); RET(c->d_step.reserve(sizeof(double) * n));
  RET(c->d_eout.reserve(sizeof(double) * EOUT * E));
  return MVICP_OK;
}

}  // extern "C"
template <bool F32> static void launch_eval(mvicp_ctx* c, int cost, int robust, const int* done_flag) {
  const int nt = c->n_eval_tiles;
  if (!nt) return;
#define MV_EVAL(NF, COSTK)                                                                                       \
  lm_eval_kernel<F32, NF, COSTK><<<nt, EVAL_THREADS, 0, c->stream>>>(                                            \
      c->d_frames.as<FrameDev>(), c->d_edges.as<EdgeDev>(), c->d_eval_tiles.as<Tile>(), c->eval_tile_len,       \
      c->d_corr.as<int32_t>(), c->d_Rt.as<Rt>(), c->d_weight.as<float>(), robust, c->d_partial.as<double>(), done_flag)
#define MV_EVALC(NF) { if (cost == COST_P2P) MV_EVAL(NF, COST_P2P); else if (cost == COST_P2PLANE) MV_EVAL(NF, COST_P2PLANE); else MV_EVAL(NF, COST_MIXED); }
  if (F32 && c->nor_f32) MV_EVALC(F32) else MV_EVALC(false)
#undef MV_EVALC
#undef MV_EVAL
}

template <bool F32> static void launch_eval_general(mvicp_ctx* c, int param, int cost, int robust, const int* done_flag) {
  const int rot0 = param == PARAM_QUAT ? 0 : 3;   // tangent order: quaternion (rotation, translation), SE3 (translation, rotation)
  const int nt = c->n_eval_tiles;
  if (!nt) return;
#define MV_EVALG(COSTK)                                                                                          \
  if (F32 && c->nor_f32) lm_eval_general_kernel<F32, F32, COSTK><<<nt, EVAL_THREADS, 0, c->stream>>>(        \
      c->d_frames.as<FrameDev>(), c->d_edges.as<EdgeDev>(), c->d_eval_tiles.as<Tile>(), c->eval_tile_len,       \
      c->d_corr.as<int32_t>(), c->d_gen.as<FrameGen>(), c->d_weight.as<float>(), robust, rot0, c->d_partial.as<double>(), done_flag); \
  else lm_eval_general_kernel<F32, false, COSTK><<<nt, EVAL_THREADS, 0, c->stream>>>(                        \
      c->d_frames.as<FrameDev>(), c->d_edges.as<EdgeDev>(), c->d_eval_tiles.as<Tile>(), c->eval_tile_len,       \
      c->d_corr.as<int32_t>(), c->d_gen.as<FrameGen>(), c->d_weight.as<float>(), robust, rot0, c->d_partial.as<double>(), done_flag)
  if (cost == COST_P2P) { MV_EVALG(COST_P2P); } else if (cost == COST_P2PLANE) { MV_EVALG(COST_P2PLANE); } else { MV_EVALG(COST_MIXED); }
#undef MV_EVALG
}
extern "C" {
int mvicp_optimize(mvicp_ctx* c, int32_t param, int32_t cost, int32_t robust, const mvicp_lm_options* opt_in, mvicp_lm_summary* summary) {
  if (!c || !c->M || !c->E) return fail(MVICP_ERR_STATE, "mvicp_optimize: frames and graph must be set first");
  if (param < 0 || param > 2 || cost < 0 || cost > 2) return fail(MVICP_ERR_INVALID, "mvicp_optimize: bad param/cost");
  if (cost != COST_P2P && !c->have_normals) return fail(MVICP_ERR_INVALID, "point-to-plane needs normals for every frame");
  CU(cudaSetDevice(c->device));
  const int M = c->M, E = c->E;
  c->fixed[0] = 1;   // frames[0]->fixed = true (icp-ceres.cpp:242-244,342-344,417-419)
  // local columns of the free frames; edges of fixed src frames contribute nothing (icp-ceres.cpp:255,353,426)
  c->h_col.assign(M, -1); int n = 0;
  for (int f = 0; f < M; ++f) if (!c->fixed[f]) { c->h_col[f] = n; n += 6; }
  c->n_free = n / 6;
  mvicp_lm_options opt; if (opt_in) opt = *opt_in; else mvicp_default_lm_options(&opt);
  if (n == 0) {   // nothing to optimise; still "writes the poses back"
    if (summary) { std::memset(summary, 0, sizeof *summary); summary->termination = MVICP_TERM_GRADIENT_TOLERANCE; }
    return MVICP_OK;
  }
  // ownership may depend on `fixed`: refresh the edge table if it changed
  bool stale = false;
  for (int e = 0; e < E; ++e) {
    if ((c->edge_owner[e] < 0) != (c->fixed[c->h_edges[e].src] != 0)) stale = true;
  }
  if (stale) {
    if (c->world > 1) return fail(MVICP_ERR_STATE, "sharded run: frame 0 was free when the edges were distributed; fix it (mvicp_set_poses) before mvicp_correspond");
    RET(refresh_after_fixed_change(c));
  }
  // the gather lists / envelope depend only on the graph and the fixed flags: build and upload them when those change
  std::vector<uint8_t> key(c->fixed); key.push_back((uint8_t)(c->graph_gen & 0xff)); key.push_back((uint8_t)((c->graph_gen >> 8) & 0xff));
  if (key != c->lm_key) {
  RET(prepare_lm(c, n));
    // block-sparse gather lists
    std::vector<std::vector<std::pair<int, int>>> blk((size_t)M * M);
    std::vector<std::vector<std::pair<int, int>>> gl(M);
    for (int e = 0; e < E; ++e) {
      const int s = c->h_edges[e].src, k = c->h_edges[e].dst;
      if (c->fixed[s]) continue;
      blk[(size_t)s * M + s].push_back({e, 0}); gl[s].push_back({e, 0});
      if (!c->fixed[k]) {
        blk[(size_t)s * M + k].push_back({e, 1}); blk[(size_t)k * M + s].push_back({e, 2}); blk[(size_t)k * M + k].push_back({e, 3});
        gl[k].push_back({e, 1});
      }
    }
    std::vector<int32_t> hb_ptr{0}, hb_row, hb_col, hc_edge, hc_sub, gb_ptr{0}, gc_edge, gc_side;
    for (int r = 0; r < M; ++r)
      for (int q = 0; q < M; ++q) {
        const auto& l = blk[(size_t)r * M + q];
        if (l.empty()) continue;
        hb_row.push_back(c->h_col[r]); hb_col.push_back(c->h_col[q]);
        for (auto& pr : l) { hc_edge.push_back(pr.first); hc_sub.push_back(pr.second); }
        hb_ptr.push_back((int32_t)hc_edge.size());
      }
    for (int f = 0; f < M; ++f) { for (auto& pr : gl[f]) { gc_edge.push_back(pr.first); gc_side.push_back(pr.second); } gb_ptr.push_back((int32_t)gc_edge.size()); }
    c->n_hblocks = (int)hb_row.size();
    // envelope: first structurally non-zero column of every row, and the last row that reaches column j
    std::vector<int32_t> rfirst(n), rlast(n);
    for (int r = 0; r < n; ++r) rfirst[r] = (r / 6) * 6;
    for (int b = 0; b < c->n_hblocks; ++b)
      if (hb_col[b] < hb_row[b]) for (int i = 0; i < 6; ++i) rfirst[hb_row[b] + i] = std::min(rfirst[hb_row[b] + i], hb_col[b]);
    for (int j = 0; j < n; ++j) { rlast[j] = j; }
    for (int r = 0; r < n; ++r) for (int j = rfirst[r]; j <= r; ++j) rlast[j] = std::max(rlast[j], r);
    for (int j = 1; j < n; ++j) rlast[j] = std::max(rlast[j], rlast[j - 1]);   // monotone (fill-in stays inside)
    auto up = [&](DevBuf& b, const std::vector<int32_t>& v) -> int {
      RET(b.reserve(sizeof(int32_t) * std::max<size_t>(1, v.size())));
      if (!v.empty()) CU(cudaMemcpyAsync(b.p, v.data(), sizeof(int32_t) * v.size(), cudaMemcpyHostToDevice, c->stream));
      return MVICP_OK;
    };
    RET(up(c->d_hb_ptr, hb_ptr)); RET(up(c->d_hb_row, hb_row)); RET(up(c->d_hb_col, hb_col)); RET(up(c->d_hc_edge, hc_edge));
    RET(up(c->d_hc_sub, hc_sub)); RET(up(c->d_gb_ptr, gb_ptr)); RET(up(c->d_gc_edge, gc_edge)); RET(up(c->d_gc_side, gc_side));
    RET(up(c->d_col, c->h_col));
    RET(up(c->d_rlast, rlast)); RET(up(c->d_rfirst, rfirst));
    // skyline storage of the Cholesky factor: row r keeps columns rfirst[r]..r, the rhs row all n
    std::vector<int32_t> rowbase(n + 1); int64_t at = 0;
    for (int r = 0; r < n; ++r) { rowbase[r] = (int32_t)(at - rfirst[r]); at += r - rfirst[r] + 1; }
    rowbase[n] = (int32_t)at; at += n;
    if (at > INT32_MAX) return fail(MVICP_ERR_INVALID, "normal matrix too large");
    c->l_size = at;
    RET(c->d_L.reserve(sizeof(double) * (size_t)at));
    RET(up(c->d_rowbase, rowbase));
    // the step kernel writes only the listed blocks of the dense normal matrix; everything else stays zero from here
    CU(cudaMemsetAsync(c->d_H.p, 0, sizeof(double) * (size_t)n * n, c->stream));
    CU(cudaMemsetAsync(c->d_Hc.p, 0, sizeof(double) * (size_t)n * n, c->stream));

    CU(cudaStreamSynchronize(c->stream));   // the host vectors above must outlive their copies
    c->lm_key = key;
  }
  LmState st; std::memset(&st, 0, sizeof st);
  st.opt = opt; st.param = param; st.cost_kind = cost; st.robust = robust ? 1 : 0; st.M = M; st.E = E; st.F = n / 6; st.n = n;
  st.G = ambient_size(param); st.radius = opt.initial_trust_region_radius; st.decrease_factor = 2.0;
  std::memcpy(c->h_state, &st, sizeof st);   // pinned staging: no synchronisation needed before the kernels
  CU(cudaMemcpyAsync(c->d_state.p, c->h_state, sizeof st, cudaMemcpyHostToDevice, c->stream));

  LmWork w{};
  w.S = c->d_state.as<LmState>(); w.edges = c->d_edges.as<EdgeDev>(); w.eout = c->d_eout.as<double>();
  w.host_flag = c->d_flag;
  if (std::getenv("MVICP_STEP_PROFILE")) { RET(c->d_prof.reserve(sizeof(long long) * 64)); w.prof = c->d_prof.as<long long>(); }
  c->nonrigid = poses_nonrigid(c->h_poses.data(), M);   // the mirror follows every solve and every mvicp_set_poses
  const bool general = c->nonrigid && param != PARAM_AA;
  if (general) { RET(c->d_gen.reserve(sizeof(FrameGen) * M)); RET(c->d_partial.reserve(sizeof(double) * GBLK * std::max<size_t>(1, c->n_eval_tiles))); }
  w.G_eval = general ? c->d_gen.as<FrameGen>() : nullptr;
  w.x = c->d_x.as<double>(); w.cand = c->d_cand.as<double>(); w.Rt_eval = c->d_Rt.as<Rt>(); w.K_eval = c->d_K.as<double>();
  w.col = c->d_col.as<int32_t>();
  w.hb_ptr = c->d_hb_ptr.as<int32_t>(); w.hb_row = c->d_hb_row.as<int32_t>(); w.hb_col = c->d_hb_col.as<int32_t>();
  w.hc_edge = c->d_hc_edge.as<int32_t>(); w.hc_sub = c->d_hc_sub.as<int32_t>(); w.n_hblocks = c->n_hblocks;
  w.rlast = c->d_rlast.as<int32_t>(); w.rfirst = c->d_rfirst.as<int32_t>(); w.rowbase = c->d_rowbase.as<int32_t>();
  w.gb_ptr = c->d_gb_ptr.as<int32_t>(); w.gc_edge = c->d_gc_edge.as<int32_t>(); w.gc_side = c->d_gc_side.as<int32_t>();
  w.H = c->d_H.as<double>(); w.g = c->d_g.as<double>(); w.Hc = c->d_Hc.as<double>(); w.gc = c->d_gc.as<double>();
  w.scale = c->d_scale.as<double>(); w.diag = c->d_diag.as<double>(); w.Lg = c->d_L.as<double>(); w.rhs = c->d_rhs.as<double>();
  w.step = c->d_step.as<double>(); w.poses16 = c->d_poses.as<double>();
  const size_t l_bytes = sizeof(double) * (size_t)c->l_size;
  const size_t vec_bytes = sizeof(double) * 3 * (size_t)(n + 1);
  w.l_in_smem = (l_bytes + vec_bytes) <= 220 * 1024 ? 1 : 0;
  const size_t dyn = vec_bytes + (w.l_in_smem ? l_bytes : 0);
  CU(cudaFuncSetAttribute(lm_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));

  CU(cudaEventRecord(c->ev[3], c->stream));
  lm_init_kernel<<<(M + 63) / 64, 64, 0, c->stream>>>(w);
  c->stats.kernel_launches += 1;
  // The loop is pipelined one iteration deep: iteration i+1 is enqueued before the host learns whether iteration i
  // terminated, so the GPU never waits for the host; kernels of an iteration issued after termination exit at once.
  const int max_evals = opt.max_num_iterations + 2;
  for (int i = 0; i < 8; ++i) c->h_flag[i] = 0;
  c->eval_ev_used = 0;
  const bool use_p2p = c->comm && c->world > 1 && c->p2p_ok && E <= mvicp_ctx::X_ECAP;
  int issued = 0, seen = 0;
  const int* done_flag = &w.S->done;
  auto issue = [&]() -> int {
    if ((int)c->eval_ev.size() < c->eval_ev_used + 2) { cudaEvent_t a, b; CU(cudaEventCreate(&a)); CU(cudaEventCreate(&b)); c->eval_ev.push_back(a); c->eval_ev.push_back(b); }
    CU(cudaEventRecord(c->eval_ev[c->eval_ev_used], c->stream));
    if (general) { if (c->f32) launch_eval_general<true>(c, param, cost, st.robust, done_flag); else launch_eval_general<false>(c, param, cost, st.robust, done_flag); }
    else if (c->f32) launch_eval<true>(c, cost, st.robust, done_flag); else launch_eval<false>(c, cost, st.robust, done_flag);
    CU(cudaEventRecord(c->eval_ev[c->eval_ev_used + 1], c->stream));
    c->eval_ev_used += 2;
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
                                                                c->d_partial.as<double>(), eout_local, done_flag, pt, xs, xcounter);
    else
      lm_edge_kernel<<<E, EDGE_THREADS, 0, c->stream>>>(c->d_edges.as<EdgeDev>(), c->d_edge_tile_begin.as<int32_t>(), c->d_partial.as<double>(),
                                                        cost == COST_P2PLANE ? NBLK_PLANE : NBLK, c->d_Rt.as<Rt>(), c->d_K.as<double>(),
                                                        eout_local, done_flag, pt, xs, xcounter);
    if (c->comm && c->world > 1 && !use_p2p)
      NC(ncclAllReduce(c->d_eout.p, c->d_eout.p, (size_t)EOUT * E, ncclDouble, ncclSum, c->comm, c->stream));
    w.eout = eout_local; w.peer_flags = use_p2p ? pt.flags[c->rank] : nullptr; w.world = c->world; w.xseq = xs;
    w.seq = issued + 1;
    lm_step_kernel<<<1, STEP_THREADS, dyn, c->stream>>>(w);
    c->stats.kernel_launches += (c->n_eval_tiles ? 1 : 0) + 2;
    ++issued;
    return MVICP_OK;
  };
  RET(issue());
  while (true) {
    if (issued - seen < 2 && issued <= max_evals) RET(issue());
    // the step kernel publishes (sequence << 1 | done) into mapped pinned memory: spin on it, no stream round trip
    const int want = seen + 1;
    int32_t v;
    long spins = 0;
    while (((v = c->h_flag[want & 7]) >> 1) != want) {
      if ((++spins & 0xfffff) == 0 && cudaStreamQuery(c->stream) != cudaErrorNotReady) {   // kernels died or stream drained
        v = c->h_flag[want & 7];
        if ((v >> 1) != want) { CU(cudaGetLastError()); return fail(MVICP_ERR_CUDA, "LM step %d never reported", want); }
        break;
      }
    }
    const bool fin = (v & 1) != 0;
    ++seen;
    if (fin || seen > max_evals) break;
  }
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
  CU(cudaEventRecord(c->ev[4], c->stream));
  CU(cudaMemcpyAsync(c->h_state, c->d_state.p, sizeof st, cudaMemcpyDeviceToHost, c->stream));
  // the host mirror follows the device: mvicp_pose_graph_knn and mvicp_set_poses' "same poses as last handed out" test read it
  CU(cudaMemcpyAsync(c->h_poses.data(), c->d_poses.p, sizeof(double) * 16 * M, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  std::memcpy(&st, c->h_state, sizeof st);
  CU(cudaGetLastError());
  c->ev_lm = true;
  c->last_lm_iters = st.iteration;
  if (summary) {
    summary->termination = st.termination; summary->num_iterations = st.iteration; summary->num_successful_steps = st.n_success;
    summary->num_evaluations = st.n_evals; summary->num_linear_solves = st.n_solves; summary->reserved = 0;
    summary->initial_cost = st.initial_cost; summary->final_cost = st.x_cost;
  }
  if (st.nonrigid == 2) return fail(MVICP_ERR_NCCL, "a peer rank never delivered its pair matrices (peer-memory exchange timed out)");
  if (st.nonrigid && !general)   // cannot happen after mvicp_set_poses; guards poses that reached the device another way
    return fail(MVICP_ERR_NONRIGID, "a pose's quaternion is not unit (non-rigid Isometry) but the unit-quaternion LM path was run");
  if (!st.done) return fail(MVICP_ERR_STATE, "LM loop did not terminate within %d evaluations", max_evals);
  return MVICP_OK;
}

int mvicp_icp_round(mvicp_ctx* c, float thresh, int32_t param, int32_t cost, int32_t robust, const mvicp_lm_options* opt, mvicp_lm_summary* summary) {
  RET(mvicp_correspond(c, thresh));
  return mvicp_optimize(c, param, cost, robust, opt, summary);
}

int mvicp_pairwise(const mvicp_config* cfg, int32_t param, int32_t cost, const double* src, const double* dst, const double* nor,
                   int64_t n, const mvicp_lm_options* opt, double* pose16_out, mvicp_lm_summary* summary) {
  if (!src || !dst || n <= 0 || !pose16_out) return fail(MVICP_ERR_INVALID, "mvicp_pairwise: bad arguments");
  if (cost != MVICP_COST_P2P && !nor) return fail(MVICP_ERR_INVALID, "mvicp_pairwise: point-to-plane needs dst normals");
  mvicp_ctx* c = nullptr;
  RET(mvicp_create(cfg, &c));
  // frame 0 = dst (constant, identity), frame 1 = src (starts at identity); edge 1 -> 0 with identity matches
  const double* pts[2] = {dst, src}; const double* nrs[2] = {nor, nor};   // src normals are never read
  const int64_t np[2] = {n, n};
  int rc = mvicp_set_frames(c, 2, pts, nor ? nrs : nullptr, np);
  const int32_t es = 1, ed = 0;
  if (rc == MVICP_OK) rc = mvicp_set_graph(c, 1, &es, &ed);
  if (rc == MVICP_OK) {
    std::vector<int32_t> id(n); std::iota(id.begin(), id.end(), 0);
    rc = mvicp_set_edge(c, 0, id.data(), id.data(), n, 1.0f);
  }
  if (rc == MVICP_OK) rc = mvicp_optimize(c, param, cost, 0, opt, summary);
  std::vector<double> poses(32);
  if (rc == MVICP_OK) rc = mvicp_get_poses(c, poses.data());
  if (rc == MVICP_OK) std::memcpy(pose16_out, poses.data() + 16, sizeof(double) * 16);
  const std::string keep = g_err;
  mvicp_destroy(c);
  g_err = keep;
  return rc;
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
int mvicp_get_stream(mvicp_ctx* c, void** stream) { if (!c || !stream) return fail(MVICP_ERR_INVALID, "bad arguments"); *stream = (void*)c->stream; return MVICP_OK; }
int mvicp_sync(mvicp_ctx* c) { if (!c) return fail(MVICP_ERR_INVALID, "null ctx"); CU(cudaSetDevice(c->device)); CU(cudaStreamSynchronize(c->stream)); return MVICP_OK; }

}  // extern "C"
