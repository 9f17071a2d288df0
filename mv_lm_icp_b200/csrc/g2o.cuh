// g2o.cuh -- the reference's g2o backend (src/internal/icp-g2o.cpp) on the device: one Edge_V_V_GICP per correspondence,
// VertexSE3 poses, OptimizationAlgorithmLevenberg with a dense linear solver, and the multiview outer loop of optimize(100)
// calls with its no-improvement counter.  Semantics marked [ext] are g2o's (tag 20170730_git), restated in DESIGN section 2.
//
// Per correspondence (first, second) of edge src -> dst: vertex 0 = dst (T0 = [F0 | t0]), vertex 1 = src (T1 = [F1 | t1]),
// pos0 = dst point, pos1 = src point, normal0 = dst normal.
//   error     e = T0^-1 (T1 pos1) - pos0, T0^-1 = [F0^T | -F0^T t0] (Eigen's isometry inverse, also for non-rigid F0)   [ext]
//   info      point-to-point: I;  point-to-plane: prec0(eps) = R0^T diag(eps, eps, 1) R0 with R0 from makeRot0(normal0)  [ext]
//   chi2      sum e^T Omega e (no 1/2, no robust kernel: the reference comments its Huber kernel out, icp-g2o.cpp:152-156)
//   Jacobians (GICP_ANALYTIC_JACOBIANS, increment order tx ty tz qx qy qz), u = T0^-1 T1 pos1, M01 = F0^T F1            [ext]
//             J_dst = [ -I | 2 [u]x ],  J_src = [ M01 | -2 M01 [pos1]x ]
// Streaming kernel: the two-lane split of lm_eval_general_kernel (lm_eval.cuh): lane pairs share a correspondence, the even
// lane owns the src half of the Jacobian row block, the odd lane the dst half; they accumulate the 12x12 pair matrix directly
// (correct for non-rigid poses) in lm_eval_general_kernel's partial layout (GBLK).  In a trial evaluation only chi2 is
// accumulated, with the same lane mapping and reduction order, so a point's chi2 is bit-identical in both modes.
#pragma once
#include <cuda_runtime.h>
#include "../../include/mvicp.h"
#include "knn.cuh"
#include "lm_eval.cuh"
#include "lm_step.cuh"
#include "se3_math.cuh"
#include "types.cuh"

namespace mv {

enum { G2O_BUILD = 0, G2O_TRIAL = 1 };   // what the pending evaluation is for

struct G2oState {
  int32_t M, E, n, max_iter, max_calls, no_impr_limit, max_trials, ortho_after;
  int32_t phase, done, ended, last_call_end, call, iter, q, no_impr;
  int32_t n_iters, n_trials, n_accepted, n_evals, n_trace, trace_cap;
  double tau, lambda, nu, chi, last_chi, chi_initial, scale;
};

// What the streaming kernels evaluate for edge e (the g2o counterpart of DoneGate): edge e belongs to g2o problem prob[e]
// (-1: to none; prob null: every edge belongs to problem 0, the joint solve), whose state says whether it is done and which
// kind of evaluation it waits for.  Problems may be at different kinds in one launch; a tile belongs to one edge, so the choice
// is uniform per CTA.
struct G2oGate {
  const G2oState* S; const int32_t* prob;
  // -1: nothing to evaluate (no problem, or its solve terminated), else G2O_BUILD / G2O_TRIAL
  __device__ __forceinline__ int phase(int e) const {
    const int k = prob ? prob[e] : 0;
    if (k < 0) return -1;
    const G2oState* s = S + k;
    return s->done ? -1 : s->phase;
  }
};

// Omega = R0^T diag(eps, eps, 1) R0 (upper triangle 00 01 02 11 12 22), R0 row by row as EdgeGICP::makeRot0 builds it:
// row 2 = normal0 (not normalised), row 1 = normalise((0,1,0) - normal0.y normal0), row 0 = normal0 x row 1.
__host__ __device__ __forceinline__ void g2o_prec0(const double* n, double eps, double* Om) {
  double y[3] = {-n[1] * n[0], 1.0 - n[1] * n[1], -n[1] * n[2]};
  const double yy = y[0] * y[0] + y[1] * y[1] + y[2] * y[2];
  if (yy > 0.0) { const double s = sqrt(yy); y[0] /= s; y[1] /= s; y[2] /= s; }   // Eigen's normalize(): a zero vector stays zero
  double x[3]; cross(n, y, x);
  const double* R[3] = {x, y, n};
  const double d[3] = {eps, eps, 1.0};
  int k = 0;
  for (int a = 0; a < 3; ++a)
    for (int b = a; b < 3; ++b) Om[k++] = (R[0][a] * d[0]) * R[0][b] + (R[1][a] * d[1]) * R[1][b] + (R[2][a] * d[2]) * R[2][b];
}

template <bool F32, bool NF32, int COST>
__global__ void __launch_bounds__(EVAL_THREADS)
g2o_eval_kernel(const FrameDev* __restrict__ frames, const EdgeDev* __restrict__ edges, const Tile* __restrict__ tiles, int tile_len,
                const int32_t* __restrict__ corr, const Rt* __restrict__ pose_eval, G2oGate gate, double eps,
                double* __restrict__ partial) {
  const Tile t = tiles[blockIdx.x];
  const int phase = gate.phase(t.edge);
  if (phase < 0) return;   // issued speculatively after the edge's solve terminated, or an edge of no problem
  const bool build = phase == G2O_BUILD;
  const EdgeDev e = edges[t.edge];
  __shared__ double sF1[9], st1[3], sF0T[9], smt[3], sM01[9];
  __shared__ double sred[EVAL_THREADS / 32][2][GACC];
  if (threadIdx.x == 0) {
    const Rt a = pose_eval[e.src], k = pose_eval[e.dst];
    for (int i = 0; i < 9; ++i) sF1[i] = a.R[i];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) sF0T[3 * i + j] = k.R[3 * j + i];
    double ft[3]; matTvec(k.R, k.t, ft);
    for (int i = 0; i < 3; ++i) { st1[i] = a.t[i]; smt[i] = -ft[i]; }
    matTmul(k.R, a.R, sM01);
  }
  __syncthreads();
  const int role = threadIdx.x & 1;   // 0: src half of the row block, 1: dst half
  // this lane's translation block B and rotation columns s * C (v x e_j):  src (M01, M01, pos1, -2), dst (-I, I, u, 2)
  double C[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) C[i] = role ? ((i % 4 == 0) ? 1.0 : 0.0) : sM01[i];
  const double tsg = role ? -1.0 : 1.0, rsg = role ? 2.0 : -2.0;
  const FrameDev fs = frames[e.src];
  const FrameDev fd = frames[e.dst];
  double acc[GACC];
#pragma unroll
  for (int i = 0; i < GACC; ++i) acc[i] = 0.0;
  const int end = min(t.start + tile_len, e.n_src);
  for (int k0 = t.start; k0 < end; k0 += EVAL_THREADS / 2) {   // uniform trip count: the pair shuffles need every lane
    const int k = k0 + (threadIdx.x >> 1);
    const int c = k < end ? __ldg(corr + e.off + k) : -1;
    const bool ok = c >= 0;
    if (!__any_sync(0xffffffffu, ok)) continue;
    double p[3] = {0, 0, 0}, q[3] = {0, 0, 0}, n[3] = {0, 0, 0}; int dummy;
    if (ok) {
      Rec<F32>::load(fs.pts_o, k, p[0], p[1], p[2], dummy);
      Rec<F32>::load(fd.pts_o, c, q[0], q[1], q[2], dummy);
      if (COST == COST_P2PLANE) Rec<NF32>::load(fd.nor_o, c, n[0], n[1], n[2], dummy);
    }
    const double live = ok ? 1.0 : 0.0;   // an empty slot adds exact zeros
    double y[3], u[3], r[3];
    matvec(sF1, p, y);
#pragma unroll
    for (int i = 0; i < 3; ++i) y[i] += st1[i];
    matvec(sF0T, y, u);
#pragma unroll
    for (int i = 0; i < 3; ++i) { u[i] += smt[i]; r[i] = u[i] - q[i]; }
    double Om[6] = {1, 0, 0, 1, 0, 1};
    if (COST == COST_P2PLANE) g2o_prec0(n, eps, Om);
    const double O3[9] = {Om[0], Om[1], Om[2], Om[1], Om[3], Om[4], Om[2], Om[4], Om[5]};
    double Or[3]; matvec(O3, r, Or);
    acc[45] += live * (r[0] * Or[0] + r[1] * Or[1] + r[2] * Or[2]);
    if (!build) continue;
    // this lane's half J (3 x 6) and W = Omega J
    const double v[3] = {role ? u[0] : p[0], role ? u[1] : p[1], role ? u[2] : p[2]};
    const double vx[3][3] = {{0.0, v[2], -v[1]}, {-v[2], 0.0, v[0]}, {v[1], -v[0], 0.0}};   // v x e_j
    double J[3][6], W[3][6];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        J[i][j] = tsg * C[3 * i + j];
        J[i][3 + j] = rsg * (C[3 * i] * vx[j][0] + C[3 * i + 1] * vx[j][1] + C[3 * i + 2] * vx[j][2]);
      }
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 6; ++j) W[i][j] = O3[3 * i] * J[0][j] + O3[3 * i + 1] * J[1][j] + O3[3 * i + 2] * J[2][j];
    int idx = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
      for (int b = a; b < 6; ++b) acc[idx++] += live * (J[0][a] * W[0][b] + J[1][a] * W[1][b] + J[2][a] * W[2][b]);
    // (src, dst) block = J_src^T W_dst: rows 0-2 on the even lane (own J cols 0-2, partner's W), rows 3-5 on the odd lane
    // (partner's J cols 3-5, own W)
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      double X[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) { const double o = __shfl_xor_sync(0xffffffffu, J[i][3 + a], 1); X[i] = role ? o : J[i][a]; }
#pragma unroll
      for (int b = 0; b < 6; ++b) {
        double Y[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) { const double o = __shfl_xor_sync(0xffffffffu, W[i][b], 1); Y[i] = role ? W[i][b] : o; }
        acc[21 + 6 * a + b] += live * (X[0] * Y[0] + X[1] * Y[1] + X[2] * Y[2]);
      }
    }
#pragma unroll
    for (int a = 0; a < 6; ++a) acc[39 + a] += live * (J[0][a] * Or[0] + J[1][a] * Or[1] + J[2][a] * Or[2]);
  }
  // sum over the lanes of equal role (xor 16, 8, 4, 2), then over the warps in order (as lm_eval_general_kernel)
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < GACC; ++i) {
    if (!build && i != 45) continue;
    double v = acc[i];
#pragma unroll
    for (int o = 16; o > 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane < 2) sred[wid][lane][i] = v;
  }
  __syncthreads();
  if (threadIdx.x < 2 * GACC) {
    const int rl = threadIdx.x / GACC, i = threadIdx.x - GACC * rl;
    if (!build && i != 45) return;
    double v = 0.0;
    for (int w = 0; w < EVAL_THREADS / 32; ++w) v += sred[w][rl][i];
    int dst = -1;
    if (i < 21) {
      int a = 0, rem = i; while (rem >= 6 - a) { rem -= 6 - a; ++a; }
      dst = u12(6 * rl + a, 6 * rl + a + rem);
    } else if (i < 39) {
      const int a = (i - 21) / 6, b = (i - 21) - 6 * a;
      dst = u12(rl ? 3 + a : a, 6 + b);
    } else if (i < 45) dst = 78 + 6 * rl + (i - 39);
    else if (rl == 0) dst = 90;
    if (dst >= 0) partial[(size_t)blockIdx.x * GBLK + dst] = v;
  }
}

// One CTA per edge: the edge's tile partials summed in tile order (deterministic) into lm_edge_general_kernel's output layout:
// pair matrix over [src | dst] (144), pair gradient J^T Omega e (12), chi2 (slot 156).  A trial evaluation sums only chi2.
__global__ void __launch_bounds__(EDGE_THREADS)
g2o_edge_kernel(const int32_t* __restrict__ edge_tile_begin, const double* __restrict__ partial, G2oGate gate,
                double* __restrict__ out) {
  const int phase = gate.phase(blockIdx.x);
  if (phase < 0) return;
  const bool build = phase == G2O_BUILD;
  const int e = blockIdx.x, tid = threadIdx.x;
  __shared__ double blk[GBLK];
  double* o = out + (size_t)EOUT_ * e;
  for (int j = tid; j < 91; j += EDGE_THREADS) {
    if (!build && j != 90) continue;
    double v = 0.0;
    for (int t = edge_tile_begin[e]; t < edge_tile_begin[e + 1]; ++t) v += partial[(size_t)t * GBLK + j];
    blk[j] = v;
  }
  __syncthreads();
  if (!build) { if (tid == 0) o[156] = blk[90]; return; }
  for (int r = tid; r < 157; r += EDGE_THREADS) {
    if (r < 144) { const int a = r / 12, b = r - 12 * a; o[r] = blk[u12(min(a, b), max(a, b))]; }
    else if (r < 156) o[r] = blk[78 + (r - 144)];
    else o[r] = blk[90];
  }
}

// inliers per edge (corr >= 0) over the g2o tile list: which vertices take part in the problem
__global__ void g2o_count_kernel(const EdgeDev* __restrict__ edges, const Tile* __restrict__ tiles, int tile_len, const int32_t* __restrict__ corr,
                                 unsigned long long* __restrict__ count) {
  const Tile t = tiles[blockIdx.x];
  const EdgeDev e = edges[t.edge];
  const int end = min(t.start + tile_len, e.n_src);
  int m = 0;
  for (int k = t.start + threadIdx.x; k < end; k += blockDim.x) m += __ldg(corr + e.off + k) >= 0 ? 1 : 0;
  if (m) atomicAdd(count + t.edge, (unsigned long long)m);
}

// What every g2o problem shares; all per-frame arrays are indexed by graph frame.
struct G2oWork {
  const double* eout;            // [E][EOUT] from g2o_edge_kernel
  Rt* x;                         // [M] current estimate of every vertex
  Rt* ev;                        // [M] evaluation point: x (build) or the trial estimate
  int32_t* n_oplus;              // [M] VertexSE3::_numOplusCalls
  double* poses16;               // [M][16]
  volatile int32_t* host_flag;   // mapped pinned ring: (sequence << 1) | done, written at the end of every step
  int32_t seq;
};

// One g2o problem as g2o_step_kernel sees it: the whole graph, or one connected component (as LmProblem).  Local frame f is
// graph frame frame[f] (ascending), local edge e is graph edge edge[e] (graph order); the layout's columns and col[] are over
// local frames, its gather lists name graph edges.
struct G2oProblem {
  G2oState* S;
  const int32_t* frame;          // [S->M]
  const int32_t* edge;           // [S->E]
  NormalLayout lay;              // a frame has a column when it is free and has a correspondence
  double *H, *g;                 // g = sum J^T Omega e: g2o's b is -g
  double* chi_calls;             // [max_calls + 1]: chi2 before the first call, then after every call
  double* trace;                 // [S->trace_cap][5]: lambda, chi, tchi, rho, accepted -- one row per trial
};

__global__ void g2o_init_kernel(G2oWork w, int M) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= M) return;
  Rt a; pose16_to_Rt(w.poses16 + 16 * f, &a);
  w.x[f] = a; w.ev[f] = a; w.n_oplus[f] = 0;
}

// VertexSE3::oplusImpl [ext]: T <- T [R(q) | t] with (t, qx, qy, qz) = d, qw = sqrt(1 - |q|^2) (identity rotation if |q|^2 > 1),
// Eigen's Quaternion::toRotationMatrix; after more than `ortho_after` updates F <- F - F (F^T F - I) / 2 and the count restarts.
__device__ __forceinline__ void g2o_oplus(const Rt& x, const double* d, int* count, int ortho_after, Rt* out) {
  const double qq = d[3] * d[3] + d[4] * d[4] + d[5] * d[5];
  double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  if (!(1.0 - qq < 0.0)) {
    const double qw = sqrt(1.0 - qq), qx = d[3], qy = d[4], qz = d[5];
    const double tx = 2 * qx, ty = 2 * qy, tz = 2 * qz;
    const double twx = tx * qw, twy = ty * qw, twz = tz * qw, txx = tx * qx, txy = ty * qx, txz = tz * qx, tyy = ty * qy, tyz = tz * qy, tzz = tz * qz;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
    R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
  }
  matmul(x.R, R, out->R);
  matvec(x.R, d, out->t);
  for (int i = 0; i < 3; ++i) out->t[i] += x.t[i];
  if (++*count > ortho_after) {
    *count = 0;
    double Em[9]; matTmul(out->R, out->R, Em);
    Em[0] -= 1; Em[4] -= 1; Em[8] -= 1;
    double FE[9]; matmul(out->R, Em, FE);
    for (int i = 0; i < 9; ++i) out->R[i] -= 0.5 * FE[i];
  }
}

// OptimizationAlgorithmLevenberg::solve + SparseOptimizer::optimize + the reference's outer loop (icp-g2o.cpp:261-303): one step
// of one problem, one CTA.  Every step consumes one evaluation (S->phase says which kind), runs trials that need no evaluation (a
// failed factorisation), and leaves the next evaluation point in ev.  Every loop over frames and edges runs over the problem's
// LOCAL indices, so a component's chi2 is associated exactly as in a context that holds only that component.  ONE: the problem is
// the whole graph, local and graph indices coincide (no frame or edge list is read).
template <bool ONE> __device__ __forceinline__ void g2o_step_body(const G2oWork& w, const G2oProblem& p) {
  extern __shared__ double smem[];
  __shared__ double red[40];
  __shared__ G2oState s_state;
  __shared__ int s_solve, s_accept, s_tobuild;
  if (p.S->done) return;
  const int tid = threadIdx.x, T = blockDim.x;
  copy_state(&s_state, p.S);
  G2oState* S = &s_state;
  const int n = S->n, M = S->M, E = S->E;
  const int phase = S->phase;   // thread 0 moves S->phase on below
  const NormalLayout& lay = p.lay;
  double* colj = smem; double* dg = smem + 2 * (n + 1);
  double* L = lay.l_in_smem ? smem + 3 * (n + 1) : lay.Lg;

  auto frame = [&](int f) { return ONE ? f : p.frame[f]; };   // local -> graph frame
  const double chi_eval = edge_cost_sum(w.eout, E, red, ONE ? nullptr : p.edge);

  // end of an iteration (Terminate: trials exhausted or rho == 0), of a call (SparseOptimizer::optimize), of the outer loop
  auto end_iter = [&](double rho) {   // thread 0 only
    S->iter += 1; S->n_iters += 1;
    const bool term = S->q == S->max_trials || rho == 0.0;
    if (term || S->iter >= S->max_iter) {
      S->last_call_end = term ? MVICP_G2O_CALL_TERMINATE : MVICP_G2O_CALL_ITERATIONS;
      p.chi_calls[S->call + 1] = S->chi;   // computeActiveErrors(); chi2() at the call's final estimate
      const double impr = (S->last_chi - S->chi) / S->last_chi;
      S->last_chi = S->chi;
      if (!(impr > 0.0)) S->no_impr += 1;
      S->call += 1;
      if (S->no_impr > S->no_impr_limit) { S->done = 1; S->ended = MVICP_G2O_END_NO_IMPROVEMENT; return; }
      if (S->call >= S->max_calls) { S->done = 1; S->ended = MVICP_G2O_END_MAX_CALLS; return; }
      S->iter = 0;
    }
    S->phase = G2O_BUILD;
    s_tobuild = 1;
  };
  auto record = [&](double tchi, double rho, bool acc) {   // thread 0 only
    if (S->n_trace < S->trace_cap) {
      double* r = p.trace + 5 * (size_t)S->n_trace;
      r[0] = S->lambda; r[1] = S->chi; r[2] = tchi; r[3] = rho; r[4] = acc ? 1.0 : 0.0;
    }
    S->n_trace += 1;
  };

  if (tid == 0) { s_solve = 0; s_accept = 0; s_tobuild = 0; S->n_evals += 1; }
  if (phase == G2O_BUILD) {
    // H = sum J^T Omega J over the listed blocks, g = sum J^T Omega e
    gather_blocks(lay, w.eout, n, p.H);
    gather_gradient(lay, w.eout, M, p.g);
    __syncthreads();
    double md = 0.0;
    for (int j = tid; j < n; j += T) md = fmax(md, fabs(p.H[(size_t)j * n + j]));
    md = block_max(md, red);
    if (tid == 0) {
      if (S->call == 0 && S->iter == 0) { S->chi_initial = S->last_chi = chi_eval; p.chi_calls[0] = chi_eval; }
      S->chi = chi_eval;
      if (S->iter == 0) { S->lambda = S->tau * md; S->nu = 2.0; }   // computeLambdaInit at iteration 0 of every call
      S->q = 0;
      s_solve = 1;
    }
  } else if (tid == 0) {   // a trial's chi2
    const double tchi = chi_eval;
    const double rho = (S->chi - tchi) / S->scale;
    const bool acc = rho > 0.0 && isfinite(tchi);
    record(tchi, rho, acc);
    if (acc) {
      const double a = 1.0 - (2.0 * rho - 1.0) * (2.0 * rho - 1.0) * (2.0 * rho - 1.0);
      S->lambda *= fmax(1.0 / 3.0, fmin(2.0 / 3.0, a));
      S->nu = 2.0; S->chi = tchi; S->n_accepted += 1;
      s_accept = 1;
    } else { S->lambda *= S->nu; S->nu *= 2.0; }
    S->q += 1;
    if (rho < 0.0 && S->q < S->max_trials) s_solve = 1; else end_iter(rho);
  }
  __syncthreads();
  if (s_accept) for (int f = tid; f < M; f += T) { const int gf = frame(f); w.x[gf] = w.ev[gf]; }   // keep the trial (discardTop); otherwise pop
  __syncthreads();

  while (s_solve) {
    // (H + lambda I) dx = b = -g, skyline Cholesky of lm_step.cuh
    const double lambda = S->lambda;
    for (int i = tid >> 5; i < n; i += T >> 5) {
      const int rbi = lay.rowbase[i];
      for (int j = lay.rfirst[i] + (tid & 31); j <= i; j += 32) L[rbi + j] = p.H[(size_t)i * n + j] + (i == j ? lambda : 0.0);
    }
    { const int rbn = lay.rowbase[n]; for (int j = tid; j < n; j += T) L[rbn + j] = -p.g[j]; }
    __syncthreads();
    bool ok = chol_solve(L, lay.rowbase, n, colj, dg, lay.rhs, lay.rlast, lay.rfirst);
    double bad = 0.0;
    if (ok) for (int j = tid; j < n; j += T) if (!isfinite(lay.rhs[j])) bad = 1.0;
    bad = block_sum(bad, red);
    ok = ok && bad == 0.0;
    double sc = 0.0;
    if (ok) for (int j = tid; j < n; j += T) sc += lay.rhs[j] * (lambda * lay.rhs[j] - p.g[j]);
    sc = block_sum(sc, red);   // computeScale()
    // the update is applied to every vertex in the problem (and counted) even when the factorisation failed; it is undone then
    for (int f = tid; f < M; f += T) {
      const int cf = lay.col[f];
      if (cf < 0) continue;
      const int gf = frame(f);
      Rt nx;
      g2o_oplus(w.x[gf], lay.rhs + cf, &w.n_oplus[gf], S->ortho_after, &nx);
      if (ok) w.ev[gf] = nx;
    }
    __syncthreads();
    if (tid == 0) {
      S->n_trials += 1;
      s_solve = 0;
      if (ok) { S->scale = sc + 1e-3; S->phase = G2O_TRIAL; }
      else {   // a non-positive pivot: tchi = +inf, a rejected trial without an evaluation
        const double rho = -INFINITY;
        record(INFINITY, rho, false);
        S->lambda *= S->nu; S->nu *= 2.0; S->q += 1;
        if (S->q < S->max_trials) s_solve = 1; else end_iter(rho);
      }
    }
    __syncthreads();
  }
  if (s_tobuild && !S->done) for (int f = tid; f < M; f += T) { const int gf = frame(f); w.ev[gf] = w.x[gf]; }
  if (S->done)   // write the vertices of the problem back; every other frame keeps its pose bit for bit
    for (int f = tid; f < M; f += T) if (lay.col[f] >= 0) { const int gf = frame(f); Rt_to_pose16(&w.x[gf], w.poses16 + 16 * gf); }
  __syncthreads();
  copy_state(p.S, &s_state);
}

// The joint solve: one CTA steps the whole graph, its view passed by value (no staging, no frame or edge list), and publishes
// (sequence << 1) | done into the ring directly.
__global__ void __launch_bounds__(STEP_THREADS) g2o_step_one_kernel(G2oWork w, G2oProblem p) {
  g2o_step_body<true>(w, p);
  __syncthreads();
  if (threadIdx.x == 0) publish_step(w.host_flag, w.seq, *(volatile const int*)&p.S->done != 0);
}

// One CTA per g2o problem (probs[blockIdx.x]), with the ticket protocol of lm_step_kernel: every CTA takes a ticket when its
// step is written, the last one publishes (sequence << 1) | (every problem done) into the ring and resets the ticket for the
// next launch.  The problem's view is staged in shared memory once per CTA.
__global__ void __launch_bounds__(STEP_THREADS) g2o_step_kernel(G2oWork w, const G2oProblem* __restrict__ probs, unsigned int* ticket) {
  __shared__ G2oProblem s_prob;
  copy_state(&s_prob, probs + blockIdx.x);
  g2o_step_body<false>(w, s_prob);
  __shared__ int s_last;
  __syncthreads();
  int open;
  {
    if (threadIdx.x == 0) { __threadfence(); s_last = atomicAdd(ticket, 1u) == gridDim.x - 1; }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    open = 0;
    for (int k = threadIdx.x; k < (int)gridDim.x; k += blockDim.x) open |= *(volatile const int*)&probs[k].S->done == 0;
    open = __syncthreads_count(open);
  }
  if (threadIdx.x == 0) { *ticket = 0u; publish_step(w.host_flag, w.seq, open == 0); }
}

}  // namespace mv
