// lm_step.cuh -- the Levenberg-Marquardt trust-region state machine, one CTA, entirely on the device.
//
// Replaces ceres::Solve(getOptionsMedium(), ...) (src/internal/icp-ceres.cpp:66-95): LEVENBERG_MARQUARDT trust
// region, normal equations + Cholesky (SPARSE_NORMAL_CHOLESKY in the reference; dense here, <= 6(M-1) unknowns),
// Jacobi scaling, Ceres' step acceptance / radius update / termination tests (SURVEY 8(a) A9; Ceres 1.13
// semantics [ext-knowledge], the same contract the CPU oracle restates).
//
// One invocation consumes the per-edge blocks evaluated at the point the previous invocation proposed
// (residuals AND Jacobian blocks are evaluated together, so an accepted candidate needs no second pass over the
// correspondences), decides accept / reject / terminate, then solves for and writes the next candidate.
#pragma once
#include <cuda_runtime.h>
#include "../../include/mvicp.h"
#include "se3_math.cuh"
#include "types.cuh"

namespace mv {

constexpr int STEP_THREADS = 512;
constexpr int EOUT = 160;   // doubles per edge produced by lm_edge_kernel: Hp 144 | gp 12 | cost | pad

struct LmState {
  mvicp_lm_options opt;
  int32_t param, cost_kind, robust, M, E, F, n, G;
  int32_t phase, done, termination, iteration, n_success, n_invalid, n_evals, n_solves, reuse_diagonal, nonrigid;
  double radius, decrease_factor, x_cost, cand_cost, x_norm, initial_cost, model_cost_change, step_norm, gmax;
};

// The normal equations as both step kernels (lm_step_kernel, g2o_step_kernel) lay them out and gather them.  Built on the host
// from the free frames' local columns (mvicp.cu, upload_problems).
struct NormalLayout {
  const int32_t* col;        // [M] first local column or -1
  // block-sparse gather lists (host-built, deterministic order)
  const int32_t* hb_ptr; const int32_t* hb_row; const int32_t* hb_col; const int32_t* hc_edge; const int32_t* hc_sub; int32_t n_hblocks;
  const int32_t* gb_ptr; const int32_t* gc_edge; const int32_t* gc_side;   // per frame
  const int32_t* rlast; const int32_t* rfirst;   // envelope of the normal matrix: last row touching column j / first column of row r
  const int32_t* rowbase;                        // skyline storage of the factor: entry (r, c) at Lg[rowbase[r] + c]; [n] = rhs row
  double *Lg, *rhs;
  int32_t l_in_smem;
};

struct LmWork {
  LmState* S;
  const EdgeDev* edges;
  const double* eout;        // [E][EOUT]: pair matrix (144), pair gradient (12), cost at the evaluation point (summed over ranks)
  volatile int* peer_flags;    // this rank's flag array (written by the peers' edge kernels), null when not sharded over peer memory
  int32_t world, xseq;
  double* x;                 // [M][7] accepted point (all frames)
  double* cand;              // [M][7] evaluation point / next candidate
  Rt* Rt_eval;               // [M]
  double* K_eval;            // [M][36]
  FrameGen* G_eval;          // [M] general frame model (null unless a quaternion is not unit)
  double* poses16;           // [M][16]
  volatile int32_t* host_flag; // mapped pinned ring: (sequence << 1) | done, written at the end of every step
  int32_t seq;
  long long* prof;           // development aid (MVICP_STEP_PROFILE=1): clock64() stamps of the last solving launch, else null
};

// One LM problem as the state machine sees it: the whole graph, or one connected component.  Local frame f is frame frame[f] of
// the graph (ascending), local edge e is edge edge[e] (graph order); the layout's columns, col[] and gb_ptr[] are over local
// frames, its gather lists name graph edges.  x, cand, Rt_eval, K_eval, G_eval and the poses stay indexed by graph frame.
struct LmProblem {
  LmState* S;
  const int32_t* frame;      // [S->M]
  const int32_t* edge;       // [S->E]
  NormalLayout lay;
  double *H, *g, *Hc, *gc, *scale, *diag, *step;
};

__device__ __forceinline__ double block_sum(double v, double* red) {
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if (lane == 0) red[wid] = v;
  __syncthreads();
  if (threadIdx.x == 0) { double s = 0; for (int w = 0; w < STEP_THREADS / 32; ++w) s += red[w]; red[32] = s; }
  __syncthreads();
  return red[32];
}
__device__ __forceinline__ double block_max(double v, double* red) {
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_down_sync(0xffffffffu, v, o));
  if (lane == 0) red[wid] = v;
  __syncthreads();
  if (threadIdx.x == 0) { double s = 0; for (int w = 0; w < STEP_THREADS / 32; ++w) s = fmax(s, red[w]); red[32] = s; }
  __syncthreads();
  return red[32];
}

// ---- the normal-equation layout, shared by lm_step_kernel and g2o_step_kernel ------------------------------------
// Dense normal matrix from the per-edge pair matrices: each listed 6x6 block summed over its (edge, sub-block) list in list
// order.  Entries outside the listed blocks are zeroed once by the host when the layout is built and never written.
__device__ __forceinline__ void gather_blocks(const NormalLayout& l, const double* eout, int n, double* H) {
  for (int idx = threadIdx.x; idx < l.n_hblocks * 36; idx += blockDim.x) {
    const int b = idx / 36, r = idx - 36 * b, i = r / 6, j = r - 6 * i;
    double s = 0;
    for (int c = l.hb_ptr[b]; c < l.hb_ptr[b + 1]; ++c) {
      const int e = l.hc_edge[c], sub = l.hc_sub[c];   // sub: 0 ss, 1 sk, 2 ks, 3 kk
      s += eout[(size_t)EOUT * e + (6 * (sub >> 1) + i) * 12 + 6 * (sub & 1) + j];
    }
    H[(size_t)(l.hb_row[b] + i) * n + l.hb_col[b] + j] = s;
  }
}
// Gradient of every frame with a column: its (edge, side) pair gradients summed in list order
__device__ __forceinline__ void gather_gradient(const NormalLayout& l, const double* eout, int M, double* g) {
  for (int idx = threadIdx.x; idx < M * 6; idx += blockDim.x) {
    const int f = idx / 6, i = idx - 6 * f;
    if (l.col[f] < 0) continue;
    double s = 0;
    for (int c = l.gb_ptr[f]; c < l.gb_ptr[f + 1]; ++c) s += eout[(size_t)EOUT * l.gc_edge[c] + 144 + 6 * l.gc_side[c] + i];
    g[l.col[f] + i] = s;
  }
}
// Total cost: edges summed in a fixed order (thread t takes edges t, t + T, ...; then the block tree) -- the same on every rank.
// edge (nullable): the problem's local edge list; the order is over local edges, so a component sums as a graph of its own would.
__device__ __forceinline__ double edge_cost_sum(const double* eout, int E, double* red, const int32_t* edge = nullptr) {
  double s = 0.0;
  for (int e = threadIdx.x; e < E; e += blockDim.x) s += eout[(size_t)EOUT * (edge ? edge[e] : e) + 156];
  return block_sum(s, red);
}
// A step kernel works on a shared-memory copy of its state (dozens of dependent scalar reads per step) and writes it back once
// at the end; nobody else touches the state while the kernel runs (lm_step_kernel stages its LmProblem the same way)
template <typename State> __device__ __forceinline__ void copy_state(State* dst, const State* src) {
  for (int i = threadIdx.x; i < (int)(sizeof(State) / sizeof(int32_t)); i += blockDim.x)
    reinterpret_cast<int32_t*>(dst)[i] = reinterpret_cast<const int32_t*>(src)[i];
  __syncthreads();
}
// One thread tells the host that this step ran: (sequence << 1) | done into the mapped ring, after every write of the step
__device__ __forceinline__ void publish_step(volatile int32_t* host_flag, int32_t seq, bool done) {
  __threadfence();
  host_flag[seq & 7] = (seq << 1) | (done ? 1 : 0);
  __threadfence_system();
}

// Per-frame set-up before the first evaluation: poses -> parameters, functor rotation, tangent map.
__global__ void lm_init_kernel(LmWork w) {
  LmState* S = w.S;
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= S->M) return;
  double x[7] = {0, 0, 0, 0, 0, 0, 0};
  param_of_pose(S->param, w.poses16 + 16 * f, x);
  if (S->param != PARAM_AA) {
    const double n2 = x[0] * x[0] + x[1] * x[1] + x[2] * x[2] + x[3] * x[3];
    if (!(fabs(n2 - 1.0) <= 1e-9)) atomicExch(&S->nonrigid, 1);
  }
  Rt a; Rt_of_param(S->param, x, &a);
  double K[36]; tangent_map(S->param, x, &a, K);
  for (int i = 0; i < 7; ++i) { w.x[7 * f + i] = x[i]; w.cand[7 * f + i] = x[i]; }
  w.Rt_eval[f] = a;
  for (int i = 0; i < 36; ++i) w.K_eval[36 * f + i] = K[i];
  if (w.G_eval && S->param != PARAM_AA) frame_general(S->param, x, &w.G_eval[f]);
}

// ---- dense Cholesky solve --------------------------------------------------------------------------------------
// L: n+1 rows; rows 0..n-1 hold the lower triangle of the SPD matrix (profile part only), row n holds the right-hand side
// (treating the rhs as an extra row performs the forward substitution for free).  n is a multiple of 6 (one 6x6 block
// per free pose), and the factorisation is right-looking over those blocks with a one-block LOOK-AHEAD -- the solve is bound
// by its dependent chain, not by arithmetic:
//   panel     one thread per row below block J solves its 6 entries against the factored diagonal block;
//   update    one warp per remaining row applies block J to the trailing matrix, while WARP 0 first updates the 21 entries
//             of the NEXT diagonal block and factors it at once (registers, every lane the same arithmetic, lane 0 stores):
//             the 6 x (rsqrt + dependent multiply-adds) of the next block overlap the other warps' update.
// Two barriers per pose, and the 6x6 factor is computed once per block instead of once per thread (ncu, round 2: the
// redundant factor with its software sqrt and division was 60 % of lm_step_kernel's instructions).  Diagonal entries are
// inverted with rsqrt (1 ulp) and L_kk = d * rsqrt(d).
// Rows whose profile starts right of the block (rfirst) and rows beyond rlast are structurally zero in the block
// (envelope of the block-sparse normal matrix; fill-in stays inside each row's profile) and are skipped: only entries
// inside the row profiles [rfirst[r], r] are ever read or written, the rest of L may hold anything.
// L is stored row by row, each row only over its profile (skyline): rowbase[r] + c addresses entry (r, c), rowbase[n] the rhs row.
// scratch: >= 3n + 2 ints (row profiles and bases staged in shared memory + the "positive definite so far" flag); dinv: reciprocal
// diagonal of the factor.  The back substitution runs block-wise in one warp.  Solution returned in y[0..n).
__device__ __forceinline__ void chol_factor_diag(double* L, const int32_t* rb, int j0, double* dinv, volatile int* s_ok, int lane) {
  double D[6][6], inv[6];
#pragma unroll
  for (int i = 0; i < 6; ++i)
#pragma unroll
    for (int k = 0; k <= i; ++k) D[i][k] = L[rb[j0 + i] + j0 + k];
  bool okb = true;
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    double d = D[k][k];
#pragma unroll
    for (int m = 0; m < k; ++m) d -= D[k][m] * D[k][m];
    if (!(d > 0.0) || !isfinite(d)) okb = false;
    inv[k] = rsqrt(d); D[k][k] = d * inv[k];
#pragma unroll
    for (int i = k + 1; i < 6; ++i) {
      double v = D[i][k];
#pragma unroll
      for (int m = 0; m < k; ++m) v -= D[i][m] * D[k][m];
      D[i][k] = v * inv[k];
    }
  }
  __syncwarp();   // every lane has read the block before lane 0 overwrites it
  if (lane == 0) {
    if (!okb) *s_ok = 0;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
#pragma unroll
      for (int k = 0; k <= i; ++k) L[rb[j0 + i] + j0 + k] = D[i][k];
      dinv[j0 + i] = inv[i];
    }
  }
}

__device__ bool chol_solve(double* L, const int32_t* __restrict__ rowbase, int n, double* scratch, double* dinv, double* y,
                           const int32_t* __restrict__ rlast, const int32_t* __restrict__ rfirst, long long* prof = nullptr) {
  const int T = blockDim.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nw = T >> 5;
  int32_t* s_rfirst = reinterpret_cast<int32_t*>(scratch);
  int32_t* s_rlast = s_rfirst + n;
  int32_t* rb = s_rlast + n;                      // row r's entry of column c sits at L[rb[r] + c] (c inside the row's profile)
  volatile int* s_ok = reinterpret_cast<volatile int*>(rb + n + 1);
  for (int i = tid; i < n; i += T) { s_rfirst[i] = rfirst[i]; s_rlast[i] = rlast[i]; }
  for (int i = tid; i <= n; i += T) rb[i] = rowbase[i];
  if (tid == 0) *s_ok = 1;
  __syncthreads();
  const int NB = n / 6;
  if (wid == 0) chol_factor_diag(L, rb, 0, dinv, s_ok, lane);
  __syncthreads();
  long long t_panel = 0, t_ahead = 0, t_bar = 0;
  for (int J = 0; J < NB; ++J) {
    if (!*s_ok) return false;                     // uniform: written before the last barrier
    const long long c0 = prof ? clock64() : 0;
    const int j0 = 6 * J;
    const int rl = s_rlast[j0 + 5];
    const int nrows = rl - (j0 + 5) + 1;          // rows j0+6..rl and the rhs row
    // panel: L[r][j0..j0+5] <- A[r][j0..j0+5] * L_JJ^-T
    for (int q = tid; q < nrows; q += T) {
      const int r = (q == nrows - 1) ? n : j0 + 6 + q;
      if (r < n && s_rfirst[r] > j0 + 5) continue;
      double* row = L + rb[r] + j0;
      double v[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        double a = row[k];
#pragma unroll
        for (int m = 0; m < k; ++m) a -= v[m] * L[rb[j0 + k] + j0 + m];
        v[k] = a * dinv[j0 + k];
      }
#pragma unroll
      for (int k = 0; k < 6; ++k) row[k] = v[k];
    }
    const long long c1 = prof ? clock64() : 0;
    __syncthreads();
    const long long c2 = prof ? clock64() : 0;
    // trailing update: A[r][c] -= sum_k L[r][j0+k] L[c][j0+k] for j0+5 < c <= min(r, rl)
    const bool next = J + 1 < NB;
    if (wid == 0 && next) {                       // look-ahead: the next diagonal block first, then its factor
      const int b0 = j0 + 6;
      if (lane < 21 && s_rfirst[b0] <= j0 + 5) {  // (the six rows of a pose share their profile start)
        int i = 0, rem = lane; while (rem > i) { rem -= i + 1; ++i; }   // lane -> (i, k), k <= i
        const int k = rem;
        double* row = L + rb[b0 + i]; const double* lc = L + rb[b0 + k] + j0;
        double a = row[b0 + k];
#pragma unroll
        for (int m = 0; m < 6; ++m) a -= row[j0 + m] * lc[m];
        row[b0 + k] = a;
      }
      __syncwarp();
      chol_factor_diag(L, rb, b0, dinv, s_ok, lane);
    } else {
      const int w0 = next ? 1 : 0, wn = next ? nw - 1 : nw;       // warps that share the remaining rows
      const int qfirst = next ? 6 : 0;                              // rows of the next diagonal block belong to warp 0
      for (int q = qfirst + (wid - w0); q < nrows; q += wn) {
        const int r = (q == nrows - 1) ? n : j0 + 6 + q;
        if (r < n && s_rfirst[r] > j0 + 5) continue;
        double* row = L + rb[r];
        double lr[6];
#pragma unroll
        for (int k = 0; k < 6; ++k) lr[k] = row[j0 + k];
        const int cend = min(r, rl);
        for (int c = j0 + 6 + lane; c <= cend; c += 32) {
          if (s_rfirst[c] > j0 + 5) continue;        // row c has nothing in this block: contributes exactly zero
          const double* lc = L + rb[c] + j0;
          double a = row[c];
#pragma unroll
          for (int k = 0; k < 6; ++k) a -= lr[k] * lc[k];
          row[c] = a;
        }
      }
    }
    const long long c3 = prof ? clock64() : 0;
    __syncthreads();
    if (prof) { const long long c4 = clock64(); t_panel += c1 - c0; t_ahead += c3 - c2; t_bar += (c2 - c1) + (c4 - c3); }
  }
  if (prof && tid == 0) { prof[8] = t_panel; prof[9] = t_ahead; prof[10] = t_bar; }
  if (!*s_ok) return false;
  for (int i = tid; i < n; i += T) y[i] = L[rb[n] + i];   // forward-substituted rhs
  __syncthreads();
  if (wid == 0) {
    for (int J = NB - 1; J >= 0; --J) {     // L^T x = z, one pose block at a time
      const int j0 = 6 * J;
      double x[6];
#pragma unroll
      for (int k = 5; k >= 0; --k) {
        double a = y[j0 + k];
#pragma unroll
        for (int m = k + 1; m < 6; ++m) a -= L[rb[j0 + m] + j0 + k] * x[m];
        x[k] = a * dinv[j0 + k];
      }
      __syncwarp();
#pragma unroll
      for (int k = 0; k < 6; ++k) if (lane == k) y[j0 + k] = x[k];
      for (int i = s_rfirst[j0] + lane; i < j0; i += 32) {
        double a = y[i];
#pragma unroll
        for (int k = 0; k < 6; ++k) a -= L[rb[j0 + k] + i] * x[k];
        y[i] = a;
      }
      __syncwarp();
    }
  }
  __syncthreads();
  return true;
}

// ---- the LM trust-region state machine: one step of one problem, one CTA -----------------------------------------------
// Every loop over frames, edges and columns runs over the problem's LOCAL indices, so a component's reductions are associated
// exactly as in a context that holds only that component.
__device__ __forceinline__ void lm_step_body(const LmWork& w, const LmProblem& p) {
  extern __shared__ double smem[];
  __shared__ double red[40];
  __shared__ int s_flag;
  if (p.S->done) return;
  const int tid = threadIdx.x, T = blockDim.x;
  __shared__ LmState s_state;
  copy_state(&s_state, p.S);
  LmState* S = &s_state;
  const int n = S->n, M = S->M, E = S->E, param = S->param;
  const NormalLayout& lay = p.lay;
  long long* prof = w.prof ? w.prof + 16 * (w.seq & 3) : nullptr;   // one row of stamps per launch, the last four launches kept
#define MV_STAMP(i) do { if (prof && tid == 0) prof[i] = clock64(); } while (0)
  MV_STAMP(0);
  if (w.peer_flags) {   // wait until every rank's edge kernel has delivered this iteration's pair matrices
    if (tid < w.world) {
      const long long t0 = clock64();
      while (w.peer_flags[tid] - w.xseq < 0) {
        if (clock64() - t0 > 4000000000LL) { S->nonrigid = 2; break; }   // ~2 s: a peer died; surface an error instead of hanging
      }
    }
    __syncthreads();
  }
  // dynamic shared memory: [scratch 2(n+1) | dg (n+1) | L (skyline) when it fits]
  double* colj = smem; double* dg = smem + 2 * (S->n + 1);
  double* L = lay.l_in_smem ? smem + 3 * (S->n + 1) : lay.Lg;

  // ================= 1. gather the per-edge pair matrices (lm_edge_kernel) into Hc, gc; total cost ===================
  gather_blocks(lay, w.eout, n, p.Hc);
  gather_gradient(lay, w.eout, M, p.gc);
  __syncthreads();
  const double eval_cost = edge_cost_sum(w.eout, E, red, p.edge);

  MV_STAMP(1);
  // ================= 2. accept / reject / terminate =================================================
  bool take = false;    // the evaluation point becomes the accepted point
  if (tid == 0) {
    s_flag = 0;
    S->n_evals += 1;
    if (!isfinite(eval_cost)) {
      if (S->phase == 0) { S->done = 1; S->termination = MVICP_TERM_EVAL_FAILURE; }
      else {   // non-finite candidate cost: Ceres treats the step as invalid
        S->n_invalid += 1;
        if (S->n_invalid >= S->opt.max_num_consecutive_invalid_steps) { S->done = 1; S->termination = MVICP_TERM_INVALID_STEPS; }
        S->radius = S->radius / S->decrease_factor; S->decrease_factor *= 2.0; S->reuse_diagonal = 1;
      }
    } else if (S->phase == 0) {
      S->x_cost = eval_cost; S->initial_cost = eval_cost; s_flag = 1;
    } else {
      S->cand_cost = eval_cost;
      if (S->step_norm <= S->opt.parameter_tolerance * (S->x_norm + S->opt.parameter_tolerance)) {
        S->done = 1; S->termination = MVICP_TERM_PARAMETER_TOLERANCE;
      } else if (fabs(S->x_cost - eval_cost) <= S->opt.function_tolerance * S->x_cost) {
        S->done = 1; S->termination = MVICP_TERM_FUNCTION_TOLERANCE;
      } else {
        const double rho = (S->x_cost - eval_cost) / S->model_cost_change;
        if (rho > S->opt.min_relative_decrease) {
          s_flag = 1; S->n_success += 1; S->x_cost = eval_cost;
          const double q = 2.0 * rho - 1.0;
          S->radius = fmin(S->opt.max_trust_region_radius, S->radius / fmax(1.0 / 3.0, 1.0 - q * q * q));
          S->decrease_factor = 2.0; S->reuse_diagonal = 0;
        } else {
          S->radius = S->radius / S->decrease_factor; S->decrease_factor *= 2.0; S->reuse_diagonal = 1;
          if (S->radius < S->opt.min_trust_region_radius) { S->done = 1; S->termination = MVICP_TERM_MIN_RADIUS; }
        }
      }
    }
  }
  __syncthreads();
  take = s_flag != 0;
  if (take) {
    for (int idx = tid; idx < lay.n_hblocks * 36; idx += T) {
      const int b = idx / 36, r = idx - 36 * b, i = r / 6, j = r - 6 * i;
      const size_t at = (size_t)(lay.hb_row[b] + i) * n + lay.hb_col[b] + j;
      p.H[at] = p.Hc[at];
    }
    for (int idx = tid; idx < n; idx += T) p.g[idx] = p.gc[idx];
    for (int idx = tid; idx < M * 7; idx += T) { const int at = 7 * p.frame[idx / 7] + idx % 7; w.x[at] = w.cand[at]; }
    __syncthreads();
    if (S->phase == 0)
      for (int j = tid; j < n; j += T) p.scale[j] = S->opt.jacobi_scaling ? 1.0 / (1.0 + sqrt(p.H[(size_t)j * n + j])) : 1.0;
    // x_norm over the free blocks, and the gradient test |x - Plus(x, -g)|_inf
    double xs = 0.0, gm = 0.0;
    for (int f = tid; f < M; f += T) {
      if (lay.col[f] < 0) continue;
      const int G = S->G;
      double xf[7], ng[6], xp[7];
      for (int i = 0; i < G; ++i) { xf[i] = w.x[7 * p.frame[f] + i]; xs += xf[i] * xf[i]; }
      for (int i = 0; i < 6; ++i) ng[i] = -p.g[lay.col[f] + i];
      param_plus(param, xf, ng, xp);
      for (int i = 0; i < G; ++i) gm = fmax(gm, fabs(xf[i] - xp[i]));
    }
    xs = block_sum(xs, red);
    gm = block_max(gm, red);
    if (tid == 0) {
      S->x_norm = sqrt(xs); S->gmax = gm;
      if (gm <= S->opt.gradient_tolerance) { S->done = 1; S->termination = MVICP_TERM_GRADIENT_TOLERANCE; }
      if (S->phase == 0) { S->phase = 1; S->iteration = 0; S->reuse_diagonal = 0; }
    }
    __syncthreads();
  }

  MV_STAMP(2);
  // ================= 3. next trust-region step ======================================================
  while (!S->done) {
    __syncthreads();
    if (S->iteration >= S->opt.max_num_iterations) {
      __syncthreads();
      if (tid == 0) { S->done = 1; S->termination = MVICP_TERM_MAX_ITERATIONS; }
      __syncthreads();
      break;
    }
    const int reuse = S->reuse_diagonal;
    const double radius = S->radius;
    __syncthreads();
    if (!reuse)
      for (int j = tid; j < n; j += T) {
        const double d = p.scale[j] * p.scale[j] * p.H[(size_t)j * n + j];
        p.diag[j] = fmin(fmax(d, S->opt.min_lm_diagonal), S->opt.max_lm_diagonal);
      }
    __syncthreads();
    for (int i = tid >> 5; i < n; i += T >> 5) {          // one warp per row, only the row's profile (see chol_solve)
      const double si = p.scale[i];
      const int rbi = lay.rowbase[i];
      for (int j = lay.rfirst[i] + (tid & 31); j <= i; j += 32) {
        double v = si * p.H[(size_t)i * n + j] * p.scale[j];
        if (i == j) { const double ldg = sqrt(p.diag[i] / radius); v += ldg * ldg; }
        L[rbi + j] = v;
      }
    }
    { const int rbn = lay.rowbase[n]; for (int j = tid; j < n; j += T) L[rbn + j] = p.scale[j] * p.g[j]; }
    __syncthreads();
    MV_STAMP(3);
    bool ok = chol_solve(L, lay.rowbase, n, colj, dg, lay.rhs, lay.rlast, lay.rfirst, prof);
    MV_STAMP(4);
    double bad = 0.0;
    if (ok) for (int j = tid; j < n; j += T) if (!isfinite(lay.rhs[j])) bad = 1.0;
    bad = block_sum(bad, red);
    ok = ok && (bad == 0.0);
    double mcc = 0.0;
    if (ok) {
      for (int j = tid; j < n; j += T) p.step[j] = -lay.rhs[j];
      __syncthreads();
      // model_cost_change = -(J s).(r + J s / 2) = -s.g~ - 1/2 s^T H~ s; with (H~ + D^2) y = g~ and s = -y this is
      // 1/2 (y.g~ + sum D_i^2 y_i^2): O(n) instead of O(n^2)
      double acc = 0.0;
      for (int i = tid; i < n; i += T) {
        const double y = lay.rhs[i];
        acc += 0.5 * (y * p.scale[i] * p.g[i] + (p.diag[i] / radius) * y * y);
      }
      mcc = block_sum(acc, red);
    }
    const bool valid = ok && (mcc > 0.0);
    __syncthreads();
    if (tid == 0) {
      S->iteration += 1; S->n_solves += 1; S->reuse_diagonal = 1; S->model_cost_change = mcc;
      if (!valid) {
        S->n_invalid += 1;
        if (S->n_invalid >= S->opt.max_num_consecutive_invalid_steps) { S->done = 1; S->termination = MVICP_TERM_INVALID_STEPS; }
        S->radius = S->radius / S->decrease_factor; S->decrease_factor *= 2.0;
      } else S->n_invalid = 0;
    }
    __syncthreads();
    if (!valid) continue;
    // candidate = Plus(x, step * scale) per free frame; step norm in the ambient space
    double sn = 0.0;
    for (int f = tid; f < M; f += T) {
      const int G = S->G, g_f = __ldg(p.frame + f);   // (read-only path: 196 instead of 216 bytes of spills, ptxas 12.9)
      double xf[7], d[6], xp[7] = {0, 0, 0, 0, 0, 0, 0};
      for (int i = 0; i < 7; ++i) xf[i] = w.x[7 * g_f + i];
      if (lay.col[f] >= 0) {
        for (int i = 0; i < 6; ++i) d[i] = p.step[lay.col[f] + i] * p.scale[lay.col[f] + i];
        param_plus(param, xf, d, xp);
        for (int i = 0; i < G; ++i) sn += (xf[i] - xp[i]) * (xf[i] - xp[i]);
      } else for (int i = 0; i < 7; ++i) xp[i] = xf[i];
      for (int i = 0; i < 7; ++i) w.cand[7 * g_f + i] = xp[i];
      Rt a; Rt_of_param(param, xp, &a);
      w.Rt_eval[g_f] = a;
      double K[36]; tangent_map(param, xp, &a, K);
      for (int i = 0; i < 36; ++i) w.K_eval[36 * g_f + i] = K[i];
      if (w.G_eval && param != PARAM_AA) frame_general(param, xp, &w.G_eval[g_f]);
    }
    sn = block_sum(sn, red);
    MV_STAMP(5);
    if (tid == 0) S->step_norm = sqrt(sn);
    __syncthreads();
    break;
  }
  __syncthreads();
  // ================= 4. on termination: write every frame's pose back (icp-ceres.cpp:318-322,392-394,472-474)
  if (S->done) {
    for (int f = tid; f < M; f += T) {
      double xf[7]; for (int i = 0; i < 7; ++i) xf[i] = w.x[7 * p.frame[f] + i];
      pose_of_param(param, xf, w.poses16 + 16 * p.frame[f]);
    }
  }
  __syncthreads();
  copy_state(p.S, &s_state);
  MV_STAMP(6);
#undef MV_STAMP
}

// One CTA per LM problem (probs[blockIdx.x]), each stepping its own problem.  Every CTA takes a ticket when its step is written;
// the last one publishes (sequence << 1) | (every problem done) into the ring and resets the ticket for the next launch (a
// single CTA publishes directly).  The problem's view is staged in shared memory once per CTA, not copied into every thread.
__global__ void __launch_bounds__(STEP_THREADS) lm_step_kernel(LmWork w, const LmProblem* __restrict__ probs, unsigned int* ticket) {
  __shared__ LmProblem s_prob;
  copy_state(&s_prob, probs + blockIdx.x);
  lm_step_body(w, s_prob);
  __shared__ int s_last;
  __syncthreads();
  int open;
  if (gridDim.x == 1) {   // one problem: no ticket (its atomic and fences cost ~2 us per step on an H100)
    open = *(volatile const int*)&s_prob.S->done == 0;
  } else {
    if (threadIdx.x == 0) { __threadfence(); s_last = atomicAdd(ticket, 1u) == gridDim.x - 1; }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    open = 0;
    for (int k = threadIdx.x; k < (int)gridDim.x; k += blockDim.x) open |= *(volatile const int*)&probs[k].S->done == 0;
    open = __syncthreads_count(open);
  }
  if (threadIdx.x == 0) {
    *ticket = 0u; publish_step(w.host_flag, w.seq, open == 0);
    if (w.prof) w.prof[16 * (w.seq & 3) + 7] = clock64();
  }
}

}  // namespace mv
