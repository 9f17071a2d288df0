// covariance.cuh -- covariance blocks of the LM problem at the current poses (mvicp_covariance, DESIGN.md section 6j).
//
// C = H^-1 over the free frames of a component, H the Gauss-Newton matrix J^T J that lm_edge_kernel / lm_edge_general_kernel
// and gather_blocks build for the first step of mvicp_optimize (the loss applied as Ceres' corrector applies it).  Ceres'
// Covariance::Compute evaluates the same matrix.  Two kernels per call, after one streaming evaluation:
//   cov_factor_kernel  one CTA per problem: gather H, Jacobi-scale it (S = diag(1 / sqrt(H_jj)), H~ = S H S with a unit diagonal)
//                      into the skyline storage of the problem's NormalLayout, factor H~ = L L^T with chol_solve (zero rhs),
//                      apply the rank rule, and leave L (global memory), 1 / L_jj and S for the next kernel;
//   cov_solve_kernel   one CTA per (problem, frame whose columns some request needs): the frame's 6 unit columns through
//                      L y = e_k, L^T z = y, then C[:, k] = S z S_k, one warp per column.
// A column's arithmetic depends only on the problem and the column (the warp's lanes take fixed strides, the warp sum is a
// xor butterfly, which leaves the same bits in every lane), never on which other columns are requested.
#pragma once
#include <cuda_runtime.h>
#include "lm_step.cuh"

namespace mv {

constexpr int COV_SOLVE_THREADS = 192;   // one warp per unit column of a frame

// One CTA of cov_solve_kernel: problem `prob`, the frame whose first local column is `col`; its 6 columns of C go to
// out[at .. at + 6 n), column by column.
struct CovJob { int32_t prob, col; int64_t at; };

// Rank rule [ext]: a component is singular when a diagonal entry of H is zero or not finite, when a pivot of the factor of H~
// is not positive or not finite (chol_solve), or when a pivot L~_jj^2 <= 64 n 2^-53, the rounding level of the normal-equation
// route for n unknowns.
__device__ __forceinline__ double cov_pivot_floor(int n) { return 64.0 * (double)n * 0x1p-53; }

// status[q]: MVICP_COV_OK, or MVICP_COV_SINGULAR.  Afterwards p.lay.Lg holds the factor's rows (skyline), p.diag 1 / L~_jj and
// p.scale S.  Dynamic shared memory as lm_step_kernel's: [scratch 2(n+1) | dinv (n+1) | factor when it fits].
__global__ void __launch_bounds__(STEP_THREADS) cov_factor_kernel(const LmProblem* __restrict__ probs, const double* __restrict__ eout,
                                                                  int32_t* __restrict__ status) {
  extern __shared__ double smem[];
  __shared__ double red[40];
  __shared__ LmProblem p;
  copy_state(&p, probs + blockIdx.x);
  const int tid = threadIdx.x, T = blockDim.x;
  const int n = p.S->n;
  const NormalLayout& lay = p.lay;
  double* scratch = smem; double* dinv = smem + 2 * (n + 1);
  double* L = lay.l_in_smem ? smem + 3 * (n + 1) : lay.Lg;
  gather_blocks(lay, eout, n, p.H);
  __syncthreads();
  double bad = 0.0;
  for (int j = tid; j < n; j += T) {
    const double h = p.H[(size_t)j * n + j];
    if (!(h > 0.0) || !isfinite(h)) bad = 1.0;
    p.scale[j] = 1.0 / sqrt(h);
  }
  bad = block_sum(bad, red);
  if (bad != 0.0) { if (tid == 0) status[blockIdx.x] = MVICP_COV_SINGULAR; return; }
  for (int i = tid >> 5; i < n; i += T >> 5) {          // one warp per row, only the row's profile (as lm_step_kernel)
    const double si = p.scale[i];
    const int rbi = lay.rowbase[i];
    for (int j = lay.rfirst[i] + (tid & 31); j <= i; j += 32) L[rbi + j] = si * p.H[(size_t)i * n + j] * p.scale[j];
  }
  { const int rbn = lay.rowbase[n]; for (int j = tid; j < n; j += T) L[rbn + j] = 0.0; }
  __syncthreads();
  bool ok = chol_solve(L, lay.rowbase, n, scratch, dinv, lay.rhs, lay.rlast, lay.rfirst);
  double low = 0.0;
  if (ok) {
    const double floor_ = cov_pivot_floor(n);
    for (int j = tid; j < n; j += T) { const double l = L[lay.rowbase[j] + j]; if (!(l * l > floor_)) low = 1.0; }
  }
  low = block_sum(low, red);
  ok = ok && low == 0.0;
  if (ok) {
    if (lay.l_in_smem) for (int i = tid; i < lay.rowbase[n]; i += T) lay.Lg[i] = L[i];   // the rows of the factor, not the rhs row
    for (int j = tid; j < n; j += T) p.diag[j] = dinv[j];
  }
  if (tid == 0) status[blockIdx.x] = ok ? MVICP_COV_OK : MVICP_COV_SINGULAR;
}

// Columns job.col .. job.col + 5 of the problem's C.  Dynamic shared memory: the 6 working vectors (6 n doubles), or none --
// then each column is worked in place in its output column (the same arithmetic).
__global__ void __launch_bounds__(COV_SOLVE_THREADS) cov_solve_kernel(const LmProblem* __restrict__ probs, const CovJob* __restrict__ jobs,
                                                                      const int32_t* __restrict__ status, double* __restrict__ out,
                                                                      int vec_in_smem) {
  extern __shared__ double smem[];
  const CovJob job = jobs[blockIdx.x];
  if (status[job.prob] != MVICP_COV_OK) return;
  const LmProblem& p = probs[job.prob];
  const int n = p.S->n, lane = threadIdx.x & 31, k = job.col + (threadIdx.x >> 5);
  const double* __restrict__ L = p.lay.Lg;
  const int32_t* __restrict__ rb = p.lay.rowbase;
  const int32_t* __restrict__ rf = p.lay.rfirst;
  const int32_t* __restrict__ rl = p.lay.rlast;
  const double* __restrict__ dinv = p.diag;
  double* col = out + job.at + (size_t)(threadIdx.x >> 5) * n;
  double* v = vec_in_smem ? smem + (size_t)(threadIdx.x >> 5) * n : col;
  for (int r = lane; r < n; r += 32) v[r] = 0.0;
  __syncwarp();
  // L y = e_k: y_r = 0 above row k; row r reads columns max(rfirst[r], k) .. r - 1
  for (int r = k; r < n; ++r) {
    double s = 0.0;
    for (int c = max(rf[r], k) + lane; c < r; c += 32) s += L[rb[r] + c] * v[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const double y = ((r == k ? 1.0 : 0.0) - s) * dinv[r];
    if (lane == 0) v[r] = y;
    __syncwarp();
  }
  // L^T z = y: column c of L holds rows c + 1 .. rlast[c] whose profile reaches c
  for (int c = n - 1; c >= 0; --c) {
    double s = 0.0;
    for (int r = c + 1 + lane; r <= rl[c]; r += 32) if (rf[r] <= c) s += L[rb[r] + c] * v[r];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const double z = (v[c] - s) * dinv[c];
    __syncwarp();
    if (lane == 0) v[c] = z;
    __syncwarp();
  }
  const double sk = p.scale[k];
  for (int i = lane; i < n; i += 32) col[i] = p.scale[i] * v[i] * sk;
}

}  // namespace mv
