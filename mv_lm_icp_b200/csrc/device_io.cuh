// device_io.cuh -- kernels of the entry points that take per-point arrays in device memory (include/mvicp.h, "device twins").
//
// Each twin returns the same bytes as its host-memory counterpart.  The batched closest-point query runs the search of
// knn_single_kernel (mvicp_closest_point) once per thread, so every query sees the same fp32 screen, fp64 re-rank and
// lowest-index tie rule; the caller-supplied matches of mvicp_set_edge_device are checked, reduced to one winner per src slot
// (the last occurrence, as the host loop's plain overwrite) and written in two launches.
#pragma once
#include <cuda_runtime.h>
#include "knn.cuh"
#include "types.cuh"

namespace mv {

// Frame::getClosestPoint for q[i] (frame-local coordinates), i < n.  A query with a non-finite coordinate gets idx -1, d2 NaN.
template <bool F32>
__global__ void __launch_bounds__(128)
closest_points_kernel(const FrameDev* __restrict__ frames, int frame, const double* __restrict__ q, long long n,
                      long long* __restrict__ out_idx, double* __restrict__ out_d2) {
  const FrameDev fd = frames[frame];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double qx = q[3 * i], qy = q[3 * i + 1], qz = q[3 * i + 2];
    long long bi = -1; double best = __longlong_as_double(0x7ff8000000000000LL);
    if (isfinite(qx) && isfinite(qy) && isfinite(qz)) {
      NNQuery nq; nn_query_init(nq, qx, qy, qz, fd.absmax);
      nn_search<F32, NNQuery>(fd, nq, -1);
      bi = nq.bi; best = nq.best;
    }
    if (out_idx) out_idx[i] = bi;
    if (out_d2) out_d2[i] = best;
  }
}

// mvicp_set_edge_device, pass 1: the range check (lowest bad position -> *bad, which starts at ~0) and, for every valid pair,
// win[first[i]] = max(win, i + 1): the last occurrence of a src index wins, as in the host loop.
__global__ void __launch_bounds__(256)
set_edge_scan_kernel(const int32_t* __restrict__ first, const int32_t* __restrict__ second, long long count, int n_src, int n_dst,
                     unsigned long long* __restrict__ win, unsigned long long* __restrict__ bad) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) {
    const int32_t f = first[i], s = second[i];
    if (f < 0 || f >= n_src || s < 0 || s >= n_dst) atomicMin(bad, (unsigned long long)i);
    else atomicMax(win + f, (unsigned long long)i + 1ull);
  }
}

// pass 2: every slot of the edge from its winner (~0 = no match), then weight and count -- nothing at all when pass 1 found a
// bad index, so that a rejected call leaves the edge as it was
__global__ void __launch_bounds__(256)
set_edge_write_kernel(const int32_t* __restrict__ second, const unsigned long long* __restrict__ win, int n_src,
                      const unsigned long long* __restrict__ bad, int32_t* __restrict__ corr, float* __restrict__ weight_slot,
                      unsigned long long* __restrict__ count_slot, float weight, unsigned long long count) {
  if (*bad != ~0ull) return;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n_src; k += (long long)gridDim.x * blockDim.x) {
    const unsigned long long w = win[k];
    corr[k] = w ? second[w - 1] : ~0;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) { *weight_slot = weight; *count_slot = count; }
}

}  // namespace mv
