// tree_gpu.cuh -- one-time construction of the per-frame search structure ON THE DEVICE (replaces the lazily built nanoflann
// index, src/internal/frame.cpp:188-193, nanoflann.hpp:859-867,1034-1085; the host version of the same construction is
// tree_build.h, kept for MVICP_FLAG_HOST_BUILD and for the host model of the engine).
//
// Same structure as tree_build.h: points in left-balanced KD order (the node that covers leaf slots [a, b) of the implicit tree
// holds the tree positions [8a, min(8b, n)); a node whose points exceed the capacity of its left half is split along the widest
// axis of their bounding box, the smallest `capacity` coordinates going left), fp32 boxes rounded outward, one-sided split
// bounds ("faces"), hybrid oriented boxes for the far rounds.  Top-down, one level at a time for the whole frame:
//   bbox   per node of the level: bounding box of its points (block / warp aggregated atomics on order-preserving ints);
//   key    per point: (node << 32 | coordinate along the node's split axis as an order-preserving uint32) -- nodes that do
//          not split keep their order (key = offset in the node);
//   sort   one radix sort of the frame's (key, index) pairs over the 32 + level significant bits (cub::DeviceRadixSort: the
//          one library primitive of this file, used at set-up only) -- every node's points stay inside its own range, sorted
//          along its axis, so its first `capacity` points are its left child's.
// Then bottom-up: fp64 leaf boxes and moments, merged level by level; fp32 boxes / faces / oriented boxes per node.
// The search is exact for ANY such tree (boxes and faces are computed from the points they bound), so the device and the host
// construction give the same matches; ties between equal fp32 keys may order two points differently, nothing else differs.
#pragma once
#ifdef __CUDACC__
#include <cub/device/device_radix_sort.cuh>
#include <cuda_runtime.h>
#include <stdint.h>
#include "adjacency.h"
#include "far.cuh"
#include "types.cuh"

namespace mv {

__device__ __forceinline__ int f2ord(float f) { const int b = __float_as_int(f); return b >= 0 ? b : b ^ 0x7fffffff; }
__device__ __forceinline__ float ord2f(int o) { return __int_as_float(o >= 0 ? o : o ^ 0x7fffffff); }
__device__ __forceinline__ unsigned f2key(float f) { const unsigned b = (unsigned)__float_as_int(f); return (b & 0x80000000u) ? ~b : (b | 0x80000000u); }
__device__ __forceinline__ float d_down(double v) { float f = __double2float_rd(v); return f; }
__device__ __forceinline__ float d_up(double v) { float f = __double2float_ru(v); return f; }

struct KdGeom { int n, L, depth; };   // points, padded leaf count (power of two), log2 L

__global__ void kd_iota_kernel(int* __restrict__ idx, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) idx[i] = i;
}

// flags[0] &= every coordinate is exactly fp32-representable; flags[1] = max |coordinate| as float bits (non-negative floats order like ints)
__global__ void kd_scan_kernel(const double* __restrict__ v, long long n3, int* __restrict__ flags) {
  bool ok = true; float am = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n3; i += (long long)gridDim.x * blockDim.x) {
    const double x = v[i];
    if ((double)(float)x != x) ok = false;
    am = fmaxf(am, __double2float_ru(fabs(x)));
  }
  if (!__all_sync(0xffffffffu, ok)) { if ((threadIdx.x & 31) == 0) atomicAnd(&flags[0], 0); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) am = fmaxf(am, __shfl_down_sync(0xffffffffu, am, o));
  if ((threadIdx.x & 31) == 0) atomicMax(&flags[1], __float_as_int(am));
}

__global__ void kd_bbox_init_kernel(int* __restrict__ bb, int n_nodes) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_nodes * 6) bb[i] = (i % 6) < 3 ? 0x7fffffff : (int)0x80000000;
}

// bounding box (fp32, order-preserving ints) of the points of every node of one level; shift = 3 + depth - level
__global__ void __launch_bounds__(256)
kd_bbox_kernel(const double* __restrict__ xyz, const int* __restrict__ idx, int n, int shift, int* __restrict__ bb) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = p < n;
  const int q = in ? p : n - 1;
  const int seg = q >> shift;
  const double* c = xyz + 3 * (size_t)idx[q];
  int lo[3], hi[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) { const float f = (float)c[a]; lo[a] = f2ord(f); hi[a] = lo[a]; }
  // a warp that lies in one node (every level but the lowest two) reduces by shuffles; the warps of a block that share a node are
  // merged through shared memory before the atomics; a warp that straddles nodes falls back to per-thread atomics
  __shared__ int s_lo[8][3], s_hi[8][3], s_seg[8];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int seg0 = __shfl_sync(0xffffffffu, seg, 0);
  const bool uniform = __all_sync(0xffffffffu, seg == seg0);
  if (uniform) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
      for (int a = 0; a < 3; ++a) { lo[a] = min(lo[a], __shfl_down_sync(0xffffffffu, lo[a], o)); hi[a] = max(hi[a], __shfl_down_sync(0xffffffffu, hi[a], o)); }
    if (lane == 0) { for (int a = 0; a < 3; ++a) { s_lo[w][a] = lo[a]; s_hi[w][a] = hi[a]; } s_seg[w] = seg0; }
  } else {
    if (in) for (int a = 0; a < 3; ++a) { atomicMin(&bb[6 * seg + a], lo[a]); atomicMax(&bb[6 * seg + 3 + a], hi[a]); }
    if (lane == 0) s_seg[w] = -1;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 0; i < 8; ++i) {
      if (s_seg[i] < 0) continue;
      int l3[3] = {s_lo[i][0], s_lo[i][1], s_lo[i][2]}, h3[3] = {s_hi[i][0], s_hi[i][1], s_hi[i][2]};
      for (int j = i + 1; j < 8; ++j) if (s_seg[j] == s_seg[i]) { for (int a = 0; a < 3; ++a) { l3[a] = min(l3[a], s_lo[j][a]); h3[a] = max(h3[a], s_hi[j][a]); } s_seg[j] = -1; }
      for (int a = 0; a < 3; ++a) { atomicMin(&bb[6 * s_seg[i] + a], l3[a]); atomicMax(&bb[6 * s_seg[i] + 3 + a], h3[a]); }
    }
  }
}

// sort key of every tree position for one level, and the split axis of every node of the level
__global__ void __launch_bounds__(256)
kd_key_kernel(const double* __restrict__ xyz, const int* __restrict__ idx, KdGeom g, int level, const int* __restrict__ bb,
              unsigned long long* __restrict__ keys, uint8_t* __restrict__ axis_of) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= g.n) return;
  const int shift = 3 + g.depth - level;
  const int seg = p >> shift;
  const long long begin = (long long)seg << shift;
  const long long count = min((long long)g.n - begin, 1ll << shift);
  const long long cap_left = 1ll << (shift - 1);
  unsigned k32 = (unsigned)(p - begin);
  if (count > cap_left) {   // the node splits: order its points along the widest axis of their bounding box
    const int* b = bb + 6 * seg;
    float ext[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) ext[a] = ord2f(b[3 + a]) - ord2f(b[a]);
    int ax = 0;
    if (ext[1] > ext[ax]) ax = 1;
    if (ext[2] > ext[ax]) ax = 2;
    k32 = f2key((float)xyz[3 * (size_t)idx[p] + ax]);
    if (p == begin) axis_of[(1 << level) + seg] = (uint8_t)ax;
  }
  keys[p] = ((unsigned long long)seg << 32) | k32;
}

// tree-order records (+ fp32 screening copy in the fp64 storage mode), original index -> tree position
template <bool F32>
__global__ void kd_pack_tree_kernel(const double* __restrict__ xyz, const int* __restrict__ order, int n, int n_pad, void* __restrict__ pts_s,
                                    float4* __restrict__ pts_sf, int32_t* __restrict__ pos_of) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pad) return;
  double x = __longlong_as_double(0x7ff0000000000000LL), y = x, z = x; int w = INT32_MAX;
  if (i < n) { const int o = order[i]; x = xyz[3 * (size_t)o]; y = xyz[3 * (size_t)o + 1]; z = xyz[3 * (size_t)o + 2]; w = o; pos_of[o] = i; }
  if (F32) reinterpret_cast<float4*>(pts_s)[i] = make_float4((float)x, (float)y, (float)z, __int_as_float(w));
  else {
    double4a r; r.x = x; r.y = y; r.z = z; r.w = __longlong_as_double((long long)w);
    reinterpret_cast<double4a*>(pts_s)[i] = r;
    pts_sf[i] = make_float4((float)x, (float)y, (float)z, __int_as_float(w));
  }
}
// caller's-order records of points or normals
template <bool F32>
__global__ void kd_pack_orig_kernel(const double* __restrict__ v, int n, void* __restrict__ rec) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (F32) reinterpret_cast<float4*>(rec)[i] = make_float4((float)v[3 * (size_t)i], (float)v[3 * (size_t)i + 1], (float)v[3 * (size_t)i + 2], 0.f);
  else { double4a r; r.x = v[3 * (size_t)i]; r.y = v[3 * (size_t)i + 1]; r.z = v[3 * (size_t)i + 2]; r.w = 0.0; reinterpret_cast<double4a*>(rec)[i] = r; }
}

struct KdMom { double n, s[3], ss[6]; };   // point count, sum p, sum p p^T (upper) of a node

// fp64 box and moments of every leaf slot (empty slots: +inf / -inf, zero moments)
__global__ void kd_leaf_kernel(const double* __restrict__ xyz, const int* __restrict__ order, KdGeom g, double* __restrict__ dbox /*[2L][6]*/,
                               KdMom* __restrict__ mom /*[2L] or null*/) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= g.L) return;
  const double inf = __longlong_as_double(0x7ff0000000000000LL);
  double lo[3] = {inf, inf, inf}, hi[3] = {-inf, -inf, -inf};
  KdMom m; m.n = 0; for (int a = 0; a < 3; ++a) m.s[a] = 0; for (int a = 0; a < 6; ++a) m.ss[a] = 0;
  for (long long i = (long long)l * LEAF; i < min((long long)g.n, (long long)(l + 1) * LEAF); ++i) {
    const double* p = xyz + 3 * (size_t)order[i];
    for (int a = 0; a < 3; ++a) { lo[a] = fmin(lo[a], p[a]); hi[a] = fmax(hi[a], p[a]); m.s[a] += p[a]; }
    m.n += 1;
    m.ss[0] += p[0] * p[0]; m.ss[1] += p[0] * p[1]; m.ss[2] += p[0] * p[2]; m.ss[3] += p[1] * p[1]; m.ss[4] += p[1] * p[2]; m.ss[5] += p[2] * p[2];
  }
  double* b = dbox + 6 * (size_t)(g.L + l);
  for (int a = 0; a < 3; ++a) { b[a] = lo[a]; b[3 + a] = hi[a]; }
  if (mom) mom[g.L + l] = m;
}
__global__ void kd_merge_kernel(int first, double* __restrict__ dbox, KdMom* __restrict__ mom) {   // nodes [first, 2 first)
  const int i = first + blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * first) return;
  const double* x = dbox + 6 * (size_t)(2 * i); const double* y = x + 6;
  double* b = dbox + 6 * (size_t)i;
  for (int a = 0; a < 3; ++a) { b[a] = fmin(x[a], y[a]); b[3 + a] = fmax(x[3 + a], y[3 + a]); }
  if (mom) {
    const KdMom &mx = mom[2 * i], &my = mom[2 * i + 1]; KdMom m;
    m.n = mx.n + my.n; for (int a = 0; a < 3; ++a) m.s[a] = mx.s[a] + my.s[a]; for (int a = 0; a < 6; ++a) m.ss[a] = mx.ss[a] + my.ss[a];
    mom[i] = m;
  }
}

// fp32 box rounded outward and the one-sided bound along the parent's split axis (tree_build.h:build_frame, same rules)
__global__ void kd_boxface_kernel(int L, const double* __restrict__ dbox, const uint8_t* __restrict__ axis_of, Box* __restrict__ boxes,
                                  float* __restrict__ faces) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * L) return;
  Box b; b.pad[0] = b.pad[1] = 0.f;
  if (i == 0) { for (int a = 0; a < 3; ++a) { b.lo[a] = __int_as_float(0x7f800000); b.hi[a] = -b.lo[a]; } boxes[0] = b; faces[0] = 0.f; return; }
  const double* d = dbox + 6 * (size_t)i;
  for (int a = 0; a < 3; ++a) { b.lo[a] = d_down(d[a]); b.hi[a] = d_up(d[3 + a]); }
  boxes[i] = b;
  float ff = 0.f;
  if (i >= 2) {
    const int axp = axis_of[i / 2]; const bool right = (i & 1) != 0;
    ff = right ? d_down(d[axp]) : d_up(d[3 + axp]);   // +inf / -inf for empty nodes
    for (int guard = 0; guard < 8 && isfinite(ff); ++guard) {   // the axis rides in the two low mantissa bits: move the bound outward until they match
      const unsigned bits = (unsigned)__float_as_int(ff);
      if ((bits & 3u) == (unsigned)axp) break;
      ff = right ? nextafterf(ff, -__int_as_float(0x7f800000)) : nextafterf(ff, __int_as_float(0x7f800000));
    }
    if (!isfinite(ff)) ff = __int_as_float(__float_as_int(ff) & ~3);   // inf: low bits 0 = axis 0, any axis prunes
  }
  faces[i] = ff;
}

// neighbour list and reach of every leaf (adjacency.h)
__global__ void kd_adj_kernel(const Box* __restrict__ boxes, int L, int n_leaf, int32_t* __restrict__ adj) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= L) return;
  int32_t o[ADJ_SLOTS];
  adj_build_leaf(boxes, L, n_leaf, l, o);
  for (int i = 0; i < ADJ_SLOTS; ++i) adj[(size_t)ADJ_SLOTS * l + i] = o[i];
}

// hybrid oriented boxes (tree_build.h:build_obb, same rules): per node the box of the coordinate axes, or -- nodes of at most
// OBB_PCA_LEAVES leaves whose principal-axes box is clearly smaller -- the box of the principal axes of its points
__global__ void kd_obb_kernel(const double* __restrict__ xyz, const int* __restrict__ order, KdGeom g, const double* __restrict__ dbox,
                              const KdMom* __restrict__ mom, ObbNode* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * g.L) return;
  ObbNode b;
  b.c[0] = b.c[1] = b.c[2] = 0.f; b.a0[0] = 1.f; b.a0[1] = b.a0[2] = 0.f; b.a1[1] = 1.f; b.a1[0] = b.a1[2] = 0.f; b.a2[2] = 1.f; b.a2[0] = b.a2[1] = 0.f;
  b.e0 = b.e1 = b.e2 = -__int_as_float(0x7f800000); b.pad = 0.f;
  if (i == 0 || mom[i].n < 1) { out[i] = b; return; }
  const KdMom mm = mom[i];
  int lev = 31 - __clz(i);
  const int first = 1 << lev, per = g.L >> lev;
  const double mean[3] = {mm.s[0] / mm.n, mm.s[1] / mm.n, mm.s[2] / mm.n};
  const double* d = dbox + 6 * (size_t)i;
  double best_vol;
  {   // candidate 0: coordinate axes -- centre and half extents from the exact fp64 box
    float cf[3]; double ext[3];
    for (int k = 0; k < 3; ++k) { cf[k] = (float)(0.5 * (d[k] + d[3 + k])); ext[k] = fmax(d[3 + k] - (double)cf[k], (double)cf[k] - d[k]); }
    const double floor_e = 1e-7 * (fabs(mean[0]) + fabs(mean[1]) + fabs(mean[2]) + 1e-3);
    best_vol = (ext[0] + floor_e) * (ext[1] + floor_e) * (ext[2] + floor_e);
    for (int k = 0; k < 3; ++k) b.c[k] = cf[k];
    b.e0 = d_up(ext[0] * (1.0 + 1e-6)); b.e1 = d_up(ext[1] * (1.0 + 1e-6)); b.e2 = d_up(ext[2] * (1.0 + 1e-6));
  }
  if (mm.n >= 3 && per <= OBB_PCA_LEAVES) {
    double C[3][3] = {{mm.ss[0] / mm.n - mean[0] * mean[0], mm.ss[1] / mm.n - mean[0] * mean[1], mm.ss[2] / mm.n - mean[0] * mean[2]},
                      {0, mm.ss[3] / mm.n - mean[1] * mean[1], mm.ss[4] / mm.n - mean[1] * mean[2]},
                      {0, 0, mm.ss[5] / mm.n - mean[2] * mean[2]}};
    C[1][0] = C[0][1]; C[2][0] = C[0][2]; C[2][1] = C[1][2];
    double V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int sweep = 0; sweep < 12; ++sweep) {   // cyclic Jacobi, symmetric 3x3
      if (fabs(C[0][1]) + fabs(C[0][2]) + fabs(C[1][2]) < 1e-30) break;
      for (int p = 0; p < 2; ++p)
        for (int q = p + 1; q < 3; ++q) {
          if (fabs(C[p][q]) < 1e-300) continue;
          const double th = (C[q][q] - C[p][p]) / (2.0 * C[p][q]);
          const double tt = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
          const double cs = 1.0 / sqrt(tt * tt + 1.0), sn = tt * cs;
          for (int k = 0; k < 3; ++k) { const double ckp = C[k][p], ckq = C[k][q]; C[k][p] = cs * ckp - sn * ckq; C[k][q] = sn * ckp + cs * ckq; }
          for (int k = 0; k < 3; ++k) { const double cpk = C[p][k], cqk = C[q][k]; C[p][k] = cs * cpk - sn * cqk; C[q][k] = sn * cpk + cs * cqk; }
          for (int k = 0; k < 3; ++k) { const double vkp = V[k][p], vkq = V[k][q]; V[k][p] = cs * vkp - sn * vkq; V[k][q] = sn * vkp + cs * vkq; }
        }
    }
    float A[3][3];
    for (int a = 0; a < 3; ++a) for (int k = 0; k < 3; ++k) A[a][k] = (float)V[k][a];
    bool ortho = true;
    for (int a = 0; a < 3; ++a)
      for (int k = a; k < 3; ++k) {
        const double dp = (double)A[a][0] * A[k][0] + (double)A[a][1] * A[k][1] + (double)A[a][2] * A[k][2];
        if (!(fabs(dp - (a == k ? 1.0 : 0.0)) < 2e-7)) ortho = false;
      }
    if (ortho) {
      const long long lo_leaf = (long long)(i - first) * per;
      const long long t0 = lo_leaf * LEAF, t1 = min((long long)g.n, (lo_leaf + per) * LEAF);
      const double inf = __longlong_as_double(0x7ff0000000000000LL);
      double mn[3] = {inf, inf, inf}, mx[3] = {-inf, -inf, -inf};
      for (long long t = t0; t < t1; ++t) {
        const double* p = xyz + 3 * (size_t)order[t];
        const double dd[3] = {p[0] - mean[0], p[1] - mean[1], p[2] - mean[2]};
        for (int a = 0; a < 3; ++a) { const double pr = (double)A[a][0] * dd[0] + (double)A[a][1] * dd[1] + (double)A[a][2] * dd[2]; mn[a] = fmin(mn[a], pr); mx[a] = fmax(mx[a], pr); }
      }
      float cf[3];
      for (int k = 0; k < 3; ++k) { double ck = mean[k]; for (int a = 0; a < 3; ++a) ck += (double)A[a][k] * 0.5 * (mn[a] + mx[a]); cf[k] = (float)ck; }
      double ext[3] = {0, 0, 0};
      for (long long t = t0; t < t1; ++t) {   // extents against the STORED fp32 centre and axes: the containment the search relies on is exact
        const double* p = xyz + 3 * (size_t)order[t];
        const double dd[3] = {p[0] - (double)cf[0], p[1] - (double)cf[1], p[2] - (double)cf[2]};
        for (int a = 0; a < 3; ++a) ext[a] = fmax(ext[a], fabs((double)A[a][0] * dd[0] + (double)A[a][1] * dd[1] + (double)A[a][2] * dd[2]));
      }
      const double floor_e = 1e-7 * (fabs(mean[0]) + fabs(mean[1]) + fabs(mean[2]) + 1e-3);
      const double vol = (ext[0] + floor_e) * (ext[1] + floor_e) * (ext[2] + floor_e);
      if (vol < 0.5 * best_vol) {
        for (int k = 0; k < 3; ++k) { b.c[k] = cf[k]; b.a0[k] = A[0][k]; b.a1[k] = A[1][k]; b.a2[k] = A[2][k]; }
        b.e0 = d_up(ext[0] * (1.0 + 1e-6)); b.e1 = d_up(ext[1] * (1.0 + 1e-6)); b.e2 = d_up(ext[2] * (1.0 + 1e-6));
      }
    }
  }
  out[i] = b;
}

// scratch of one build, reused across frames (sized for the largest)
struct KdScratch {
  unsigned long long* keys[2] = {nullptr, nullptr}; int* vals[2] = {nullptr, nullptr};
  void* cub_tmp = nullptr; size_t cub_bytes = 0;
  int* bb = nullptr; uint8_t* axis_of = nullptr; double* dbox = nullptr; KdMom* mom = nullptr;
  size_t cap_n = 0, cap_L = 0;
  void release() {
    for (int i = 0; i < 2; ++i) { cudaFree(keys[i]); cudaFree(vals[i]); keys[i] = nullptr; vals[i] = nullptr; }
    cudaFree(cub_tmp); cudaFree(bb); cudaFree(axis_of); cudaFree(dbox); cudaFree(mom);
    cub_tmp = nullptr; bb = nullptr; axis_of = nullptr; dbox = nullptr; mom = nullptr; cap_n = cap_L = 0; cub_bytes = 0;
  }
  cudaError_t reserve(size_t n, size_t L) {
    if (n <= cap_n && L <= cap_L) return cudaSuccess;
    release();
    cudaError_t e;
    for (int i = 0; i < 2; ++i) { if ((e = cudaMalloc(&keys[i], 8 * n)) != cudaSuccess) return e; if ((e = cudaMalloc(&vals[i], 4 * n)) != cudaSuccess) return e; }
    cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, keys[0], keys[1], vals[0], vals[1], (int)n, 0, 64);
    if ((e = cudaMalloc(&cub_tmp, cub_bytes + 16)) != cudaSuccess) return e;
    if ((e = cudaMalloc(&bb, sizeof(int) * 6 * L)) != cudaSuccess) return e;
    if ((e = cudaMalloc(&axis_of, 2 * L)) != cudaSuccess) return e;
    if ((e = cudaMalloc(&dbox, sizeof(double) * 6 * 2 * L)) != cudaSuccess) return e;
    if ((e = cudaMalloc(&mom, sizeof(KdMom) * 2 * L)) != cudaSuccess) return e;
    cap_n = n; cap_L = L;
    return cudaSuccess;
  }
};

// Orders the frame's points (d_xyz: n x 3 doubles on the device) and fills the frame's arrays (allocated by the caller).
// order_out: tree position -> original index.  Returns the first CUDA error.
template <bool F32>
static cudaError_t kd_build_device(cudaStream_t st, KdScratch& S, const double* d_xyz, KdGeom g, void* pts_s, float4* pts_sf, int32_t* pos_of,
                                   Box* boxes, float* faces, int32_t* adj, ObbNode* obb /*nullable*/, int64_t* launches) {
  const int n = g.n, L = g.L, T = 256;
  cudaError_t e = S.reserve((size_t)n, (size_t)L);
  if (e != cudaSuccess) return e;
  int cur = 0;
  kd_iota_kernel<<<(n + T - 1) / T, T, 0, st>>>(S.vals[0], n);
  cudaMemsetAsync(S.axis_of, 0, 2 * (size_t)L, st);
  *launches += 1;
  for (int level = 0; level < g.depth; ++level) {
    const int nodes = 1 << level, shift = 3 + g.depth - level;
    if ((long long)n <= (1ll << (shift - 1))) continue;   // even the first node of the level does not exceed its left half: nothing splits
    kd_bbox_init_kernel<<<(nodes * 6 + T - 1) / T, T, 0, st>>>(S.bb, nodes);
    kd_bbox_kernel<<<(n + T - 1) / T, T, 0, st>>>(d_xyz, S.vals[cur], n, shift, S.bb);
    kd_key_kernel<<<(n + T - 1) / T, T, 0, st>>>(d_xyz, S.vals[cur], g, level, S.bb, S.keys[cur], S.axis_of);
    size_t tmp = S.cub_bytes;
    e = cub::DeviceRadixSort::SortPairs(S.cub_tmp, tmp, S.keys[cur], S.keys[cur ^ 1], S.vals[cur], S.vals[cur ^ 1], n, 0, 32 + level, st);
    if (e != cudaSuccess) return e;
    cur ^= 1;
    *launches += 4;
  }
  const int* order = S.vals[cur];
  const int n_pad = ((n + LEAF - 1) / LEAF) * LEAF;
  kd_pack_tree_kernel<F32><<<(n_pad + T - 1) / T, T, 0, st>>>(d_xyz, order, n, n_pad, pts_s, pts_sf, pos_of);
  kd_leaf_kernel<<<(L + T - 1) / T, T, 0, st>>>(d_xyz, order, g, S.dbox, obb ? S.mom : nullptr);
  for (int first = L / 2; first >= 1; first /= 2) kd_merge_kernel<<<(first + T - 1) / T, T, 0, st>>>(first, S.dbox, obb ? S.mom : nullptr);
  kd_boxface_kernel<<<(2 * L + T - 1) / T, T, 0, st>>>(L, S.dbox, S.axis_of, boxes, faces);
  kd_adj_kernel<<<(L + 63) / 64, 64, 0, st>>>(boxes, L, (n + LEAF - 1) / LEAF, adj);
  if (obb) kd_obb_kernel<<<(2 * L + T - 1) / T, T, 0, st>>>(d_xyz, order, g, S.dbox, S.mom, obb);
  *launches += 4 + g.depth + (obb ? 1 : 0);
  return cudaGetLastError();
}

}  // namespace mv
#endif  // __CUDACC__
