// tools/hostshim/cuda_runtime.h -- stands in for <cuda_runtime.h> when the engine's .cuh files are compiled by g++ for the
// host checks (tools/knn_host_check.cpp): the device intrinsics the search uses, as plain C++.  Directed-rounding
// intrinsics are emulated in double and rounded in the stated direction (conservative: never below the hardware result's
// true value), so the SEARCH LOGIC and the exactness argument are exercised; the hardware's exact roundings are not.
#pragma once
#include <vector_types.h>   // the real CUDA header: plain structs (float4, double2, ...), usable by host compilers
#include <cmath>
#include <cstdint>
#include <cstring>
#include <algorithm>
using std::min; using std::max;
#ifndef __launch_bounds__
#define __launch_bounds__(...)
#endif
struct HostDim3 { unsigned x = 0, y = 0, z = 0; };
static thread_local HostDim3 threadIdx, blockIdx;
static HostDim3 blockDim, gridDim;
typedef void* cudaStream_t;
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline int __float_as_int(float f) { int i; std::memcpy(&i, &f, 4); return i; }
static inline float __int_as_float(int i) { float f; std::memcpy(&f, &i, 4); return f; }
static inline long long __double_as_longlong(double d) { long long l; std::memcpy(&l, &d, 8); return l; }
static inline double __longlong_as_double(long long l) { double d; std::memcpy(&d, &l, 8); return d; }
static inline double __dmul_rn(double a, double b) { return a * b; }   // compile with -ffp-contract=off
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline double __dsub_rn(double a, double b) { return a - b; }
static inline double __ddiv_rn(double a, double b) { return a / b; }
static inline double __dsqrt_rn(double a) { return std::sqrt(a); }
static inline float hs_up(double v) { float f = (float)v; if ((double)f < v) f = std::nextafterf(f, INFINITY); return f; }
static inline float __double2float_ru(double a) { return hs_up(a); }
static inline float __fsqrt_ru(float a) { return std::nextafterf(hs_up(std::sqrt((double)a)), INFINITY); }
static inline float __fadd_ru(float a, float b) { return hs_up((double)a + (double)b); }
static inline float4 make_float4(float x, float y, float z, float w) { float4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }
static inline int2 make_int2(int x, int y) { int2 r; r.x = x; r.y = y; return r; }
static inline int __ffs(unsigned x) { return __builtin_ffs((int)x); }
static inline float __fmul_ru(float a, float b) { return hs_up((double)a * (double)b); }
static inline float hs_down(double v) { float f = (float)v; if ((double)f > v) f = std::nextafterf(f, -INFINITY); return f; }
static inline float __fmul_rd(float a, float b) { return hs_down((double)a * (double)b); }
static inline float __fsub_rd(float a, float b) { return hs_down((double)a - (double)b); }
static inline float __fmaf_ru(float a, float b, float c) { return std::nextafterf(hs_up((double)a * (double)b + (double)c), INFINITY); }
static inline void __syncthreads() {}
// declarations only, so that the kernels' text parses: the host check calls the search functions, never a kernel
unsigned __ballot_sync(unsigned, int);
unsigned __match_any_sync(unsigned, int);
unsigned __reduce_min_sync(unsigned, unsigned);
unsigned __reduce_max_sync(unsigned, unsigned);
template <class T> T __shfl_sync(unsigned, T, int, int = 32);
static inline unsigned __float_as_uint(float f) { unsigned i; std::memcpy(&i, &f, 4); return i; }
static inline float __uint_as_float(unsigned i) { float f; std::memcpy(&f, &i, 4); return f; }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
template <class T> T atomicAdd(T*, T);
static inline void __syncwarp() {}
static inline int __any_sync(unsigned, int p) { return p; }   // one-lane "warp"
