// tools/hostemu/cuda_runtime.h -- TEST INFRASTRUCTURE.  A miniature CUDA execution model for the host, so that the engine's
// own sources (csrc/*.cuh, mvicp.cu) can be compiled by g++ and their LOGIC exercised by the CPU test-suite
// (tests/test_hostemu_*.py; built by tools/hostemu/build_hostemu.py).  It is not a CPU path of the product: nothing under
// mv_lm_icp_b200/ knows about it, and it models neither the hardware's roundings nor its memory model.
//
//  * every CTA of a launch runs to completion before the next (blocks are independent in CUDA);
//  * the threads of a CTA are fibers (ucontext) of one OS thread, switched only at __syncthreads / __syncwarp / shuffles /
//    votes; a thread that returns from the kernel simply stops taking part in later barriers, as on the device;
//  * __shared__ becomes `static` (one CTA at a time), dynamic shared memory is a per-launch buffer (dyn_smem());
//  * device memory is host memory, streams/events are no-ops, atomics are plain (one OS thread);
//  * directed-rounding float intrinsics are evaluated in double and rounded outward (conservative).
#pragma once
#include <vector_types.h>   // the real CUDA header: float4, double2, dim3, uint3 ... as plain structs
#undef __shared__
#define __shared__ static
#undef __launch_bounds__
#define __launch_bounds__(...)
#include <ucontext.h>
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>
using std::min; using std::max;

// ---- execution model --------------------------------------------------------------------------------------------
static uint3 threadIdx, blockIdx;
static dim3 blockDim, gridDim;
namespace hostemu {
enum { RUN = 0, AT_BLOCK = 1, AT_WARP = 2, DONE = 3 };
// Context switch: on x86-64 a six-register stack switch (a barrier costs ~20 ns per thread); elsewhere ucontext (~1 us).
#if defined(__x86_64__)
extern "C" void hostemu_switch(void** save_sp, void* load_sp);
__asm__(".text\n.globl hostemu_switch\n.type hostemu_switch,@function\nhostemu_switch:\n"
        "  pushq %rbp\n  pushq %rbx\n  pushq %r12\n  pushq %r13\n  pushq %r14\n  pushq %r15\n"
        "  movq %rsp, (%rdi)\n  movq %rsi, %rsp\n"
        "  popq %r15\n  popq %r14\n  popq %r13\n  popq %r12\n  popq %rbx\n  popq %rbp\n  ret\n"
        ".size hostemu_switch, .-hostemu_switch\n");
struct Fiber { void* sp; int state; char* stack; };
static void* sched_sp = nullptr;
#else
struct Fiber { ucontext_t ctx; int state; char* stack; };
static ucontext_t sched_ctx;
#endif
static std::vector<Fiber> fibers; static int cur = -1, n_threads = 0;
static const std::function<void()>* body = nullptr;
static std::vector<char> dyn; static long long warp_slot[64][32]; static int vote_slot[64][32];
static const size_t STACK = 256 * 1024;
static std::vector<int> perm; static unsigned long long rng_state = 0x9E3779B97F4A7C15ULL;
static const int order_mode = []() { const char* e = std::getenv("HOSTEMU_ORDER"); return !e ? 0 : (e[0] == 'r' && e[1] == 'e' ? 1 : (e[0] == 'r' ? 2 : 0)); }();
inline void* dyn_smem() { return dyn.data(); }
#if defined(__x86_64__)
inline void to_sched() { hostemu_switch(&fibers[cur].sp, sched_sp); }
inline void to_fiber(int t) { hostemu_switch(&sched_sp, fibers[t].sp); }
#else
inline void to_sched() { swapcontext(&fibers[cur].ctx, &sched_ctx); }
inline void to_fiber(int t) { swapcontext(&sched_ctx, &fibers[t].ctx); }
#endif
inline void fiber_main() { (*body)(); fibers[cur].state = DONE; to_sched(); std::abort(); }
inline void yield(int st) { fibers[cur].state = st; to_sched(); }
inline void set_ids(int t) { threadIdx.x = (unsigned)t % blockDim.x; threadIdx.y = ((unsigned)t / blockDim.x) % blockDim.y; threadIdx.z = (unsigned)t / (blockDim.x * blockDim.y); }
inline void run_block() {
  const int n = n_threads;
  if ((int)fibers.size() < n) { const size_t o = fibers.size(); fibers.resize(n); for (size_t i = o; i < (size_t)n; ++i) fibers[i].stack = (char*)std::malloc(STACK); }
  for (int t = 0; t < n; ++t) {
#if defined(__x86_64__)
    void** sp = (void**)(((uintptr_t)fibers[t].stack + STACK) & ~(uintptr_t)15);
    *--sp = nullptr;                       // fake return address of fiber_main (it never returns)
    *--sp = (void*)fiber_main;             // `ret` of the first switch jumps here with rsp = 16k + 8, as after a call
    for (int r = 0; r < 6; ++r) *--sp = nullptr;
    fibers[t].sp = sp;
#else
    getcontext(&fibers[t].ctx); fibers[t].ctx.uc_stack.ss_sp = fibers[t].stack; fibers[t].ctx.uc_stack.ss_size = STACK; fibers[t].ctx.uc_link = nullptr;
    makecontext(&fibers[t].ctx, (void (*)())fiber_main, 0);
#endif
    fibers[t].state = RUN;
  }
  std::memset(vote_slot, 0, sizeof vote_slot);
  while (true) {
    bool progressed = false, alive = false;
    // scheduling order between two barriers: ascending thread index, descending (HOSTEMU_ORDER=reverse) or a fresh
    // pseudo-random permutation every phase (HOSTEMU_ORDER=random): code that lacks a barrier passes under one order at most
    for (int i = 0; i < n; ++i) {
      int t = i;
      if (order_mode == 1) t = n - 1 - i;
      else if (order_mode == 2) { if (i == 0) { perm.resize(n); for (int k = 0; k < n; ++k) perm[k] = k; for (int k = n - 1; k > 0; --k) { rng_state = rng_state * 6364136223846793005ULL + 1442695040888963407ULL; std::swap(perm[k], perm[(rng_state >> 33) % (unsigned)(k + 1)]); } } t = perm[i]; }
      if (fibers[t].state == RUN) { cur = t; set_ids(t); to_fiber(t); progressed = true; }
    }
    // release barriers whose participants (all threads that have not returned) have all arrived
    bool all_block = true; int n_wait = 0;
    for (int t = 0; t < n; ++t) { if (fibers[t].state == DONE) continue; alive = true; if (fibers[t].state != AT_BLOCK) all_block = false; else ++n_wait; }
    if (!alive) break;
    if (all_block && n_wait) { for (int t = 0; t < n; ++t) if (fibers[t].state == AT_BLOCK) fibers[t].state = RUN; continue; }
    bool released = false;
    for (int w = 0; w * 32 < n; ++w) {
      bool all = true; int cnt = 0;
      for (int t = 32 * w; t < std::min(n, 32 * w + 32); ++t) { if (fibers[t].state == DONE) continue; if (fibers[t].state != AT_WARP) all = false; else ++cnt; }
      if (all && cnt) { for (int t = 32 * w; t < std::min(n, 32 * w + 32); ++t) if (fibers[t].state == AT_WARP) fibers[t].state = RUN; released = true; }
    }
    if (!released && !progressed) { std::fprintf(stderr, "hostemu: barrier deadlock (threads wait at different barriers)\n"); std::abort(); }
  }
  cur = -1;
}
template <class F> inline void launch(dim3 g, dim3 b, size_t smem, F&& f) {
  const std::function<void()> fn(f); body = &fn;
  gridDim = g; blockDim = b; n_threads = (int)(b.x * b.y * b.z);
  if (dyn.size() < smem + 64) dyn.resize(smem + 64);
  for (unsigned z = 0; z < g.z; ++z) for (unsigned y = 0; y < g.y; ++y) for (unsigned x = 0; x < g.x; ++x) { blockIdx.x = x; blockIdx.y = y; blockIdx.z = z; run_block(); }
  body = nullptr;
}
}  // namespace hostemu
template <class K, class... A> inline void hostemu_launch(K k, dim3 g, dim3 b, size_t smem, A... a) { hostemu::launch(g, b, smem, [=]() { k(a...); }); }

inline void __syncthreads() { hostemu::yield(hostemu::AT_BLOCK); }
inline void __syncwarp(unsigned = 0xffffffffu) { hostemu::yield(hostemu::AT_WARP); }
static int block_vote[2048];
inline int __syncthreads_count(int p) {
  block_vote[hostemu::cur] = p ? 1 : 0;
  hostemu::yield(hostemu::AT_BLOCK);
  int r = 0; for (int i = 0; i < hostemu::n_threads; ++i) if (hostemu::fibers[i].state != hostemu::DONE) r += block_vote[i];
  hostemu::yield(hostemu::AT_BLOCK);
  return r;
}
template <class T> inline T __shfl_down_sync(unsigned, T v, unsigned delta, int = 32) {
  static_assert(sizeof(T) <= 8, "shuffle of > 8 bytes");
  const int w = hostemu::cur / 32, l = hostemu::cur % 32;
  long long raw = 0; std::memcpy(&raw, &v, sizeof(T)); hostemu::warp_slot[w][l] = raw;
  hostemu::yield(hostemu::AT_WARP);
  const int src = l + (int)delta < 32 && 32 * w + l + (int)delta < hostemu::n_threads ? l + (int)delta : l;
  raw = hostemu::warp_slot[w][src]; T r; std::memcpy(&r, &raw, sizeof(T));
  hostemu::yield(hostemu::AT_WARP);
  return r;
}
template <class T> inline T __shfl_up_sync(unsigned, T v, unsigned delta, int = 32) {
  static_assert(sizeof(T) <= 8, "shuffle of > 8 bytes");
  const int w = hostemu::cur / 32, l = hostemu::cur % 32;
  long long raw = 0; std::memcpy(&raw, &v, sizeof(T)); hostemu::warp_slot[w][l] = raw;
  hostemu::yield(hostemu::AT_WARP);
  const int src = l - (int)delta >= 0 ? l - (int)delta : l;
  raw = hostemu::warp_slot[w][src]; T r; std::memcpy(&r, &raw, sizeof(T));
  hostemu::yield(hostemu::AT_WARP);
  return r;
}
inline int __any_sync(unsigned, int p) {
  const int w = hostemu::cur / 32, l = hostemu::cur % 32;
  hostemu::vote_slot[w][l] = p ? 1 : 0;
  hostemu::yield(hostemu::AT_WARP);
  int r = 0; for (int i = 0; i < 32; ++i) if (32 * w + i < hostemu::n_threads && hostemu::fibers[32 * w + i].state != hostemu::DONE) r |= hostemu::vote_slot[w][i];
  hostemu::yield(hostemu::AT_WARP);
  return r;
}
inline unsigned __ballot_sync(unsigned, int p) {
  const int w = hostemu::cur / 32, l = hostemu::cur % 32;
  hostemu::vote_slot[w][l] = p ? 1 : 0;
  hostemu::yield(hostemu::AT_WARP);
  unsigned r = 0; for (int i = 0; i < 32; ++i) if (32 * w + i < hostemu::n_threads && hostemu::fibers[32 * w + i].state != hostemu::DONE && hostemu::vote_slot[w][i]) r |= 1u << i;
  hostemu::yield(hostemu::AT_WARP);
  return r;
}
// whole-warp integer reductions (redux.sync): min / max over the lanes that have not returned
static unsigned reduce_slot[64][32];
template <class Op> inline unsigned hostemu_reduce(unsigned v, Op op) {
  const int w = hostemu::cur / 32, l = hostemu::cur % 32;
  reduce_slot[w][l] = v;
  hostemu::yield(hostemu::AT_WARP);
  bool first = true; unsigned r = 0;
  for (int i = 0; i < 32; ++i)
    if (32 * w + i < hostemu::n_threads && hostemu::fibers[32 * w + i].state != hostemu::DONE) { r = first ? reduce_slot[w][i] : op(r, reduce_slot[w][i]); first = false; }
  hostemu::yield(hostemu::AT_WARP);
  return r;
}
inline unsigned __reduce_min_sync(unsigned, unsigned v) { return hostemu_reduce(v, [](unsigned a, unsigned b) { return a < b ? a : b; }); }
inline unsigned __reduce_max_sync(unsigned, unsigned v) { return hostemu_reduce(v, [](unsigned a, unsigned b) { return a > b ? a : b; }); }
// sub-warp collectives (mask names the participants): modelled on the whole-warp barrier, so every lane of the warp that is
// still alive must reach SOME warp-level barrier while the named lanes exchange -- true for the engine's uses, where the
// lanes outside the mask wait at the __syncwarp that follows.
static long long match_slot[64][32]; static int match_in[64][32];
template <class T> inline unsigned __match_any_sync(unsigned mask, T v) {
  const int w = hostemu::cur / 32, l = hostemu::cur % 32;
  long long raw = 0; std::memcpy(&raw, &v, sizeof(T)); match_slot[w][l] = raw; match_in[w][l] = 1;
  hostemu::yield(hostemu::AT_WARP);
  unsigned r = 0; for (int i = 0; i < 32; ++i) if ((mask >> i & 1u) && match_in[w][i] && match_slot[w][i] == raw) r |= 1u << i;
  hostemu::yield(hostemu::AT_WARP);
  match_in[w][l] = 0;
  return r;
}
template <class T> inline T __shfl_sync(unsigned, T v, int src, int = 32) {
  static_assert(sizeof(T) <= 8, "shuffle of > 8 bytes");
  const int w = hostemu::cur / 32, l = hostemu::cur % 32;
  long long raw = 0; std::memcpy(&raw, &v, sizeof(T)); hostemu::warp_slot[w][l] = raw;
  hostemu::yield(hostemu::AT_WARP);
  raw = hostemu::warp_slot[w][src & 31]; T r; std::memcpy(&r, &raw, sizeof(T));
  hostemu::yield(hostemu::AT_WARP);
  return r;
}
template <class T> inline T __shfl_xor_sync(unsigned m, T v, int lane_mask, int = 32) { return __shfl_sync(m, v, (hostemu::cur % 32) ^ lane_mask); }
inline int __clzll(long long x) { return x ? __builtin_clzll((unsigned long long)x) : 64; }
inline int __popc(unsigned x) { return __builtin_popcount(x); }
inline int __ffs(unsigned x) { return __builtin_ffs((int)x); }
inline uint2 make_uint2(unsigned x, unsigned y) { uint2 r; r.x = x; r.y = y; return r; }
template <class T> inline T atomicAdd(T* p, T v) { const T o = *p; *p = o + v; return o; }
template <class T> inline T atomicExch(T* p, T v) { const T o = *p; *p = v; return o; }
template <class T> inline T atomicMin(T* p, T v) { const T o = *p; if (v < o) *p = v; return o; }
template <class T> inline T atomicMax(T* p, T v) { const T o = *p; if (v > o) *p = v; return o; }
inline void __threadfence() {} inline void __threadfence_system() {} inline void __threadfence_block() {}
inline long long clock64() { return std::chrono::steady_clock::now().time_since_epoch().count(); }

// ---- device intrinsics ----------------------------------------------------------------------------------------------
template <class T> inline T __ldg(const T* p) { return *p; }
inline int __float_as_int(float f) { int i; std::memcpy(&i, &f, 4); return i; }
inline float __int_as_float(int i) { float f; std::memcpy(&f, &i, 4); return f; }
inline unsigned __float_as_uint(float f) { unsigned i; std::memcpy(&i, &f, 4); return i; }
inline float __uint_as_float(unsigned i) { float f; std::memcpy(&f, &i, 4); return f; }
inline long long __double_as_longlong(double d) { long long l; std::memcpy(&l, &d, 8); return l; }
inline double __longlong_as_double(long long l) { double d; std::memcpy(&d, &l, 8); return d; }
inline double __dmul_rn(double a, double b) { return a * b; }   // compile with -ffp-contract=off
inline double __dadd_rn(double a, double b) { return a + b; }
inline double __dsub_rn(double a, double b) { return a - b; }
inline double __ddiv_rn(double a, double b) { return a / b; }
inline double __dsqrt_rn(double a) { return std::sqrt(a); }
inline float __double2float_rn(double a) { return (float)a; }
inline float hs_up(double v) { float f = (float)v; if ((double)f < v) f = std::nextafterf(f, INFINITY); return f; }
inline float __double2float_ru(double a) { return hs_up(a); }
inline float __fsqrt_ru(float a) { return std::nextafterf(hs_up(std::sqrt((double)a)), INFINITY); }
inline float __fadd_ru(float a, float b) { return hs_up((double)a + (double)b); }
inline float4 make_float4(float x, float y, float z, float w) { float4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }
inline int2 make_int2(int x, int y) { int2 r; r.x = x; r.y = y; return r; }
inline float __fmul_ru(float a, float b) { return hs_up((double)a * (double)b); }
inline float hs_down(double v) { float f = (float)v; if ((double)f > v) f = std::nextafterf(f, -INFINITY); return f; }
inline float __fmul_rd(float a, float b) { return hs_down((double)a * (double)b); }
inline float __fsub_rd(float a, float b) { return hs_down((double)a - (double)b); }
inline float __fmaf_ru(float a, float b, float c) { return std::nextafterf(hs_up((double)a * (double)b + (double)c), INFINITY); }
inline double rsqrt(double a) { return 1.0 / std::sqrt(a); }

// ---- runtime API (device memory = host memory; streams and events do nothing) -----------------------------------------
typedef int cudaError_t; typedef void* cudaStream_t; typedef void* cudaEvent_t;
enum { cudaSuccess = 0, cudaErrorNotReady = 600, cudaErrorNotSupported = 801 };
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
enum { cudaStreamNonBlocking = 1, cudaHostAllocMapped = 2, cudaHostAllocPortable = 1, cudaIpcMemLazyEnablePeerAccess = 1, cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
struct cudaIpcMemHandle_t { char reserved[64]; };
inline cudaError_t cudaMalloc(void** p, size_t n) { return posix_memalign(p, 256, n ? n : 1) ? 2 : cudaSuccess; }
template <class T> inline cudaError_t cudaMalloc(T** p, size_t n) { return cudaMalloc((void**)p, n); }
inline cudaError_t cudaFree(void* p) { std::free(p); return cudaSuccess; }
inline cudaError_t cudaMallocHost(void** p, size_t n) { return cudaMalloc(p, n); }
template <class T> inline cudaError_t cudaMallocHost(T** p, size_t n) { return cudaMalloc((void**)p, n); }
inline cudaError_t cudaHostAlloc(void** p, size_t n, unsigned) { return cudaMalloc(p, n); }
template <class T> inline cudaError_t cudaHostAlloc(T** p, size_t n, unsigned f) { return cudaMalloc((void**)p, n); }
inline cudaError_t cudaFreeHost(void* p) { std::free(p); return cudaSuccess; }
template <class T> inline cudaError_t cudaHostGetDevicePointer(T** d, void* h, unsigned) { *d = (T*)h; return cudaSuccess; }
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { std::memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { std::memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemset(void* d, int v, size_t n) { std::memset(d, v, n); return cudaSuccess; }
inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = nullptr) { std::memset(d, v, n); return cudaSuccess; }
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = (void*)0x1; return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamQuery(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = (void*)0x1; return cudaSuccess; }
inline cudaError_t cudaEventDestroy(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0.f; return cudaSuccess; }
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline const char* cudaGetErrorString(cudaError_t) { return "hostemu"; }
template <class K> inline cudaError_t cudaFuncSetAttribute(K, int, int) { return cudaSuccess; }
inline cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t*, void*) { return cudaErrorNotSupported; }
inline cudaError_t cudaIpcOpenMemHandle(void**, cudaIpcMemHandle_t, unsigned) { return cudaErrorNotSupported; }
inline cudaError_t cudaIpcCloseMemHandle(void*) { return cudaSuccess; }
// every allocation is host memory here, and all of it stands for device memory of device 0: the `_device` entry points accept
// numpy buffers on this model (a null pointer is unregistered, as on the device)
enum cudaMemoryType { cudaMemoryTypeUnregistered = 0, cudaMemoryTypeHost = 1, cudaMemoryTypeDevice = 2, cudaMemoryTypeManaged = 3 };
struct cudaPointerAttributes { cudaMemoryType type; int device; void* devicePointer; void* hostPointer; };
inline cudaError_t cudaPointerGetAttributes(cudaPointerAttributes* a, const void* p) {
  a->type = p ? cudaMemoryTypeDevice : cudaMemoryTypeUnregistered; a->device = 0;
  a->devicePointer = const_cast<void*>(p); a->hostPointer = nullptr;
  return cudaSuccess;
}
