// cuda_emu.h -- a small CUDA-on-CPU emulation layer (TEST INFRASTRUCTURE, never shipped): lets the library's .cu
// sources be compiled by g++ and its kernels be EXECUTED on the host, so that kernel logic can be checked against the
// oracle in a container without a GPU (tools/emu/build_emu.py, tests/test_emulated_kernels.py).
//
// Model: a launch runs its blocks one after the other; the threads of a block are cooperative fibers (ucontext) of
// one OS thread, switched only at synchronisation points:
//   __syncthreads / __syncwarp / __shfl*_sync / __ballot_sync / __any_sync / __all_sync  (block / warp barriers)
//   mbarrier waits (the TMA ring of the tile kernels: cp.async.bulk is a memcpy that completes at issue time)
// Atomics are plain read-modify-writes (single OS thread).  `__shared__` variables are function-local statics (one
// block runs at a time); dynamic shared memory is one global buffer.  A pass of the scheduler in which no fiber makes
// progress is reported as a deadlock.  This checks LOGIC (indexing, protocols, collectives under divergence), not
// timing and not real concurrency.
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <cmath>
#include <functional>

// ---------------------------------------------------------------------------------------------- qualifiers
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __shared__ static
#define __align__(n) alignas(n)
#define __constant__ static

// ---------------------------------------------------------------------------------------------- vector types
struct dim3 {
  unsigned x, y, z;
  dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {}
};
struct uint3 { unsigned x, y, z; };
struct int2 { int x, y; };
struct alignas(16) int4 { int x, y, z, w; };
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(16) double2 { double x, y; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
static inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{x, y, z, w}; }
// IEEE binary16 on g++'s _Float16: float -> half rounds to nearest even, subnormals included, as __float2half_rn does.  Only
// the conversions exist (no arithmetic operators), so emulated kernels cannot compute in half by accident.
struct __half {
  _Float16 v;
};
static inline __half __float2half_rn(float f) { return __half{(_Float16)f}; }
static inline float __half2float(__half h) { return (float)h.v; }
static inline unsigned short __half_as_ushort(__half h) { unsigned short b; memcpy(&b, &h, 2); return b; }
static inline __half __ushort_as_half(unsigned short b) { __half h; memcpy(&h, &b, 2); return h; }
static inline int2 make_int2(int x, int y) { return int2{x, y}; }
static inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
static inline double2 make_double2(double x, double y) { return double2{x, y}; }

// ---------------------------------------------------------------------------------------------- runtime (fake)
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorNotReady = 600, cudaErrorMemoryAllocation = 2 };
typedef struct b200emu_stream* cudaStream_t;
typedef struct b200emu_event* cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyDefault };
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount = 16, cudaDevAttrComputeCapabilityMajor = 75 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
enum { cudaEventDisableTiming = 2, cudaStreamNonBlocking = 1 };

namespace b200emu {
void* device_alloc(size_t bytes);
void device_free(void* p);
}  // namespace b200emu

static inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "emulated CUDA error"; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaDeviceGetAttribute(int* v, int attr, int) {
  *v = attr == cudaDevAttrMultiProcessorCount ? 4 : (attr == cudaDevAttrComputeCapabilityMajor ? 9 : 0);
  return cudaSuccess;
}
static inline cudaError_t cudaMalloc(void** p, size_t n) { *p = b200emu::device_alloc(n); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
template <class T> static inline cudaError_t cudaMalloc(T** p, size_t n) { return cudaMalloc((void**)p, n); }
static inline cudaError_t cudaMallocAsync(void** p, size_t n, cudaStream_t) { return cudaMalloc(p, n); }
template <class T> static inline cudaError_t cudaMallocAsync(T** p, size_t n, cudaStream_t) { return cudaMalloc((void**)p, n); }
static inline cudaError_t cudaMallocHost(void** p, size_t n) { return cudaMalloc(p, n); }
static inline cudaError_t cudaFree(void* p) { b200emu::device_free(p); return cudaSuccess; }
static inline cudaError_t cudaFreeAsync(void* p, cudaStream_t) { return cudaFree(p); }
static inline cudaError_t cudaFreeHost(void* p) { return cudaFree(p); }
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { if (n) memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind k, cudaStream_t = nullptr) { return cudaMemcpy(d, s, n, k); }
static inline cudaError_t cudaMemset(void* d, int v, size_t n) { if (n) memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = nullptr) { return cudaMemset(d, v, n); }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = nullptr; return cudaSuccess; }
static inline cudaError_t cudaStreamCreate(cudaStream_t* s) { *s = nullptr; return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = (cudaEvent_t)(uintptr_t)1; return cudaSuccess; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { return cudaEventCreate(e); }
static inline cudaError_t cudaEventDestroy(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return cudaSuccess; }
static inline cudaError_t cudaEventQuery(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 1.0f; return cudaSuccess; }
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, int, int) { return cudaSuccess; }
template <class F> static inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* n, F, int, size_t) { *n = 2; return cudaSuccess; }

// ---------------------------------------------------------------------------------------------- execution model
namespace b200emu {

struct Fiber;
struct ThreadCtx {
  uint3 tid, bid;
  dim3 bdim, gdim;
  int linear;  // thread index within the block
};
ThreadCtx* cur();                       // context of the running fiber
void* dyn_smem();                       // dynamic shared memory of the running block
void launch(dim3 grid, dim3 block, size_t smem, const std::function<void()>& body);
void block_barrier();                   // __syncthreads
void warp_barrier(unsigned mask);       // __syncwarp and the two halves of every warp collective
unsigned long long* warp_slots();       // 32 exchange slots of the running fiber's warp
unsigned warp_alive();                  // lanes of the running fiber's warp that exist and have not exited
void yield_blocked();                   // give up the processor while waiting on something (mbarrier)
void note_progress();

// mbarrier emulation (keyed by the shared-memory address of the barrier object; reset at block start)
void mbar_init(void* bar, unsigned count);
void mbar_arrive(void* bar);
void mbar_arrive_expect_tx(void* bar, unsigned bytes);
void mbar_complete_tx(void* bar, unsigned bytes);
bool mbar_test_wait(void* bar, unsigned parity);
void bulk_copy_async(void* smem_dst, const void* gsrc, unsigned bytes, void* bar);

}  // namespace b200emu

#ifndef B200EMU_HOST_PROGRAM  // host programs (tools/emu/cuda_runtime.h) only need the runtime API, not the built-ins
#define threadIdx (b200emu::cur()->tid)
#define blockIdx (b200emu::cur()->bid)
#define blockDim (b200emu::cur()->bdim)
#define gridDim (b200emu::cur()->gdim)
#endif

#define B200_EMU_LAUNCH(KERN, GRID, BLOCK, SMEM, ...) \
  b200emu::launch(dim3(GRID), dim3(BLOCK), (size_t)(SMEM), [&]() { KERN(__VA_ARGS__); })

// ---------------------------------------------------------------------------------------------- device intrinsics
static inline void __syncthreads() { b200emu::block_barrier(); }
template <class T> static inline T __ldcg(const T* p) { return *p; }
static inline void __syncwarp(unsigned mask = 0xffffffffu) { b200emu::warp_barrier(mask); }
static inline void __threadfence() {}  // one fiber runs at a time: memory is always coherent here
static inline void __threadfence_block() {}
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline int __popcll(unsigned long long v) { return __builtin_popcountll(v); }
static inline int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline double __dmul_rn(double a, double b) { return a * b; }  // built with -ffp-contract=off: no fusion
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline double __dsub_rn(double a, double b) { return a - b; }
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
static inline int __double2loint(double v) { unsigned long long b; memcpy(&b, &v, 8); return (int)(unsigned)(b & 0xffffffffull); }
static inline int __double2hiint(double v) { unsigned long long b; memcpy(&b, &v, 8); return (int)(unsigned)(b >> 32); }
static inline double __hiloint2double(int hi, int lo) {
  const unsigned long long b = ((unsigned long long)(unsigned)hi << 32) | (unsigned long long)(unsigned)lo;
  double v; memcpy(&v, &b, 8); return v;
}
static inline int __float_as_int(float v) { int b; memcpy(&b, &v, 4); return b; }
static inline float __int_as_float(int b) { float v; memcpy(&v, &b, 4); return v; }
static inline size_t __cvta_generic_to_shared(const void* p) { return (size_t)(uintptr_t)p; }

static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
static inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
static inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }
static inline long long min(long long a, long long b) { return a < b ? a : b; }
static inline long long max(long long a, long long b) { return a > b ? a : b; }
static inline long min(long a, long b) { return a < b ? a : b; }
static inline long max(long a, long b) { return a > b ? a : b; }
static inline long long min(long long a, int b) { return a < b ? a : b; }

namespace b200emu {
template <class T> static inline unsigned long long to_bits(T v) {
  static_assert(sizeof(T) <= 8, "warp collectives move at most 8 bytes");
  unsigned long long b = 0;
  memcpy(&b, &v, sizeof(T));
  return b;
}
template <class T> static inline T from_bits(unsigned long long b) {
  T v;
  memcpy(&v, &b, sizeof(T));
  return v;
}
static inline int lane_id() { return cur()->linear & 31; }
// every participating lane publishes `mine`, all see the published values between the two barriers
template <class T, class F> static inline auto collective(unsigned mask, T mine, F&& read) {
  unsigned long long* slot = warp_slots();
  slot[lane_id()] = to_bits(mine);
  warp_barrier(mask);
  auto r = read(slot);
  warp_barrier(mask);
  return r;
}
}  // namespace b200emu

template <class T> static inline T __shfl_sync(unsigned mask, T v, int src, int width = 32) {
  return b200emu::collective(mask, v, [&](unsigned long long* s) {
    const int lane = b200emu::lane_id();
    const int base = lane & ~(width - 1);
    const int from = base + (src & (width - 1));
    return ((mask >> from) & 1u) && ((b200emu::warp_alive() >> from) & 1u) ? b200emu::from_bits<T>(s[from]) : v;
  });
}
template <class T> static inline T __shfl_up_sync(unsigned mask, T v, unsigned delta, int width = 32) {
  return b200emu::collective(mask, v, [&](unsigned long long* s) {
    const int lane = b200emu::lane_id();
    const int base = lane & ~(width - 1);
    const int from = lane - (int)delta;
    return (from >= base && ((b200emu::warp_alive() >> from) & 1u)) ? b200emu::from_bits<T>(s[from]) : v;
  });
}
template <class T> static inline T __shfl_down_sync(unsigned mask, T v, unsigned delta, int width = 32) {
  return b200emu::collective(mask, v, [&](unsigned long long* s) {
    const int lane = b200emu::lane_id();
    const int base = lane & ~(width - 1);
    const int from = lane + (int)delta;
    return (from < base + width && ((b200emu::warp_alive() >> from) & 1u)) ? b200emu::from_bits<T>(s[from]) : v;
  });
}
template <class T> static inline T __shfl_xor_sync(unsigned mask, T v, int lanemask, int width = 32) {
  return b200emu::collective(mask, v, [&](unsigned long long* s) {
    const int lane = b200emu::lane_id();
    const int from = lane ^ lanemask;
    return ((lane & ~(width - 1)) == (from & ~(width - 1)) && ((b200emu::warp_alive() >> from) & 1u)) ? b200emu::from_bits<T>(s[from]) : v;
  });
}
static inline unsigned __ballot_sync(unsigned mask, int pred) {
  return b200emu::collective(mask, (int)(pred != 0), [&](unsigned long long* s) {
    unsigned r = 0;
    const unsigned part = mask & b200emu::warp_alive();
    for (int l = 0; l < 32; ++l)
      if (((part >> l) & 1u) && s[l]) r |= 1u << l;
    return r;
  });
}
static inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
static inline int __all_sync(unsigned mask, int pred) { return __ballot_sync(mask, !pred) == 0; }
static inline int __syncthreads_or(int pred) {
  static int acc;
  __syncthreads();
  if (b200emu::cur()->linear == 0) acc = 0;
  __syncthreads();
  if (pred) acc = 1;
  __syncthreads();
  return acc;
}

template <class T> static inline T atomicAdd(T* p, T v) { T o = *p; *p = o + v; b200emu::note_progress(); return o; }
static inline int atomicAdd(int* p, int v) { int o = *p; *p = o + v; b200emu::note_progress(); return o; }
static inline int atomicMin(int* p, int v) { int o = *p; if (v < o) *p = v; b200emu::note_progress(); return o; }
static inline int __ffsll(long long v) { return __builtin_ffsll(v); }
static inline int __ffs(int v) { return __builtin_ffs(v); }
static inline int atomicMax(int* p, int v) { int o = *p; if (v > o) *p = v; b200emu::note_progress(); return o; }
static inline unsigned atomicOr(unsigned* p, unsigned v) { unsigned o = *p; *p = o | v; b200emu::note_progress(); return o; }
static inline int atomicCAS(int* p, int cmp, int v) { int o = *p; if (o == cmp) *p = v; b200emu::note_progress(); return o; }
static inline unsigned long long atomicCAS(unsigned long long* p, unsigned long long cmp, unsigned long long v) {
  unsigned long long o = *p; if (o == cmp) *p = v; b200emu::note_progress(); return o;
}
static inline int atomicExch(int* p, int v) { int o = *p; *p = v; b200emu::note_progress(); return o; }
