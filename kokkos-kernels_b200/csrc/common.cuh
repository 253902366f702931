// common.cuh -- shared helpers of libb200sparse (sm_90a only).
#pragma once
#ifdef B200SP_EMU
#include "cuda_emu.h"  // tools/emu: CUDA-on-CPU emulation of the kernels (test infrastructure)
#else
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#endif
#include <stdint.h>
#include <stdio.h>
#include <assert.h>
#include <algorithm>
#include <atomic>
#include "../../include/b200sparse.h"

namespace b200sp {

// ---- error plumbing -------------------------------------------------------
void set_error(const char* fmt, ...);
extern std::atomic<long long> g_launches;

#define B200SP_CUDA_TRY(expr)                                                        \
  do {                                                                               \
    cudaError_t _e = (expr);                                                         \
    if (_e != cudaSuccess) {                                                         \
      ::b200sp::set_error("%s failed at %s:%d: %s", #expr, __FILE__, __LINE__,       \
                          cudaGetErrorString(_e));                                   \
      return B200SP_ERR_CUDA;                                                        \
    }                                                                                \
  } while (0)

#define B200SP_LAUNCH_CHECK()                                                        \
  do {                                                                               \
    ::b200sp::g_launches.fetch_add(1, std::memory_order_relaxed);                    \
    cudaError_t _e = cudaGetLastError();                                             \
    if (_e != cudaSuccess) {                                                         \
      ::b200sp::set_error("kernel launch failed at %s:%d: %s", __FILE__, __LINE__,   \
                          cudaGetErrorString(_e));                                   \
      return B200SP_ERR_CUDA;                                                        \
    }                                                                                \
  } while (0)

#define B200SP_REQUIRE(cond, ...)                                                    \
  do {                                                                               \
    if (!(cond)) {                                                                   \
      ::b200sp::set_error(__VA_ARGS__);                                              \
      return B200SP_ERR_INVALID_ARGUMENT;                                            \
    }                                                                                \
  } while (0)

int sm_count();  // SMs of the current device (cached per device)

// CTAs of `per_block` threads for a grid-stride loop over `work` items: one item per thread, at most per_sm CTAs per SM
inline int grid_for(int64_t work, int per_block = 256, int per_sm = 8) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((work + per_block - 1) / per_block, (int64_t)sm_count() * per_sm));
}
// Scratch is allocated with cudaMallocAsync.  The default pool hands unused memory back to the driver at every synchronisation
// point (release threshold 0), and the symbolic phases synchronise by contract (they return counts to the host): each call would
// then map its scratch again, which can cost more than its kernels (spadd_symbolic most of all).  Keeps the pool's memory (once per device); called by every scratch allocation scope (DevTmp) and by the plans that own
// stream-ordered memory.
void keep_async_pool_memory();

// Launch setup of a kernel with more than 48 KB of dynamic shared memory: the opt-in attribute and the occupancy are
// per DEVICE, so they are cached per (kernel instantiation, device) -- one process may drive several GPUs.
struct KernelSetup {
  std::atomic<int> occ[32];
  KernelSetup() {
    for (auto& o : occ) o.store(0);
  }
};
template <class K>
static inline int kernel_setup(KernelSetup& ks, K kern, int threads, size_t smem, int* occ_out) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) dev = 0;
  const bool cacheable = dev >= 0 && dev < 32;
  int occ = cacheable ? ks.occ[dev].load(std::memory_order_acquire) : 0;
  if (occ == 0) {
    B200SP_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    B200SP_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, smem));
    if (occ < 1) occ = 1;
    if (cacheable) ks.occ[dev].store(occ, std::memory_order_release);
  }
  *occ_out = occ;
  return B200SP_OK;
}

// stream-ordered temporaries of one host call
struct DevTmp {  // frees stream-ordered on scope exit
  cudaStream_t st;
  void* ptrs[32];
  int n = 0;
  explicit DevTmp(cudaStream_t s) : st(s) { keep_async_pool_memory(); }
  ~DevTmp() {
    for (int i = 0; i < n; ++i) cudaFreeAsync(ptrs[i], st);
  }
  template <typename T>
  cudaError_t alloc(T** out, size_t count) {
    void* q = nullptr;
    cudaError_t e = cudaMallocAsync(&q, sizeof(T) * (count > 0 ? count : 1), st);
    if (e == cudaSuccess) ptrs[n++] = q;
    *out = (T*)q;
    return e;
  }
};

// stream-ordered device memory a plan keeps between calls: one owner, freed by release() on the caller's stream.  The
// destructor frees nothing (a plan is destroyed with the stream its memory goes back on).  Buffers whose scalar type is
// chosen per call are DevArray<char>, sized in bytes.  A move leaves the source empty; the target must be empty (asserted:
// a block it held would be lost).
template <typename T>
struct DevArray {
  T* ptr = nullptr;
  size_t count = 0;
  DevArray() = default;
  DevArray(const DevArray&) = delete;
  DevArray& operator=(const DevArray&) = delete;
  DevArray(DevArray&& o) noexcept : ptr(o.ptr), count(o.count) { o.ptr = nullptr, o.count = 0; }
  DevArray& operator=(DevArray&& o) noexcept {
    assert(ptr == nullptr);
    ptr = o.ptr, count = o.count;
    o.ptr = nullptr, o.count = 0;
    return *this;
  }
  operator T*() const { return ptr; }
  template <typename U>
  U* as() const {
    return reinterpret_cast<U*>(ptr);
  }
  void release(cudaStream_t st) {
    if (ptr) cudaFreeAsync(ptr, st);
    ptr = nullptr;
    count = 0;
  }
  // exactly n elements, in place of what the array held
  cudaError_t alloc(size_t n, cudaStream_t st) {
    release(st);
    const cudaError_t e = cudaMallocAsync((void**)&ptr, sizeof(T) * n, st);
    if (e == cudaSuccess) count = n;
    else ptr = nullptr;
    return e;
  }
  // at least n elements: the block is kept when it is large enough
  cudaError_t grow(size_t n, cudaStream_t st) { return n <= count ? cudaSuccess : alloc(n, st); }
};

// what a plan's cached product was built from, compared whole; the default key matches no call (row_ptr is never null there)
struct PlanKey {
  const void* row_ptr = nullptr;
  const void* col_idx = nullptr;
  int64_t m = -1, n = -1, nnz = -1, a = -1, b = -1;  // a, b: the product's own parameters (cfg, stage, row limit, ...)
  bool operator==(const PlanKey& o) const {
    return row_ptr == o.row_ptr && col_idx == o.col_idx && m == o.m && n == o.n && nnz == o.nnz && a == o.a && b == o.b;
  }
  bool operator!=(const PlanKey& o) const { return !(*this == o); }
};

#ifdef B200SP_EMU
// ---- emulation of the PTX wrappers (tools/emu/cuda_emu.h): same names, same protocol -------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)(uintptr_t)p; }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) { b200emu::mbar_init(bar, count); }
__device__ __forceinline__ void fence_mbar_init() {}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) { b200emu::mbar_arrive(bar); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) { b200emu::mbar_arrive_expect_tx(bar, bytes); }
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) { return b200emu::mbar_test_wait(bar, parity); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// asynchronous like the real thing: the destination is poisoned at issue time and the bytes land only when a thread
// waits on the barrier (tools/emu/emu_runtime.cpp); alignment rules of cp.async.bulk are checked
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar, uint64_t) {
  b200emu::bulk_copy_async(smem_dst, gsrc, bytes, bar);
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() { return 0; }
__device__ __forceinline__ uint64_t l2_policy_evict_last() { return 0; }
// per-thread asynchronous copies (cp.async): the emulation copies at issue time
template <int BYTES>
__device__ __forceinline__ void cp_async(void* smem_dst, const void* gsrc) { memcpy(smem_dst, gsrc, BYTES); }
__device__ __forceinline__ void cp_async_wait_all() {}
template <typename T>
__device__ __forceinline__ T ldg(const T* p) {
  return *p;
}
__device__ __forceinline__ int ld_stream(const int* p) { return *p; }
__device__ __forceinline__ double ld_stream(const double* p) { return *p; }
__device__ __forceinline__ float ld_stream(const float* p) { return *p; }
__device__ __forceinline__ int ld_once(const int* p, uint64_t) { return *p; }
__device__ __forceinline__ double ld_once(const double* p, uint64_t) { return *p; }
__device__ __forceinline__ float ld_once(const float* p, uint64_t) { return *p; }
__device__ __forceinline__ int4 ld_once(const int4* p, uint64_t) { return *p; }
__device__ __forceinline__ void st_once(int* p, int v, uint64_t) { *p = v; }
__device__ __forceinline__ void st_once(float* p, float v, uint64_t) { *p = v; }
__device__ __forceinline__ void st_once(double* p, double v, uint64_t) { *p = v; }
__device__ __forceinline__ void st_once(float4* p, const float4& v, uint64_t) { *p = v; }
__device__ __forceinline__ void st_once(double2* p, const double2& v, uint64_t) { *p = v; }
__device__ __forceinline__ __half ld_once(const __half* p, uint64_t) { return *p; }
__device__ __forceinline__ void st_once(__half* p, __half v, uint64_t) { *p = v; }
__device__ __forceinline__ void st_once(uint4* p, const uint4& v, uint64_t) { *p = v; }
#else
// ---- PTX wrappers: mbarrier + 1-D bulk (TMA) copies ------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(20000u) /* suspend-time hint, ns: sleep instead of spinning */
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// global -> shared bulk async copy (TMA engine, SASS UBLKCP); completes `bytes`
// on `bar`.  src/dst 16-byte aligned, bytes a multiple of 16.  `policy` is an
// L2 cache-hint descriptor (createpolicy).
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes,
                                         uint64_t* bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint "
      "[%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}
// per-thread asynchronous copy global -> shared of 4 / 8 / 16 bytes (SASS LDGSTS): no destination register is held while the
// load is in flight; completion by cp_async_wait_all() in the issuing thread, visibility to others by a barrier after it
template <int BYTES>
__device__ __forceinline__ void cp_async(void* smem_dst, const void* gsrc) {
  static_assert(BYTES == 4 || BYTES == 8 || BYTES == 16, "cp.async moves 4, 8 or 16 bytes");
  asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "n"(BYTES) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}

// read-only gathers (LDG.CONSTANT, L1-allocating)
template <typename T>
__device__ __forceinline__ T ldg(const T* p) {
  return __ldg(p);
}
// streaming loads that should not displace x in L1
__device__ __forceinline__ int ld_stream(const int* p) {
  int v;
  asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ double ld_stream(const double* p) {
  double v;
  asm volatile("ld.global.nc.L1::no_allocate.f64 %0, [%1];" : "=d"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ float ld_stream(const float* p) {
  float v;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}

// data that is touched ONCE per kernel (matrix streams, work-item lists, results): no L1 allocation and an L2 evict-first
// policy (createpolicy, l2_policy_evict_first()), so that it does not push the gathered operand (x / X rows) out of L2
__device__ __forceinline__ int ld_once(const int* p, uint64_t pol) {
  int v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.s32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ float ld_once(const float* p, uint64_t pol) {
  float v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ double ld_once(const double* p, uint64_t pol) {
  double v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ int4 ld_once(const int4* p, uint64_t pol) {
  int4 v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.s32 {%0, %1, %2, %3}, [%4], %5;"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ void st_once(int* p, int v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.s32 [%0], %1, %2;" ::"l"(p), "r"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_once(float* p, float v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.f32 [%0], %1, %2;" ::"l"(p), "f"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_once(double* p, double v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.f64 [%0], %1, %2;" ::"l"(p), "d"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_once(float4* p, const float4& v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol)
               : "memory");
}
__device__ __forceinline__ void st_once(double2* p, const double2& v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v2.f64 [%0], {%1, %2}, %3;" ::"l"(p), "d"(v.x), "d"(v.y), "l"(pol) : "memory");
}
// binary16: one value, or 8 packed in a uint4 (the 16-byte form of the half-precision rank-2 kernels)
__device__ __forceinline__ __half ld_once(const __half* p, uint64_t pol) {
  unsigned short v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.b16 %0, [%1], %2;" : "=h"(v) : "l"(p), "l"(pol));
  return __ushort_as_half(v);
}
__device__ __forceinline__ void st_once(__half* p, __half v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.b16 [%0], %1, %2;" ::"l"(p), "h"(__half_as_ushort(v)), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_once(uint4* p, const uint4& v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v4.b32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "l"(pol)
               : "memory");
}

#endif  // B200SP_EMU

template <typename T>
__device__ __forceinline__ T shfl_xor(T v, int mask) {
  return __shfl_xor_sync(0xffffffffu, v, mask);
}

}  // namespace b200sp
