// scan.cuh -- exclusive scan of per-row counts (int32) into CSR offsets, shared by spgemm.cu and
// crs_utils.cu (the analogue of kk_exclusive_parallel_prefix_sum,
// reference common/src/KokkosKernels_SimpleUtils.hpp:86-134).  Three kernels: block-local scan,
// scan of the block sums (+ total as int64, + maximum count), offset add.  out has m+1 entries;
// when the total exceeds INT32_MAX every offset is written as 0 and the caller reports the overflow.
#pragma once
#include <limits.h>
#include "common.cuh"

namespace b200sp {

// ---- exclusive scan of row counts -> row_ptr (int32) + total (int64) + max --
static constexpr int SCAN_ITEMS = 2048;  // per CTA (256 threads x 8)
static __global__ void __launch_bounds__(256) scan_local_kernel(int m, const int* __restrict__ cnt, int* __restrict__ out,
                                                         long long* __restrict__ block_sum, int* __restrict__ block_max) {
  __shared__ long long wsum[8];
  __shared__ int wmax[8];
  const int base = blockIdx.x * SCAN_ITEMS + threadIdx.x * 8;
  int v[8];
  long long s = 0;
  int mx = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    v[i] = (base + i < m) ? cnt[base + i] : 0;
    s += v[i];
    mx = max(mx, v[i]);
  }
  // warp inclusive scan of s
  long long inc = s;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    long long t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 31) wsum[w] = inc;
  if (lane == 0) wmax[w] = mx;
  __syncthreads();
  long long woff = 0;
  for (int i = 0; i < w; ++i) woff += wsum[i];
  long long run = woff + inc - s;  // exclusive prefix of this thread within the block
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (base + i < m) out[base + i] = (int)run;  // block-local; offset added later
    run += v[i];
  }
  if (threadIdx.x == 255) {
    long long tot = 0;
    int bm = 0;
    for (int i = 0; i < 8; ++i) {
      tot += wsum[i];
      bm = max(bm, wmax[i]);
    }
    block_sum[blockIdx.x] = tot;
    block_max[blockIdx.x] = bm;
  }
}
static __global__ void scan_blocks_kernel(int nblocks, long long* __restrict__ block_sum, const int* __restrict__ block_max,
                                   long long* __restrict__ total, int* __restrict__ maxv) {
  // single thread block; serial over chunks of 1024 (nblocks is m/2048: small)
  __shared__ long long carry;
  __shared__ long long ws[32];
  __shared__ int gm;
  if (threadIdx.x == 0) {
    carry = 0;
    gm = 0;
  }
  __syncthreads();
  for (int b0 = 0; b0 < nblocks; b0 += 1024) {
    const int i = b0 + threadIdx.x;
    const long long v = i < nblocks ? block_sum[i] : 0;
    if (i < nblocks) atomicMax(&gm, block_max[i]);
    long long inc = v;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      long long t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    if (lane == 31) ws[w] = inc;
    __syncthreads();
    long long woff = 0;
    for (int k = 0; k < w; ++k) woff += ws[k];
    const long long excl = carry + woff + inc - v;
    if (i < nblocks) block_sum[i] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) carry = excl + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    *total = carry;
    *maxv = gm;
  }
}
static __global__ void __launch_bounds__(256) scan_add_kernel(int m, int* __restrict__ out, const long long* __restrict__ block_off,
                                                       const long long* __restrict__ total) {
  const long long off = block_off[blockIdx.x];
  const int base = blockIdx.x * SCAN_ITEMS + threadIdx.x * 8;
  const bool ok = *total <= (long long)INT_MAX;
#pragma unroll
  for (int i = 0; i < 8; ++i)
    if (base + i < m) out[base + i] = ok ? (int)(out[base + i] + off) : 0;
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) out[m] = ok ? (int)*total : 0;
}

// counts[0..m) -> out[0..m] (exclusive offsets, out[m] = total); d_total / d_max receive the int64
// total and the largest count.  block_sum / block_max: scratch of scan_blocks(m) entries each.
static inline int scan_blocks(int m) { return (m + SCAN_ITEMS - 1) / SCAN_ITEMS; }
static inline int launch_exclusive_scan(cudaStream_t st, int m, const int* counts, int* out, long long* block_sum,
                                        int* block_max, long long* d_total, int* d_max) {
  const int nblocks = scan_blocks(m);
  scan_local_kernel<<<nblocks, 256, 0, st>>>(m, counts, out, block_sum, block_max);
  B200SP_LAUNCH_CHECK();
  scan_blocks_kernel<<<1, 1024, 0, st>>>(nblocks, block_sum, block_max, d_total, d_max);
  B200SP_LAUNCH_CHECK();
  scan_add_kernel<<<nblocks, 256, 0, st>>>(m, out, block_sum, d_total);
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

// ---- the same scan into int64 offsets, for totals past 2^31 (spgemm64.cu) ----------------------------------------------
// Templates on the count type so that only the translation units that use them compile them.
template <typename Cnt>
static __global__ void __launch_bounds__(256) scan64_local_kernel(int m, const Cnt* __restrict__ cnt, int64_t* __restrict__ out,
                                                                  long long* __restrict__ block_sum, int* __restrict__ block_max) {
  __shared__ long long wsum[8];
  const int base = blockIdx.x * SCAN_ITEMS + threadIdx.x * 8;
  long long v[8];
  long long s = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    v[i] = (base + i < m) ? (long long)cnt[base + i] : 0;
    s += v[i];
  }
  long long inc = s;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    long long t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) wsum[w] = inc;
  __syncthreads();
  long long run = inc - s;
  for (int i = 0; i < w; ++i) run += wsum[i];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (base + i < m) out[base + i] = run;
    run += v[i];
  }
  if (threadIdx.x == 255) {
    long long tot = 0;
    for (int i = 0; i < 8; ++i) tot += wsum[i];
    block_sum[blockIdx.x] = tot;
    block_max[blockIdx.x] = 0;
  }
}
template <typename Cnt>
static __global__ void __launch_bounds__(256) scan64_add_kernel(int m, int64_t* __restrict__ out, const long long* __restrict__ block_off,
                                                                const long long* __restrict__ total) {
  const long long off = block_off[blockIdx.x];
  const int base = blockIdx.x * SCAN_ITEMS + threadIdx.x * 8;
#pragma unroll
  for (int i = 0; i < 8; ++i)
    if (base + i < m) out[base + i] += off;
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) out[m] = *total;
}

// counts[0..m) -> out[0..m] as int64 (exclusive offsets, out[m] = *d_total = total); scratch as launch_exclusive_scan's.
template <typename Cnt>
static inline int launch_exclusive_scan64(cudaStream_t st, int m, const Cnt* counts, int64_t* out, long long* block_sum,
                                          int* block_max, long long* d_total, int* d_max) {
  const int nblocks = scan_blocks(m);  // m > 0
  scan64_local_kernel<Cnt><<<nblocks, 256, 0, st>>>(m, counts, out, block_sum, block_max);
  B200SP_LAUNCH_CHECK();
  scan_blocks_kernel<<<1, 1024, 0, st>>>(nblocks, block_sum, block_max, d_total, d_max);
  B200SP_LAUNCH_CHECK();
  scan64_add_kernel<Cnt><<<nblocks, 256, 0, st>>>(m, out, block_sum, d_total);
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

}  // namespace b200sp
