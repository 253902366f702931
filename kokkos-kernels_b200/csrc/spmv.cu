// spmv.cu -- rank-1 CrsMatrix SpMV for H100 (sm_90a): y = beta*y + alpha*op(A)*x.
//
// Replaces the reference's Kokkos::Cuda SpMV legs:
//   native  SPMV_Functor team kernel   sparse/impl/KokkosSparse_spmv_impl.hpp:134-165,337-379
//   native  merge path                 sparse/impl/KokkosSparse_spmv_impl_merge.hpp:70-334
//   native  transpose (atomics)        sparse/impl/KokkosSparse_spmv_impl.hpp:36-84,463-513
//   TPL     cusparseSpMV               sparse/tpls/KokkosSparse_spmv_tpl_spec_decl.hpp:31-197
//
// Kernels (DESIGN.md section 3):
//   spmv_tile_kernel    persistent CTAs; one producer warp streams row-aligned
//                       tiles of (vals, col_idx, row_ptr) into a shared-memory
//                       ring with 1-D TMA bulk copies (cp.async.bulk + mbarrier),
//                       NW consumer warps do sub-warp-per-row dot products out of
//                       shared memory, x gathered through L1 (ld.global.nc),
//                       warp-shuffle reduction, fused alpha/beta epilogue.
//                       IDX16 form: col_idx is replaced by the plan's 16-bit in-row
//                       column deltas + one 32-bit anchor column per row (section 3.5).
//                       Pattern form: one 16-bit pattern start per row into a dictionary
//                       of in-row column offsets, + the anchors (section 3.6).
//   spmv_longrow_kernel rows longer than the tile's row limit: one CTA per row (default), or -- opt-in,
//                       B200SP_SPMV_LONGROWS=seg -- segments of <= 4096 entries + ordered combine.
//   spmv_vector_kernel  no-analysis fallback (FAST_SETUP, tiny or misaligned
//                       inputs): sub-warp per row straight from global memory.
//   spmv_transpose_kernel  T/H modes: y pre-scaled, atomicAdd scatter.
#include "common.cuh"
#include "spmv_plan.h"
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <mutex>
#include <type_traits>

namespace b200sp {

// ---------------------------------------------------------------------------
// error string + launch counter + device props
// ---------------------------------------------------------------------------
static thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int sm_count() {
  static int cached[64];
  static std::once_flag once;
  std::call_once(once, [] { memset(cached, 0, sizeof(cached)); });
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

void keep_async_pool_memory() {
#ifndef B200SP_EMU
  static std::atomic<unsigned> done{0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 32) return;
  if (done.load() & (1u << dev)) return;
  const char* keep_env = getenv("B200SP_KEEP_POOL");  // 0: leave the device's default pool as the application configured it
  if (keep_env && keep_env[0] == '0') {
    done.fetch_or(1u << dev);
    return;
  }
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
    uint64_t keep = UINT64_MAX;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
  }
  done.fetch_or(1u << dev);
#endif
}

// ---------------------------------------------------------------------------
// y = beta*y (beta == 0 writes exact zeros without reading y)
// ---------------------------------------------------------------------------
template <typename S>
__global__ void scale_kernel(int64_t n, S beta, S* __restrict__ y) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  if (beta == S(0)) {
    for (; i < n; i += stride) y[i] = S(0);
  } else {
    for (; i < n; i += stride) y[i] = beta * y[i];
  }
}

template <typename S>
static int launch_scale(cudaStream_t st, int64_t n, S beta, S* y) {
  if (n <= 0) return B200SP_OK;
  if (beta == S(1)) return B200SP_OK;
  int blocks = (int)std::min<int64_t>((n + 255) / 256, (int64_t)sm_count() * 8);
  scale_kernel<S><<<blocks, 256, 0, st>>>(n, beta, y);
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

// ---------------------------------------------------------------------------
// sub-warp reduction: sum over the LPR lanes that share a row
// ---------------------------------------------------------------------------
template <int LPR, typename S>
__device__ __forceinline__ S subwarp_sum(S v) {
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) v += shfl_xor(v, o);
  return v;
}

// ex.n > 0: every value is also stored to ex.n further destinations (P2P mappings of the peers' buffers, or one NVSwitch
// multicast mapping).  ex.n < 0 ("forward", one destination ex.p[0]) is seen by the forwarding form of the tiled kernel only,
// whose producer warp copies whole finished tiles (the loop below then stores nothing); every other kernel of a forwarding
// call gets the same destination as an ordinary extra one (direct_extra()).
template <typename S>
__device__ __forceinline__ void store_y(S* __restrict__ y, int r, S sum, S alpha, S beta, const YExtra& ex) {
  // reference epilogue (spmv_impl.hpp:124-131): sum *= alpha; y = beta*y + sum
  sum *= alpha;
  const S v = (beta == S(0)) ? sum : beta * y[r] + sum;
  y[r] = v;
  for (int d = 0; d < ex.n; ++d) static_cast<S*>(ex.p[d])[r] = v;  // P2P stores
}
static inline YExtra direct_extra(YExtra ex) {
  if (ex.n < 0) ex.n = 1;
  return ex;
}

// rows [r0, r1) of y -> the forward destination, by one warp: 32 lanes x 8 bytes = 256 contiguous bytes per store instruction
// (whole 128-byte NVLink writes instead of one 8-byte packet per row).  The loads bypass L1: the values were written by other
// warps of this CTA a moment ago.
template <typename S>
__device__ __forceinline__ void forward_rows(const S* __restrict__ y, S* __restrict__ dst, int r0, int r1, int lane) {
  for (int r = r0 + lane; r < r1; r += 32) dst[r] = __ldcg(y + r);
}

// ---------------------------------------------------------------------------
// fallback: sub-warp per row, straight from global memory
// ---------------------------------------------------------------------------
template <typename S, int LPR>
__global__ void __launch_bounds__(256) spmv_vector_kernel(int m, const int* __restrict__ row_ptr,
                                                          const int* __restrict__ col_idx,
                                                          const S* __restrict__ vals,
                                                          const S* __restrict__ x, S* __restrict__ y,
                                                          S alpha, S beta, YExtra ex, int lmax) {
  // rows longer than lmax are left to spmv_longrow_kernel, as the tiled kernel leaves them: whichever of the two kernels a
  // self-tuning plan settles on, every row is summed in the same order (INT_MAX: this kernel takes every row)
  constexpr int RPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR, sl = lane % LPR;
  const int64_t warp_global = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t g = warp_global; g * RPW < m; g += nwarps) {
    const int r = (int)(g * RPW) + sub;
    int rs = 0, re = 0;
    if (r < m) {
      rs = row_ptr[r];
      re = row_ptr[r + 1];
    }
    const bool is_long = (re - rs) > lmax;
    if (is_long) re = rs;
    S sum = S(0);
    constexpr int UNR = 8;
    for (int j0 = rs + sl; j0 < re; j0 += UNR * LPR) {
      int c[UNR];
      S av[UNR], xv[UNR];
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        const int j = j0 + u * LPR;
        const bool ok = j < re;
        c[u] = ok ? ld_stream(col_idx + j) : 0;
        av[u] = ok ? ld_stream(vals + j) : S(0);
      }
#pragma unroll
      for (int u = 0; u < UNR; ++u) xv[u] = (j0 + u * LPR < re) ? ldg(x + c[u]) : S(0);
#pragma unroll
      for (int u = 0; u < UNR; ++u) sum += av[u] * xv[u];
    }
    sum = subwarp_sum<LPR>(sum);
    if (r < m && sl == 0 && !is_long) store_y(y, r, sum, alpha, beta, ex);
  }
}

// ---------------------------------------------------------------------------
// long rows: one CTA per row taken from a device-side list
// ---------------------------------------------------------------------------
template <typename S>
__global__ void __launch_bounds__(256) spmv_longrow_kernel(const int* __restrict__ long_rows,
                                                           const int* __restrict__ n_long_ptr,
                                                           const int* __restrict__ row_ptr,
                                                           const int* __restrict__ col_idx,
                                                           const S* __restrict__ vals,
                                                           const S* __restrict__ x, S* __restrict__ y,
                                                           S alpha, S beta, YExtra ex) {
  __shared__ S warp_part[8];
  const int n_long = *n_long_ptr;
  for (int i = blockIdx.x; i < n_long; i += gridDim.x) {
    const int r = long_rows[i];
    const int rs = row_ptr[r], re = row_ptr[r + 1];
    S sum = S(0);
    for (int j = rs + threadIdx.x; j < re; j += 256)
      sum += ld_stream(vals + j) * ldg(x + ld_stream(col_idx + j));
    sum = subwarp_sum<32>(sum);
    if ((threadIdx.x & 31) == 0) warp_part[threadIdx.x >> 5] = sum;
    __syncthreads();
    if (threadIdx.x == 0) {
      S t = S(0);
#pragma unroll
      for (int w = 0; w < 8; ++w) t += warp_part[w];
      store_y(y, r, t, alpha, beta, ex);
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------
// long rows, adaptive row splitting (opt-in, B200SP_SPMV_LONGROWS=seg): every long row is cut into segments of
// <= SEG entries (build_row_segments_kernel, once per matrix), one CTA sums a segment, and a second small kernel
// adds a row's partial sums in segment order -- the longest row no longer serialises on one CTA (R-MAT scale 23:
// 152,801 entries), and the result stays deterministic (fixed association, no atomics).
// ---------------------------------------------------------------------------
__global__ void build_row_segments_kernel(const int* __restrict__ long_rows, const int* __restrict__ n_long,
                                          const int* __restrict__ row_ptr, int SEG, int4* __restrict__ segs,
                                          int* __restrict__ n_seg, int2* __restrict__ row_seg) {
  const int nl = *n_long;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nl; i += gridDim.x * blockDim.x) {
    const int r = long_rows[i];
    const int s = row_ptr[r], e = row_ptr[r + 1];
    const int nseg = (e - s + SEG - 1) / SEG;
    const int base = atomicAdd(n_seg, nseg);
    row_seg[i] = make_int2(base, nseg);
    for (int q = 0; q < nseg; ++q) segs[base + q] = make_int4(r, s + q * SEG, min(e, s + (q + 1) * SEG), q);
  }
}

template <typename S>
__global__ void __launch_bounds__(256) spmv_seg_partial_kernel(const int4* __restrict__ segs, const int* __restrict__ n_seg_ptr,
                                                               const int* __restrict__ col_idx, const S* __restrict__ vals,
                                                               const S* __restrict__ x, S* __restrict__ partial) {
  __shared__ S warp_part[8];
  const int n_seg = *n_seg_ptr;
  for (int q = blockIdx.x; q < n_seg; q += gridDim.x) {
    const int4 d = segs[q];
    S sum = S(0);
    constexpr int UNR = 4;
    for (int j0 = d.y + threadIdx.x; j0 < d.z; j0 += 256 * UNR) {
      int c[UNR];
      S av[UNR];
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        const int j = j0 + u * 256;
        const bool ok = j < d.z;
        c[u] = ok ? ld_stream(col_idx + j) : 0;
        av[u] = ok ? ld_stream(vals + j) : S(0);
      }
#pragma unroll
      for (int u = 0; u < UNR; ++u) sum += (j0 + u * 256 < d.z) ? av[u] * ldg(x + c[u]) : S(0);
    }
    sum = subwarp_sum<32>(sum);
    if ((threadIdx.x & 31) == 0) warp_part[threadIdx.x >> 5] = sum;
    __syncthreads();
    if (threadIdx.x == 0) {
      S t = S(0);
#pragma unroll
      for (int w = 0; w < 8; ++w) t += warp_part[w];
      partial[q] = t;
    }
    __syncthreads();
  }
}

template <typename S>
__global__ void __launch_bounds__(256) spmv_seg_combine_kernel(const int* __restrict__ long_rows, const int* __restrict__ n_long_ptr,
                                                               const int2* __restrict__ row_seg, const S* __restrict__ partial,
                                                               S* __restrict__ y, S alpha, S beta, YExtra ex) {
  const int n_long = *n_long_ptr;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_long; i += gridDim.x * blockDim.x) {
    const int2 rs = row_seg[i];
    S t = S(0);
    for (int q = 0; q < rs.y; ++q) t += partial[rs.x + q];
    store_y(y, long_rows[i], t, alpha, beta, ex);
  }
}

// ---------------------------------------------------------------------------
// transpose modes: y (pre-scaled) += alpha * A^T x, atomics like the reference
// ---------------------------------------------------------------------------
template <typename S, int LPR>
__global__ void __launch_bounds__(256) spmv_transpose_kernel(int m, const int* __restrict__ row_ptr,
                                                             const int* __restrict__ col_idx,
                                                             const S* __restrict__ vals,
                                                             const S* __restrict__ x, S* __restrict__ y,
                                                             S alpha) {
  constexpr int RPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR, sl = lane % LPR;
  const int64_t warp_global = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t g = warp_global; g * RPW < m; g += nwarps) {
    const int r = (int)(g * RPW) + sub;
    if (r >= m) continue;
    const int rs = row_ptr[r], re = row_ptr[r + 1];
    const S xv = alpha * x[r];  // serial reference order: x_val = alpha*x[i] (spmv_impl.hpp:426)
    for (int j = rs + sl; j < re; j += LPR) atomicAdd(&y[ld_stream(col_idx + j)], ld_stream(vals + j) * xv);
  }
}

// ---------------------------------------------------------------------------
// tile analysis.  Tile b owns the rows whose first entry lies in
// [b*T, (b+1)*T); descriptor = {r0, r1, s = row_ptr[r0], e = staged end}.
// Rows longer than LMAX (found by find_long_rows_kernel) are skipped by the
// tile kernel and computed by spmv_longrow_kernel; T + LMAX + 8 <= CAP makes
// every other row fit the stage.
// ---------------------------------------------------------------------------
__device__ __forceinline__ int lower_bound_rows(const int* __restrict__ row_ptr, int m, int64_t v) {
  // first r in [0, m) with row_ptr[r] >= v, else m
  int lo = 0, hi = m;
  while (lo < hi) {
    const int mid = lo + ((hi - lo) >> 1);
    if ((int64_t)row_ptr[mid] < v) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

__global__ void build_tiles_kernel(int m, const int* __restrict__ row_ptr, int n_tiles, int T, int CAP,
                                   int4* __restrict__ tiles) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n_tiles) return;
  const int r0 = lower_bound_rows(row_ptr, m, (int64_t)b * T);
  const int r1 = lower_bound_rows(row_ptr, m, (int64_t)(b + 1) * T);
  int s = 0, e = 0;
  if (r1 > r0) {
    s = row_ptr[r0];
    e = row_ptr[r1];
    // every row but the last ends before (b+1)*T; only a long (> LMAX) last row can exceed the stage.  The clamp also holds
    // for the 16-bit column form, whose stages start at s & ~7: cap_end <= (s & ~7) + CAP, and every row <= LMAX ends at
    // most at s + T + LMAX - 1 = s + CAP - 9 < cap_end.
    const int cap_end = (s & ~3) + CAP - 4;
    if (e > cap_end) e = cap_end;
  }
  tiles[b] = make_int4(r0, r1, s, e);
}

// rows longer than LMAX are skipped by the tile kernel and handled by spmv_longrow_kernel
__global__ void find_long_rows_kernel(int m, const int* __restrict__ row_ptr, int LMAX, int* __restrict__ long_rows,
                                      int* __restrict__ n_long) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < m; r += gridDim.x * blockDim.x)
    if (row_ptr[r + 1] - row_ptr[r] > LMAX) long_rows[atomicAdd(n_long, 1)] = r;
}

// The tiles and long rows of the tile kernels (spmv_tile_kernel, the BSR ones of bsr.cu with blocks for
// entries) for a stage of cap entries and a row limit of lmax.  *out owns what it allocated, also on an error.
int tile_analyse(cudaStream_t st, int m, int64_t nnz, const int* row_ptr, int cap, int lmax, TileAnalysis* out) {
  out->LMAX = lmax;
  out->T = cap - lmax - 8;
  out->n_tiles = (int)(nnz / out->T) + 1;
  out->long_cap = (int)(nnz / (lmax + 1)) + 1;  // every long row holds more than lmax entries
  B200SP_CUDA_TRY(out->tiles.alloc((size_t)out->n_tiles, st));
  B200SP_CUDA_TRY(out->long_rows.alloc((size_t)out->long_cap, st));
  B200SP_CUDA_TRY(out->n_long.alloc(1, st));
  B200SP_CUDA_TRY(cudaMemsetAsync(out->n_long, 0, sizeof(int), st));
  build_tiles_kernel<<<(out->n_tiles + 255) / 256, 256, 0, st>>>(m, row_ptr, out->n_tiles, out->T, cap, out->tiles);
  B200SP_LAUNCH_CHECK();
  find_long_rows_kernel<<<std::max(1, std::min((m + 255) / 256, sm_count() * 8)), 256, 0, st>>>(m, row_ptr, lmax, out->long_rows,
                                                                                                out->n_long);
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

// 16-bit column form of the tiled kernel (DESIGN.md section 3.5): d[j] = col_idx[j] - col_idx[j-1] inside a row, 0 for the
// first entry of a row; anchor[r] = col_idx[row_ptr[r]], 0 for an empty row.  *bad is set when a row the tiled kernel reads
// (<= LMAX entries) has an in-row delta outside [0, 65535] (unsorted, or a gap too wide); longer rows go to the long-row
// kernel, which reads col_idx.  The differences are taken modulo 2^32, so the kernel's anchor + sum of deltas is col_idx[j]
// exactly whenever no delta was flagged.  8 lanes per row.
__global__ void build_idx16_kernel(int m, const int* __restrict__ row_ptr, const int* __restrict__ col_idx, int LMAX,
                                   uint16_t* __restrict__ d, int* __restrict__ anchor, int* __restrict__ bad) {
  constexpr int G = 8;
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int sl = (int)(t % G);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x / G;
  bool wide = false;
  for (int64_t r = t / G; r < m; r += stride) {
    const int rs = row_ptr[r], re = row_ptr[r + 1];
    if (sl == 0) anchor[r] = re > rs ? col_idx[rs] : 0;
    const bool checked = re - rs <= LMAX;
    for (int j = rs + sl; j < re; j += G) {
      const unsigned dl = j == rs ? 0u : (unsigned)col_idx[j] - (unsigned)col_idx[j - 1];
      wide |= checked && dl > 65535u;
      d[j] = (uint16_t)dl;
    }
  }
  if (wide) *bad = 1;
}

// Pattern form of the tiled kernel (DESIGN.md section 3.6): the offsets col_idx[j] - anchor[r] of a row, taken over the row,
// form its pattern.  Matrices from structured grids have a handful of patterns (lap27: 8), so a row's columns are its anchor
// plus one uint16 pid[r], the start of its pattern in a dictionary of at most DCAP offsets that the tiled kernel keeps in
// shared memory.  dict[DCAP] holds the dictionary's used length.  Three passes, stream-ordered: hash every row of 1..LMAX
// entries into a small open-addressing table; lay the table's patterns out in the dictionary; then set pid[r] and check every
// entry of every such row against the dictionary, so that a hash collision only makes the matrix fall back.  *bad is set
// when the table or the dictionary overflows or an entry does not match.
constexpr int DCAP = 1024;         // dictionary offsets (4 KB of shared memory)
constexpr int PAT_SLOTS = 2048;    // hash table slots: a qualifying matrix has at most DCAP patterns
constexpr int PAT_PROBES = 64;     // linear probes before the table counts as full

__device__ __forceinline__ unsigned long long pat_mix(unsigned long long z) {  // splitmix64 finaliser
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

// 8 lanes per row: the hash of (length, offsets) is a sum of per-entry hashes, so the lanes add theirs with three shuffles
__global__ void pattern_hash_kernel(int m, const int* __restrict__ row_ptr, const int* __restrict__ col_idx, int LMAX,
                                    unsigned long long* __restrict__ table, int* __restrict__ rep, int* __restrict__ row_slot,
                                    int* __restrict__ bad) {
  constexpr int G = 8;
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int sl = (int)(t % G);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x / G;
  const int64_t r_end = ((int64_t)m + G - 1) / G * G;  // whole warps (4 rows each) run every pass: the shuffles
  for (int64_t r = t / G; r < r_end; r += stride) {
    int rs = 0, re = 0;
    if (r < m) {
      rs = row_ptr[r];
      re = row_ptr[r + 1];
    }
    const int len = re - rs;
    const bool mine = len >= 1 && len <= LMAX;
    unsigned long long h = 0;
    if (mine) {
      const unsigned c0 = (unsigned)col_idx[rs];
      for (int k = sl; k < len; k += G) h += pat_mix(((unsigned long long)k << 32) | ((unsigned)col_idx[rs + k] - c0));
    }
#pragma unroll
    for (int o = 1; o < G; o <<= 1) h += __shfl_xor_sync(0xffffffffu, h, o);
    if (!mine || sl != 0) continue;
    h += pat_mix(0x9e3779b97f4a7c15ull ^ (unsigned long long)len);
    if (h == 0) h = 1;  // 0 marks an empty slot
    int slot = -1;
    if (__ldcg(bad) == 0) {
      // load first: the few distinct keys are inserted once, then every row finds its key without an atomic
      for (int q = 0, s = (int)(h % PAT_SLOTS); q < PAT_PROBES; ++q, s = (s + 1) % PAT_SLOTS) {
        unsigned long long k = __ldcg(table + s);
        if (k == 0) {
          k = atomicCAS(table + s, 0ull, h);
          if (k == 0) rep[s] = (int)r;  // the inserting row represents the slot
        }
        if (k == 0 || k == h) {
          slot = s;
          break;
        }
      }
      if (slot < 0) *bad = 1;
    }
    row_slot[r] = slot;
  }
}

// one CTA of 256 threads, PAT_SLOTS / 256 consecutive slots each: pattern starts in slot order
__global__ void __launch_bounds__(256) pattern_dict_kernel(const int* __restrict__ row_ptr, const int* __restrict__ col_idx,
                                                           const unsigned long long* __restrict__ table, const int* __restrict__ rep,
                                                           int* __restrict__ slot_start, int* __restrict__ slot_len,
                                                           int* __restrict__ dict, int* __restrict__ bad) {
  constexpr int PER = PAT_SLOTS / 256;
  __shared__ int part[257];
  if (*bad) return;  // the same value for every thread
  const int s0 = threadIdx.x * PER;
  int len[PER], sum = 0;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    len[i] = 0;
    if (table[s0 + i]) len[i] = row_ptr[rep[s0 + i] + 1] - row_ptr[rep[s0 + i]];
    sum += len[i];
  }
  part[threadIdx.x + 1] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    part[0] = 0;
    for (int i = 1; i <= 256; ++i) part[i] += part[i - 1];
    dict[DCAP] = part[256];
    if (part[256] > DCAP) *bad = 1;
  }
  __syncthreads();
  if (part[256] > DCAP) return;
  int base = part[threadIdx.x];
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    slot_start[s0 + i] = base;
    slot_len[s0 + i] = len[i];
    if (len[i]) {
      const int rs = row_ptr[rep[s0 + i]];
      const unsigned c0 = (unsigned)col_idx[rs];
      for (int k = 0; k < len[i]; ++k) dict[base + k] = (int)((unsigned)col_idx[rs + k] - c0);
    }
    base += len[i];
  }
}

// pid[r] for every row (0 for empty and long rows), and the check of every entry the tiled kernel will rebuild
__global__ void pattern_assign_kernel(int m, const int* __restrict__ row_ptr, const int* __restrict__ col_idx, int LMAX,
                                      const int* __restrict__ row_slot, const int* __restrict__ slot_start,
                                      const int* __restrict__ slot_len, const int* __restrict__ dict,
                                      uint16_t* __restrict__ pid, int* __restrict__ bad) {
  constexpr int G = 8;
  if (*bad) return;
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int sl = (int)(t % G);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x / G;
  bool wrong = false;
  for (int64_t r = t / G; r < m; r += stride) {
    const int rs = row_ptr[r], len = row_ptr[r + 1] - rs;
    int start = 0;
    if (len >= 1 && len <= LMAX) {
      const int s = row_slot[r];
      start = slot_start[s];
      if (slot_len[s] != len) {
        wrong = true;
      } else {
        const unsigned c0 = (unsigned)col_idx[rs];
        for (int k = sl; k < len; k += G) wrong |= (int)((unsigned)col_idx[rs + k] - c0) != dict[start + k];
      }
    }
    if (sl == 0) pid[r] = (uint16_t)start;
  }
  if (wrong) *bad = 1;
}

// ---------------------------------------------------------------------------
// the TMA-tiled kernel
// ---------------------------------------------------------------------------
__device__ __forceinline__ int64_t dmin64(int64_t a, int64_t b) { return a < b ? a : b; }
__device__ __forceinline__ int64_t dmax64(int64_t a, int64_t b) { return a > b ? a : b; }

// The pattern form's layout, for every configuration (DESIGN.md sections 3.6 and 7): stages of PAT_CAP entries with PAT_RCAP
// row slots, two CTAs of 16 consumer warps per SM in f64.  The form streams no per-entry columns, so a stage holds only values
// and row slots -- row_ptr (TileRing::rows), anchor (cols[0, RCAP)) and pattern start (cols[RCAP, 3*RCAP/2) as uint16) --
// and the dictionary follows the ring, once per CTA.  Rows of a tile past the row slots read the three from global memory.
constexpr int PAT_CAP = 4096, PAT_STAGES = 3, PAT_RCAP = 256;
// The form's value copies start and end on 128-byte lines (EAL below), so that two tiles never split a line between them:
// up to 2 * (32 - 1) entries of f32 more than the tile, which its tiles leave room for (tile_analyse's T = cap - LMAX - 8).
constexpr int PAT_TILE_CAP = PAT_CAP - 2 * 32 + 8;
template <typename S, int CAP, int RCAP, int STAGES>
using PatTileRing = TileRing<S, CAP, RCAP * 3 / 2, RCAP, STAGES>;

// the ring of spmv_tile_kernel in each column form, and the dynamic shared memory past it (the pattern form's dictionary)
template <typename S, int CAP, int STAGES, int COLS>
using TileSmem = std::conditional_t<COLS == COLS_PAT, PatTileRing<S, CAP, PAT_RCAP, STAGES>, CsrTileRing<S, CAP, STAGES>>;
template <int COLS>
constexpr int tile_smem_extra() { return COLS == COLS_PAT ? (int)sizeof(int) * DCAP : 0; }

// CTAs per SM with 56 registers per thread and the kernel's ring.  Both column forms are held to it: left alone, the compiler
// gives the 16-bit form's decode up to 91 registers, and the 32-bit form 80 once both share this kernel -- one CTA per SM
// instead of two in the default configuration.
template <typename S, int NW, int STAGES, int CAP, int COLS>
constexpr int tile_ctas_per_sm() {
  const int by_regs = 65536 / ((NW + 1) * 32 * 56);
  const int by_smem = (227 * 1024) / (int)(sizeof(TileSmem<S, CAP, STAGES, COLS>) + tile_smem_extra<COLS>() + 128 + 1024);
  const int c = by_regs < by_smem ? by_regs : by_smem;
  return c > 1 ? c : 1;
}

// FWD: the fused all-gather form (b200sp_spmv_forward_f64_i32): the producer warp forwards finished tiles of y to ex.p[0].
// A template parameter, so that the plain kernel -- the one every roofline number of this repository is measured on -- carries
// no trace of it.
// COLS_DELTA: columns come from c16 (deltas) / anchor (build_idx16_kernel) instead of col_idx: 2 bytes per entry plus 4 per
// row instead of 4 per entry.  COLS_PAT: from c16 (pattern starts) / anchor / dict (pattern_*_kernel): 6 bytes per row.
// Same lanes, same entries per lane, same order: the same bits as the 32-bit form.
template <typename S, int LPR, int NW, int STAGES, int CAP, int UNR, int COLS = COLS_I32, bool FWD = false>
__global__ void __launch_bounds__((NW + 1) * 32, tile_ctas_per_sm<S, NW, STAGES, CAP, COLS>())
    spmv_tile_kernel(int m, int64_t nnz, int n_tiles, int LMAX, const int4* __restrict__ tiles,
                     const int* __restrict__ row_ptr, const int* __restrict__ col_idx,
                     const uint16_t* __restrict__ c16, const int* __restrict__ anchor, const int* __restrict__ dict,
                     const S* __restrict__ vals, const S* __restrict__ x, S* __restrict__ y, S alpha,
                     S beta, YExtra ex) {
  using Smem = TileSmem<S, CAP, STAGES, COLS>;
  constexpr int RCAP = Smem::RCAP;
  constexpr bool IDX16 = COLS == COLS_DELTA, PAT = COLS == COLS_PAT;
  // a stage starts at an entry that is a multiple of EAL: 16 bytes of the narrowest entry stream (bulk-copy alignment), and
  // in the pattern form, whose only entry stream is the values, a 128-byte line of them (PAT_TILE_CAP)
  constexpr int EAL = IDX16 ? 8 : PAT ? 128 / (int)sizeof(S) : 4;
  // ... and at a row that is a multiple of RAL: 16 bytes of the narrowest row stream
  constexpr int RAL = PAT ? 8 : 4;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>(smem_raw);
  int* sdict = reinterpret_cast<int*>(smem_raw + sizeof(Smem));  // PAT: the dictionary, after the ring

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if constexpr (PAT) {
    const int dl = dict[DCAP];  // used length
    for (int i = threadIdx.x; i < dl; i += blockDim.x) sdict[i] = dict[i];
  }
  tile_ring_init(sm, NW);

  if (warp == NW) {
    // ------------------------- producer warp ------------------------------
    const uint64_t pol = l2_policy_evict_first();
    const int64_t nnz_al = nnz & ~(int64_t)3;           // bulk copies stay below this entry
    const int rp_al_end = (m + 1) & ~3;                 // ... and below this row_ptr entry
    int4 mine = make_int4(0, 0, 0, 0);
    constexpr bool forward = FWD;  // fused all-gather: finished tiles of y go on to ex.p[0] (see store_y)
    int n_mine = 0;
    int fr0 = 0, fr1 = 0;  // rows of the tile whose values (fv0: row fr0 + lane, fv1: row fr0 + 32 + lane) wait to be stored
    S fv0 = S(0), fv1 = S(0);
    for (int it = 0;; ++it) {
      const int64_t tile = blockIdx.x + (int64_t)it * gridDim.x;
      if (tile >= n_tiles) break;
      if ((it & 31) == 0) {
        const int64_t t = blockIdx.x + (int64_t)(it + lane) * gridDim.x;
        if (t < n_tiles) mine = tiles[t];
      }
      int4 d;
      d.x = __shfl_sync(0xffffffffu, mine.x, it & 31);
      d.y = __shfl_sync(0xffffffffu, mine.y, it & 31);
      d.z = __shfl_sync(0xffffffffu, mine.z, it & 31);
      d.w = __shfl_sync(0xffffffffu, mine.w, it & 31);
      const int stage = it % STAGES;
      const uint32_t ph = (uint32_t)(it / STAGES) & 1u;
      mbar_wait(&sm.empty[stage], ph ^ 1u);
      // every consumer warp has left tile it - STAGES: its rows of y are final.  They are forwarded AFTER the refill of the
      // stage has been issued (below), so that the copy to the peers rides behind the TMA and not in front of it.
      int4 dp = make_int4(0, 0, 0, 0);
      if (forward) {
        if (it >= STAGES) dp = sm.desc[stage];
        __syncwarp();  // (lane 0 overwrites the descriptor below)
      }

      const int r0 = d.x, r1 = d.y, s = d.z, e = d.w;
      S* sv = sm.vals[stage];
      int* sc = sm.cols[stage];
      int* sr = sm.rows[stage];
      uint16_t* sd = reinterpret_cast<uint16_t*>(sc);  // IDX16: deltas, then anchors
      int* sa = PAT ? sc : reinterpret_cast<int*>(sd + CAP);
      uint16_t* sp = reinterpret_cast<uint16_t*>(sc + RCAP);  // PAT: pattern starts, after the anchors
      // entries [s_al, e) -> smem[0 ..); bulk part [s_al, bulk_end), tail by plain loads.  nnz_al is a multiple of 4 and
      // s_al of EAL, so every bulk length is a multiple of 16 bytes.  The delta stream is padded to a multiple of 8 entries
      // by the plan: its copy [s_al, e_up) is always whole.
      const int s_al = s & ~(EAL - 1);
      const int e_up = (e + EAL - 1) & ~(EAL - 1);
      const int bulk_end = (int)dmin64(e_up, nnz_al);
      const int nb = (r1 > r0 && bulk_end > s_al) ? bulk_end - s_al : 0;
      const int nd = (IDX16 && r1 > r0) ? e_up - s_al : 0;
      if (r1 > r0 && (int64_t)e > nnz_al) {
        const int t0 = (int)dmax64(s_al, nnz_al);
        for (int i = t0 + lane; i < e; i += 32) {
          sv[i - s_al] = vals[i];
          if (COLS == COLS_I32) sc[i - s_al] = col_idx[i];
        }
      }
      // row_ptr[r0_al .. r1] -> rows[0 ..], at most RCAP entries
      const int r0_al = r0 & ~(RAL - 1);
      int nrp = 0, na = 0, np = 0;
      if (r1 > r0) {
        const int want_end = min(r1 + 1, r0_al + RCAP);  // exclusive
        const int want_up = (want_end + 3) & ~3;
        const int rbulk_end = min(min(want_up, r0_al + RCAP), rp_al_end);
        nrp = rbulk_end > r0_al ? rbulk_end - r0_al : 0;
        if (want_end > rp_al_end) {
          const int t0 = max(r0_al, rp_al_end);
          for (int i = t0 + lane; i < want_end; i += 32) sr[i - r0_al] = row_ptr[i];
        }
        // anchors of rows [r0_al, r1), at most RCAP; the plan pads the anchor stream to a multiple of 4 rows
        if (COLS != COLS_I32) na = min((r1 + 3) & ~3, r0_al + RCAP) - r0_al;
        // PAT: pattern starts of the same rows; the plan pads that stream to a multiple of 8 rows
        if (PAT) np = min((r1 + 7) & ~7, r0_al + RCAP) - r0_al;
      }
      __syncwarp();
      if (lane == 0) {
        sm.desc[stage] = d;
        const uint32_t col_bytes = COLS == COLS_I32 ? (uint32_t)(nb * 4) : (uint32_t)(nd * 2 + na * 4 + np * 2);
        mbar_arrive_expect_tx(&sm.full[stage], (uint32_t)(nb * sizeof(S)) + col_bytes + (uint32_t)(nrp * 4));
        if (nb > 0) {
          bulk_g2s(sv, vals + s_al, (uint32_t)(nb * sizeof(S)), &sm.full[stage], pol);
          if (COLS == COLS_I32) bulk_g2s(sc, col_idx + s_al, (uint32_t)(nb * 4), &sm.full[stage], pol);
        }
        if (nd > 0) bulk_g2s(sd, c16 + s_al, (uint32_t)(nd * 2), &sm.full[stage], pol);
        if (np > 0) bulk_g2s(sp, c16 + r0_al, (uint32_t)(np * 2), &sm.full[stage], pol);
        if (na > 0) bulk_g2s(sa, anchor + r0_al, (uint32_t)(na * 4), &sm.full[stage], pol);
        if (nrp > 0) bulk_g2s(sr, row_ptr + r0_al, (uint32_t)(nrp * 4), &sm.full[stage], pol);
      }
      __syncwarp();
      if (forward) {
        // Software-pipelined by one tile: the values of the tile that just left are only LOADED here (from L2) and stored
        // when the next tile comes round -- a load-then-store in one go made the producer warp the bottleneck of the
        // kernel.  Tiles of more than 64
        // rows are forwarded in one go.
        S* dst = static_cast<S*>(ex.p[0]);
        if (fr1 > fr0) {
          if (fr0 + lane < fr1) dst[fr0 + lane] = fv0;
          if (fr0 + 32 + lane < fr1) dst[fr0 + 32 + lane] = fv1;
        }
        fr0 = fr1 = 0;
        if (dp.y - dp.x <= 64) {
          fr0 = dp.x;
          fr1 = dp.y;
          if (fr0 + lane < fr1) fv0 = __ldcg(y + fr0 + lane);
          if (fr0 + 32 + lane < fr1) fv1 = __ldcg(y + fr0 + 32 + lane);
        } else {
          forward_rows<S>(y, dst, dp.x, dp.y, lane);
        }
        n_mine = it + 1;
      }
    }
    if (forward) {  // the pending tile, then the last tiles of this CTA: wait for the consumers to leave each, then forward it
      S* dst = static_cast<S*>(ex.p[0]);
      if (fr1 > fr0) {
        if (fr0 + lane < fr1) dst[fr0 + lane] = fv0;
        if (fr0 + 32 + lane < fr1) dst[fr0 + 32 + lane] = fv1;
      }
      for (int j = n_mine > STAGES ? n_mine - STAGES : 0; j < n_mine; ++j) {
        const int stage = j % STAGES;
        mbar_wait(&sm.empty[stage], (uint32_t)(j / STAGES) & 1u);
        const int4 dp = sm.desc[stage];
        forward_rows<S>(y, static_cast<S*>(ex.p[0]), dp.x, dp.y, lane);
      }
    }
  } else {
    // ------------------------- consumer warps -----------------------------
    constexpr int RPW = 32 / LPR;
    const int sub = lane / LPR, sl = lane % LPR;
    for (int it = 0; tile_ring_more(it, n_tiles); ++it) {
      const TileView tv = tile_ring_acquire<EAL, RAL>(sm, it);
      const int stage = tv.stage, r0 = tv.r0, r1 = tv.r1, s_al = tv.s_al;
      const S* sv = sm.vals[stage];
      const int* sc = sm.cols[stage];
      const uint16_t* sd = reinterpret_cast<const uint16_t*>(sc);
      const int* sa = PAT ? sc : reinterpret_cast<const int*>(sd + CAP);
      const uint16_t* sp = reinterpret_cast<const uint16_t*>(sc + RCAP);
      // absolute row groups of RPW rows are dealt round-robin to the warps
      const int g_first = r0 / RPW;
      int g = g_first + ((warp - g_first % NW) + NW) % NW;
      for (; g * RPW < r1; g += NW) {
        const int r = g * RPW + sub;
        const bool valid = (r >= r0) && (r < r1);
        int rs = 0, re = 0, col = 0, pb = 0;
        if (valid) {
          const int o = r - tv.r0_al;
          if (tile_row_bounds(sm, stage, row_ptr, r, o, rs, re)) {
            if (COLS != COLS_I32) col = sa[o];
            if (PAT) pb = sp[o];
          } else {
            if (COLS != COLS_I32) col = anchor[r];
            if (PAT) pb = c16[r];
          }
        }
        const bool is_long = (re - rs) > LMAX;
        if (is_long) re = rs;
        S sum = S(0);
        const int jend = re - s_al;
        if constexpr (IDX16) {
          // The passes run over the row, not over the lane's own entries, so that the LPR lanes of a row take the same
          // number of passes and can shuffle; a lane's extra passes only add +0.0, which leaves its sum's bits alone.
          // Entry jb + u*LPR + sl is the lane's u-th of the pass, as in the 32-bit form.  Its column is col (the column of
          // the entry before the pass, the row's anchor at first) plus the deltas of the pass up to it: the totals of slices
          // 0..u-1 plus the inclusive prefix of slice u over the row's lanes.  One butterfly per slice gives both the prefix
          // and the total in log2(LPR) shuffles; the UNR slices are independent, so their shuffles overlap.
          const unsigned gmask = LPR == 32 ? 0xffffffffu : ((1u << LPR) - 1u) << (sub * LPR);
          for (int jb = rs - s_al; jb < jend; jb += UNR * LPR) {
            int c[UNR], tot[UNR];
            S av[UNR], xv[UNR];
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
              const int j = jb + u * LPR + sl;
              c[u] = tot[u] = j < jend ? (int)sd[j] : 0;  // entries past the row contribute 0
            }
#pragma unroll
            for (int o = 1; o < LPR; o <<= 1) {
#pragma unroll
              for (int u = 0; u < UNR; ++u) {
                const int t = __shfl_xor_sync(gmask, tot[u], o);
                if (sl & o) c[u] += t;
                tot[u] += t;
              }
            }
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
              c[u] += col;
              col += tot[u];
            }
            // the values are read after the gathers are issued: fewer registers live across the scan
#pragma unroll
            for (int u = 0; u < UNR; ++u) xv[u] = (jb + u * LPR + sl < jend) ? ldg(x + c[u]) : S(0);
#pragma unroll
            for (int u = 0; u < UNR; ++u) av[u] = (jb + u * LPR + sl < jend) ? sv[jb + u * LPR + sl] : S(0);
#pragma unroll
            for (int u = 0; u < UNR; ++u) sum += av[u] * xv[u];
          }
        } else {
          // UNR predicated entries per lane per pass: all gathers of a row (<= UNR*LPR entries) are
          // in flight together -- one memory latency per row instead of one per remainder step.  PAT: the column of the
          // row's entry k is col + dict[pb + k]; the rows of a warp mostly share a pattern, so the dictionary reads are
          // mostly broadcasts
          const int db = pb - (rs - s_al);
          for (int j0 = rs + sl - s_al; j0 < jend; j0 += UNR * LPR) {
            int c[UNR];
            S av[UNR], xv[UNR];
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
              const int j = j0 + u * LPR;
              const bool ok = j < jend;
              if constexpr (PAT) c[u] = ok ? col + sdict[db + j] : 0;
              else c[u] = ok ? sc[j] : 0;
              av[u] = ok ? sv[j] : S(0);
            }
#pragma unroll
            for (int u = 0; u < UNR; ++u) xv[u] = (j0 + u * LPR < jend) ? ldg(x + c[u]) : S(0);
#pragma unroll
            for (int u = 0; u < UNR; ++u) sum += av[u] * xv[u];
          }
        }
        sum = subwarp_sum<LPR>(sum);
        if (valid && !is_long && sl == 0) store_y(y, r, sum, alpha, beta, ex);
      }
      tile_ring_release(sm, stage, lane);
    }
  }
}

// ---------------------------------------------------------------------------
// plan
// ---------------------------------------------------------------------------
struct TileCfg {
  int cap, stages, nw;
};
static const TileCfg kCfgs[] = {
    {2048, 4, 8},   // 0: 100 KB / CTA (f64) -> 2 CTAs per SM
    {4096, 4, 16},  // 1: 200 KB / CTA -> 1 CTA per SM
    {4096, 3, 8},   // 2: 150 KB
    {1024, 6, 8},   // 3:  75 KB -> 3 CTAs per SM
    {2048, 3, 16},  // 4:  84 KB -> 2 CTAs per SM
    {2048, 3, 24},  // 5
    {2048, 3, 31},  // 6: 1024 threads, 2 CTAs per SM = 64 warps
    {1024, 5, 16},  // 7:  70 KB -> 3 CTAs per SM
    {2048, 4, 16},  // 8: 112 KB -> 2 CTAs per SM
    {2048, 3, 16},  // 9: as 4 with UNR=4
    {4096, 3, 31},  // 10: 168 KB, 1 CTA per SM, 32 warps
};
static constexpr int kNumCfgs = sizeof(kCfgs) / sizeof(kCfgs[0]);

// ---------------------------------------------------------------------------
// Push a finished piece of y to the NVSwitch multicast mapping of the next-x buffer with 16-byte stores
// (on sm_90, as the SASS of this kernel shows, multimem.st to a multicast address is a plain STG: the switch replicates
// it into every GPU's copy, so store_y and the forwarding kernel write the multicast mapping with plain stores).  A few CTAs are enough (80 MB per step); they co-reside with the persistent SpMV CTAs.
// ---------------------------------------------------------------------------
// 16-byte store to a multicast address: multimem.st (the switch writes the value into every GPU's copy)
__device__ __forceinline__ void mc_store16(double2* dst, const double2& v) {
#ifdef B200SP_EMU
  *dst = v;
#else
  asm volatile("multimem.st.weak.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "r"(__double2loint(v.x)),
               "r"(__double2hiint(v.x)), "r"(__double2loint(v.y)), "r"(__double2hiint(v.y))
               : "memory");
#endif
}
__device__ __forceinline__ void mc_store8(double* dst, double v) {
#ifdef B200SP_EMU
  *dst = v;
#else
  asm volatile("multimem.st.weak.global.v2.f32 [%0], {%1, %2};" ::"l"(dst), "r"(__double2loint(v)), "r"(__double2hiint(v))
               : "memory");
#endif
}

// MC = true: dst is the multicast mapping (multimem.st); false: a plain store (also used for a peer's unicast mapping)
template <bool MC>
__global__ void __launch_bounds__(128, 16) multicast_push_kernel(const double* __restrict__ src, double* __restrict__ dst, int64_t n) {
  // head: up to one element so that both pointers are 16-byte aligned (they share their 8-byte phase)
  int64_t head = (((uintptr_t)dst & 15u) != 0 && n > 0) ? 1 : 0;
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
  if (head && tid == 0) {
    if (MC) mc_store8(dst, src[0]); else dst[0] = src[0];
  }
  const int64_t n2 = (n - head) >> 1;
  const double2* s2 = reinterpret_cast<const double2*>(src + head);
  double2* d2 = reinterpret_cast<double2*>(dst + head);
  int64_t i = tid;
#pragma unroll 1
  for (; i + 3 * nthreads < n2; i += 4 * nthreads) {  // 4 independent 16-byte loads in flight per thread
    const double2 a = s2[i], b = s2[i + nthreads], c = s2[i + 2 * nthreads], d = s2[i + 3 * nthreads];
    if (MC) {
      mc_store16(d2 + i, a); mc_store16(d2 + i + nthreads, b); mc_store16(d2 + i + 2 * nthreads, c); mc_store16(d2 + i + 3 * nthreads, d);
    } else {
      d2[i] = a; d2[i + nthreads] = b; d2[i + 2 * nthreads] = c; d2[i + 3 * nthreads] = d;
    }
  }
#pragma unroll 1
  for (; i < n2; i += nthreads) {
    const double2 a = s2[i];
    if (MC) mc_store16(d2 + i, a); else d2[i] = a;
  }
  if (((n - head) & 1) && tid == 0) {
    if (MC) mc_store8(dst + n - 1, src[n - 1]); else dst[n - 1] = src[n - 1];
  }
}

// SM-driven unicast push: every 16 bytes of src are read once and stored to the same offset of n_dst peer buffers
// (P2P stores over NVLink).  src and all destinations share their 16-byte phase.
struct PeerDsts {
  double* p[8];
  int n;
};
__global__ void __launch_bounds__(128, 16) peer_push_sm_kernel(const double* __restrict__ src, PeerDsts dsts, int64_t n) {
  const int64_t head = (((uintptr_t)src & 15u) != 0 && n > 0) ? 1 : 0;
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
  if (head && tid == 0)
    for (int d = 0; d < dsts.n; ++d) dsts.p[d][0] = src[0];
  const int64_t n2 = (n - head) >> 1;
  const double2* s2 = reinterpret_cast<const double2*>(src + head);
  int64_t i = tid;
#pragma unroll 1
  for (; i + nthreads < n2; i += 2 * nthreads) {
    const double2 a = s2[i], b = s2[i + nthreads];
#pragma unroll
    for (int d = 0; d < 8; ++d)
      if (d < dsts.n) {
        double2* q = reinterpret_cast<double2*>(dsts.p[d] + head);
        q[i] = a;
        q[i + nthreads] = b;
      }
  }
#pragma unroll 1
  for (; i < n2; i += nthreads) {
    const double2 a = s2[i];
#pragma unroll
    for (int d = 0; d < 8; ++d)
      if (d < dsts.n) reinterpret_cast<double2*>(dsts.p[d] + head)[i] = a;
  }
  if (((n - head) & 1) && tid == 0)
    for (int d = 0; d < dsts.n; ++d) dsts.p[d][n - 1] = src[n - 1];
}

}  // namespace b200sp

using namespace b200sp;

namespace b200sp {

// what plan_analyse builds and b200sp_spmv_plan_invalidate drops: the tiles, the column forms and the long-row segments
static void plan_reset_analysis(b200sp_spmv_plan* p, cudaStream_t st) {
  p->r1.reset(st);
  p->cols.reset(st);
  p->segs.release(st);
}

template <typename S>
static int plan_analyse(b200sp_spmv_plan* p, cudaStream_t st, int cfg, int m, int n, int64_t nnz,
                        const int* row_ptr) {
  const PlanKey key{row_ptr, nullptr, m, n, nnz, cfg};
  if (p->r1.key == key) return B200SP_OK;
  plan_reset_analysis(p, st);
  const TileCfg c = kCfgs[cfg];
  TileAnalysis a;
  const int rc = tile_analyse(st, m, nnz, row_ptr, c.cap, c.cap / 4, &a);
  p->r1.a = std::move(a);
  p->r1.cut = ++p->cuts;
  if (rc != B200SP_OK) return rc;
  if (int rc2 = p->r1.n_long.fetch(p->r1.a.n_long, 1, st)) return rc2;
  p->r1.key = key;
  p->at.reset();
  return B200SP_OK;
}

// The 16-bit column forms of the analysed matrix (after plan_analyse): built once per col_idx, stream-ordered.  The verdicts
// (deltas: every in-row delta of the rows <= LMAX within [0, 65535]; patterns: every such row matches the dictionary, which
// holds at most DCAP offsets) reach the host together through a pinned mirror and an event.  The pattern form wins when the
// matrix qualifies for both.  A matrix that qualifies for neither, or whose streams do not fit in device memory, keeps the
// 32-bit columns: the call does not fail.  B200SP_SPMV_PATTERN=0 at the build leaves out the pattern analysis.
static int plan_idx16(b200sp_spmv_plan* p, cudaStream_t st, int m, int64_t nnz, const int* row_ptr, const int* col_idx) {
  SpmvCols& c = p->cols;
  const int LMAX = p->r1.a.LMAX;
  // the deltas of a pattern-form matrix go on the call after the one that learnt the verdict: a call never frees the streams
  // it has built, so what a handle holds after its first call does not depend on how soon the verdict arrived
  if (c.state == COLS_PAT) c.d.release(st);
  if (c.key_ci != col_idx) {
    c.release_streams(st);
    c.key_ci = col_idx;
    c.state = COLS_I32;
    const char* pe = getenv("B200SP_SPMV_PATTERN");
    const bool pat = !(pe && pe[0] == '0');
    const size_t nd = ((size_t)nnz + 7) & ~(size_t)7, na = ((size_t)m + 3) & ~(size_t)3, np = ((size_t)m + 7) & ~(size_t)7;
    // hash table, slot representatives, slot starts, slot lengths, row slots: freed once the pattern passes are issued
    const size_t scratch = sizeof(unsigned long long) * PAT_SLOTS + sizeof(int) * (3 * (size_t)PAT_SLOTS + (size_t)m);
    unsigned long long* table = nullptr;
    if (c.d.alloc(nd, st) != cudaSuccess || c.anchor.alloc(na, st) != cudaSuccess || c.bad.alloc(2, st) != cudaSuccess ||
        (pat && (c.pid.alloc(np, st) != cudaSuccess || c.dict.alloc(DCAP + 1, st) != cudaSuccess ||
                 cudaMallocAsync((void**)&table, scratch, st) != cudaSuccess))) {
      (void)cudaGetLastError();  // not an error of the call: it runs on the 32-bit columns
      if (table) cudaFreeAsync(table, st);
      c.release_streams(st);
      return B200SP_OK;
    }
    B200SP_CUDA_TRY(cudaMemsetAsync(c.d + nnz, 0, sizeof(uint16_t) * (nd - (size_t)nnz), st));
    B200SP_CUDA_TRY(cudaMemsetAsync(c.anchor + m, 0, sizeof(int) * (na - (size_t)m), st));
    B200SP_CUDA_TRY(cudaMemsetAsync(c.bad, 0, 2 * sizeof(int), st));
    const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>(((int64_t)m + 31) / 32, (int64_t)sm_count() * 16));
    build_idx16_kernel<<<blocks, 256, 0, st>>>(m, row_ptr, col_idx, LMAX, c.d, c.anchor, c.bad);
    B200SP_LAUNCH_CHECK();
    if (pat) {
      int* rep = reinterpret_cast<int*>(table + PAT_SLOTS);
      int* slot_start = rep + PAT_SLOTS;
      int* slot_len = slot_start + PAT_SLOTS;
      int* row_slot = slot_len + PAT_SLOTS;
      B200SP_CUDA_TRY(cudaMemsetAsync(table, 0, sizeof(unsigned long long) * PAT_SLOTS, st));
      B200SP_CUDA_TRY(cudaMemsetAsync(c.pid + m, 0, sizeof(uint16_t) * (np - (size_t)m), st));
      pattern_hash_kernel<<<blocks, 256, 0, st>>>(m, row_ptr, col_idx, LMAX, table, rep, row_slot, c.bad + 1);
      B200SP_LAUNCH_CHECK();
      pattern_dict_kernel<<<1, 256, 0, st>>>(row_ptr, col_idx, table, rep, slot_start, slot_len, c.dict, c.bad + 1);
      B200SP_LAUNCH_CHECK();
      pattern_assign_kernel<<<blocks, 256, 0, st>>>(m, row_ptr, col_idx, LMAX, row_slot, slot_start, slot_len, c.dict, c.pid,
                                                    c.bad + 1);
      B200SP_LAUNCH_CHECK();
      cudaFreeAsync(table, st);
    }
    if (int rc = c.verdict.fetch(c.bad, 2, st)) return rc;
    c.state = -1;
  }
  if (c.state < 0 && c.verdict.ready()) {
    const int* bad = c.verdict.h;
    c.state = (c.pid && bad[1] == 0) ? COLS_PAT : bad[0] == 0 ? COLS_DELTA : COLS_I32;
    if (c.state == COLS_PAT) {
      // the pattern form's own tiles, for its larger stages, ahead of its first launch; its long rows are the cfg's (same
      // LMAX), so the cut's copy of them is dropped.  A table that cannot be built leaves the matrix on the deltas.
      TileAnalysis a;
      const int rc = tile_analyse(st, m, nnz, row_ptr, PAT_TILE_CAP, LMAX, &a);
      a.release_long_rows(st);
      c.pat = std::move(a);
      c.pat_cut = ++p->cuts;
      if (rc != B200SP_OK) {
        (void)cudaGetLastError();
        c.pat.release(st);
        c.state = COLS_DELTA;
      }
    }
    if (c.state == COLS_I32) c.release_streams(st);  // the key stays: not built again for this matrix
    if (c.state == COLS_DELTA) {
      c.pid.release(st);
      c.dict.release(st);
    }
  }
  return B200SP_OK;
}

// The column form of the next tiled launch (p->cols.launch), and so its tile table (plan_tiles).
// B200SP_SPMV_IDX16=0: the 32-bit columns (A/B comparisons; the 16-bit streams are not built for this call).
static int plan_cols(b200sp_spmv_plan* p, cudaStream_t st, int cfg, int m, int64_t nnz, const int* row_ptr, const int* col_idx) {
  const char* i16 = getenv("B200SP_SPMV_IDX16");
  p->cols.launch = COLS_I32;
  if (!(i16 && i16[0] == '0')) {
    const int rc = plan_idx16(p, st, m, nnz, row_ptr, col_idx);
    if (rc) return rc;
    if (p->cols.state > 0) p->cols.launch = p->cols.state;
  }
  // one tile table at a time: the pattern form's while it runs, else the cfg's, cut again when a call goes back to them
  TileAnalysis& a = p->r1.a;
  if (p->cols.launch == COLS_PAT) {
    a.tiles.release(st);
    a.n_tiles = 0;
  } else if (!a.tiles) {
    TileAnalysis cut;
    const int rc = tile_analyse(st, m, nnz, row_ptr, kCfgs[cfg].cap, a.LMAX, &cut);
    cut.release_long_rows(st);  // the analysis keeps the list its segments were built from
    a.tiles = std::move(cut.tiles);
    a.n_tiles = cut.n_tiles;
    p->r1.cut = ++p->cuts;
    if (rc != B200SP_OK) return rc;
  }
  return B200SP_OK;
}

static const TileAnalysis& plan_tiles(const b200sp_spmv_plan* p) { return p->cols.launch == COLS_PAT ? p->cols.pat : p->r1.a; }

int spmv_lanes_per_row(int64_t m, int64_t nnz);
static int pick_lpr(int m, int64_t nnz) { return spmv_lanes_per_row(m, nnz); }
int spmv_lanes_per_row(int64_t m, int64_t nnz) {  // also used by spmv64.cu: one choice for all windows of a matrix
  const double avg = m > 0 ? (double)nnz / (double)m : 0.0;
  // tuned by tools/tune_spmv.py: fewer lanes per row win until rows get long
  if (avg <= 8.0) return 2;
  if (avg <= 96.0) return 4;
  if (avg <= 384.0) return 8;
  if (avg <= 1536.0) return 16;
  return 32;
}

// STAGES and CAP are the cfg's; the pattern form runs its own layout (PAT_STAGES stages of PAT_CAP) on the plan's pattern
// tiles, and reports it after the cfg's label
template <typename S, int LPR, int NW, int STAGES, int CAP, int UNR, int COLS>
static int launch_tile_form(b200sp_spmv_plan* p, cudaStream_t st, int m, int64_t nnz, const int* row_ptr,
                            const int* col_idx, const S* vals, const S* x, S* y, S alpha, S beta) {
  constexpr bool PAT = COLS == COLS_PAT;
  constexpr int KSTAGES = PAT ? PAT_STAGES : STAGES, KCAP = PAT ? PAT_CAP : CAP;
  using Smem = TileSmem<S, KCAP, KSTAGES, COLS>;
  auto kern = spmv_tile_kernel<S, LPR, NW, KSTAGES, KCAP, UNR, COLS, false>;
  const uint16_t* c16 = PAT ? p->cols.pid : p->cols.d;
  const int* anchor = p->cols.anchor;
  const int* dict = p->cols.dict;
  const int n_tiles = plan_tiles(p).n_tiles;
  const int4* tiles = plan_tiles(p).tiles;
  const size_t smem = sizeof(Smem) + tile_smem_extra<COLS>() + 128;
  static KernelSetup ks;
  int occ_dev = 1;
  if (int rc = kernel_setup(ks, kern, (NW + 1) * 32, smem, &occ_dev)) return rc;
  int per_sm = p->ctas_per_sm;
  if (per_sm <= 0) per_sm = occ_dev;
  const int lo = p->range_hi < 0 ? 0 : p->range_lo;
  const int hi = p->range_hi < 0 ? n_tiles : p->range_hi;
  int grid = std::min(hi - lo, sm_count() * per_sm);
  if (grid < 1) grid = 1;
  bool launched = false;
  if constexpr (sizeof(S) == 8 && NW == 16 && STAGES == 4 && CAP == 2048 && UNR == 8) {
    // the forwarding form exists for the default configuration; elsewhere the consumers store to the destination themselves
    if (p->extra.n < 0) {
      auto kf = spmv_tile_kernel<S, LPR, NW, KSTAGES, KCAP, UNR, COLS, true>;
      static KernelSetup ksf;
      int occ_f = 1;
      if (int rc = kernel_setup(ksf, kf, (NW + 1) * 32, smem, &occ_f)) return rc;
      kf<<<grid, (NW + 1) * 32, smem, st>>>(m, nnz, hi - lo, p->r1.a.LMAX, tiles + lo, row_ptr, col_idx, c16, anchor, dict, vals, x,
                                            y, alpha, beta, p->extra);
      launched = true;
    }
  }
  if (!launched)
    kern<<<grid, (NW + 1) * 32, smem, st>>>(m, nnz, hi - lo, p->r1.a.LMAX, tiles + lo, row_ptr, col_idx, c16, anchor, dict, vals, x,
                                            y, alpha, beta, direct_extra(p->extra));
  B200SP_LAUNCH_CHECK();
  // the pattern form is a sub-form of the 16-bit column data (pattern starts + anchors): IDX=u16, and COLS names the source
  static const char* const kColsLabel[] = {"IDX=i32", "IDX=u16,COLS=delta", "IDX=u16,COLS=pat"};
  char layout[48] = "";
  if (PAT) snprintf(layout, sizeof(layout), "pat<STAGES=%d,CAP=%d,RCAP=%d>", KSTAGES, KCAP, PAT_RCAP);
  snprintf(p->last_kernel, sizeof(p->last_kernel), "tile<%s,LPR=%d,NW=%d,STAGES=%d,CAP=%d,UNR=%d,%s>%sgrid=%d",
           sizeof(S) == 8 ? "f64" : "f32", LPR, NW, STAGES, CAP, UNR, kColsLabel[COLS], layout, grid);
  return B200SP_OK;
}

template <typename S, int LPR, int NW, int STAGES, int CAP, int UNR = 8>
static int launch_tile(b200sp_spmv_plan* p, cudaStream_t st, int m, int64_t nnz, const int* row_ptr,
                       const int* col_idx, const S* vals, const S* x, S* y, S alpha, S beta) {
  if (p->cols.launch == COLS_PAT)
    return launch_tile_form<S, LPR, NW, STAGES, CAP, UNR, COLS_PAT>(p, st, m, nnz, row_ptr, col_idx, vals, x, y, alpha, beta);
  if (p->cols.launch == COLS_DELTA)
    return launch_tile_form<S, LPR, NW, STAGES, CAP, UNR, COLS_DELTA>(p, st, m, nnz, row_ptr, col_idx, vals, x, y, alpha, beta);
  return launch_tile_form<S, LPR, NW, STAGES, CAP, UNR, COLS_I32>(p, st, m, nnz, row_ptr, col_idx, vals, x, y, alpha, beta);
}

template <typename S, int LPR>
static int launch_tile_cfg(b200sp_spmv_plan* p, int cfg, cudaStream_t st, int m, int64_t nnz,
                           const int* row_ptr, const int* col_idx, const S* vals, const S* x, S* y,
                           S alpha, S beta) {
  switch (cfg) {
    case 0: return launch_tile<S, LPR, 8, 4, 2048>(p, st, m, nnz, row_ptr, col_idx, vals, x, y, alpha, beta);
    case 1: return launch_tile<S, LPR, 16, 4, 4096>(p, st, m, nnz, row_ptr, col_idx, vals, x, y, alpha, beta);
    case 2: return launch_tile<S, LPR, 8, 3, 4096>(p, st, m, nnz, row_ptr, col_idx, vals, x, y, alpha, beta);
    case 3: return launch_tile<S, LPR, 8, 6, 1024>(p, st, m, nnz, row_ptr, col_idx, vals, x, y, alpha, beta);
    case 4: return launch_tile<S, LPR, 16, 3, 2048>(p, st, m, nnz, row_ptr, col_idx, vals, x, y, alpha, beta);
    case 5: return launch_tile<S, LPR, 24, 3, 2048>(p, st, m, nnz, row_ptr, col_idx, vals, x, y, alpha, beta);
    case 6: return launch_tile<S, LPR, 31, 3, 2048>(p, st, m, nnz, row_ptr, col_idx, vals, x, y, alpha, beta);
    case 7: return launch_tile<S, LPR, 16, 5, 1024>(p, st, m, nnz, row_ptr, col_idx, vals, x, y, alpha, beta);
    case 8: return launch_tile<S, LPR, 16, 4, 2048>(p, st, m, nnz, row_ptr, col_idx, vals, x, y, alpha, beta);
    case 9: return launch_tile<S, LPR, 16, 3, 2048, 4>(p, st, m, nnz, row_ptr, col_idx, vals, x, y, alpha, beta);
    case 10: return launch_tile<S, LPR, 31, 3, 4096>(p, st, m, nnz, row_ptr, col_idx, vals, x, y, alpha, beta);
  }
  set_error("bad tile cfg %d", cfg);
  return B200SP_ERR_INVALID_ARGUMENT;
}

template <typename S>
static int launch_vector(b200sp_spmv_plan* p, cudaStream_t st, int lpr, int m, const int* row_ptr,
                         const int* col_idx, const S* vals, const S* x, S* y, S alpha, S beta, int lmax = INT32_MAX) {
  const int rpw = 32 / lpr;
  const int64_t warps = ((int64_t)m + rpw - 1) / rpw;
  int blocks = (int)std::min<int64_t>((warps + 7) / 8, (int64_t)sm_count() * 16);
  if (blocks < 1) blocks = 1;
  YExtra ex = {{nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr}, 0};
  if (p) ex = direct_extra(p->extra);
#define B200SP_VEC(L)                                                                              \
  case L:                                                                                          \
    spmv_vector_kernel<S, L><<<blocks, 256, 0, st>>>(m, row_ptr, col_idx, vals, x, y, alpha, beta, ex, lmax); \
    break;
  switch (lpr) {
    B200SP_VEC(2)
    B200SP_VEC(4)
    B200SP_VEC(8)
    B200SP_VEC(16)
    B200SP_VEC(32)
    default: set_error("bad lanes-per-row %d", lpr); return B200SP_ERR_INVALID_ARGUMENT;
  }
#undef B200SP_VEC
  B200SP_LAUNCH_CHECK();
  if (p) snprintf(p->last_kernel, sizeof(p->last_kernel), "vector<%s,LPR=%d>grid=%d", sizeof(S) == 8 ? "f64" : "f32", lpr, blocks);
  return B200SP_OK;
}

// crs_utils.cu
int transpose_structure(cudaStream_t st, int m, int n, int64_t nnz, const int* rp, const int* ci, int* trp, int* tci,
                        int* t_src);
template <typename S>
int gather_values(cudaStream_t st, int64_t nnz, const int* t_src, const S* v, S* tv);

template <typename S>
static int spmv_impl(b200sp_spmv_plan* p, cudaStream_t st, char mode, int m, int n, int64_t nnz, S alpha,
                     const int* row_ptr, const int* col_idx, const S* vals, const S* x, S beta, S* y);

// y = beta*y + alpha*A^T*x through an explicit A^T kept in the plan: the transposed product becomes the
// gather kernel's (deterministic, no atomics).  The structure is built once per matrix (synchronises the
// stream), the values are re-gathered on every call.
template <typename S>
static int spmv_cached_transpose(b200sp_spmv_plan* p, cudaStream_t st, int m, int n, int64_t nnz, S alpha,
                                 const int* row_ptr, const int* col_idx, const S* vals, const S* x, S beta, S* y) {
  SpmvTranspose& t = p->t;
  const PlanKey key{row_ptr, col_idx, m, n, nnz};
  if (t.key != key) {
    t.key = PlanKey();
    B200SP_CUDA_TRY(t.rp.alloc((size_t)n + 1, st));
    B200SP_CUDA_TRY(t.ci.alloc((size_t)nnz, st));
    B200SP_CUDA_TRY(t.src.alloc((size_t)nnz, st));
    int rc = transpose_structure(st, m, n, nnz, row_ptr, col_idx, t.rp, t.ci, t.src);
    if (rc) return rc;
    t.key = key;
    if (!t.plan) {
      rc = b200sp_spmv_plan_create(&t.plan, p->algo);
      if (rc) return rc;
      t.plan->cfg = p->cfg;
      t.plan->ctas_per_sm = p->ctas_per_sm;
    }
  }
  B200SP_CUDA_TRY(t.vals.grow(sizeof(S) * (size_t)nnz, st));
  int rc = gather_values<S>(st, nnz, t.src, vals, t.vals.as<S>());
  if (rc) return rc;
  rc = spmv_impl<S>(t.plan, st, 'N', n, m, nnz, alpha, t.rp, t.ci, t.vals.as<S>(), x, beta, y);
  if (rc) return rc;
  snprintf(p->last_kernel, sizeof(p->last_kernel), "cached_transpose+%.70s", t.plan->last_kernel);
  return B200SP_OK;
}

template <typename S>
static int spmv_impl(b200sp_spmv_plan* p, cudaStream_t st, char mode, int m, int n, int64_t nnz, S alpha,
                     const int* row_ptr, const int* col_idx, const S* vals, const S* x, S beta, S* y) {
  B200SP_REQUIRE(m >= 0 && n >= 0 && nnz >= 0, "spmv: negative dimension (m=%d n=%d nnz=%lld)", m, n,
                 (long long)nnz);
  B200SP_REQUIRE(nnz <= INT32_MAX, "spmv: nnz=%lld exceeds int32 offsets", (long long)nnz);
  bool trans;
  switch (mode) {
    case 'N': case 'n': case 'C': case 'c': trans = false; break;
    case 'T': case 't': case 'H': case 'h': trans = true; break;
    default:
      // same condition the reference throws on (spmv_impl.hpp:537-541)
      set_error("Invalid transpose mode %c for KokkosSparse::spmv()", mode);
      return B200SP_ERR_INVALID_ARGUMENT;
  }
  const int ylen = trans ? n : m;
  // alpha*op(A) == 0: y = beta*y  (KokkosSparse_spmv.hpp:145-154)
  if (alpha == S(0) || m == 0 || n == 0 || nnz == 0) {
    if (ylen > 0) B200SP_REQUIRE(y != nullptr, "spmv: y is null");
    if (p) snprintf(p->last_kernel, sizeof(p->last_kernel), "scale");
    return launch_scale<S>(st, ylen, beta, y);
  }
  B200SP_REQUIRE(row_ptr && col_idx && vals && x && y, "spmv: null pointer argument");

  const int lpr_auto = pick_lpr(m, nnz);
  if (trans && p && p->cache_transpose)
    return spmv_cached_transpose<S>(p, st, m, n, nnz, alpha, row_ptr, col_idx, vals, x, beta, y);
  if (trans) {
    int rc = launch_scale<S>(st, ylen, beta, y);
    if (rc) return rc;
    const int lpr = lpr_auto;
    const int rpw = 32 / lpr;
    const int64_t warps = ((int64_t)m + rpw - 1) / rpw;
    int blocks = (int)std::min<int64_t>((warps + 7) / 8, (int64_t)sm_count() * 16);
    if (blocks < 1) blocks = 1;
    switch (lpr) {
      case 2: spmv_transpose_kernel<S, 2><<<blocks, 256, 0, st>>>(m, row_ptr, col_idx, vals, x, y, alpha); break;
      case 4: spmv_transpose_kernel<S, 4><<<blocks, 256, 0, st>>>(m, row_ptr, col_idx, vals, x, y, alpha); break;
      case 8: spmv_transpose_kernel<S, 8><<<blocks, 256, 0, st>>>(m, row_ptr, col_idx, vals, x, y, alpha); break;
      case 16: spmv_transpose_kernel<S, 16><<<blocks, 256, 0, st>>>(m, row_ptr, col_idx, vals, x, y, alpha); break;
      default: spmv_transpose_kernel<S, 32><<<blocks, 256, 0, st>>>(m, row_ptr, col_idx, vals, x, y, alpha); break;
    }
    B200SP_LAUNCH_CHECK();
    if (p) snprintf(p->last_kernel, sizeof(p->last_kernel), "transpose<%s,LPR=%d>", sizeof(S) == 8 ? "f64" : "f32", lpr);
    return B200SP_OK;
  }

  const bool aligned = (((uintptr_t)vals | (uintptr_t)col_idx | (uintptr_t)row_ptr) & 15u) == 0;
  const bool use_tile = p && p->algo != B200SP_SPMV_FAST_SETUP && aligned &&
                        (nnz >= 32768 || p->cfg >= 0);
  if (!use_tile) return launch_vector<S>(p, st, (p && p->lpr > 0) ? p->lpr : lpr_auto, m, row_ptr, col_idx, vals, x, y, alpha, beta);

  const int cfg = p->cfg >= 0 ? p->cfg : 8;  // CAP=2048, 4 stages, 16 consumer warps, 2 CTAs/SM
  int rc = plan_analyse<S>(p, st, cfg, m, n, nnz, row_ptr);
  if (rc) return rc;
  // a piece of the host-vector pipeline runs the form its call settled on, with the tiles its bounds were cut from
  if (p->range_hi < 0) {
    rc = plan_cols(p, st, cfg, m, nnz, row_ptr, col_idx);
    if (rc) return rc;
  }
  const int lpr = p->lpr > 0 ? p->lpr : lpr_auto;
  // ---- self-tuning (only for untuned plans on whole-matrix launches)
  const bool autotune = p->cfg < 0 && p->range_hi < 0 && p->extra.n == 0 && getenv("B200SP_NO_AUTOTUNE") == nullptr;
  int phase = -1;  // 1: time the tiled kernel, 2: time the vector kernel
  bool use_vec = false;
  if (autotune) {
    SpmvTuning& at = p->at;
    if (at.choice < 0 && at.calls >= 3 && cudaEventQuery(at.ev[1]) == cudaSuccess && cudaEventQuery(at.ev[3]) == cudaSuccess) {
      if (cudaEventElapsedTime(&at.tile_ms, at.ev[0], at.ev[1]) == cudaSuccess &&
          cudaEventElapsedTime(&at.vec_ms, at.ev[2], at.ev[3]) == cudaSuccess)
        at.choice = (at.vec_ms < 0.9f * at.tile_ms) ? 1 : 0;
    }
    if (at.calls == 1 || at.calls == 2) {
      phase = at.calls;
      for (int i = 0; i < 4; ++i)
        if (!at.ev[i]) B200SP_CUDA_TRY(cudaEventCreate(&at.ev[i]));
    }
    at.calls++;
    use_vec = phase == 2 || (phase < 0 && at.choice == 1);
    if (phase > 0) B200SP_CUDA_TRY(cudaEventRecord(at.ev[phase == 1 ? 0 : 2], st));
  }
  if (use_vec) {
    // same split as the tiled kernel: rows beyond LMAX go to the long-row kernel below, so the choice never changes a bit
    rc = launch_vector<S>(p, st, lpr, m, row_ptr, col_idx, vals, x, y, alpha, beta, p->r1.a.LMAX);
  } else {
    switch (lpr) {
      case 2: rc = launch_tile_cfg<S, 2>(p, cfg, st, m, nnz, row_ptr, col_idx, vals, x, y, alpha, beta); break;
      case 4: rc = launch_tile_cfg<S, 4>(p, cfg, st, m, nnz, row_ptr, col_idx, vals, x, y, alpha, beta); break;
      case 8: rc = launch_tile_cfg<S, 8>(p, cfg, st, m, nnz, row_ptr, col_idx, vals, x, y, alpha, beta); break;
      case 16: rc = launch_tile_cfg<S, 16>(p, cfg, st, m, nnz, row_ptr, col_idx, vals, x, y, alpha, beta); break;
      case 32: rc = launch_tile_cfg<S, 32>(p, cfg, st, m, nnz, row_ptr, col_idx, vals, x, y, alpha, beta); break;
      default: set_error("bad lanes-per-row %d", lpr); return B200SP_ERR_INVALID_ARGUMENT;
    }
  }
  if (rc) return rc;
  // long rows: skip the launch once the (asynchronously fetched) count is known to be 0
  SpmvTiles& r1 = p->r1;
  if (!r1.n_long_known && r1.n_long.ready()) r1.n_long_known = true;
  if (!(r1.n_long_known && *r1.n_long.h == 0) && (p->range_hi < 0 || p->range_lo == 0)) {
    const char* lr = getenv("B200SP_SPMV_LONGROWS");
    if (lr && lr[0] == 's') {
      constexpr int SEG = 4096;
      SpmvSegs& g = p->segs;
      const int long_cap = r1.a.long_cap;
      if (!g.built) {
        g.cap = (int)(nnz / SEG) + long_cap + 1;
        B200SP_CUDA_TRY(g.segs.alloc((size_t)g.cap, st));
        B200SP_CUDA_TRY(g.n_seg.alloc(1, st));
        B200SP_CUDA_TRY(g.row_seg.alloc((size_t)long_cap, st));
        B200SP_CUDA_TRY(g.partial.alloc(sizeof(double) * (size_t)g.cap, st));
        B200SP_CUDA_TRY(cudaMemsetAsync(g.n_seg, 0, sizeof(int), st));
        build_row_segments_kernel<<<std::max(1, std::min((long_cap + 255) / 256, sm_count() * 4)), 256, 0, st>>>(
            r1.a.long_rows, r1.a.n_long, row_ptr, SEG, g.segs, g.n_seg, g.row_seg);
        B200SP_LAUNCH_CHECK();
        g.built = true;
      }
      spmv_seg_partial_kernel<S><<<sm_count() * 4, 256, 0, st>>>(g.segs, g.n_seg, col_idx, vals, x, g.partial.as<S>());
      B200SP_LAUNCH_CHECK();
      spmv_seg_combine_kernel<S><<<std::max(1, std::min((long_cap + 255) / 256, sm_count())), 256, 0, st>>>(
          r1.a.long_rows, r1.a.n_long, g.row_seg, g.partial.as<const S>(), y, alpha, beta, direct_extra(p->extra));
      B200SP_LAUNCH_CHECK();
      snprintf(p->last_kernel + strlen(p->last_kernel), sizeof(p->last_kernel) - strlen(p->last_kernel), "+seg");
    } else {
      int blocks = r1.n_long_known ? std::min(*r1.n_long.h, sm_count() * 4) : sm_count() * 2;
      spmv_longrow_kernel<S><<<blocks, 256, 0, st>>>(r1.a.long_rows, r1.a.n_long, row_ptr, col_idx, vals, x, y, alpha, beta,
                                                     direct_extra(p->extra));
      B200SP_LAUNCH_CHECK();
    }
  }
  if (phase > 0) B200SP_CUDA_TRY(cudaEventRecord(p->at.ev[phase == 1 ? 1 : 3], st));
  return B200SP_OK;
}

}  // namespace b200sp

// ---------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------
extern "C" {

const char* b200sp_last_error_string(void) { return b200sp::g_err; }
int b200sp_version(void) { return 100; }
int64_t b200sp_launch_count(void) { return (int64_t)b200sp::g_launches.load(); }

int b200sp_device_ok(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  int major = 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
  return major == 9 ? 1 : 0;
}

int b200sp_spmv_plan_create(b200sp_spmv_plan** plan, int algo) {
  B200SP_REQUIRE(plan != nullptr, "spmv_plan_create: null output pointer");
  B200SP_REQUIRE(algo >= 0 && algo <= 2, "spmv_plan_create: unknown algorithm %d", algo);
  b200sp_spmv_plan* p = new (std::nothrow) b200sp_spmv_plan();
  if (!p) {
    set_error("spmv_plan_create: out of host memory");
    return B200SP_ERR_ALLOC;
  }
  p->algo = algo;
  *plan = p;
  return B200SP_OK;
}

int b200sp_spmv_plan_destroy(b200sp_spmv_plan* p, void* stream) {
  if (!p) return B200SP_OK;
  cudaStream_t st = (cudaStream_t)stream;
  p->r1.release(st);
  p->cols.release(st);
  p->segs.release(st);
  p->mm.release(st);
  p->t.release(st);
  p->at.release();
  p->dx.release(st);
  p->dy.release(st);
  p->pipe.release();
  delete p;
  return B200SP_OK;
}

int b200sp_spmv_plan_set_option(b200sp_spmv_plan* p, int option, int value) {
  B200SP_REQUIRE(p != nullptr, "spmv_plan_set_option: null plan");
  switch (option) {
    case B200SP_SPMV_OPT_CACHE_TRANSPOSE: p->cache_transpose = value != 0; return B200SP_OK;
    case B200SP_SPMV_OPT_HOSTVEC_DEFER:
      if (p->pipe.defer && value == 0 && p->pipe.last_b >= 0) {
        set_error("spmv_plan_set_option: downloads are outstanding, call b200sp_spmv_hostvec_flush first");
        return B200SP_ERR_STATE;
      }
      p->pipe.defer = value != 0;
      return B200SP_OK;
  }
  set_error("spmv_plan_set_option: unknown option %d", option);
  return B200SP_ERR_INVALID_ARGUMENT;
}

int b200sp_spmv_plan_invalidate(b200sp_spmv_plan* p, void* stream) {
  B200SP_REQUIRE(p != nullptr, "spmv_plan_invalidate: null plan");
  cudaStream_t st = (cudaStream_t)stream;
  // everything derived from the STRUCTURE of the matrix the plan last saw: tiles, long rows, 16-bit column stream, rank-2
  // tiles / segments / items, chunk table, cached transpose, host-vector piece bounds, self-tuning state.  Buffers that only depend on sizes stay.
  plan_reset_analysis(p, st);
  p->mm.reset(st);
  p->t.key = PlanKey();
  p->pipe.key = PlanKey();
  p->at.reset();
  if (p->t.plan) return b200sp_spmv_plan_invalidate(p->t.plan, stream);
  return B200SP_OK;
}

int b200sp_spmv_plan_tune(b200sp_spmv_plan* p, int cfg, int lanes_per_row, int ctas_per_sm) {
  B200SP_REQUIRE(p != nullptr, "spmv_plan_tune: null plan");
  B200SP_REQUIRE(cfg >= -1 && cfg < kNumCfgs, "spmv_plan_tune: cfg %d out of range", cfg);
  B200SP_REQUIRE(lanes_per_row == -1 || lanes_per_row == 2 || lanes_per_row == 4 || lanes_per_row == 8 ||
                     lanes_per_row == 16 || lanes_per_row == 32,
                 "spmv_plan_tune: lanes_per_row %d not in {2,4,8,16,32}", lanes_per_row);
  B200SP_REQUIRE(ctas_per_sm >= -1 && ctas_per_sm <= 8, "spmv_plan_tune: ctas_per_sm %d out of range", ctas_per_sm);
  p->cfg = cfg;
  p->lpr = lanes_per_row;
  p->ctas_per_sm = ctas_per_sm;
  return B200SP_OK;
}

const char* b200sp_spmv_last_kernel(const b200sp_spmv_plan* p) { return p ? p->last_kernel : "none"; }

int b200sp_spmv_f64_i32(b200sp_spmv_plan* plan, void* stream, char mode, int m, int n, int64_t nnz, double alpha,
                        const int* row_ptr, const int* col_idx, const double* vals, const double* x, double beta,
                        double* y) {
  return spmv_impl<double>(plan, (cudaStream_t)stream, mode, m, n, nnz, alpha, row_ptr, col_idx, vals, x, beta, y);
}

int b200sp_spmv_f32_i32(b200sp_spmv_plan* plan, void* stream, char mode, int m, int n, int64_t nnz, float alpha,
                        const int* row_ptr, const int* col_idx, const float* vals, const float* x, float beta,
                        float* y) {
  return spmv_impl<float>(plan, (cudaStream_t)stream, mode, m, n, nnz, alpha, row_ptr, col_idx, vals, x, beta, y);
}

int b200sp_spmv_scatter_f64_i32(b200sp_spmv_plan* p, void* stream, int m, int n, int64_t nnz, double alpha,
                                const int* row_ptr, const int* col_idx, const double* vals, const double* x,
                                double* y, int n_extra, void* const* y_extra) {
  B200SP_REQUIRE(p != nullptr, "spmv_scatter: a plan is required");
  B200SP_REQUIRE(n_extra >= 0 && n_extra <= 7, "spmv_scatter: at most 7 extra destinations (8 GPUs), got %d", n_extra);
  B200SP_REQUIRE(n_extra == 0 || y_extra != nullptr, "spmv_scatter: y_extra is null");
  if (alpha == 0.0 || m == 0 || n == 0 || nnz == 0) {
    set_error("spmv_scatter: alpha == 0 / empty matrix is not supported by the fused all-gather form");
    return B200SP_ERR_INVALID_ARGUMENT;
  }
  p->extra.n = n_extra;
  for (int d = 0; d < n_extra; ++d) p->extra.p[d] = y_extra[d];
  const int rc = spmv_impl<double>(p, (cudaStream_t)stream, 'N', m, n, nnz, alpha, row_ptr, col_idx, vals, x, 0.0, y);
  p->extra.n = 0;
  return rc;
}

int b200sp_spmv_forward_f64_i32(b200sp_spmv_plan* p, void* stream, int m, int n, int64_t nnz, double alpha,
                                const int* row_ptr, const int* col_idx, const double* vals, const double* x,
                                double* y, void* y_forward) {
  B200SP_REQUIRE(p != nullptr, "spmv_forward: a plan is required");
  B200SP_REQUIRE(y_forward != nullptr, "spmv_forward: y_forward is null");
  if (alpha == 0.0 || m == 0 || n == 0 || nnz == 0) {
    set_error("spmv_forward: alpha == 0 / empty matrix is not supported by the fused all-gather form");
    return B200SP_ERR_INVALID_ARGUMENT;
  }
  p->extra.n = -1;
  p->extra.p[0] = y_forward;
  const int rc = spmv_impl<double>(p, (cudaStream_t)stream, 'N', m, n, nnz, alpha, row_ptr, col_idx, vals, x, 0.0, y);
  p->extra.n = 0;
  return rc;
}

// event pool for the push / join helpers (events may be re-recorded once the waits on them are enqueued)
static cudaEvent_t pool_event() {
  static cudaEvent_t ev[64];
  static bool init[64];
  static std::atomic<unsigned> next{0};
  const unsigned i = next.fetch_add(1) % 64;
  if (!init[i]) {
    if (cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming) != cudaSuccess) return nullptr;
    init[i] = true;
  }
  return ev[i];
}

int b200sp_peer_push_async(void* compute_stream, void* const* comm_streams, int n_dst, void* const* dsts,
                           const void* src, int64_t bytes) {
  B200SP_REQUIRE(bytes >= 0 && n_dst >= 0 && (n_dst == 0 || (dsts && comm_streams)), "peer_push_async: bad arguments");
  if (n_dst == 0) return B200SP_OK;
  cudaEvent_t ev = pool_event();
  B200SP_REQUIRE(ev != nullptr, "peer_push_async: cannot create event");
  B200SP_CUDA_TRY(cudaEventRecord(ev, (cudaStream_t)compute_stream));
  for (int d = 0; d < n_dst; ++d) {
    B200SP_CUDA_TRY(cudaStreamWaitEvent((cudaStream_t)comm_streams[d], ev, 0));
    B200SP_CUDA_TRY(cudaMemcpyAsync(dsts[d], src, (size_t)bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)comm_streams[d]));
  }
  return B200SP_OK;
}

int b200sp_peer_join(void* compute_stream, void* const* comm_streams, int n) {
  for (int d = 0; d < n; ++d) {
    cudaEvent_t ev = pool_event();
    B200SP_REQUIRE(ev != nullptr, "peer_join: cannot create event");
    B200SP_CUDA_TRY(cudaEventRecord(ev, (cudaStream_t)comm_streams[d]));
    B200SP_CUDA_TRY(cudaStreamWaitEvent((cudaStream_t)compute_stream, ev, 0));
  }
  return B200SP_OK;
}

int b200sp_multicast_push(void* stream, const void* src, void* mc_dst, int64_t bytes, int ctas) {
  B200SP_REQUIRE(bytes >= 0 && (bytes % 8) == 0, "multicast_push: byte count must be a non-negative multiple of 8");
  B200SP_REQUIRE(bytes == 0 || (src && mc_dst), "multicast_push: null pointer");
  B200SP_REQUIRE((((uintptr_t)src ^ (uintptr_t)mc_dst) & 15u) == 0 && ((uintptr_t)src & 7u) == 0,
                 "multicast_push: source and destination must be 8-byte aligned with the same 16-byte phase");
  if (bytes == 0) return B200SP_OK;
  // ctas < 0: plain stores to the multicast mapping instead of multimem.st (|ctas| CTAs)
  const bool plain = ctas < 0;
  if (ctas < 0) ctas = -ctas;
  if (ctas == 0) ctas = 32;
  if (plain)
    multicast_push_kernel<false><<<ctas, 128, 0, (cudaStream_t)stream>>>((const double*)src, (double*)mc_dst, bytes / 8);
  else
    multicast_push_kernel<true><<<ctas, 128, 0, (cudaStream_t)stream>>>((const double*)src, (double*)mc_dst, bytes / 8);
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

int b200sp_peer_push_sm(void* stream, const void* src, int64_t bytes, int n_dst, void* const* dsts, int ctas) {
  B200SP_REQUIRE(bytes >= 0 && (bytes % 8) == 0, "peer_push_sm: byte count must be a non-negative multiple of 8");
  B200SP_REQUIRE(n_dst >= 0 && n_dst <= 8 && (n_dst == 0 || dsts != nullptr), "peer_push_sm: 0..8 destinations");
  if (bytes == 0 || n_dst == 0) return B200SP_OK;
  B200SP_REQUIRE(src != nullptr && ((uintptr_t)src & 7u) == 0, "peer_push_sm: source must be 8-byte aligned");
  PeerDsts pd;
  pd.n = n_dst;
  for (int d = 0; d < 8; ++d) pd.p[d] = d < n_dst ? (double*)dsts[d] : nullptr;
  for (int d = 0; d < n_dst; ++d)
    B200SP_REQUIRE(dsts[d] != nullptr && ((((uintptr_t)src) ^ ((uintptr_t)dsts[d])) & 15u) == 0,
                   "peer_push_sm: every destination must share the source's 16-byte phase");
  if (ctas <= 0) ctas = 32;
  peer_push_sm_kernel<<<ctas, 128, 0, (cudaStream_t)stream>>>((const double*)src, pd, bytes / 8);
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

int b200sp_peer_push(void* stream, const void* src, int64_t bytes, int n_dst, void* const* dsts) {
  B200SP_REQUIRE(bytes >= 0 && n_dst >= 0 && (n_dst == 0 || dsts != nullptr), "peer_push: bad arguments");
  for (int d = 0; d < n_dst; ++d)
    B200SP_CUDA_TRY(cudaMemcpyAsync(dsts[d], src, (size_t)bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return B200SP_OK;
}

// Host-vector SpMV.  Large non-transposed products run as a pipeline: x goes up on a copy stream into
// one of two device buffers (so the upload of call k+1 overlaps call k), the rows are computed in
// pieces (tile sub-ranges of the TMA-tiled kernel) and every finished piece of y goes down on a second
// copy stream while the next piece is computed.  x_host must be ready when the call is made (it is
// read asynchronously); y_host is valid once `stream` has been synchronised.
static int hostvec_simple(b200sp_spmv_plan* p, cudaStream_t st, char mode, int m, int n, int64_t nnz, double alpha,
                          const int* row_ptr, const int* col_idx, const double* vals, const double* x_host,
                          double beta, double* y_host, size_t xb, size_t yb) {
  B200SP_CUDA_TRY(p->dx.grow(xb, st));
  B200SP_CUDA_TRY(p->dy.grow(yb, st));
  if (xb) B200SP_CUDA_TRY(cudaMemcpyAsync(p->dx, x_host, xb, cudaMemcpyHostToDevice, st));
  if (beta != 0.0 && yb) B200SP_CUDA_TRY(cudaMemcpyAsync(p->dy, y_host, yb, cudaMemcpyHostToDevice, st));
  int rc = spmv_impl<double>(p, st, mode, m, n, nnz, alpha, row_ptr, col_idx, vals, p->dx.as<const double>(), beta,
                             p->dy.as<double>());
  if (rc) return rc;
  if (yb) B200SP_CUDA_TRY(cudaMemcpyAsync(y_host, p->dy, yb, cudaMemcpyDeviceToHost, st));
  return B200SP_OK;
}

int b200sp_spmv_hostvec_f64_i32(b200sp_spmv_plan* p, void* stream, char mode, int m, int n, int64_t nnz,
                                double alpha, const int* row_ptr, const int* col_idx, const double* vals,
                                const double* x_host, double beta, double* y_host) {
  B200SP_REQUIRE(p != nullptr, "spmv_hostvec: a plan is required");
  B200SP_REQUIRE(m >= 0 && n >= 0, "spmv_hostvec: negative dimension");
  cudaStream_t st = (cudaStream_t)stream;
  const bool trans = (mode == 'T' || mode == 't' || mode == 'H' || mode == 'h');
  const size_t xb = sizeof(double) * (size_t)(trans ? m : n);
  const size_t yb = sizeof(double) * (size_t)(trans ? n : m);
  const bool aligned = (((uintptr_t)vals | (uintptr_t)col_idx | (uintptr_t)row_ptr) & 15u) == 0;
  const bool piped = !trans && (mode == 'N' || mode == 'n' || mode == 'C' || mode == 'c') && alpha != 0.0 &&
                     nnz >= (1 << 22) && aligned && p->algo != B200SP_SPMV_FAST_SETUP && getenv("B200SP_HOSTVEC_SIMPLE") == nullptr;
  if (!piped) return hostvec_simple(p, st, mode, m, n, nnz, alpha, row_ptr, col_idx, vals, x_host, beta, y_host, xb, yb);

  auto& q = p->pipe;
  if (!q.init) {
    B200SP_CUDA_TRY(cudaStreamCreateWithFlags(&q.sH, cudaStreamNonBlocking));
    B200SP_CUDA_TRY(cudaStreamCreateWithFlags(&q.sD, cudaStreamNonBlocking));
    for (int b = 0; b < 2; ++b) {
      B200SP_CUDA_TRY(cudaEventCreateWithFlags(&q.ev_x[b], cudaEventDisableTiming));
      B200SP_CUDA_TRY(cudaEventCreateWithFlags(&q.ev_c[b], cudaEventDisableTiming));
      B200SP_CUDA_TRY(cudaEventCreateWithFlags(&q.ev_done[b], cudaEventDisableTiming));
    }
    for (int c = 0; c < 8; ++c) B200SP_CUDA_TRY(cudaEventCreateWithFlags(&q.ev_chunk[c], cudaEventDisableTiming));
    q.init = true;
  }
  if (xb > q.xb || yb > q.yb) {
    B200SP_CUDA_TRY(cudaDeviceSynchronize());
    for (int b = 0; b < 2; ++b) {
      if (q.dx[b]) cudaFree(q.dx[b]);
      if (q.dy[b]) cudaFree(q.dy[b]);
      q.dx[b] = q.dy[b] = nullptr;
      B200SP_CUDA_TRY(cudaMalloc(&q.dx[b], std::max(xb, q.xb)));
      B200SP_CUDA_TRY(cudaMalloc(&q.dy[b], std::max(yb, q.yb)));
    }
    q.xb = std::max(xb, q.xb);
    q.yb = std::max(yb, q.yb);
    q.call = 0;
  }
  // tile analysis + piece boundaries (once per matrix; the only synchronous part)
  const int cfg = p->cfg >= 0 ? p->cfg : 8;
  int rc = plan_analyse<double>(p, st, cfg, m, n, nnz, row_ptr);
  if (rc) return rc;
  // the column form is settled once per call, so that every piece launches on the table the bounds come from
  rc = plan_cols(p, st, cfg, m, nnz, row_ptr, col_idx);
  if (rc) return rc;
  const int n_tiles = plan_tiles(p).n_tiles;
  const int4* tiles = plan_tiles(p).tiles;
  // keyed on the cut that made the table this call launches on, not on its address: a new table may come back at the address
  // of the one the bounds were cut from, and the plan may hold both tables
  const uint64_t cut = p->cols.launch == COLS_PAT ? p->cols.pat_cut : p->r1.cut;
  const PlanKey key{row_ptr, nullptr, m, -1, nnz, cfg, (int64_t)cut};
  if (q.key != key) {
    q.nc = 4;  // pieces of y that go down while the next piece is computed (B200SP_HOSTVEC_PIECES: 1..8, tuning)
    if (const char* e = getenv("B200SP_HOSTVEC_PIECES")) {
      const int v = atoi(e);
      if (v >= 1 && v <= 8) q.nc = v;
    }
    int4 d[9];
    for (int c = 0; c <= q.nc; ++c) {
      q.tile_b[c] = (int)(((int64_t)n_tiles * c) / q.nc);
      if (c < q.nc) B200SP_CUDA_TRY(cudaMemcpyAsync(&d[c], tiles + q.tile_b[c], sizeof(int4), cudaMemcpyDeviceToHost, st));
    }
    B200SP_CUDA_TRY(cudaStreamSynchronize(st));
    for (int c = 0; c < q.nc; ++c) q.row_b[c] = d[c].x;  // first row of the first tile of piece c
    q.row_b[q.nc] = m;
    q.row_b[0] = 0;
    q.key = key;
  }
  const int b = (int)(q.call & 1ull);
  if (q.defer && q.call >= 2) {
    // deferred mode: nothing made `stream` wait for the download of call k-2, which reads the y buffer this call writes
    B200SP_CUDA_TRY(cudaStreamWaitEvent(st, q.ev_done[b], 0));
    if (beta != 0.0) B200SP_CUDA_TRY(cudaStreamWaitEvent(q.sH, q.ev_done[b], 0));
  }
  // upload: wait until the compute that last read this x buffer (call k-2) is done
  if (q.call >= 2) B200SP_CUDA_TRY(cudaStreamWaitEvent(q.sH, q.ev_c[b], 0));
  B200SP_CUDA_TRY(cudaMemcpyAsync(q.dx[b], x_host, xb, cudaMemcpyHostToDevice, q.sH));
  if (beta != 0.0) {
    // dy[b] was last read by the download of call k-2, which `stream` already waited for
    B200SP_CUDA_TRY(cudaMemcpyAsync(q.dy[b], y_host, yb, cudaMemcpyHostToDevice, q.sH));
  }
  B200SP_CUDA_TRY(cudaEventRecord(q.ev_x[b], q.sH));
  B200SP_CUDA_TRY(cudaStreamWaitEvent(st, q.ev_x[b], 0));
  for (int c = 0; c < q.nc; ++c) {
    p->range_lo = q.tile_b[c];
    p->range_hi = q.tile_b[c + 1];
    rc = spmv_impl<double>(p, st, mode, m, n, nnz, alpha, row_ptr, col_idx, vals, (const double*)q.dx[b], beta,
                           (double*)q.dy[b]);
    p->range_lo = 0;
    p->range_hi = -1;
    if (rc) return rc;
    B200SP_CUDA_TRY(cudaEventRecord(q.ev_chunk[c], st));
    B200SP_CUDA_TRY(cudaStreamWaitEvent(q.sD, q.ev_chunk[c], 0));
    const size_t r0 = (size_t)q.row_b[c], r1 = (size_t)q.row_b[c + 1];
    if (r1 > r0)
      B200SP_CUDA_TRY(cudaMemcpyAsync(y_host + r0, (double*)q.dy[b] + r0, sizeof(double) * (r1 - r0), cudaMemcpyDeviceToHost, q.sD));
  }
  B200SP_CUDA_TRY(cudaEventRecord(q.ev_c[b], st));
  B200SP_CUDA_TRY(cudaEventRecord(q.ev_done[b], q.sD));
  if (q.defer) {
    q.last_b = b;  // y_host is valid once b200sp_spmv_hostvec_flush has been called and `stream` synchronised
  } else {
    B200SP_CUDA_TRY(cudaStreamWaitEvent(st, q.ev_done[b], 0));  // y_host is valid once `stream` is synchronised
  }
  q.call++;
  return B200SP_OK;
}

int b200sp_spmv_hostvec_flush(b200sp_spmv_plan* p, void* stream) {
  B200SP_REQUIRE(p != nullptr, "spmv_hostvec_flush: null plan");
  auto& q = p->pipe;
  if (q.init && q.last_b >= 0) {
    // the download stream is in order: waiting for the latest download covers all earlier ones
    B200SP_CUDA_TRY(cudaStreamWaitEvent((cudaStream_t)stream, q.ev_done[q.last_b], 0));
    q.last_b = -1;
  }
  return B200SP_OK;
}

}  // extern "C"
