// crs_utils.cu -- the CrsMatrix utilities either side of the SpMV / SpGEMM hot path on H100
// (SURVEY.md section 8f): in-row sort, sort-and-merge, sparse add, transpose.
//
// Replaces the reference's Kokkos::Cuda legs
//   sort_crs_matrix / sort_crs_graph        sparse/src/KokkosSparse_SortCrs.hpp:43-120,209-270
//                                           (GPU: bitonic per thread or one bulk sort of row*ncols+col keys)
//   sort_and_merge_matrix / _graph          sparse/src/KokkosSparse_SortCrs.hpp:303-380,426-491,
//                                           sparse/impl/KokkosSparse_sort_crs_impl.hpp:130-248
//   spadd_symbolic / spadd_numeric          sparse/impl/KokkosSparse_spadd_symbolic_impl.hpp:33-512,
//                                           sparse/impl/KokkosSparse_spadd_numeric_impl.hpp:27-242
//   transpose_matrix / transpose_graph      sparse/src/KokkosSparse_Utils.hpp:245-450
// Results follow the reference's Serial path bit for bit:
//   * the sort is STABLE (the Serial path is an LSD radix sort, common/src/KokkosKernels_Sorting.hpp:301-380):
//     keys are (column << 32 | position in the row), all distinct, so any sorting network gives the
//     stable order;
//   * merged / added values are accumulated sequentially in the reference's order by one thread per row;
//   * the transpose lists every column's entries in (row, position) order like the Serial loop.
#include "common.cuh"
#include "scan.cuh"
#include <algorithm>
#include <limits.h>
#include <stdlib.h>
#include <new>

namespace b200sp {

typedef unsigned long long u64;

static constexpr int SORT_WARP_MAX = 256;   // rows up to this length: one warp, keys in shared memory
static constexpr int SORT_CTA_MAX = 4096;   // up to this length: one CTA of 256 threads

// ---------------------------------------------------------------------------
// classification: rows that are already sorted (or have <= 1 entry) are left alone; the others
// are listed by length class.  8 lanes per row.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    sort_classify_kernel(int m, const int* __restrict__ rp, const int* __restrict__ ci, const int* __restrict__ payload,
                         int* __restrict__ lists, int* __restrict__ counts) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t r = t >> 3;
  const int sl = (int)(t & 7);
  const int lane = threadIdx.x & 31;
  bool uns = false;
  int len = 0;
  if (r < m) {
    const int s = rp[r], e = rp[r + 1];
    len = e - s;
    if (payload == nullptr) {
      for (int j = s + 1 + sl; j < e; j += 8) uns |= ci[j - 1] > ci[j];
    } else {  // MODE 2: the payload is the second half of the key
      for (int j = s + 1 + sl; j < e; j += 8)
        uns |= (ci[j - 1] > ci[j]) || (ci[j - 1] == ci[j] && payload[j - 1] > payload[j]);
    }
  }
  const unsigned b = __ballot_sync(0xffffffffu, uns);
  const bool any = ((b >> (lane & ~7)) & 0xffu) != 0u;
  if (r < m && sl == 0 && any && len > 1) {
    const int cls = len <= SORT_WARP_MAX ? 0 : (len <= SORT_CTA_MAX ? 1 : 2);
    lists[(size_t)cls * m + atomicAdd(&counts[cls], 1)] = (int)r;
  }
}

// Bitonic network with every comparator ascending (first step of each merge mirrors, idx ^ (size-1)):
// +inf padding beyond n never moves, so it is not stored.  NT threads, keys k[0..n).
template <typename SyncT>
__device__ __forceinline__ void bitonic_keys(u64* k, int n, int tid, int nt, SyncT&& sync) {
  int P = 1;
  while (P < n) P <<= 1;
  for (int size = 2; size <= P; size <<= 1) {
    for (int stride = size >> 1, first = 1; stride > 0; stride >>= 1, first = 0) {
      for (int idx = tid; idx < n; idx += nt) {
        const int l = first ? (idx ^ (size - 1)) : (idx ^ stride);
        if (l > idx && l < n) {
          const u64 a = k[idx], b = k[l];
          if (a > b) {
            k[idx] = b;
            k[l] = a;
          }
        }
      }
      sync();
    }
  }
}

__device__ __forceinline__ u64 make_key(int col, int pos) {
  return ((u64)(unsigned)col << 32) | (u64)(unsigned)pos;
}

// MODE 0: column indices only; 1: values follow the stable order (gathered through the position bits of
// the key); 2: the values are non-negative int payloads that ARE the tie-break (key = column << 32 | payload)
// -- used for (row, entry id) in the transpose and for the A/B permutation of the unsorted spadd.
template <typename V, int MODE>
__device__ __forceinline__ u64 load_key(const int* __restrict__ ci, const V* __restrict__ vals, int s, int j) {
  if (MODE == 2) return make_key(ci[s + j], (int)vals[s + j]);
  return make_key(ci[s + j], j);
}

// one warp per listed row (2 <= n <= SORT_WARP_MAX)
template <typename V, int MODE>
__global__ void __launch_bounds__(256)
    sort_rows_warp_kernel(const int* __restrict__ list, const int* __restrict__ n_list_ptr, const int* __restrict__ rp,
                          int* __restrict__ ci, V* __restrict__ vals) {
  __shared__ u64 sk[8][SORT_WARP_MAX];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  u64* k = sk[warp];
  const int n_list = *n_list_ptr;
  for (int q = blockIdx.x * 8 + warp; q < n_list; q += gridDim.x * 8) {
    const int r = list[q];
    const int s = rp[r], n = rp[r + 1] - s;
    for (int j = lane; j < n; j += 32) k[j] = load_key<V, MODE>(ci, vals, s, j);
    __syncwarp();
    bitonic_keys(k, n, lane, 32, [] { __syncwarp(); });
    constexpr int U = SORT_WARP_MAX / 32;
    V tmp[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int p = lane + 32 * u;
      if (MODE == 1 && p < n) tmp[u] = vals[s + (int)(k[p] & 0xffffffffu)];
    }
    __syncwarp();  // every source value is in a register before any destination is written
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int p = lane + 32 * u;
      if (p < n) {
        const u64 key = k[p];
        ci[s + p] = (int)(key >> 32);
        if (MODE == 1) vals[s + p] = tmp[u];
        if (MODE == 2) vals[s + p] = (V)(int)(key & 0xffffffffu);
      }
    }
    __syncwarp();  // k is reused by the next row
  }
}

// one CTA (256 threads) per listed row (SORT_WARP_MAX < n <= SORT_CTA_MAX)
template <typename V, int MODE>
__global__ void __launch_bounds__(256)
    sort_rows_cta_kernel(const int* __restrict__ list, const int* __restrict__ n_list_ptr, const int* __restrict__ rp,
                         int* __restrict__ ci, V* __restrict__ vals) {
  __shared__ u64 k[SORT_CTA_MAX];
  const int n_list = *n_list_ptr;
  for (int q = blockIdx.x; q < n_list; q += gridDim.x) {
    const int r = list[q];
    const int s = rp[r], n = rp[r + 1] - s;
    for (int j = threadIdx.x; j < n; j += 256) k[j] = load_key<V, MODE>(ci, vals, s, j);
    __syncthreads();
    bitonic_keys(k, n, (int)threadIdx.x, 256, [] { __syncthreads(); });
    constexpr int U = SORT_CTA_MAX / 256;
    V tmp[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int p = threadIdx.x + 256 * u;
      if (MODE == 1 && p < n) tmp[u] = vals[s + (int)(k[p] & 0xffffffffu)];
    }
    __syncthreads();
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int p = threadIdx.x + 256 * u;
      if (p < n) {
        const u64 key = k[p];
        ci[s + p] = (int)(key >> 32);
        if (MODE == 1) vals[s + p] = tmp[u];
        if (MODE == 2) vals[s + p] = (V)(int)(key & 0xffffffffu);
      }
    }
    __syncthreads();
  }
}

// rows longer than SORT_CTA_MAX: keys (and a copy of the values) in global scratch indexed like the matrix
template <typename V, int MODE>
__global__ void __launch_bounds__(256)
    sort_rows_global_kernel(const int* __restrict__ list, const int* __restrict__ n_list_ptr, const int* __restrict__ rp,
                            int* __restrict__ ci, V* __restrict__ vals, u64* __restrict__ gkeys, V* __restrict__ gvals) {
  const int n_list = *n_list_ptr;
  for (int q = blockIdx.x; q < n_list; q += gridDim.x) {
    const int r = list[q];
    const int s = rp[r], n = rp[r + 1] - s;
    u64* k = gkeys + s;
    for (int j = threadIdx.x; j < n; j += 256) {
      k[j] = load_key<V, MODE>(ci, vals, s, j);
      if (MODE == 1) gvals[s + j] = vals[s + j];
    }
    __syncthreads();
    bitonic_keys(k, n, (int)threadIdx.x, 256, [] { __syncthreads(); });
    for (int p = threadIdx.x; p < n; p += 256) {
      const u64 key = k[p];
      ci[s + p] = (int)(key >> 32);
      if (MODE == 1) vals[s + p] = gvals[s + (int)(key & 0xffffffffu)];
      if (MODE == 2) vals[s + p] = (V)(int)(key & 0xffffffffu);
    }
    __syncthreads();
  }
}

// Sorts every row of (rp, ci[, vals]) in place.  Synchronises `st` once (class counts).
template <typename V, int MODE>
static int sort_crs_impl(cudaStream_t st, int m, const int* rp, int* ci, V* vals, int64_t nnz_hint) {
  if (m <= 0) return B200SP_OK;
  DevTmp tmp(st);
  int *lists, *counts;
  B200SP_CUDA_TRY(tmp.alloc(&lists, (size_t)3 * m));
  B200SP_CUDA_TRY(tmp.alloc(&counts, 4));
  B200SP_CUDA_TRY(cudaMemsetAsync(counts, 0, sizeof(int) * 4, st));
  sort_classify_kernel<<<(unsigned)(((int64_t)m * 8 + 255) / 256), 256, 0, st>>>(
      m, rp, ci, MODE == 2 ? reinterpret_cast<const int*>(vals) : nullptr, lists, counts);
  B200SP_LAUNCH_CHECK();
  int h[4] = {0, 0, 0, 0};
  B200SP_CUDA_TRY(cudaMemcpyAsync(h, counts, sizeof(int) * 3, cudaMemcpyDeviceToHost, st));
  B200SP_CUDA_TRY(cudaStreamSynchronize(st));
  if (h[0] > 0) {
    const int blocks = std::min((h[0] + 7) / 8, sm_count() * 8);
    sort_rows_warp_kernel<V, MODE><<<blocks, 256, 0, st>>>(lists, counts + 0, rp, ci, vals);
    B200SP_LAUNCH_CHECK();
  }
  if (h[1] > 0) {
    const int blocks = std::min(h[1], sm_count() * 4);
    sort_rows_cta_kernel<V, MODE><<<blocks, 256, 0, st>>>(lists + (size_t)m, counts + 1, rp, ci, vals);
    B200SP_LAUNCH_CHECK();
  }
  if (h[2] > 0) {
    int64_t nnz = nnz_hint;
    if (nnz < 0) {
      int last = 0;
      B200SP_CUDA_TRY(cudaMemcpyAsync(&last, rp + m, sizeof(int), cudaMemcpyDeviceToHost, st));
      B200SP_CUDA_TRY(cudaStreamSynchronize(st));
      nnz = last;
    }
    u64* gkeys;
    V* gvals = nullptr;
    B200SP_CUDA_TRY(tmp.alloc(&gkeys, (size_t)nnz));
    if (MODE == 1) B200SP_CUDA_TRY(tmp.alloc(&gvals, (size_t)nnz));
    const int blocks = std::min(h[2], sm_count() * 2);
    sort_rows_global_kernel<V, MODE><<<blocks, 256, 0, st>>>(lists + (size_t)2 * m, counts + 2, rp, ci, vals, gkeys, gvals);
    B200SP_LAUNCH_CHECK();
  }
  return B200SP_OK;
}

// ---------------------------------------------------------------------------
// sort_and_merge: unique columns per (sorted) row, then sequential accumulation per row
// (MergedRowmapFunctor / MatrixMergedEntriesFunctor, sort_crs_impl.hpp:130-205).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    merged_count_kernel(int m, const int* __restrict__ rp, const int* __restrict__ ci, int* __restrict__ counts) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t r = t >> 3;
  const int sl = (int)(t & 7);
  int u = 0;
  if (r < m) {
    const int s = rp[r], e = rp[r + 1];
    if (sl == 0 && e > s) u = 1;
    for (int j = s + 1 + sl; j < e; j += 8) u += (ci[j - 1] != ci[j]);
  }
#pragma unroll
  for (int o = 4; o > 0; o >>= 1) u += __shfl_xor_sync(0xffffffffu, u, o);
  if (r < m && sl == 0) counts[r] = u;
}

// 8 lanes per row: a lane that sits on the first entry of a run of equal columns writes that run -- its place is the number of runs
// that start before it (ballot / popc), its value the run's entries added in storage order (`acc = v[first]; acc += v[next] ...`, the
// serial loop's operations).  Runs are short (a merged matrix has none longer than one), so the lanes work side by side where one
// thread per row walked the row in a serial chain of dependent loads.
template <typename V, bool HAS_VALS>
__global__ void __launch_bounds__(256)
    merged_fill_kernel(int m, const int* __restrict__ rp, const int* __restrict__ ci, const V* __restrict__ vals,
                       const int* __restrict__ rp_out, int* __restrict__ ci_out, V* __restrict__ vals_out) {
  constexpr int G = 8;
  const int lane = (int)threadIdx.x & (G - 1);
  const int gbase = ((int)threadIdx.x & 31) & ~(G - 1);
  const unsigned gmask = ((1u << G) - 1u) << gbase;
  const unsigned below = (1u << (gbase + lane)) - 1u;
  const int groups = (int)(gridDim.x * blockDim.x) / G;
  for (int r = (int)(blockIdx.x * blockDim.x + threadIdx.x) / G; r < m; r += groups) {
    const int s = rp[r], e = rp[r + 1];
    int before = rp_out[r];  // place of the next run start
    for (int base = s; base < e; base += G) {
      const int j = base + lane;
      int col = 0;
      bool start = false;
      if (j < e) {
        col = ci[j];
        start = j == s || ci[j - 1] != col;
      }
      const unsigned sb = __ballot_sync(gmask, start);
      if (start) {
        const int pos = before + __popc(sb & below);
        ci_out[pos] = col;
        if (HAS_VALS) {
          V acc = vals[j];
          for (int q = j + 1; q < e && ci[q] == col; ++q) acc += vals[q];
          vals_out[pos] = acc;
        }
      }
      before += __popc(sb);
    }
  }
}

// counts -> offsets with the shared scan; returns the int64 total (synchronises st)
static int counts_to_offsets(cudaStream_t st, int m, const int* counts, int* offsets, long long* total_out, int* max_out) {
  DevTmp tmp(st);
  long long *block_sum, *d_total;
  int *block_max, *d_max;
  B200SP_CUDA_TRY(tmp.alloc(&block_sum, (size_t)scan_blocks(m)));
  B200SP_CUDA_TRY(tmp.alloc(&block_max, (size_t)scan_blocks(m)));
  B200SP_CUDA_TRY(tmp.alloc(&d_total, 1));
  B200SP_CUDA_TRY(tmp.alloc(&d_max, 1));
  int rc = launch_exclusive_scan(st, m, counts, offsets, block_sum, block_max, d_total, d_max);
  if (rc) return rc;
  long long total = 0;
  int mx = 0;
  B200SP_CUDA_TRY(cudaMemcpyAsync(&total, d_total, sizeof(total), cudaMemcpyDeviceToHost, st));
  B200SP_CUDA_TRY(cudaMemcpyAsync(&mx, d_max, sizeof(mx), cudaMemcpyDeviceToHost, st));
  B200SP_CUDA_TRY(cudaStreamSynchronize(st));
  if (total_out) *total_out = total;
  if (max_out) *max_out = mx;
  return B200SP_OK;
}

__global__ void fill_zero_int_kernel(int64_t n, int* __restrict__ p) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = 0;
}
static int zero_ints(cudaStream_t st, int64_t n, int* p) {
  if (n <= 0) return B200SP_OK;
  const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)sm_count() * 8));
  fill_zero_int_kernel<<<blocks, 256, 0, st>>>(n, p);
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

// ---------------------------------------------------------------------------
// spadd: C = alpha*A + beta*B  (row by row; one thread per row, the reference's operation order)
// The products are rounded before they are added (no FMA contraction), like the C expression
// `accum += alpha * a` compiled without contraction: bit-identical to the oracle for any alpha, beta.
// ---------------------------------------------------------------------------
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__global__ void __launch_bounds__(256)
    spadd_sorted_count_kernel(int m, const int* __restrict__ rpA, const int* __restrict__ ciA,
                              const int* __restrict__ rpB, const int* __restrict__ ciB, int* __restrict__ counts) {
  // SortedCountEntriesRange (spadd_symbolic_impl.hpp:33-77)
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
    int ai = rpA[i], bi = rpB[i];
    const int ae = rpA[i + 1], be = rpB[i + 1];
    int n = 0;
    int acol = ai < ae ? ciA[ai] : INT_MAX;
    int bcol = bi < be ? ciB[bi] : INT_MAX;
    while (acol != INT_MAX || bcol != INT_MAX) {
      const int c = acol < bcol ? acol : bcol;
      ++n;
      while (acol == c) acol = (++ai < ae) ? ciA[ai] : INT_MAX;
      while (bcol == c) bcol = (++bi < be) ? ciB[bi] : INT_MAX;
    }
    counts[i] = n;
  }
}

template <typename S>
__global__ void __launch_bounds__(256)
    spadd_sorted_numeric_kernel(int m, const int* __restrict__ rpA, const int* __restrict__ ciA, const S* __restrict__ vA,
                                S alpha, const int* __restrict__ rpB, const int* __restrict__ ciB,
                                const S* __restrict__ vB, S beta, const int* __restrict__ rpC, int* __restrict__ ciC,
                                S* __restrict__ vC) {
  // SortedNumericSumFunctor (spadd_numeric_impl.hpp:50-92): accum = 0; += alpha*a ...; += beta*b ...
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
    int ai = rpA[i], bi = rpB[i];
    const int ae = rpA[i + 1], be = rpB[i + 1];
    int pos = rpC[i];
    int acol = ai < ae ? ciA[ai] : INT_MAX;
    int bcol = bi < be ? ciB[bi] : INT_MAX;
    while (acol != INT_MAX || bcol != INT_MAX) {
      const int c = acol < bcol ? acol : bcol;
      S acc = S(0);
      while (acol == c) {
        acc += mul_rn(alpha, vA[ai]);
        acol = (++ai < ae) ? ciA[ai] : INT_MAX;
      }
      while (bcol == c) {
        acc += mul_rn(beta, vB[bi]);
        bcol = (++bi < be) ? ciB[bi] : INT_MAX;
      }
      ciC[pos] = c;
      vC[pos] = acc;
      ++pos;
    }
  }
}

// ---- sorted spadd by a GROUP of lanes per row -------------------------------------------------------------------------------
// One thread per row walks two sorted rows in a serial chain of dependent loads (latency-bound, far from the HBM roof).
// Rows WITHOUT a repeated column inside A_i or inside B_i (any merged matrix) need no walk: the place of an
// entry in C_i is its rank in the union,
//     pos(a_k) = k + |{b in B_i : b < a_k}| - |{j < k : a_j in B_i}|,      pos(b_k) likewise, written only when b_k is not in A_i,
// found by one binary search in the other row per entry (the rows were just read: the probes hit L1) and a ballot / popc prefix
// over the match flags.  The value is the serial loop's, operation for operation: (0 + alpha a) + beta b for a matched pair,
// 0 + alpha a or 0 + beta b otherwise (the leading 0 + keeps -0 -> +0 as `acc = 0; acc += ...` does).  A row with a repeated
// column falls back to the serial walk by lane 0 (the reference accumulates the repeats in order).
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }

__device__ __forceinline__ int row_lower_bound(const int* __restrict__ c, int len, int key) {
  int lo = 0, hi = len;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (c[mid] < key) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// true if some column repeats inside the sorted row [s, e) (uniform over the group)
template <int G>
__device__ __forceinline__ bool row_has_repeat(const int* __restrict__ ci, int s, int e, int lane, unsigned gmask) {
  bool rep = false;
  for (int base = s; base < e; base += G) {
    const int k = base + lane;
    rep |= (k < e && k > s && ci[k] == ci[k - 1]);
  }
  return __ballot_sync(gmask, rep) != 0u;
}

__device__ __forceinline__ int spadd_serial_count(const int* __restrict__ ciA, int ai, int ae, const int* __restrict__ ciB, int bi, int be) {
  int n = 0;
  int acol = ai < ae ? ciA[ai] : INT_MAX;
  int bcol = bi < be ? ciB[bi] : INT_MAX;
  while (acol != INT_MAX || bcol != INT_MAX) {
    const int c = acol < bcol ? acol : bcol;
    ++n;
    while (acol == c) acol = (++ai < ae) ? ciA[ai] : INT_MAX;
    while (bcol == c) bcol = (++bi < be) ? ciB[bi] : INT_MAX;
  }
  return n;
}

template <int G>
__global__ void __launch_bounds__(256)
    spadd_sorted_count_group_kernel(int m, const int* __restrict__ rpA, const int* __restrict__ ciA, const int* __restrict__ rpB,
                                    const int* __restrict__ ciB, int* __restrict__ counts) {
  const int lane = (int)threadIdx.x & (G - 1);
  const int gbase = ((int)threadIdx.x & 31) & ~(G - 1);
  const unsigned gmask = G == 32 ? 0xffffffffu : (((1u << (G & 31)) - 1u) << gbase);
  const int groups = (int)(gridDim.x * blockDim.x) / G;
  for (int i = (int)(blockIdx.x * blockDim.x + threadIdx.x) / G; i < m; i += groups) {
    const int as = rpA[i], ae = rpA[i + 1], bs = rpB[i], be = rpB[i + 1];
    const bool rep = row_has_repeat<G>(ciA, as, ae, lane, gmask) | row_has_repeat<G>(ciB, bs, be, lane, gmask);
    if (rep) {
      if (lane == 0) counts[i] = spadd_serial_count(ciA, as, ae, ciB, bs, be);
      continue;
    }
    int matches = 0;
    for (int base = as; base < ae; base += G) {
      const int k = base + lane;
      bool match = false;
      if (k < ae) {
        const int col = ciA[k];
        const int lb = row_lower_bound(ciB + bs, be - bs, col);
        match = lb < be - bs && ciB[bs + lb] == col;
      }
      matches += __popc(__ballot_sync(gmask, match));
    }
    if (lane == 0) counts[i] = (ae - as) + (be - bs) - matches;
  }
}

template <typename S, int G>
__global__ void __launch_bounds__(256)
    spadd_sorted_numeric_group_kernel(int m, const int* __restrict__ rpA, const int* __restrict__ ciA, const S* __restrict__ vA, S alpha,
                                      const int* __restrict__ rpB, const int* __restrict__ ciB, const S* __restrict__ vB, S beta,
                                      const int* __restrict__ rpC, int* __restrict__ ciC, S* __restrict__ vC) {
  const int lane = (int)threadIdx.x & (G - 1);
  const int gbase = ((int)threadIdx.x & 31) & ~(G - 1);
  const unsigned gmask = G == 32 ? 0xffffffffu : (((1u << (G & 31)) - 1u) << gbase);
  const unsigned below = (1u << (gbase + lane)) - 1u;  // the lanes before this one (masked with the group's ballot)
  const int groups = (int)(gridDim.x * blockDim.x) / G;
  for (int i = (int)(blockIdx.x * blockDim.x + threadIdx.x) / G; i < m; i += groups) {
    const int as = rpA[i], ae = rpA[i + 1], bs = rpB[i], be = rpB[i + 1];
    const int cs = rpC[i];
    const bool rep = row_has_repeat<G>(ciA, as, ae, lane, gmask) | row_has_repeat<G>(ciB, bs, be, lane, gmask);
    if (rep) {
      if (lane == 0) {  // the serial walk (SortedNumericSumFunctor, spadd_numeric_impl.hpp:50-92)
        int ai = as, bi = bs, pos = cs;
        int acol = ai < ae ? ciA[ai] : INT_MAX;
        int bcol = bi < be ? ciB[bi] : INT_MAX;
        while (acol != INT_MAX || bcol != INT_MAX) {
          const int c = acol < bcol ? acol : bcol;
          S acc = S(0);
          while (acol == c) {
            acc += mul_rn(alpha, vA[ai]);
            acol = (++ai < ae) ? ciA[ai] : INT_MAX;
          }
          while (bcol == c) {
            acc += mul_rn(beta, vB[bi]);
            bcol = (++bi < be) ? ciB[bi] : INT_MAX;
          }
          ciC[pos] = c;
          vC[pos] = acc;
          ++pos;
        }
      }
      continue;
    }
    const int alen = ae - as, blen = be - bs;
    int before = 0;  // matched entries of A in the batches done
    for (int base = 0; base < alen; base += G) {
      const int k = base + lane;
      bool match = false;
      int col = 0, lb = 0;
      if (k < alen) {
        col = ciA[as + k];
        lb = row_lower_bound(ciB + bs, blen, col);
        match = lb < blen && ciB[bs + lb] == col;
      }
      const unsigned mb = __ballot_sync(gmask, match);
      if (k < alen) {
        const int pos = cs + k + lb - (before + __popc(mb & below));
        S acc = add_rn(S(0), mul_rn(alpha, vA[as + k]));
        if (match) acc = add_rn(acc, mul_rn(beta, vB[bs + lb]));
        ciC[pos] = col;
        vC[pos] = acc;
      }
      before += __popc(mb);
    }
    before = 0;  // matched entries of B in the batches done
    for (int base = 0; base < blen; base += G) {
      const int k = base + lane;
      bool match = false;
      int col = 0, lb = 0;
      if (k < blen) {
        col = ciB[bs + k];
        lb = row_lower_bound(ciA + as, alen, col);
        match = lb < alen && ciA[as + lb] == col;
      }
      const unsigned mb = __ballot_sync(gmask, match);
      if (k < blen && !match) {
        const int pos = cs + k + lb - (before + __popc(mb & below));
        ciC[pos] = col;
        vC[pos] = add_rn(S(0), mul_rn(beta, vB[bs + k]));
      }
      before += __popc(mb);
    }
  }
}

// lanes per row of the sorted spadd kernels by the mean length of A_i plus B_i; 0 = the one-thread-per-row kernels
// (B200SP_SPADD_GROUP = 0 | 8 | 32 overrides)
static int spadd_group(int m, int64_t nnzA, int64_t nnzB) {
  if (const char* e = getenv("B200SP_SPADD_GROUP")) {
    const int g = atoi(e);
    if (g == 0 || g == 8 || g == 32) return g;
  }
  // tools/bench_spadd.py on an H100 (400 W), 54 + 54 entries per row: numeric 0.60-0.69 ms with 32 lanes, 1.0-1.9 ms with 8,
  // 6.6-7.3 ms with one thread per row (symbolic 0.39-0.44 vs 0.33-0.40 ms), same bits.  Rows this long fill a warp; shorter
  // rows keep 8 lanes (more rows in flight), a choice not re-measured on the H100.
  return (double)(nnzA + nnzB) / (double)std::max(m, 1) >= 64.0 ? 32 : 8;
}

__global__ void __launch_bounds__(256)
    spadd_upper_bound_kernel(int m, const int* __restrict__ rpA, const int* __restrict__ rpB, int* __restrict__ counts) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x)
    counts[i] = (rpA[i + 1] - rpA[i]) + (rpB[i + 1] - rpB[i]);
}

// UnmergedSumFunctor (spadd_symbolic_impl.hpp:232-276): A's entries then B's; perm = j or j + len(A_i)
__global__ void __launch_bounds__(256)
    spadd_unmerged_kernel(int m, const int* __restrict__ rpA, const int* __restrict__ ciA, const int* __restrict__ rpB,
                          const int* __restrict__ ciB, const int* __restrict__ rpU, int* __restrict__ ciU,
                          int* __restrict__ perm) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t i = t >> 3;
  const int sl = (int)(t & 7);
  if (i >= m) return;
  const int as = rpA[i], alen = rpA[i + 1] - as;
  const int bs = rpB[i], blen = rpB[i + 1] - bs;
  const int cs = rpU[i];
  for (int j = sl; j < alen; j += 8) {
    ciU[cs + j] = ciA[as + j];
    perm[cs + j] = j;
  }
  for (int j = sl; j < blen; j += 8) {
    ciU[cs + alen + j] = ciB[bs + j];
    perm[cs + alen + j] = j + alen;
  }
}

// MergeEntriesFunctor (spadd_symbolic_impl.hpp:278-343), 8 lanes per row: the place of a union entry in C_i is the number of column
// changes up to it (ballot / popc prefix).  simple[i] = no column occurs twice in A_i or twice in B_i: then no two entries of one
// matrix share a place in C_i and the numeric phase may add a row's entries side by side (below).
__global__ void __launch_bounds__(256)
    spadd_merge_entries_kernel(int m, const int* __restrict__ rpA, const int* __restrict__ rpB,
                               const int* __restrict__ rpU, const int* __restrict__ ciU, const int* __restrict__ perm,
                               int* __restrict__ counts, int* __restrict__ apos, int* __restrict__ bpos, int* __restrict__ simple) {
  constexpr int G = 8;
  const int lane = (int)threadIdx.x & (G - 1);
  const int gbase = ((int)threadIdx.x & 31) & ~(G - 1);
  const unsigned gmask = ((1u << G) - 1u) << gbase;
  const unsigned upto = (2u << (gbase + lane)) - 1u;  // this lane and the ones before it
  const int groups = (int)(gridDim.x * blockDim.x) / G;
  for (int i = (int)(blockIdx.x * blockDim.x + threadIdx.x) / G; i < m; i += groups) {
    const int cs = rpU[i], ce = rpU[i + 1];
    if (ce == cs) {
      if (lane == 0) {
        counts[i] = 0;
        simple[i] = 1;
      }
      continue;
    }
    const int as = rpA[i], alen = rpA[i + 1] - as;
    const int bs = rpB[i];
    int before = 0;  // column changes in the batches done
    bool twice = false;
    for (int base = cs; base < ce; base += G) {
      const int it = base + lane;
      bool change = false;
      int pv = 0;
      if (it < ce) {
        pv = perm[it];
        if (it > cs) {
          change = ciU[it] != ciU[it - 1];
          // equal columns are ordered A's entries first (the stable sort keeps the unmerged order): two neighbours of one matrix
          twice |= !change && ((perm[it - 1] < alen) == (pv < alen));
        }
      }
      const unsigned cb = __ballot_sync(gmask, change);
      if (it < ce) {
        const int cf = before + __popc(cb & upto);
        if (pv < alen) apos[as + pv] = cf;
        else bpos[bs + (pv - alen)] = cf;
      }
      before += __popc(cb);
    }
    const unsigned tw = __ballot_sync(gmask, twice);
    if (lane == 0) {
      counts[i] = before + 1;
      simple[i] = tw == 0u;
    }
  }
}

// UnsortedNumericSumFunctor (spadd_numeric_impl.hpp:131-152), 8 lanes per row.  The three passes of the serial loop -- C_i = 0;
// C_i[apos] += alpha a in storage order; C_i[bpos] += beta b -- run pass by pass with the lanes side by side when the row is
// `simple` (inside one pass no two entries then touch the same place, so each place sees the serial loop's operations in its order:
// (0 + alpha a) + beta b); other rows are walked by lane 0.
template <typename S>
__global__ void __launch_bounds__(256)
    spadd_unsorted_numeric_kernel(int m, const int* __restrict__ rpA, const int* __restrict__ ciA,
                                  const S* __restrict__ vA, S alpha, const int* __restrict__ rpB,
                                  const int* __restrict__ ciB, const S* __restrict__ vB, S beta,
                                  const int* __restrict__ rpC, int* __restrict__ ciC, S* vC,
                                  const int* __restrict__ apos, const int* __restrict__ bpos, const int* __restrict__ simple) {
  constexpr int G = 8;
  const int lane = (int)threadIdx.x & (G - 1);
  const int gbase = ((int)threadIdx.x & 31) & ~(G - 1);
  const unsigned gmask = ((1u << G) - 1u) << gbase;
  const int groups = (int)(gridDim.x * blockDim.x) / G;
  for (int i = (int)(blockIdx.x * blockDim.x + threadIdx.x) / G; i < m; i += groups) {
    const int cs = rpC[i], ce = rpC[i + 1];
    const int as = rpA[i], ae = rpA[i + 1], bs = rpB[i], be = rpB[i + 1];
    if (!simple[i]) {
      if (lane == 0) {
        for (int j = cs; j < ce; ++j) vC[j] = S(0);
        for (int j = as; j < ae; ++j) {
          vC[cs + apos[j]] += mul_rn(alpha, vA[j]);
          ciC[cs + apos[j]] = ciA[j];
        }
        for (int j = bs; j < be; ++j) {
          vC[cs + bpos[j]] += mul_rn(beta, vB[j]);
          ciC[cs + bpos[j]] = ciB[j];
        }
      }
      continue;
    }
    for (int j = cs + lane; j < ce; j += G) vC[j] = S(0);
    __syncwarp(gmask);
    for (int j = as + lane; j < ae; j += G) {
      const int q = cs + apos[j];
      vC[q] = add_rn(vC[q], mul_rn(alpha, vA[j]));
      ciC[q] = ciA[j];
    }
    __syncwarp(gmask);
    for (int j = bs + lane; j < be; j += G) {
      const int q = cs + bpos[j];
      vC[q] = add_rn(vC[q], mul_rn(beta, vB[j]));
      ciC[q] = ciB[j];
    }
  }
}

// ---------------------------------------------------------------------------
// transpose: histogram of columns, scan, atomic fill of (row, entry id) keys, stable in-row sort
// by (row, entry id), gather of the values through the entry id.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    transpose_count_kernel(int64_t nnz, const int* __restrict__ ci, int* __restrict__ counts) {
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < nnz; j += (int64_t)gridDim.x * blockDim.x)
    atomicAdd(&counts[ci[j]], 1);
}

__global__ void __launch_bounds__(256)
    transpose_fill_kernel(int m, const int* __restrict__ rp, const int* __restrict__ ci, int* __restrict__ cursor,
                          int* __restrict__ t_row, int* __restrict__ t_src) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t i = t >> 3;
  const int sl = (int)(t & 7);
  if (i >= m) return;
  for (int j = rp[i] + sl; j < rp[i + 1]; j += 8) {
    const int p = atomicAdd(&cursor[ci[j]], 1);
    t_row[p] = (int)i;
    t_src[p] = j;
  }
}

template <typename S>
__global__ void __launch_bounds__(256)
    transpose_gather_kernel(int64_t nnz, const int* __restrict__ t_src, const S* __restrict__ vals, S* __restrict__ t_vals) {
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < nnz; j += (int64_t)gridDim.x * blockDim.x)
    t_vals[j] = vals[t_src[j]];
}

static inline int grid_for(int64_t work, int per_block = 256, int mult = 8) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((work + per_block - 1) / per_block, (int64_t)sm_count() * mult));
}

// structure of the transpose + source entry of every transposed entry (t_src); nnz = row_ptr[m] (host value)
int transpose_structure(cudaStream_t st, int m, int n, int64_t nnz, const int* rp, const int* ci, int* trp, int* tci,
                        int* t_src) {
  DevTmp tmp(st);
  int *counts, *cursor;
  B200SP_CUDA_TRY(tmp.alloc(&counts, (size_t)n));
  B200SP_CUDA_TRY(tmp.alloc(&cursor, (size_t)n + 1));
  B200SP_CUDA_TRY(cudaMemsetAsync(counts, 0, sizeof(int) * (size_t)n, st));
  transpose_count_kernel<<<grid_for(nnz), 256, 0, st>>>(nnz, ci, counts);
  B200SP_LAUNCH_CHECK();
  int rc = counts_to_offsets(st, n, counts, trp, nullptr, nullptr);
  if (rc) return rc;
  B200SP_CUDA_TRY(cudaMemcpyAsync(cursor, trp, sizeof(int) * ((size_t)n + 1), cudaMemcpyDeviceToDevice, st));
  transpose_fill_kernel<<<(unsigned)(((int64_t)m * 8 + 255) / 256), 256, 0, st>>>(m, rp, ci, cursor, tci, t_src);
  B200SP_LAUNCH_CHECK();
  // (row, entry id) order inside every transposed row: the Serial loop's order, whatever the atomics did
  return sort_crs_impl<int, 2>(st, n, trp, tci, t_src, nnz);
}

template <typename S>
int gather_values(cudaStream_t st, int64_t nnz, const int* t_src, const S* v, S* tv) {
  if (nnz <= 0) return B200SP_OK;
  transpose_gather_kernel<S><<<grid_for(nnz), 256, 0, st>>>(nnz, t_src, v, tv);
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}
template int gather_values<double>(cudaStream_t, int64_t, const int*, const double*, double*);
template int gather_values<float>(cudaStream_t, int64_t, const int*, const float*, float*);

template <typename S, bool HAS_VALS>
static int transpose_impl(cudaStream_t st, int m, int n, const int* rp, const int* ci, const S* v, int* trp, int* tci,
                          S* tv) {
  B200SP_REQUIRE(m >= 0 && n >= 0, "transpose_matrix: negative dimension");
  B200SP_REQUIRE(trp != nullptr, "transpose_matrix: output row map is null");
  int64_t nnz = 0;
  if (m > 0) {
    B200SP_REQUIRE(rp != nullptr, "transpose_matrix: row map is null");
    int last = 0;
    B200SP_CUDA_TRY(cudaMemcpyAsync(&last, rp + m, sizeof(int), cudaMemcpyDeviceToHost, st));
    B200SP_CUDA_TRY(cudaStreamSynchronize(st));
    nnz = last;
  }
  if (n == 0 || nnz == 0) return zero_ints(st, (int64_t)n + 1, trp);
  B200SP_REQUIRE(ci && tci && (!HAS_VALS || (v && tv)), "transpose_matrix: null pointer argument");
  DevTmp tmp(st);
  int* t_src;
  B200SP_CUDA_TRY(tmp.alloc(&t_src, (size_t)nnz));
  int rc = transpose_structure(st, m, n, nnz, rp, ci, trp, tci, t_src);
  if (rc) return rc;
  if (HAS_VALS) return gather_values<S>(st, nnz, t_src, v, tv);
  return B200SP_OK;
}

}  // namespace b200sp

using namespace b200sp;

// ---------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------
struct b200sp_spadd_plan {
  bool input_sorted = false, input_merged = false;
  bool symbolic_done = false;
  int m = 0, n = 0;
  int64_t c_nnz = 0;
  int64_t nnzA = 0, nnzB = 0;
  int *apos = nullptr, *bpos = nullptr;  // unsorted path: position of every A / B entry in its C row
  int* simple = nullptr;                 // unsorted path, per row: no repeated column inside A_i or inside B_i
};

namespace b200sp {
static void spadd_release(b200sp_spadd_plan* p, cudaStream_t st) {
  if (p->apos) cudaFreeAsync(p->apos, st);
  if (p->bpos) cudaFreeAsync(p->bpos, st);
  if (p->simple) cudaFreeAsync(p->simple, st);
  p->apos = p->bpos = p->simple = nullptr;
  p->symbolic_done = false;
}

template <typename S>
static int sort_and_merge_count(cudaStream_t st, int m, const int* rp, int* ci, S* v, bool has_vals, int* rp_out,
                                int64_t* merged_nnz) {
  B200SP_REQUIRE(m >= 0, "sort_and_merge: negative row count");
  B200SP_REQUIRE(merged_nnz != nullptr, "sort_and_merge: merged_nnz is null");
  *merged_nnz = 0;
  if (m == 0) {
    // zero rows: a length-one row map, if present, is [0] (SortCrs.hpp:329-334)
    return rp_out ? zero_ints(st, 1, rp_out) : B200SP_OK;
  }
  B200SP_REQUIRE(rp && rp_out, "sort_and_merge: null row map");
  int rc = has_vals ? sort_crs_impl<S, 1>(st, m, rp, ci, v, -1) : sort_crs_impl<S, 0>(st, m, rp, ci, nullptr, -1);
  if (rc) return rc;
  DevTmp tmp(st);
  int* counts;
  B200SP_CUDA_TRY(tmp.alloc(&counts, (size_t)m));
  merged_count_kernel<<<(unsigned)(((int64_t)m * 8 + 255) / 256), 256, 0, st>>>(m, rp, ci, counts);
  B200SP_LAUNCH_CHECK();
  long long total = 0;
  rc = counts_to_offsets(st, m, counts, rp_out, &total, nullptr);
  if (rc) return rc;
  *merged_nnz = total;
  return B200SP_OK;
}

template <typename S>
static int sort_and_merge_fill(cudaStream_t st, int m, const int* rp, const int* ci, const S* v, bool has_vals,
                               const int* rp_out, int* ci_out, S* v_out) {
  if (m <= 0) return B200SP_OK;
  B200SP_REQUIRE(rp && rp_out, "sort_and_merge: null row map");
  const int fill_blocks = grid_for((int64_t)m * 8);  // 8 lanes per row
  if (has_vals) merged_fill_kernel<S, true><<<fill_blocks, 256, 0, st>>>(m, rp, ci, v, rp_out, ci_out, v_out);
  else merged_fill_kernel<S, false><<<fill_blocks, 256, 0, st>>>(m, rp, ci, nullptr, rp_out, ci_out, nullptr);
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

template <typename S>
static int spadd_numeric_impl(b200sp_spadd_plan* p, cudaStream_t st, int m, int n, const int* rpA, const int* ciA,
                              const S* vA, S alpha, const int* rpB, const int* ciB, const S* vB, S beta, const int* rpC,
                              int* ciC, S* vC) {
  B200SP_REQUIRE(p != nullptr, "spadd_numeric: null plan");
  if (!p->symbolic_done) {
    set_error("spadd_numeric: spadd_symbolic was not called on this handle");
    return B200SP_ERR_STATE;
  }
  if (p->m != m || p->n != n) {
    set_error("spadd_numeric: dimensions (%d,%d) differ from symbolic (%d,%d)", m, n, p->m, p->n);
    return B200SP_ERR_STATE;
  }
  if (m == 0 || p->c_nnz == 0) return B200SP_OK;
  B200SP_REQUIRE(rpA && rpB && rpC && ciC && vC, "spadd_numeric: null pointer argument");
  B200SP_REQUIRE((p->nnzA == 0 || (ciA && vA)) && (p->nnzB == 0 || (ciB && vB)), "spadd_numeric: null pointer argument");
  const int blocks = grid_for(m);
  if (p->input_sorted) {
    const int g = spadd_group(m, p->nnzA, p->nnzB);
    if (g == 32) spadd_sorted_numeric_group_kernel<S, 32><<<grid_for((int64_t)m * 32), 256, 0, st>>>(m, rpA, ciA, vA, alpha, rpB, ciB, vB, beta, rpC, ciC, vC);
    else if (g == 8) spadd_sorted_numeric_group_kernel<S, 8><<<grid_for((int64_t)m * 8), 256, 0, st>>>(m, rpA, ciA, vA, alpha, rpB, ciB, vB, beta, rpC, ciC, vC);
    else spadd_sorted_numeric_kernel<S><<<blocks, 256, 0, st>>>(m, rpA, ciA, vA, alpha, rpB, ciB, vB, beta, rpC, ciC, vC);
  } else {
    spadd_unsorted_numeric_kernel<S><<<grid_for((int64_t)m * 8), 256, 0, st>>>(m, rpA, ciA, vA, alpha, rpB, ciB, vB, beta, rpC, ciC, vC,
                                                                              p->apos, p->bpos, p->simple);
  }
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}
}  // namespace b200sp

extern "C" {

int b200sp_sort_crs_f64_i32(void* stream, int m, const int* row_ptr, int* col_idx, double* vals) {
  B200SP_REQUIRE(m >= 0, "sort_crs_matrix: negative row count");
  if (m == 0) return B200SP_OK;
  B200SP_REQUIRE(row_ptr != nullptr, "sort_crs_matrix: row map is null");
  return vals ? sort_crs_impl<double, 1>((cudaStream_t)stream, m, row_ptr, col_idx, vals, -1)
              : sort_crs_impl<double, 0>((cudaStream_t)stream, m, row_ptr, col_idx, nullptr, -1);
}
int b200sp_sort_crs_f32_i32(void* stream, int m, const int* row_ptr, int* col_idx, float* vals) {
  B200SP_REQUIRE(m >= 0, "sort_crs_matrix: negative row count");
  if (m == 0) return B200SP_OK;
  B200SP_REQUIRE(row_ptr != nullptr, "sort_crs_matrix: row map is null");
  return vals ? sort_crs_impl<float, 1>((cudaStream_t)stream, m, row_ptr, col_idx, vals, -1)
              : sort_crs_impl<float, 0>((cudaStream_t)stream, m, row_ptr, col_idx, nullptr, -1);
}
int b200sp_sort_crs_graph_i32(void* stream, int m, const int* row_ptr, int* col_idx) {
  return b200sp_sort_crs_f32_i32(stream, m, row_ptr, col_idx, nullptr);
}

int b200sp_sort_and_merge_count_f64_i32(void* stream, int m, const int* row_ptr, int* col_idx, double* vals,
                                        int* row_ptr_out, int64_t* merged_nnz) {
  return sort_and_merge_count<double>((cudaStream_t)stream, m, row_ptr, col_idx, vals, vals != nullptr, row_ptr_out, merged_nnz);
}
int b200sp_sort_and_merge_count_f32_i32(void* stream, int m, const int* row_ptr, int* col_idx, float* vals,
                                        int* row_ptr_out, int64_t* merged_nnz) {
  return sort_and_merge_count<float>((cudaStream_t)stream, m, row_ptr, col_idx, vals, vals != nullptr, row_ptr_out, merged_nnz);
}
int b200sp_sort_and_merge_fill_f64_i32(void* stream, int m, const int* row_ptr, const int* col_idx, const double* vals,
                                       const int* row_ptr_out, int* col_idx_out, double* vals_out) {
  return sort_and_merge_fill<double>((cudaStream_t)stream, m, row_ptr, col_idx, vals, vals != nullptr, row_ptr_out, col_idx_out, vals_out);
}
int b200sp_sort_and_merge_fill_f32_i32(void* stream, int m, const int* row_ptr, const int* col_idx, const float* vals,
                                       const int* row_ptr_out, int* col_idx_out, float* vals_out) {
  return sort_and_merge_fill<float>((cudaStream_t)stream, m, row_ptr, col_idx, vals, vals != nullptr, row_ptr_out, col_idx_out, vals_out);
}

int b200sp_transpose_f64_i32(void* stream, int m, int n, const int* row_ptr, const int* col_idx, const double* vals,
                             int* t_row_ptr, int* t_col_idx, double* t_vals) {
  return (vals || t_vals) ? transpose_impl<double, true>((cudaStream_t)stream, m, n, row_ptr, col_idx, vals, t_row_ptr, t_col_idx, t_vals)
                          : transpose_impl<double, false>((cudaStream_t)stream, m, n, row_ptr, col_idx, nullptr, t_row_ptr, t_col_idx, nullptr);
}
int b200sp_transpose_f32_i32(void* stream, int m, int n, const int* row_ptr, const int* col_idx, const float* vals,
                             int* t_row_ptr, int* t_col_idx, float* t_vals) {
  return (vals || t_vals) ? transpose_impl<float, true>((cudaStream_t)stream, m, n, row_ptr, col_idx, vals, t_row_ptr, t_col_idx, t_vals)
                          : transpose_impl<float, false>((cudaStream_t)stream, m, n, row_ptr, col_idx, nullptr, t_row_ptr, t_col_idx, nullptr);
}

int b200sp_spadd_plan_create(b200sp_spadd_plan** plan, int input_sorted, int input_merged) {
  B200SP_REQUIRE(plan != nullptr, "spadd_plan_create: null output pointer");
  b200sp_spadd_plan* p = new (std::nothrow) b200sp_spadd_plan();
  if (!p) {
    set_error("spadd_plan_create: out of host memory");
    return B200SP_ERR_ALLOC;
  }
  p->input_sorted = input_sorted != 0;
  p->input_merged = input_merged != 0;
  *plan = p;
  return B200SP_OK;
}

int b200sp_spadd_plan_destroy(b200sp_spadd_plan* p, void* stream) {
  if (!p) return B200SP_OK;
  spadd_release(p, (cudaStream_t)stream);
  delete p;
  return B200SP_OK;
}

int b200sp_spadd_symbolic_i32(b200sp_spadd_plan* p, void* stream, int m, int n, const int* rpA, const int* ciA,
                              const int* rpB, const int* ciB, int* rpC, int64_t* c_nnz) {
  B200SP_REQUIRE(p != nullptr, "spadd_symbolic: null plan");
  B200SP_REQUIRE(m >= 0 && n >= 0, "spadd_symbolic: negative dimension");
  cudaStream_t st = (cudaStream_t)stream;
  spadd_release(p, st);
  p->m = m;
  p->n = n;
  p->c_nnz = 0;
  p->nnzA = p->nnzB = 0;
  if (c_nnz) *c_nnz = 0;
  if (m == 0) {
    // zero rows: nnz(C) = 0; a length-one row map must hold 0 (spadd_symbolic_impl.hpp:443-450)
    if (rpC) {
      int rc = zero_ints(st, 1, rpC);
      if (rc) return rc;
    }
    p->symbolic_done = true;
    return B200SP_OK;
  }
  B200SP_REQUIRE(rpA && rpB && rpC, "spadd_symbolic: null row map");
  int lastA = 0, lastB = 0;
  B200SP_CUDA_TRY(cudaMemcpyAsync(&lastA, rpA + m, sizeof(int), cudaMemcpyDeviceToHost, st));
  B200SP_CUDA_TRY(cudaMemcpyAsync(&lastB, rpB + m, sizeof(int), cudaMemcpyDeviceToHost, st));
  B200SP_CUDA_TRY(cudaStreamSynchronize(st));
  p->nnzA = lastA;
  p->nnzB = lastB;
  B200SP_REQUIRE((lastA == 0 || ciA) && (lastB == 0 || ciB), "spadd_symbolic: null column index array");
  if ((int64_t)lastA + (int64_t)lastB > (int64_t)INT_MAX) {
    set_error("spadd_symbolic: nnz(A) + nnz(B) = %lld exceeds int32 offsets", (long long)lastA + lastB);
    return B200SP_ERR_OVERFLOW;
  }
  DevTmp tmp(st);
  int* counts;
  B200SP_CUDA_TRY(tmp.alloc(&counts, (size_t)m));
  const int blocks = grid_for(m);
  long long total = 0;
  int rc;
  if (p->input_sorted) {
    const int g = spadd_group(m, lastA, lastB);
    if (g == 32) spadd_sorted_count_group_kernel<32><<<grid_for((int64_t)m * 32), 256, 0, st>>>(m, rpA, ciA, rpB, ciB, counts);
    else if (g == 8) spadd_sorted_count_group_kernel<8><<<grid_for((int64_t)m * 8), 256, 0, st>>>(m, rpA, ciA, rpB, ciB, counts);
    else spadd_sorted_count_kernel<<<blocks, 256, 0, st>>>(m, rpA, ciA, rpB, ciB, counts);
    B200SP_LAUNCH_CHECK();
    rc = counts_to_offsets(st, m, counts, rpC, &total, nullptr);
    if (rc) return rc;
  } else {
    int *rpU, *ciU, *perm;
    B200SP_CUDA_TRY(tmp.alloc(&rpU, (size_t)m + 1));
    spadd_upper_bound_kernel<<<blocks, 256, 0, st>>>(m, rpA, rpB, counts);
    B200SP_LAUNCH_CHECK();
    long long ub = 0;
    rc = counts_to_offsets(st, m, counts, rpU, &ub, nullptr);
    if (rc) return rc;
    B200SP_CUDA_TRY(tmp.alloc(&ciU, (size_t)ub));
    B200SP_CUDA_TRY(tmp.alloc(&perm, (size_t)ub));
    spadd_unmerged_kernel<<<(unsigned)(((int64_t)m * 8 + 255) / 256), 256, 0, st>>>(m, rpA, ciA, rpB, ciB, rpU, ciU, perm);
    B200SP_LAUNCH_CHECK();
    rc = sort_crs_impl<int, 2>(st, m, rpU, ciU, perm, ub);
    if (rc) return rc;
    B200SP_CUDA_TRY(cudaMallocAsync((void**)&p->apos, sizeof(int) * (size_t)std::max(lastA, 1), st));
    B200SP_CUDA_TRY(cudaMallocAsync((void**)&p->bpos, sizeof(int) * (size_t)std::max(lastB, 1), st));
    B200SP_CUDA_TRY(cudaMallocAsync((void**)&p->simple, sizeof(int) * (size_t)m, st));
    spadd_merge_entries_kernel<<<grid_for((int64_t)m * 8), 256, 0, st>>>(m, rpA, rpB, rpU, ciU, perm, counts, p->apos, p->bpos, p->simple);
    B200SP_LAUNCH_CHECK();
    rc = counts_to_offsets(st, m, counts, rpC, &total, nullptr);
    if (rc) return rc;
  }
  if (total > (long long)INT_MAX) {
    set_error("spadd_symbolic: nnz(C) = %lld exceeds int32 offsets", total);
    return B200SP_ERR_OVERFLOW;
  }
  p->c_nnz = total;
  p->symbolic_done = true;
  if (c_nnz) *c_nnz = total;
  return B200SP_OK;
}

int b200sp_spadd_numeric_f64_i32(b200sp_spadd_plan* plan, void* stream, int m, int n, const int* rpA, const int* ciA,
                                 const double* vA, double alpha, const int* rpB, const int* ciB, const double* vB,
                                 double beta, const int* rpC, int* ciC, double* vC) {
  return spadd_numeric_impl<double>(plan, (cudaStream_t)stream, m, n, rpA, ciA, vA, alpha, rpB, ciB, vB, beta, rpC, ciC, vC);
}
int b200sp_spadd_numeric_f32_i32(b200sp_spadd_plan* plan, void* stream, int m, int n, const int* rpA, const int* ciA,
                                 const float* vA, float alpha, const int* rpB, const int* ciB, const float* vB,
                                 float beta, const int* rpC, int* ciC, float* vC) {
  return spadd_numeric_impl<float>(plan, (cudaStream_t)stream, m, n, rpA, ciA, vA, alpha, rpB, ciB, vB, beta, rpC, ciC, vC);
}

}  // extern "C"
