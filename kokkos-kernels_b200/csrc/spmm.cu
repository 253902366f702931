// spmm.cu -- rank-2 (multivector) CrsMatrix SpMV: Y = beta*Y + alpha*op(A)*X.
//
// Replaces the reference's Kokkos::Cuda legs
//   native  SPMV_MV_LayoutLeft_Functor   sparse/impl/KokkosSparse_spmv_impl.hpp:634-1004,1057-1119
//   native  SPMV_MV_Transpose_Functor    sparse/impl/KokkosSparse_spmv_impl.hpp:547-632,1163-1229
//   TPL     cusparseSpMM                 sparse/tpls/KokkosSparse_spmv_mv_tpl_spec_decl.hpp:97-196
//
// Kernels:
//   spmm_item_coop_kernel X, Y LayoutRight with a plan: length-sorted runs of
//                         <= LMAX entries of one row (DESIGN.md 4.2), pieces
//                         of longer rows added up by spmm_item_reduce_kernel.
//   spmm_rowmajor_kernel  X, Y LayoutRight without a plan: a group of KT lanes
//                         owns one row of A and one strip of <= KT columns;
//                         (col,val) pairs are loaded coalesced KT at a time and
//                         broadcast by shuffle, X rows are read as contiguous
//                         KT*sizeof(S) segments.  One pass over A per 32-column
//                         strip, no reduction.
//   spmm_general_kernel   any LayoutLeft / LayoutRight mix: thread per (row, j).
//   spmm_transpose_kernel T/H modes: Y pre-scaled, atomicAdd scatter.
// Column-major (LayoutLeft) X with k >= 4 goes through a transposed copy so the
// gather touches one segment per nonzero instead of k sectors (DESIGN.md 3.4).
// binary16 (b200sp_spmm_f16_i32): the item, general and relayout kernels with fp32 accumulators, and an fp32 scratch for
// T/H (DESIGN.md 4.3).
#include <limits.h>
#include "spmv_plan.h"
#include <algorithm>
#include <type_traits>
#include <atomic>
#include <stdlib.h>

namespace b200sp {

static void set_last_kernel(b200sp_spmv_plan* p, const char* s) {
  if (p) snprintf(p->last_kernel, sizeof(p->last_kernel), "%s", s);
}

// Storage type S -> accumulator type: fp32 and fp64 accumulate in their own type, binary16 (__half) in fp32.  wide() is exact;
// narrow() rounds once, to nearest even (a result beyond the fp16 range becomes +-inf).  Kernels that serve fp16 compute in
// AccT<S> and touch S only to load and store.
template <typename S> struct AccOf { using type = S; };
template <> struct AccOf<__half> { using type = float; };
template <typename S> using AccT = typename AccOf<S>::type;
__device__ __forceinline__ float wide(float v) { return v; }
__device__ __forceinline__ double wide(double v) { return v; }
__device__ __forceinline__ float wide(__half v) { return __half2float(v); }
template <typename S> __device__ __forceinline__ S narrow(AccT<S> v) { return v; }
template <> __device__ __forceinline__ __half narrow<__half>(float v) { return __float2half_rn(v); }

template <typename S>
__global__ void scale2d_kernel(int64_t rows, int k, AccT<S> beta, S* __restrict__ Y, int64_t yr, int64_t yc) {
  using A = AccT<S>;
  const int64_t total = rows * k;
  const bool by_rows = (yc == 1 || yr != 1);  // walk memory-contiguously for either layout
  if (total <= (int64_t)INT32_MAX) {  // 32-bit index arithmetic: a 64-bit division per element costs more than the element's traffic
    const unsigned t32 = (unsigned)total, k32 = (unsigned)k, r32 = (unsigned)rows, step = gridDim.x * blockDim.x;
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < t32; i += step) {
      unsigned r, j;
      if (by_rows) { r = i / k32; j = i - r * k32; } else { j = i / r32; r = i - j * r32; }
      S* p = &Y[(int64_t)r * yr + (int64_t)j * yc];
      *p = narrow<S>((beta == A(0)) ? A(0) : beta * wide(*p));
    }
    return;
  }
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r, j;
    if (by_rows) { r = i / k; j = i % k; } else { j = i / rows; r = i % rows; }
    S* p = &Y[r * yr + j * yc];
    *p = narrow<S>((beta == A(0)) ? A(0) : beta * wide(*p));
  }
}

// out(r, j) row-major [rows x k] <- in(r, j) with strides (sr, sc)   (or the reverse).  256 threads move tiles of 128 rows x
// <= 32 columns through shared memory: on the strided side consecutive threads touch consecutive rows of one column (512
// contiguous bytes per column of a LayoutLeft operand in fp32), on the row-major side consecutive elements (the whole tile is
// one contiguous run when k <= 32); the odd row pitch keeps both phases free of bank conflicts.  Grid-stride over the tiles.
template <typename S, bool TO_ROWMAJOR>
__global__ void __launch_bounds__(256) relayout_kernel(int64_t rows, int k, S* __restrict__ rm, const S* __restrict__ strided_in,
                                                       S* __restrict__ strided_out, int64_t sr, int64_t sc) {
  constexpr int R = 128, KC = 32;
  __shared__ S tile[R][KC + 1];
  const int tid = threadIdx.x;
  const int64_t ntiles = (rows + R - 1) / R;
  for (int64_t tI = blockIdx.x; tI < ntiles; tI += gridDim.x) {
    const int64_t r0 = tI * R;
    const int nr = (int)((rows - r0) < (int64_t)R ? (rows - r0) : (int64_t)R);
    for (int j0 = 0; j0 < k; j0 += KC) {
      const int nc = (k - j0) < KC ? (k - j0) : KC;
      if (TO_ROWMAJOR) {
        for (int idx = tid; idx < R * nc; idx += 256) {
          const int r = idx % R, j = idx / R;
          if (r < nr) tile[r][j] = strided_in[(r0 + r) * sr + (int64_t)(j0 + j) * sc];
        }
        __syncthreads();
        for (int idx = tid; idx < nr * nc; idx += 256) {
          const int r = idx / nc, j = idx - r * nc;
          rm[(r0 + r) * k + j0 + j] = tile[r][j];
        }
      } else {
        for (int idx = tid; idx < nr * nc; idx += 256) {
          const int r = idx / nc, j = idx - r * nc;
          tile[r][j] = rm[(r0 + r) * k + j0 + j];
        }
        __syncthreads();
        for (int idx = tid; idx < R * nc; idx += 256) {
          const int r = idx % R, j = idx / R;
          if (r < nr) strided_out[(r0 + r) * sr + (int64_t)(j0 + j) * sc] = tile[r][j];
        }
      }
      __syncthreads();
    }
  }
}

template <typename S, int KT>
__global__ void __launch_bounds__(256)
    spmm_rowmajor_kernel(int m, int k, const int* __restrict__ row_ptr, const int* __restrict__ col_idx,
                         const S* __restrict__ vals, const S* __restrict__ X, int64_t ldx, S* __restrict__ Y,
                         int64_t ldy, S alpha, S beta) {
  constexpr int GPW = 32 / KT;  // row groups per warp
  const int lane = threadIdx.x & 31;
  const int grp = lane / KT, t = lane % KT;
  const int nstrips = (k + KT - 1) / KT;
  const int64_t warp_global = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t work = (int64_t)((m + GPW - 1) / GPW) * nstrips;
  for (int64_t w = warp_global; w < work; w += nwarps) {
    const int strip = (int)(w % nstrips);
    const int r = (int)(w / nstrips) * GPW + grp;
    const int j = strip * KT + t;
    int rs = 0, re = 0;
    if (r < m) {
      rs = row_ptr[r];
      re = row_ptr[r + 1];
    }
    // all groups of the warp iterate to the longest row (shuffles are warp-wide)
    int len = re - rs;
    int maxlen = len;
#pragma unroll
    for (int o = 16; o >= KT; o >>= 1) maxlen = max(maxlen, __shfl_xor_sync(0xffffffffu, maxlen, o));
    S acc = S(0);
    const bool jok = (j < k);
    for (int b = 0; b < maxlen; b += KT) {
      int c = 0;
      S v = S(0);
      if (b + t < len) {
        c = ld_stream(col_idx + rs + b + t);
        v = ld_stream(vals + rs + b + t);
      }
      const int nb = min(KT, maxlen - b);
#pragma unroll 4
      for (int e = 0; e < nb; ++e) {
        const int ce = __shfl_sync(0xffffffffu, c, e, KT);
        const S ve = __shfl_sync(0xffffffffu, v, e, KT);
        if (jok && b + e < len) acc += ve * ldg(X + (int64_t)ce * ldx + j);
      }
    }
    if (r < m && jok) {
      S* yp = Y + (int64_t)r * ldy + j;
      acc *= alpha;
      *yp = (beta == S(0)) ? acc : beta * *yp + acc;
    }
  }
}

template <typename S>
__global__ void __launch_bounds__(256)
    spmm_general_kernel(int m, int k, const int* __restrict__ row_ptr, const int* __restrict__ col_idx,
                        const S* __restrict__ vals, const S* __restrict__ X, int64_t xr, int64_t xc,
                        S* __restrict__ Y, int64_t yr, int64_t yc, AccT<S> alpha, AccT<S> beta) {
  using A = AccT<S>;
  const int64_t total = (int64_t)m * k;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / k), j = (int)(i % k);
    A acc = A(0);
    for (int e = row_ptr[r]; e < row_ptr[r + 1]; ++e) acc += wide(vals[e]) * wide(ldg(X + (int64_t)col_idx[e] * xr + (int64_t)j * xc));
    acc *= alpha;
    S* yp = Y + (int64_t)r * yr + (int64_t)j * yc;
    *yp = narrow<S>((beta == A(0)) ? acc : beta * wide(*yp) + acc);
  }
}

template <typename S>
__global__ void __launch_bounds__(256)
    spmm_transpose_kernel(int m, int k, const int* __restrict__ row_ptr, const int* __restrict__ col_idx,
                          const S* __restrict__ vals, const S* __restrict__ X, int64_t xr, int64_t xc,
                          S* __restrict__ Y, int64_t yr, int64_t yc, S alpha) {
  const int64_t total = (int64_t)m * k;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / k), j = (int)(i % k);
    const S xv = X[(int64_t)r * xr + (int64_t)j * xc];
    for (int e = row_ptr[r]; e < row_ptr[r + 1]; ++e)
      atomicAdd(Y + (int64_t)col_idx[e] * yr + (int64_t)j * yc, alpha * vals[e] * xv);
  }
}

// T/H for fp16: exact fp32 products a*x added into a zeroed fp32 row-major [yrows x k] scratch, then ONE rounding per entry of Y
// in spmm_acc_epilogue_kernel (a half atomicAdd into Y would round at every addition)
__global__ void __launch_bounds__(256)
    spmm_transpose_acc_kernel(int m, int k, const int* __restrict__ row_ptr, const int* __restrict__ col_idx,
                              const __half* __restrict__ vals, const __half* __restrict__ X, int64_t xr, int64_t xc,
                              float* __restrict__ acc) {
  const int64_t total = (int64_t)m * k;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / k), j = (int)(i % k);
    const float xv = wide(X[(int64_t)r * xr + (int64_t)j * xc]);
    for (int e = row_ptr[r]; e < row_ptr[r + 1]; ++e) atomicAdd(acc + (int64_t)col_idx[e] * k + j, wide(vals[e]) * xv);
  }
}

// 16-byte loads and stores of VW adjacent columns of a row-major X or Y row.  Needs k, ldx, ldy multiples of VW and 16-byte
// aligned X / Y (items_vec).
template <typename S> struct VecOf;
template <> struct VecOf<float> { using type = float4; static constexpr int W = 4; };
template <> struct VecOf<double> { using type = double2; static constexpr int W = 2; };
__device__ __forceinline__ void vec_unpack(const float4& v, float* a) { a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w; }
__device__ __forceinline__ void vec_unpack(const double2& v, double* a) { a[0] = v.x; a[1] = v.y; }
__device__ __forceinline__ float4 vec_pack(const float* a) { return make_float4(a[0], a[1], a[2], a[3]); }
__device__ __forceinline__ double2 vec_pack(const double* a) { return make_double2(a[0], a[1]); }
// binary16: 8 halves per 16-byte load, unpacked straight to fp32 (item kernels only)
template <> struct VecOf<__half> { using type = uint4; static constexpr int W = 8; };
__device__ __forceinline__ void vec_unpack(const uint4& v, float* a) {
  const unsigned w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    a[2 * i] = __half2float(__ushort_as_half((unsigned short)(w[i] & 0xffffu)));
    a[2 * i + 1] = __half2float(__ushort_as_half((unsigned short)(w[i] >> 16)));
  }
}
__device__ __forceinline__ uint4 vec_pack(const __half* a) {
  unsigned w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) w[i] = (unsigned)__half_as_ushort(a[2 * i]) | ((unsigned)__half_as_ushort(a[2 * i + 1]) << 16);
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// the VW adjacent columns a lane accumulates in registers
template <typename S, int VW>
struct Acc {
  S a[VW];
};

// beta*y + alpha*acc as alpha*acc rounded, then one fused multiply-add.  Written out so that every instantiation rounds the
// same way: left to the compiler, the contraction of this expression differed between the 16-byte-load (VW > 1) and the
// scalar variants of the item kernel, and misaligned operands then gave other bits than aligned ones.
__device__ __forceinline__ float axpby_rn(float alpha, float acc, float beta, float y) { return fmaf(beta, y, __fmul_rn(alpha, acc)); }
__device__ __forceinline__ double axpby_rn(double alpha, double acc, double beta, double y) { return fma(beta, y, __dmul_rn(alpha, acc)); }

// the fp16 transpose's epilogue: Y = beta*Y + alpha*acc in fp32, rounded once to fp16; beta == 0 never reads Y
__global__ void __launch_bounds__(256)
    spmm_acc_epilogue_kernel(int64_t rows, int k, const float* __restrict__ acc, float alpha, float beta, __half* __restrict__ Y,
                             int64_t yr, int64_t yc) {
  const int64_t total = rows * k;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / k, j = i % k;
    __half* yp = Y + r * yr + j * yc;
    *yp = narrow<__half>(beta == 0.0f ? __fmul_rn(alpha, acc[i]) : axpby_rn(alpha, acc[i], beta, wide(*yp)));
  }
}

// X rows (and Y for beta != 0) in the accumulator type: VW == 1 one element, else one 16-byte load of VW elements
template <typename S, int VW>
__device__ __forceinline__ Acc<AccT<S>, VW> load_x(const S* __restrict__ p) {
  static_assert(VW == 1 || VW == VecOf<S>::W, "VW is 1 or the 16-byte vector width");
  Acc<AccT<S>, VW> r;
  if constexpr (VW == 1) {
    r.a[0] = wide(ldg(p));
  } else {
    using V = typename VecOf<S>::type;
    const V v = __ldg(reinterpret_cast<const V*>(p));
    vec_unpack(v, r.a);
  }
  return r;
}

// VW accumulator values rounded to T and stored evict-first: VW == 1 one element, else 16-byte stores (two for 8 fp32 partial
// sums of the fp16 kernels)
template <int VW, typename T>
__device__ __forceinline__ void st_vec_once(T* dst, const AccT<T>* o, uint64_t once) {
  if constexpr (VW == 1) {
    st_once(dst, narrow<T>(o[0]), once);
  } else {
    constexpr int PER = VecOf<T>::W;
    static_assert(VW % PER == 0, "whole 16-byte stores");
#pragma unroll
    for (int h = 0; h < VW; h += PER) {
      T t[PER];
#pragma unroll
      for (int i = 0; i < PER; ++i) t[i] = narrow<T>(o[h + i]);
      st_once(reinterpret_cast<typename VecOf<T>::type*>(dst + h), vec_pack(t), once);
    }
  }
}

// an item that is a whole row: o = alpha*acc (beta == 0: Y is not read) or beta*y + alpha*acc, in the accumulator type
template <typename S, int VW>
__device__ __forceinline__ void item_epilogue(AccT<S>* o, const Acc<AccT<S>, VW>& acc, AccT<S> alpha, AccT<S> beta, const S* y) {
  if (beta == AccT<S>(0)) {
#pragma unroll
    for (int cc = 0; cc < VW; ++cc) o[cc] = alpha * acc.a[cc];
  } else {
    const Acc<AccT<S>, VW> old = load_x<S, VW>(y);
#pragma unroll
    for (int cc = 0; cc < VW; ++cc) o[cc] = axpby_rn(alpha, acc.a[cc], beta, old.a[cc]);
  }
}

template <typename S>
static int launch_rowmajor(cudaStream_t st, int m, int k, const int* row_ptr, const int* col_idx, const S* vals,
                           const S* X, int64_t ldx, S* Y, int64_t ldy, S alpha, S beta) {
  int KT = 1;
  while (KT < k && KT < 32) KT <<= 1;
  const int gpw = 32 / KT;
  const int nstrips = (k + KT - 1) / KT;
  const int64_t work = (int64_t)((m + gpw - 1) / gpw) * nstrips;
  int blocks = (int)std::min<int64_t>((work + 7) / 8, (int64_t)sm_count() * 16);
  if (blocks < 1) blocks = 1;
#define B200SP_RM(K)                                                                                              \
  case K:                                                                                                         \
    spmm_rowmajor_kernel<S, K><<<blocks, 256, 0, st>>>(m, k, row_ptr, col_idx, vals, X, ldx, Y, ldy, alpha, beta); \
    break;
  switch (KT) {
    B200SP_RM(1)
    B200SP_RM(2)
    B200SP_RM(4)
    B200SP_RM(8)
    B200SP_RM(16)
    B200SP_RM(32)
  }
#undef B200SP_RM
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

// ---------------------------------------------------------------------------
// Item kernel (row-major X and Y with a plan): the gather-bound formulation.  On power-law matrices row groups of one
// warp that each own a whole row run loops of very different lengths and wait for the longest; here the unit of work is
// an ITEM -- a run of <= LMAX consecutive entries of one row (MMItems, spmv_plan.h) -- and the items are sorted by length,
// longest first.  A group of KTL lanes (VW adjacent columns each, one 16-byte load of the X row segment per lane and
// entry) owns one item, so the 32/KTL groups of a warp run loops of equal length, nothing waits, and the long items are
// scheduled first.  Single-item rows write Y; the pieces of longer rows write partial sums that spmm_item_reduce_kernel
// adds up in piece order (no atomics: deterministic).  Per entry the sum order is the storage order.
// ---------------------------------------------------------------------------
static constexpr int MMI_MAXL = 256;
static constexpr int MMI_LONG_PIECES = 64;  // rows of more pieces are added up by a whole CTA (spmm_item_reduce_long_kernel)

// histogram of item lengths (0..lmax), number of multi-piece rows and of their pieces
__global__ void __launch_bounds__(256) mmi_count_kernel(int m, const int* __restrict__ row_ptr, int lmax, int* __restrict__ hist,
                                                        int* __restrict__ counters) {
  __shared__ int sh[MMI_MAXL + 1];
  __shared__ int sc[3];
  for (int i = threadIdx.x; i <= lmax; i += 256) sh[i] = 0;
  if (threadIdx.x < 3) sc[threadIdx.x] = 0;
  __syncthreads();
  for (int r = blockIdx.x * 256 + threadIdx.x; r < m; r += gridDim.x * 256) {
    const int len = row_ptr[r + 1] - row_ptr[r];
    const int pieces = len <= lmax ? 1 : (len + lmax - 1) / lmax;
    if (pieces == 1) {
      atomicAdd(&sh[len], 1);
    } else {
      atomicAdd(&sh[lmax], pieces - 1);
      atomicAdd(&sh[len - (pieces - 1) * lmax], 1);
      atomicAdd(&sc[0], 1);
      atomicAdd(&sc[1], pieces);
      if (pieces > MMI_LONG_PIECES) atomicAdd(&sc[2], 1);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i <= lmax; i += 256)
    if (sh[i]) atomicAdd(&hist[i], sh[i]);
  if (threadIdx.x < 2 && sc[threadIdx.x]) atomicAdd(&counters[threadIdx.x], sc[threadIdx.x]);
  if (threadIdx.x == 2 && sc[2]) atomicAdd(&counters[4], sc[2]);
}

// cursor[len] = first position of the items of that length (longest first); block-aggregated reservation of ranges
__global__ void __launch_bounds__(256) mmi_fill_kernel(int m, const int* __restrict__ row_ptr, int lmax, int* __restrict__ cursor,
                                                       int* __restrict__ counters /* [2] multi cursor, [3] partial cursor, [5] long-row cursor */,
                                                       int4* __restrict__ items, int4* __restrict__ multi, int n_multi) {
  __shared__ int sh[MMI_MAXL + 1];
  __shared__ int sbase[MMI_MAXL + 1];
  const int passes = (m + (int)(gridDim.x * 256) - 1) / (int)(gridDim.x * 256);
  for (int it = 0; it < passes; ++it) {
    const int r = (it * gridDim.x + blockIdx.x) * 256 + threadIdx.x;
    for (int i = threadIdx.x; i <= lmax; i += 256) sh[i] = 0;
    __syncthreads();
    int len = 0, pieces = 0, rank_last = 0, rank_full = 0, last = 0;
    if (r < m) {
      len = row_ptr[r + 1] - row_ptr[r];
      pieces = len <= lmax ? 1 : (len + lmax - 1) / lmax;
      last = len - (pieces - 1) * lmax;
      if (pieces > 1) rank_full = atomicAdd(&sh[lmax], pieces - 1);
      rank_last = atomicAdd(&sh[last], 1);
    }
    __syncthreads();
    for (int i = threadIdx.x; i <= lmax; i += 256)
      if (sh[i]) sbase[i] = atomicAdd(&cursor[i], sh[i]);
    __syncthreads();
    if (r < m) {
      const int e0 = row_ptr[r];
      if (pieces == 1) {
        items[sbase[len] + rank_last] = make_int4(r, e0, len, -1);
      } else {
        const int slot0 = atomicAdd(&counters[3], pieces);
        // rows of many pieces at the END of the list (they get a CTA each in the reduce), the others at the front
        const int mpos = pieces > MMI_LONG_PIECES ? n_multi - 1 - atomicAdd(&counters[5], 1) : atomicAdd(&counters[2], 1);
        multi[mpos] = make_int4(r, slot0, pieces, 0);
        for (int s = 0; s < pieces - 1; ++s) items[sbase[lmax] + rank_full + s] = make_int4(r, e0 + s * lmax, lmax, slot0 + s);
        items[sbase[last] + rank_last] = make_int4(r, e0 + (pieces - 1) * lmax, last, slot0 + pieces - 1);
      }
    }
    __syncthreads();
  }
}

static int plan_analyse_items(MMItems* mi, cudaStream_t st, int lmax, int m, int64_t nnz, const int* row_ptr) {
  const PlanKey key{row_ptr, nullptr, m, -1, nnz, lmax};
  if (mi->key == key) return B200SP_OK;
  mi->release(st);
  DevTmp tmp(st);
  int *hist, *counters;
  B200SP_CUDA_TRY(tmp.alloc(&hist, lmax + 1));
  B200SP_CUDA_TRY(tmp.alloc(&counters, 8));
  B200SP_CUDA_TRY(cudaMemsetAsync(hist, 0, sizeof(int) * (size_t)(lmax + 1), st));
  B200SP_CUDA_TRY(cudaMemsetAsync(counters, 0, sizeof(int) * 8, st));
  const int blocks = std::max(1, std::min((m + 255) / 256, sm_count() * 8));
  mmi_count_kernel<<<blocks, 256, 0, st>>>(m, row_ptr, lmax, hist, counters);
  B200SP_LAUNCH_CHECK();
  int h_hist[MMI_MAXL + 1], h_cnt[8];
  B200SP_CUDA_TRY(cudaMemcpyAsync(h_hist, hist, sizeof(int) * (size_t)(lmax + 1), cudaMemcpyDeviceToHost, st));
  B200SP_CUDA_TRY(cudaMemcpyAsync(h_cnt, counters, sizeof(int) * 8, cudaMemcpyDeviceToHost, st));
  B200SP_CUDA_TRY(cudaStreamSynchronize(st));  // once per matrix
  int h_cur[MMI_MAXL + 1];
  long long total = 0;
  for (int l = lmax; l >= 0; --l) {  // longest first
    h_cur[l] = (int)total;
    total += h_hist[l];
  }
  B200SP_REQUIRE(total <= (long long)INT_MAX, "spmm: too many work items");
  mi->n_items = (int)total;
  mi->n_multi = h_cnt[0];
  mi->n_multi_long = h_cnt[4];
  mi->n_partial = h_cnt[1];
  mi->lmax = lmax;
  B200SP_CUDA_TRY(mi->items.alloc((size_t)std::max(mi->n_items, 1), st));
  B200SP_CUDA_TRY(mi->multi.alloc((size_t)std::max(mi->n_multi, 1), st));
  B200SP_CUDA_TRY(cudaMemcpyAsync(hist, h_cur, sizeof(int) * (size_t)(lmax + 1), cudaMemcpyHostToDevice, st));
  mmi_fill_kernel<<<blocks, 256, 0, st>>>(m, row_ptr, lmax, hist, counters, mi->items, mi->multi, mi->n_multi);
  B200SP_LAUNCH_CHECK();
  B200SP_CUDA_TRY(cudaStreamSynchronize(st));  // h_cur is pageable host memory: consumed before it goes out of scope
  mi->key = key;
  return B200SP_OK;
}

// Cooperative loads: the KTL lanes of a group do not each read the same (col, val) address -- that costs one L1 wavefront
// per group and entry for the column, one for the value and one for the X row: 3 per nonzero at 8 groups per warp, and a
// kernel that did so was bound by exactly that (one wavefront per SM and clock).  The group reads a batch of EB
// consecutive entries with ONE load per lane (adjacent lanes, adjacent entries: the group's EB/KTL loads cover a
// contiguous 32..64-byte run) and passes them round with shuffles, which run on a different pipe: 1 + 2 * 4/32
// wavefronts per nonzero for k = 16 fp32, with EB gathers of X in flight per lane (EB = 4: 40 registers, 6 CTAs per SM;
// EB = 8, 80 registers and 3 CTAs, was slower when tuned).
template <typename S, int VW, int KTL, int EB /* entries per batch */>
__global__ void __launch_bounds__(256)
    spmm_item_coop_kernel(int n_items, const int4* __restrict__ items, int k, const int* __restrict__ col_idx,
                          const S* __restrict__ vals, const S* __restrict__ X, int64_t ldx, S* __restrict__ Y, int64_t ldy,
                          AccT<S>* __restrict__ partial, AccT<S> alpha, AccT<S> beta) {
  using A = AccT<S>;
  constexpr int PL = (EB + KTL - 1) / KTL;    // entries a lane loads per batch (KTL > EB: lanes >= EB load nothing)
  const int64_t gt = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t q = gt / KTL;
  const int t = (int)(gt % KTL);
  if (q >= n_items) return;  // whole groups leave: 256 % KTL == 0
  const unsigned gmask = KTL == 32 ? 0xffffffffu : (((1u << (KTL & 31)) - 1u) << ((threadIdx.x & 31) & ~(KTL - 1)));
  const uint64_t once = l2_policy_evict_first();
  const int4 it = ld_once(items + q, once);
  const int row = it.x, e0 = it.y, len = it.z, slot = it.w;
  const int eend = e0 + len;
  const int nstrips = (k + KTL * VW - 1) / (KTL * VW);
  for (int strip = 0; strip < nstrips; ++strip) {
    const int j = (strip * KTL + t) * VW;
    const bool live = j < k;  // k % VW == 0: a lane's VW columns are all in or all out; dead lanes still load and shuffle
    Acc<A, VW> acc;
#pragma unroll
    for (int c = 0; c < VW; ++c) acc.a[c] = A(0);
    const S* xb = X + (live ? j : 0);
    int e = e0;
    for (; e + EB <= eend; e += EB) {
      int cl[PL];
      S vl[PL];
#pragma unroll
      for (int i = 0; i < PL; ++i) {
        const int idx = i * KTL + t;
        cl[i] = 0;
        vl[i] = S();
        if (KTL <= EB || idx < EB) {
          cl[i] = ld_once(col_idx + e + idx, once);
          vl[i] = ld_once(vals + e + idx, once);
        }
      }
      int c[EB];
      A av[EB];
#pragma unroll
      for (int u = 0; u < EB; ++u) {
        if constexpr (KTL == 1) {
          c[u] = cl[u];
          av[u] = wide(vl[u]);
        } else {
          c[u] = __shfl_sync(gmask, cl[u / KTL], u % KTL, KTL);
          av[u] = wide(__shfl_sync(gmask, vl[u / KTL], u % KTL, KTL));
        }
      }
      if (live) {
        Acc<A, VW> xv[EB];
#pragma unroll
        for (int u = 0; u < EB; ++u) xv[u] = load_x<S, VW>(xb + (int64_t)c[u] * ldx);
#pragma unroll
        for (int u = 0; u < EB; ++u)
#pragma unroll
          for (int cc = 0; cc < VW; ++cc) acc.a[cc] += av[u] * xv[u].a[cc];
      }
    }
    const int rem = eend - e;  // 0 .. EB-1, uniform over the group
    if (rem > 0) {
      int cl[PL];
      S vl[PL];
#pragma unroll
      for (int i = 0; i < PL; ++i) {
        const int idx = i * KTL + t;
        cl[i] = 0;
        vl[i] = S();
        if (idx < rem) {
          cl[i] = ld_once(col_idx + e + idx, once);
          vl[i] = ld_once(vals + e + idx, once);
        }
      }
      int c[EB];
      A av[EB];
#pragma unroll
      for (int u = 0; u < EB; ++u) {
        if constexpr (KTL == 1) {
          c[u] = cl[u];
          av[u] = wide(vl[u]);
        } else {
          c[u] = __shfl_sync(gmask, cl[u / KTL], u % KTL, KTL);
          av[u] = wide(__shfl_sync(gmask, vl[u / KTL], u % KTL, KTL));
        }
      }
      if (live) {
        Acc<A, VW> xv[EB];
#pragma unroll
        for (int u = 0; u < EB - 1; ++u)
          if (u < rem) xv[u] = load_x<S, VW>(xb + (int64_t)c[u] * ldx);
#pragma unroll
        for (int u = 0; u < EB - 1; ++u)
          if (u < rem) {
#pragma unroll
            for (int cc = 0; cc < VW; ++cc) acc.a[cc] += av[u] * xv[u].a[cc];
          }
      }
    }
    if (!live) continue;
    A o[VW];
    if constexpr (std::is_same<S, A>::value) {  // fp32 / fp64: Y and the partial sums share a type, one store
      S* dst;
      if (slot < 0) {
        dst = Y + (int64_t)row * ldy + j;
        item_epilogue<S, VW>(o, acc, alpha, beta, dst);
      } else {
        dst = partial + (int64_t)slot * k + j;  // raw sums; alpha and beta are applied by the reduce kernel
#pragma unroll
        for (int cc = 0; cc < VW; ++cc) o[cc] = acc.a[cc];
      }
      st_vec_once<VW>(dst, o, once);
    } else if (slot < 0) {  // fp16: Y in S, the partial sums in A
      S* dst = Y + (int64_t)row * ldy + j;
      item_epilogue<S, VW>(o, acc, alpha, beta, dst);
      st_vec_once<VW>(dst, o, once);
    } else {
      st_vec_once<VW>(partial + (int64_t)slot * k + j, acc.a, once);
    }
  }
}

// rows of several pieces: Y(row, :) = beta * Y(row, :) + alpha * (sum of the pieces).  One WARP per row: the lanes are
// KC columns x 32/KC interleaved piece subsequences (k = 16: lane = (piece parity, column)); a lane adds its subsequence in
// piece order, a fixed xor tree joins the subsequences -- the order of additions depends on the row alone, so the result is
// reproducible run to run.  (One thread per (row, column) made the longest row of R-MAT scale 23, 2388 pieces, a tail that
// took a fifth of the whole product.)
template <typename S>
__global__ void __launch_bounds__(256)
    spmm_item_reduce_kernel(int n_multi, const int4* __restrict__ multi, int k, const AccT<S>* __restrict__ partial,
                            S* __restrict__ Y, int64_t ldy, AccT<S> alpha, AccT<S> beta) {
  using A = AccT<S>;
  const int lane = threadIdx.x & 31;
  int KC = 1;
  while (KC < k && KC < 32) KC <<= 1;
  const int SUB = 32 / KC;
  const int j0 = lane % KC, sub = lane / KC;
  const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n_multi; w += warps) {
    const int4 d = multi[w];  // (row, first partial slot, pieces, 0)
    for (int jb = 0; jb < k; jb += KC) {
      const int j = jb + j0;
      A sum = A(0);
      if (j < k) {
        const A* src = partial + (int64_t)d.y * k + j;
        for (int s = sub; s < d.z; s += SUB) sum += src[(int64_t)s * k];
      }
      for (int o = 16; o >= KC; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      if (sub == 0 && j < k) {
        S* yp = Y + (int64_t)d.x * ldy + j;
        *yp = narrow<S>((beta == A(0)) ? alpha * sum : beta * wide(*yp) + alpha * sum);
      }
    }
  }
}

// the same for the rows of more than MMI_LONG_PIECES pieces (the hubs of a power-law matrix: 2388 pieces in the longest row of
// R-MAT scale 23), one CTA per row: thread = (piece subsequence, column), 256 / KC subsequences added in piece order each, then
// joined in subsequence order through shared memory by the threads of subsequence 0.  Fixed order: reproducible.
template <typename S>
__global__ void __launch_bounds__(256)
    spmm_item_reduce_long_kernel(int n_long, const int4* __restrict__ multi_long, int k, const AccT<S>* __restrict__ partial,
                                 S* __restrict__ Y, int64_t ldy, AccT<S> alpha, AccT<S> beta) {
  using A = AccT<S>;
  __shared__ A part[256];
  int KC = 1;
  while (KC < k && KC < 32) KC <<= 1;
  const int SUB = 256 / KC;
  const int j0 = threadIdx.x % KC, sub = threadIdx.x / KC;
  for (int w = blockIdx.x; w < n_long; w += gridDim.x) {
    const int4 d = multi_long[w];
    for (int jb = 0; jb < k; jb += KC) {
      const int j = jb + j0;
      A sum = A(0);
      if (j < k) {
        const A* src = partial + (int64_t)d.y * k + j;
        for (int s = sub; s < d.z; s += SUB) sum += src[(int64_t)s * k];
      }
      part[threadIdx.x] = sum;
      __syncthreads();
      if (sub == 0 && j < k) {
        A t = part[j0];
        for (int q = 1; q < SUB; ++q) t += part[q * KC + j0];
        S* yp = Y + (int64_t)d.x * ldy + j;
        *yp = narrow<S>((beta == A(0)) ? alpha * t : beta * wide(*yp) + alpha * t);
      }
      __syncthreads();
    }
  }
}

// the 16-byte item kernels can take row-major X and Y: k, ldx and ldy multiples of the vector width, X and Y 16-byte aligned
template <typename S>
static bool items_vec(int k, int64_t ldx, int64_t ldy, const S* X, const S* Y) {
  constexpr int W = VecOf<S>::W;
  return (k % W == 0) && (ldx % W == 0) && (ldy % W == 0) && ((((uintptr_t)X) | ((uintptr_t)Y)) & 15u) == 0;
}

// the item path on row-major X and Y: the plan's items (built once per matrix), the item kernel, then the reduce kernels
template <typename S>
static int launch_mm_items(b200sp_spmv_plan* p, cudaStream_t st, int m, int k, int64_t nnz, const int* row_ptr,
                           const int* col_idx, const S* vals, const S* X, int64_t ldx, S* Y, int64_t ldy, AccT<S> alpha, AccT<S> beta) {
  using A = AccT<S>;
  int LMAX = 64;  // entries per item (B200SP_SPMM_ITEM_LMAX: 16..256); 64 was the best of 32..256 on R-MAT scale 23 when tuned
  if (const char* e = getenv("B200SP_SPMM_ITEM_LMAX")) {
    const int v = atoi(e);
    if (v >= 16 && v <= MMI_MAXL) LMAX = v;
  }
  MMItems* mi = &p->mm.items;
  int rc = plan_analyse_items(mi, st, LMAX, m, nnz, row_ptr);
  if (rc) return rc;
  B200SP_CUDA_TRY(mi->partial.grow(sizeof(A) * (size_t)mi->n_partial * (size_t)k, st));
  const bool vec = items_vec(k, ldx, ldy, X, Y);
  constexpr int W = VecOf<S>::W;
  const int lanes_needed = vec ? (k + W - 1) / W : k;
  int KTL = 1;
  while (KTL < lanes_needed && KTL < 32) KTL <<= 1;
  const int64_t threads = (int64_t)mi->n_items * KTL;
  const unsigned grid = (unsigned)((threads + 255) / 256);
  if (grid > 0) {
#define B200SP_MMI(V, L)                                                                                                   \
  case L:                                                                                                                  \
    spmm_item_coop_kernel<S, V, L, 4><<<grid, 256, 0, st>>>(mi->n_items, mi->items, k, col_idx, vals, X, ldx, Y, ldy,      \
                                                            mi->partial.as<A>(), alpha, beta);                             \
    break;
    if (vec) {
      switch (KTL) { B200SP_MMI(W, 1) B200SP_MMI(W, 2) B200SP_MMI(W, 4) B200SP_MMI(W, 8) B200SP_MMI(W, 16) B200SP_MMI(W, 32) }
    } else {
      switch (KTL) { B200SP_MMI(1, 1) B200SP_MMI(1, 2) B200SP_MMI(1, 4) B200SP_MMI(1, 8) B200SP_MMI(1, 16) B200SP_MMI(1, 32) }
    }
#undef B200SP_MMI
    B200SP_LAUNCH_CHECK();
  }
  const int n_short = mi->n_multi - mi->n_multi_long;
  if (n_short > 0) {
    const int g = (int)std::min<int64_t>(((int64_t)n_short + 7) / 8, (int64_t)sm_count() * 16);  // a warp per row
    spmm_item_reduce_kernel<S><<<std::max(g, 1), 256, 0, st>>>(n_short, mi->multi, k, mi->partial.as<const A>(), Y, ldy, alpha, beta);
    B200SP_LAUNCH_CHECK();
  }
  if (mi->n_multi_long > 0) {
    const int g = std::min(mi->n_multi_long, sm_count() * 8);  // a CTA per row
    spmm_item_reduce_long_kernel<S><<<g, 256, 0, st>>>(mi->n_multi_long, mi->multi + n_short, k, mi->partial.as<const A>(), Y, ldy, alpha, beta);
    B200SP_LAUNCH_CHECK();
  }
  return B200SP_OK;
}

// Y = beta*Y + alpha*op(A)*X for S = double, float and __half (binary16 A, X and Y with fp32 products, sums and epilogue:
// include/b200sparse.h, DESIGN.md 4.3).  Mode N with a plan takes the item path, through row-major copies for LayoutLeft
// operands when k >= 4; without a plan, LayoutRight X and Y take spmm_rowmajor_kernel (fp32 / fp64) and everything else
// spmm_general_kernel.  T/H scatter with atomics.
template <typename S>
static int spmm_impl(b200sp_spmv_plan* p, cudaStream_t st, char mode, int m, int n, int64_t nnz, int k, AccT<S> alpha,
                     const int* row_ptr, const int* col_idx, const S* vals, const S* X, int64_t ldx, int xrm,
                     AccT<S> beta, S* Y, int64_t ldy, int yrm) {
  using A = AccT<S>;
  constexpr bool f16 = std::is_same<S, __half>::value;
  B200SP_REQUIRE(m >= 0 && n >= 0 && nnz >= 0 && k >= 0, "spmm: negative dimension");
  bool trans;
  switch (mode) {
    case 'N': case 'n': case 'C': case 'c': trans = false; break;
    case 'T': case 't': case 'H': case 'h': trans = true; break;
    default: set_error("Invalid transpose mode %c for KokkosSparse::spmv()", mode); return B200SP_ERR_INVALID_ARGUMENT;
  }
  const int64_t xrows = trans ? m : n, yrows = trans ? n : m;
  const int64_t xr = xrm ? ldx : 1, xc = xrm ? 1 : ldx;
  const int64_t yr = yrm ? ldy : 1, yc = yrm ? 1 : ldy;
  if (k == 0 || yrows == 0) return B200SP_OK;
  B200SP_REQUIRE(Y != nullptr, "spmm: Y is null");
  B200SP_REQUIRE((xrm ? ldx >= k : ldx >= xrows) && (yrm ? ldy >= k : ldy >= yrows), "spmm: leading dimension too small");
  const int grid_elem = (int)std::min<int64_t>((yrows * k + 255) / 256, (int64_t)sm_count() * 16);
  if (alpha == A(0) || m == 0 || n == 0 || nnz == 0) {
    if (beta != A(1)) {
      scale2d_kernel<S><<<std::max(grid_elem, 1), 256, 0, st>>>(yrows, k, beta, Y, yr, yc);
      B200SP_LAUNCH_CHECK();
    }
    return B200SP_OK;
  }
  B200SP_REQUIRE(row_ptr && col_idx && vals && X, "spmm: null pointer argument");
  if (trans) {
    const int g = (int)std::min<int64_t>(((int64_t)m * k + 255) / 256, (int64_t)sm_count() * 16);
    if constexpr (f16) {  // fp32 scratch, then one rounding per entry of Y
      DevTmp tmp(st);
      float* acc = nullptr;
      const size_t acc_bytes = sizeof(float) * (size_t)yrows * (size_t)k;
      if (p) {
        B200SP_CUDA_TRY(p->mm.yt.grow(acc_bytes, st));
        acc = p->mm.yt.as<float>();
      } else {
        B200SP_CUDA_TRY(tmp.alloc(&acc, (size_t)yrows * (size_t)k));
      }
      B200SP_CUDA_TRY(cudaMemsetAsync(acc, 0, acc_bytes, st));
      spmm_transpose_acc_kernel<<<std::max(g, 1), 256, 0, st>>>(m, k, row_ptr, col_idx, vals, X, xr, xc, acc);
      B200SP_LAUNCH_CHECK();
      spmm_acc_epilogue_kernel<<<std::max(grid_elem, 1), 256, 0, st>>>(yrows, k, acc, alpha, beta, Y, yr, yc);
      B200SP_LAUNCH_CHECK();
    } else {
      if (beta != A(1)) {
        scale2d_kernel<S><<<std::max(grid_elem, 1), 256, 0, st>>>(yrows, k, beta, Y, yr, yc);
        B200SP_LAUNCH_CHECK();
      }
      spmm_transpose_kernel<S><<<std::max(g, 1), 256, 0, st>>>(m, k, row_ptr, col_idx, vals, X, xr, xc, Y, yr, yc, alpha);
      B200SP_LAUNCH_CHECK();
    }
    set_last_kernel(p, "spmm_transpose");
    return B200SP_OK;
  }
  if (p && xrm && yrm) {
    set_last_kernel(p, items_vec(k, ldx, ldy, X, Y) ? "spmm_items_vec" : "spmm_items");
    return launch_mm_items<S>(p, st, m, k, nnz, row_ptr, col_idx, vals, X, ldx, Y, ldy, alpha, beta);
  }
  // LayoutLeft operands: with a plan and k >= 4, relayout to row-major scratch and take the item path
  if (p && k >= 4) {
    B200SP_CUDA_TRY(p->mm.xt.grow(xrm ? 0 : sizeof(S) * (size_t)xrows * k, st));
    B200SP_CUDA_TRY(p->mm.yt.grow(yrm ? 0 : sizeof(S) * (size_t)yrows * k, st));
    S* xt = p->mm.xt.as<S>();
    S* yt = p->mm.yt.as<S>();
    auto rl_grid = [](int64_t rows) { return (unsigned)std::max<int64_t>(1, std::min<int64_t>((rows + 127) / 128, (int64_t)sm_count() * 16)); };
    const S* Xr = X;
    int64_t ldxr = ldx;
    if (!xrm) {
      relayout_kernel<S, true><<<rl_grid(xrows), 256, 0, st>>>(xrows, k, xt, X, nullptr, xr, xc);
      B200SP_LAUNCH_CHECK();
      Xr = xt;
      ldxr = k;
    }
    S* Yr = Y;
    int64_t ldyr = ldy;
    if (!yrm) {
      Yr = yt;
      ldyr = k;
      if (beta != A(0)) {
        relayout_kernel<S, true><<<rl_grid(yrows), 256, 0, st>>>(yrows, k, Yr, Y, nullptr, yr, yc);
        B200SP_LAUNCH_CHECK();
      }
    }
    if (int rc = launch_mm_items<S>(p, st, m, k, nnz, row_ptr, col_idx, vals, Xr, ldxr, Yr, ldyr, alpha, beta)) return rc;
    if (!yrm) {
      relayout_kernel<S, false><<<rl_grid(yrows), 256, 0, st>>>(yrows, k, Yr, nullptr, Y, yr, yc);
      B200SP_LAUNCH_CHECK();
    }
    set_last_kernel(p, "spmm_relayout+items");
    return B200SP_OK;
  }
  if constexpr (!f16) {
    if (xrm && yrm) return launch_rowmajor<S>(st, m, k, row_ptr, col_idx, vals, X, ldx, Y, ldy, alpha, beta);  // no plan
  }
  const int g = (int)std::min<int64_t>(((int64_t)m * k + 255) / 256, (int64_t)sm_count() * 16);
  spmm_general_kernel<S><<<std::max(g, 1), 256, 0, st>>>(m, k, row_ptr, col_idx, vals, X, xr, xc, Y, yr, yc, alpha, beta);
  B200SP_LAUNCH_CHECK();
  set_last_kernel(p, "spmm_general");
  return B200SP_OK;
}

}  // namespace b200sp

using namespace b200sp;

extern "C" {
int b200sp_spmm_f64_i32(b200sp_spmv_plan* plan, void* stream, char mode, int m, int n, int64_t nnz, int k,
                        double alpha, const int* row_ptr, const int* col_idx, const double* vals, const double* X,
                        int64_t ldx, int x_row_major, double beta, double* Y, int64_t ldy, int y_row_major) {
  return spmm_impl<double>(plan, (cudaStream_t)stream, mode, m, n, nnz, k, alpha, row_ptr, col_idx, vals, X, ldx,
                           x_row_major, beta, Y, ldy, y_row_major);
}
int b200sp_spmm_f32_i32(b200sp_spmv_plan* plan, void* stream, char mode, int m, int n, int64_t nnz, int k,
                        float alpha, const int* row_ptr, const int* col_idx, const float* vals, const float* X,
                        int64_t ldx, int x_row_major, float beta, float* Y, int64_t ldy, int y_row_major) {
  return spmm_impl<float>(plan, (cudaStream_t)stream, mode, m, n, nnz, k, alpha, row_ptr, col_idx, vals, X, ldx,
                          x_row_major, beta, Y, ldy, y_row_major);
}
int b200sp_spmm_f16_i32(b200sp_spmv_plan* plan, void* stream, char mode, int m, int n, int64_t nnz, int k, float alpha,
                        const int* row_ptr, const int* col_idx, const uint16_t* vals, const uint16_t* X, int64_t ldx,
                        int x_row_major, float beta, uint16_t* Y, int64_t ldy, int y_row_major) {
  static_assert(sizeof(__half) == sizeof(uint16_t), "binary16 bit patterns");
  return spmm_impl<__half>(plan, (cudaStream_t)stream, mode, m, n, nnz, k, alpha, row_ptr, col_idx, reinterpret_cast<const __half*>(vals),
                           reinterpret_cast<const __half*>(X), ldx, x_row_major, beta, reinterpret_cast<__half*>(Y), ldy, y_row_major);
}
}
