// spmm.cu -- rank-2 (multivector) CrsMatrix SpMV: Y = beta*Y + alpha*op(A)*X.
//
// Replaces the reference's Kokkos::Cuda legs
//   native  SPMV_MV_LayoutLeft_Functor   sparse/impl/KokkosSparse_spmv_impl.hpp:634-1004,1057-1119
//   native  SPMV_MV_Transpose_Functor    sparse/impl/KokkosSparse_spmv_impl.hpp:547-632,1163-1229
//   TPL     cusparseSpMM                 sparse/tpls/KokkosSparse_spmv_mv_tpl_spec_decl.hpp:97-196
//
// Kernels:
//   spmm_rowmajor_kernel  X, Y LayoutRight: a group of KT lanes owns one row of
//                         A and one strip of <= KT columns; (col,val) pairs are
//                         loaded coalesced KT at a time and broadcast by shuffle,
//                         X rows are read as contiguous KT*sizeof(S) segments.
//                         One pass over A per 32-column strip, no reduction.
//   spmm_general_kernel   any LayoutLeft / LayoutRight mix: thread per (row, j).
//   spmm_transpose_kernel T/H modes: Y pre-scaled, atomicAdd scatter.
// Column-major (LayoutLeft) X with k >= 4 goes through a transposed copy so the
// gather touches one segment per nonzero instead of k sectors (DESIGN.md 3.4).
#include <limits.h>
#include "common.cuh"
#include "tile_ring.cuh"
#include "spmm_items.h"
#include <algorithm>
#include <atomic>
#include <stdlib.h>

struct b200sp_spmv_plan;  // defined in spmv.cu

namespace b200sp {

// scratch owned by the plan (spmv.cu)
int plan_mv_scratch(b200sp_spmv_plan* p, cudaStream_t st, size_t xt_bytes, size_t yt_bytes, void** xt, void** yt);
void plan_set_last_kernel(b200sp_spmv_plan* p, const char* s);
MMItems* plan_mm_items(b200sp_spmv_plan* p);

template <typename S>
__global__ void scale2d_kernel(int64_t rows, int k, S beta, S* __restrict__ Y, int64_t yr, int64_t yc) {
  const int64_t total = rows * k;
  const bool by_rows = (yc == 1 || yr != 1);  // walk memory-contiguously for either layout
  if (total <= (int64_t)INT32_MAX) {  // 32-bit index arithmetic: a 64-bit division per element costs more than the element's traffic
    const unsigned t32 = (unsigned)total, k32 = (unsigned)k, r32 = (unsigned)rows, step = gridDim.x * blockDim.x;
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < t32; i += step) {
      unsigned r, j;
      if (by_rows) { r = i / k32; j = i - r * k32; } else { j = i / r32; r = i - j * r32; }
      S* p = &Y[(int64_t)r * yr + (int64_t)j * yc];
      *p = (beta == S(0)) ? S(0) : beta * *p;
    }
    return;
  }
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r, j;
    if (by_rows) { r = i / k; j = i % k; } else { j = i / rows; r = i % rows; }
    S* p = &Y[r * yr + j * yc];
    *p = (beta == S(0)) ? S(0) : beta * *p;
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
                        S* __restrict__ Y, int64_t yr, int64_t yc, S alpha, S beta) {
  const int64_t total = (int64_t)m * k;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / k), j = (int)(i % k);
    S acc = S(0);
    for (int e = row_ptr[r]; e < row_ptr[r + 1]; ++e) acc += vals[e] * ldg(X + (int64_t)col_idx[e] * xr + (int64_t)j * xc);
    acc *= alpha;
    S* yp = Y + (int64_t)r * yr + (int64_t)j * yc;
    *yp = (beta == S(0)) ? acc : beta * *yp + acc;
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

// ---------------------------------------------------------------------------
// nnz-split kernel (power-law rows): a group of KT lanes (one per column of the strip) walks a chunk
// of Q consecutive nonzeros; rows that lie inside the chunk are stored directly, the (at most two)
// rows cut by the chunk borders are pre-scaled by spmm_prescale_split_rows and accumulated with
// atomicAdd.  chunk_row[c] = row holding nonzero c*Q (built once per matrix, cached in the plan).
// ---------------------------------------------------------------------------
__global__ void build_chunk_rows_kernel(int m, const int* __restrict__ row_ptr, int n_chunks, int Q,
                                        int* __restrict__ chunk_row) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_chunks) return;
  // first row r with row_ptr[r+1] > c*Q
  const int64_t pos = (int64_t)c * Q;
  int lo = 0, hi = m;
  while (lo < hi) {
    const int mid = lo + ((hi - lo) >> 1);
    if ((int64_t)row_ptr[mid + 1] <= pos) lo = mid + 1;
    else hi = mid;
  }
  chunk_row[c] = lo;
}

template <typename S>
__global__ void spmm_prescale_split_rows(int m, int k, int Q, const int* __restrict__ row_ptr, S beta,
                                         S* __restrict__ Y, int64_t ldy) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < m; r += gridDim.x * blockDim.x) {
    const int s = row_ptr[r], e = row_ptr[r + 1];
    if (e > s && (s / Q) != ((e - 1) / Q)) {
      S* yp = Y + (int64_t)r * ldy;
      for (int j = 0; j < k; ++j) yp[j] = (beta == S(0)) ? S(0) : beta * yp[j];
    }
  }
}

template <typename S, int KT>
__global__ void __launch_bounds__(256)
    spmm_split_kernel(int m, int k, int64_t nnz, int Q, int n_chunks, const int* __restrict__ chunk_row,
                      const int* __restrict__ row_ptr, const int* __restrict__ col_idx, const S* __restrict__ vals,
                      const S* __restrict__ X, int64_t ldx, S* __restrict__ Y, int64_t ldy, S alpha, S beta) {
  constexpr int GPW = 32 / KT;
  const int lane = threadIdx.x & 31;
  const int grp = lane / KT, t = lane % KT;
  const unsigned gmask = (KT == 32) ? 0xffffffffu : (((1u << KT) - 1u) << (grp * KT));
  const int gbase = grp * KT;  // shuffle source lanes are absolute
  const int nstrips = (k + KT - 1) / KT;
  const int64_t gid = ((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5) * GPW + grp;
  const int64_t ngroups = (((int64_t)gridDim.x * blockDim.x) >> 5) * GPW;
  const int64_t work_total = (int64_t)n_chunks * nstrips;
  for (int64_t w = gid; w < work_total; w += ngroups) {
    const int chunk = (int)(w / nstrips);
    const int j = (int)(w % nstrips) * KT + t;
    const bool jok = j < k;
    // chunk 0 starts at the first entry of row 0: the windows of the 64-bit-offset path (spmv64.cu) pass relative row maps
    // that start at 1..3, and the entries before row_ptr[0] belong to the previous window's last row
    const int64_t cq = (int64_t)chunk * Q;
    const int64_t c0 = (chunk == 0) ? (int64_t)row_ptr[0] : cq;
    const int64_t c1 = (cq + Q < nnz) ? cq + Q : nnz;
    int row = (chunk == 0) ? 0 : chunk_row[chunk];
    // cache of KT row ends: lane t holds row_ptr[ebase + 1 + t]
    int ebase = row;
    int ends = row_ptr[min(ebase + 1 + t, m)];
    int64_t row_start = row_ptr[row];
    int64_t next_end = __shfl_sync(gmask, ends, gbase);
    S acc = S(0);
    auto flush = [&]() {
      // row `row` ends at next_end; acc holds this chunk's share of it
      if (jok) {
        S* yp = Y + (int64_t)row * ldy + j;
        const S a = alpha * acc;
        if (row_start >= c0 && next_end <= c1) *yp = (beta == S(0)) ? a : beta * *yp + a;
        else atomicAdd(yp, a);
      }
      acc = S(0);
      row_start = next_end;
      ++row;
      if (row - ebase == KT) {
        ebase = row;
        ends = row_ptr[min(ebase + 1 + t, m)];
      }
      next_end = __shfl_sync(gmask, ends, gbase + (row - ebase));
    };
    for (int64_t b = c0; b < c1; b += KT) {
      const int64_t e = b + t;
      int c = 0;
      S v = S(0);
      if (e < c1) {
        c = ld_stream(col_idx + e);
        v = ld_stream(vals + e);
      }
      const int nb = (int)((c1 - b < KT) ? (c1 - b) : KT);
      S xv[KT];
#pragma unroll
      for (int u = 0; u < KT; ++u) {
        const int cu = __shfl_sync(gmask, c, gbase + u);
        xv[u] = (u < nb && jok) ? ldg(X + (int64_t)cu * ldx + j) : S(0);
      }
#pragma unroll
      for (int u = 0; u < KT; ++u) {
        const S vu = __shfl_sync(gmask, v, gbase + u);
        if (u < nb) {
          while (b + u >= next_end) flush();  // uniform within the group
          acc += vu * xv[u];
        }
      }
    }
    // rows ending inside (or exactly at the end of) this chunk, incl. empty rows
    while (row < m && next_end <= c1) flush();
    // a row that continues into the next chunk: its share goes in atomically
    if (row < m && row_start < c1 && jok) atomicAdd(Y + (int64_t)row * ldy + j, alpha * acc);
  }
}


// Vectorised variant: every lane owns VW adjacent columns (one 16-byte load of the X row per nonzero),
// a group of KT lanes covers KT*VW columns, so a warp advances 32/KT chunks at once.  Needs k, ldx,
// ldy multiples of VW and 16-byte aligned X / Y.
template <typename S> struct VecOf;
template <> struct VecOf<float> { using type = float4; static constexpr int W = 4; };
template <> struct VecOf<double> { using type = double2; static constexpr int W = 2; };
__device__ __forceinline__ void vec_unpack(const float4& v, float* a) { a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w; }
__device__ __forceinline__ void vec_unpack(const double2& v, double* a) { a[0] = v.x; a[1] = v.y; }
__device__ __forceinline__ float4 vec_pack(const float* a) { return make_float4(a[0], a[1], a[2], a[3]); }
__device__ __forceinline__ double2 vec_pack(const double* a) { return make_double2(a[0], a[1]); }

// ---------------------------------------------------------------------------
// Tile kernel (B200SP_SPMM_KERNEL=tile|tilev; row-major X and Y): the matrix is streamed ONCE, whatever k,
// through the same TMA-fed shared-memory ring as the rank-1 kernel (tile_ring.cuh); a group of KTL lanes
// owns one row at a time (rows dealt round-robin to the groups like spmv_tile_kernel does), every lane
// accumulates VW adjacent columns in registers: per nonzero a broadcast read of (col, val) from shared
// memory, one gather of the X row segment (VW = 1: 4/8-byte, VW = 4/2: 16-byte loads) and VW FMAs -- no
// shuffles, no atomics, no row bookkeeping in the inner loop, deterministic.  Rows longer than the tile
// row limit are cut into segments (plan_analyse_mm, spmv.cu) and done by spmm_seg_kernel.
// ---------------------------------------------------------------------------
template <typename S, int VW>
struct Acc {
  S a[VW];
};

template <typename S, int VW>
__device__ __forceinline__ Acc<S, VW> load_x(const S* __restrict__ p) {
  static_assert(VW == 1 || VW == VecOf<S>::W, "VW is 1 or the 16-byte vector width");
  Acc<S, VW> r;
  if constexpr (VW == 1) {
    r.a[0] = ldg(p);
  } else {
    using V = typename VecOf<S>::type;
    const V v = __ldg(reinterpret_cast<const V*>(p));
    vec_unpack(v, r.a);
  }
  return r;
}

template <typename S, int VW, int KTL, int NW, int STAGES, int CAP, int UNR>
__global__ void __launch_bounds__((NW + 1) * 32)
    spmm_tile_kernel(int m, int k, int64_t nnz, int n_tiles, int LMAX, const int4* __restrict__ tiles,
                     const int* __restrict__ row_ptr, const int* __restrict__ col_idx, const S* __restrict__ vals,
                     const S* __restrict__ X, int64_t ldx, S* __restrict__ Y, int64_t ldy, S alpha, S beta) {
  using Ring = TileRing<S, CAP, STAGES>;
  constexpr int RCAP = Ring::RCAP;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Ring& sm = *reinterpret_cast<Ring*>(smem_raw);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  tile_ring_init(sm, NW);
  if (warp == NW) {
    tile_ring_produce<S, CAP, STAGES>(sm, lane, m, nnz, n_tiles, tiles, row_ptr, col_idx, vals);
    return;
  }
  constexpr int RPW = 32 / KTL;  // rows per warp
  const int sub = lane / KTL, t = lane % KTL;
  const int nstrips = (k + KTL * VW - 1) / (KTL * VW);
  for (int it = 0;; ++it) {
    const int64_t tile = blockIdx.x + (int64_t)it * gridDim.x;
    if (tile >= n_tiles) break;
    const int stage = it % STAGES;
    const uint32_t ph = (uint32_t)(it / STAGES) & 1u;
    mbar_wait(&sm.full[stage], ph);
    const int4 d = sm.desc[stage];
    const int r0 = d.x, r1 = d.y;
    const int s_al = d.z & ~3;
    const int r0_al = r0 & ~3;
    const S* sv = sm.vals[stage];
    const int* sc = sm.cols[stage];
    const int* sr = sm.rows[stage];
    const int g_first = r0 / RPW;
    int g = g_first + ((warp - g_first % NW) + NW) % NW;
    for (; g * RPW < r1; g += NW) {
      const int r = g * RPW + sub;
      const bool valid = (r >= r0) && (r < r1);
      int rs = 0, re = 0;
      if (valid) {
        const int o = r - r0_al;
        if (o + 1 < RCAP) {
          rs = sr[o];
          re = sr[o + 1];
        } else {
          rs = row_ptr[r];
          re = row_ptr[r + 1];
        }
      }
      const bool is_long = (re - rs) > LMAX;
      if (is_long) re = rs;
      const int jbeg = rs - s_al, jend = re - s_al;
      for (int strip = 0; strip < nstrips; ++strip) {
        const int j = (strip * KTL + t) * VW;
        const bool jok = j < k;  // k % VW == 0: a lane's VW columns are all in or all out
        Acc<S, VW> acc;
#pragma unroll
        for (int q = 0; q < VW; ++q) acc.a[q] = S(0);
        for (int e0 = jbeg; e0 < jend; e0 += UNR) {
          int c[UNR];
          S av[UNR];
          Acc<S, VW> xv[UNR];
#pragma unroll
          for (int u = 0; u < UNR; ++u) {
            const bool ok = e0 + u < jend;
            c[u] = ok ? sc[e0 + u] : 0;
            av[u] = ok ? sv[e0 + u] : S(0);
          }
#pragma unroll
          for (int u = 0; u < UNR; ++u) {
            if (jok && e0 + u < jend) {
              xv[u] = load_x<S, VW>(X + (int64_t)c[u] * ldx + j);
            } else {
#pragma unroll
              for (int q = 0; q < VW; ++q) xv[u].a[q] = S(0);
            }
          }
#pragma unroll
          for (int u = 0; u < UNR; ++u)
#pragma unroll
            for (int q = 0; q < VW; ++q) acc.a[q] += av[u] * xv[u].a[q];
        }
        if (valid && !is_long && jok) {
          S* yp = Y + (int64_t)r * ldy + j;
          S o[VW];
          if (beta == S(0)) {
#pragma unroll
            for (int q = 0; q < VW; ++q) o[q] = alpha * acc.a[q];
          } else {
            const Acc<S, VW> old = load_x<S, VW>(yp);
#pragma unroll
            for (int q = 0; q < VW; ++q) o[q] = beta * old.a[q] + alpha * acc.a[q];
          }
          if constexpr (VW == 1) {
            yp[0] = o[0];
          } else {
            using V = typename VecOf<S>::type;
            *reinterpret_cast<V*>(yp) = vec_pack(o);
          }
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm.empty[stage]);
  }
}

// rows of several segments: y_row = beta*y_row before the pieces are added atomically
template <typename S>
__global__ void __launch_bounds__(256)
    spmm_seg_prescale_kernel(const int4* __restrict__ segs, const int* __restrict__ n_seg_ptr, int k, S beta,
                             S* __restrict__ Y, int64_t ldy) {
  const int n_seg = *n_seg_ptr;
  const int64_t total = (int64_t)n_seg * k;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int4 d = segs[i / k];
    if ((d.w & 3) == 3) {
      S* yp = Y + (int64_t)d.x * ldy + (i % k);
      *yp = (beta == S(0)) ? S(0) : beta * *yp;
    }
  }
}

// one CTA (256 threads = 256/KT groups of KT lanes) per segment of a long row
template <typename S, int KT>
__global__ void __launch_bounds__(256)
    spmm_seg_kernel(const int4* __restrict__ segs, const int* __restrict__ n_seg_ptr, int k,
                    const int* __restrict__ col_idx, const S* __restrict__ vals, const S* __restrict__ X, int64_t ldx,
                    S* __restrict__ Y, int64_t ldy, S alpha, S beta) {
  constexpr int G = 256 / KT;
  constexpr int UNR = 4;
  __shared__ S red[G][KT];
  const int grp = threadIdx.x / KT, t = threadIdx.x % KT;
  const int n_seg = *n_seg_ptr;
  const int nstrips = (k + KT - 1) / KT;
  for (int q = blockIdx.x; q < n_seg; q += gridDim.x) {
    const int4 d = segs[q];
    const int row = d.x, e0 = d.y, e1 = d.z;
    const bool multi = (d.w & 1) != 0;
    for (int strip = 0; strip < nstrips; ++strip) {
      const int j = strip * KT + t;
      const bool jok = j < k;
      S acc = S(0);
      for (int e = e0 + grp; e < e1; e += G * UNR) {
        int c[UNR];
        S av[UNR], xv[UNR];
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
          const int ee = e + u * G;
          const bool ok = ee < e1;
          c[u] = ok ? ld_stream(col_idx + ee) : 0;
          av[u] = ok ? ld_stream(vals + ee) : S(0);
        }
#pragma unroll
        for (int u = 0; u < UNR; ++u) xv[u] = (jok && e + u * G < e1) ? ldg(X + (int64_t)c[u] * ldx + j) : S(0);
#pragma unroll
        for (int u = 0; u < UNR; ++u) acc += av[u] * xv[u];
      }
      red[grp][t] = acc;
      __syncthreads();
      if (grp == 0 && jok) {
        S sum = S(0);
#pragma unroll 4
        for (int gg = 0; gg < G; ++gg) sum += red[gg][t];
        S* yp = Y + (int64_t)row * ldy + j;
        const S a = alpha * sum;
        if (multi) atomicAdd(yp, a);
        else *yp = (beta == S(0)) ? a : beta * *yp + a;
      }
      __syncthreads();
    }
  }
}

// 16-byte-load flavour of spmm_seg_kernel (opt-in, B200SP_SPMM_SEG=vec): groups of KTL lanes with VW adjacent columns
// each (the tile kernel's vec layout), so that a 256-thread CTA keeps 256/KTL nonzeros' X rows in flight per step
// instead of 256/KT; partial sums are reduced by shuffles inside a warp and through shared memory across the 8 warps.
template <typename S, int KTL>
__global__ void __launch_bounds__(256)
    spmm_seg_vec_kernel(const int4* __restrict__ segs, const int* __restrict__ n_seg_ptr, int k,
                        const int* __restrict__ col_idx, const S* __restrict__ vals, const S* __restrict__ X, int64_t ldx,
                        S* __restrict__ Y, int64_t ldy, S alpha, S beta) {
  constexpr int VW = VecOf<S>::W;
  constexpr int G = 256 / KTL;       // groups per CTA
  constexpr int GPW = 32 / KTL;      // groups per warp
  constexpr int UNR = 4;
  __shared__ S red[8][KTL * VW];
  const int grp = threadIdx.x / KTL, t = threadIdx.x % KTL;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_seg = *n_seg_ptr;
  const int nstrips = (k + KTL * VW - 1) / (KTL * VW);
  for (int q = blockIdx.x; q < n_seg; q += gridDim.x) {
    const int4 d = segs[q];
    const int row = d.x, e0 = d.y, e1 = d.z;
    const bool multi = (d.w & 1) != 0;
    for (int strip = 0; strip < nstrips; ++strip) {
      const int j = (strip * KTL + t) * VW;
      const bool jok = j < k;
      Acc<S, VW> acc;
#pragma unroll
      for (int c = 0; c < VW; ++c) acc.a[c] = S(0);
      for (int e = e0 + grp; e < e1; e += G * UNR) {
        int c[UNR];
        S av[UNR];
        Acc<S, VW> xv[UNR];
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
          const int ee = e + u * G;
          const bool ok = ee < e1;
          c[u] = ok ? ld_stream(col_idx + ee) : 0;
          av[u] = ok ? ld_stream(vals + ee) : S(0);
        }
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
          if (jok && e + u * G < e1) {
            xv[u] = load_x<S, VW>(X + (int64_t)c[u] * ldx + j);
          } else {
#pragma unroll
            for (int cc = 0; cc < VW; ++cc) xv[u].a[cc] = S(0);
          }
        }
#pragma unroll
        for (int u = 0; u < UNR; ++u)
#pragma unroll
          for (int cc = 0; cc < VW; ++cc) acc.a[cc] += av[u] * xv[u].a[cc];
      }
      // groups of one warp: lanes with the same t are KTL apart
#pragma unroll
      for (int o = KTL; o < 32; o <<= 1)
#pragma unroll
        for (int cc = 0; cc < VW; ++cc) acc.a[cc] += __shfl_xor_sync(0xffffffffu, acc.a[cc], o);
      if (lane < KTL) {
#pragma unroll
        for (int cc = 0; cc < VW; ++cc) red[warp][lane * VW + cc] = acc.a[cc];
      }
      __syncthreads();
      if (threadIdx.x < KTL && jok) {
        S* yp = Y + (int64_t)row * ldy + j;
#pragma unroll
        for (int cc = 0; cc < VW; ++cc) {
          S sum = S(0);
#pragma unroll
          for (int w = 0; w < 8; ++w) sum += red[w][threadIdx.x * VW + cc];
          const S a = alpha * sum;
          if (multi) atomicAdd(yp + cc, a);
          else yp[cc] = (beta == S(0)) ? a : beta * yp[cc] + a;
        }
      }
      __syncthreads();
    }
  }
  (void)GPW;
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

template <typename S, int KT>
__global__ void __launch_bounds__(256)
    spmm_split_vec_kernel(int m, int k, int64_t nnz, int Q, int n_chunks, const int* __restrict__ chunk_row,
                          const int* __restrict__ row_ptr, const int* __restrict__ col_idx, const S* __restrict__ vals,
                          const S* __restrict__ X, int64_t ldx, S* __restrict__ Y, int64_t ldy, S alpha, S beta) {
  using V = typename VecOf<S>::type;
  constexpr int VW = VecOf<S>::W;
  constexpr int GPW = 32 / KT;
  constexpr int EB = (KT >= 8) ? 1 : (8 / KT);  // entries per lane per batch
  constexpr int BATCH = KT * EB;
  const int lane = threadIdx.x & 31;
  const int grp = lane / KT, t = lane % KT;
  const unsigned gmask = (KT == 32) ? 0xffffffffu : (((1u << KT) - 1u) << (grp * KT));
  const int gbase = grp * KT;
  const int strip_cols = KT * VW;
  const int nstrips = (k + strip_cols - 1) / strip_cols;
  const int64_t gid = ((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5) * GPW + grp;
  const int64_t ngroups = (((int64_t)gridDim.x * blockDim.x) >> 5) * GPW;
  const int64_t work_total = (int64_t)n_chunks * nstrips;
  for (int64_t w = gid; w < work_total; w += ngroups) {
    const int chunk = (int)(w / nstrips);
    const int j = (int)(w % nstrips) * strip_cols + t * VW;
    const bool jok = j < k;  // k % VW == 0: a lane's VW columns are all in or all out
    const int64_t c0 = (int64_t)chunk * Q;
    const int64_t c1 = (c0 + Q < nnz) ? c0 + Q : nnz;
    int row = (chunk == 0) ? 0 : chunk_row[chunk];
    int ebase = row;
    int ends = row_ptr[min(ebase + 1 + t, m)];
    int64_t row_start = row_ptr[row];
    int64_t next_end = __shfl_sync(gmask, ends, gbase);
    S acc[VW];
#pragma unroll
    for (int q = 0; q < VW; ++q) acc[q] = S(0);
    auto flush = [&]() {
      if (jok) {
        S* yp = Y + (int64_t)row * ldy + j;
        if (row_start >= c0 && next_end <= c1) {
          S o[VW];
          if (beta == S(0)) {
#pragma unroll
            for (int q = 0; q < VW; ++q) o[q] = alpha * acc[q];
          } else {
            S old[VW];
            vec_unpack(*reinterpret_cast<const V*>(yp), old);
#pragma unroll
            for (int q = 0; q < VW; ++q) o[q] = beta * old[q] + alpha * acc[q];
          }
          *reinterpret_cast<V*>(yp) = vec_pack(o);
        } else {
#pragma unroll
          for (int q = 0; q < VW; ++q) atomicAdd(yp + q, alpha * acc[q]);
        }
      }
#pragma unroll
      for (int q = 0; q < VW; ++q) acc[q] = S(0);
      row_start = next_end;
      ++row;
      if (row - ebase == KT) {
        ebase = row;
        ends = row_ptr[min(ebase + 1 + t, m)];
      }
      next_end = __shfl_sync(gmask, ends, gbase + (row - ebase));
    };
    for (int64_t b = c0; b < c1; b += BATCH) {
      int c[EB];
      S v[EB];
#pragma unroll
      for (int i = 0; i < EB; ++i) {
        const int64_t e = b + i * KT + t;
        c[i] = 0;
        v[i] = S(0);
        if (e < c1) {
          c[i] = ld_stream(col_idx + e);
          v[i] = ld_stream(vals + e);
        }
      }
      const int nb = (int)((c1 - b < BATCH) ? (c1 - b) : BATCH);
      V xv[BATCH];
#pragma unroll
      for (int u = 0; u < BATCH; ++u) {
        const int cu = __shfl_sync(gmask, c[u / KT], gbase + (u % KT));
        if (u < nb && jok) xv[u] = __ldg(reinterpret_cast<const V*>(X + (int64_t)cu * ldx + j));
      }
#pragma unroll
      for (int u = 0; u < BATCH; ++u) {
        const S vu = __shfl_sync(gmask, v[u / KT], gbase + (u % KT));
        if (u < nb) {
          while (b + u >= next_end) flush();  // uniform within the group
          if (jok) {
            S xs[VW];
            vec_unpack(xv[u], xs);
#pragma unroll
            for (int q = 0; q < VW; ++q) acc[q] += vu * xs[q];
          }
        }
      }
    }
    while (row < m && next_end <= c1) flush();
    if (row < m && row_start < c1 && jok) {
      S* yp = Y + (int64_t)row * ldy + j;
#pragma unroll
      for (int q = 0; q < VW; ++q) atomicAdd(yp + q, alpha * acc[q]);
    }
  }
}

int plan_chunk_rows(b200sp_spmv_plan* p, cudaStream_t st, int m, int64_t nnz, const int* row_ptr, int Q, int** chunk_row,
                    int* n_chunks);

template <typename S>
static int launch_split(b200sp_spmv_plan* p, cudaStream_t st, int m, int k, int64_t nnz, const int* row_ptr,
                        const int* col_idx, const S* vals, const S* X, int64_t ldx, S* Y, int64_t ldy, S alpha, S beta) {
  const int Q = 256;
  int* chunk_row = nullptr;
  int n_chunks = 0;
  int rc = plan_chunk_rows(p, st, m, nnz, row_ptr, Q, &chunk_row, &n_chunks);
  if (rc) return rc;
  {
    const int blocks = std::max(1, std::min((m + 255) / 256, sm_count() * 8));
    spmm_prescale_split_rows<S><<<blocks, 256, 0, st>>>(m, k, Q, row_ptr, beta, Y, ldy);
    B200SP_LAUNCH_CHECK();
  }
  {
    constexpr int VW = 16 / (int)sizeof(S);
    const bool vec_ok = (k % VW == 0) && (ldx % VW == 0) && (ldy % VW == 0) &&
                        ((((uintptr_t)X) | ((uintptr_t)Y)) & 15u) == 0 && getenv("B200SP_SPMM_VEC") != nullptr;
    // opt-in: slower than the scalar-lane kernel on config 3 when it was tuned -- fewer lanes per chunk means fewer
    // chunks in flight per SM at its register count; kept for the tuning round
    if (vec_ok) {
      int KTv = 1;
      while (KTv * VW < k && KTv < 32) KTv <<= 1;
      const int gpwv = 32 / KTv;
      const int nstripsv = (k + KTv * VW - 1) / (KTv * VW);
      const int64_t workv = (int64_t)n_chunks * nstripsv;
      int blocksv = (int)std::min<int64_t>((workv + 8 * gpwv - 1) / (8 * gpwv), (int64_t)sm_count() * 16);
      if (blocksv < 1) blocksv = 1;
#define B200SP_SPLITV(K)                                                                                          \
  case K:                                                                                                         \
    spmm_split_vec_kernel<S, K><<<blocksv, 256, 0, st>>>(m, k, nnz, Q, n_chunks, chunk_row, row_ptr, col_idx, vals, X, \
                                                         ldx, Y, ldy, alpha, beta);                               \
    break;
      switch (KTv) {
        B200SP_SPLITV(1)
        B200SP_SPLITV(2)
        B200SP_SPLITV(4)
        B200SP_SPLITV(8)
        B200SP_SPLITV(16)
        B200SP_SPLITV(32)
      }
#undef B200SP_SPLITV
      B200SP_LAUNCH_CHECK();
      return B200SP_OK;
    }
  }
  int KT = 1;
  while (KT < k && KT < 32) KT <<= 1;
  const int gpw = 32 / KT;
  const int nstrips = (k + KT - 1) / KT;
  const int64_t work = (int64_t)n_chunks * nstrips;
  int blocks = (int)std::min<int64_t>((work + 8 * gpw - 1) / (8 * gpw), (int64_t)sm_count() * 16);
  if (blocks < 1) blocks = 1;
#define B200SP_SPLIT(K)                                                                                       \
  case K:                                                                                                     \
    spmm_split_kernel<S, K><<<blocks, 256, 0, st>>>(m, k, nnz, Q, n_chunks, chunk_row, row_ptr, col_idx, vals, X, ldx, \
                                                    Y, ldy, alpha, beta);                                     \
    break;
  switch (KT) {
    B200SP_SPLIT(1)
    B200SP_SPLIT(2)
    B200SP_SPLIT(4)
    B200SP_SPLIT(8)
    B200SP_SPLIT(16)
    B200SP_SPLIT(32)
  }
#undef B200SP_SPLIT
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

int plan_analyse_mm(b200sp_spmv_plan* p, cudaStream_t st, int cap, int lmax, int seg, int m, int64_t nnz, const int* row_ptr,
                    MMTileView* out);

template <typename S, int VW, int KTL, int NW, int STAGES, int CAP, int UNR>
static int launch_mm_tile_k(cudaStream_t st, const MMTileView& tv, int m, int k, int64_t nnz, const int* row_ptr,
                            const int* col_idx, const S* vals, const S* X, int64_t ldx, S* Y, int64_t ldy, S alpha, S beta) {
  using Ring = TileRing<S, CAP, STAGES>;
  auto kern = spmm_tile_kernel<S, VW, KTL, NW, STAGES, CAP, UNR>;
  const size_t smem = sizeof(Ring) + 128;
  static KernelSetup ks;  // per instantiation and device: attribute set + occupancy queried once
  int occ = 1;
  if (int rc = kernel_setup(ks, kern, (NW + 1) * 32, smem, &occ)) return rc;
  int grid = std::min(tv.n_tiles, sm_count() * occ);
  if (grid < 1) grid = 1;
  kern<<<grid, (NW + 1) * 32, smem, st>>>(m, k, nnz, tv.n_tiles, tv.LMAX, tv.tiles, row_ptr, col_idx, vals, X, ldx, Y, ldy, alpha, beta);
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

// ring / unroll configurations of the tile kernel.  0 is the default; 1-3 exist for the 16-byte-load path only
// (B200SP_SPMM_CFG, tuning sweeps): 1 = small ring (8 consumer warps, 1024-entry stages: 5 CTAs per SM for fp32),
// 2 = default ring with twice the gathers in flight per lane, 3 = small ring with 16 consumer warps.
template <typename S, int VW, int KTL>
static int launch_mm_tile_cfg(int cfg, cudaStream_t st, const MMTileView& tv, int m, int k, int64_t nnz, const int* row_ptr,
                              const int* col_idx, const S* vals, const S* X, int64_t ldx, S* Y, int64_t ldy, S alpha, S beta) {
  if constexpr (VW > 1) {
    switch (cfg) {
      case 1: return launch_mm_tile_k<S, VW, KTL, 8, 4, 1024, 4>(st, tv, m, k, nnz, row_ptr, col_idx, vals, X, ldx, Y, ldy, alpha, beta);
      case 2: return launch_mm_tile_k<S, VW, KTL, 16, 4, 2048, 8>(st, tv, m, k, nnz, row_ptr, col_idx, vals, X, ldx, Y, ldy, alpha, beta);
      case 3: return launch_mm_tile_k<S, VW, KTL, 16, 3, 1024, 4>(st, tv, m, k, nnz, row_ptr, col_idx, vals, X, ldx, Y, ldy, alpha, beta);
      default: break;
    }
  }
  return launch_mm_tile_k<S, VW, KTL, 16, 4, 2048, (VW == 1 ? 8 : 4)>(st, tv, m, k, nnz, row_ptr, col_idx, vals, X, ldx, Y, ldy, alpha, beta);
}

template <typename S>
static int launch_mm_tile(b200sp_spmv_plan* p, cudaStream_t st, bool vec, int m, int k, int64_t nnz, const int* row_ptr,
                          const int* col_idx, const S* vals, const S* X, int64_t ldx, S* Y, int64_t ldy, S alpha, S beta) {
  constexpr int SEG = 2048;
  int cfg = 0;
  if (const char* e = getenv("B200SP_SPMM_CFG")) cfg = atoi(e);
  if (!vec || cfg < 0 || cfg > 3) cfg = 0;
  const int CAP = (cfg == 1 || cfg == 3) ? 1024 : 2048;
  int LMAX = 256;  // rows longer than this leave the tiles for the segment kernel (B200SP_SPMM_LMAX: 16..512)
  if (const char* e = getenv("B200SP_SPMM_LMAX")) {
    const int v = atoi(e);
    if (v >= 16 && v <= 512) LMAX = v;
  }
  MMTileView tv;
  int rc = plan_analyse_mm(p, st, CAP, LMAX, SEG, m, nnz, row_ptr, &tv);
  if (rc) return rc;
  constexpr int W = VecOf<S>::W;
  const int lanes_needed = vec ? (k + W - 1) / W : k;
  int KTL = 1;
  while (KTL < lanes_needed && KTL < 32) KTL <<= 1;
#define B200SP_MMT(V, L)                                                                                                    \
  case L:                                                                                                                   \
    rc = launch_mm_tile_cfg<S, V, L>(cfg, st, tv, m, k, nnz, row_ptr, col_idx, vals, X, ldx, Y, ldy, alpha, beta);          \
    break;
  if (vec) {
    switch (KTL) {
      B200SP_MMT(W, 1) B200SP_MMT(W, 2) B200SP_MMT(W, 4) B200SP_MMT(W, 8) B200SP_MMT(W, 16) B200SP_MMT(W, 32)
    }
  } else {
    switch (KTL) {
      B200SP_MMT(1, 1) B200SP_MMT(1, 2) B200SP_MMT(1, 4) B200SP_MMT(1, 8) B200SP_MMT(1, 16) B200SP_MMT(1, 32)
    }
  }
#undef B200SP_MMT
  if (rc) return rc;
  // long rows: segments of <= SEG entries, one CTA each
  const int grid = sm_count() * 4;
  spmm_seg_prescale_kernel<S><<<grid, 256, 0, st>>>(tv.segs, tv.n_seg, k, beta, Y, ldy);
  B200SP_LAUNCH_CHECK();
  if (vec) {
    const char* e = getenv("B200SP_SPMM_SEG");
    if (e && e[0] == 'v') {
#define B200SP_SEGV(L)                                                                                               \
  case L:                                                                                                            \
    spmm_seg_vec_kernel<S, L><<<grid, 256, 0, st>>>(tv.segs, tv.n_seg, k, col_idx, vals, X, ldx, Y, ldy, alpha, beta); \
    break;
      switch (KTL) {
        B200SP_SEGV(1) B200SP_SEGV(2) B200SP_SEGV(4) B200SP_SEGV(8) B200SP_SEGV(16) B200SP_SEGV(32)
      }
#undef B200SP_SEGV
      B200SP_LAUNCH_CHECK();
      return B200SP_OK;
    }
  }
  int KT = 1;
  while (KT < k && KT < 32) KT <<= 1;
#define B200SP_SEG(K)                                                                                              \
  case K:                                                                                                          \
    spmm_seg_kernel<S, K><<<grid, 256, 0, st>>>(tv.segs, tv.n_seg, k, col_idx, vals, X, ldx, Y, ldy, alpha, beta); \
    break;
  switch (KT) {
    B200SP_SEG(1) B200SP_SEG(2) B200SP_SEG(4) B200SP_SEG(8) B200SP_SEG(16) B200SP_SEG(32)
  }
#undef B200SP_SEG
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

// ---------------------------------------------------------------------------
// Item kernel (default for row-major X and Y with a plan; B200SP_SPMM_KERNEL=items): the gather-bound formulation.
// On power-law matrices the tile kernel's row groups of one warp run loops of very different lengths and wait for
// the longest; here the unit of work is an ITEM -- a run of <= LMAX consecutive entries of one row (spmm_items.h) --
// and the items are sorted by length, longest first.  A group of KTL lanes (VW adjacent columns each, one 16-byte
// load of the X row segment per lane and entry) owns one item, so the 32/KTL groups of a warp run loops of equal
// length with 4 independent gathers in flight per lane, nothing waits, and the long items are scheduled first.
// (col, val) are read straight from global memory (every lane of the group the same address: one request).
// Single-item rows write Y; the pieces of longer rows write partial sums that spmm_item_reduce_kernel adds up in
// piece order (no atomics: deterministic).  Per entry the sum order is the storage order.
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

static int plan_analyse_items(b200sp_spmv_plan* p, cudaStream_t st, int lmax, int m, int64_t nnz, const int* row_ptr, MMItems** out) {
  MMItems* mi = plan_mm_items(p);
  *out = mi;
  if (mi->items && mi->key_row_ptr == row_ptr && mi->key_m == m && mi->key_nnz == nnz && mi->key_lmax == lmax) return B200SP_OK;
  void* old[] = {mi->items, mi->multi, mi->partial};
  for (void* q : old)
    if (q) cudaFreeAsync(q, st);
  *mi = MMItems();
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
  B200SP_CUDA_TRY(cudaMallocAsync((void**)&mi->items, sizeof(int4) * (size_t)std::max(mi->n_items, 1), st));
  B200SP_CUDA_TRY(cudaMallocAsync((void**)&mi->multi, sizeof(int4) * (size_t)std::max(mi->n_multi, 1), st));
  B200SP_CUDA_TRY(cudaMemcpyAsync(hist, h_cur, sizeof(int) * (size_t)(lmax + 1), cudaMemcpyHostToDevice, st));
  mmi_fill_kernel<<<blocks, 256, 0, st>>>(m, row_ptr, lmax, hist, counters, mi->items, mi->multi, mi->n_multi);
  B200SP_LAUNCH_CHECK();
  B200SP_CUDA_TRY(cudaStreamSynchronize(st));  // h_cur is pageable host memory: consumed before it goes out of scope
  mi->key_row_ptr = row_ptr;
  mi->key_m = m;
  mi->key_nnz = nnz;
  mi->key_lmax = lmax;
  return B200SP_OK;
}

template <typename S, int VW, int KTL>
__global__ void __launch_bounds__(256)
    spmm_item_kernel(int n_items, const int4* __restrict__ items, int k, const int* __restrict__ col_idx,
                     const S* __restrict__ vals, const S* __restrict__ X, int64_t ldx, S* __restrict__ Y, int64_t ldy,
                     S* __restrict__ partial, S alpha, S beta) {
  const int64_t gt = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t q = gt / KTL;
  const int t = (int)(gt % KTL);
  if (q >= n_items) return;
  // the matrix, the item list and Y pass through once: evict-first in L2, which then belongs to the gathered rows of X
  const uint64_t once = l2_policy_evict_first();
  const int4 it = ld_once(items + q, once);
  const int row = it.x, e0 = it.y, len = it.z, slot = it.w;
  const int nstrips = (k + KTL * VW - 1) / (KTL * VW);
  for (int strip = 0; strip < nstrips; ++strip) {
    const int j = (strip * KTL + t) * VW;
    if (j >= k) break;  // k % VW == 0: a lane's VW columns are all in or all out
    Acc<S, VW> acc;
#pragma unroll
    for (int c = 0; c < VW; ++c) acc.a[c] = S(0);
    const S* xb = X + j;
    int e = e0;
    const int e4 = e0 + (len & ~3);
    for (; e < e4; e += 4) {
      int c[4];
      S av[4];
      Acc<S, VW> xv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        c[u] = ld_once(col_idx + e + u, once);
        av[u] = ld_once(vals + e + u, once);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) xv[u] = load_x<S, VW>(xb + (int64_t)c[u] * ldx);
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int cc = 0; cc < VW; ++cc) acc.a[cc] += av[u] * xv[u].a[cc];
    }
    for (; e < e0 + len; ++e) {
      const int c = ld_once(col_idx + e, once);
      const S av = ld_once(vals + e, once);
      const Acc<S, VW> xv = load_x<S, VW>(xb + (int64_t)c * ldx);
#pragma unroll
      for (int cc = 0; cc < VW; ++cc) acc.a[cc] += av * xv.a[cc];
    }
    S o[VW];
    S* dst;
    if (slot < 0) {
      dst = Y + (int64_t)row * ldy + j;
      if (beta == S(0)) {
#pragma unroll
        for (int cc = 0; cc < VW; ++cc) o[cc] = alpha * acc.a[cc];
      } else {
        const Acc<S, VW> old = load_x<S, VW>(dst);
#pragma unroll
        for (int cc = 0; cc < VW; ++cc) o[cc] = beta * old.a[cc] + alpha * acc.a[cc];
      }
    } else {
      dst = partial + (int64_t)slot * k + j;  // raw sums; alpha and beta are applied by the reduce kernel
#pragma unroll
      for (int cc = 0; cc < VW; ++cc) o[cc] = acc.a[cc];
    }
    if constexpr (VW == 1) {
      st_once(dst, o[0], once);
    } else {
      using V = typename VecOf<S>::type;
      st_once(reinterpret_cast<V*>(dst), vec_pack(o), once);
    }
  }
}

// Cooperative variant (default; B200SP_SPMM_ITEM_COOP=0 selects the kernel above): the same items, the same order of
// additions (bit-identical Y), but the KTL lanes of a group no longer read the same (col, val) address each -- that
// costs one L1 wavefront per group and entry for the column, one for the value and one for the X row: 3 per
// nonzero at 8 groups per warp, and the kernel is bound by exactly that (one wavefront per SM and clock).  Here the
// group reads a batch of EB consecutive entries with ONE load per lane (adjacent lanes, adjacent entries: the group's
// EB/KTL loads cover a contiguous 32..64-byte run) and passes them round with shuffles, which run on a different
// pipe: 1 + 2 * 4/32 wavefronts per nonzero for k = 16 fp32, with EB gathers of X in flight per lane (EB = 4: 40 registers,
// 6 CTAs per SM; EB = 8: 80 registers, 3 CTAs -- the same number of gathers in flight per SM, and 4 was faster when tuned).
template <typename S, int VW, int KTL, int EB /* entries per batch: 4 or 8 */>
__global__ void __launch_bounds__(256)
    spmm_item_coop_kernel(int n_items, const int4* __restrict__ items, int k, const int* __restrict__ col_idx,
                          const S* __restrict__ vals, const S* __restrict__ X, int64_t ldx, S* __restrict__ Y, int64_t ldy,
                          S* __restrict__ partial, S alpha, S beta) {
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
    Acc<S, VW> acc;
#pragma unroll
    for (int c = 0; c < VW; ++c) acc.a[c] = S(0);
    const S* xb = X + (live ? j : 0);
    int e = e0;
    for (; e + EB <= eend; e += EB) {
      int cl[PL];
      S vl[PL];
#pragma unroll
      for (int i = 0; i < PL; ++i) {
        const int idx = i * KTL + t;
        cl[i] = 0;
        vl[i] = S(0);
        if (KTL <= EB || idx < EB) {
          cl[i] = ld_once(col_idx + e + idx, once);
          vl[i] = ld_once(vals + e + idx, once);
        }
      }
      int c[EB];
      S av[EB];
#pragma unroll
      for (int u = 0; u < EB; ++u) {
        if constexpr (KTL == 1) {
          c[u] = cl[u];
          av[u] = vl[u];
        } else {
          c[u] = __shfl_sync(gmask, cl[u / KTL], u % KTL, KTL);
          av[u] = __shfl_sync(gmask, vl[u / KTL], u % KTL, KTL);
        }
      }
      if (live) {
        Acc<S, VW> xv[EB];
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
        vl[i] = S(0);
        if (idx < rem) {
          cl[i] = ld_once(col_idx + e + idx, once);
          vl[i] = ld_once(vals + e + idx, once);
        }
      }
      int c[EB];
      S av[EB];
#pragma unroll
      for (int u = 0; u < EB; ++u) {
        if constexpr (KTL == 1) {
          c[u] = cl[u];
          av[u] = vl[u];
        } else {
          c[u] = __shfl_sync(gmask, cl[u / KTL], u % KTL, KTL);
          av[u] = __shfl_sync(gmask, vl[u / KTL], u % KTL, KTL);
        }
      }
      if (live) {
        Acc<S, VW> xv[EB];
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
    S o[VW];
    S* dst;
    if (slot < 0) {
      dst = Y + (int64_t)row * ldy + j;
      if (beta == S(0)) {
#pragma unroll
        for (int cc = 0; cc < VW; ++cc) o[cc] = alpha * acc.a[cc];
      } else {
        const Acc<S, VW> old = load_x<S, VW>(dst);
#pragma unroll
        for (int cc = 0; cc < VW; ++cc) o[cc] = beta * old.a[cc] + alpha * acc.a[cc];
      }
    } else {
      dst = partial + (int64_t)slot * k + j;  // raw sums; alpha and beta are applied by the reduce kernel
#pragma unroll
      for (int cc = 0; cc < VW; ++cc) o[cc] = acc.a[cc];
    }
    if constexpr (VW == 1) {
      st_once(dst, o[0], once);
    } else {
      using V = typename VecOf<S>::type;
      st_once(reinterpret_cast<V*>(dst), vec_pack(o), once);
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
    spmm_item_reduce_kernel(int n_multi, const int4* __restrict__ multi, int k, const S* __restrict__ partial, S* __restrict__ Y,
                            int64_t ldy, S alpha, S beta) {
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
      S sum = S(0);
      if (j < k) {
        const S* src = partial + (int64_t)d.y * k + j;
        for (int s = sub; s < d.z; s += SUB) sum += src[(int64_t)s * k];
      }
      for (int o = 16; o >= KC; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      if (sub == 0 && j < k) {
        S* yp = Y + (int64_t)d.x * ldy + j;
        *yp = (beta == S(0)) ? alpha * sum : beta * *yp + alpha * sum;
      }
    }
  }
}

// the same for the rows of more than MMI_LONG_PIECES pieces (the hubs of a power-law matrix: 2388 pieces in the longest row of
// R-MAT scale 23), one CTA per row: thread = (piece subsequence, column), 256 / KC subsequences added in piece order each, then
// joined in subsequence order through shared memory by the threads of subsequence 0.  Fixed order: reproducible.
template <typename S>
__global__ void __launch_bounds__(256)
    spmm_item_reduce_long_kernel(int n_long, const int4* __restrict__ multi_long, int k, const S* __restrict__ partial,
                                 S* __restrict__ Y, int64_t ldy, S alpha, S beta) {
  __shared__ S part[256];
  int KC = 1;
  while (KC < k && KC < 32) KC <<= 1;
  const int SUB = 256 / KC;
  const int j0 = threadIdx.x % KC, sub = threadIdx.x / KC;
  for (int w = blockIdx.x; w < n_long; w += gridDim.x) {
    const int4 d = multi_long[w];
    for (int jb = 0; jb < k; jb += KC) {
      const int j = jb + j0;
      S sum = S(0);
      if (j < k) {
        const S* src = partial + (int64_t)d.y * k + j;
        for (int s = sub; s < d.z; s += SUB) sum += src[(int64_t)s * k];
      }
      part[threadIdx.x] = sum;
      __syncthreads();
      if (sub == 0 && j < k) {
        S t = part[j0];
        for (int q = 1; q < SUB; ++q) t += part[q * KC + j0];
        S* yp = Y + (int64_t)d.x * ldy + j;
        *yp = (beta == S(0)) ? alpha * t : beta * *yp + alpha * t;
      }
      __syncthreads();
    }
  }
}

template <typename S>
static int launch_mm_items(b200sp_spmv_plan* p, cudaStream_t st, bool vec, int m, int k, int64_t nnz, const int* row_ptr,
                           const int* col_idx, const S* vals, const S* X, int64_t ldx, S* Y, int64_t ldy, S alpha, S beta) {
  int LMAX = 64;  // entries per item (B200SP_SPMM_ITEM_LMAX: 16..256); 64 was the best of 32..256 on R-MAT scale 23 when tuned
  if (const char* e = getenv("B200SP_SPMM_ITEM_LMAX")) {
    const int v = atoi(e);
    if (v >= 16 && v <= MMI_MAXL) LMAX = v;
  }
  MMItems* mi;
  int rc = plan_analyse_items(p, st, LMAX, m, nnz, row_ptr, &mi);
  if (rc) return rc;
  const size_t need = sizeof(S) * (size_t)mi->n_partial * (size_t)k;
  if (need > mi->partial_bytes) {
    if (mi->partial) cudaFreeAsync(mi->partial, st);
    mi->partial = nullptr;
    mi->partial_bytes = 0;
    B200SP_CUDA_TRY(cudaMallocAsync(&mi->partial, need, st));
    mi->partial_bytes = need;
  }
  constexpr int W = VecOf<S>::W;
  const int lanes_needed = vec ? (k + W - 1) / W : k;
  int KTL = 1;
  while (KTL < lanes_needed && KTL < 32) KTL <<= 1;
  const int64_t threads = (int64_t)mi->n_items * KTL;
  const unsigned grid = (unsigned)((threads + 255) / 256);
  if (grid > 0) {
    static const int coop = [] {  // B200SP_SPMM_ITEM_COOP=0: every lane reads (col, val) itself (the first item kernel); 4 (default) | 8: batch
      const char* e = getenv("B200SP_SPMM_ITEM_COOP");
      return e && e[0] == '0' ? 0 : (e && e[0] == '8' ? 8 : 4);  // 4 was the fastest of 0 / 4 / 8 on R-MAT scale 23 x 16 when tuned
    }();
#define B200SP_MMI(V, L)                                                                                                   \
  case L:                                                                                                                  \
    if (coop == 8)                                                                                                         \
      spmm_item_coop_kernel<S, V, L, 8><<<grid, 256, 0, st>>>(mi->n_items, mi->items, k, col_idx, vals, X, ldx, Y, ldy,    \
                                                              (S*)mi->partial, alpha, beta);                               \
    else if (coop == 4)                                                                                                    \
      spmm_item_coop_kernel<S, V, L, 4><<<grid, 256, 0, st>>>(mi->n_items, mi->items, k, col_idx, vals, X, ldx, Y, ldy,    \
                                                              (S*)mi->partial, alpha, beta);                               \
    else                                                                                                                   \
      spmm_item_kernel<S, V, L><<<grid, 256, 0, st>>>(mi->n_items, mi->items, k, col_idx, vals, X, ldx, Y, ldy,            \
                                                      (S*)mi->partial, alpha, beta);                                       \
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
    spmm_item_reduce_kernel<S><<<std::max(g, 1), 256, 0, st>>>(n_short, mi->multi, k, (const S*)mi->partial, Y, ldy, alpha, beta);
    B200SP_LAUNCH_CHECK();
  }
  if (mi->n_multi_long > 0) {
    const int g = std::min(mi->n_multi_long, sm_count() * 8);  // a CTA per row
    spmm_item_reduce_long_kernel<S><<<g, 256, 0, st>>>(mi->n_multi_long, mi->multi + n_short, k, (const S*)mi->partial, Y, ldy, alpha, beta);
    B200SP_LAUNCH_CHECK();
  }
  return B200SP_OK;
}

// which rank-2 kernel: 0 = row per group, 1 = nnz-split, 2 = tile, 3 = tile with 16-byte X loads (default: about twice
// as fast as the split kernel on R-MAT scale 21 x 16 columns when it was tuned).
// B200SP_SPMM_KERNEL=row|split|tile|tilev overrides.
static int mm_kernel_choice(b200sp_spmv_plan* p) {
  if (!p) return 0;  // the others need a plan (chunk table / tile analysis)
  const char* e = getenv("B200SP_SPMM_KERNEL");
  if (e && e[0] == 'r') return 0;
  if (e && e[0] == 's') return 1;
  if (e && e[0] == 't') return (e[1] == 'i' && e[2] == 'l' && e[3] == 'e' && e[4] == 'v') ? 3 : 2;
  if (e && e[0] == 'i') return 4;
  return 4;  // items (B200SP_SPMM_KERNEL=items)
}

static bool use_split_kernel(b200sp_spmv_plan* p) {
  // needs a plan (chunk table); B200SP_SPMM_KERNEL=row|split overrides for experiments
  if (!p) return false;
  const char* e = getenv("B200SP_SPMM_KERNEL");
  if (e && e[0] == 'r') return false;
  return true;
}

template <typename S>
static int spmm_impl(b200sp_spmv_plan* p, cudaStream_t st, char mode, int m, int n, int64_t nnz, int k, S alpha,
                     const int* row_ptr, const int* col_idx, const S* vals, const S* X, int64_t ldx, int xrm,
                     S beta, S* Y, int64_t ldy, int yrm) {
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
  if (alpha == S(0) || m == 0 || n == 0 || nnz == 0) {
    if (beta != S(1)) {
      scale2d_kernel<S><<<std::max(grid_elem, 1), 256, 0, st>>>(yrows, k, beta, Y, yr, yc);
      B200SP_LAUNCH_CHECK();
    }
    return B200SP_OK;
  }
  B200SP_REQUIRE(row_ptr && col_idx && vals && X, "spmm: null pointer argument");
  if (trans) {
    if (beta != S(1)) {
      scale2d_kernel<S><<<std::max(grid_elem, 1), 256, 0, st>>>(yrows, k, beta, Y, yr, yc);
      B200SP_LAUNCH_CHECK();
    }
    const int g = (int)std::min<int64_t>(((int64_t)m * k + 255) / 256, (int64_t)sm_count() * 16);
    spmm_transpose_kernel<S><<<std::max(g, 1), 256, 0, st>>>(m, k, row_ptr, col_idx, vals, X, xr, xc, Y, yr, yc, alpha);
    B200SP_LAUNCH_CHECK();
    plan_set_last_kernel(p, "spmm_transpose");
    return B200SP_OK;
  }
  const bool split = use_split_kernel(p);
  const int choice = mm_kernel_choice(p);
  if (xrm && yrm) {
    if (choice == 4) {
      constexpr int W = VecOf<S>::W;
      const bool vec = (k % W == 0) && (ldx % W == 0) && (ldy % W == 0) && ((((uintptr_t)X) | ((uintptr_t)Y)) & 15u) == 0;
      plan_set_last_kernel(p, vec ? "spmm_items_vec" : "spmm_items");
      return launch_mm_items<S>(p, st, vec, m, k, nnz, row_ptr, col_idx, vals, X, ldx, Y, ldy, alpha, beta);
    }
    if (choice >= 2 && (((uintptr_t)vals | (uintptr_t)col_idx | (uintptr_t)row_ptr) & 15u) == 0) {
      constexpr int W = VecOf<S>::W;
      const bool vec = choice == 3 && (k % W == 0) && (ldx % W == 0) && (ldy % W == 0) && ((((uintptr_t)X) | ((uintptr_t)Y)) & 15u) == 0;
      plan_set_last_kernel(p, vec ? "spmm_tile_vec" : "spmm_tile");
      return launch_mm_tile<S>(p, st, vec, m, k, nnz, row_ptr, col_idx, vals, X, ldx, Y, ldy, alpha, beta);
    }
    plan_set_last_kernel(p, split ? "spmm_split" : "spmm_rowmajor");
    if (split) return launch_split<S>(p, st, m, k, nnz, row_ptr, col_idx, vals, X, ldx, Y, ldy, alpha, beta);
    return launch_rowmajor<S>(st, m, k, row_ptr, col_idx, vals, X, ldx, Y, ldy, alpha, beta);
  }
  // LayoutLeft operands: with a plan and k >= 4, relayout to row-major scratch and use the row-major kernel
  if (p && k >= 4) {
    void *xt = nullptr, *yt = nullptr;
    const size_t xtb = xrm ? 0 : sizeof(S) * (size_t)xrows * k;
    const size_t ytb = yrm ? 0 : sizeof(S) * (size_t)yrows * k;
    int rc = plan_mv_scratch(p, st, xtb, ytb, &xt, &yt);
    if (rc) return rc;
    const int tb = 256;
    auto rl_grid = [](int64_t rows) { return (unsigned)std::max<int64_t>(1, std::min<int64_t>((rows + 127) / 128, (int64_t)sm_count() * 16)); };
    const S* Xr = X;
    int64_t ldxr = ldx;
    if (!xrm) {
      relayout_kernel<S, true><<<rl_grid(xrows), tb, 0, st>>>(xrows, k, (S*)xt, X, nullptr, xr, xc);
      B200SP_LAUNCH_CHECK();
      Xr = (const S*)xt;
      ldxr = k;
    }
    S* Yr = Y;
    int64_t ldyr = ldy;
    if (!yrm) {
      Yr = (S*)yt;
      ldyr = k;
      if (beta != S(0)) {
        relayout_kernel<S, true><<<rl_grid(yrows), tb, 0, st>>>(yrows, k, Yr, Y, nullptr, yr, yc);
        B200SP_LAUNCH_CHECK();
      }
    }
    const bool tile_ok = choice >= 2 && (choice == 4 || (((uintptr_t)vals | (uintptr_t)col_idx | (uintptr_t)row_ptr) & 15u) == 0);
    if (choice == 4) {
      constexpr int W = VecOf<S>::W;
      const bool vec = (k % W == 0) && (ldxr % W == 0) && (ldyr % W == 0) && ((((uintptr_t)Xr) | ((uintptr_t)Yr)) & 15u) == 0;
      rc = launch_mm_items<S>(p, st, vec, m, k, nnz, row_ptr, col_idx, vals, Xr, ldxr, Yr, ldyr, alpha, beta);
    } else if (tile_ok) {
      constexpr int W = VecOf<S>::W;
      const bool vec = choice == 3 && (k % W == 0) && (ldxr % W == 0) && (ldyr % W == 0) && ((((uintptr_t)Xr) | ((uintptr_t)Yr)) & 15u) == 0;
      rc = launch_mm_tile<S>(p, st, vec, m, k, nnz, row_ptr, col_idx, vals, Xr, ldxr, Yr, ldyr, alpha, beta);
    } else {
      rc = split ? launch_split<S>(p, st, m, k, nnz, row_ptr, col_idx, vals, Xr, ldxr, Yr, ldyr, alpha, beta)
                 : launch_rowmajor<S>(st, m, k, row_ptr, col_idx, vals, Xr, ldxr, Yr, ldyr, alpha, beta);
    }
    if (rc) return rc;
    if (!yrm) {
      relayout_kernel<S, false><<<rl_grid(yrows), tb, 0, st>>>(yrows, k, Yr, nullptr, Y, yr, yc);
      B200SP_LAUNCH_CHECK();
    }
    plan_set_last_kernel(p, choice == 4 ? "spmm_relayout+items" : tile_ok ? "spmm_relayout+tile" : (split ? "spmm_relayout+split" : "spmm_relayout+rowmajor"));
    return B200SP_OK;
  }
  const int g = (int)std::min<int64_t>(((int64_t)m * k + 255) / 256, (int64_t)sm_count() * 16);
  spmm_general_kernel<S><<<std::max(g, 1), 256, 0, st>>>(m, k, row_ptr, col_idx, vals, X, xr, xc, Y, yr, yc, alpha, beta);
  B200SP_LAUNCH_CHECK();
  plan_set_last_kernel(p, "spmm_general");
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
}
