// bsr.cu -- BsrMatrix SpMV / SpMM for sm_90a (SURVEY.md section 8f rank 3; DESIGN.md section 7c).
//
// Replaces, behind the C ABI (include/b200sparse.h, b200sp_bsr_*):
//   SPMV_BSRMATRIX<Cuda,...>::spmv_bsrmatrix        sparse/impl/KokkosSparse_spmv_bsrmatrix_spec.hpp:165-283
//     = today either cusparse{S,D}bsrmv             sparse/tpls/KokkosSparse_spmv_bsrmatrix_tpl_spec_decl.hpp:279-352
//       (mode N only) or the native functors BsrSpmvV42NonTrans (impl_v42.hpp:35-121) and, for T / H,
//       BSR_GEMV_Transpose_Functor                  sparse/impl/KokkosSparse_spmv_bsrmatrix_impl.hpp:707-834
//   SPMV_MV_BSRMATRIX<Cuda,...>::spmv_mv_bsrmatrix  (cusparse{S,D}bsrmm :372-455 / the same native functors)
//
// A BsrMatrix is three arrays (sparse/src/KokkosSparse_BsrMatrix.hpp:355-370): the block row map (mb+1), block
// column indices (nnzb) and values, nnzb*bs*bs, every block row-major.  The tensor-core BSR kernel of the reference
// (impl.hpp:24-459, Volta/Ampere wmma, half or fp64 8x8x4) is NOT what this file does: for fp64/fp32 SpMV the bound is
// the HBM stream of the values (8 + 4/bs^2 bytes per multiply-add against > 40 flop/byte of CUDA-core fp64), so the
// kernel below is the CSR tile kernel's design (spmv.cu) with blocks as the unit of the stream:
//
//   * the block rows are cut into tiles of about T blocks; a producer warp streams each tile's values, block columns
//     and row-map slice into a shared-memory ring with 1-D bulk (TMA) copies, evict-first in L2;
//   * bs in {2,3,4,5}: element-per-lane consumers (bsr_tile_e_kernel, block size compile-time); other bs <= 16:
//     consumer warps give every point row (block row, local row) LPR lanes; lane `sl` walks the entries
//     sl, sl+LPR, ... of its point row -- entry k is element (lr, k % bs) of block k / bs -- with all index arithmetic
//     carried incrementally (no division in the loop, bs is a run-time value); UNR gathers of x are in flight per lane;
//   * the epilogue is the reference functor's: y = beta*y (exact 0 for beta == 0), y += alpha*sum.
//
// Block rows too long for a stage, unaligned arrays and bs > 16 use bsr_vector_kernel (same walk, straight from global
// memory).  T / H scale y and scatter alpha * (column of block)^T x with atomics, like the reference.
#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <cstring>

#include <limits.h>
#include "common.cuh"
#include "tile_ring.cuh"

namespace b200sp {

namespace {

template <typename S>
__global__ void bsr_scale_kernel(int64_t rows, int k, S beta, S* __restrict__ y, int64_t yr, int64_t yc) {
  const int64_t total = rows * k;
  if (total <= (int64_t)INT32_MAX) {  // 32-bit index arithmetic (a 64-bit division per element costs more than its traffic)
    const unsigned t32 = (unsigned)total, r32 = (unsigned)rows, step = gridDim.x * blockDim.x;
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < t32; i += step) {
      const unsigned c = i / r32, r = i - c * r32;
      S* p = y + (int64_t)r * yr + (int64_t)c * yc;
      *p = (beta == S(0)) ? S(0) : beta * *p;
    }
    return;
  }
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i % rows, c = i / rows;
    S* p = y + r * yr + c * yc;
    *p = (beta == S(0)) ? S(0) : beta * *p;
  }
}

template <typename S>
int launch_scale2d(cudaStream_t st, int64_t rows, int k, S beta, S* y, int64_t yr, int64_t yc) {
  if (rows <= 0 || k <= 0 || beta == S(1)) return B200SP_OK;
  const int64_t total = rows * k;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, (int64_t)sm_count() * 8);
  bsr_scale_kernel<S><<<blocks, 256, 0, st>>>(rows, k, beta, y, yr, yc);
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

// reference epilogue (impl_v42.hpp:56-60,85): y *= beta (0 -> exact 0), y += alpha*accum
template <typename S>
__device__ __forceinline__ void bsr_store(S* __restrict__ p, S sum, S alpha, S beta) {
  sum *= alpha;
  *p = (beta == S(0)) ? sum : beta * *p + sum;
}

// ---------------------------------------------------------------------------------------------------------------
// the walk over one point row: entries k = sl, sl+lpr, ... < nk; entry k = element (lr, k % bs) of block k / bs.
// `vrow` points at element (lr, 0) of the row's first block, `crow` at its first block column.
// ---------------------------------------------------------------------------------------------------------------
template <typename S, int UNR, bool STREAM>
__device__ __forceinline__ S bsr_row_dot(const S* __restrict__ vrow, const int* __restrict__ crow, const S* __restrict__ x, int nk,
                                         int bs, int vpe, int lpr, int sl, int j0, int i0, int dj, int di) {
  // (j, i) = (block, column in block) of the lane's current entry; off = j*vpe + i, its value offset from vrow.  One step
  // adds (dj, di) with a carry into j when i passes bs -- carried as additions, no multiplication or division per entry.
  // Entries past the end of the row read entry (j0, i0) again (always inside the row here) and contribute exactly 0.
  S sum = S(0);
  int j = j0, i = i0;
  int off = j0 * vpe + i0;
  const int doff = dj * vpe + di, carry = vpe - bs;
  const int off0 = off;
  for (int k = sl; k < nk; k += UNR * lpr) {
    unsigned c[UNR];
    S av[UNR], xv[UNR];
    bool ok[UNR];
#pragma unroll
    for (int u = 0; u < UNR; ++u) {
      ok[u] = (k + u * lpr) < nk;
      const int jj = ok[u] ? j : j0, ii = ok[u] ? i : i0, oo = ok[u] ? off : off0;
      c[u] = (unsigned)((STREAM ? ld_stream(crow + jj) : crow[jj]) * bs + ii);
      av[u] = STREAM ? ld_stream(vrow + oo) : vrow[oo];
      i += di;
      j += dj;
      off += doff;
      if (i >= bs) {
        i -= bs;
        ++j;
        off += carry;
      }
    }
#pragma unroll
    for (int u = 0; u < UNR; ++u) xv[u] = ok[u] ? ldg(x + c[u]) : S(0);
#pragma unroll
    for (int u = 0; u < UNR; ++u) sum += av[u] * xv[u];
  }
  return sum;
}

template <typename S>
__device__ __forceinline__ S bsr_group_sum(S v, int lpr) {
  for (int o = lpr >> 1; o > 0; o >>= 1) v += shfl_xor(v, o);
  return v;
}

// ---------------------------------------------------------------------------------------------------------------
// fallback / long block rows: lpr lanes per point row, straight from global memory.  row_list == nullptr: all mb
// block rows; else the *n_list block rows it names.
// ---------------------------------------------------------------------------------------------------------------
template <typename S>
__global__ void __launch_bounds__(256) bsr_vector_kernel(int mb, int bs, int lpr, const int* __restrict__ row_ptr,
                                                         const int* __restrict__ col_idx, const S* __restrict__ vals,
                                                         const S* __restrict__ x, S* __restrict__ y, S alpha, S beta,
                                                         const int* __restrict__ row_list, const int* __restrict__ n_list) {
  const int nb_rows = row_list ? *n_list : mb;
  const int64_t n_point = (int64_t)nb_rows * bs;
  const int lane = threadIdx.x & 31;
  const int sl = lane % lpr;
  const int j0 = sl / bs, i0 = sl % bs, dj = lpr / bs, di = lpr % bs;
  const int vpe = bs * bs;
  const int64_t groups_per_pass = ((int64_t)gridDim.x * blockDim.x) / lpr;
  // every lane of a warp runs the same number of passes (the group sum is a full-warp shuffle)
  const int64_t first = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / lpr;
  const int64_t warp_first = ((int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31)) / lpr;
  for (int64_t base = 0; warp_first + base < n_point; base += groups_per_pass) {
    const int64_t g = first + base;
    const bool valid = g < n_point;
    int brow = 0, lr = 0, rs = 0, re = 0;
    if (valid) {
      const int bi = (int)(g / bs);
      lr = (int)(g % bs);
      brow = row_list ? row_list[bi] : bi;
      rs = row_ptr[brow];
      re = row_ptr[brow + 1];
    }
    S sum = bsr_row_dot<S, 4, true>(vals + (int64_t)rs * vpe + lr * bs, col_idx + rs, x, (re - rs) * bs, bs, vpe, lpr, sl, j0, i0, dj, di);
    sum = bsr_group_sum(sum, lpr);
    if (valid && sl == 0) bsr_store(y + (int64_t)brow * bs + lr, sum, alpha, beta);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// the TMA-tiled kernel
// ---------------------------------------------------------------------------------------------------------------
// the ring of the BSR kernels: VCAP values per stage, columns and row-map entries for VCAP / 4 blocks (bs >= 2)
template <typename S, int VCAP, int STAGES>
using BsrTileRing = TileRing<S, VCAP, VCAP / 4, VCAP / 4, STAGES>;

template <typename S, int NW, int STAGES, int VCAP, int UNR>
__global__ void __launch_bounds__((NW + 1) * 32)
    bsr_tile_kernel(int mb, int64_t nnzb, int bs, int lpr, int lmaxb, int n_tiles, const int4* __restrict__ tiles,
                    const int* __restrict__ row_ptr, const int* __restrict__ col_idx, const S* __restrict__ vals,
                    const S* __restrict__ x, S* __restrict__ y, S alpha, S beta) {
  using Smem = BsrTileRing<S, VCAP, STAGES>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>(smem_raw);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int vpe = bs * bs;

  tile_ring_init(sm, NW);

  if (warp == NW) {
    tile_ring_produce(sm, lane, mb, nnzb, vpe, n_tiles, tiles, row_ptr, col_idx, vals);
  } else {
    // ------------------------------------------------ consumer warps
    const int G = bs * lpr;    // lanes of one block row
    const int BRW = 32 / G;    // block rows of one warp pass (>= 1: the host guarantees bs*lpr <= 32)
    const int b_in = lane / G;
    const int lr = (lane % G) / lpr, sl = lane % lpr;
    const bool lane_used = b_in < BRW;
    const int j0 = sl / bs, i0 = sl % bs, dj = lpr / bs, di = lpr % bs;
    for (int it = 0; tile_ring_more(it, n_tiles); ++it) {
      const TileView tv = tile_ring_acquire<4, 4>(sm, it);
      const int stage = tv.stage, r0 = tv.r0, r1 = tv.r1, s_al = tv.s_al;
      const S* sv = sm.vals[stage];
      const int* sc = sm.cols[stage];
      // absolute groups of BRW block rows are dealt round-robin to the warps
      const int g_first = r0 / BRW;
      int g = g_first + ((warp - g_first % NW) + NW) % NW;
      for (; g * BRW < r1; g += NW) {
        const int brow = g * BRW + b_in;
        const bool valid = lane_used && (brow >= r0) && (brow < r1);
        int rs = 0, re = 0;
        if (valid) tile_row_bounds(sm, stage, row_ptr, brow, brow - tv.r0_al, rs, re);
        const bool is_long = (re - rs) > lmaxb;  // left to bsr_vector_kernel
        if (is_long) re = rs;
        S sum = bsr_row_dot<S, UNR, false>(sv + (rs - s_al) * vpe + lr * bs, sc + (rs - s_al), x, (re - rs) * bs, bs, vpe, lpr, sl, j0, i0,
                                           dj, di);
        sum = bsr_group_sum(sum, lpr);
        if (valid && !is_long && sl == 0) bsr_store(y + (int64_t)brow * bs + lr, sum, alpha, beta);
      }
      tile_ring_release(sm, stage, lane);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// The tile kernel for the common small block sizes (BS compile-time, BS*BS <= 32): ELEMENT per lane.  A warp takes one
// block row at a time; lane L owns element e = L % BS^2 = (lr, i) of block slot p = L / BS^2, so a warp pass covers
// P = 32 / BS^2 whole blocks, read from the stage as ONE contiguous run of values (no bank conflicts, no index
// arithmetic beyond j*BS^2 + e) while the BS lanes that share a column i gather the same x entry (one request).  Per
// entry: LDS value, LDS block column, multiply-add for the x index, LDG x, FMA -- a quarter of the instructions of the
// run-time-bs walk above, which matters because 8 + 4/BS^2 bytes per entry leave fewer issue slots per byte than CSR's 12.
// After the row: sum over the BS lanes of a local row and over the P slots by shuffles, lanes (p = 0, i = 0) store.
// ---------------------------------------------------------------------------------------------------------------
template <typename S, int BS, int NW, int STAGES, int VCAP, int UNR>
__global__ void __launch_bounds__((NW + 1) * 32)
    bsr_tile_e_kernel(int mb, int64_t nnzb, int lmaxb, int n_tiles, const int4* __restrict__ tiles, const int* __restrict__ row_ptr,
                      const int* __restrict__ col_idx, const S* __restrict__ vals, const S* __restrict__ x, S* __restrict__ y, S alpha,
                      S beta) {
  using Smem = BsrTileRing<S, VCAP, STAGES>;
  constexpr int VPE = BS * BS;
  constexpr int P = 32 / VPE;
  static_assert(P >= 1, "element-per-lane kernel needs BS*BS <= 32");
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>(smem_raw);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  tile_ring_init(sm, NW);

  if (warp == NW) {
    tile_ring_produce(sm, lane, mb, nnzb, VPE, n_tiles, tiles, row_ptr, col_idx, vals);
  } else {
    const int p = lane / VPE, e = lane % VPE;
    const int lr = e / BS, i = e % BS;
    const bool lane_used = p < P;
    for (int it = 0; tile_ring_more(it, n_tiles); ++it) {
      const TileView tv = tile_ring_acquire<4, 4>(sm, it);
      const int stage = tv.stage, r0 = tv.r0, r1 = tv.r1, s_al = tv.s_al;
      const S* sv = sm.vals[stage];
      const int* sc = sm.cols[stage];
      // block rows dealt round-robin to the warps by absolute index
      for (int brow = r0 + ((warp - r0 % NW) + NW) % NW; brow < r1; brow += NW) {
        int rs, re;
        tile_row_bounds(sm, stage, row_ptr, brow, brow - tv.r0_al, rs, re);
        if (re - rs > lmaxb) continue;  // left to bsr_vector_kernel (uniform across the warp)
        const int nblk = re - rs;
        const S* vb = sv + (rs - s_al) * VPE + e;
        const int* cb = sc + (rs - s_al);
        S sum = S(0);
        const int nb_eff = lane_used ? nblk : 0;  // lanes beyond the last whole slot (32 % BS^2 of them) idle
        int j = p;
        for (; j + (UNR - 1) * P < nb_eff; j += UNR * P) {  // UNR blocks per lane in flight, no predicates
          unsigned c[UNR];
          S av[UNR], xv[UNR];
#pragma unroll
          for (int u = 0; u < UNR; ++u) {
            c[u] = (unsigned)(cb[j + u * P] * BS + i);
            av[u] = vb[(j + u * P) * VPE];
          }
#pragma unroll
          for (int u = 0; u < UNR; ++u) xv[u] = ldg(x + c[u]);
#pragma unroll
          for (int u = 0; u < UNR; ++u) sum += av[u] * xv[u];
        }
        for (; j < nb_eff; j += P) sum += vb[j * VPE] * ldg(x + (unsigned)(cb[j] * BS + i));
        // local row total: the BS lanes (lr, 0..BS-1) of a slot, then the P slots
        S t = sum;
#pragma unroll
        for (int q = 1; q < BS; ++q) t += __shfl_down_sync(0xffffffffu, sum, q);
        S r = t;
#pragma unroll
        for (int q = 1; q < P; ++q) r += __shfl_down_sync(0xffffffffu, t, q * VPE);
        if (p == 0 && i == 0) bsr_store(y + (int64_t)brow * BS + lr, r, alpha, beta);
      }
      tile_ring_release(sm, stage, lane);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// T / H: y (already scaled) += alpha * A^T x.  One warp per block row; lane q handles output (block q / bs, column
// q % bs): t = sum_ii a(ii, jj) * x(brow*bs + ii); t *= alpha; atomic add -- the reference functor's operations
// (impl.hpp:750-775).  X / Y strided so that the same kernel serves every multivector layout (grid.y = column).
// ---------------------------------------------------------------------------------------------------------------
template <typename S>
__global__ void __launch_bounds__(256) bsr_transpose_kernel(int mb, int bs, const int* __restrict__ row_ptr, const int* __restrict__ col_idx,
                                                            const S* __restrict__ vals, const S* __restrict__ X, int64_t xr, int64_t xc,
                                                            S* __restrict__ Y, int64_t yr, int64_t yc, S alpha) {
  const int lane = threadIdx.x & 31;
  const int vpe = bs * bs;
  const S* x = X + (int64_t)blockIdx.y * xc;
  S* y = Y + (int64_t)blockIdx.y * yc;
  const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int dj = 32 / bs, di = 32 % bs;
  for (int64_t brow = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; brow < mb; brow += warps) {
    const int rs = row_ptr[brow], re = row_ptr[brow + 1];
    const int nq = (re - rs) * bs;
    int j = lane / bs, jj = lane % bs;
    for (int q = lane; q < nq; q += 32) {
      const S* a = vals + (int64_t)(rs + j) * vpe + jj;
      S t = S(0);
      for (int ii = 0; ii < bs; ++ii) t += ld_stream(a + ii * bs) * ldg(x + (brow * bs + ii) * xr);
      t *= alpha;
      atomicAdd(y + ((int64_t)col_idx[rs + j] * bs + jj) * yr, t);
      jj += di;
      j += dj;
      if (jj >= bs) {
        jj -= bs;
        ++j;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// N, multivector: lpr lanes per point row, KT columns of Y in registers; grid.y = column tile.  Accumulation per
// (row, column) in the order of the rank-1 walk.
// ---------------------------------------------------------------------------------------------------------------
template <typename S, int KT>
__global__ void __launch_bounds__(256) bsr_mm_kernel(int mb, int bs, int lpr, int k, const int* __restrict__ row_ptr,
                                                     const int* __restrict__ col_idx, const S* __restrict__ vals, const S* __restrict__ X,
                                                     int64_t xr, int64_t xc, S* __restrict__ Y, int64_t yr, int64_t yc, S alpha, S beta) {
  const int64_t n_point = (int64_t)mb * bs;
  const int lane = threadIdx.x & 31;
  const int sl = lane % lpr;
  const int vpe = bs * bs;
  const int c0 = blockIdx.y * KT;
  const int kc = min(KT, k - c0);
  const int j0 = sl / bs, i0 = sl % bs, dj = lpr / bs, di = lpr % bs;
  const int64_t groups_per_pass = ((int64_t)gridDim.x * blockDim.x) / lpr;
  const int64_t first = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / lpr;
  const int64_t warp_first = ((int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31)) / lpr;
  for (int64_t base = 0; warp_first + base < n_point; base += groups_per_pass) {
    const int64_t g = first + base;
    const bool valid = g < n_point;
    int brow = 0, lr = 0, rs = 0, re = 0;
    if (valid) {
      brow = (int)(g / bs);
      lr = (int)(g % bs);
      rs = row_ptr[brow];
      re = row_ptr[brow + 1];
    }
    S acc[KT];
#pragma unroll
    for (int t = 0; t < KT; ++t) acc[t] = S(0);
    const S* vrow = vals + (int64_t)rs * vpe + lr * bs;
    const int* crow = col_idx + rs;
    const int nk = (re - rs) * bs;
    int j = j0, i = i0;
    for (int q = sl; q < nk; q += lpr) {
      const S a = ld_stream(vrow + (int64_t)j * vpe + i);
      const S* xp = X + ((int64_t)ld_stream(crow + j) * bs + i) * xr + (int64_t)c0 * xc;
#pragma unroll
      for (int t = 0; t < KT; ++t)
        if (t < kc) acc[t] += a * ldg(xp + t * xc);
      i += di;
      j += dj;
      if (i >= bs) {
        i -= bs;
        ++j;
      }
    }
#pragma unroll
    for (int t = 0; t < KT; ++t) acc[t] = bsr_group_sum(acc[t], lpr);
    if (valid && sl == 0) {
#pragma unroll
      for (int t = 0; t < KT; ++t)
        if (t < kc) bsr_store(Y + ((int64_t)brow * bs + lr) * yr + (int64_t)(c0 + t) * yc, acc[t], alpha, beta);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// N, multivector, tensor cores (SPMV_BSR_TC; fp64): one warp per block row and super-tile of 8*NT columns of X.
// The reference's only architecture-specific kernel is this product on wmma fragments (m8n8k4 for double,
// sparse/impl/KokkosSparse_spmv_bsrmatrix_impl.hpp:74-459, opt-in through SPMV_BSR_TC, spmv_bsrmatrix_spec.hpp:165-245);
// here it is mma.sync.m8n8k4.f64 issued directly, fragments loaded straight from global memory:
//   A fragment (8 x 4, row):  lane l holds A_blk(mt*8 + l/4, ks*4 + l%4)  -- 4 lanes read 32 contiguous bytes of a block row
//   B fragment (4 x 8, col):  lane l holds X(cb*bs + ks*4 + l%4, n0 + l/4) -- 8 lanes read 64 contiguous bytes of a row-major X row
//   C fragment (8 x 8):       lane l holds Y(mt*8 + l/4, n0 + 2*(l%4) + {0, 1})
// Rows / columns of a block beyond bs are fed as zeros (any bs <= 8*MT), columns of X beyond k likewise.  Each block of
// A is read once for all 8*NT columns (the scalar kernel re-reads it per 4 columns).  The sums inside an MMA are the
// tensor core's; between blocks the order is the storage order.
// ---------------------------------------------------------------------------------------------------------------
#ifdef B200SP_EMU
__device__ __forceinline__ void dmma_m8n8k4(double (&c)[2], double a, double b) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  for (int kk = 0; kk < 4; ++kk) {
    const double av = __shfl_sync(0xffffffffu, a, g * 4 + kk);
    const double b0 = __shfl_sync(0xffffffffu, b, (2 * t) * 4 + kk);
    const double b1 = __shfl_sync(0xffffffffu, b, (2 * t + 1) * 4 + kk);
    c[0] += av * b0;
    c[1] += av * b1;
  }
}
#else
__device__ __forceinline__ void dmma_m8n8k4(double (&c)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
               : "+d"(c[0]), "+d"(c[1])
               : "d"(a), "d"(b));
}
#endif

template <int MT, int NT>
__global__ void __launch_bounds__(256) bsr_mm_tc_kernel(int mb, int bs, int k, const int* __restrict__ row_ptr,
                                                        const int* __restrict__ col_idx, const double* __restrict__ vals,
                                                        const double* __restrict__ X, int64_t xr, int64_t xc,
                                                        double* __restrict__ Y, int64_t yr, int64_t yc, double alpha, double beta) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int n0 = blockIdx.y * (8 * NT);
  const int vpe = bs * bs;
  const int KS = (bs + 3) >> 2;
  const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t brow = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; brow < mb; brow += warps) {
    const int rs = row_ptr[brow], re = row_ptr[brow + 1];
    double acc[MT][NT][2];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) acc[mt][nt][0] = acc[mt][nt][1] = 0.0;
    for (int j = rs; j < re; ++j) {
      const int cb = ld_stream(col_idx + j);
      const double* ab = vals + (int64_t)j * vpe;
      for (int ks = 0; ks < KS; ++ks) {
        const int kk = ks * 4 + t;  // column of the block = row of the X panel
        const bool kin = kk < bs;
        double b[NT];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
          const int n = n0 + nt * 8 + g;
          b[nt] = (kin && n < k) ? ldg(X + ((int64_t)cb * bs + kk) * xr + (int64_t)n * xc) : 0.0;
        }
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
          const int r = mt * 8 + g;
          const double a = (kin && r < bs) ? ld_stream(ab + r * bs + kk) : 0.0;
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) dmma_m8n8k4(acc[mt][nt], a, b[nt]);
        }
      }
    }
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      const int r = mt * 8 + g;
      if (r < bs) {
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int n = n0 + nt * 8 + 2 * t + e;
            if (n < k) bsr_store(Y + ((int64_t)brow * bs + r) * yr + (int64_t)n * yc, acc[mt][nt][e], alpha, beta);
          }
      }
    }
  }
}

int pick_lpr(double avg_entries_per_point_row, int bs, int cap) {
  int lpr = avg_entries_per_point_row <= 8.0 ? 2 : avg_entries_per_point_row <= 96.0 ? 4 : avg_entries_per_point_row <= 384.0 ? 8 : 16;
  while (lpr > 1 && bs * lpr > cap) lpr >>= 1;
  return lpr;
}

}  // namespace
}  // namespace b200sp

using namespace b200sp;

struct b200sp_spmv_plan;
extern "C" int b200sp_spmv_plan_create(b200sp_spmv_plan** plan, int algo);
extern "C" int b200sp_spmv_plan_destroy(b200sp_spmv_plan* p, void* stream);

struct b200sp_bsr_plan {
  b200sp::TileAnalysis a;  // of the block rows, blocks for entries
  b200sp::PlanKey key;     // of the analysed structure
  // blockDim() == 1 is a CrsMatrix (KokkosSparse_spmv.hpp:169-185): forwarded to the CSR path
  b200sp_spmv_plan* crs = nullptr;
  int algo = 0;  // B200SP_BSR_ALGO_*: 1 = tensor cores for the multivector product (SPMV_BSR_TC)
  char last_kernel[128] = "none";
};

namespace b200sp {
namespace {

int bsr_analyse(b200sp_bsr_plan* p, cudaStream_t st, int mb, int64_t nnzb, int bs, int capb, const int* row_ptr) {
  const PlanKey key{row_ptr, nullptr, mb, -1, nnzb, bs, capb};
  if (p->key == key) return B200SP_OK;
  p->key = PlanKey();
  p->a.release(st);
  const int rc = tile_analyse(st, mb, nnzb, row_ptr, capb, capb / 4, &p->a);  // blocks for entries
  if (rc != B200SP_OK) return rc;
  p->key = key;
  return B200SP_OK;
}

template <typename S>
int launch_vector(b200sp_bsr_plan* p, cudaStream_t st, int mb, int64_t nnzb, int bs, const int* rp, const int* ci, const S* v, const S* x,
                  S* y, S alpha, S beta) {
  const double avg = mb > 0 ? (double)nnzb * bs / (double)mb : 0.0;
  const int lpr = pick_lpr(avg, 1, 32);
  const int64_t threads = (int64_t)mb * bs * lpr;
  const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>((threads + 255) / 256, (int64_t)sm_count() * 16));
  bsr_vector_kernel<S><<<blocks, 256, 0, st>>>(mb, bs, lpr, rp, ci, v, x, y, alpha, beta, nullptr, nullptr);
  B200SP_LAUNCH_CHECK();
  snprintf(p->last_kernel, sizeof(p->last_kernel), "bsr_vector<%s,bs=%d,LPR=%d>", sizeof(S) == 8 ? "f64" : "f32", bs, lpr);
  return B200SP_OK;
}

template <typename S, int NW, int STAGES, int VCAP>
int launch_tile(b200sp_bsr_plan* p, cudaStream_t st, int mb, int64_t nnzb, int bs, const int* rp, const int* ci, const S* v, const S* x,
                S* y, S alpha, S beta) {
  using Smem = BsrTileRing<S, VCAP, STAGES>;
  constexpr int UNR = 4;
  auto kern = bsr_tile_kernel<S, NW, STAGES, VCAP, UNR>;
  const size_t smem = sizeof(Smem) + 128;
  static KernelSetup ks;
  int occ_dev = 1;
  if (int rc0 = kernel_setup(ks, kern, (NW + 1) * 32, smem, &occ_dev)) return rc0;
  int capb = std::min(Smem::CCAP, VCAP / (bs * bs)) & ~3;
  int rc = bsr_analyse(p, st, mb, nnzb, bs, capb, rp);
  if (rc != B200SP_OK) return rc;
  const double avg = mb > 0 ? (double)nnzb * bs / (double)mb : 0.0;
  const int lpr = pick_lpr(avg, bs, 32);
  const int grid = std::max(1, std::min(p->a.n_tiles, sm_count() * occ_dev));
  kern<<<grid, (NW + 1) * 32, smem, st>>>(mb, nnzb, bs, lpr, p->a.LMAX, p->a.n_tiles, p->a.tiles, rp, ci, v, x, y, alpha, beta);
  B200SP_LAUNCH_CHECK();
  // block rows longer than a stage: one warp per point row, list and count stay on the device
  const int lblocks = sm_count() * 2;
  bsr_vector_kernel<S><<<lblocks, 256, 0, st>>>(mb, bs, 32, rp, ci, v, x, y, alpha, beta, p->a.long_rows, p->a.n_long);
  B200SP_LAUNCH_CHECK();
  snprintf(p->last_kernel, sizeof(p->last_kernel), "bsr_tile<%s,bs=%d,LPR=%d,NW=%d,STAGES=%d,VCAP=%d>grid=%d", sizeof(S) == 8 ? "f64" : "f32",
           bs, lpr, NW, STAGES, VCAP, grid);
  return B200SP_OK;
}

template <typename S, int BS, int NW, int STAGES, int VCAP>
int launch_tile_e(b200sp_bsr_plan* p, cudaStream_t st, int mb, int64_t nnzb, const int* rp, const int* ci, const S* v, const S* x, S* y,
                  S alpha, S beta) {
  using Smem = BsrTileRing<S, VCAP, STAGES>;
  constexpr int UNR = 4;
  auto kern = bsr_tile_e_kernel<S, BS, NW, STAGES, VCAP, UNR>;
  const size_t smem = sizeof(Smem) + 128;
  static KernelSetup ks;
  int occ_dev = 1;
  if (int rc0 = kernel_setup(ks, kern, (NW + 1) * 32, smem, &occ_dev)) return rc0;
  const int capb = std::min(Smem::CCAP, VCAP / (BS * BS)) & ~3;
  int rc = bsr_analyse(p, st, mb, nnzb, BS, capb, rp);
  if (rc != B200SP_OK) return rc;
  const int grid = std::max(1, std::min(p->a.n_tiles, sm_count() * occ_dev));
  kern<<<grid, (NW + 1) * 32, smem, st>>>(mb, nnzb, p->a.LMAX, p->a.n_tiles, p->a.tiles, rp, ci, v, x, y, alpha, beta);
  B200SP_LAUNCH_CHECK();
  bsr_vector_kernel<S><<<sm_count() * 2, 256, 0, st>>>(mb, BS, 32, rp, ci, v, x, y, alpha, beta, p->a.long_rows, p->a.n_long);
  B200SP_LAUNCH_CHECK();
  snprintf(p->last_kernel, sizeof(p->last_kernel), "bsr_tile_e<%s,BS=%d,NW=%d,STAGES=%d,VCAP=%d>grid=%d", sizeof(S) == 8 ? "f64" : "f32", BS,
           NW, STAGES, VCAP, grid);
  return B200SP_OK;
}

bool aligned16(const void* a, const void* b, const void* c) { return ((((uintptr_t)a) | ((uintptr_t)b) | ((uintptr_t)c)) & 15u) == 0; }

template <typename S>
int crs_forward(b200sp_bsr_plan* p, cudaStream_t st, char mode, int m, int n, int64_t nnz, S alpha, const int* rp, const int* ci,
                const S* v, const S* x, S beta, S* y);
template <>
int crs_forward<double>(b200sp_bsr_plan* p, cudaStream_t st, char mode, int m, int n, int64_t nnz, double alpha, const int* rp,
                        const int* ci, const double* v, const double* x, double beta, double* y) {
  return b200sp_spmv_f64_i32(p->crs, st, mode, m, n, nnz, alpha, rp, ci, v, x, beta, y);
}
template <>
int crs_forward<float>(b200sp_bsr_plan* p, cudaStream_t st, char mode, int m, int n, int64_t nnz, float alpha, const int* rp, const int* ci,
                       const float* v, const float* x, float beta, float* y) {
  return b200sp_spmv_f32_i32(p->crs, st, mode, m, n, nnz, alpha, rp, ci, v, x, beta, y);
}

int check_common(b200sp_bsr_plan* p, char& mode, int mb, int nb, int64_t nnzb, int bs, const void* rp, const void* ci, const void* v) {
  B200SP_REQUIRE(p != nullptr, "bsr spmv: null plan");
  if (mode >= 'a' && mode <= 'z') mode = (char)(mode - 'a' + 'A');
  B200SP_REQUIRE(mode == 'N' || mode == 'C' || mode == 'T' || mode == 'H', "bsr spmv: invalid mode '%c' (N, C, T or H)", mode);
  B200SP_REQUIRE(mb >= 0 && nb >= 0 && nnzb >= 0, "bsr spmv: negative dimension (mb=%d nb=%d nnzb=%lld)", mb, nb, (long long)nnzb);
  B200SP_REQUIRE(bs >= 1, "bsr spmv: inappropriate block size %d", bs);  // BsrMatrix.hpp:429-433
  B200SP_REQUIRE((int64_t)mb * bs <= INT32_MAX && (int64_t)nb * bs <= INT32_MAX, "bsr spmv: point dimensions exceed int32");
  B200SP_REQUIRE(nnzb <= INT32_MAX, "bsr spmv: nnzb exceeds the int32 offset type");
  B200SP_REQUIRE(mb == 0 || rp != nullptr, "bsr spmv: null row map");
  B200SP_REQUIRE(nnzb == 0 || (ci != nullptr && v != nullptr), "bsr spmv: null entries / values");
  return B200SP_OK;
}

template <typename S>
int bsr_spmv_impl(b200sp_bsr_plan* p, cudaStream_t st, char mode, int mb, int nb, int64_t nnzb, int bs, S alpha, const int* rp,
                  const int* ci, const S* v, const S* x, S beta, S* y) {
  int rc = check_common(p, mode, mb, nb, nnzb, bs, rp, ci, v);
  if (rc != B200SP_OK) return rc;
  const bool trans = (mode == 'T' || mode == 'H');
  const int64_t ylen = (int64_t)(trans ? nb : mb) * bs;
  const int64_t xlen = (int64_t)(trans ? mb : nb) * bs;
  B200SP_REQUIRE(ylen == 0 || y != nullptr, "bsr spmv: null y");
  if (ylen == 0) return B200SP_OK;
  if (alpha == S(0) || nnzb == 0 || mb == 0 || xlen == 0) {
    snprintf(p->last_kernel, sizeof(p->last_kernel), "scale");
    return launch_scale2d<S>(st, ylen, 1, beta, y, 1, 0);
  }
  B200SP_REQUIRE(x != nullptr, "bsr spmv: null x");
  if (bs == 1) {
    if (!p->crs) {
      rc = b200sp_spmv_plan_create(&p->crs, B200SP_SPMV_DEFAULT);
      if (rc != B200SP_OK) return rc;
    }
    snprintf(p->last_kernel, sizeof(p->last_kernel), "crs(blockDim=1)");
    return crs_forward<S>(p, st, mode, mb, nb, nnzb, alpha, rp, ci, v, x, beta, y);
  }
  if (trans) {
    rc = launch_scale2d<S>(st, ylen, 1, beta, y, 1, 0);
    if (rc != B200SP_OK) return rc;
    const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>(((int64_t)mb + 7) / 8, (int64_t)sm_count() * 16));
    bsr_transpose_kernel<S><<<dim3(blocks, 1), 256, 0, st>>>(mb, bs, rp, ci, v, x, 1, 0, y, 1, 0, alpha);
    B200SP_LAUNCH_CHECK();
    snprintf(p->last_kernel, sizeof(p->last_kernel), "bsr_transpose<%s,bs=%d>", sizeof(S) == 8 ? "f64" : "f32", bs);
    return B200SP_OK;
  }
  const char* force = getenv("B200SP_BSR_KERNEL");
  bool tile = aligned16(rp, ci, v) && bs <= 16 && nnzb >= 64;
  if (force && !strcmp(force, "vector")) tile = false;
  if (!tile) return launch_vector<S>(p, st, mb, nnzb, bs, rp, ci, v, x, y, alpha, beta);
  if (!(force && !strcmp(force, "walk"))) {  // element-per-lane kernel for the block sizes it is instantiated for
    switch (bs) {
      case 2: return launch_tile_e<S, 2, 16, 4, 2048>(p, st, mb, nnzb, rp, ci, v, x, y, alpha, beta);
      case 3: return launch_tile_e<S, 3, 16, 4, 2048>(p, st, mb, nnzb, rp, ci, v, x, y, alpha, beta);
      case 4: return launch_tile_e<S, 4, 16, 4, 2048>(p, st, mb, nnzb, rp, ci, v, x, y, alpha, beta);
      case 5: return launch_tile_e<S, 5, 16, 3, 4096>(p, st, mb, nnzb, rp, ci, v, x, y, alpha, beta);
      default: break;
    }
  }
  // The run-time block size ("walk") tile kernel lost to the row-vector kernel from bs = 5 on when it was tuned (lap27 pattern,
  // 6.9 M blocks): it serves bs <= 4 and explicit requests only.
  if constexpr (sizeof(S) == 8) {
    // bs 6..16 in double: the tensor-core multivector kernel with ONE column (x contiguous: row stride 1).  Seven of the eight
    // columns of each MMA are zeros, but the MMA is not what bounds the product -- the loads of the blocks are, and the fragment
    // loads of that kernel (4 lanes x 32 contiguous bytes of a block row) are cheaper than the row-vector kernel's walk.
    // B200SP_BSR_KERNEL=vector|walk keeps the other kernels; SPMV_BSR_V41 / V42 requests keep the scalar ones as well.
    if (bs >= 6 && bs <= 16 && !force && p->algo != B200SP_BSR_ALGO_SCALAR) {
      const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>(((int64_t)mb + 7) / 8, (int64_t)sm_count() * 16));
      if (bs <= 8)
        bsr_mm_tc_kernel<1, 1><<<dim3(blocks, 1), 256, 0, st>>>(mb, bs, 1, rp, ci, (const double*)v, (const double*)x, 1, 0, (double*)y, 1, 0,
                                                                (double)alpha, (double)beta);
      else
        bsr_mm_tc_kernel<2, 1><<<dim3(blocks, 1), 256, 0, st>>>(mb, bs, 1, rp, ci, (const double*)v, (const double*)x, 1, 0, (double*)y, 1, 0,
                                                                (double)alpha, (double)beta);
      B200SP_LAUNCH_CHECK();
      snprintf(p->last_kernel, sizeof(p->last_kernel), "bsr_mm_tc<f64,bs=%d,m8n8k4,MT=%d,NT=1>x1", bs, bs <= 8 ? 1 : 2);
      return B200SP_OK;
    }
  }
  if (bs > 4 && !(force && !strcmp(force, "walk"))) return launch_vector<S>(p, st, mb, nnzb, bs, rp, ci, v, x, y, alpha, beta);
  if (bs <= 4) return launch_tile<S, 16, 4, 2048>(p, st, mb, nnzb, bs, rp, ci, v, x, y, alpha, beta);
  return launch_tile<S, 16, 3, 4096>(p, st, mb, nnzb, bs, rp, ci, v, x, y, alpha, beta);
}

template <typename S>
int bsr_spmm_impl(b200sp_bsr_plan* p, cudaStream_t st, char mode, int mb, int nb, int64_t nnzb, int bs, int k, S alpha, const int* rp,
                  const int* ci, const S* v, const S* X, int64_t ldx, int x_row_major, S beta, S* Y, int64_t ldy, int y_row_major) {
  int rc = check_common(p, mode, mb, nb, nnzb, bs, rp, ci, v);
  if (rc != B200SP_OK) return rc;
  B200SP_REQUIRE(k >= 0, "bsr spmm: negative column count");
  const bool trans = (mode == 'T' || mode == 'H');
  const int64_t ylen = (int64_t)(trans ? nb : mb) * bs;
  const int64_t xlen = (int64_t)(trans ? mb : nb) * bs;
  if (ylen == 0 || k == 0) return B200SP_OK;
  B200SP_REQUIRE(Y != nullptr, "bsr spmm: null Y");
  B200SP_REQUIRE(y_row_major ? ldy >= k : ldy >= ylen, "bsr spmm: leading dimension of Y too small");
  const int64_t yr = y_row_major ? ldy : 1, yc = y_row_major ? 1 : ldy;
  if (alpha == S(0) || nnzb == 0 || mb == 0 || xlen == 0) {
    snprintf(p->last_kernel, sizeof(p->last_kernel), "scale");
    return launch_scale2d<S>(st, ylen, k, beta, Y, yr, yc);
  }
  B200SP_REQUIRE(X != nullptr, "bsr spmm: null X");
  B200SP_REQUIRE(x_row_major ? ldx >= k : ldx >= xlen, "bsr spmm: leading dimension of X too small");
  const int64_t xr = x_row_major ? ldx : 1, xc = x_row_major ? 1 : ldx;
  if (trans) {
    rc = launch_scale2d<S>(st, ylen, k, beta, Y, yr, yc);
    if (rc != B200SP_OK) return rc;
    const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>(((int64_t)mb + 7) / 8, (int64_t)sm_count() * 16));
    for (int c0 = 0; c0 < k; c0 += 65535) {  // grid.y limit
      const int kc = std::min(k - c0, 65535);
      bsr_transpose_kernel<S><<<dim3(blocks, kc), 256, 0, st>>>(mb, bs, rp, ci, v, X + (int64_t)c0 * xc, xr, xc, Y + (int64_t)c0 * yc, yr, yc,
                                                                alpha);
      B200SP_LAUNCH_CHECK();
    }
    snprintf(p->last_kernel, sizeof(p->last_kernel), "bsr_transpose<%s,bs=%d>x%d", sizeof(S) == 8 ? "f64" : "f32", bs, k);
    return B200SP_OK;
  }
  if constexpr (sizeof(S) == 8) {
    // SPMV_BSR_TC (spmv_bsrmatrix_spec.hpp:176-245): no-transpose multivector products in double; anything else falls back,
    // as the reference does when its tensor-core functor is unavailable.  B200SP_BSR_MM=tc|scalar overrides the plan.
    // Default = tensor cores from 4 columns on, several times faster than the scalar kernel at k = 16 when it was tuned
    // (differences between the two at the 1e-14 level, far inside the reference's tolerance law).
    const char* fm = getenv("B200SP_BSR_MM");
    const bool tc = fm ? !strcmp(fm, "tc") : (p->algo == B200SP_BSR_ALGO_TENSOR_CORES || (p->algo == B200SP_BSR_ALGO_DEFAULT && k >= 4));
    if (tc && bs >= 2 && bs <= 16) {
      const int NT = k > 8 ? 2 : 1;
      const int warps_per_cta = 8;
      const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>(((int64_t)mb + warps_per_cta - 1) / warps_per_cta, (int64_t)sm_count() * 16));
      const int tiles = (k + 8 * NT - 1) / (8 * NT);
      for (int t0 = 0; t0 < tiles; t0 += 65535) {
        const int tn = std::min(tiles - t0, 65535);
        const int c0 = t0 * 8 * NT;
        const int kc = std::min(k - c0, tn * 8 * NT);
        const dim3 grid(blocks, tn);
        const double* Xc = (const double*)X + (int64_t)c0 * xc;
        double* Yc = (double*)Y + (int64_t)c0 * yc;
#define B200SP_TC(MT_, NT_) bsr_mm_tc_kernel<MT_, NT_><<<grid, 256, 0, st>>>(mb, bs, kc, rp, ci, (const double*)v, Xc, xr, xc, Yc, yr, yc, (double)alpha, (double)beta)
        if (bs <= 8) {
          if (NT == 2) B200SP_TC(1, 2); else B200SP_TC(1, 1);
        } else {
          if (NT == 2) B200SP_TC(2, 2); else B200SP_TC(2, 1);
        }
#undef B200SP_TC
        B200SP_LAUNCH_CHECK();
      }
      snprintf(p->last_kernel, sizeof(p->last_kernel), "bsr_mm_tc<f64,bs=%d,m8n8k4,MT=%d,NT=%d>", bs, bs <= 8 ? 1 : 2, NT);
      return B200SP_OK;
    }
  }
  constexpr int KT = 4;
  const double avg = (double)nnzb * bs / (double)mb;
  const int lpr = pick_lpr(avg, 1, 32);
  const int64_t threads = (int64_t)mb * bs * lpr;
  const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>((threads + 255) / 256, (int64_t)sm_count() * 16));
  for (int c0 = 0; c0 < k; c0 += 65535 * KT) {
    const int kc = std::min(k - c0, 65535 * KT);
    bsr_mm_kernel<S, KT><<<dim3(blocks, (kc + KT - 1) / KT), 256, 0, st>>>(mb, bs, lpr, kc, rp, ci, v, X + (int64_t)c0 * xc, xr, xc,
                                                                          Y + (int64_t)c0 * yc, yr, yc, alpha, beta);
    B200SP_LAUNCH_CHECK();
  }
  snprintf(p->last_kernel, sizeof(p->last_kernel), "bsr_mm<%s,bs=%d,LPR=%d,KT=%d>", sizeof(S) == 8 ? "f64" : "f32", bs, lpr, KT);
  return B200SP_OK;
}

}  // namespace
}  // namespace b200sp

extern "C" {

int b200sp_bsr_plan_create(b200sp_bsr_plan** plan) {
  B200SP_REQUIRE(plan != nullptr, "bsr plan_create: null output pointer");
  *plan = new (std::nothrow) b200sp_bsr_plan();
  B200SP_REQUIRE(*plan != nullptr, "bsr plan_create: out of host memory");
  return B200SP_OK;
}

int b200sp_bsr_plan_destroy(b200sp_bsr_plan* p, void* stream) {
  if (!p) return B200SP_OK;
  p->a.release((cudaStream_t)stream);
  if (p->crs) b200sp_spmv_plan_destroy(p->crs, stream);
  delete p;
  return B200SP_OK;
}

const char* b200sp_bsr_last_kernel(const b200sp_bsr_plan* p) { return p ? p->last_kernel : "none"; }

int b200sp_bsr_plan_set_algorithm(b200sp_bsr_plan* p, int algo) {
  B200SP_REQUIRE(p != nullptr, "bsr_plan_set_algorithm: null plan");
  B200SP_REQUIRE(algo == B200SP_BSR_ALGO_DEFAULT || algo == B200SP_BSR_ALGO_TENSOR_CORES || algo == B200SP_BSR_ALGO_SCALAR,
                 "bsr_plan_set_algorithm: unknown algorithm %d", algo);
  p->algo = algo;
  return B200SP_OK;
}

int b200sp_bsr_spmv_f64_i32(b200sp_bsr_plan* plan, void* stream, char mode, int mb, int nb, int64_t nnzb, int bs, double alpha,
                            const int* row_ptr, const int* col_idx, const double* vals, const double* x, double beta, double* y) {
  return bsr_spmv_impl<double>(plan, (cudaStream_t)stream, mode, mb, nb, nnzb, bs, alpha, row_ptr, col_idx, vals, x, beta, y);
}
int b200sp_bsr_spmv_f32_i32(b200sp_bsr_plan* plan, void* stream, char mode, int mb, int nb, int64_t nnzb, int bs, float alpha,
                            const int* row_ptr, const int* col_idx, const float* vals, const float* x, float beta, float* y) {
  return bsr_spmv_impl<float>(plan, (cudaStream_t)stream, mode, mb, nb, nnzb, bs, alpha, row_ptr, col_idx, vals, x, beta, y);
}
int b200sp_bsr_spmm_f64_i32(b200sp_bsr_plan* plan, void* stream, char mode, int mb, int nb, int64_t nnzb, int bs, int k, double alpha,
                            const int* row_ptr, const int* col_idx, const double* vals, const double* X, int64_t ldx, int x_row_major,
                            double beta, double* Y, int64_t ldy, int y_row_major) {
  return bsr_spmm_impl<double>(plan, (cudaStream_t)stream, mode, mb, nb, nnzb, bs, k, alpha, row_ptr, col_idx, vals, X, ldx, x_row_major,
                               beta, Y, ldy, y_row_major);
}
int b200sp_bsr_spmm_f32_i32(b200sp_bsr_plan* plan, void* stream, char mode, int mb, int nb, int64_t nnzb, int bs, int k, float alpha,
                            const int* row_ptr, const int* col_idx, const float* vals, const float* X, int64_t ldx, int x_row_major,
                            float beta, float* Y, int64_t ldy, int y_row_major) {
  return bsr_spmm_impl<float>(plan, (cudaStream_t)stream, mode, mb, nb, nnzb, bs, k, alpha, row_ptr, col_idx, vals, X, ldx, x_row_major,
                              beta, Y, ldy, y_row_major);
}

}  // extern "C"
