// spgemm.cu -- C = A*B on CrsMatrix data for H100 (sm_90a): symbolic + numeric.
//
// Replaces the reference's Kokkos::Cuda SpGEMM legs
//   native  KokkosSPGEMM symbolic (compression + StructureC hash kernels)
//           sparse/impl/KokkosSparse_spgemm_impl_symbolic.hpp:903-1100,1513-1957
//   native  numeric PortableNumericCHASH / NumericCMEM + sort_crs_matrix
//           sparse/impl/KokkosSparse_spgemm_impl_kkmem.hpp:410-1021,1173-1258,
//           sparse/impl/KokkosSparse_spgemm_numeric_spec.hpp:138-140
//   TPL     cusparseSpGEMMreuse_*
//           sparse/tpls/KokkosSparse_spgemm_{symbolic,numeric}_tpl_spec_decl.hpp
// Results follow the reference's SPGEMM_DEBUG host path (impl_seq.hpp:23-182)
// after sort_crs_matrix: row_ptr / col_idx bit-identical, values by its
// accumulation law (sum of b_val*a_val, association differs).
//
// Design (DESIGN.md section 4)
//  symbolic: per-row flop bound f_i and column span [cmin_i, cmax_i] from one
//    pass over A (+ a min/max pass over B's rows); rows binned by f_i; each bin
//    runs a shared-memory hash-set kernel (group of G threads per row, atomicCAS
//    on keys) that counts distinct columns; rows too big for shared memory use
//    a per-CTA global bitmap.  Exclusive scan -> row_ptr_C, c_nnz, max row.
//  numeric: rows binned by nnz(C_i); a group of threads builds the row in a
//    shared-memory accumulator addressed by a MONOTONE map of the column
//    (dense accumulator when the row's span fits the table, order-preserving
//    hash with linear probing otherwise), so the table is already sorted up to
//    its probe clusters; an in-cluster rank turns slots into sorted output
//    positions -- the separate sort_crs_matrix pass of the reference is gone.
//    Rows that overflow or exceed shared memory go to a global-memory hash +
//    in-place bitonic sort kernel.
#include "common.cuh"
#include "scan.cuh"
#include "spgemm_esc.cuh"
#include "bspgemm.cuh"
#include <algorithm>
#include <limits.h>
#include <stdlib.h>
#include <time.h>
#include <new>

namespace b200sp {

static constexpr int EMPTY = -1;

// ---------------------------------------------------------------------------
// small utilities
// ---------------------------------------------------------------------------
__global__ void fill_int_kernel(int64_t n, int v, int* __restrict__ p) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}

// per-row min / max column of B (EMPTY rows: min = INT_MAX, max = -1)
__global__ void brow_minmax_kernel(int n, const int* __restrict__ rp, const int* __restrict__ ci,
                                   int* __restrict__ bmin, int* __restrict__ bmax) {
  // 8 lanes per row
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int r = (int)(t >> 3), sl = (int)(t & 7);
  int mn = INT_MAX, mx = -1;
  if (r < n)
    for (int j = rp[r] + sl; j < rp[r + 1]; j += 8) {
      const int c = ci[j];
      mn = min(mn, c);
      mx = max(mx, c);
    }
#pragma unroll
  for (int o = 4; o > 0; o >>= 1) {
    mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if (r < n && sl == 0) {
    bmin[r] = mn;
    bmax[r] = mx;
  }
}

// per A-row: flop bound, column span of the product row
__global__ void arow_analyse_kernel(int m, const int* __restrict__ rpA, const int* __restrict__ ciA,
                                    const int* __restrict__ rpB, const int* __restrict__ bmin,
                                    const int* __restrict__ bmax, int* __restrict__ flops,
                                    int* __restrict__ cmin, int* __restrict__ cmax) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int r = (int)(t >> 3), sl = (int)(t & 7);
  long long f = 0;
  int mn = INT_MAX, mx = -1;
  if (r < m)
    for (int j = rpA[r] + sl; j < rpA[r + 1]; j += 8) {
      const int c = ciA[j];
      f += rpB[c + 1] - rpB[c];
      mn = min(mn, bmin[c]);
      mx = max(mx, bmax[c]);
    }
#pragma unroll
  for (int o = 4; o > 0; o >>= 1) {
    f += __shfl_xor_sync(0xffffffffu, f, o);
    mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if (r < m && sl == 0) {
    flops[r] = (int)min(f, (long long)INT_MAX);
    cmin[r] = mn;
    cmax[r] = mx;
  }
}

// ---- binning: rows -> bins by a key array and ascending thresholds ---------
static constexpr int MAXBINS = 8;
struct BinSpec {
  int nb;               // number of bins (last bin = everything above thr[nb-2])
  int thr[MAXBINS];     // bin b holds keys <= thr[b] (and > thr[b-1])
};
__device__ __forceinline__ int bin_of(const BinSpec& s, int key) {
  int b = 0;
  while (b < s.nb - 1 && key > s.thr[b]) ++b;
  return b;
}
__global__ void bin_count_kernel(int m, const int* __restrict__ key, BinSpec spec, int* __restrict__ counts) {
  __shared__ int sc[MAXBINS];
  if (threadIdx.x < MAXBINS) sc[threadIdx.x] = 0;
  __syncthreads();
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < m; r += gridDim.x * blockDim.x) atomicAdd(&sc[bin_of(spec, key[r])], 1);
  __syncthreads();
  if (threadIdx.x < MAXBINS && sc[threadIdx.x]) atomicAdd(&counts[threadIdx.x], sc[threadIdx.x]);
}
__global__ void __launch_bounds__(256) bin_scatter_kernel(int m, const int* __restrict__ key, BinSpec spec, int* __restrict__ cursors,
                                   int* __restrict__ rows_out) {
  // block-aggregated: one global atomic per (CTA pass, bin) instead of one per row (2M atomics on ONE counter serialise for
  // milliseconds when every row falls into the same bin); the rows of a pass stay together, so a bin's list follows the
  // natural row order up to the order in which the passes reserve their ranges -- consecutive CTAs of the row kernels then
  // read neighbouring rows of A and write neighbouring rows of C
  __shared__ int scnt[MAXBINS];
  __shared__ int sbase[MAXBINS];
  const int passes = (m + (int)(gridDim.x * blockDim.x) - 1) / (int)(gridDim.x * blockDim.x);
  for (int it = 0; it < passes; ++it) {
    const int r = (it * gridDim.x + blockIdx.x) * blockDim.x + threadIdx.x;
    if (threadIdx.x < MAXBINS) scnt[threadIdx.x] = 0;
    __syncthreads();
    int b = -1, rank = 0;
    if (r < m) {
      b = bin_of(spec, key[r]);
      rank = atomicAdd(&scnt[b], 1);
    }
    __syncthreads();
    if (threadIdx.x < MAXBINS && scnt[threadIdx.x] > 0) sbase[threadIdx.x] = atomicAdd(&cursors[threadIdx.x], scnt[threadIdx.x]);
    __syncthreads();
    if (b >= 0) rows_out[sbase[b] + rank] = r;
    __syncthreads();
  }
}

// ESC bin key of a row (spgemm_esc.cuh): max(products, 2 * nnz(A_i)), saturated
__global__ void esc_key_kernel(int m, const int* __restrict__ flops, const int* __restrict__ rpA, int* __restrict__ key) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < m; r += gridDim.x * blockDim.x) {
    const long long na2 = 2LL * (rpA[r + 1] - rpA[r]);
    key[r] = (int)min(max((long long)flops[r], na2), (long long)INT_MAX);
  }
}
// old-path bin key: 0 for rows the ESC kernels take (key <= cap), else max(nnz(C_i), 1); all_rows: every row by nnz(C_i)
__global__ void rest_key_kernel(int m, const int* __restrict__ esc_key, int cap, const int* __restrict__ rpC, int all_rows,
                                int* __restrict__ key) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < m; r += gridDim.x * blockDim.x) {
    const int nz = rpC[r + 1] - rpC[r];
    key[r] = all_rows ? nz : (esc_key[r] <= cap ? 0 : max(nz, 1));
  }
}

// ---------------------------------------------------------------------------
// Product walker shared by symbolic and numeric.  A group of G threads expands row i of A*B:
// per batch of <= G entries of A it stages (B row start, B row length, A value) in shared memory
// with two rounds of independent loads; then sub-warps of LB lanes (LB ~ mean row length of B)
// each take staged entries round-robin, UT entries at a time, so that UT independent B-row reads
// per lane are in flight (a naive walk chains row_ptr_B -> col_idx_B loads per entry of A and is
// bound by HBM latency).  f(c, v) is called once per product; stop() lets the caller abandon the row.
// ---------------------------------------------------------------------------
template <int G, typename S>
struct WalkSmem {
  int bs[G];   // start of the B row of staged entry t
  int len[G];  // its length
  S va[G];     // A value of staged entry t
};

template <int G, bool WITH_VALS, typename S, typename F, typename Stop>
__device__ __forceinline__ void walk_products(int tg, int lb, int a0, int a1, const int* __restrict__ ciA,
                                              const S* __restrict__ vA, const int* __restrict__ rpB,
                                              const int* __restrict__ ciB, const S* __restrict__ vB,
                                              WalkSmem<G, S>& w, F&& f, Stop&& stop) {
  constexpr int UT = 4;
  auto gsync = [&]() {
    if (G <= 32) __syncwarp(); else __syncthreads();
  };
  const int nsub = G / lb;
  const int q = tg / lb, sl = tg % lb;
  for (int ab = a0; ab < a1; ab += G) {
    const int nA = min(G, a1 - ab);
    if (tg < nA) {
      const int ca = ciA[ab + tg];
      const int b0 = rpB[ca];
      w.bs[tg] = b0;
      w.len[tg] = rpB[ca + 1] - b0;
      if (WITH_VALS) w.va[tg] = vA[ab + tg];
    }
    gsync();
    for (int t0 = q; t0 < nA; t0 += nsub * UT) {
      int c[UT];
      S v[UT];
#pragma unroll
      for (int u = 0; u < UT; ++u) {
        const int t = t0 + u * nsub;
        c[u] = -1;
        if (t < nA && sl < w.len[t]) {
          const int jb = w.bs[t] + sl;
          c[u] = ld_stream(ciB + jb);
          if (WITH_VALS) v[u] = ld_stream(vB + jb) * w.va[t];  // b_val * val (impl_seq.hpp:163)
        }
      }
#pragma unroll
      for (int u = 0; u < UT; ++u)
        if (c[u] >= 0) f(c[u], WITH_VALS ? v[u] : S(0));
      // B rows longer than the sub-warp
#pragma unroll 1
      for (int u = 0; u < UT; ++u) {
        const int t = t0 + u * nsub;
        if (t < nA)
          for (int off = sl + lb; off < w.len[t]; off += lb) {
            const int jb = w.bs[t] + off;
            f(ld_stream(ciB + jb), WITH_VALS ? ld_stream(vB + jb) * w.va[t] : S(0));
          }
      }
      if (stop()) break;
    }
    gsync();  // staging is rewritten by the next batch
    if (stop()) break;
  }
}

// ---------------------------------------------------------------------------
// SYMBOLIC: count distinct columns of row i of A*B with a shared-memory hash set.
// G threads cooperate on one row; LB lanes walk one row of B.
// ---------------------------------------------------------------------------
__device__ __forceinline__ unsigned hash_mul(int c, int log2slots) {
  return ((unsigned)c * 0x9E3779B1u) >> (32 - log2slots);
}

template <int G, int LOG2SLOTS, bool V2 = false>
__global__ void __launch_bounds__(G <= 32 ? 256 : G)
    sym_hash_kernel(int nrows_bin, const int* __restrict__ rows, int lb, const int* __restrict__ rpA,
                    const int* __restrict__ ciA, const int* __restrict__ rpB, const int* __restrict__ ciB,
                    int* __restrict__ row_nnz) {
  constexpr int SLOTS = 1 << LOG2SLOTS;
  constexpr int THREADS = (G <= 32 ? 256 : G);
  constexpr int RPC = THREADS / G;
  extern __shared__ __align__(16) int sm_keys[];  // RPC * SLOTS
  __shared__ int sm_cnt[RPC];
  __shared__ WalkSmem<G, float> sm_walk[RPC];
  const int g = threadIdx.x / G, tg = threadIdx.x % G;
  int* keys = sm_keys + g * SLOTS;
  const int ridx = blockIdx.x * RPC + g;
  const bool active = ridx < nrows_bin;
  if (V2) {  // variant 2: 16-byte stores
    int4* k4 = reinterpret_cast<int4*>(keys);
    for (int s = tg; s < SLOTS / 4; s += G) k4[s] = make_int4(EMPTY, EMPTY, EMPTY, EMPTY);
  } else {
    for (int s = tg; s < SLOTS; s += G) keys[s] = EMPTY;
  }
  if (tg == 0) sm_cnt[g] = 0;
  if (G <= 32) __syncwarp(); else __syncthreads();
  int mine = 0;
  // inactive groups (tail CTA) walk an empty row so that block-wide barriers stay matched
  const int i = active ? rows[ridx] : 0;
  const int a0 = active ? rpA[i] : 0, a1 = active ? rpA[i + 1] : 0;
  walk_products<G, false, float>(
      tg, lb, a0, a1, ciA, (const float*)nullptr, rpB, ciB, (const float*)nullptr, sm_walk[g],
      [&](int c, float) {
        unsigned h = hash_mul(c, LOG2SLOTS);
        while (true) {
          const int kcur = ((volatile int*)keys)[h];
          if (kcur == c) break;
          if (kcur == EMPTY) {
            const int old = atomicCAS(&keys[h], EMPTY, c);
            if (old == EMPTY) {
              ++mine;
              break;
            }
            if (old == c) break;
          }
          h = (h + 1) & (SLOTS - 1);
        }
      },
      []() { return false; });
  // group reduce
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
  if (G <= 32) {
    if (active && tg == 0) row_nnz[i] = mine;
  } else {
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(&sm_cnt[g], mine);
    __syncthreads();
    if (active && tg == 0) row_nnz[i] = sm_cnt[g];
  }
}

// rows whose flop bound exceeds the largest shared-memory table: k-bit bitmap per CTA in global memory
__global__ void __launch_bounds__(256)
    sym_bitmap_kernel(int nrows_bin, const int* __restrict__ rows, int k, unsigned* __restrict__ bitmaps,
                      const int* __restrict__ rpA, const int* __restrict__ ciA, const int* __restrict__ rpB,
                      const int* __restrict__ ciB, int* __restrict__ row_nnz) {
  const int words = (k + 31) / 32;
  unsigned* bm = bitmaps + (size_t)blockIdx.x * words;
  __shared__ int cnt;
  for (int ridx = blockIdx.x; ridx < nrows_bin; ridx += gridDim.x) {
    const int i = rows[ridx];
    for (int w = threadIdx.x; w < words; w += 256) bm[w] = 0u;
    if (threadIdx.x == 0) cnt = 0;
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int ja = rpA[i] + warp; ja < rpA[i + 1]; ja += 8) {
      const int ca = ciA[ja];
      for (int jb = rpB[ca] + lane; jb < rpB[ca + 1]; jb += 32) {
        const int c = ciB[jb];
        atomicOr(&bm[c >> 5], 1u << (c & 31));
      }
    }
    __syncthreads();
    int local = 0;
    for (int w = threadIdx.x; w < words; w += 256) local += __popc(bm[w]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
    if (lane == 0 && local) atomicAdd(&cnt, local);
    __syncthreads();
    if (threadIdx.x == 0) row_nnz[i] = cnt;
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------
// NUMERIC: monotone-addressed shared-memory accumulator -> sorted row.
// ---------------------------------------------------------------------------
template <typename S>
__device__ __forceinline__ void smem_add(S* p, S v) {
  atomicAdd(p, v);
}

template <typename S, int G, int KSLOTS, int PAD, int VCAP>
struct NumLayout {
  static constexpr int TOT = KSLOTS + PAD;
  static constexpr int WORDS = (TOT + 31) / 32;
  // per row-group: vals[VCAP] | keys[TOT] | wpre[WORDS+1] | wmask[WORDS]
  static constexpr size_t PER = sizeof(S) * VCAP + sizeof(int) * TOT + sizeof(int) * (2 * WORDS + 2);
  static constexpr size_t PER_AL = (PER + 15) & ~(size_t)15;
};

template <typename S, int G, int KSLOTS, int PAD, int VCAP>
__global__ void __launch_bounds__(G <= 32 ? 256 : G)
    num_hash_kernel(int nrows_bin, const int* __restrict__ rows, int lb, const int* __restrict__ rpA,
                    const int* __restrict__ ciA, const S* __restrict__ vA, const int* __restrict__ rpB,
                    const int* __restrict__ ciB, const S* __restrict__ vB, const int* __restrict__ rpC,
                    int* __restrict__ ciC, S* __restrict__ vC, const int* __restrict__ cmin_arr,
                    const int* __restrict__ cmax_arr, int* __restrict__ fb_rows, int* __restrict__ fb_count) {
  // Sorted-by-construction accumulator.  The key table has >= 4x the row's nnz slots (load <= 0.25);
  // the slot of column c starts at the MONOTONE map h(c); keys are placed with atomicMin and the
  // displaced (larger) key is carried to the next slot -- ordered linear probing.  Every slot only
  // ever decreases and a carried key is never smaller than what it leaves behind, so at quiescence
  // each probe cluster is ascending and clusters are ordered by the monotone map: the occupied slots
  // read left to right ARE the sorted row.  An occupancy prefix turns slot -> output position; values
  // are accumulated by output position in a second walk over the products (keys no longer move) and
  // leave fully coalesced.  Dense rows (span <= KSLOTS) use h(c) = c - cmin: no probing at all.
  using L = NumLayout<S, G, KSLOTS, PAD, VCAP>;
  constexpr int THREADS = (G <= 32 ? 256 : G);
  constexpr int RPC = THREADS / G;
  constexpr int TOT = L::TOT;
  constexpr int WORDS = L::WORDS;
  constexpr int INF = INT_MAX;
  extern __shared__ __align__(16) unsigned char smraw[];
  __shared__ int sm_flag[RPC];
  __shared__ WalkSmem<G, S> sm_walk[RPC];
  const int g = threadIdx.x / G, tg = threadIdx.x % G;
  unsigned char* base = smraw + (size_t)g * L::PER_AL;
  S* vals = reinterpret_cast<S*>(base);
  int* keys = reinterpret_cast<int*>(base + sizeof(S) * VCAP);
  int* wpre = keys + TOT;
  unsigned* wmask = reinterpret_cast<unsigned*>(wpre + WORDS + 1);
  const int ridx = blockIdx.x * RPC + g;
  const bool active = ridx < nrows_bin;
  auto gsync = [&]() {
    if (G <= 32) __syncwarp(); else __syncthreads();
  };
  for (int s = tg; s < TOT; s += G) keys[s] = INF;
  for (int s = tg; s < VCAP; s += G) vals[s] = S(0);
  if (tg == 0) sm_flag[g] = 0;
  gsync();
  int i = 0, cbase = 0, nz = 0;
  if (active) {
    i = rows[ridx];
    cbase = rpC[i];
    nz = rpC[i + 1] - cbase;
  }
  const bool work = active && nz > 0;
  const int cmin = work ? cmin_arr[i] : 0;
  const long long span = work ? ((long long)cmax_arr[i] - cmin + 1) : 1;
  const bool dense = span <= KSLOTS;
  const unsigned long long mult = dense ? 0ull : (((unsigned long long)KSLOTS << 32) / (unsigned long long)span);
  const int a0 = work ? rpA[i] : 0, a1 = work ? rpA[i + 1] : 0;
  auto slot_of = [&](int c) -> int {
    return dense ? (c - cmin) : (int)(((unsigned long long)(unsigned)(c - cmin) * mult) >> 32);
  };
  auto stopped = [&]() { return ((volatile int*)sm_flag)[g] != 0; };
  // ---- walk 1: keys
  walk_products<G, false, S>(
      tg, lb, a0, a1, ciA, vA, rpB, ciB, vB, sm_walk[g],
      [&](int c, S) {
        int h = slot_of(c);
        while (true) {
          const int old = atomicMin(&keys[h], c);
          if (old == c || old == INF) return;  // already there / took an empty slot
          if (old > c) c = old;                // displaced a larger key: carry it on
          if (++h >= TOT) {
            sm_flag[g] = 1;  // ran off the pad: row goes to the fallback kernel
            return;
          }
        }
      },
      stopped);
  gsync();
  const bool overflow = sm_flag[g] != 0;
  if (active && overflow && tg == 0) fb_rows[atomicAdd(fb_count, 1)] = i;
  // ---- occupancy prefix: wpre[w] = occupied slots before word w; column indices leave now
  if (work && !overflow) {
    for (int w = tg; w < WORDS; w += G) {
      unsigned msk = 0u;
      const int s0 = w * 32;
#pragma unroll 8
      for (int b = 0; b < 32; ++b)
        if (s0 + b < TOT && keys[s0 + b] != INF) msk |= (1u << b);
      wmask[w] = msk;
      wpre[w] = __popc(msk);
    }
  }
  gsync();
  if (work && !overflow && tg < 32) {
    int carry = 0;
    for (int w0 = 0; w0 < WORDS; w0 += 32) {
      const int w = w0 + tg;
      const int v = w < WORDS ? wpre[w] : 0;
      int inc = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (tg >= o) inc += t;
      }
      if (w < WORDS) wpre[w] = carry + inc - v;
      carry += __shfl_sync(0xffffffffu, inc, 31);
    }
  }
  gsync();
  if (work && !overflow) {
    for (int s = tg; s < TOT; s += G) {
      const int key = keys[s];
      if (key != INF) ciC[cbase + wpre[s >> 5] + __popc(wmask[s >> 5] & ((1u << (s & 31)) - 1u))] = key;
    }
  }
  // ---- walk 2: values, accumulated by output position (a0 == a1 for idle / overflowed groups)
  const int b0 = overflow ? 0 : a0, b1 = overflow ? 0 : a1;
  walk_products<G, true, S>(
      tg, lb, b0, b1, ciA, vA, rpB, ciB, vB, sm_walk[g],
      [&](int c, S v) {
        int h = slot_of(c);
        while (keys[h] != c) ++h;  // present by construction
        smem_add(&vals[wpre[h >> 5] + __popc(wmask[h >> 5] & ((1u << (h & 31)) - 1u))], v);
      },
      []() { return false; });
  gsync();
  if (work && !overflow)
    for (int q = tg; q < nz; q += G) vC[cbase + q] = vals[q];
}

// ---------------------------------------------------------------------------
// NUMERIC, variant 2 ("staged"): same sorted-by-construction accumulator as num_hash_kernel, but
//  * ONE walk over the products: while the keys are inserted, every product (column, b*a) is parked
//    in shared memory at its ordinal within the row (ordinals come from a group-wide exclusive scan
//    of the B row lengths), so the value pass reads shared memory instead of gathering the B rows
//    from HBM a second time (rows with more than PCAP products fall back to a second walk);
//  * occupancy words by warp ballot (one instruction per 32 slots instead of a 32-step loop),
//    16-byte table initialisation;
//  * rows whose product count equals nnz(C_i) have no duplicate column: their values are placed
//    with plain stores (no shared-memory atomics, no zero fill).
// Selected with B200SP_SPGEMM_NUMERIC=2|3|4 (3 = half-size key tables, load factor <= 0.5; 4 = no parking:
// only the cheaper table passes, same footprint as variant 1).
// ---------------------------------------------------------------------------
template <int G, typename S>
struct Walk2Smem {
  int bs[G];    // start of the B row of staged entry t
  int len[G];   // its length
  int off[G];   // ordinal (within the C row's product list) of its first product
  S va[G];      // A value of staged entry t
  int wsum[G > 32 ? G / 32 : 1];
};

// exclusive scan of one int per thread over a group of G threads (G = 32: one warp, else the CTA)
template <int G>
__device__ __forceinline__ int group_excl_scan(int v, int tg, int* wsum, int& total) {
  const int lane = tg & 31;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (G == 32) {
    total = __shfl_sync(0xffffffffu, inc, 31);
    return inc - v;
  }
  const int w = tg >> 5;
  if (lane == 31) wsum[w] = inc;
  __syncthreads();
  int woff = 0, tot = 0;
#pragma unroll
  for (int i = 0; i < (G > 32 ? G / 32 : 1); ++i) {
    const int s = wsum[i];
    if (i < w) woff += s;
    tot += s;
  }
  total = tot;
  return woff + inc - v;
}

// f(column, b_val*a_val, ordinal) once per product of row i; with_vals == false skips the value loads
// jac_row >= 0 (spgemm_jacobi): the row gets one extra leading entry (column jac_row, value 1) -- row jac_row of B
// itself -- and every value of A is multiplied by jac_mult = -omega * dinv[row]
// (sparse/impl/KokkosSparse_spgemm_jacobi_seq_impl.hpp:78-108).
template <int G, typename S, typename F>
__device__ __forceinline__ void walk_products2(int tg, int lb, int a0, int a1, bool with_vals, int jac_row, S jac_mult,
                                               const int* __restrict__ ciA, const S* __restrict__ vA,
                                               const int* __restrict__ rpB, const int* __restrict__ ciB,
                                               const S* __restrict__ vB, Walk2Smem<G, S>& w, F&& f) {
  constexpr int UT = 4;
  auto gsync = [&]() {
    if (G <= 32) __syncwarp(); else __syncthreads();
  };
  const int nsub = G / lb;
  const int q = tg / lb, sl = tg % lb;
  int pbase = 0;
  const int lo = jac_row >= 0 ? a0 - 1 : a0;  // index a0 - 1 stands for the extra entry
  for (int ab = lo; ab < a1; ab += G) {
    const int nA = min(G, a1 - ab);
    int b0 = 0, ln = 0;
    S va = S(0);
    if (tg < nA) {
      const int j = ab + tg;
      int ca;
      if (jac_row >= 0 && j == a0 - 1) {
        ca = jac_row;
        if (with_vals) va = S(1);
      } else {
        ca = ciA[j];
        if (with_vals) va = jac_row >= 0 ? vA[j] * jac_mult : vA[j];
      }
      b0 = rpB[ca];
      ln = rpB[ca + 1] - b0;
    }
    int total;
    const int excl = group_excl_scan<G>(ln, tg, w.wsum, total);
    w.bs[tg] = b0;
    w.len[tg] = ln;
    w.off[tg] = pbase + excl;
    w.va[tg] = va;
    pbase += total;
    gsync();
    for (int t0 = q; t0 < nA; t0 += nsub * UT) {
      int c[UT], id[UT];
      S v[UT];
#pragma unroll
      for (int u = 0; u < UT; ++u) {
        const int t = t0 + u * nsub;
        c[u] = -1;
        id[u] = 0;
        v[u] = S(0);
        if (t < nA && sl < w.len[t]) {
          const int jb = w.bs[t] + sl;
          c[u] = ld_stream(ciB + jb);
          id[u] = w.off[t] + sl;
          if (with_vals) v[u] = ld_stream(vB + jb) * w.va[t];  // b_val * val (impl_seq.hpp:163)
        }
      }
#pragma unroll
      for (int u = 0; u < UT; ++u)
        if (c[u] >= 0) f(c[u], v[u], id[u]);
      // B rows longer than the sub-warp
#pragma unroll 1
      for (int u = 0; u < UT; ++u) {
        const int t = t0 + u * nsub;
        if (t < nA)
          for (int off = sl + lb; off < w.len[t]; off += lb) {
            const int jb = w.bs[t] + off;
            f(ld_stream(ciB + jb), with_vals ? ld_stream(vB + jb) * w.va[t] : S(0), w.off[t] + off);
          }
      }
    }
    gsync();  // staging is rewritten by the next batch
  }
}

template <typename S, int G, int KSLOTS, int PAD, int VCAP, int PCAP>
struct Num2Layout {
  static constexpr int TOT = KSLOTS + PAD;  // multiple of 32
  static constexpr int WORDS = TOT / 32;
  // per row-group: vals[VCAP] | pval[PCAP] | keys[TOT] | pcol[PCAP] | wpre[WORDS] | wmask[WORDS]
  static constexpr size_t OFF_PVAL = sizeof(S) * VCAP;
  static constexpr size_t OFF_KEYS = OFF_PVAL + sizeof(S) * PCAP;
  static constexpr size_t OFF_PCOL = OFF_KEYS + sizeof(int) * TOT;
  static constexpr size_t OFF_WPRE = OFF_PCOL + sizeof(int) * PCAP;
  static constexpr size_t OFF_WMASK = OFF_WPRE + sizeof(int) * WORDS;
  static constexpr size_t PER = OFF_WMASK + sizeof(int) * WORDS;
  static constexpr size_t PER_AL = (PER + 15) & ~(size_t)15;
  static_assert(TOT % 32 == 0 && VCAP % 4 == 0 && PCAP % 4 == 0, "table sizes keep 16-byte alignment");
};

template <typename S, int G, int KSLOTS, int PAD, int VCAP, int PCAP, bool EMIT2 = false, bool JAC = false, bool FASTW = false>
__global__ void __launch_bounds__(G <= 32 ? 256 : G)
    num2_kernel(int nrows_bin, const int* __restrict__ rows, int lb, const int* __restrict__ rpA,
                const int* __restrict__ ciA, const S* __restrict__ vA, const int* __restrict__ rpB,
                const int* __restrict__ ciB, const S* __restrict__ vB, const int* __restrict__ rpC,
                int* __restrict__ ciC, S* __restrict__ vC, const int* __restrict__ cmin_arr,
                const int* __restrict__ cmax_arr, const int* __restrict__ flops_arr, int* __restrict__ fb_rows,
                int* __restrict__ fb_count, S omega, const S* __restrict__ dinv) {
  using L = Num2Layout<S, G, KSLOTS, PAD, VCAP, PCAP>;
  constexpr int THREADS = (G <= 32 ? 256 : G);
  constexpr int RPC = THREADS / G;
  constexpr int NWG = G / 32;  // warps per row group
  constexpr int TOT = L::TOT;
  constexpr int WORDS = L::WORDS;
  constexpr int INF = INT_MAX;
  extern __shared__ __align__(16) unsigned char smraw[];
  __shared__ int sm_flag[RPC];
  __shared__ Walk2Smem<G, S> sm_walk[RPC];
  const int g = threadIdx.x / G, tg = threadIdx.x % G;
  const int lane = tg & 31, wg = tg >> 5;
  unsigned char* base = smraw + (size_t)g * L::PER_AL;
  S* vals = reinterpret_cast<S*>(base);
  S* pval = reinterpret_cast<S*>(base + L::OFF_PVAL);
  int* keys = reinterpret_cast<int*>(base + L::OFF_KEYS);
  int* pcol = reinterpret_cast<int*>(base + L::OFF_PCOL);
  int* wpre = reinterpret_cast<int*>(base + L::OFF_WPRE);
  unsigned* wmask = reinterpret_cast<unsigned*>(base + L::OFF_WMASK);
  const int ridx = blockIdx.x * RPC + g;
  const bool active = ridx < nrows_bin;
  auto gsync = [&]() {
    if (G <= 32) __syncwarp(); else __syncthreads();
  };
  int i = 0, cbase = 0, nz = 0, np = 0;
  if (active) {
    i = rows[ridx];
    cbase = rpC[i];
    nz = rpC[i + 1] - cbase;
    np = flops_arr[i];  // exact number of products of the row (clamped at INT_MAX)
  }
  const bool work = active && nz > 0;
  // spgemm_jacobi: row i of B joins the products (its columns are expected inside the symbolic pattern, i.e. A
  // has its diagonal, like the reference's kernels assume): duplicates are the rule, nothing is parked
  const bool dupfree = !JAC && work && np == nz;  // every product has its own column
  const bool staged = !JAC && PCAP > 0 && work && np <= PCAP;
  const int jac_row = (JAC && work) ? i : -1;
  const S jac_mult = (JAC && work) ? -omega * dinv[i] : S(1);
  {
    int4* k4 = reinterpret_cast<int4*>(keys);
    for (int s = tg; s < TOT / 4; s += G) k4[s] = make_int4(INF, INF, INF, INF);
    if (work && !dupfree)
      for (int s = tg; s < nz; s += G) vals[s] = S(0);
    if (tg == 0) sm_flag[g] = 0;
  }
  gsync();
  const int cmin = work ? cmin_arr[i] : 0;
  const int cmax = work ? cmax_arr[i] : 0;
  const long long span = work ? ((long long)cmax - cmin + 1) : 1;
  const bool dense = span <= KSLOTS;
  const unsigned long long mult = dense ? 0ull : (((unsigned long long)KSLOTS << 32) / (unsigned long long)span);
  const int a0 = work ? rpA[i] : 0, a1 = work ? rpA[i + 1] : 0;
  auto slot_of = [&](int c) -> int {
    return dense ? (c - cmin) : (int)(((unsigned long long)(unsigned)(c - cmin) * mult) >> 32);
  };
  // position of the (present) column c in the sorted row
  auto rank_of = [&](int c) -> int {
    int h = slot_of(c);
    while (keys[h] != c) ++h;
    return wpre[h >> 5] + __popc(wmask[h >> 5] & ((1u << (h & 31)) - 1u));
  };
  // ---- the walk: ordered insertion of the keys (+ products parked in shared memory)
  walk_products2<G, S>(tg, lb, a0, a1, staged, jac_row, jac_mult, ciA, vA, rpB, ciB, vB, sm_walk[g], [&](int c, S v, int id) {
    if (PCAP > 0 && staged) {
      pcol[id] = c;
      pval[id] = v;
    }
    if (JAC && (c < cmin || c > cmax)) {
      // a column of row i of B outside the span of A*B's row (A without its diagonal): it has no slot in the table; the
      // row goes to the fallback kernel, which drops such columns
      sm_flag[g] = 1;
      return;
    }
    int h = slot_of(c);
    while (true) {
      const int old = atomicMin(&keys[h], c);
      if (old == c || old == INF) return;  // already there / took an empty slot
      if (old > c) c = old;                // displaced a larger key: carry it on
      if (++h >= TOT) {
        sm_flag[g] = 1;  // ran off the pad: row goes to the fallback kernel
        return;
      }
    }
  });
  gsync();
  const bool overflow = sm_flag[g] != 0;
  if (active && overflow && tg == 0) fb_rows[atomicAdd(fb_count, 1)] = i;
  bool emit = work && !overflow;  // uniform within the group
  // ---- occupancy words and their exclusive prefix
  if (FASTW) {
    // variant 6: 128 slots per step -- every lane reads 4 keys with one 16-byte load, its 4 occupancy bits are
    // OR-reduced over the 8 lanes that make up a word; then every thread scans a contiguous run of words and the
    // runs are combined with one group-wide scan (all warps busy, instead of warp 0 walking every word)
    if (emit) {
      for (int chunk = wg; chunk * 128 < TOT; chunk += NWG) {
        const int s0 = chunk * 128 + lane * 4;
        unsigned nib = 0u;
        if (s0 < TOT) {  // TOT % 4 == 0: the four keys are all in range or all out
          const int4 kk = *reinterpret_cast<const int4*>(&keys[s0]);
          nib = (kk.x != INF ? 1u : 0u) | (kk.y != INF ? 2u : 0u) | (kk.z != INF ? 4u : 0u) | (kk.w != INF ? 8u : 0u);
        }
        unsigned word = nib << (4 * (lane & 7));
        word |= __shfl_xor_sync(0xffffffffu, word, 1);
        word |= __shfl_xor_sync(0xffffffffu, word, 2);
        word |= __shfl_xor_sync(0xffffffffu, word, 4);
        const int w = chunk * 4 + (lane >> 3);
        if ((lane & 7) == 0 && w < WORDS) {
          wmask[w] = word;
          wpre[w] = __popc(word);
        }
      }
    }
    gsync();
    constexpr int WPT = (WORDS + G - 1) / G;  // words per thread
    int local[WPT];
    int tsum = 0;
#pragma unroll
    for (int q = 0; q < WPT; ++q) {
      const int w = tg * WPT + q;
      const int v = (emit && w < WORDS) ? wpre[w] : 0;
      local[q] = tsum;
      tsum += v;
    }
    int total_words;
    const int excl = group_excl_scan<G>(tsum, tg, sm_walk[g].wsum, total_words);  // barrier inside for G > 32
    (void)total_words;
    gsync();  // every wpre[] read above precedes the writes below
#pragma unroll
    for (int q = 0; q < WPT; ++q) {
      const int w = tg * WPT + q;
      if (emit && w < WORDS) wpre[w] = excl + local[q];
    }
    gsync();
  } else {
    if (emit) {
      for (int w = wg; w < WORDS; w += NWG) {
        const unsigned msk = __ballot_sync(0xffffffffu, keys[w * 32 + lane] != INF);
        if (lane == 0) {
          wmask[w] = msk;
          wpre[w] = __popc(msk);
        }
      }
    }
    gsync();
    if (emit && tg < 32) {
      int carry = 0;
      for (int w0 = 0; w0 < WORDS; w0 += 32) {
        const int w = w0 + tg;
        const int v = w < WORDS ? wpre[w] : 0;
        int inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int t = __shfl_up_sync(0xffffffffu, inc, o);
          if (tg >= o) inc += t;
        }
        if (w < WORDS) wpre[w] = carry + inc - v;
        carry += __shfl_sync(0xffffffffu, inc, 31);
      }
    }
    gsync();
  }
  if (JAC && emit) {
    // row i of B brought columns the symbolic pattern does not hold (A without its diagonal): hand the row to the
    // fallback kernel, which drops the surplus instead of writing past the row
    const int total = wpre[WORDS - 1] + __popc(wmask[WORDS - 1]);
    if (total != nz) {
      emit = false;
      if (tg == 0) fb_rows[atomicAdd(fb_count, 1)] = i;
    }
  }
  // ---- column indices leave in sorted order (EMIT2: written from the value pass instead, one scattered 4-byte
  //      store per product -- no scan over the whole key table)
  if (emit && !EMIT2) {
    const unsigned lt = (1u << lane) - 1u;
    for (int w = wg; w < WORDS; w += NWG) {
      const int key = keys[w * 32 + lane];
      if (key != INF) ciC[cbase + wpre[w] + __popc(wmask[w] & lt)] = key;
    }
  }
  // ---- values by output position
  if (PCAP > 0 && staged) {
    if (emit) {
      for (int id = tg; id < np; id += G) {
        const int c = pcol[id];
        const int pos = rank_of(c);
        if (EMIT2) ciC[cbase + pos] = c;
        if (dupfree) vals[pos] = pval[id]; else smem_add(&vals[pos], pval[id]);
      }
    }
  } else {
    // too many products to park: second walk (idle / overflowed groups walk an empty row)
    const int b0 = emit ? a0 : 0, b1 = emit ? a1 : 0;
    walk_products2<G, S>(tg, lb, b0, b1, true, emit ? jac_row : -1, jac_mult, ciA, vA, rpB, ciB, vB, sm_walk[g], [&](int c, S v, int) {
      const int pos = rank_of(c);
      if (EMIT2) ciC[cbase + pos] = c;
      if (dupfree) vals[pos] = v; else smem_add(&vals[pos], v);
    });
  }
  gsync();
  if (emit)
    for (int q = tg; q < nz; q += G) vC[cbase + q] = vals[q];
}

// spgemm_jacobi rows that do not fit shared memory, overflowed, or whose row i of B brought columns outside the symbolic
// pattern: num_fallback_kernel with A's values scaled by -omega*dinv[i], then row i of B added where its column is in the
// pattern.  The products go in first: their distinct columns ARE the symbolic pattern, so at most nz keys enter a table of
// at least 2*nz slots and every probe ends.  Row i of B only looks its columns up and drops the ones it does not find: for
// an A without its diagonal the row is C restricted to the pattern of A*B.
template <typename S>
__global__ void __launch_bounds__(256)
    num_fallback_jacobi_kernel(const int* __restrict__ fb_rows, const int* __restrict__ fb_count, int log2slots,
                               int* __restrict__ gkeys, S* __restrict__ gvals, const int* __restrict__ rpA,
                               const int* __restrict__ ciA, const S* __restrict__ vA, const int* __restrict__ rpB,
                               const int* __restrict__ ciB, const S* __restrict__ vB, const int* __restrict__ rpC,
                               int* __restrict__ ciC, S* __restrict__ vC, S omega, const S* __restrict__ dinv) {
  const size_t slots = (size_t)1 << log2slots;
  int* keys = gkeys + (size_t)blockIdx.x * slots;
  S* vals = gvals + (size_t)blockIdx.x * slots;
  __shared__ int cursor;
  const int nfb = *fb_count;
  for (int q = blockIdx.x; q < nfb; q += gridDim.x) {
    const int i = fb_rows[q];
    const int cbase = rpC[i];
    const int nz = rpC[i + 1] - cbase;
    int lg = 1;
    while (((size_t)1 << lg) < (size_t)2 * (size_t)nz) ++lg;
    const size_t tsz = (size_t)1 << lg;
    for (size_t s = threadIdx.x; s < tsz; s += 256) {
      keys[s] = EMPTY;
      vals[s] = S(0);
    }
    if (threadIdx.x == 0) cursor = 0;
    __syncthreads();
    const S mult = -omega * dinv[i];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int a0 = rpA[i], a1 = rpA[i + 1];
    for (int ja = a0 + warp; ja < a1; ja += 8) {
      const int ca = ciA[ja];
      const S va = vA[ja] * mult;
      for (int jb = rpB[ca] + lane; jb < rpB[ca + 1]; jb += 32) {
        const int c = ciB[jb];
        const S v = vB[jb] * va;
        size_t h = hash_mul(c, lg);
        while (true) {
          const int kcur = ((volatile int*)keys)[h];
          if (kcur == c) break;
          if (kcur == EMPTY) {
            const int old = atomicCAS(&keys[h], EMPTY, c);
            if (old == EMPTY || old == c) break;
          }
          h = (h + 1) & (tsz - 1);
        }
        atomicAdd(&vals[h], v);
      }
    }
    __syncthreads();
    // row i of B, weight 1: lookups only (the table holds at most nz keys, so an absent column meets an empty slot)
    for (int jb = rpB[i] + threadIdx.x; jb < rpB[i + 1]; jb += 256) {
      const int c = ciB[jb];
      size_t h = hash_mul(c, lg);
      int kcur;
      while ((kcur = keys[h]) != c && kcur != EMPTY) h = (h + 1) & (tsz - 1);
      if (kcur == c) atomicAdd(&vals[h], vB[jb]);
    }
    __syncthreads();
    for (size_t s = threadIdx.x; s < tsz; s += 256) {
      const int key = keys[s];
      if (key != EMPTY) {
        const int p = atomicAdd(&cursor, 1);
        if (p < nz) {  // a structure other than the symbolic phase's: drop, do not write past the row
          ciC[cbase + p] = key;
          vC[cbase + p] = vals[s];
        }
      }
    }
    __syncthreads();
    int P = 1;
    while (P < nz) P <<= 1;
    for (int size = 2; size <= P; size <<= 1) {
      for (int stride = size >> 1, first = 1; stride > 0; stride >>= 1, first = 0) {
        for (int idx = threadIdx.x; idx < P; idx += 256) {
          const int l = first ? (idx ^ (size - 1)) : (idx ^ stride);
          if (l > idx && l < nz) {
            const int ka = ciC[cbase + idx], kb = ciC[cbase + l];
            if (ka > kb) {
              ciC[cbase + idx] = kb;
              ciC[cbase + l] = ka;
              const S ta = vC[cbase + idx];
              vC[cbase + idx] = vC[cbase + l];
              vC[cbase + l] = ta;
            }
          }
        }
        __syncthreads();
      }
    }
    __syncthreads();
  }
}

// fallback: global-memory hash (wrap-around, multiplicative) + in-place bitonic sort of the C row
template <typename S>
__global__ void __launch_bounds__(256)
    num_fallback_kernel(const int* __restrict__ fb_rows, const int* __restrict__ fb_count, int log2slots,
                        int* __restrict__ gkeys, S* __restrict__ gvals, const int* __restrict__ rpA,
                        const int* __restrict__ ciA, const S* __restrict__ vA, const int* __restrict__ rpB,
                        const int* __restrict__ ciB, const S* __restrict__ vB, const int* __restrict__ rpC,
                        int* __restrict__ ciC, S* __restrict__ vC) {
  const size_t slots = (size_t)1 << log2slots;
  int* keys = gkeys + (size_t)blockIdx.x * slots;
  S* vals = gvals + (size_t)blockIdx.x * slots;
  __shared__ int cursor;
  const int nfb = *fb_count;
  for (int q = blockIdx.x; q < nfb; q += gridDim.x) {
    const int i = fb_rows[q];
    const int cbase = rpC[i];
    const int nz = rpC[i + 1] - cbase;
    // table sized for this row: smallest power of two >= 2*nz (<= slots)
    int lg = 1;
    while (((size_t)1 << lg) < (size_t)2 * (size_t)nz) ++lg;
    const size_t tsz = (size_t)1 << lg;
    for (size_t s = threadIdx.x; s < tsz; s += 256) {
      keys[s] = EMPTY;
      vals[s] = S(0);
    }
    if (threadIdx.x == 0) cursor = 0;
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int ja = rpA[i] + warp; ja < rpA[i + 1]; ja += 8) {
      const int ca = ciA[ja];
      const S va = vA[ja];
      for (int jb = rpB[ca] + lane; jb < rpB[ca + 1]; jb += 32) {
        const int c = ciB[jb];
        const S v = vB[jb] * va;
        size_t h = hash_mul(c, lg);
        while (true) {
          const int kcur = ((volatile int*)keys)[h];
          if (kcur == c) break;
          if (kcur == EMPTY) {
            const int old = atomicCAS(&keys[h], EMPTY, c);
            if (old == EMPTY || old == c) break;
          }
          h = (h + 1) & (tsz - 1);
        }
        atomicAdd(&vals[h], v);
      }
    }
    __syncthreads();
    for (size_t s = threadIdx.x; s < tsz; s += 256) {
      const int key = keys[s];
      if (key != EMPTY) {
        const int p = atomicAdd(&cursor, 1);
        ciC[cbase + p] = key;
        vC[cbase + p] = vals[s];
      }
    }
    __syncthreads();
    // bitonic network with all comparators ascending (virtual +inf padding never moves)
    int P = 1;
    while (P < nz) P <<= 1;
    for (int size = 2; size <= P; size <<= 1) {
      for (int stride = size >> 1, first = 1; stride > 0; stride >>= 1, first = 0) {
        for (int idx = threadIdx.x; idx < P; idx += 256) {
          const int l = first ? (idx ^ (size - 1)) : (idx ^ stride);
          if (l > idx && l < nz) {
            const int ka = ciC[cbase + idx], kb = ciC[cbase + l];
            if (ka > kb) {
              ciC[cbase + idx] = kb;
              ciC[cbase + l] = ka;
              const S ta = vC[cbase + idx];
              vC[cbase + idx] = vC[cbase + l];
              vC[cbase + l] = ta;
            }
          }
        }
        __syncthreads();
      }
    }
    __syncthreads();
  }
}

}  // namespace b200sp

using namespace b200sp;

// ---------------------------------------------------------------------------
// plan + host drivers
// ---------------------------------------------------------------------------
// symbolic bins by flop bound f (table slots >= 2f); last bin -> global bitmap
static const int kSymThr[] = {128, 512, 2048, 8192, 16384};
static constexpr int kSymBins = 6;
// numeric bins by nnz(C_i); last bin -> global fallback
static const int kNumThr[] = {64, 256, 1024, 4096, 8192};
static constexpr int kNumBins = 6;
static constexpr int kFbCtas = 16;
// ESC kernels (spgemm_esc.cuh): bins by max(products, 2 nnz(A_i)); rows above the last threshold -> hash kernels
static const int kEscThr[] = {256, 1024, 4096, 8192};
static constexpr int kEscBins = 4;
static constexpr int kEscCap = 8192;
// b200sp_spgemm_plan_paths: ESC bins, symbolic hash bin, bitmap, numeric hash bins, static and overflowed fallback rows
static constexpr int kSpgemmPaths = kEscBins + 2 + kNumBins + 1;

struct b200sp_spgemm_plan {
  bool symbolic_done = false;
  int m = 0, n = 0, k = 0;
  const int *rpA = nullptr, *ciA = nullptr, *rpB = nullptr, *ciB = nullptr;
  int64_t c_nnz = 0;
  int c_max = 0;
  int lb = 8;  // lanes walking one B row
  // device state kept for numeric
  b200sp::DevArray<int> cmin, cmax;
  b200sp::DevArray<int> flops;  // products per row of A*B (numeric variant 2 parks them in shared memory)
  int numeric_variant = 7;  // 7: ESC kernels (spgemm_esc.cuh) + hash kernels for long rows; 1: two-walk num_hash_kernel, 2..6: num2_kernel flavours (B200SP_SPGEMM_NUMERIC)
  b200sp::DevArray<int> num_rows;  // rows grouped by numeric bin (hash kernels): the rows beyond the ESC kernels' capacity
  int num_off[kNumBins + 1] = {0};
  b200sp::DevArray<int> all_rows;  // every row grouped by nnz(C_i): built on demand for the hash variants and spgemm_jacobi
  int all_off[kNumBins + 1] = {0};
  bool all_built = false;
  const int* cur_rows = nullptr;  // the grouping the hash-kernel launchers read (num_rows or all_rows)
  const int* cur_off = nullptr;
  const int* last_off = nullptr;  // the grouping of the last numeric / jacobi call (num_off or all_off), for plan_paths
  b200sp::DevArray<int> esc_key;   // per row: max(products, 2 nnz(A_i))
  b200sp::DevArray<int> esc_rows;  // rows grouped by ESC bin
  int esc_off[kEscBins + 3] = {0};
  b200sp::DevArray<int> fb_rows, fb_count;
  int fb_static = 0;
  int fb_log2 = 1;
  b200sp::DevArray<int> fb_keys;
  b200sp::DevArray<char> fb_vals;
  b200sp::BspState* bsp = nullptr;  // block-row grouping of the block numeric phase (bspgemm.cu), built on first use
  b200sp::Spgemm64State* s64 = nullptr;  // a product with 64-bit offsets (spgemm64.cu): the 32-bit entries refuse the plan
};

namespace b200sp {

static void spgemm_release(b200sp_spgemm_plan* p, cudaStream_t st) {
  for (DevArray<int>* q : {&p->cmin, &p->cmax, &p->flops, &p->num_rows, &p->fb_rows, &p->fb_count, &p->fb_keys, &p->all_rows,
                           &p->esc_key, &p->esc_rows})
    q->release(st);
  p->fb_vals.release(st);
  p->all_built = false;
  p->cur_rows = nullptr;
  p->cur_off = nullptr;
  p->last_off = nullptr;
  bsp_state_free(p->bsp, st);
  p->bsp = nullptr;
  p->symbolic_done = false;
}

SpgemmPlanView spgemm_plan_view(b200sp_spgemm_plan* p) {
  return SpgemmPlanView{p->symbolic_done, p->m, p->n, p->k, p->c_nnz, p->c_max, p->flops, &p->bsp, &p->s64};
}

static int bin_rows(cudaStream_t st, int m, const int* key, const BinSpec& spec, int* d_counts /*MAXBINS*/,
                    int* rows_out, int* h_off /*nb+1*/) {
  B200SP_CUDA_TRY(cudaMemsetAsync(d_counts, 0, sizeof(int) * MAXBINS, st));
  const int blocks = std::max(1, std::min((m + 255) / 256, sm_count() * 8));
  bin_count_kernel<<<blocks, 256, 0, st>>>(m, key, spec, d_counts);
  B200SP_LAUNCH_CHECK();
  int h_counts[MAXBINS];
  B200SP_CUDA_TRY(cudaMemcpyAsync(h_counts, d_counts, sizeof(int) * MAXBINS, cudaMemcpyDeviceToHost, st));
  B200SP_CUDA_TRY(cudaStreamSynchronize(st));
  h_off[0] = 0;
  for (int b = 0; b < spec.nb; ++b) h_off[b + 1] = h_off[b] + h_counts[b];
  B200SP_CUDA_TRY(cudaMemcpyAsync(d_counts, h_off, sizeof(int) * spec.nb, cudaMemcpyHostToDevice, st));
  bin_scatter_kernel<<<blocks, 256, 0, st>>>(m, key, spec, d_counts, rows_out);
  B200SP_LAUNCH_CHECK();
  // h_off is pageable host memory: make sure the H2D copy consumed it before it can change
  B200SP_CUDA_TRY(cudaStreamSynchronize(st));
  return B200SP_OK;
}

template <int G, int LOG2SLOTS, bool V2 = false>
static int launch_sym(cudaStream_t st, int nrows, const int* rows, int lb, const int* rpA, const int* ciA,
                      const int* rpB, const int* ciB, int* row_nnz) {
  if (nrows <= 0) return B200SP_OK;
  constexpr int THREADS = (G <= 32 ? 256 : G);
  constexpr int RPC = THREADS / G;
  const size_t smem = sizeof(int) * (size_t)RPC * ((size_t)1 << LOG2SLOTS);
  auto kern = sym_hash_kernel<G, LOG2SLOTS, V2>;
  // always: the 48 KB default limit counts the kernel's STATIC shared memory too (walker staging, flags)
  B200SP_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<(nrows + RPC - 1) / RPC, THREADS, smem, st>>>(nrows, rows, std::min(lb, 32), rpA, ciA, rpB, ciB, row_nnz);
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

template <typename S, int G, int KSLOTS, int PAD, int VCAP>
static int launch_num(cudaStream_t st, b200sp_spgemm_plan* p, int bin, const int* rpA, const int* ciA, const S* vA,
                      const int* rpB, const int* ciB, const S* vB, const int* rpC, int* ciC, S* vC) {
  const int nrows = p->cur_off[bin + 1] - p->cur_off[bin];
  if (nrows <= 0) return B200SP_OK;
  using L = NumLayout<S, G, KSLOTS, PAD, VCAP>;
  constexpr int THREADS = (G <= 32 ? 256 : G);
  constexpr int RPC = THREADS / G;
  const size_t smem = L::PER_AL * RPC;
  auto kern = num_hash_kernel<S, G, KSLOTS, PAD, VCAP>;
  // always: the 48 KB default limit counts the kernel's STATIC shared memory too (walker staging, flags)
  B200SP_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<(nrows + RPC - 1) / RPC, THREADS, smem, st>>>(nrows, p->cur_rows + p->cur_off[bin], std::min(p->lb, 32), rpA, ciA, vA,
                                                      rpB, ciB, vB, rpC, ciC, vC, p->cmin, p->cmax, p->fb_rows, p->fb_count);
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

template <typename S, int G, int KSLOTS, int PAD, int VCAP, int PCAP, bool EMIT2 = false, bool JAC = false, bool FASTW = false>
static int launch_num2(cudaStream_t st, b200sp_spgemm_plan* p, int bin, const int* rpA, const int* ciA, const S* vA,
                       const int* rpB, const int* ciB, const S* vB, const int* rpC, int* ciC, S* vC, S omega = S(0),
                       const S* dinv = nullptr) {
  const int nrows = p->cur_off[bin + 1] - p->cur_off[bin];
  if (nrows <= 0) return B200SP_OK;
  using L = Num2Layout<S, G, KSLOTS, PAD, VCAP, PCAP>;
  constexpr int THREADS = (G <= 32 ? 256 : G);
  constexpr int RPC = THREADS / G;
  const size_t smem = L::PER_AL * RPC;
  auto kern = num2_kernel<S, G, KSLOTS, PAD, VCAP, PCAP, EMIT2, JAC, FASTW>;
  // always: the 48 KB default limit counts the kernel's STATIC shared memory too (walker staging, flags)
  B200SP_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<(nrows + RPC - 1) / RPC, THREADS, smem, st>>>(nrows, p->cur_rows + p->cur_off[bin], std::min(p->lb, 32), rpA, ciA, vA,
                                                      rpB, ciB, vB, rpC, ciC, vC, p->cmin, p->cmax, p->flops, p->fb_rows,
                                                      p->fb_count, omega, dinv);
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

// The ESC kernels are persistent: one wave of CTAs (SMs x resident CTAs per SM), each working through every grid-th row of
// its bin with the row pipeline of spgemm_esc.cuh.  B200SP_ESC_PERSIST=0 launches one CTA per row instead (the pipeline
// then degenerates to the plain dependent chain) -- an A/B switch for measurements.
static int esc_grid(int nrows, int occ) {
  static const bool persist = [] {
    const char* e = getenv("B200SP_ESC_PERSIST");
    return !(e && e[0] == '0');
  }();
  if (!persist) return nrows;
  return (int)std::min<int64_t>((int64_t)nrows, (int64_t)sm_count() * std::max(occ, 1));
}

template <int T, int I, int LOG2NB, int MINB>
static int launch_esc_sym(cudaStream_t st, int nrows, const int* rows, const int* rpA, const int* ciA, const int* rpB,
                          const int* ciB, const int* flops, const int* cmin, const int* cmax, int* row_nnz) {
  if (nrows <= 0) return B200SP_OK;
  using L = EscSymLayout<T, I, LOG2NB>;
  auto kern = esc_sym_kernel<T, I, LOG2NB, MINB>;
  static KernelSetup ks;  // per instantiation and device: shared-memory opt-in + occupancy, queried once
  int occ = 1;
  if (int rc = kernel_setup(ks, kern, T, L::BYTES, &occ)) return rc;
  const int grid = esc_grid(nrows, occ);
  kern<<<grid, T, L::BYTES, st>>>(nrows, rows, rpA, ciA, rpB, ciB, flops, cmin, cmax, row_nnz);
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

template <typename S, int T, int I, int LOG2NB, int MINB>
static int launch_esc_num(cudaStream_t st, b200sp_spgemm_plan* p, int bin, const int* rpA, const int* ciA, const S* vA,
                          const int* rpB, const int* ciB, const S* vB, const int* rpC, int* ciC, S* vC) {
  const int nrows = p->esc_off[bin + 1] - p->esc_off[bin];
  if (nrows <= 0) return B200SP_OK;
  using L = EscNumLayout<S, T, I, LOG2NB>;
  auto kern = esc_num_kernel<S, T, I, LOG2NB, MINB>;
  static KernelSetup ks;
  int occ = 1;
  if (int rc = kernel_setup(ks, kern, T, L::BYTES, &occ)) return rc;
  const int grid = esc_grid(nrows, occ);
  kern<<<grid, T, L::BYTES, st>>>(nrows, p->esc_rows + p->esc_off[bin], rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC, p->cmin,
                                   p->cmax, p->flops);
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

// B200SP_SPGEMM_TRACE=1: host wall clock between the phases of spgemm_symbolic (each mark synchronises the stream): a
// diagnostic for the synchronous phase, never on by default
struct SymTrace {
  bool on;
  cudaStream_t st;
  double t0;
  static double now() {
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6;
  }
  explicit SymTrace(cudaStream_t s) : on(getenv("B200SP_SPGEMM_TRACE") != nullptr), st(s), t0(0) {
    if (on) {
      cudaStreamSynchronize(st);
      t0 = now();
    }
  }
  void mark(const char* what) {
    if (!on) return;
    cudaStreamSynchronize(st);
    const double t = now();
    fprintf(stderr, "[spgemm_symbolic] %-28s %8.3f ms\n", what, t - t0);
    t0 = t;
  }
};

// every row grouped by nnz(C_i) (the hash variants B200SP_SPGEMM_NUMERIC=1..6 and spgemm_jacobi); built once, synchronises
static int ensure_all_bins(b200sp_spgemm_plan* p, cudaStream_t st, const int* rpC) {
  if (p->all_built) return B200SP_OK;
  DevTmp tmp(st);
  int *key, *d_counts;
  B200SP_CUDA_TRY(tmp.alloc(&key, p->m));
  B200SP_CUDA_TRY(tmp.alloc(&d_counts, MAXBINS));
  if (!p->all_rows) B200SP_CUDA_TRY(p->all_rows.alloc((size_t)p->m, st));
  const int blocks = std::max(1, std::min((p->m + 255) / 256, sm_count() * 8));
  rest_key_kernel<<<blocks, 256, 0, st>>>(p->m, nullptr, 0, rpC, 1, key);
  B200SP_LAUNCH_CHECK();
  BinSpec nspec;
  nspec.nb = kNumBins;
  for (int b = 0; b < kNumBins - 1; ++b) nspec.thr[b] = kNumThr[b];
  const int rc = bin_rows(st, p->m, key, nspec, d_counts, p->all_rows, p->all_off);
  if (rc) return rc;
  p->all_built = true;
  return B200SP_OK;
}

template <typename S>
static int numeric_impl(b200sp_spgemm_plan* p, cudaStream_t st, int m, int n, int k, const int* rpA, const int* ciA,
                        const S* vA, const int* rpB, const int* ciB, const S* vB, const int* rpC, int* ciC, S* vC) {
  B200SP_REQUIRE(p != nullptr, "spgemm_numeric: null plan");
  if (spgemm64_holds_product(p->s64)) {
    set_error("spgemm_numeric: the symbolic phase on this handle had 64-bit offsets; use the _i64 numeric");
    return B200SP_ERR_STATE;
  }
  if (!p->symbolic_done) {
    set_error("Call spgemm symbolic before spgemm numeric");
    return B200SP_ERR_STATE;
  }
  if (p->m != m || p->n != n || p->k != k) {
    set_error("spgemm_numeric: dimensions (%d,%d,%d) differ from symbolic (%d,%d,%d)", m, n, k, p->m, p->n, p->k);
    return B200SP_ERR_STATE;
  }
  p->last_off = nullptr;
  if (m == 0 || p->c_nnz == 0) return B200SP_OK;
  B200SP_REQUIRE(rpA && ciA && vA && rpB && ciB && vB && rpC && ciC && vC, "spgemm_numeric: null pointer argument");
  // fallback scratch for values (type-dependent; keys were sized in symbolic)
  const size_t need = sizeof(S) * (size_t)kFbCtas * ((size_t)1 << p->fb_log2);
  B200SP_CUDA_TRY(p->fb_vals.grow(need, st));
  // fallback list starts as the rows that are too long for shared memory
  B200SP_CUDA_TRY(cudaMemcpyAsync(p->fb_count, &p->fb_static, sizeof(int), cudaMemcpyHostToDevice, st));
  int rc;
  int variant = p->numeric_variant;
  if (const char* e = getenv("B200SP_SPGEMM_NUMERIC")) variant = atoi(e);
  if (variant >= 7 && p->esc_rows) {
    // default: register-resident expand / sort / compress kernels (spgemm_esc.cuh) for rows of <= 8192 products,
    // the two-walk hash kernels for the rest
    // <S, threads, products per thread, log2(buckets), CTAs per SM for the register budget>.  B200SP_ESC_CFG selects the
    // alternatives of the 1024-product bin for A/B runs
    int esc_cfg = 0;
    if (const char* e = getenv("B200SP_ESC_CFG")) esc_cfg = atoi(e);
    if ((rc = launch_esc_num<S, 32, 8, 9, 32>(st, p, 0, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC))) return rc;
    switch (esc_cfg) {  // bin 1; the default was the fastest on config 4 when it was tuned (B200-era, not re-tuned on the H100)
      case 1: rc = launch_esc_num<S, 256, 4, 11, 6>(st, p, 1, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC); break;
      case 2: rc = launch_esc_num<S, 128, 8, 10, 8>(st, p, 1, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC); break;
      case 4: rc = launch_esc_num<S, 256, 4, 10, 5>(st, p, 1, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC); break;
      case 5: rc = launch_esc_num<S, 512, 2, 10, 4>(st, p, 1, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC); break;
      case 7: rc = launch_esc_num<S, 256, 4, 10, 7>(st, p, 1, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC); break;
      case 8: rc = launch_esc_num<S, 128, 8, 11, 8>(st, p, 1, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC); break;
      default: rc = launch_esc_num<S, 256, 4, 10, 6>(st, p, 1, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC); break;
    }
    if (rc) return rc;
    if ((rc = launch_esc_num<S, 512, 8, 12, 2>(st, p, 2, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC))) return rc;
    if ((rc = launch_esc_num<S, 1024, 8, 13, 1>(st, p, 3, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC))) return rc;
    p->last_off = p->num_off;
    if (p->esc_off[kEscBins] < m) {
      p->cur_rows = p->num_rows;
      p->cur_off = p->num_off;
      if ((rc = launch_num<S, 32, 256, 32, 64>(st, p, 0, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC))) return rc;
      if ((rc = launch_num<S, 32, 1024, 64, 256>(st, p, 1, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC))) return rc;
      if ((rc = launch_num<S, 128, 4096, 128, 1024>(st, p, 2, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC))) return rc;
      if ((rc = launch_num<S, 256, 16384, 256, 4096>(st, p, 3, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC))) return rc;
      if ((rc = launch_num<S, 512, 32768, 512, 8192>(st, p, 4, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC))) return rc;
      num_fallback_kernel<S><<<kFbCtas, 256, 0, st>>>(p->fb_rows, p->fb_count, p->fb_log2, p->fb_keys, p->fb_vals.as<S>(), rpA,
                                                      ciA, vA, rpB, ciB, vB, rpC, ciC, vC);
      B200SP_LAUNCH_CHECK();
    }
    return B200SP_OK;
  }
  if (variant >= 7) variant = 1;
  if ((rc = ensure_all_bins(p, st, rpC))) return rc;
  p->cur_rows = p->all_rows;
  p->cur_off = p->all_off;
  p->last_off = p->all_off;
  if (variant == 6) {  // variant 5 + occupancy words from 16-byte key loads and a scan that keeps every warp busy
#define NUM6(B, G, KS, PAD, VCAP)                                                                                 \
  if ((rc = launch_num2<S, G, KS, PAD, VCAP, 0, true, false, true>(st, p, B, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC))) return rc;
    NUM6(0, 32, 256, 32, 64)
    NUM6(1, 32, 1024, 64, 256)
    NUM6(2, 128, 4096, 128, 1024)
    NUM6(3, 256, 16384, 256, 4096)
    NUM6(4, 512, 32768, 512, 8192)
#undef NUM6
    num_fallback_kernel<S><<<kFbCtas, 256, 0, st>>>(p->fb_rows, p->fb_count, p->fb_log2, p->fb_keys, p->fb_vals.as<S>(), rpA,
                                                    ciA, vA, rpB, ciB, vB, rpC, ciC, vC);
    B200SP_LAUNCH_CHECK();
    return B200SP_OK;
  }
  if (variant == 5) {  // variant 4 + column indices written from the value pass (no scan of the key table for them)
#define NUM5(B, G, KS, PAD, VCAP)                                                                                 \
  if ((rc = launch_num2<S, G, KS, PAD, VCAP, 0, true>(st, p, B, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC))) return rc;
    NUM5(0, 32, 256, 32, 64)
    NUM5(1, 32, 1024, 64, 256)
    NUM5(2, 128, 4096, 128, 1024)
    NUM5(3, 256, 16384, 256, 4096)
    NUM5(4, 512, 32768, 512, 8192)
#undef NUM5
    num_fallback_kernel<S><<<kFbCtas, 256, 0, st>>>(p->fb_rows, p->fb_count, p->fb_log2, p->fb_keys, p->fb_vals.as<S>(), rpA,
                                                    ciA, vA, rpB, ciB, vB, rpC, ciC, vC);
    B200SP_LAUNCH_CHECK();
    return B200SP_OK;
  }
  if (variant >= 2 && variant <= 4) {
    // <S, G, key slots, pad, max nnz(C_i) of the bin, parked products>
#define NUM2(B, G, KS, PAD, VCAP, PCAP)                                                                          \
  if ((rc = launch_num2<S, G, KS, PAD, VCAP, PCAP>(st, p, B, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC))) return rc;
    if (variant == 2) {  // key tables >= 4 x nnz (load <= 0.25)
      NUM2(0, 32, 256, 32, 64, 128)
      NUM2(1, 64, 1024, 64, 256, 512)
      NUM2(2, 128, 4096, 128, 1024, 1024)
      NUM2(3, 256, 16384, 256, 4096, 2048)
      NUM2(4, 512, 32768, 512, 8192, 0)
    } else if (variant == 3) {  // >= 2 x nnz (load <= 0.5): half the table to initialise and scan, longer probe chains
      NUM2(0, 32, 128, 32, 64, 128)
      NUM2(1, 64, 512, 64, 256, 512)
      NUM2(2, 128, 2048, 128, 1024, 1024)
      NUM2(3, 256, 8192, 256, 4096, 2048)
      NUM2(4, 512, 16384, 512, 8192, 0)
    } else {  // 4: variant 2's cheaper table passes (16-byte init, ballot words) WITHOUT parking the products:
              // two walks like variant 1 and the same shared-memory footprint (same resident CTAs per SM)
      NUM2(0, 32, 256, 32, 64, 0)
      NUM2(1, 32, 1024, 64, 256, 0)
      NUM2(2, 128, 4096, 128, 1024, 0)
      NUM2(3, 256, 16384, 256, 4096, 0)
      NUM2(4, 512, 32768, 512, 8192, 0)
    }
#undef NUM2
    num_fallback_kernel<S><<<kFbCtas, 256, 0, st>>>(p->fb_rows, p->fb_count, p->fb_log2, p->fb_keys, p->fb_vals.as<S>(), rpA,
                                                    ciA, vA, rpB, ciB, vB, rpC, ciC, vC);
    B200SP_LAUNCH_CHECK();
    return B200SP_OK;
  }
  // <S, G, key slots (>= 4 x bin's max nnz), pad, max nnz>
  if ((rc = launch_num<S, 32, 256, 32, 64>(st, p, 0, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC))) return rc;
  if ((rc = launch_num<S, 32, 1024, 64, 256>(st, p, 1, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC))) return rc;
  if ((rc = launch_num<S, 128, 4096, 128, 1024>(st, p, 2, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC))) return rc;
  if ((rc = launch_num<S, 256, 16384, 256, 4096>(st, p, 3, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC))) return rc;
  if ((rc = launch_num<S, 512, 32768, 512, 8192>(st, p, 4, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC))) return rc;
  num_fallback_kernel<S><<<kFbCtas, 256, 0, st>>>(p->fb_rows, p->fb_count, p->fb_log2, p->fb_keys, p->fb_vals.as<S>(), rpA,
                                                  ciA, vA, rpB, ciB, vB, rpC, ciC, vC);
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

template <typename S>
static int jacobi_impl(b200sp_spgemm_plan* p, cudaStream_t st, int m, int n, int k, const int* rpA, const int* ciA,
                       const S* vA, const int* rpB, const int* ciB, const S* vB, const int* rpC, int* ciC, S* vC, S omega,
                       const S* dinv) {
  B200SP_REQUIRE(p != nullptr, "spgemm_jacobi: null plan");
  if (spgemm64_holds_product(p->s64)) {
    set_error("spgemm_jacobi: not provided on 64-bit offsets (the symbolic phase on this handle had them)");
    return B200SP_ERR_STATE;
  }
  if (!p->symbolic_done) {
    set_error("KokkosSparse::spgemm_jacobi: must first call spgemm_symbolic with the same handle.");
    return B200SP_ERR_STATE;
  }
  if (p->m != m || p->n != n || p->k != k) {
    set_error("spgemm_jacobi: dimensions (%d,%d,%d) differ from symbolic (%d,%d,%d)", m, n, k, p->m, p->n, p->k);
    return B200SP_ERR_STATE;
  }
  B200SP_REQUIRE(m == n, "spgemm_jacobi: C = (I - omega D^-1 A) B needs a square A (m = %d, n = %d)", m, n);
  p->last_off = nullptr;
  if (m == 0 || p->c_nnz == 0) return B200SP_OK;
  B200SP_REQUIRE(rpA && ciA && vA && rpB && ciB && vB && rpC && ciC && vC && dinv, "spgemm_jacobi: null pointer argument");
  const size_t need = sizeof(S) * (size_t)kFbCtas * ((size_t)1 << p->fb_log2);
  B200SP_CUDA_TRY(p->fb_vals.grow(need, st));
  B200SP_CUDA_TRY(cudaMemcpyAsync(p->fb_count, &p->fb_static, sizeof(int), cudaMemcpyHostToDevice, st));
  int rc;
  if ((rc = ensure_all_bins(p, st, rpC))) return rc;
  p->cur_rows = p->all_rows;
  p->cur_off = p->all_off;
  p->last_off = p->all_off;
#define NUMJ(B, G, KS, PAD, VCAP)                                                                                       \
  if ((rc = launch_num2<S, G, KS, PAD, VCAP, 0, false, true>(st, p, B, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC, omega, \
                                                            dinv)))                                                     \
    return rc;
  NUMJ(0, 32, 256, 32, 64)
  NUMJ(1, 32, 1024, 64, 256)
  NUMJ(2, 128, 4096, 128, 1024)
  NUMJ(3, 256, 16384, 256, 4096)
  NUMJ(4, 512, 32768, 512, 8192)
#undef NUMJ
  num_fallback_jacobi_kernel<S><<<kFbCtas, 256, 0, st>>>(p->fb_rows, p->fb_count, p->fb_log2, p->fb_keys, p->fb_vals.as<S>(), rpA,
                                                         ciA, vA, rpB, ciB, vB, rpC, ciC, vC, omega, dinv);
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

}  // namespace b200sp

extern "C" {

int b200sp_spgemm_plan_create(b200sp_spgemm_plan** plan) {
  B200SP_REQUIRE(plan != nullptr, "spgemm_plan_create: null output pointer");
  b200sp::keep_async_pool_memory();
  b200sp_spgemm_plan* p = new (std::nothrow) b200sp_spgemm_plan();
  if (!p) {
    set_error("spgemm_plan_create: out of host memory");
    return B200SP_ERR_ALLOC;
  }
  *plan = p;
  return B200SP_OK;
}

int b200sp_spgemm_plan_destroy(b200sp_spgemm_plan* p, void* stream) {
  if (!p) return B200SP_OK;
  spgemm_release(p, (cudaStream_t)stream);
  spgemm64_state_free(p->s64, (cudaStream_t)stream);
  delete p;
  return B200SP_OK;
}

int b200sp_spgemm_symbolic_i32(b200sp_spgemm_plan* p, void* stream, int m, int n, int k, const int* rpA,
                               const int* ciA, const int* rpB, const int* ciB, int* rpC, int64_t* c_nnz,
                               int* c_max_row_nnz) {
  B200SP_REQUIRE(p != nullptr, "spgemm_symbolic: null plan");
  B200SP_REQUIRE(m >= 0 && n >= 0 && k >= 0, "spgemm_symbolic: negative dimension");
  B200SP_REQUIRE(rpC != nullptr, "spgemm_symbolic: row_ptr_C is null");
  cudaStream_t st = (cudaStream_t)stream;
  if (spgemm64_holds_product(p->s64)) {
    set_error("spgemm_symbolic: handle was already used for a product with 64-bit offsets; create a new handle");
    return B200SP_ERR_STATE;
  }
  if (p->symbolic_done) {
    // one handle, one product (reference debug build throws std::invalid_argument, spgemm_handle.hpp:706-746)
    if (p->m != m || p->n != n || p->k != k || p->rpA != rpA || p->ciA != ciA || p->rpB != rpB || p->ciB != ciB) {
      set_error("spgemm_symbolic: handle was already used for a different product; create a new handle");
      return B200SP_ERR_STATE;
    }
  }
  spgemm_release(p, st);
  p->m = m; p->n = n; p->k = k;
  p->rpA = rpA; p->ciA = ciA; p->rpB = rpB; p->ciB = ciB;
  p->c_nnz = 0; p->c_max = 0; p->fb_static = 0;
  for (int b = 0; b <= kNumBins; ++b) p->num_off[b] = 0;
  for (int b = 0; b < kEscBins + 3; ++b) p->esc_off[b] = 0;

  // degenerate shapes: zero row_ptr, c_nnz = 0 (symbolic_spec.hpp:101-107, numeric_tpl_spec_decl.hpp:55-68)
  int64_t nnzA = 0, nnzB = 0;
  if (m > 0) {
    B200SP_REQUIRE(rpA != nullptr, "spgemm_symbolic: row_ptr_A is null");
    int last = 0;
    B200SP_CUDA_TRY(cudaMemcpyAsync(&last, rpA + m, sizeof(int), cudaMemcpyDeviceToHost, st));
    B200SP_CUDA_TRY(cudaStreamSynchronize(st));
    nnzA = last;
  }
  if (n > 0 && nnzA > 0) {
    B200SP_REQUIRE(rpB != nullptr, "spgemm_symbolic: row_ptr_B is null");
    int last = 0;
    B200SP_CUDA_TRY(cudaMemcpyAsync(&last, rpB + n, sizeof(int), cudaMemcpyDeviceToHost, st));
    B200SP_CUDA_TRY(cudaStreamSynchronize(st));
    nnzB = last;
  }
  // numeric needs these even for empty products
  B200SP_CUDA_TRY(p->fb_count.alloc(1, st));
  if (m == 0 || n == 0 || k == 0 || nnzA == 0 || nnzB == 0) {
    const int blocks = std::max(1, std::min((m + 1 + 255) / 256, sm_count() * 8));
    fill_int_kernel<<<blocks, 256, 0, st>>>((int64_t)m + 1, 0, rpC);
    B200SP_LAUNCH_CHECK();
    B200SP_CUDA_TRY(cudaStreamSynchronize(st));
    p->symbolic_done = true;
    if (c_nnz) *c_nnz = 0;
    if (c_max_row_nnz) *c_max_row_nnz = 0;
    return B200SP_OK;
  }
  B200SP_REQUIRE(ciA && ciB, "spgemm_symbolic: null column index array");

  SymTrace trace(st);
  DevTmp tmp(st);
  int *bmin, *bmax, *row_nnz, *sym_rows, *d_counts, *block_max, *d_max;
  long long *block_sum, *d_total;
  const int nblocks = (m + SCAN_ITEMS - 1) / SCAN_ITEMS;
  B200SP_CUDA_TRY(tmp.alloc(&bmin, n));
  B200SP_CUDA_TRY(tmp.alloc(&bmax, n));
  B200SP_CUDA_TRY(tmp.alloc(&row_nnz, m));
  B200SP_CUDA_TRY(tmp.alloc(&sym_rows, m));
  B200SP_CUDA_TRY(tmp.alloc(&d_counts, MAXBINS));
  B200SP_CUDA_TRY(tmp.alloc(&block_sum, nblocks));
  B200SP_CUDA_TRY(tmp.alloc(&block_max, nblocks));
  B200SP_CUDA_TRY(tmp.alloc(&d_total, 1));
  B200SP_CUDA_TRY(tmp.alloc(&d_max, 1));
  B200SP_CUDA_TRY(p->cmin.alloc((size_t)m, st));
  B200SP_CUDA_TRY(p->cmax.alloc((size_t)m, st));
  B200SP_CUDA_TRY(p->flops.alloc((size_t)m, st));
  int* const flops = p->flops;
  B200SP_CUDA_TRY(p->num_rows.alloc((size_t)m, st));
  B200SP_CUDA_TRY(p->fb_rows.alloc((size_t)m, st));

  // lanes per B row from B's mean row length
  {
    const double avg = (double)nnzB / (double)n;
    int lb = 4;
    while (lb < 32 && lb < avg) lb <<= 1;
    p->lb = lb;
  }
  brow_minmax_kernel<<<(unsigned)(((int64_t)n * 8 + 255) / 256), 256, 0, st>>>(n, rpB, ciB, bmin, bmax);
  B200SP_LAUNCH_CHECK();
  arow_analyse_kernel<<<(unsigned)(((int64_t)m * 8 + 255) / 256), 256, 0, st>>>(m, rpA, ciA, rpB, bmin, bmax, flops,
                                                                                p->cmin, p->cmax);
  B200SP_LAUNCH_CHECK();

  trace.mark("allocations + row analysis");
  // ---- count distinct columns per row
  // default (3): rows binned by max(products, 2 nnz(A_i)); up to 8192 -> esc_sym_kernel (spgemm_esc.cuh: products held in
  // registers, hash set of 2x the bin's capacity); above -> the group-walk hash kernel / global bitmap.
  // B200SP_SPGEMM_SYMBOLIC=1: round-1 kernels (bins by flop bound, tables of up to 4x); 2: tables of 2x, 16-byte init
  int sym_variant = 3;
  if (const char* e = getenv("B200SP_SPGEMM_SYMBOLIC")) sym_variant = atoi(e);
  BinSpec sspec;
  int soff[MAXBINS + 1];
  int rc;
  const int lb = p->lb;
  int big_bin;
  // ESC bins (kept on the plan: the numeric phase uses the same grouping)
  B200SP_CUDA_TRY(p->esc_key.alloc((size_t)m, st));
  B200SP_CUDA_TRY(p->esc_rows.alloc((size_t)m, st));
  {
    const int blocks = std::max(1, std::min((m + 255) / 256, sm_count() * 8));
    esc_key_kernel<<<blocks, 256, 0, st>>>(m, flops, rpA, p->esc_key);
    B200SP_LAUNCH_CHECK();
    BinSpec espec;
    espec.nb = kEscBins + 2;  // 4 ESC bins, <= 16384 (hash kernel), the rest (bitmap)
    for (int b = 0; b < kEscBins; ++b) espec.thr[b] = kEscThr[b];
    espec.thr[kEscBins] = 16384;
    rc = bin_rows(st, m, p->esc_key, espec, d_counts, p->esc_rows, p->esc_off);
    if (rc) return rc;
  }
  trace.mark("bin keys + grouping");
  if (sym_variant >= 3) {
    const int* er = p->esc_rows;
    const int* eo = p->esc_off;
    // bin 1 (<= 1024 products, config 4's bin): 256 threads x 4 products, 1024 buckets (the best of the alternatives when
    // the kernel was tuned); B200SP_ESC_SYM_CFG selects the alternatives for A/B runs
    int sym_cfg = 0;
    if (const char* e = getenv("B200SP_ESC_SYM_CFG")) sym_cfg = atoi(e);
    if ((rc = launch_esc_sym<32, 8, 9, 1>(st, eo[1] - eo[0], er + eo[0], rpA, ciA, rpB, ciB, flops, p->cmin, p->cmax, row_nnz))) return rc;
    switch (sym_cfg) {
      case 1: rc = launch_esc_sym<256, 4, 10, 1>(st, eo[2] - eo[1], er + eo[1], rpA, ciA, rpB, ciB, flops, p->cmin, p->cmax, row_nnz); break;
      case 2: rc = launch_esc_sym<256, 4, 10, 6>(st, eo[2] - eo[1], er + eo[1], rpA, ciA, rpB, ciB, flops, p->cmin, p->cmax, row_nnz); break;
      case 3: rc = launch_esc_sym<128, 8, 11, 1>(st, eo[2] - eo[1], er + eo[1], rpA, ciA, rpB, ciB, flops, p->cmin, p->cmax, row_nnz); break;
      case 4: rc = launch_esc_sym<512, 2, 10, 1>(st, eo[2] - eo[1], er + eo[1], rpA, ciA, rpB, ciB, flops, p->cmin, p->cmax, row_nnz); break;
      default: rc = launch_esc_sym<256, 4, 10, 8>(st, eo[2] - eo[1], er + eo[1], rpA, ciA, rpB, ciB, flops, p->cmin, p->cmax, row_nnz); break;
    }
    if (rc) return rc;
    if ((rc = launch_esc_sym<512, 8, 12, 1>(st, eo[3] - eo[2], er + eo[2], rpA, ciA, rpB, ciB, flops, p->cmin, p->cmax, row_nnz))) return rc;
    if ((rc = launch_esc_sym<1024, 8, 13, 1>(st, eo[4] - eo[3], er + eo[3], rpA, ciA, rpB, ciB, flops, p->cmin, p->cmax, row_nnz))) return rc;
    if ((rc = launch_sym<512, 15>(st, eo[5] - eo[4], er + eo[4], lb, rpA, ciA, rpB, ciB, row_nnz))) return rc;
    for (int b = 0; b <= kEscBins + 2; ++b) soff[b] = eo[b];
    sym_rows = p->esc_rows;
    big_bin = kEscBins + 1;
  } else
  if (sym_variant == 2) {
    static const int thr2[] = {128, 512, 1024, 2048, 4096, 8192, 16384};
    sspec.nb = 8;
    for (int b = 0; b < 7; ++b) sspec.thr[b] = thr2[b];
    rc = bin_rows(st, m, flops, sspec, d_counts, sym_rows, soff);
    if (rc) return rc;
#define SYM_BIN2(B, G, LG)                                                                                              \
  if ((rc = launch_sym<G, LG, true>(st, soff[B + 1] - soff[B], sym_rows + soff[B], lb, rpA, ciA, rpB, ciB, row_nnz))) \
    return rc;
    SYM_BIN2(0, 32, 8)     // f <= 128   -> 256 slots, warp per row
    SYM_BIN2(1, 32, 10)    // f <= 512   -> 1024 slots
    SYM_BIN2(2, 128, 11)   // f <= 1024  -> 2048 slots
    SYM_BIN2(3, 128, 12)   // f <= 2048  -> 4096 slots
    SYM_BIN2(4, 256, 13)   // f <= 4096  -> 8192 slots
    SYM_BIN2(5, 256, 14)   // f <= 8192  -> 16384 slots
    SYM_BIN2(6, 512, 15)   // f <= 16384 -> 32768 slots
#undef SYM_BIN2
    big_bin = 7;
  } else {
    sspec.nb = kSymBins;
    for (int b = 0; b < kSymBins - 1; ++b) sspec.thr[b] = kSymThr[b];
    rc = bin_rows(st, m, flops, sspec, d_counts, sym_rows, soff);
    if (rc) return rc;
#define SYM_BIN(B, G, LG)                                                                                          \
  if ((rc = launch_sym<G, LG>(st, soff[B + 1] - soff[B], sym_rows + soff[B], lb, rpA, ciA, rpB, ciB, row_nnz))) \
    return rc;
    SYM_BIN(0, 32, 8)     // f <= 128   -> 256 slots, warp per row
    SYM_BIN(1, 32, 10)    // f <= 512   -> 1024 slots
    SYM_BIN(2, 128, 12)   // f <= 2048  -> 4096 slots
    SYM_BIN(3, 256, 14)   // f <= 8192  -> 16384 slots (64 KB)
    SYM_BIN(4, 512, 15)   // f <= 16384 -> 32768 slots (128 KB)
#undef SYM_BIN
    big_bin = kSymBins - 1;
  }
  {
    const int nbig = soff[big_bin + 1] - soff[big_bin];
    if (nbig > 0) {
      const int ctas = std::min(nbig, sm_count());
      unsigned* bitmaps;
      B200SP_CUDA_TRY(tmp.alloc(&bitmaps, (size_t)ctas * ((k + 31) / 32)));
      sym_bitmap_kernel<<<ctas, 256, 0, st>>>(nbig, sym_rows + soff[big_bin], k, bitmaps, rpA, ciA, rpB, ciB, row_nnz);
      B200SP_LAUNCH_CHECK();
    }
  }

  trace.mark("distinct-column kernels");
  // ---- row_ptr_C = exclusive scan(row_nnz); total and longest row
  scan_local_kernel<<<nblocks, 256, 0, st>>>(m, row_nnz, rpC, block_sum, block_max);
  B200SP_LAUNCH_CHECK();
  scan_blocks_kernel<<<1, 1024, 0, st>>>(nblocks, block_sum, block_max, d_total, d_max);
  B200SP_LAUNCH_CHECK();
  scan_add_kernel<<<nblocks, 256, 0, st>>>(m, rpC, block_sum, d_total);
  B200SP_LAUNCH_CHECK();
  long long total = 0;
  int mx = 0;
  B200SP_CUDA_TRY(cudaMemcpyAsync(&total, d_total, sizeof(total), cudaMemcpyDeviceToHost, st));
  B200SP_CUDA_TRY(cudaMemcpyAsync(&mx, d_max, sizeof(mx), cudaMemcpyDeviceToHost, st));
  B200SP_CUDA_TRY(cudaStreamSynchronize(st));
  if (total > (long long)INT_MAX) {
    set_error("spgemm_symbolic: nnz(C) = %lld exceeds int32 offsets", total);
    return B200SP_ERR_OVERFLOW;
  }
  p->c_nnz = total;
  p->c_max = mx;
  trace.mark("scan -> row_ptr_C");

  // ---- numeric: the ESC grouping above serves rows of <= 8192 products; the rows beyond it are grouped by nnz(C_i) for
  // the hash kernels here (kept on the plan so that numeric stays asynchronous)
  for (int b = 0; b <= kNumBins; ++b) p->num_off[b] = 0;
  p->fb_static = 0;
  if (p->esc_off[kEscBins] < m) {
    int* key2;
    B200SP_CUDA_TRY(tmp.alloc(&key2, m));
    const int blocks = std::max(1, std::min((m + 255) / 256, sm_count() * 8));
    rest_key_kernel<<<blocks, 256, 0, st>>>(m, p->esc_key, kEscCap, rpC, 0, key2);
    B200SP_LAUNCH_CHECK();
    BinSpec nspec;
    nspec.nb = kNumBins + 1;  // bin 0: the ESC rows (key 0), then the hash bins
    nspec.thr[0] = 0;
    for (int b = 0; b < kNumBins - 1; ++b) nspec.thr[b + 1] = kNumThr[b];
    int h_off[MAXBINS + 1];
    rc = bin_rows(st, m, key2, nspec, d_counts, p->num_rows, h_off);
    if (rc) return rc;
    for (int b = 0; b <= kNumBins; ++b) p->num_off[b] = h_off[b + 1];
    p->fb_static = p->num_off[kNumBins] - p->num_off[kNumBins - 1];
    if (p->fb_static > 0)
      B200SP_CUDA_TRY(cudaMemcpyAsync(p->fb_rows, p->num_rows + p->num_off[kNumBins - 1], sizeof(int) * (size_t)p->fb_static,
                                      cudaMemcpyDeviceToDevice, st));
  }
  int lg = 1;
  while (((long long)1 << lg) < 2LL * std::max(mx, 1)) ++lg;
  p->fb_log2 = lg;
  B200SP_CUDA_TRY(p->fb_keys.alloc((size_t)kFbCtas * ((size_t)1 << lg), st));
  B200SP_CUDA_TRY(cudaStreamSynchronize(st));
  trace.mark("hash-bin grouping + scratch");
  p->symbolic_done = true;
  if (c_nnz) *c_nnz = total;
  if (c_max_row_nnz) *c_max_row_nnz = mx;
  return B200SP_OK;
}

int b200sp_spgemm_numeric_f64_i32(b200sp_spgemm_plan* plan, void* stream, int m, int n, int k, const int* rpA,
                                  const int* ciA, const double* vA, const int* rpB, const int* ciB, const double* vB,
                                  const int* rpC, int* ciC, double* vC) {
  return numeric_impl<double>(plan, (cudaStream_t)stream, m, n, k, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC);
}
int b200sp_spgemm_jacobi_f64_i32(b200sp_spgemm_plan* plan, void* stream, int m, int n, int k, const int* rpA,
                                 const int* ciA, const double* vA, const int* rpB, const int* ciB, const double* vB,
                                 const int* rpC, int* ciC, double* vC, double omega, const double* dinv) {
  return jacobi_impl<double>(plan, (cudaStream_t)stream, m, n, k, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC, omega, dinv);
}
int b200sp_spgemm_jacobi_f32_i32(b200sp_spgemm_plan* plan, void* stream, int m, int n, int k, const int* rpA,
                                 const int* ciA, const float* vA, const int* rpB, const int* ciB, const float* vB,
                                 const int* rpC, int* ciC, float* vC, float omega, const float* dinv) {
  return jacobi_impl<float>(plan, (cudaStream_t)stream, m, n, k, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC, omega, dinv);
}
int b200sp_spgemm_numeric_f32_i32(b200sp_spgemm_plan* plan, void* stream, int m, int n, int k, const int* rpA,
                                  const int* ciA, const float* vA, const int* rpB, const int* ciB, const float* vB,
                                  const int* rpC, int* ciC, float* vC) {
  return numeric_impl<float>(plan, (cudaStream_t)stream, m, n, k, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC);
}

int b200sp_spgemm_plan_paths(const b200sp_spgemm_plan* plan, int64_t* counts, int n) {
  B200SP_REQUIRE(plan != nullptr && (counts != nullptr || n <= 0), "spgemm_plan_paths: null argument");
  int64_t c[kSpgemmPaths] = {0};
  // a product with 64-bit offsets: the sum over the plans of its windows
  const bool wide = spgemm64_holds_product(plan->s64);
  const int nplans = wide ? spgemm64_window_count(plan->s64) : 1;
  for (int w = 0; w < nplans; ++w) {
    const b200sp_spgemm_plan* p = wide ? spgemm64_window_plan(plan->s64, w) : plan;
    if (!p->symbolic_done) continue;
    for (int b = 0; b < kEscBins + 2; ++b) c[b] += p->esc_off[b + 1] - p->esc_off[b];
    if (!p->last_off) continue;
    for (int b = 0; b < kNumBins; ++b) c[kEscBins + 2 + b] += p->last_off[b + 1] - p->last_off[b];
    // the run-time overflows: rows the shared-memory kernels appended to the fallback list after the static ones
    int fb = p->fb_static;
    B200SP_CUDA_TRY(cudaDeviceSynchronize());
    B200SP_CUDA_TRY(cudaMemcpy(&fb, p->fb_count.ptr, sizeof(int), cudaMemcpyDeviceToHost));
    c[kSpgemmPaths - 1] += fb - p->fb_static;
  }
  for (int i = 0; i < n; ++i) counts[i] = i < kSpgemmPaths ? c[i] : 0;
  return B200SP_OK;
}

}  // extern "C"
