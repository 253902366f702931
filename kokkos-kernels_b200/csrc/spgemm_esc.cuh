// spgemm_esc.cuh -- register-resident expand / sort / compress kernels of the SpGEMM (included by spgemm.cu).
//
// One CTA of T threads builds one row of C = A*B whose product count f = sum_j nnz(B_{a_ij}) is at most T*I:
// product p (its ORDINAL in the reference's accumulation order: A's row in storage order, each B row in storage
// order, sparse/impl/KokkosSparse_spgemm_impl_seq.hpp:147-164) belongs to thread p % T, item p / T, so the T*I
// gathers of a row are issued back to back from registers (I independent col/val loads per thread in flight)
// and consecutive lanes read consecutive entries of one B row.  Nothing is gathered twice.
//
// Both phases sort the row's columns with one counting sort over a MONOTONE bucket map
//      bucket(c) = c - cmin                                          (row span <= NB: injective)
//                = ((c - cmin) * floor(NB*2^32 / span)) >> 32        otherwise
//   histogram (shared atomicAdd; the returned count is the product's arrival rank in its bucket) -> exclusive
//   scan -> scatter of the keys to bucket order.  Buckets hold 0.5 products on average, so what is left is local:
//  symbolic  esc_sym_kernel : a bitmap pre-filter settles the rows with few duplicates without sorting (see there);
//            otherwise a product is a duplicate iff its bucket holds an equal column at a smaller position;
//            nnz(C_i) = f - duplicates.
//  numeric   esc_num_kernel : every product ranks itself among the members of its bucket by (column, ordinal) and
//            stores (column, value) at its sorted position.  Rows without duplicate columns (f == nnz(C_i), known
//            from symbolic) leave at once with coalesced stores; otherwise the first product of each run of equal
//            columns adds the run up in ordinal order -- the oracle's order, and the product is an unfused multiply,
//            so the VALUES equal the reference's SPGEMM_DEBUG result bit for bit when that is compiled without FMA
//            contraction -- and a ballot scan of the run heads gives the output positions.
//  No floating-point atomics, no second walk over B, deterministic, rows come out sorted by column: the reference's
//  separate sort_crs_matrix pass (sparse/impl/KokkosSparse_spgemm_numeric_spec.hpp:138-140) is not needed.
//
// A row qualifies when max(f, 2 * nnz(A_i)) <= T*I (the staged A row shares memory with the sorted output).
#pragma once
#include "common.cuh"
#include <limits.h>

namespace b200sp {

template <typename S>
__device__ __forceinline__ S mul_rn(S a, S b);
template <>
__device__ __forceinline__ double mul_rn<double>(double a, double b) { return __dmul_rn(a, b); }
template <>
__device__ __forceinline__ float mul_rn<float>(float a, float b) { return __fmul_rn(a, b); }

constexpr int esc_log2(int v) { return v <= 1 ? 0 : 1 + esc_log2(v >> 1); }

// (column, value) pairs of the sorted row: one 16-byte (fp64) / 8-byte (fp32) shared-memory access each
template <typename S>
struct EscKV;
template <>
struct EscKV<double> {
  using type = int4;
  static __device__ __forceinline__ int4 pack(int k, double v) {
    return make_int4(k, 0, __double2loint(v), __double2hiint(v));
  }
  static __device__ __forceinline__ int key(const int4& q) { return q.x; }
  static __device__ __forceinline__ double val(const int4& q) { return __hiloint2double(q.w, q.z); }
};
template <>
struct EscKV<float> {
  using type = int2;
  static __device__ __forceinline__ int2 pack(int k, float v) { return make_int2(k, __float_as_int(v)); }
  static __device__ __forceinline__ int key(const int2& q) { return q.x; }
  static __device__ __forceinline__ float val(const int2& q) { return __int_as_float(q.y); }
};

// exclusive scan in place of a[0..n), n <= T*K, thread t owns a[t*K .. t*K+K); every thread gets the total.
// wsum: 34 ints of shared memory.  Ends with a barrier (a[] and the total are visible to all).
// PACK: the result word is prefix | (count << 16) (both < 65536 here): one shared-memory read per look-up instead of two.
template <int T, int K, bool PACK = false>
__device__ __forceinline__ int esc_block_scan(int* a, int n, int* wsum) {
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  constexpr int NW = T / 32;
  int v[K];
  int s = 0;
  const int base = tid * K;
  if (K % 4 == 0 && base + K <= n) {
#pragma unroll
    for (int c = 0; c < K / 4; ++c) {
      const int4 q = reinterpret_cast<const int4*>(a + base)[c];
      v[4 * c] = q.x; v[4 * c + 1] = q.y; v[4 * c + 2] = q.z; v[4 * c + 3] = q.w;
    }
#pragma unroll
    for (int i = 0; i < K; ++i) s += v[i];
  } else {
#pragma unroll
    for (int i = 0; i < K; ++i) {
      v[i] = (base + i < n) ? a[base + i] : 0;
      s += v[i];
    }
  }
  int inc = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  int woff = 0, total;
  if (NW > 1) {
    if (lane == 31) wsum[w] = inc;
    __syncthreads();
    if (w == 0) {
      const int x = lane < NW ? wsum[lane] : 0;
      int xi = x;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, xi, o);
        if (lane >= o) xi += t;
      }
      if (lane < NW) wsum[lane] = xi - x;
      if (lane == 31) wsum[32] = xi;
    }
    __syncthreads();
    woff = wsum[w];
    total = wsum[32];
  } else {
    total = __shfl_sync(0xffffffffu, inc, 31);
  }
  int run = woff + inc - s;
  if (K % 4 == 0 && base + K <= n) {
#pragma unroll
    for (int c = 0; c < K / 4; ++c) {
      int4 q;
      q.x = PACK ? (run | (v[4 * c] << 16)) : run; run += v[4 * c];
      q.y = PACK ? (run | (v[4 * c + 1] << 16)) : run; run += v[4 * c + 1];
      q.z = PACK ? (run | (v[4 * c + 2] << 16)) : run; run += v[4 * c + 2];
      q.w = PACK ? (run | (v[4 * c + 3] << 16)) : run; run += v[4 * c + 3];
      reinterpret_cast<int4*>(a + base)[c] = q;
    }
  } else {
#pragma unroll
    for (int i = 0; i < K; ++i) {
      if (base + i < n) a[base + i] = PACK ? (run | (v[i] << 16)) : run;
      run += v[i];
    }
  }
  __syncthreads();
  return total;
}

// exclusive scan of one int per thread over the CTA (registers only + wsum); total to all threads.
template <int T>
__device__ __forceinline__ int esc_block_scan1(int v, int* wsum, int& total) {
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  constexpr int NW = T / 32;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  int woff = 0;
  if (NW > 1) {
    __syncthreads();  // wsum may still be read from an earlier scan
    if (lane == 31) wsum[w] = inc;
    __syncthreads();
    if (w == 0) {
      const int x = lane < NW ? wsum[lane] : 0;
      int xi = x;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, xi, o);
        if (lane >= o) xi += t;
      }
      if (lane < NW) wsum[lane] = xi - x;
      if (lane == 31) wsum[32] = xi;
    }
    __syncthreads();
    woff = wsum[w];
    total = wsum[32];
  } else {
    total = __shfl_sync(0xffffffffu, inc, 31);
  }
  return woff + inc - v;
}

// ---- staging of A's row and the product -> (entry of A, offset in its B row) map -------------------
// bs[j] = start of the B row of A's j-th entry, pre[j] = ordinal of its first product (pre[nA] = f), va[j] = its value
// (numeric).  Returns the common length of the B rows (>= 1) when all of them have the same length, else 0.
// Rows of up to 32 entries are staged by warp 0 alone (shuffle scan, one barrier).
template <int T, typename S, bool WITH_VALS>
__device__ __forceinline__ int esc_stage_row(int a0, int nA, int f, const int* __restrict__ ciA, const S* __restrict__ vA,
                                             const int* __restrict__ rpB, int* bs, int* pre, S* va, int* wsum) {
  const int tid = threadIdx.x, lane = tid & 31;
  int* sflag = wsum + 35;
  if (nA <= 32) {
    if (tid < 32) {
      int len = 0;
      if (lane < nA) {
        const int c = ldg(ciA + a0 + lane);
        const int b0 = ldg(rpB + c);
        len = ldg(rpB + c + 1) - b0;
        bs[lane] = b0;
        if (WITH_VALS) va[lane] = ldg(vA + a0 + lane);
      }
      const int len0 = __shfl_sync(0xffffffffu, len, 0);
      const bool uni = __all_sync(0xffffffffu, lane >= nA || len == len0) != 0;
      int inc = len;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
      }
      if (lane < nA) pre[lane] = inc - len;
      if (lane == 0) {
        pre[nA] = f;
        *sflag = (uni && len0 > 0) ? len0 : 0;
      }
    }
    __syncthreads();
    return *sflag;
  }
  if (tid == 0) *sflag = 0;
  __syncthreads();
  int carry = 0;
  int len0 = -1;
  for (int base = 0; base < nA; base += T) {
    const int j = base + tid;
    int len = 0;
    if (j < nA) {
      const int c = ldg(ciA + a0 + j);
      const int b0 = ldg(rpB + c);
      len = ldg(rpB + c + 1) - b0;
      bs[j] = b0;
      if (WITH_VALS) va[j] = ldg(vA + a0 + j);
    }
    if (base == 0) {
      if (tid == 0) wsum[34] = len;
      __syncthreads();
      len0 = wsum[34];
    }
    int total;
    const int excl = esc_block_scan1<T>(len, wsum, total);
    if (j < nA) {
      pre[j] = carry + excl;
      if (len != len0) *sflag = 1;  // benign race: every writer stores 1
    }
    carry += total;
  }
  if (tid == 0) pre[nA] = f;
  __syncthreads();
  return (*sflag == 0 && len0 > 0) ? len0 : 0;
}

// ---- row pipeline of the persistent kernels -------------------------------------------------------------------------
// A CTA works through the rows r = blockIdx.x, blockIdx.x + gridDim.x, ... of its bin ("sequence" k = 0, 1, ...).  What a
// row needs before its first gather is a chain of four dependent global loads (row list -> row header -> A's columns ->
// B's row pointers) that a one-row-per-CTA launch pays once per row (stall sampling put most of both kernels' stalls on
// that chain and on the barrier behind it).  The chain therefore runs as a software
// pipeline, one stage per row built: at the top of row k the B row pointers of row k+1, the A entries of row k+2, the
// header of row k+3 and the list entry of row k+4 are requested, each from what the previous row's requests brought.
// The requests are cp.async copies global -> shared memory (LDGSTS): no register is held while they are in flight.
// (A first version kept the stages in registers of warp 0; under the kernels' register budget they were spilled, a spilled
// destination of a load in flight waits for the load at the spill store, the reloads missed L1 -- the pipeline ran slower
// than the chain it replaced: ncu r02c8.)  The four jobs of a step touch disjoint state, so four different warps do them
// concurrently; every thread waits for its own copies at the END of the row, and the end-of-row barrier publishes them.
//   list     row index of sequence k+3 (or -1)
//   hdr[4]   ring of headers by sequence & 3:  0: rpA[i]  1: rpA[i+1]  2: flops[i]  3: rpC[i]  4: rpC[i+1]  5: cmin[i]
//                                              6: cmax[i]  7: i (or -1: no row)
//   c[2], b0[2], b1[2]   A's columns / the start and end of their B rows, by sequence & 1 (rows of <= 32 entries of A)
//   va[4]    A's values by sequence & 3
// Rows of more than 32 entries of A are pipelined up to their header only (esc_stage_row stages them).
template <typename S, bool WITH_VALS>
struct EscPipeMem {
  int list[4];
  int hdr[4][8];
  int c[2][32];
  int b0[2][32];
  int b1[2][32];
  S va[WITH_VALS ? 4 : 1][32];
};

template <typename S, bool WITH_VALS>
__device__ __forceinline__ void esc_pipe_init(EscPipeMem<S, WITH_VALS>& pm) {  // all threads; followed by a barrier
  const int t = threadIdx.x;
  if (t < 32) pm.hdr[t >> 3][t & 7] = ((t & 7) == 7) ? -1 : 0;
  if (t == 0) pm.list[0] = -1;
}

// job A (one warp): header of sequence k+3 from the list entry that arrived, list entry of sequence k+4
template <typename S, bool WITH_VALS>
__device__ __forceinline__ void esc_pipe_headers(EscPipeMem<S, WITH_VALS>& pm, int k, int nrows, int G,
                                                 const int* __restrict__ rows, const int* __restrict__ rpA,
                                                 const int* __restrict__ flops, const int* __restrict__ rpC,
                                                 const int* __restrict__ cmin, const int* __restrict__ cmax) {
  const int lane = threadIdx.x & 31;
  const int i = pm.list[0];
  __syncwarp();  // every lane has read the entry before lane 0 requests the next one into its place
  int* h = pm.hdr[(k + 3) & 3];
  if (lane < 8) {
    const int* src = nullptr;
    if (i >= 0) {
      switch (lane) {
        case 0: src = rpA + i; break;
        case 1: src = rpA + i + 1; break;
        case 2: src = flops + i; break;
        case 3: src = rpC ? rpC + i : nullptr; break;
        case 4: src = rpC ? rpC + i + 1 : nullptr; break;
        case 5: src = cmin + i; break;
        case 6: src = cmax + i; break;
        default: break;
      }
    }
    if (src) cp_async<4>(&h[lane], src);
    else h[lane] = (lane == 7) ? i : 0;
  }
  if (lane == 0) {
    const long long pos = (long long)blockIdx.x + (long long)(k + 4) * (long long)G;
    if (pos < (long long)nrows) cp_async<4>(&pm.list[0], rows + pos);
    else pm.list[0] = -1;
  }
}

// job B (one warp): A's entries of sequence k+2
template <typename S, bool WITH_VALS>
__device__ __forceinline__ void esc_pipe_aentries(EscPipeMem<S, WITH_VALS>& pm, int k, const int* __restrict__ ciA,
                                                  const S* __restrict__ vA) {
  const int lane = threadIdx.x & 31;
  const int* h = pm.hdr[(k + 2) & 3];
  const int a0 = h[0], nA = h[1] - a0;
  if (nA <= 32 && lane < nA) {
    cp_async<4>(&pm.c[(k + 2) & 1][lane], ciA + a0 + lane);
    if (WITH_VALS) cp_async<(int)sizeof(S)>(&pm.va[WITH_VALS ? ((k + 2) & 3) : 0][lane], vA + a0 + lane);
  }
}

// job C (one warp): start and end of the B rows of sequence k+1
template <typename S, bool WITH_VALS>
__device__ __forceinline__ void esc_pipe_bptrs(EscPipeMem<S, WITH_VALS>& pm, int k, const int* __restrict__ rpB) {
  const int lane = threadIdx.x & 31;
  const int* h = pm.hdr[(k + 1) & 3];
  const int nA = h[1] - h[0];
  if (nA <= 32 && lane < nA) {
    const int c = pm.c[(k + 1) & 1][lane];
    cp_async<4>(&pm.b0[(k + 1) & 1][lane], rpB + c);
    cp_async<4>(&pm.b1[(k + 1) & 1][lane], rpB + c + 1);
  }
}

// job D (one warp): sequence k -> the header and, for a row of <= 32 entries of A, the staging arrays of esc_stage_row
// (bs, pre, va, the uniform-length flag wsum[35]) the CTA builds the row from
template <typename S, bool WITH_VALS>
__device__ __forceinline__ void esc_pipe_publish(const EscPipeMem<S, WITH_VALS>& pm, int k, int* shdr, int* bs, int* pre, S* va,
                                                 int* wsum) {
  const int lane = threadIdx.x & 31;
  const int* h = pm.hdr[k & 3];
  if (lane < 8) shdr[lane] = h[lane];
  const int nA = h[1] - h[0];
  const int f = h[2];
  if (nA > 32) return;
  int len = 0;
  if (lane < nA) {
    const int b0 = pm.b0[k & 1][lane];
    len = pm.b1[k & 1][lane] - b0;
    bs[lane] = b0;
    if (WITH_VALS) va[lane] = pm.va[WITH_VALS ? (k & 3) : 0][lane];
  }
  const int len0 = __shfl_sync(0xffffffffu, len, 0);
  const bool uni = __all_sync(0xffffffffu, lane >= nA || len == len0) != 0;
  if (uni && len0 > 0) {  // (the regular case needs no scan)
    if (lane < nA) pre[lane] = lane * len0;
    if (lane == 0) {
      pre[nA] = f;
      wsum[35] = len0;
    }
    return;
  }
  int inc = len;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane < nA) pre[lane] = inc - len;
  if (lane == 0) {
    pre[nA] = f;
    wsum[35] = 0;
  }
}

// one step of the pipeline at the top of sequence k (k < 0: the prologue), jobs dealt to warps 0..3 (or fewer)
template <int T, typename S, bool WITH_VALS>
__device__ __forceinline__ void esc_pipe_step(EscPipeMem<S, WITH_VALS>& pm, int k, int nrows, int G, const int* __restrict__ rows,
                                              const int* __restrict__ rpA, const int* __restrict__ ciA, const S* __restrict__ vA,
                                              const int* __restrict__ rpB, const int* __restrict__ flops,
                                              const int* __restrict__ rpC, const int* __restrict__ cmin,
                                              const int* __restrict__ cmax, int* shdr, int* bs, int* pre, S* va, int* wsum) {
  constexpr int NW = T / 32;
  const int warp = threadIdx.x >> 5;
  if (warp == 0 % NW && k >= 0) esc_pipe_publish<S, WITH_VALS>(pm, k, shdr, bs, pre, va, wsum);
  if (warp == 1 % NW) esc_pipe_bptrs<S, WITH_VALS>(pm, k, rpB);
  if (warp == 2 % NW) esc_pipe_aentries<S, WITH_VALS>(pm, k, ciA, vA);
  if (warp == 3 % NW) esc_pipe_headers<S, WITH_VALS>(pm, k, nrows, G, rows, rpA, flops, rpC, cmin, cmax);
}

// ---- the products of this thread: columns (and values) in registers ------------------------------------------------
template <int T, int I, typename S, bool WITH_VALS>
__device__ __forceinline__ void esc_expand(int f, int nA, int L0, const int* bs, const int* pre, const S* va,
                                           const int* __restrict__ ciB, const S* __restrict__ vB, int nokey, int (&col)[I],
                                           S (&val)[I]) {
  const int tid = threadIdx.x;
  if (L0 == 32 && f == T * I) {
    // the regular case (config 4: 32 entries in every row of B, a full bin): item k of this thread is entry `lane` of the
    // B row of A's entry k * (T/32) + warp -- no index arithmetic, no predicates
    const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int k = 0; k < I; ++k) {
      const int j = k * (T / 32) + warp;
      const int jb = bs[j] + lane;
      col[k] = ld_stream(ciB + jb);
      if (WITH_VALS) val[k] = mul_rn(ld_stream(vB + jb), va[j]);  // b_val * a_val (impl_seq.hpp:163)
    }
  } else if (L0 > 0) {
    int j = tid / L0, t = tid - j * L0;
    const int dj = T / L0, dt = T - dj * L0;
#pragma unroll
    for (int k = 0; k < I; ++k) {
      col[k] = nokey;
      if (WITH_VALS) val[k] = S(0);
      if (k * T + tid < f) {
        const int jb = bs[j] + t;
        col[k] = ld_stream(ciB + jb);
        if (WITH_VALS) val[k] = mul_rn(ld_stream(vB + jb), va[j]);  // b_val * a_val (impl_seq.hpp:163)
      }
      j += dj;
      t += dt;
      if (t >= L0) {
        t -= L0;
        ++j;
      }
    }
  } else {
    int lo = 0;
#pragma unroll
    for (int k = 0; k < I; ++k) {
      const int p = k * T + tid;
      col[k] = nokey;
      if (WITH_VALS) val[k] = S(0);
      if (p < f) {
        int hi = nA;  // largest j with pre[j] <= p (pre[nA] = f > p); p grows with k: search from the last answer
        while (hi - lo > 1) {
          const int mid = (lo + hi) >> 1;
          if (pre[mid] <= p) lo = mid; else hi = mid;
        }
        const int jb = bs[lo] + (p - pre[lo]);
        col[k] = ld_stream(ciB + jb);
        if (WITH_VALS) val[k] = mul_rn(ld_stream(vB + jb), va[lo]);
      }
    }
  }
}

// ---- counting sort of the columns into bucket order.  On return skey[] holds the keys grouped by bucket,
// pos[k] = position of item k in skey, lc[k] = first position of its bucket | (members of the bucket << 16).
template <int T, int I, int LOG2NB>
__device__ __forceinline__ void esc_bucket_sort(int f, int cmin, long long span, int nokey, const int (&col)[I], int* off,
                                                int* skey, int* wsum, int (&pos)[I], int (&lc)[I]) {
  constexpr int NB = 1 << LOG2NB;
  const bool dense = span <= NB;
  const unsigned long long mult = dense ? 0ull : (((unsigned long long)NB << 32) / (unsigned long long)span);
#pragma unroll
  for (int k = 0; k < I; ++k) {
    pos[k] = 0;
    if (col[k] != nokey) {
      const unsigned d = (unsigned)(col[k] - cmin);
      const int b = dense ? (int)d : (int)(((unsigned long long)d * mult) >> 32);
      const int r = atomicAdd(&off[b], 1);
      pos[k] = b | (r << LOG2NB);
    }
  }
  __syncthreads();
  esc_block_scan<T, NB / T, true>(off, NB, wsum);  // off[b] = first position of bucket b | (members << 16)
#pragma unroll
  for (int k = 0; k < I; ++k) {
    lc[k] = 0;
    if (col[k] != nokey) {
      const int w = off[pos[k] & (NB - 1)];
      const int p0 = (w & 0xffff) + (pos[k] >> LOG2NB);
      skey[p0] = col[k];
      pos[k] = p0;
      lc[k] = w;
    }
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------------
// SYMBOLIC
// ---------------------------------------------------------------------------------------------------
// Most product rows have few or no duplicate columns (config 4: 0.26 per 1024 products).  Before sorting anything the
// columns are therefore hashed into a BITMAP of 128 bits per product slot (atomicOr): a product whose bit was clear is
// certainly a new column; the few whose bit was already set ("suspects": true duplicates + about f/256 false positives)
// are resolved exactly -- a suspect is a duplicate iff a non-suspect product holds the same column, or an equal suspect
// precedes it in the suspect list.  Only rows with more than SUSCAP suspects (duplicate-heavy products such as stencils)
// go through the bucket sort.
template <int T, int I, int LOG2NB>
struct EscSymLayout {
  static constexpr int CAP = T * I;
  static constexpr int NB = 1 << LOG2NB;
  static constexpr int NA = CAP / 2;
  static constexpr int LOG2BITS = esc_log2(CAP) + 7;
  static constexpr int BMW = (1 << LOG2BITS) / 32;       // bitmap words
  static constexpr int SORTW = NB + 4 + CAP + 8;         // off[NB + 4] | skey[CAP] of the fallback, aliased with the bitmap
  static constexpr int REGW = BMW > SORTW ? BMW : SORTW;
  static constexpr int SUSCAP = 64;
  // region[REGW] | bs[NA] | pre[NA + 4] | wsum[36] | sus_n[4] | sus_col[SUSCAP] | sus_dup[SUSCAP] | shdr[8] | pipeline state
  static constexpr size_t BYTES = sizeof(int) * (size_t)(REGW + NA + NA + 4 + 36 + 4 + 2 * SUSCAP + 8) + sizeof(EscPipeMem<float, false>);
  static_assert(BYTES <= 227 * 1024, "esc_sym_kernel: configuration exceeds the shared memory of an SM");
};

// one row: shdr holds its header, and for nA <= 32 warp 0 has staged bs / pre / the uniform-length flag already
template <int T, int I, int LOG2NB>
__device__ __forceinline__ void esc_sym_row(int* region, int* bs, int* pre, int* wsum, int* sus_n, int* sus_col, int* sus_dup,
                                            const int* shdr, const int* __restrict__ ciA, const int* __restrict__ rpB,
                                            const int* __restrict__ ciB, int* __restrict__ row_nnz) {
  using L = EscSymLayout<T, I, LOG2NB>;
  constexpr int NB = L::NB;
  constexpr int NOKEY = INT_MAX;
  constexpr int SUSCAP = L::SUSCAP;
  unsigned* bm = reinterpret_cast<unsigned*>(region);
  int* off = region;               // fallback view
  int* skey = region + NB + 4;
  const int tid = threadIdx.x;
  const int i = shdr[7];
  const int f = shdr[2];
  if (f == 0) {
    if (tid == 0) row_nnz[i] = 0;
    return;
  }
  const int a0 = shdr[0], nA = shdr[1] - a0;
  const int L0 = nA <= 32 ? wsum[35]
                          : esc_stage_row<T, float, false>(a0, nA, f, ciA, (const float*)nullptr, rpB, bs, pre, (float*)nullptr, wsum);
  int col[I];
  float dummy[I];
  esc_expand<T, I, float, false>(f, nA, L0, bs, pre, (const float*)nullptr, ciB, (const float*)nullptr, NOKEY, col, dummy);
  // ---- bitmap pass
  unsigned smask = 0;  // bit k: item k is a suspect
#pragma unroll
  for (int k = 0; k < I; ++k)
    if (col[k] != NOKEY) {
      const unsigned h = ((unsigned)col[k] * 0x9E3779B1u) >> (32 - L::LOG2BITS);
      const unsigned bit = 1u << (h & 31u);
      const unsigned old = atomicOr(&bm[h >> 5], bit);
      if (old & bit) {
        smask |= 1u << k;
        const int idx = atomicAdd(sus_n, 1);
        if (idx < SUSCAP) sus_col[idx] = col[k];
      }
    }
  __syncthreads();
  const int ns = *sus_n;
  if (ns == 0) {
    if (tid == 0) row_nnz[i] = f;
    return;
  }
  if (ns <= SUSCAP) {
    // a suspect equal to a product that was counted as new is a duplicate
    for (int s = 0; s < ns; ++s) {
      const int c = sus_col[s];
      bool hit = false;
#pragma unroll
      for (int k = 0; k < I; ++k) hit = hit || (col[k] == c && !((smask >> k) & 1u));
      if (hit) sus_dup[s] = 1;  // benign race: every writer stores 1
    }
    __syncthreads();
    // ... and so is one that an equal suspect precedes in the list (one of each group of equal suspects counts)
    if (tid < 32) {
      int dups = 0;
      for (int s = tid; s < ns; s += 32) {
        bool dup = sus_dup[s] != 0;
        const int c = sus_col[s];
        for (int s2 = 0; s2 < s && !dup; ++s2) dup = (sus_col[s2] == c);
        dups += dup ? 1 : 0;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) dups += __shfl_xor_sync(0xffffffffu, dups, o);
      if (tid == 0) row_nnz[i] = f - dups;
    }
    return;
  }
  // ---- duplicate-heavy row: counting sort over the monotone buckets, duplicates found inside the buckets
  __syncthreads();  // every thread has read *sus_n and the bitmap is dead
  {
    int4* o4 = reinterpret_cast<int4*>(off);
    for (int s = tid; s < (NB + 4) / 4; s += T) o4[s] = make_int4(0, 0, 0, 0);
  }
  __syncthreads();
  const int cmin = shdr[5];
  const long long span = (long long)shdr[6] - cmin + 1;
  int pos[I], lc[I];
  esc_bucket_sort<T, I, LOG2NB>(f, cmin, span, NOKEY, col, off, skey, wsum, pos, lc);
  // a product is a duplicate iff an equal column sits at a smaller position of its bucket
  int dups = 0;
#pragma unroll
  for (int k = 0; k < I; ++k)
    if (col[k] != NOKEY) {
      const int lo = lc[k] & 0xffff, cnt = lc[k] >> 16;
      if (cnt > 1) {
        const int c = col[k];
        bool dup = false;
#pragma unroll
        for (int u = 0; u < 3; ++u)
          if (u < cnt && lo + u < pos[k]) dup = dup || (skey[lo + u] == c);
        for (int m = lo + 3; m < pos[k]; ++m) dup = dup || (skey[m] == c);
        dups += dup ? 1 : 0;
      }
    }
  int total;
  esc_block_scan1<T>(dups, wsum, total);
  if (tid == 0) row_nnz[i] = f - total;
}

template <int T, int I, int LOG2NB, int MINB>
__global__ void __launch_bounds__(T, MINB)
    esc_sym_kernel(int nrows_bin, const int* __restrict__ rows, const int* __restrict__ rpA, const int* __restrict__ ciA,
                   const int* __restrict__ rpB, const int* __restrict__ ciB, const int* __restrict__ flops,
                   const int* __restrict__ cmin_arr, const int* __restrict__ cmax_arr, int* __restrict__ row_nnz) {
  using L = EscSymLayout<T, I, LOG2NB>;
  constexpr int SUSCAP = L::SUSCAP;
  extern __shared__ __align__(16) int esc_sm[];
  int* region = esc_sm;
  int* bs = region + L::REGW;
  int* pre = bs + L::NA;
  int* wsum = pre + L::NA + 4;
  int* sus_n = wsum + 36;
  int* sus_col = sus_n + 4;
  int* sus_dup = sus_col + SUSCAP;
  int* shdr = sus_dup + SUSCAP;
  auto& pm = *reinterpret_cast<EscPipeMem<float, false>*>(shdr + 8);
  const int tid = threadIdx.x;
  const int G = (int)gridDim.x;
  esc_pipe_init(pm);
  __syncthreads();
#pragma unroll 1
  for (int k = -4; k < 0; ++k) {
    esc_pipe_step<T, float, false>(pm, k, nrows_bin, G, rows, rpA, ciA, (const float*)nullptr, rpB, flops, nullptr, cmin_arr, cmax_arr,
                                   shdr, bs, pre, (float*)nullptr, wsum);
    cp_async_wait_all();
    __syncthreads();
  }
  int k = 0;
#pragma unroll 1
  for (int r = (int)blockIdx.x; r < nrows_bin; r += G, ++k) {
    {
      int4* b4 = reinterpret_cast<int4*>(region);
      for (int s = tid; s < L::BMW / 4; s += T) b4[s] = make_int4(0, 0, 0, 0);
      if (tid == 0) *sus_n = 0;
      if (tid < SUSCAP) sus_dup[tid] = 0;
      if (T < SUSCAP)
        for (int s = tid + T; s < SUSCAP; s += T) sus_dup[s] = 0;
    }
    esc_pipe_step<T, float, false>(pm, k, nrows_bin, G, rows, rpA, ciA, (const float*)nullptr, rpB, flops, nullptr, cmin_arr, cmax_arr,
                                   shdr, bs, pre, (float*)nullptr, wsum);
    __syncthreads();
    esc_sym_row<T, I, LOG2NB>(region, bs, pre, wsum, sus_n, sus_col, sus_dup, shdr, ciA, rpB, ciB, row_nnz);
    cp_async_wait_all();  // this thread's requests of the step above have had the whole row to arrive
    __syncthreads();      // ... and are visible to every warp; the next row reuses every array
  }
}

// ---------------------------------------------------------------------------------------------------
// NUMERIC
// ---------------------------------------------------------------------------------------------------
template <typename S, int T, int I, int LOG2NB>
struct EscNumLayout {
  using KV = typename EscKV<S>::type;
  static constexpr int CAP = T * I;
  static constexpr int NB = 1 << LOG2NB;
  static constexpr int NA = CAP / 2;
  static constexpr int NW = T / 32;
  // off[NB + 4] | skey[CAP] | wsum[36] | hpre[I * NW + 4] | shdr[8] | sord[CAP] (u16) | union { va[NA], bs[NA], pre[NA + 4] ; skv[CAP] }
  static constexpr size_t OFF_BYTES = sizeof(int) * (size_t)(NB + 4);
  static constexpr size_t KEY_BYTES = sizeof(int) * (size_t)CAP;
  static constexpr size_t WS_BYTES = sizeof(int) * (size_t)(36 + I * NW + 4 + 8);
  static constexpr size_t ORD_BYTES = ((sizeof(unsigned short) * (size_t)CAP) + 15) & ~(size_t)15;
  static constexpr size_t STAGE_BYTES = sizeof(int) * (size_t)(NA + NA + 4) + sizeof(S) * (size_t)NA;
  static constexpr size_t SORT_BYTES = sizeof(KV) * (size_t)CAP;
  static constexpr size_t UNION_BYTES = ((STAGE_BYTES > SORT_BYTES ? STAGE_BYTES : SORT_BYTES) + 15) & ~(size_t)15;
  static constexpr size_t PIPE_BYTES = (sizeof(EscPipeMem<S, true>) + 15) & ~(size_t)15;
  static constexpr size_t BYTES = OFF_BYTES + KEY_BYTES + WS_BYTES + ORD_BYTES + UNION_BYTES + PIPE_BYTES;
  static_assert(BYTES <= 227 * 1024, "esc_num_kernel: configuration exceeds the shared memory of an SM");
};

// one row: shdr holds its header, and for nA <= 32 warp 0 has staged bs / pre / va / the uniform-length flag already
template <typename S, int T, int I, int LOG2NB>
__device__ __forceinline__ void esc_num_row(unsigned char* esc_raw, const int* shdr, const int* __restrict__ ciA,
                                            const S* __restrict__ vA, const int* __restrict__ rpB,
                                            const int* __restrict__ ciB, const S* __restrict__ vB, int* __restrict__ ciC,
                                            S* __restrict__ vC) {
  using L = EscNumLayout<S, T, I, LOG2NB>;
  using KVT = EscKV<S>;
  using KV = typename KVT::type;
  constexpr int NW = L::NW;
  constexpr int NOKEY = INT_MAX;
  int* off = reinterpret_cast<int*>(esc_raw);
  int* skey = reinterpret_cast<int*>(esc_raw + L::OFF_BYTES);
  int* wsum = reinterpret_cast<int*>(esc_raw + L::OFF_BYTES + L::KEY_BYTES);
  int* hpre = wsum + 36;
  unsigned short* sord = reinterpret_cast<unsigned short*>(esc_raw + L::OFF_BYTES + L::KEY_BYTES + L::WS_BYTES);
  unsigned char* un = esc_raw + L::OFF_BYTES + L::KEY_BYTES + L::WS_BYTES + L::ORD_BYTES;
  // staging view (S first: 8-byte alignment)
  S* va = reinterpret_cast<S*>(un);
  int* bs = reinterpret_cast<int*>(un + sizeof(S) * (size_t)L::NA);
  int* pre = bs + L::NA;
  // sorted view
  KV* skv = reinterpret_cast<KV*>(un);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cbase = shdr[3];
  const int nz = shdr[4] - cbase;
  if (nz == 0) return;
  const int f = shdr[2];
  const int a0 = shdr[0], nA = shdr[1] - a0;
  const int cmin = shdr[5];
  const long long span = (long long)shdr[6] - cmin + 1;
  const bool nodup = (nz == f);  // no duplicate column in this row (uniform over the CTA)
  const int L0 = nA <= 32 ? wsum[35] : esc_stage_row<T, S, true>(a0, nA, f, ciA, vA, rpB, bs, pre, va, wsum);
  int col[I];
  S val[I];
  esc_expand<T, I, S, true>(f, nA, L0, bs, pre, va, ciB, vB, NOKEY, col, val);
  int pos[I], lc[I];
  // (the first barrier inside the sort retires the staging arrays: skv aliases them)
  esc_bucket_sort<T, I, LOG2NB>(f, cmin, span, NOKEY, col, off, skey, wsum, pos, lc);
  if (nodup) {
    // ---- rank inside the bucket by column -> sorted position; (column, value) stored there
#pragma unroll
    for (int k = 0; k < I; ++k)
      if (col[k] != NOKEY) {
        const int lo = lc[k] & 0xffff, cnt = lc[k] >> 16;
        int less = 0;
        if (cnt > 1) {
          const int c = col[k];
#pragma unroll
          for (int u = 0; u < 3; ++u)
            if (u < cnt) less += (skey[lo + u] < c) ? 1 : 0;
          for (int u = 3; u < cnt; ++u) less += (skey[lo + u] < c) ? 1 : 0;
        }
        skv[lo + less] = KVT::pack(col[k], val[k]);
      }
    __syncthreads();
    const uint64_t once = l2_policy_evict_first();  // C is written once: keep L2 for the gathered rows of B
    for (int q = tid; q < f; q += T) {
      const KV e = skv[q];
      st_once(ciC + cbase + q, KVT::key(e), once);
      st_once(vC + cbase + q, KVT::val(e), once);
    }
    return;
  }
  // ---- rows with duplicate columns: rank by (column, ordinal), then compress the runs
#pragma unroll
  for (int k = 0; k < I; ++k)
    if (col[k] != NOKEY) sord[pos[k]] = (unsigned short)(k * T + tid);
  __syncthreads();
#pragma unroll
  for (int k = 0; k < I; ++k)
    if (col[k] != NOKEY) {
      const int lo = lc[k] & 0xffff, cnt = lc[k] >> 16;
      int less = 0;
      if (cnt > 1) {
        // by column first; the ordinals are read only when the bucket holds another product of the same column (rare in
        // products with few duplicates: the ordinal reads were 9 % of all instructions of the config-4 run, ncu r02c6)
        const int c = col[k];
        int eq = 0;
#pragma unroll
        for (int u = 0; u < 3; ++u)
          if (u < cnt) {
            const int km = skey[lo + u];
            less += (km < c) ? 1 : 0;
            eq += (km == c) ? 1 : 0;
          }
        for (int u = 3; u < cnt; ++u) {
          const int km = skey[lo + u];
          less += (km < c) ? 1 : 0;
          eq += (km == c) ? 1 : 0;
        }
        if (eq > 1) {  // (eq counts the product itself)
          const int p = k * T + tid;
          for (int u = 0; u < cnt; ++u) less += (skey[lo + u] == c && (int)sord[lo + u] < p) ? 1 : 0;
        }
      }
      skv[lo + less] = KVT::pack(col[k], val[k]);
    }
  __syncthreads();
  // run heads in position order q = k*T + tid; output position = heads before q (ballot scan over (k, warp) groups)
  unsigned hmask = 0;  // bit k: position k*T + tid starts a run
#pragma unroll
  for (int k = 0; k < I; ++k) {
    const int q = k * T + tid;
    bool head = false;
    if (q < f) head = (q == 0) || (KVT::key(skv[q]) != KVT::key(skv[q - 1]));
    const unsigned bal = __ballot_sync(0xffffffffu, head);
    if (head) hmask |= 1u << k;
    if (lane == 0) hpre[k * NW + warp] = __popc(bal);
  }
  __syncthreads();
  // exclusive scan of the I * NW group counts (<= 256 values): warp 0
  if (warp == 0) {
    int carry = 0;
    for (int g0 = 0; g0 < I * NW; g0 += 32) {
      const int g = g0 + lane;
      const int v = g < I * NW ? hpre[g] : 0;
      int inc = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
      }
      if (g < I * NW) hpre[g] = carry + inc - v;
      carry += __shfl_sync(0xffffffffu, inc, 31);
    }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < I; ++k) {
    const int q = k * T + tid;
    const bool head = (hmask >> k) & 1u;
    const unsigned bal = __ballot_sync(0xffffffffu, head);
    if (head) {
      const int o = hpre[k * NW + warp] + __popc(bal & ((1u << lane) - 1u));
      if (o < nz) {  // more distinct columns than the symbolic pattern holds = precondition violated: drop, do not corrupt
        const KV e = skv[q];
        const int c = KVT::key(e);
        S v = KVT::val(e);
        for (int q2 = q + 1; q2 < f; ++q2) {  // ordinal order = the oracle's order
          const KV e2 = skv[q2];
          if (KVT::key(e2) != c) break;
          v += KVT::val(e2);
        }
        ciC[cbase + o] = c;
        vC[cbase + o] = v;
      }
    }
  }
}

template <typename S, int T, int I, int LOG2NB, int MINB>
__global__ void __launch_bounds__(T, MINB)
    esc_num_kernel(int nrows_bin, const int* __restrict__ rows, const int* __restrict__ rpA, const int* __restrict__ ciA,
                   const S* __restrict__ vA, const int* __restrict__ rpB, const int* __restrict__ ciB,
                   const S* __restrict__ vB, const int* __restrict__ rpC, int* __restrict__ ciC, S* __restrict__ vC,
                   const int* __restrict__ cmin_arr, const int* __restrict__ cmax_arr, const int* __restrict__ flops) {
  using L = EscNumLayout<S, T, I, LOG2NB>;
  constexpr int NB = L::NB;
  extern __shared__ __align__(16) unsigned char esc_raw[];
  int* off = reinterpret_cast<int*>(esc_raw);
  int* wsum = reinterpret_cast<int*>(esc_raw + L::OFF_BYTES + L::KEY_BYTES);
  int* shdr = wsum + 36 + I * L::NW + 4;
  unsigned char* un = esc_raw + L::OFF_BYTES + L::KEY_BYTES + L::WS_BYTES + L::ORD_BYTES;
  S* va = reinterpret_cast<S*>(un);
  int* bs = reinterpret_cast<int*>(un + sizeof(S) * (size_t)L::NA);
  int* pre = bs + L::NA;
  auto& pm = *reinterpret_cast<EscPipeMem<S, true>*>(esc_raw + L::OFF_BYTES + L::KEY_BYTES + L::WS_BYTES + L::ORD_BYTES + L::UNION_BYTES);
  const int tid = threadIdx.x;
  const int G = (int)gridDim.x;
  esc_pipe_init(pm);
  __syncthreads();
#pragma unroll 1
  for (int k = -4; k < 0; ++k) {
    esc_pipe_step<T, S, true>(pm, k, nrows_bin, G, rows, rpA, ciA, vA, rpB, flops, rpC, cmin_arr, cmax_arr, shdr, bs, pre, va, wsum);
    cp_async_wait_all();
    __syncthreads();
  }
  int k = 0;
#pragma unroll 1
  for (int r = (int)blockIdx.x; r < nrows_bin; r += G, ++k) {
    {
      int4* o4 = reinterpret_cast<int4*>(off);
      for (int s = tid; s < (NB + 4) / 4; s += T) o4[s] = make_int4(0, 0, 0, 0);
    }
    esc_pipe_step<T, S, true>(pm, k, nrows_bin, G, rows, rpA, ciA, vA, rpB, flops, rpC, cmin_arr, cmax_arr, shdr, bs, pre, va, wsum);
    __syncthreads();
    esc_num_row<S, T, I, LOG2NB>(esc_raw, shdr, ciA, vA, rpB, ciB, vB, ciC, vC);
    cp_async_wait_all();  // this thread's requests of the step above have had the whole row to arrive
    __syncthreads();      // ... and are visible to every warp; the next row's staging arrays alias the sorted pairs
  }
}

}  // namespace b200sp
