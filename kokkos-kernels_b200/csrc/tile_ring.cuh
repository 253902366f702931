// tile_ring.cuh -- the shared-memory ring of row-aligned tiles that a producer warp fills with 1-D TMA bulk copies
// (cp.async.bulk + mbarrier) for the consumer warps of the tile kernels: spmv_tile_kernel (spmv.cu, DESIGN.md 3.1) and
// the BsrMatrix tile kernels (bsr.cu), whose entries are blocks of bs*bs values.  The tile descriptors are made once for
// all of them by tile_analyse (build_tiles_kernel, spmv.cu).
#pragma once
#include "common.cuh"

namespace b200sp {

// STAGES stages of VCAP values, CCAP 32-bit columns (entries) and RCAP row_ptr entries
template <typename S_, int VCAP_, int CCAP_, int RCAP_, int STAGES_>
struct TileRing {
  using S = S_;
  static constexpr int VCAP = VCAP_, CCAP = CCAP_, RCAP = RCAP_, STAGES = STAGES_;
  alignas(128) S vals[STAGES][VCAP];
  alignas(128) int cols[STAGES][CCAP];
  alignas(128) int rows[STAGES][RCAP];
  int4 desc[STAGES];
  alignas(8) uint64_t full[STAGES];
  alignas(8) uint64_t empty[STAGES];
};

// the ring of the CSR kernels: CAP entries per stage, row_ptr entries for CAP/2 rows
template <typename S, int CAP, int STAGES>
using CsrTileRing = TileRing<S, CAP, CAP, CAP / 2, STAGES>;

template <typename Ring>
__device__ __forceinline__ void tile_ring_init(Ring& sm, int n_consumer_warps) {
  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < Ring::STAGES; ++s) {
      mbar_init(&sm.full[s], 1);                    // producer's arrive.expect_tx (+ TMA byte count)
      mbar_init(&sm.empty[s], n_consumer_warps);    // one arrive per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
}

// Tile `it` of this CTA is tiles[blockIdx.x + it*gridDim.x]; it goes to stage it % STAGES.
__device__ __forceinline__ bool tile_ring_more(int it, int n_tiles) { return blockIdx.x + (int64_t)it * gridDim.x < n_tiles; }

// ---------------------------------------------------------------------------------------------------------------------
// producer: ONE warp (all 32 lanes)
// ---------------------------------------------------------------------------------------------------------------------
// Descriptor {r0, r1, s, e} of tile `it` into d (the descriptors of 32 tiles are loaded at a time, one per lane, and handed
// out by shuffles), then waits until the consumers have left its stage.  False past this CTA's last tile.
template <typename Ring>
__device__ __forceinline__ bool tile_ring_next(Ring& sm, int it, int lane, int n_tiles, const int4* __restrict__ tiles, int4& mine,
                                               int4& d) {
  if (!tile_ring_more(it, n_tiles)) return false;
  if ((it & 31) == 0) {
    const int64_t t = blockIdx.x + (int64_t)(it + lane) * gridDim.x;
    if (t < n_tiles) mine = tiles[t];
  }
  d.x = __shfl_sync(0xffffffffu, mine.x, it & 31);
  d.y = __shfl_sync(0xffffffffu, mine.y, it & 31);
  d.z = __shfl_sync(0xffffffffu, mine.z, it & 31);
  d.w = __shfl_sync(0xffffffffu, mine.w, it & 31);
  const int stage = it % Ring::STAGES;
  const uint32_t ph = (uint32_t)(it / Ring::STAGES) & 1u;
  mbar_wait(&sm.empty[stage], ph ^ 1u);
  return true;
}

// what tile_ring_stage leaves to lane 0's bulk copies
struct TileStage {
  int s_al, r0_al;  // first staged entry, first staged row_ptr entry
  int nb, nrp;      // entries and row_ptr entries copied in bulk
};

// Stages tile d: entries [s_al, e) -- vpe values each and their 32-bit columns -- at vals/cols[0..), and row_ptr[r0_al ..]
// at rows[0..) (at most RCAP entries), where s_al = s & ~3 and r0_al = r0 & ~3.  Bulk copies stay below entry
// nnz_al = nnz & ~3 and row_ptr entry rp_al_end = (m + 1) & ~3, which keeps them inside the arrays and every length a
// multiple of 16 bytes; here the rest of the tile is copied with plain loads, and tile_ring_issue then issues the bulk part.
template <typename Ring>
__device__ __forceinline__ TileStage tile_ring_stage(Ring& sm, int stage, int4 d, int lane, int64_t nnz_al, int rp_al_end, int vpe,
                                                     const int* __restrict__ row_ptr, const int* __restrict__ col_idx,
                                                     const typename Ring::S* __restrict__ vals) {
  constexpr int RCAP = Ring::RCAP;
  const int r0 = d.x, r1 = d.y, s = d.z, e = d.w;
  typename Ring::S* sv = sm.vals[stage];
  int* sc = sm.cols[stage];
  int* sr = sm.rows[stage];
  TileStage ts;
  ts.s_al = s & ~3;
  const int e_up = (e + 3) & ~3;
  const int64_t bulk_end64 = (int64_t)e_up < nnz_al ? (int64_t)e_up : nnz_al;
  const int bulk_end = (int)bulk_end64;
  ts.nb = (r1 > r0 && bulk_end > ts.s_al) ? bulk_end - ts.s_al : 0;
  if (r1 > r0 && (int64_t)e > nnz_al) {
    const int t0 = (int)((int64_t)ts.s_al > nnz_al ? (int64_t)ts.s_al : nnz_al);
    if constexpr (Ring::CCAP == Ring::VCAP) {  // a column slot per value: one value per entry (CSR, vpe == 1)
      for (int i = t0 + lane; i < e; i += 32) {
        sv[i - ts.s_al] = vals[i];
        sc[i - ts.s_al] = col_idx[i];
      }
    } else {
      for (int b = t0 + lane; b < e; b += 32) sc[b - ts.s_al] = col_idx[b];
      const int64_t v0 = (int64_t)t0 * vpe, v1 = (int64_t)e * vpe, voff = (int64_t)ts.s_al * vpe;
      for (int64_t q = v0 + lane; q < v1; q += 32) sv[q - voff] = vals[q];
    }
  }
  ts.r0_al = r0 & ~3;
  ts.nrp = 0;
  if (r1 > r0) {
    const int want_end = min(r1 + 1, ts.r0_al + RCAP);  // exclusive
    const int want_up = (want_end + 3) & ~3;
    const int rbulk_end = min(min(want_up, ts.r0_al + RCAP), rp_al_end);
    ts.nrp = rbulk_end > ts.r0_al ? rbulk_end - ts.r0_al : 0;
    if (want_end > rp_al_end) {
      const int t0 = max(ts.r0_al, rp_al_end);
      for (int i = t0 + lane; i < want_end; i += 32) sr[i - ts.r0_al] = row_ptr[i];
    }
  }
  return ts;
}

// Lane 0, after a __syncwarp behind tile_ring_stage: publishes the descriptor, arms the stage's `full` barrier with the bytes
// of the bulk copies and issues them.
template <typename Ring>
__device__ __forceinline__ void tile_ring_issue(Ring& sm, int stage, int4 d, const TileStage& ts, int vpe, const int* __restrict__ row_ptr,
                                                const int* __restrict__ col_idx, const typename Ring::S* __restrict__ vals,
                                                uint64_t pol) {
  sm.desc[stage] = d;
  const uint32_t vbytes = (uint32_t)((size_t)ts.nb * vpe * sizeof(typename Ring::S));
  mbar_arrive_expect_tx(&sm.full[stage], vbytes + (uint32_t)(ts.nb * 4) + (uint32_t)(ts.nrp * 4));
  if (ts.nb > 0) {
    bulk_g2s(sm.vals[stage], vals + (int64_t)ts.s_al * vpe, vbytes, &sm.full[stage], pol);
    bulk_g2s(sm.cols[stage], col_idx + ts.s_al, (uint32_t)(ts.nb * 4), &sm.full[stage], pol);
  }
  if (ts.nrp > 0) bulk_g2s(sm.rows[stage], row_ptr + ts.r0_al, (uint32_t)(ts.nrp * 4), &sm.full[stage], pol);
}

// The producer of the BSR tile kernels (vpe values per entry: bs*bs).
// spmv_tile_kernel has its own, which also streams its 16-bit column forms.
template <typename Ring>
__device__ __forceinline__ void tile_ring_produce(Ring& sm, int lane, int m, int64_t nnz, int vpe, int n_tiles,
                                                  const int4* __restrict__ tiles, const int* __restrict__ row_ptr,
                                                  const int* __restrict__ col_idx, const typename Ring::S* __restrict__ vals) {
  const uint64_t pol = l2_policy_evict_first();
  const int64_t nnz_al = nnz & ~(int64_t)3;
  const int rp_al_end = (m + 1) & ~3;
  int4 mine = make_int4(0, 0, 0, 0), d;
  for (int it = 0; tile_ring_next(sm, it, lane, n_tiles, tiles, mine, d); ++it) {
    const int stage = it % Ring::STAGES;
    const TileStage ts = tile_ring_stage(sm, stage, d, lane, nnz_al, rp_al_end, vpe, row_ptr, col_idx, vals);
    __syncwarp();
    if (lane == 0) tile_ring_issue(sm, stage, d, ts, vpe, row_ptr, col_idx, vals, pol);
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// consumers
// ---------------------------------------------------------------------------------------------------------------------
// the stage of tile `it`, once the producer's copies have landed: its rows [r0, r1) and where its entries (s_al) and row_ptr
// entries (r0_al) start, aligned as tile_ring_stage aligned them
struct TileView {
  int stage, r0, r1, s_al, r0_al;
};

template <int EAL, int RAL, typename Ring>
__device__ __forceinline__ TileView tile_ring_acquire(Ring& sm, int it) {
  TileView t;
  t.stage = it % Ring::STAGES;
  const uint32_t ph = (uint32_t)(it / Ring::STAGES) & 1u;
  mbar_wait(&sm.full[t.stage], ph);
  const int4 d = sm.desc[t.stage];
  t.r0 = d.x;
  t.r1 = d.y;
  t.s_al = d.z & ~(EAL - 1);
  t.r0_al = t.r0 & ~(RAL - 1);
  return t;
}

// every lane of the warp: the warp is done with the stage
template <typename Ring>
__device__ __forceinline__ void tile_ring_release(Ring& sm, int stage, int lane) {
  __syncwarp();
  if (lane == 0) mbar_arrive(&sm.empty[stage]);
}

// row_ptr[r] and row_ptr[r + 1] of row r of the tile: from the stage when both are staged (o = r - r0_al), else from global
// memory.  Returns whether they were staged.
template <typename Ring>
__device__ __forceinline__ bool tile_row_bounds(const Ring& sm, int stage, const int* __restrict__ row_ptr, int r, int o, int& rs,
                                                int& re) {
  if (o + 1 < Ring::RCAP) {
    rs = sm.rows[stage][o];
    re = sm.rows[stage][o + 1];
    return true;
  }
  rs = row_ptr[r];
  re = row_ptr[r + 1];
  return false;
}

// ---------------------------------------------------------------------------------------------------------------------
// tile analysis (spmv.cu): tile b owns the rows whose first entry lies in [b*T, (b+1)*T), T = cap - lmax - 8; rows longer
// than lmax are listed for the caller's long-row kernel.  Stream-ordered, no host synchronisation.
// ---------------------------------------------------------------------------------------------------------------------
struct TileAnalysis {
  DevArray<int4> tiles;  // {r0, r1, s, e} per tile
  int n_tiles = 0, T = 0, LMAX = 0;
  DevArray<int> long_rows;  // long_cap entries, *n_long of them used
  DevArray<int> n_long;
  int long_cap = 0;
  void release_long_rows(cudaStream_t st) {
    long_rows.release(st);
    n_long.release(st);
  }
  void release(cudaStream_t st) {
    tiles.release(st);
    release_long_rows(st);
    n_tiles = 0;
  }
};
// *out is empty on entry
int tile_analyse(cudaStream_t st, int m, int64_t nnz, const int* row_ptr, int cap, int lmax, TileAnalysis* out);

}  // namespace b200sp
