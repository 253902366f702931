// spmv_plan.h -- the SpMV plan (b200sp_spmv_plan) of spmv.cu (rank 1) and spmm.cu (rank 2), as parts that each own their
// device memory, know what it was built from (a PlanKey, set once a build has succeeded) and give it back.  reset() drops
// what a part derived from the STRUCTURE of the matrix (b200sp_spmv_plan_invalidate); release() frees all of it
// (b200sp_spmv_plan_destroy).  Everything is freed stream-ordered on the caller's stream.
#pragma once
#include "common.cuh"
#include "tile_ring.cuh"

namespace b200sp {

// extra destinations of y: peer GPUs' x buffers (fused all-gather over NVLink, DESIGN.md section 6)
struct YExtra {
  void* p[7];
  int n;
};

// which columns the tiled kernel reads: col_idx, the plan's 16-bit deltas + anchors (section 3.5), or its pattern starts +
// anchors + dictionary (section 3.6)
enum TileCols { COLS_I32 = 0, COLS_DELTA = 1, COLS_PAT = 2 };

// A pinned host copy of a few device ints, fetched without a host synchronisation: valid once ready().  Kept across matrices.
struct HostMirror {
  int* h = nullptr;
  cudaEvent_t ev = nullptr;
  int fetch(const int* d, int count, cudaStream_t st) {
    if (!h) B200SP_CUDA_TRY(cudaMallocHost((void**)&h, sizeof(int) * count));
    if (!ev) B200SP_CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    B200SP_CUDA_TRY(cudaMemcpyAsync(h, d, sizeof(int) * count, cudaMemcpyDeviceToHost, st));
    B200SP_CUDA_TRY(cudaEventRecord(ev, st));
    return B200SP_OK;
  }
  bool ready() const { return cudaEventQuery(ev) == cudaSuccess; }
  void release() {
    if (ev) {
      cudaEventSynchronize(ev);  // the mirror must not be written after it is freed
      cudaEventDestroy(ev);
    }
    if (h) cudaFreeHost(h);
    h = nullptr;
    ev = nullptr;
  }
};

// rank-1 tile analysis for the cfg's stage (plan_analyse).  Its tile table is dropped while the pattern form runs and cut
// again when a call goes back to the cfg's tiles; the long rows stay.
struct SpmvTiles {
  TileAnalysis a;
  uint64_t cut = 0;  // which of the plan's cuts made a.tiles
  PlanKey key;
  HostMirror n_long;  // number of long rows
  bool n_long_known = false;
  void reset(cudaStream_t st) {
    a.release(st);
    key = PlanKey();
    n_long_known = false;
  }
  void release(cudaStream_t st) {
    reset(st);
    n_long.release();
  }
};

// 16-bit column forms of the tiled kernel (plan_idx16, DESIGN.md sections 3.5 and 3.6), keyed on col_idx on top of the
// analysis and reset with it
struct SpmvCols {
  DevArray<uint16_t> d;    // nnz deltas, padded to a multiple of 8 entries
  DevArray<int> anchor;    // m anchors, padded to a multiple of 4 rows
  DevArray<uint16_t> pid;  // m pattern starts, padded to a multiple of 8 rows
  DevArray<int> dict;      // DCAP offsets + the used length
  DevArray<int> bad;       // device flags: [0] deltas, [1] patterns
  TileAnalysis pat;        // the pattern form's tiles (PAT_TILE_CAP entries, the cfg's LMAX), built with its verdict
  uint64_t pat_cut = 0;    // which of the plan's cuts made pat.tiles
  HostMirror verdict;      // of `bad`
  const int* key_ci = nullptr;  // col_idx the state below belongs to
  int state = 0;                // -1: verdict pending, else the TileCols of the matrix
  int launch = COLS_I32;        // the current call's tiled launch takes this form
  void release_streams(cudaStream_t st) {
    d.release(st);
    anchor.release(st);
    pid.release(st);
    dict.release(st);
    bad.release(st);
    pat.release(st);
  }
  void reset(cudaStream_t st) {
    release_streams(st);
    key_ci = nullptr;
    state = 0;
  }
  void release(cudaStream_t st) {
    reset(st);
    verdict.release();
  }
};

// adaptive row splitting of the long rows (B200SP_SPMV_LONGROWS=seg): segments, per-row (first segment, count), partial sums
struct SpmvSegs {
  DevArray<int4> segs;
  DevArray<int> n_seg;
  DevArray<int2> row_seg;
  DevArray<char> partial;
  int cap = 0;
  bool built = false;
  void release(cudaStream_t st) {
    segs.release(st);
    n_seg.release(st);
    row_seg.release(st);
    partial.release(st);
    built = false;
  }
};

// A work item of the rank-2 item kernel is a run of <= LMAX consecutive entries of one row: (row, first entry, length,
// partial slot or -1).  Rows of up to LMAX entries are one item (it writes Y directly); longer rows are cut into pieces whose
// sums go to `partial` and are added up in piece order by a second kernel.  Items are sorted by length, longest first, so
// that the row groups of a warp run loops of equal length and the long items start first.
struct MMItems {
  DevArray<int4> items;
  int n_items = 0;
  DevArray<int4> multi;  // rows of several pieces: (row, first partial slot, pieces, 0)
  int n_multi = 0;
  int n_multi_long = 0;  // of them, at the END of `multi`: rows of more than 64 pieces (added up by a CTA each)
  int n_partial = 0;
  DevArray<char> partial;
  int lmax = 0;
  PlanKey key;
  void release(cudaStream_t st) {
    items.release(st);
    multi.release(st);
    partial.release(st);
    *this = MMItems();
  }
};

// rank-2 state (spmm.cu)
struct SpmmState {
  MMItems items;  // item kernel
  DevArray<char> xt, yt;  // row-major copies of LayoutLeft operands: size-only, kept by reset()
  void reset(cudaStream_t st) { items.release(st); }
  void release(cudaStream_t st) {
    reset(st);
    xt.release(st);
    yt.release(st);
  }
};

// cached transpose (B200SP_SPMV_OPT_CACHE_TRANSPOSE): structure of A^T + source entry of each of its entries, values
// re-gathered on every call (they may have changed in place), and a plan of its own for A^T
struct SpmvTranspose {
  DevArray<int> rp, ci, src;
  DevArray<char> vals;
  PlanKey key;
  b200sp_spmv_plan* plan = nullptr;
  void release(cudaStream_t st) {
    rp.release(st);
    ci.release(st);
    src.release(st);
    vals.release(st);
    key = PlanKey();
    if (plan) b200sp_spmv_plan_destroy(plan, st);
    plan = nullptr;
  }
};

// self-tuning between the tiled and the row-vector kernel (same bits, different speed by matrix):
// call 0 tile, call 1 tile timed, call 2 vector timed, then the faster one (DESIGN.md section 3.3)
struct SpmvTuning {
  int calls = 0, choice = -1;
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  float tile_ms = 0.f, vec_ms = 0.f;
  void reset() {
    calls = 0;
    choice = -1;
  }
  void release() {
    for (cudaEvent_t e : ev)
      if (e) cudaEventDestroy(e);
    *this = SpmvTuning();
  }
};

// host-vector pipeline (b200sp_spmv_hostvec_*): double-buffered device x / y, copy streams, events
struct HostPipe {
  bool init = false;
  cudaStream_t sH = nullptr, sD = nullptr;
  void* dx[2] = {nullptr, nullptr};
  void* dy[2] = {nullptr, nullptr};
  size_t xb = 0, yb = 0;
  cudaEvent_t ev_x[2], ev_c[2], ev_done[2], ev_chunk[8];
  unsigned long long call = 0;
  int nc = 0;
  int tile_b[9];
  int row_b[9];
  PlanKey key;         // of the piece bounds: the matrix, the cfg and the cut of the tile table they come from
  bool defer = false;  // B200SP_SPMV_OPT_HOSTVEC_DEFER: `stream` does not wait for a call's download before the next call computes
  int last_b = -1;     // buffer of the latest call whose download `stream` has not been made to wait for
  void release() {
    if (!init) return;
    cudaStreamSynchronize(sH);
    cudaStreamSynchronize(sD);
    for (int b = 0; b < 2; ++b) {
      if (dx[b]) cudaFree(dx[b]);
      if (dy[b]) cudaFree(dy[b]);
      cudaEventDestroy(ev_x[b]);
      cudaEventDestroy(ev_c[b]);
      cudaEventDestroy(ev_done[b]);
    }
    for (int c = 0; c < 8; ++c) cudaEventDestroy(ev_chunk[c]);
    cudaStreamDestroy(sH);
    cudaStreamDestroy(sD);
    init = false;
  }
};

}  // namespace b200sp

struct b200sp_spmv_plan {
  int algo = B200SP_SPMV_DEFAULT;
  // tuning overrides (-1 = auto)
  int cfg = -1, lpr = -1, ctas_per_sm = -1;
  b200sp::SpmvTiles r1;
  b200sp::SpmvCols cols;
  b200sp::SpmvSegs segs;
  uint64_t cuts = 0;  // tile tables cut so far (r1's or the pattern form's), to stamp each table with its own cut
  b200sp::SpmmState mm;
  bool cache_transpose = false;
  b200sp::SpmvTranspose t;
  b200sp::SpmvTuning at;
  char last_kernel[160] = "none";
  b200sp::YExtra extra = {{nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr}, 0};
  // tile sub-range of the next tiled launch (host-vector pipeline computes y piece by piece); hi < 0 = all
  int range_lo = 0, range_hi = -1;
  b200sp::DevArray<char> dx, dy;  // host-vector staging of the simple path
  b200sp::HostPipe pipe;
};
