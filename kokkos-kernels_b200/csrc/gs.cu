// gs.cu -- point (multicolour) Gauss-Seidel: symbolic (colouring), numeric (inverse diagonal), apply (sweeps).
// SURVEY.md section 8f rank 4: the preconditioner of the reference's CG driver.
//
// Replaces, behind the C ABI (b200sp_gs_*), the point algorithm of
//   KokkosSparse::gauss_seidel_symbolic / gauss_seidel_numeric          sparse/src/KokkosSparse_gauss_seidel.hpp:49-360
//   symmetric_ / forward_sweep_ / backward_sweep_gauss_seidel_apply      sparse/src/KokkosSparse_gauss_seidel.hpp:363-1100
//   = PointGaussSeidel (GS_DEFAULT: GS_TEAM on GPUs, GS_PERMUTED elsewhere) sparse/impl/KokkosSparse_gauss_seidel_impl.hpp
// The reference colours the graph (KokkosGraph), PERMUTES the matrix so that every colour set is a contiguous row range
// (a second copy of A in HBM, rebuilt in every numeric call), and sweeps the sets; the arithmetic of a row is PSGS::operator()
// (:159-179): sum = y_i - sum_j a_ij x_j (diagonal included), x_i += omega * sum * inv_diag_i.
//
// Here the matrix stays where it is: symbolic produces the colour of every row and the row LIST of every colour set (rows
// ascending inside a set), numeric only extracts 1 / a_ii, and a sweep launches, per colour set, one kernel that gives every
// listed row LPR lanes.  No second copy of A; the price is that a set's rows are not contiguous (the row map and x are
// gathered anyway, the values of a row are contiguous as before).
//   * colouring: Jones-Plassmann with a hashed priority -- per round, every uncoloured row that beats all its uncoloured
//     neighbours takes the smallest colour no coloured neighbour holds; the rows coloured in one round are pairwise
//     non-adjacent, so they only read colours fixed in earlier rounds (no race, deterministic result).  A structurally
//     nonsymmetric matrix is coloured on the union of its pattern and its transpose's (is_graph_symmetric = 0).
//   * same arithmetic per row as the reference, dot product split over the row's lanes and summed by shuffles.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "common.cuh"
#include "scan.cuh"

namespace b200sp {
int transpose_structure(cudaStream_t st, int m, int n, int64_t nnz, const int* rp, const int* ci, int* trp, int* tci, int* t_src);

namespace {

__device__ __forceinline__ unsigned gs_priority(unsigned v) {  // a fixed hash: the colouring is reproducible
  v ^= v >> 16;
  v *= 0x7feb352du;
  v ^= v >> 15;
  v *= 0x846ca68bu;
  v ^= v >> 16;
  return v;
}
__device__ __forceinline__ bool gs_beats(int a, int b) {  // does row a outrank row b?
  const unsigned pa = gs_priority((unsigned)a), pb = gs_priority((unsigned)b);
  return pa > pb || (pa == pb && a > b);
}

// One Jones-Plassmann round.  colors[v] < 0: uncoloured.  Rows coloured in this round write `next` only; the caller swaps.
__global__ void __launch_bounds__(256) gs_color_round_kernel(int n, const int* __restrict__ rp, const int* __restrict__ ci,
                                                             const int* __restrict__ trp, const int* __restrict__ tci,
                                                             const int* __restrict__ colors, int* __restrict__ next, int* __restrict__ remaining) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) {
    const int cv = colors[v];
    if (cv >= 0) {
      next[v] = cv;
      continue;
    }
    bool top = true;
    for (int pass = 0; pass < 2 && top; ++pass) {
      const int* p = pass ? trp : rp;
      const int* c = pass ? tci : ci;
      if (!p) continue;
      for (int j = p[v]; j < p[v + 1]; ++j) {
        const int u = c[j];
        if (u == v || u >= n) continue;
        if (colors[u] < 0 && gs_beats(u, v)) {
          top = false;
          break;
        }
      }
    }
    if (!top) {
      next[v] = -1;
      atomicAdd(remaining, 1);
      continue;
    }
    // smallest colour not held by a coloured neighbour: windows of 64 colours
    int chosen = -1;
    for (int base = 0; chosen < 0; base += 64) {
      unsigned long long used = 0ull;
      for (int pass = 0; pass < 2; ++pass) {
        const int* p = pass ? trp : rp;
        const int* c = pass ? tci : ci;
        if (!p) continue;
        for (int j = p[v]; j < p[v + 1]; ++j) {
          const int u = c[j];
          if (u == v || u >= n) continue;
          const int cu = colors[u];
          if (cu >= base && cu < base + 64) used |= 1ull << (cu - base);
        }
      }
      if (~used) chosen = base + (__ffsll((long long)~used) - 1);
    }
    next[v] = chosen;
  }
}

// Iterated greedy (Culberson): a NEW colouring is built from nothing, visiting the old colour classes from the last to the
// first; the rows of one class -- an independent set, so they can be coloured together -- each take the smallest colour no
// already re-coloured neighbour holds.  Never uses more colours than the old colouring (a class can always share one colour),
// and usually fewer: a hashed Jones-Plassmann order needs about twice the colours of a good sequential order.
__global__ void __launch_bounds__(256) gs_recolor_class_kernel(int n, int cls, const int* __restrict__ rp, const int* __restrict__ ci,
                                                               const int* __restrict__ trp, const int* __restrict__ tci,
                                                               const int* __restrict__ old_colors, int* __restrict__ colors) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) {
    if (old_colors[v] != cls) continue;
    int chosen = -1;
    for (int base = 0; chosen < 0; base += 64) {
      unsigned long long used = 0ull;
      for (int pass = 0; pass < 2; ++pass) {
        const int* p = pass ? trp : rp;
        const int* c = pass ? tci : ci;
        if (!p) continue;
        for (int j = p[v]; j < p[v + 1]; ++j) {
          const int u = c[j];
          if (u == v || u >= n) continue;
          const int cu = colors[u];  // -1: not re-coloured yet; never a row of this class (independent set)
          if (cu >= base && cu < base + 64) used |= 1ull << (cu - base);
        }
      }
      if (~used) chosen = base + (__ffsll((long long)~used) - 1);
    }
    colors[v] = chosen;
  }
}

// used[c] = 1 for every colour that still has a row; then colours are renumbered densely through the scan of used[]
__global__ void __launch_bounds__(256) gs_mark_used_kernel(int n, const int* __restrict__ colors, int* __restrict__ used) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) used[colors[v]] = 1;
}
__global__ void __launch_bounds__(256) gs_relabel_kernel(int n, const int* __restrict__ newid, int* __restrict__ colors) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) colors[v] = newid[colors[v]];
}

__global__ void __launch_bounds__(256) gs_max_color_kernel(int n, const int* __restrict__ colors, int* __restrict__ out) {
  int m = -1;
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) m = max(m, colors[v]);
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_down_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(out, m);
}

__global__ void __launch_bounds__(256) gs_flag_kernel(int n, const int* __restrict__ colors, int c, int* __restrict__ flag) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) flag[v] = colors[v] == c;
}
// rows of colour c, ascending, behind the sets already written; pos = exclusive scan of the flags (pos[n] = the set's size)
__global__ void __launch_bounds__(256) gs_scatter_kernel(int n, const int* __restrict__ colors, int c, const int* __restrict__ pos,
                                                         int* __restrict__ color_ptr, int* __restrict__ color_rows) {
  const int base = color_ptr[c];
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) {
    if (colors[v] == c) color_rows[base + pos[v]] = v;
    if (v == 0) color_ptr[c + 1] = base + pos[n];
  }
}

template <typename S>
__global__ void __launch_bounds__(256) gs_inverse_diagonal_kernel(int n, const int* __restrict__ rp, const int* __restrict__ ci,
                                                                  const S* __restrict__ v, S* __restrict__ dinv, int* __restrict__ missing) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
    S d = S(0);
    bool found = false;
    for (int j = rp[r]; j < rp[r + 1]; ++j)
      if (ci[j] == r) {  // duplicates of the diagonal entry add up, as they do in the row's dot product
        d += v[j];
        found = true;
      }
    if (!found || d == S(0)) {
      atomicAdd(missing, 1);
      dinv[r] = S(1);
    } else {
      dinv[r] = S(1) / d;
    }
  }
}

// one colour set: LPR lanes per listed row
template <typename S, int LPR>
__global__ void __launch_bounds__(256) gs_set_kernel(const int* __restrict__ rows, int count, const int* __restrict__ rp,
                                                     const int* __restrict__ ci, const S* __restrict__ v, const S* __restrict__ dinv,
                                                     const S* __restrict__ y, S* __restrict__ x, S omega) {
  const int lane = threadIdx.x & 31, sl = lane % LPR;
  const int64_t groups = ((int64_t)gridDim.x * blockDim.x) / LPR;
  const int64_t first = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / LPR;
  const int64_t warp_first = ((int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31)) / LPR;
  for (int64_t base = 0; warp_first + base < count; base += groups) {
    const int64_t q = first + base;
    const bool valid = q < count;
    int ii = 0, rs = 0, re = 0;
    if (valid) {
      ii = rows[q];
      rs = rp[ii];
      re = rp[ii + 1];
    }
    S part = S(0);
    // x is read through the ordinary path: other colour sets wrote it in earlier kernels of this sweep
    for (int j = rs + sl; j < re; j += LPR) part += ld_stream(v + j) * x[ld_stream(ci + j)];
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) part += shfl_xor(part, o);
    if (valid && sl == 0) {
      const S sum = y[ii] - part;
      x[ii] += omega * sum * dinv[ii];
    }
  }
}

}  // namespace
}  // namespace b200sp

using namespace b200sp;

struct b200sp_gs_plan {
  int ncols = 0;  // num_cols of the matrix symbolic saw (>= n: columns beyond n are ghost entries of x)
  int n = -1;
  int num_colors = 0;
  DevArray<int> colors;      // n
  DevArray<int> color_ptr;   // num_colors + 1
  DevArray<int> color_rows;  // n
  std::vector<int> h_color_ptr;
  DevArray<char> dinv;  // n scalars of the numeric call's type
  int dinv_bytes_per = 0;
  bool symbolic_done = false, numeric_done = false;
  int lpr = 4;
  char last_kernel[64] = "none";  // the set kernel of the last apply and its launch count (tests)
};

namespace b200sp {
namespace {

void gs_release(b200sp_gs_plan* p, cudaStream_t st) {
  p->colors.release(st);
  p->color_ptr.release(st);
  p->color_rows.release(st);
  p->dinv.release(st);
  p->symbolic_done = p->numeric_done = false;
}

template <typename S>
int gs_numeric_impl(b200sp_gs_plan* p, cudaStream_t st, int n, const int* rp, const int* ci, const S* v) {
  B200SP_REQUIRE(p != nullptr, "gauss_seidel_numeric: null plan");
  if (!p->symbolic_done || p->n != n) {
    set_error("gauss_seidel_numeric: call gauss_seidel_symbolic first (same handle, same matrix size)");
    return B200SP_ERR_STATE;
  }
  if (n == 0) {
    p->numeric_done = true;
    p->dinv_bytes_per = (int)sizeof(S);
    return B200SP_OK;
  }
  B200SP_REQUIRE(rp && ci && v, "gauss_seidel_numeric: null array");
  B200SP_CUDA_TRY(p->dinv.grow(sizeof(S) * (size_t)n, st));
  p->dinv_bytes_per = (int)sizeof(S);
  DevTmp tmp(st);
  int* missing = nullptr;
  B200SP_CUDA_TRY(tmp.alloc(&missing, 1));
  B200SP_CUDA_TRY(cudaMemsetAsync(missing, 0, sizeof(int), st));
  gs_inverse_diagonal_kernel<S><<<grid_for(n), 256, 0, st>>>(n, rp, ci, v, p->dinv.as<S>(), missing);
  B200SP_LAUNCH_CHECK();
  int h_missing = 0;
  B200SP_CUDA_TRY(cudaMemcpyAsync(&h_missing, missing, sizeof(int), cudaMemcpyDeviceToHost, st));
  B200SP_CUDA_TRY(cudaStreamSynchronize(st));
  if (h_missing > 0) {
    set_error("gauss_seidel_numeric: %d rows have no (or a zero) diagonal entry", h_missing);
    return B200SP_ERR_INVALID_ARGUMENT;
  }
  p->numeric_done = true;
  return B200SP_OK;
}

template <typename S>
int gs_apply_impl(b200sp_gs_plan* p, cudaStream_t st, int n, const int* rp, const int* ci, const S* v, S* x, const S* y, int init_zero_x,
                  S omega, int sweeps, int direction) {
  B200SP_REQUIRE(p != nullptr, "gauss_seidel_apply: null plan");
  B200SP_REQUIRE(direction >= 0 && direction <= 2, "gauss_seidel_apply: direction must be 0 (symmetric), 1 (forward) or 2 (backward)");
  B200SP_REQUIRE(sweeps >= 0, "gauss_seidel_apply: negative sweep count");
  if (!p->numeric_done || p->n != n || p->dinv_bytes_per != (int)sizeof(S)) {
    set_error("gauss_seidel_apply: call gauss_seidel_symbolic and gauss_seidel_numeric (same scalar type) first");
    return B200SP_ERR_STATE;
  }
  if (n == 0) return B200SP_OK;
  B200SP_REQUIRE(rp && ci && v && x && y, "gauss_seidel_apply: null array");
  if (init_zero_x)  // all of x, ghost entries included, as the reference's zero_vector(num_cols, ...) does (gauss_seidel_impl.hpp:1426-1428)
    B200SP_CUDA_TRY(cudaMemsetAsync(x, 0, sizeof(S) * (size_t)std::max(n, p->ncols), st));
  const S* dinv = p->dinv.as<const S>();
  int launches = 0;
  for (int s = 0; s < sweeps; ++s) {
    for (int backward = 0; backward < 2; ++backward) {
      if (!backward && direction == 2) continue;
      if (backward && direction == 1) continue;
      for (int it = 0; it < p->num_colors; ++it) {
        const int c = backward ? p->num_colors - 1 - it : it;
        const int b = p->h_color_ptr[c], e = p->h_color_ptr[c + 1];
        if (e <= b) continue;
        const int count = e - b;
        const int64_t threads = (int64_t)count * p->lpr;
        const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>((threads + 255) / 256, (int64_t)sm_count() * 16));
        switch (p->lpr) {
          case 2: gs_set_kernel<S, 2><<<blocks, 256, 0, st>>>(p->color_rows + b, count, rp, ci, v, dinv, y, x, omega); break;
          case 4: gs_set_kernel<S, 4><<<blocks, 256, 0, st>>>(p->color_rows + b, count, rp, ci, v, dinv, y, x, omega); break;
          case 8: gs_set_kernel<S, 8><<<blocks, 256, 0, st>>>(p->color_rows + b, count, rp, ci, v, dinv, y, x, omega); break;
          case 16: gs_set_kernel<S, 16><<<blocks, 256, 0, st>>>(p->color_rows + b, count, rp, ci, v, dinv, y, x, omega); break;
          default: gs_set_kernel<S, 32><<<blocks, 256, 0, st>>>(p->color_rows + b, count, rp, ci, v, dinv, y, x, omega); break;
        }
        B200SP_LAUNCH_CHECK();
        ++launches;
      }
    }
  }
  snprintf(p->last_kernel, sizeof(p->last_kernel), "gs_set<%s,LPR=%d>x%d", sizeof(S) == 8 ? "f64" : "f32", p->lpr, launches);
  return B200SP_OK;
}

}  // namespace
}  // namespace b200sp

extern "C" {

int b200sp_gs_plan_create(b200sp_gs_plan** plan) {
  B200SP_REQUIRE(plan != nullptr, "gs plan_create: null output pointer");
  *plan = new (std::nothrow) b200sp_gs_plan();
  B200SP_REQUIRE(*plan != nullptr, "gs plan_create: out of host memory");
  return B200SP_OK;
}

int b200sp_gs_plan_destroy(b200sp_gs_plan* p, void* stream) {
  if (!p) return B200SP_OK;
  gs_release(p, (cudaStream_t)stream);
  delete p;
  return B200SP_OK;
}

int b200sp_gs_symbolic_i32(b200sp_gs_plan* p, void* stream, int n, const int* row_ptr, const int* col_idx, int is_graph_symmetric) {
  return b200sp_gs_symbolic_nc_i32(p, stream, n, n, row_ptr, col_idx, is_graph_symmetric);
}

// num_cols >= num_rows: the local matrix of a distributed one; columns >= num_rows address ghost entries of x (read by the sweeps,
// never written) and take no part in the colouring
int b200sp_gs_symbolic_nc_i32(b200sp_gs_plan* p, void* stream, int n, int ncols, const int* row_ptr, const int* col_idx,
                              int is_graph_symmetric) {
  B200SP_REQUIRE(p != nullptr, "gauss_seidel_symbolic: null plan");
  B200SP_REQUIRE(n >= 0 && ncols >= n, "gauss_seidel_symbolic: needs 0 <= num_rows <= num_cols (got %d x %d)", n, ncols);
  cudaStream_t st = (cudaStream_t)stream;
  gs_release(p, st);
  p->n = n;
  p->ncols = ncols;
  p->num_colors = 0;
  p->h_color_ptr.assign(1, 0);
  if (n == 0) {
    p->symbolic_done = true;
    return B200SP_OK;
  }
  B200SP_REQUIRE(row_ptr != nullptr, "gauss_seidel_symbolic: null row map");
  int nnz = 0;
  B200SP_CUDA_TRY(cudaMemcpyAsync(&nnz, row_ptr + n, sizeof(int), cudaMemcpyDeviceToHost, st));
  B200SP_CUDA_TRY(cudaStreamSynchronize(st));
  B200SP_REQUIRE(nnz == 0 || col_idx != nullptr, "gauss_seidel_symbolic: null entries");
  DevTmp tmp(st);
  int *trp = nullptr, *tci = nullptr, *tsrc = nullptr, *next = nullptr, *remaining = nullptr, *flag = nullptr, *pos = nullptr, *maxc = nullptr,
      *bmax = nullptr, *dmax = nullptr;
  long long *bsum = nullptr, *dtotal = nullptr;
  if (!is_graph_symmetric && nnz > 0) {  // colour on pattern(A) + pattern(A^T)
    B200SP_CUDA_TRY(tmp.alloc(&trp, (size_t)ncols + 1));  // rows 0 .. n-1 of A^T are the ones the colouring reads
    B200SP_CUDA_TRY(tmp.alloc(&tci, (size_t)nnz));
    B200SP_CUDA_TRY(tmp.alloc(&tsrc, (size_t)nnz));
    const int rc = transpose_structure(st, n, ncols, nnz, row_ptr, col_idx, trp, tci, tsrc);
    if (rc != B200SP_OK) return rc;
  }
  B200SP_CUDA_TRY(p->colors.alloc((size_t)n, st));
  B200SP_CUDA_TRY(p->color_rows.alloc((size_t)n, st));
  B200SP_CUDA_TRY(tmp.alloc(&next, (size_t)n));
  B200SP_CUDA_TRY(tmp.alloc(&remaining, 1));
  B200SP_CUDA_TRY(tmp.alloc(&flag, (size_t)n));
  B200SP_CUDA_TRY(tmp.alloc(&pos, (size_t)n + 1));
  B200SP_CUDA_TRY(tmp.alloc(&bsum, (size_t)scan_blocks(n)));
  B200SP_CUDA_TRY(tmp.alloc(&bmax, (size_t)scan_blocks(n)));
  B200SP_CUDA_TRY(tmp.alloc(&dtotal, 1));
  B200SP_CUDA_TRY(tmp.alloc(&dmax, 1));
  B200SP_CUDA_TRY(tmp.alloc(&maxc, 1));
  B200SP_CUDA_TRY(cudaMemsetAsync(p->colors, 0xFF, sizeof(int) * (size_t)n, st));  // -1: uncoloured
  int* cur = p->colors;
  int* nxt = next;
  const int grid = grid_for(n);
  for (int round = 0;; ++round) {
    B200SP_CUDA_TRY(cudaMemsetAsync(remaining, 0, sizeof(int), st));
    gs_color_round_kernel<<<grid, 256, 0, st>>>(n, row_ptr, col_idx, trp, tci, cur, nxt, remaining);
    B200SP_LAUNCH_CHECK();
    std::swap(cur, nxt);
    int h_remaining = 0;
    B200SP_CUDA_TRY(cudaMemcpyAsync(&h_remaining, remaining, sizeof(int), cudaMemcpyDeviceToHost, st));
    B200SP_CUDA_TRY(cudaStreamSynchronize(st));
    if (h_remaining == 0) break;
    B200SP_REQUIRE(round < 4 * 1024, "gauss_seidel_symbolic: colouring did not finish");  // the top row of every round always colours
  }
  if (cur != p->colors) B200SP_CUDA_TRY(cudaMemcpyAsync(p->colors, cur, sizeof(int) * (size_t)n, cudaMemcpyDeviceToDevice, st));
  // colour count
  auto count_colors = [&](int* h_max) -> int {
    B200SP_CUDA_TRY(cudaMemsetAsync(maxc, 0xFF, sizeof(int), st));
    gs_max_color_kernel<<<grid, 256, 0, st>>>(n, p->colors, maxc);
    B200SP_LAUNCH_CHECK();
    B200SP_CUDA_TRY(cudaMemcpyAsync(h_max, maxc, sizeof(int), cudaMemcpyDeviceToHost, st));
    B200SP_CUDA_TRY(cudaStreamSynchronize(st));
    return B200SP_OK;
  };
  int h_max = -1;
  int rcc = count_colors(&h_max);
  if (rcc != B200SP_OK) return rcc;
  // two passes of iterated greedy over the classes, last to first, then dense renumbering (B200SP_GS_RECOLOR=0 skips them)
  const char* rec = getenv("B200SP_GS_RECOLOR");
  const int passes = rec ? atoi(rec) : 2;
  int *oldc = nullptr, *used = nullptr, *newid = nullptr;
  if (passes > 0 && h_max > 0) {
    B200SP_CUDA_TRY(tmp.alloc(&oldc, (size_t)n));
    B200SP_CUDA_TRY(tmp.alloc(&used, (size_t)h_max + 1));
    B200SP_CUDA_TRY(tmp.alloc(&newid, (size_t)h_max + 2));
  }
  for (int pass = 0; pass < passes && h_max > 0; ++pass) {
    B200SP_CUDA_TRY(cudaMemcpyAsync(oldc, p->colors, sizeof(int) * (size_t)n, cudaMemcpyDeviceToDevice, st));
    B200SP_CUDA_TRY(cudaMemsetAsync(p->colors, 0xFF, sizeof(int) * (size_t)n, st));
    for (int cls = h_max; cls >= 0; --cls) {
      gs_recolor_class_kernel<<<grid, 256, 0, st>>>(n, cls, row_ptr, col_idx, trp, tci, oldc, p->colors);
      B200SP_LAUNCH_CHECK();
    }
    B200SP_CUDA_TRY(cudaMemsetAsync(used, 0, sizeof(int) * ((size_t)h_max + 1), st));
    gs_mark_used_kernel<<<grid, 256, 0, st>>>(n, p->colors, used);
    B200SP_LAUNCH_CHECK();
    const int rcs = launch_exclusive_scan(st, h_max + 1, used, newid, bsum, bmax, dtotal, dmax);
    if (rcs != B200SP_OK) return rcs;
    gs_relabel_kernel<<<grid, 256, 0, st>>>(n, newid, p->colors);
    B200SP_LAUNCH_CHECK();
    rcc = count_colors(&h_max);
    if (rcc != B200SP_OK) return rcc;
  }
  // the row list of every set (stream compaction per colour: rows stay ascending inside a set)
  p->num_colors = h_max + 1;
  B200SP_CUDA_TRY(p->color_ptr.alloc((size_t)(p->num_colors + 1), st));
  B200SP_CUDA_TRY(cudaMemsetAsync(p->color_ptr, 0, sizeof(int) * (size_t)(p->num_colors + 1), st));
  for (int c = 0; c < p->num_colors; ++c) {
    gs_flag_kernel<<<grid, 256, 0, st>>>(n, p->colors, c, flag);
    B200SP_LAUNCH_CHECK();
    const int rc = launch_exclusive_scan(st, n, flag, pos, bsum, bmax, dtotal, dmax);
    if (rc != B200SP_OK) return rc;
    gs_scatter_kernel<<<grid, 256, 0, st>>>(n, p->colors, c, pos, p->color_ptr, p->color_rows);
    B200SP_LAUNCH_CHECK();
  }
  p->h_color_ptr.assign((size_t)p->num_colors + 1, 0);
  B200SP_CUDA_TRY(cudaMemcpyAsync(p->h_color_ptr.data(), p->color_ptr, sizeof(int) * (size_t)(p->num_colors + 1), cudaMemcpyDeviceToHost, st));
  B200SP_CUDA_TRY(cudaStreamSynchronize(st));
  const double avg = (double)nnz / (double)n;
  p->lpr = avg <= 8.0 ? 2 : avg <= 96.0 ? 4 : avg <= 384.0 ? 8 : avg <= 1536.0 ? 16 : 32;
  if (const char* f = getenv("B200SP_GS_LPR")) {  // lanes per row forced (tests): 2, 4, 8, 16 or 32
    const int l = atoi(f);
    B200SP_REQUIRE(l == 2 || l == 4 || l == 8 || l == 16 || l == 32, "gauss_seidel_symbolic: B200SP_GS_LPR must be 2, 4, 8, 16 or 32 (got %s)", f);
    p->lpr = l;
  }
  p->symbolic_done = true;
  return B200SP_OK;
}

int b200sp_gs_numeric_f64_i32(b200sp_gs_plan* p, void* stream, int n, const int* row_ptr, const int* col_idx, const double* vals) {
  return gs_numeric_impl<double>(p, (cudaStream_t)stream, n, row_ptr, col_idx, vals);
}
int b200sp_gs_numeric_f32_i32(b200sp_gs_plan* p, void* stream, int n, const int* row_ptr, const int* col_idx, const float* vals) {
  return gs_numeric_impl<float>(p, (cudaStream_t)stream, n, row_ptr, col_idx, vals);
}
int b200sp_gs_apply_f64_i32(b200sp_gs_plan* p, void* stream, int n, const int* row_ptr, const int* col_idx, const double* vals, double* x,
                            const double* y, int init_zero_x, double omega, int sweeps, int direction) {
  return gs_apply_impl<double>(p, (cudaStream_t)stream, n, row_ptr, col_idx, vals, x, y, init_zero_x, omega, sweeps, direction);
}
int b200sp_gs_apply_f32_i32(b200sp_gs_plan* p, void* stream, int n, const int* row_ptr, const int* col_idx, const float* vals, float* x,
                            const float* y, int init_zero_x, float omega, int sweeps, int direction) {
  return gs_apply_impl<float>(p, (cudaStream_t)stream, n, row_ptr, col_idx, vals, x, y, init_zero_x, omega, sweeps, direction);
}

const char* b200sp_gs_last_kernel(const b200sp_gs_plan* p) { return p ? p->last_kernel : "none"; }

// colouring produced by symbolic (tests, and callers that want to reuse it): device pointers owned by the plan
int b200sp_gs_get_coloring(const b200sp_gs_plan* p, int* num_colors, const int** colors, const int** color_ptr, const int** color_rows) {
  B200SP_REQUIRE(p != nullptr && p->symbolic_done, "gs get_coloring: symbolic has not run");
  if (num_colors) *num_colors = p->num_colors;
  if (colors) *colors = p->colors;
  if (color_ptr) *color_ptr = p->color_ptr;
  if (color_rows) *color_rows = p->color_rows;
  return B200SP_OK;
}

// the same, copied to host arrays of n, num_colors + 1 and n entries (any of them may be NULL); synchronises
int b200sp_gs_copy_coloring(const b200sp_gs_plan* p, void* stream, int* colors_host, int* color_ptr_host, int* color_rows_host) {
  B200SP_REQUIRE(p != nullptr && p->symbolic_done, "gs copy_coloring: symbolic has not run");
  cudaStream_t st = (cudaStream_t)stream;
  if (p->n > 0) {
    if (colors_host) B200SP_CUDA_TRY(cudaMemcpyAsync(colors_host, p->colors, sizeof(int) * (size_t)p->n, cudaMemcpyDeviceToHost, st));
    if (color_rows_host)
      B200SP_CUDA_TRY(cudaMemcpyAsync(color_rows_host, p->color_rows, sizeof(int) * (size_t)p->n, cudaMemcpyDeviceToHost, st));
    B200SP_CUDA_TRY(cudaStreamSynchronize(st));
  }
  if (color_ptr_host)
    for (int c = 0; c <= p->num_colors; ++c) color_ptr_host[c] = p->h_color_ptr[(size_t)c];
  return B200SP_OK;
}

}  // extern "C"
