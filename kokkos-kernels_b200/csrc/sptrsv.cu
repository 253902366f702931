// sptrsv.cu -- sparse triangular solve on a CrsMatrix by level sets: what the classic (two_stage = false) form of the two-stage
// Gauss-Seidel needs (sparse/impl/KokkosSparse_twostage_gauss_seidel_impl.hpp:685-697, 880-925: Z = (L + D)^{-1} R through
// KokkosSparse::sptrsv_symbolic / sptrsv_solve, sparse/src/KokkosSparse_sptrsv.hpp) and, behind the same C ABI, a stand-alone
// b200sp_sptrsv_* for callers of sptrsv_symbolic / sptrsv_solve on a lower or upper triangular matrix with its diagonal stored.
//
//   symbolic: level(i) = 1 + max level(j) over the off-diagonal entries j of row i (0 for a row without any): the longest
//             dependency chain that ends in row i.  Computed by relaxation sweeps over the still unresolved rows, each sweep
//             reading the levels of the sweep before (two arrays: the result is the exact longest-path level, independent of
//             thread timing); as many sweeps as there are levels.  Rows are then grouped by level (counting sort).
//   solve   : one launch per level, a GROUP of 8 / 16 / 32 lanes per row (by the mean row length):  acc = b_i;  acc -= a_ij * x_j in
//             STORAGE order (unfused multiply and subtract);  x_i = acc / a_ii  -- operation for operation the serial substitution
//             loop of the oracle (oracle/kk_oracle_sptrsv.c: okk_sptrsv), so the result is bit-identical to it whatever the level
//             schedule is.  The lanes of a group load a batch of the row's (column, value, x[column]) and form the products IN
//             PARALLEL (each product is rounded on its own either way); only the chain of subtractions runs in order, on values
//             passed by shuffle.  One thread per row (the first version) spends its time in ~14 serial rounds of dependent
//             loads per row on the 27-point operator; a group needs three
//             (row record -> columns / values -> x).  The row record (row, begin, end) is stored with the level lists.
//             The Gauss-Seidel form solves with the lower (upper) triangle of a general matrix: the entries on the other side and
//             the ghost columns are skipped (`filter`), no copy of the triangle is made; with a caller-supplied inverse diagonal
//             the diagonal is 1 / dinv_i, as in the reference.
//             Runs of consecutive SMALL levels (one row per lane group of a 1024-thread CTA: the first and last planes of a stencil,
//             all of a banded matrix) are solved by ONE launch of a single CTA that walks them with a CTA barrier in between -- the
//             dependent-launch latency of a level becomes a barrier plus one load round trip (B200SP_SPTRSV_CHAIN=0: off).
//   symbolic sweeps are launched TR_SWEEP_BATCH at a time between two read-backs of the progress counter (a sweep after the
//             last row was resolved changes nothing).
#include <algorithm>
#include <cstdlib>
#include <new>
#include <vector>

#include "common.cuh"

struct b200sp_sptrsv_plan {
  int n = 0;
  bool lower = true;
  bool filter = false;  // the triangle of a general matrix (the Gauss-Seidel form) instead of a triangular matrix
  bool symbolic = false;
  const int *key_rp = nullptr, *key_ci = nullptr;
  int n_levels = 0;
  b200sp::DevArray<int4> level_rows;  // rows grouped by level (device): (row, first entry, end of the row, -)
  int group = 8;                  // lanes per row of the solve kernels
  int* level_ptr_host = nullptr;  // n_levels + 1 offsets (host)
  b200sp::DevArray<int> level_ptr_dev;  // the same on the device (the chain kernel walks it)
  struct Segment {
    int l0, l1;  // levels [l0, l1): one launch per level, or one single-CTA launch for the whole run when `chain`
    bool chain;
    int threads;  // chain: CTA size = lanes of the largest level of the run (a narrow CTA has a cheaper barrier)
  };
  std::vector<Segment> segments;
};

namespace b200sp {
namespace {

constexpr int TR_CHAIN_THREADS = 1024;  // a level of at most TR_CHAIN_THREADS / group rows is "small": one CTA solves it in one pass
constexpr int TR_SWEEP_BATCH   = 8;     // symbolic: relaxation sweeps per read-back

inline bool tr_chain_enabled() {
  const char* e = getenv("B200SP_SPTRSV_CHAIN");
  return !(e && e[0] == '0');
}

// one relaxation sweep: rows whose dependencies all had a level BEFORE this sweep get theirs; counts the rows resolved and flags
// entries on the wrong side of the diagonal
__global__ void __launch_bounds__(256) tr_level_sweep_kernel(int n, const int* __restrict__ rp, const int* __restrict__ ci, int lower,
                                                             int filter, const int* __restrict__ prev, int* __restrict__ cur,
                                                             int* __restrict__ resolved, int* __restrict__ bad,
                                                             int* __restrict__ max_level) {
  int mine = 0, top = -1;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    int lv = prev[i];
    if (lv < 0) {
      int mx = -1;
      bool ready = true;
      for (int k = rp[i]; k < rp[i + 1]; ++k) {
        const int c = ci[k];
        if (c == i) continue;
        if ((lower ? (c > i) : (c < i)) || c >= n) {
          // filter: the triangle of a general matrix is solved with (the Gauss-Seidel form), the other entries and the ghost
          // columns do not take part; otherwise the matrix must be triangular
          if (!filter) atomicMin(bad, i);
          continue;
        }
        const int lj = prev[c];
        if (lj < 0) {
          ready = false;
          break;
        }
        mx = lj > mx ? lj : mx;
      }
      if (ready) {
        lv = mx + 1;
        ++mine;
        top = lv > top ? lv : top;
      }
    }
    cur[i] = lv;
  }
  if (mine) {
    atomicAdd(resolved, mine);
    atomicMax(max_level, top);
  }
}

__global__ void __launch_bounds__(256) tr_fill_kernel(int n, int* __restrict__ a, int v) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) a[i] = v;
}
__global__ void __launch_bounds__(256) tr_hist_kernel(int n, const int* __restrict__ level, int* __restrict__ count) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) atomicAdd(&count[level[i]], 1);
}
// rows of one level, in whatever order the atomics hand out (the solve does not depend on it: a row reads only rows of lower levels)
__global__ void __launch_bounds__(256) tr_place_kernel(int n, const int* __restrict__ rp, const int* __restrict__ level,
                                                       int* __restrict__ cursor, int4* __restrict__ rows) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    rows[atomicAdd(&cursor[level[i]], 1)] = make_int4(i, rp[i], rp[i + 1], 0);
}

template <typename S>
__device__ __forceinline__ S tr_mul(S a, S b);
template <>
__device__ __forceinline__ double tr_mul<double>(double a, double b) { return __dmul_rn(a, b); }
template <>
__device__ __forceinline__ float tr_mul<float>(float a, float b) { return __fmul_rn(a, b); }
template <typename S>
__device__ __forceinline__ S tr_sub(S a, S b);
template <>
__device__ __forceinline__ double tr_sub<double>(double a, double b) { return __dsub_rn(a, b); }
template <>
__device__ __forceinline__ float tr_sub<float>(float a, float b) { return __fsub_rn(a, b); }

// one row of the substitution by a group of G lanes (gmask: the lanes of the group, gbase: its first lane in the warp)
// side: 0 = every off-diagonal entry takes part (a triangular matrix), 1 = only columns < i (the lower triangle of a general
// matrix), 2 = only columns in (i, n) (its upper triangle).  dinv: the caller's inverse diagonal or null.
template <typename S, int G>
__device__ __forceinline__ void tr_solve_row(int4 r, int lane, unsigned gmask, int gbase, int n, const int* __restrict__ ci,
                                             const S* __restrict__ v, const S* __restrict__ b, S* x, int side, const S* __restrict__ dinv) {
  const int i = r.x;
  S acc = b[i];
  S d = S(1);
  for (int base = r.y; base < r.z; base += G) {
    const int k = base + lane;
    const bool valid = k < r.z;
    const int c = valid ? ci[k] : -1;
    const S a = valid ? v[k] : S(0);
    const bool diag = valid && c == i;
    bool take = valid && !diag;
    if (side == 1 && c > i) take = false;
    if (side == 2 && (c < i || c >= n)) take = false;
    const S prod = take ? tr_mul(a, x[c]) : S(0);
    const unsigned tk = __ballot_sync(gmask, take) >> gbase;
    const unsigned dg = (__ballot_sync(gmask, diag) >> gbase) & (G == 32 ? 0xffffffffu : ((1u << (G & 31)) - 1u));
    const int cnt = min(G, r.z - base);
    for (int j = 0; j < cnt; ++j) {  // the serial part: the subtractions, in storage order
      const S pj = __shfl_sync(gmask, prod, j, G);
      if ((tk >> j) & 1u) acc = tr_sub(acc, pj);
    }
    if (dg) d = __shfl_sync(gmask, a, 31 - __clz(dg), G);  // the last diagonal entry of the batch, as the serial loop keeps it
  }
  // a caller-supplied INVERSE diagonal enters as the diagonal 1 / dinv_i (twostage_gauss_seidel_impl.hpp:446-456)
  if (lane == 0) x[i] = dinv ? acc / (S(1) / dinv[i]) : acc / d;
}

template <int G>
__device__ __forceinline__ unsigned tr_group_mask(int gbase) {
  return G == 32 ? 0xffffffffu : (((1u << (G & 31)) - 1u) << gbase);
}

// the rows of one level
template <typename S, int G>
__global__ void __launch_bounds__(256) tr_solve_level_kernel(int count, const int4* __restrict__ rows, int n, const int* __restrict__ ci,
                                                             const S* __restrict__ v, const S* __restrict__ b, S* x, int side,
                                                             const S* __restrict__ dinv) {
  const int lane = (int)threadIdx.x & (G - 1);
  const int gbase = ((int)threadIdx.x & 31) & ~(G - 1);
  const unsigned gmask = tr_group_mask<G>(gbase);
  const int groups = (int)(gridDim.x * blockDim.x) / G;
  for (int q = (int)(blockIdx.x * blockDim.x + threadIdx.x) / G; q < count; q += groups)
    tr_solve_row<S, G>(rows[q], lane, gmask, gbase, n, ci, v, b, x, side, dinv);
}

// levels [l0, l1), each of at most blockDim.x / G rows, by ONE CTA: the x written in a level is read by the next one after the CTA
// barrier (global writes of a CTA are visible to its own threads after __syncthreads)
template <typename S, int G>
__global__ void __launch_bounds__(TR_CHAIN_THREADS) tr_solve_chain_kernel(int l0, int l1, const int* __restrict__ level_ptr,
                                                                          const int4* __restrict__ rows, int n, const int* __restrict__ ci,
                                                                          const S* __restrict__ v, const S* __restrict__ b, S* x, int side,
                                                                          const S* __restrict__ dinv) {
  const int lane = (int)threadIdx.x & (G - 1);
  const int gbase = ((int)threadIdx.x & 31) & ~(G - 1);
  const unsigned gmask = tr_group_mask<G>(gbase);
  const int g = (int)threadIdx.x / G, groups = (int)blockDim.x / G;
  int q0 = level_ptr[l0];
  for (int l = l0; l < l1; ++l) {
    const int q1 = level_ptr[l + 1];
    for (int q = q0 + g; q < q1; q += groups) tr_solve_row<S, G>(rows[q], lane, gmask, gbase, n, ci, v, b, x, side, dinv);
    q0 = q1;
    __syncthreads();
  }
}

template <typename S, int G>
void tr_launch_solve(const b200sp_sptrsv_plan* p, cudaStream_t st, int n, const int* ci, const S* v, const S* b, S* x, const S* dinv) {
  const int side = p->filter ? (p->lower ? 1 : 2) : 0;
  for (const auto& sg : p->segments) {
    if (sg.chain) {
      tr_solve_chain_kernel<S, G><<<1, sg.threads, 0, st>>>(sg.l0, sg.l1, p->level_ptr_dev, p->level_rows, n, ci, v, b, x, side, dinv);
      continue;
    }
    const int q0 = p->level_ptr_host[sg.l0], cntl = p->level_ptr_host[sg.l1] - q0;
    if (cntl <= 0) continue;
    tr_solve_level_kernel<S, G><<<grid_for((int64_t)cntl * G), 256, 0, st>>>(cntl, p->level_rows + q0, n, ci, v, b, x, side, dinv);
  }
}

void tr_release(b200sp_sptrsv_plan* p, cudaStream_t st) {
  p->level_rows.release(st);
  p->level_ptr_dev.release(st);
  delete[] p->level_ptr_host;
  p->level_ptr_host = nullptr;
  p->segments.clear();
  p->n_levels = 0;
  p->symbolic = false;
}

}  // namespace

// used by gs2.cu as well (the classic form of the two-stage Gauss-Seidel)
int sptrsv_symbolic_impl(b200sp_sptrsv_plan* p, cudaStream_t st, int n, const int* rp, const int* ci, bool lower, bool filter) {
  tr_release(p, st);
  p->n = n;
  p->lower = lower;
  p->filter = filter;
  p->key_rp = rp;
  p->key_ci = ci;
  if (n == 0) {
    p->level_ptr_host = new (std::nothrow) int[1]{0};
    p->symbolic = true;
    return B200SP_OK;
  }
  DevTmp tmp(st);
  int *lv[2], *cnt;
  B200SP_CUDA_TRY(tmp.alloc(&lv[0], n));
  B200SP_CUDA_TRY(tmp.alloc(&lv[1], n));
  B200SP_CUDA_TRY(tmp.alloc(&cnt, 3));
  tr_fill_kernel<<<grid_for(n), 256, 0, st>>>(n, lv[0], -1);
  B200SP_LAUNCH_CHECK();
  int h[3] = {0, n, -1};  // rows resolved so far, smallest offending row, highest level handed out
  int nnz = 0;
  B200SP_CUDA_TRY(cudaMemcpyAsync(cnt, h, sizeof(h), cudaMemcpyHostToDevice, st));
  B200SP_CUDA_TRY(cudaMemcpyAsync(&nnz, rp + n, sizeof(int), cudaMemcpyDeviceToHost, st));
  B200SP_CUDA_TRY(cudaStreamSynchronize(st));
  // lanes per row: one batch covers the mean row (all its stored entries: the filtered form scans the other triangle too)
  const double mean = (double)nnz / (double)n;
  p->group = mean <= 8.0 ? 8 : (mean <= 20.0 ? 16 : 32);
  if (const char* e = getenv("B200SP_SPTRSV_GROUP")) {
    const int g = atoi(e);
    if (g == 8 || g == 16 || g == 32) p->group = g;
  }
  int cur = 0, done = 0;
  while (done < n) {
    // a sweep resolves exactly the rows of the next level; sweeps after the last one copy the levels unchanged
    for (int k = 0; k < TR_SWEEP_BATCH; ++k) {
      tr_level_sweep_kernel<<<grid_for(n), 256, 0, st>>>(n, rp, ci, lower ? 1 : 0, filter ? 1 : 0, lv[cur], lv[cur ^ 1], cnt, cnt + 1,
                                                           cnt + 2);
      B200SP_LAUNCH_CHECK();
      cur ^= 1;
    }
    B200SP_CUDA_TRY(cudaMemcpyAsync(h, cnt, sizeof(h), cudaMemcpyDeviceToHost, st));
    B200SP_CUDA_TRY(cudaStreamSynchronize(st));
    if (h[1] < n) {
      set_error("sptrsv_symbolic: row %d has an entry on the wrong side of the diagonal of a%s triangular matrix", h[1],
                lower ? " lower" : "n upper");
      return B200SP_ERR_INVALID_ARGUMENT;
    }
    if (h[0] == done) {  // no progress: impossible for a triangular matrix (kept as a guard against an endless loop)
      set_error("sptrsv_symbolic: the dependency graph has a cycle");
      return B200SP_ERR_INVALID_ARGUMENT;
    }
    done = h[0];
  }
  const int levels = h[2] + 1;
  // rows grouped by level
  int *count, *cursor;
  B200SP_CUDA_TRY(tmp.alloc(&count, levels + 1));
  B200SP_CUDA_TRY(tmp.alloc(&cursor, levels + 1));
  B200SP_CUDA_TRY(cudaMemsetAsync(count, 0, sizeof(int) * (size_t)(levels + 1), st));
  tr_hist_kernel<<<grid_for(n), 256, 0, st>>>(n, lv[cur], count);
  B200SP_LAUNCH_CHECK();
  p->level_ptr_host = new (std::nothrow) int[levels + 1];
  if (!p->level_ptr_host) {
    set_error("sptrsv_symbolic: out of host memory");
    return B200SP_ERR_ALLOC;
  }
  int* hc = new (std::nothrow) int[levels + 1];
  if (!hc) {
    set_error("sptrsv_symbolic: out of host memory");
    return B200SP_ERR_ALLOC;
  }
  cudaError_t ce = cudaMemcpyAsync(hc, count, sizeof(int) * (size_t)levels, cudaMemcpyDeviceToHost, st);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
  if (ce != cudaSuccess) {
    delete[] hc;
    set_error("sptrsv_symbolic: %s", cudaGetErrorString(ce));
    return B200SP_ERR_CUDA;
  }
  p->level_ptr_host[0] = 0;
  for (int l = 0; l < levels; ++l) p->level_ptr_host[l + 1] = p->level_ptr_host[l] + hc[l];
  delete[] hc;
  B200SP_CUDA_TRY(cudaMemcpyAsync(cursor, p->level_ptr_host, sizeof(int) * (size_t)(levels + 1), cudaMemcpyHostToDevice, st));
  B200SP_CUDA_TRY(p->level_rows.alloc((size_t)n, st));
  tr_place_kernel<<<grid_for(n), 256, 0, st>>>(n, rp, lv[cur], cursor, p->level_rows);
  B200SP_LAUNCH_CHECK();
  B200SP_CUDA_TRY(p->level_ptr_dev.alloc((size_t)(levels + 1), st));
  B200SP_CUDA_TRY(cudaMemcpyAsync(p->level_ptr_dev, p->level_ptr_host, sizeof(int) * (size_t)(levels + 1), cudaMemcpyHostToDevice, st));
  B200SP_CUDA_TRY(cudaStreamSynchronize(st));  // level_ptr_host was the source of asynchronous copies; tmp is released below
  // launch plan: runs of two or more consecutive small levels become one single-CTA launch
  const bool chain = tr_chain_enabled();
  const int small = TR_CHAIN_THREADS / p->group;
  for (int l = 0; l < levels;) {
    int e = l;
    while (chain && e < levels && p->level_ptr_host[e + 1] - p->level_ptr_host[e] <= small) ++e;
    if (e - l >= 2) {
      int widest = 1;
      for (int q = l; q < e; ++q) widest = std::max(widest, p->level_ptr_host[q + 1] - p->level_ptr_host[q]);
      p->segments.push_back({l, e, true, std::min(TR_CHAIN_THREADS, (widest * p->group + 31) / 32 * 32)});
      l = e;
    } else {
      p->segments.push_back({l, l + 1, false, 0});
      ++l;
    }
  }
  p->n_levels = levels;
  p->symbolic = true;
  return B200SP_OK;
}

template <typename S>
int sptrsv_solve_impl(b200sp_sptrsv_plan* p, cudaStream_t st, int n, const int* rp, const int* ci, const S* v, const S* b, S* x,
                      const S* dinv) {
  if (!p->symbolic || p->n != n || p->key_rp != rp || p->key_ci != ci) {
    set_error("sptrsv_solve: symbolic was not called on this plan with this matrix");
    return B200SP_ERR_STATE;
  }
  (void)rp;  // the row limits travel with the level lists
  switch (p->group) {
    case 8: tr_launch_solve<S, 8>(p, st, n, ci, v, b, x, dinv); break;
    case 16: tr_launch_solve<S, 16>(p, st, n, ci, v, b, x, dinv); break;
    default: tr_launch_solve<S, 32>(p, st, n, ci, v, b, x, dinv); break;
  }
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}
template int sptrsv_solve_impl<double>(b200sp_sptrsv_plan*, cudaStream_t, int, const int*, const int*, const double*, const double*, double*,
                                       const double*);
template int sptrsv_solve_impl<float>(b200sp_sptrsv_plan*, cudaStream_t, int, const int*, const int*, const float*, const float*, float*,
                                      const float*);

}  // namespace b200sp

extern "C" {

int b200sp_sptrsv_plan_create(b200sp_sptrsv_plan** plan) {
  B200SP_REQUIRE(plan != nullptr, "sptrsv_plan_create: null output pointer");
  b200sp_sptrsv_plan* p = new (std::nothrow) b200sp_sptrsv_plan();
  if (!p) {
    b200sp::set_error("sptrsv_plan_create: out of host memory");
    return B200SP_ERR_ALLOC;
  }
  b200sp::keep_async_pool_memory();
  *plan = p;
  return B200SP_OK;
}

int b200sp_sptrsv_plan_destroy(b200sp_sptrsv_plan* p, void* stream) {
  if (!p) return B200SP_OK;
  b200sp::tr_release(p, (cudaStream_t)stream);
  delete p;
  return B200SP_OK;
}

int b200sp_sptrsv_symbolic_i32(b200sp_sptrsv_plan* p, void* stream, int n, const int* row_ptr, const int* col_idx, int is_lower) {
  B200SP_REQUIRE(p != nullptr, "sptrsv_symbolic: null plan");
  B200SP_REQUIRE(n >= 0, "sptrsv_symbolic: negative dimension");
  B200SP_REQUIRE(n == 0 || (row_ptr && col_idx), "sptrsv_symbolic: null pointer argument");
  return b200sp::sptrsv_symbolic_impl(p, (cudaStream_t)stream, n, row_ptr, col_idx, is_lower != 0, false);
}

int b200sp_sptrsv_levels(const b200sp_sptrsv_plan* p) { return p ? p->n_levels : 0; }
int b200sp_sptrsv_launches(const b200sp_sptrsv_plan* p) { return p ? (int)p->segments.size() : 0; }

int b200sp_sptrsv_solve_f64_i32(b200sp_sptrsv_plan* p, void* stream, int n, const int* row_ptr, const int* col_idx, const double* vals,
                                const double* b, double* x) {
  B200SP_REQUIRE(p != nullptr, "sptrsv_solve: null plan");
  B200SP_REQUIRE(n == 0 || (vals && b && x), "sptrsv_solve: null pointer argument");
  return b200sp::sptrsv_solve_impl<double>(p, (cudaStream_t)stream, n, row_ptr, col_idx, vals, b, x, (const double*)nullptr);
}
int b200sp_sptrsv_solve_f32_i32(b200sp_sptrsv_plan* p, void* stream, int n, const int* row_ptr, const int* col_idx, const float* vals,
                                const float* b, float* x) {
  B200SP_REQUIRE(p != nullptr, "sptrsv_solve: null plan");
  B200SP_REQUIRE(n == 0 || (vals && b && x), "sptrsv_solve: null pointer argument");
  return b200sp::sptrsv_solve_impl<float>(p, (cudaStream_t)stream, n, row_ptr, col_idx, vals, b, x, (const float*)nullptr);
}

}  // extern "C"
