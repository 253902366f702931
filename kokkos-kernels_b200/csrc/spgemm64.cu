// spgemm64.cu -- SpGEMM C = A*B on CrsMatrix data with 64-bit offsets and 32-bit ordinals: products past 2^31 entries.
//
// Replaces the (int ordinal, size_t offset) instantiations of the SPGEMM_SYMBOLIC / SPGEMM_NUMERIC legs, Kokkos' default
// offset type in a Trilinos build (cmake/kokkoskernels_eti_offsets.cmake:1-11).  The cuSPARSE slot cannot take them (it
// requires 32-bit offsets and ordinals, sparse/tpls/KokkosSparse_spgemm_numeric_tpl_spec_avail.hpp:38-41), so the reference
// runs them on the native KokkosSPGEMM.
//
// C is the array that outgrows int32 first.  Every row of C is computed on its own, so the rows can be cut into windows
// that each fit 32-bit offsets and run through the 32-bit entry points (spgemm.cu), as spmv64.cu does for SpMV:
//   * B's row map is narrowed to int32 once (nnz(B) must stay within 2^31 - 65537: every window reads all of B);
//   * per row of A: its entries and its products sum_{j in A_i} len(B_{col_j}), scanned into int64 prefixes;
//   * windows of consecutive rows with at most `limit` products and at most `limit` entries of A -- the products bound
//     makes a window's nnz(C) fit int32 before anything is counted, so symbolic and numeric share one cut;
//   * per window a 32-bit row map of A relative to the window's first entry, a child b200sp_spgemm_plan that runs the
//     32-bit symbolic on it and keeps the window's relative C row map, which is widened into the caller's row_ptr_C.
// Numeric runs the 32-bit numeric per window on `col_idx + base`, `vals + base` of A and C.  The kernels read and write
// those arrays element by element (vector accesses are to shared memory only), so the bases need no rounding.  Every row
// runs the kernel the 32-bit path runs it on: same structure, and the same value bits wherever those are deterministic
// (rows of at most 8192 products; longer rows are summed with atomics by the hash kernels).
#include <algorithm>
#include <new>
#include <vector>

#include "common.cuh"
#include "scan.cuh"
#include "bspgemm.cuh"

namespace {
constexpr int kMaxWindows = 4096;
constexpr int64_t kDefaultWindow = (int64_t)INT32_MAX - 65536;  // products / entries per window, as spmv64.cu

struct Window {
  int r0 = 0, r1 = 0;      // rows [r0, r1)
  int64_t a_base = 0;      // row_ptr_A[r0]
  int64_t c_base = 0;      // row_ptr_C[r0]
  int64_t c_nnz = 0;       // entries of C in the window
  int64_t rel_off = 0;     // offset of the window's relative row maps (r1 - r0 + 1 entries) in rel_a / rel_c
  b200sp_spgemm_plan* plan = nullptr;
};
}  // namespace

namespace b200sp {

struct Spgemm64State {
  int64_t window = kDefaultWindow;
  bool done = false;  // a 64-bit symbolic completed on this plan
  int m = 0, n = 0, k = 0;
  const void *rpA = nullptr, *ciA = nullptr, *rpB = nullptr, *ciB = nullptr;
  int64_t c_nnz = 0;
  int c_max = 0;
  std::vector<Window> win;
  int* rel_a = nullptr;  // device: relative row maps of A, all windows (4 B per row)
  int* rel_c = nullptr;  // device: relative row maps of C, all windows (4 B per row)
  int* rp_b = nullptr;   // device: B's row map narrowed to int32 (4 B per row)
};

namespace {

__global__ void __launch_bounds__(256) s64g_fill_kernel(int64_t n, int64_t* __restrict__ p) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = 0;
}

__global__ void __launch_bounds__(256) s64g_narrow_kernel(int64_t n, const int64_t* __restrict__ in, int* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = (int)in[i];
}

// products per row of A, 8 lanes per row; a row past INT_MAX products is clamped (it exceeds every window limit)
__global__ void __launch_bounds__(256) s64g_products_kernel(int m, const int64_t* __restrict__ rpA, const int* __restrict__ ciA,
                                                            const int* __restrict__ rpB, int* __restrict__ prod) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int r = (int)(t >> 3), sl = (int)(t & 7);
  long long f = 0;
  if (r < m)
    for (int64_t j = rpA[r] + sl; j < rpA[r + 1]; j += 8) {
      const int c = ciA[j];
      f += rpB[c + 1] - rpB[c];
    }
#pragma unroll
  for (int o = 4; o > 0; o >>= 1) f += __shfl_xor_sync(0xffffffffu, f, o);
  if (r < m && sl == 0) prod[r] = (int)min(f, (long long)INT_MAX);
}

// One thread, one binary search per window over the prefixes P (products) and rpA (entries): window k starts at row R_k
// and ends at the largest R' with P[R'] - P[R_k] <= limit and rpA[R'] - rpA[R_k] <= limit.  out[3k .. 3k+2] = (R_k,
// R_{k+1}, rpA[R_k]); *n_out = windows, -1 when one row alone exceeds the limit (out[0] = that row), -2 when there are more
// than max_windows.
__global__ void s64g_windows_kernel(int64_t m, const int64_t* __restrict__ P, const int64_t* __restrict__ rpA, int64_t limit,
                                    int max_windows, int64_t* __restrict__ out, int* __restrict__ n_out) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  int k = 0;
  int64_t R = 0;
  while (R < m) {
    const int64_t ptop = P[R] + limit, atop = rpA[R] + limit;
    int64_t lo = R, hi = m;
    while (lo < hi) {
      const int64_t mid = lo + ((hi - lo + 1) >> 1);
      if (P[mid] <= ptop && rpA[mid] <= atop) lo = mid;
      else hi = mid - 1;
    }
    if (lo == R) {
      *n_out = -1;
      out[0] = R;
      return;
    }
    if (k == max_windows) {
      *n_out = -2;
      return;
    }
    out[3 * k] = R;
    out[3 * k + 1] = lo;
    out[3 * k + 2] = rpA[R];
    ++k;
    R = lo;
  }
  *n_out = k;
}

__global__ void __launch_bounds__(256) s64g_relative_kernel(int64_t r0, int64_t count, int64_t base, const int64_t* __restrict__ rp,
                                                            int* __restrict__ rel) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
    rel[i] = (int)(rp[r0 + i] - base);
}

__global__ void __launch_bounds__(256) s64g_widen_kernel(int64_t r0, int64_t count, int64_t base, const int* __restrict__ rel,
                                                         int64_t* __restrict__ rp) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
    rp[r0 + i] = base + rel[i];
}

inline int grid_for(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)sm_count() * 8)); }

// frees the windows, their child plans and the narrowed arrays; keeps the window limit
void release_windows(Spgemm64State* s, cudaStream_t st) {
  for (Window& w : s->win)
    if (w.plan) b200sp_spgemm_plan_destroy(w.plan, (void*)st);
  s->win.clear();
  void* ptrs[] = {s->rel_a, s->rel_c, s->rp_b};
  for (void* q : ptrs)
    if (q) cudaFreeAsync(q, st);
  s->rel_a = s->rel_c = s->rp_b = nullptr;
  s->done = false;
  s->c_nnz = 0;
  s->c_max = 0;
}

Spgemm64State* state_of(b200sp_spgemm_plan* p, bool create) {
  Spgemm64State** slot = spgemm_plan_view(p).s64;
  if (!*slot && create) *slot = new (std::nothrow) Spgemm64State();
  return *slot;
}

int symbolic64(b200sp_spgemm_plan* p, cudaStream_t st, int m, int n, int k, const int64_t* rpA, const int* ciA,
               const int64_t* rpB, const int* ciB, int64_t* rpC, int64_t* c_nnz, int* c_max_row_nnz) {
  B200SP_REQUIRE(p != nullptr, "spgemm_symbolic (64-bit offsets): null plan");
  B200SP_REQUIRE(m >= 0 && n >= 0 && k >= 0, "spgemm_symbolic: negative dimension");
  B200SP_REQUIRE(rpC != nullptr, "spgemm_symbolic: row_ptr_C is null");
  if (spgemm_plan_view(p).symbolic_done) {
    set_error("spgemm_symbolic (64-bit offsets): handle was already used for a product with 32-bit offsets; create a new handle");
    return B200SP_ERR_STATE;
  }
  Spgemm64State* s = state_of(p, true);
  if (!s) {
    set_error("spgemm_symbolic (64-bit offsets): out of host memory");
    return B200SP_ERR_ALLOC;
  }
  // one handle, one product (spgemm_handle.hpp:706-746); the same product again is analysed again
  if (s->done && (s->m != m || s->n != n || s->k != k || s->rpA != rpA || s->ciA != ciA || s->rpB != rpB || s->ciB != ciB)) {
    set_error("spgemm_symbolic: handle was already used for a different product; create a new handle");
    return B200SP_ERR_STATE;
  }
  release_windows(s, st);
  s->m = m; s->n = n; s->k = k;
  s->rpA = rpA; s->ciA = ciA; s->rpB = rpB; s->ciB = ciB;

  int64_t nnzA = 0, nnzB = 0;
  if (m > 0) {
    B200SP_REQUIRE(rpA != nullptr, "spgemm_symbolic: row_ptr_A is null");
    B200SP_CUDA_TRY(cudaMemcpyAsync(&nnzA, rpA + m, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    B200SP_CUDA_TRY(cudaStreamSynchronize(st));
  }
  if (n > 0 && nnzA > 0) {
    B200SP_REQUIRE(rpB != nullptr, "spgemm_symbolic: row_ptr_B is null");
    B200SP_CUDA_TRY(cudaMemcpyAsync(&nnzB, rpB + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    B200SP_CUDA_TRY(cudaStreamSynchronize(st));
  }
  // degenerate shapes: zero row_ptr, c_nnz = 0, no windows (symbolic_spec.hpp:101-107)
  if (m == 0 || n == 0 || k == 0 || nnzA == 0 || nnzB == 0) {
    s64g_fill_kernel<<<grid_for((int64_t)m + 1), 256, 0, st>>>((int64_t)m + 1, rpC);
    B200SP_LAUNCH_CHECK();
    B200SP_CUDA_TRY(cudaStreamSynchronize(st));
    s->done = true;
    if (c_nnz) *c_nnz = 0;
    if (c_max_row_nnz) *c_max_row_nnz = 0;
    return B200SP_OK;
  }
  // B is read whole by every window through 32-bit offsets: the default limit, whatever set_window chose for A's rows
  if (nnzB > kDefaultWindow) {
    set_error("spgemm_symbolic (64-bit offsets): nnz(B) = %lld exceeds %lld entries (every window reads all of B through "
              "32-bit offsets)", (long long)nnzB, (long long)kDefaultWindow);
    return B200SP_ERR_OVERFLOW;
  }
  B200SP_REQUIRE(ciA && ciB, "spgemm_symbolic: null column index array");

  DevTmp tmp(st);
  int *prod, *block_max, *d_max, *d_n;
  int64_t *P, *d_win;
  long long *block_sum, *d_total;
  const int nblocks = scan_blocks(m);
  B200SP_CUDA_TRY(tmp.alloc(&prod, m));
  B200SP_CUDA_TRY(tmp.alloc(&P, (size_t)m + 1));
  B200SP_CUDA_TRY(tmp.alloc(&block_sum, nblocks));
  B200SP_CUDA_TRY(tmp.alloc(&block_max, nblocks));
  B200SP_CUDA_TRY(tmp.alloc(&d_total, 1));
  B200SP_CUDA_TRY(tmp.alloc(&d_max, 1));
  B200SP_CUDA_TRY(tmp.alloc(&d_win, (size_t)3 * kMaxWindows));
  B200SP_CUDA_TRY(tmp.alloc(&d_n, 1));
  B200SP_CUDA_TRY(cudaMallocAsync((void**)&s->rp_b, sizeof(int) * ((size_t)n + 1), st));
  s64g_narrow_kernel<<<grid_for((int64_t)n + 1), 256, 0, st>>>((int64_t)n + 1, rpB, s->rp_b);
  B200SP_LAUNCH_CHECK();
  s64g_products_kernel<<<(unsigned)(((int64_t)m * 8 + 255) / 256), 256, 0, st>>>(m, rpA, ciA, s->rp_b, prod);
  B200SP_LAUNCH_CHECK();
  if (int rc = launch_exclusive_scan64<int>(st, m, prod, P, block_sum, block_max, d_total, d_max)) return rc;
  s64g_windows_kernel<<<1, 32, 0, st>>>(m, P, rpA, s->window, kMaxWindows, d_win, d_n);
  B200SP_LAUNCH_CHECK();
  int nw = 0;
  B200SP_CUDA_TRY(cudaMemcpyAsync(&nw, d_n, sizeof(int), cudaMemcpyDeviceToHost, st));
  B200SP_CUDA_TRY(cudaStreamSynchronize(st));
  if (nw == -1) {
    int64_t row = 0;
    B200SP_CUDA_TRY(cudaMemcpyAsync(&row, d_win, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    B200SP_CUDA_TRY(cudaStreamSynchronize(st));
    release_windows(s, st);
    set_error("spgemm_symbolic (64-bit offsets): row %lld holds more than %lld entries or products (window limit)",
              (long long)row, (long long)s->window);
    return B200SP_ERR_OVERFLOW;
  }
  if (nw == -2) {
    release_windows(s, st);
    set_error("spgemm_symbolic (64-bit offsets): more than %d windows of %lld products", kMaxWindows, (long long)s->window);
    return B200SP_ERR_OVERFLOW;
  }
  std::vector<int64_t> h_win((size_t)3 * nw);
  B200SP_CUDA_TRY(cudaMemcpyAsync(h_win.data(), d_win, sizeof(int64_t) * 3 * (size_t)nw, cudaMemcpyDeviceToHost, st));
  B200SP_CUDA_TRY(cudaStreamSynchronize(st));
  s->win.resize((size_t)nw);
  int64_t total = 0;
  for (int w = 0; w < nw; ++w) {
    Window& x = s->win[(size_t)w];
    x.r0 = (int)h_win[3 * (size_t)w];
    x.r1 = (int)h_win[3 * (size_t)w + 1];
    x.a_base = h_win[3 * (size_t)w + 2];
    x.rel_off = total;
    total += (int64_t)(x.r1 - x.r0) + 1;
  }
  B200SP_CUDA_TRY(cudaMallocAsync((void**)&s->rel_a, sizeof(int) * (size_t)total, st));
  B200SP_CUDA_TRY(cudaMallocAsync((void**)&s->rel_c, sizeof(int) * (size_t)total, st));
  int64_t c_base = 0;
  int c_max = 0;
  for (Window& x : s->win) {
    const int wm = x.r1 - x.r0;
    const int64_t count = (int64_t)wm + 1;
    s64g_relative_kernel<<<grid_for(count), 256, 0, st>>>(x.r0, count, x.a_base, rpA, s->rel_a + x.rel_off);
    B200SP_LAUNCH_CHECK();
    if (int rc = b200sp_spgemm_plan_create(&x.plan)) return rc;
    int64_t w_nnz = 0;
    int w_max = 0;
    if (int rc = b200sp_spgemm_symbolic_i32(x.plan, (void*)st, wm, n, k, s->rel_a + x.rel_off, ciA + x.a_base, s->rp_b, ciB,
                                            s->rel_c + x.rel_off, &w_nnz, &w_max))
      return rc;
    x.c_base = c_base;
    x.c_nnz = w_nnz;
    s64g_widen_kernel<<<grid_for(count), 256, 0, st>>>(x.r0, count, c_base, s->rel_c + x.rel_off, rpC);
    B200SP_LAUNCH_CHECK();
    c_base += w_nnz;
    c_max = std::max(c_max, w_max);
  }
  B200SP_CUDA_TRY(cudaStreamSynchronize(st));
  s->c_nnz = c_base;
  s->c_max = c_max;
  s->done = true;
  if (c_nnz) *c_nnz = c_base;
  if (c_max_row_nnz) *c_max_row_nnz = c_max;
  return B200SP_OK;
}

inline int call32(b200sp_spgemm_plan* pl, void* st, int m, int n, int k, const int* rA, const int* cA, const double* vA,
                  const int* rB, const int* cB, const double* vB, const int* rC, int* cC, double* vC) {
  return b200sp_spgemm_numeric_f64_i32(pl, st, m, n, k, rA, cA, vA, rB, cB, vB, rC, cC, vC);
}
inline int call32(b200sp_spgemm_plan* pl, void* st, int m, int n, int k, const int* rA, const int* cA, const float* vA,
                  const int* rB, const int* cB, const float* vB, const int* rC, int* cC, float* vC) {
  return b200sp_spgemm_numeric_f32_i32(pl, st, m, n, k, rA, cA, vA, rB, cB, vB, rC, cC, vC);
}

template <typename S>
int numeric64(b200sp_spgemm_plan* p, void* stream, int m, int n, int k, const int64_t* rpA, const int* ciA, const S* vA,
              const int64_t* rpB, const int* ciB, const S* vB, const int64_t* rpC, int* ciC, S* vC) {
  B200SP_REQUIRE(p != nullptr, "spgemm_numeric: null plan");
  const Spgemm64State* s = state_of(p, false);
  if (!s || !s->done) {
    set_error(spgemm_plan_view(p).symbolic_done
                  ? "spgemm_numeric (64-bit offsets): the symbolic phase on this handle had 32-bit offsets"
                  : "Call spgemm symbolic before spgemm numeric");
    return B200SP_ERR_STATE;
  }
  if (s->m != m || s->n != n || s->k != k) {
    set_error("spgemm_numeric: dimensions (%d,%d,%d) differ from symbolic (%d,%d,%d)", m, n, k, s->m, s->n, s->k);
    return B200SP_ERR_STATE;
  }
  if (m == 0 || s->c_nnz == 0) return B200SP_OK;
  B200SP_REQUIRE(rpA && ciA && vA && rpB && ciB && vB && rpC && ciC && vC, "spgemm_numeric: null pointer argument");
  // the windows' relative row maps stand for rpA / rpB / rpC, which symbolic has read
  for (const Window& x : s->win) {
    if (int rc = call32(x.plan, stream, x.r1 - x.r0, n, k, s->rel_a + x.rel_off, ciA + x.a_base, vA + x.a_base, s->rp_b, ciB, vB,
                        s->rel_c + x.rel_off, ciC + x.c_base, vC + x.c_base))
      return rc;
  }
  return B200SP_OK;
}

}  // namespace

bool spgemm64_holds_product(const Spgemm64State* s) { return s && s->done; }

void spgemm64_state_free(Spgemm64State* s, cudaStream_t st) {
  if (!s) return;
  release_windows(s, st);
  delete s;
}

}  // namespace b200sp

extern "C" {

int b200sp_spgemm_plan_set_window(b200sp_spgemm_plan* plan, int64_t max_entries) {
  B200SP_REQUIRE(plan != nullptr, "spgemm_plan_set_window: null plan");
  B200SP_REQUIRE(max_entries >= 8 && max_entries <= kDefaultWindow, "spgemm_plan_set_window: %lld not in [8, %lld]",
                 (long long)max_entries, (long long)kDefaultWindow);
  b200sp::Spgemm64State* s = b200sp::state_of(plan, true);
  if (!s) {
    b200sp::set_error("spgemm_plan_set_window: out of host memory");
    return B200SP_ERR_ALLOC;
  }
  s->window = max_entries;  // the next 64-bit symbolic cuts by it
  return B200SP_OK;
}

int b200sp_spgemm_plan_windows(const b200sp_spgemm_plan* plan) {
  if (!plan) return 0;
  const b200sp::Spgemm64State* s = b200sp::state_of(const_cast<b200sp_spgemm_plan*>(plan), false);
  return s ? (int)s->win.size() : 0;
}

int b200sp_spgemm_symbolic_i64(b200sp_spgemm_plan* plan, void* stream, int m, int n, int k, const int64_t* row_ptr_A,
                               const int* col_idx_A, const int64_t* row_ptr_B, const int* col_idx_B, int64_t* row_ptr_C,
                               int64_t* c_nnz, int* c_max_row_nnz) {
  return b200sp::symbolic64(plan, (cudaStream_t)stream, m, n, k, row_ptr_A, col_idx_A, row_ptr_B, col_idx_B, row_ptr_C, c_nnz,
                            c_max_row_nnz);
}

int b200sp_spgemm_numeric_f64_i64(b200sp_spgemm_plan* plan, void* stream, int m, int n, int k, const int64_t* row_ptr_A,
                                  const int* col_idx_A, const double* vals_A, const int64_t* row_ptr_B, const int* col_idx_B,
                                  const double* vals_B, const int64_t* row_ptr_C, int* col_idx_C, double* vals_C) {
  return b200sp::numeric64<double>(plan, stream, m, n, k, row_ptr_A, col_idx_A, vals_A, row_ptr_B, col_idx_B, vals_B, row_ptr_C,
                                   col_idx_C, vals_C);
}

int b200sp_spgemm_numeric_f32_i64(b200sp_spgemm_plan* plan, void* stream, int m, int n, int k, const int64_t* row_ptr_A,
                                  const int* col_idx_A, const float* vals_A, const int64_t* row_ptr_B, const int* col_idx_B,
                                  const float* vals_B, const int64_t* row_ptr_C, int* col_idx_C, float* vals_C) {
  return b200sp::numeric64<float>(plan, stream, m, n, k, row_ptr_A, col_idx_A, vals_A, row_ptr_B, col_idx_B, vals_B, row_ptr_C,
                                  col_idx_C, vals_C);
}

}  // extern "C"
