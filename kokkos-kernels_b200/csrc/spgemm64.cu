// spgemm64.cu -- SpGEMM C = A*B on CrsMatrix data with 64-bit offsets and 32-bit ordinals: products past 2^31 entries.
//
// Replaces the (int ordinal, size_t offset) instantiations of the SPGEMM_SYMBOLIC / SPGEMM_NUMERIC legs, Kokkos' default
// offset type in a Trilinos build (cmake/kokkoskernels_eti_offsets.cmake:1-11).  The cuSPARSE slot cannot take them (it
// requires 32-bit offsets and ordinals, sparse/tpls/KokkosSparse_spgemm_numeric_tpl_spec_avail.hpp:38-41), so the reference
// runs them on the native KokkosSPGEMM.
//
// C is the array that outgrows int32 first.  Every row of C is computed on its own, so the rows can be cut into windows
// that each fit 32-bit offsets and run through the 32-bit entry points (spgemm.cu), on the row windows of spmv64.cu
// (windows64.cuh):
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
#include "windows64.cuh"

namespace b200sp {

struct Spgemm64State {
  int64_t window = kDefaultWindow;  // products / entries of A per window
  bool done = false;  // a 64-bit symbolic completed on this plan
  int m = 0, n = 0, k = 0;
  const void *rpA = nullptr, *ciA = nullptr, *rpB = nullptr, *ciB = nullptr;
  int64_t c_nnz = 0;
  int c_max = 0;
  RowWindows cut;                           // windows of A's rows, bases not rounded; cut.rel: relative row maps of A
  std::vector<int64_t> c_base;              // per window: row_ptr_C[r0]
  std::vector<b200sp_spgemm_plan*> plans;   // per window: the 32-bit product
  DevArray<int> rel_c;  // relative row maps of C, laid out as cut.rel (4 B per row)
  DevArray<int> rp_b;   // B's row map narrowed to int32 (4 B per row)
};

namespace {

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

// frees the windows, their child plans and the narrowed arrays; keeps the window limit
void release_windows(Spgemm64State* s, cudaStream_t st) {
  for (b200sp_spgemm_plan* pl : s->plans) b200sp_spgemm_plan_destroy(pl, (void*)st);
  s->plans.clear();
  s->c_base.clear();
  s->cut.release(st);
  s->rel_c.release(st);
  s->rp_b.release(st);
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
    B200SP_CUDA_TRY(cudaMemsetAsync(rpC, 0, sizeof(int64_t) * ((size_t)m + 1), st));
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
  int *prod, *block_max, *d_max;
  int64_t* P;
  long long *block_sum, *d_total;
  const int nblocks = scan_blocks(m);
  B200SP_CUDA_TRY(tmp.alloc(&prod, m));
  B200SP_CUDA_TRY(tmp.alloc(&P, (size_t)m + 1));
  B200SP_CUDA_TRY(tmp.alloc(&block_sum, nblocks));
  B200SP_CUDA_TRY(tmp.alloc(&block_max, nblocks));
  B200SP_CUDA_TRY(tmp.alloc(&d_total, 1));
  B200SP_CUDA_TRY(tmp.alloc(&d_max, 1));
  B200SP_CUDA_TRY(s->rp_b.alloc((size_t)n + 1, st));
  win64_narrow_kernel<<<grid_for((int64_t)n + 1), 256, 0, st>>>((int64_t)n + 1, rpB, s->rp_b, nullptr);
  B200SP_LAUNCH_CHECK();
  s64g_products_kernel<<<(unsigned)(((int64_t)m * 8 + 255) / 256), 256, 0, st>>>(m, rpA, ciA, s->rp_b, prod);
  B200SP_LAUNCH_CHECK();
  if (int rc = launch_exclusive_scan64<int>(st, m, prod, P, block_sum, block_max, d_total, d_max)) return rc;
  int64_t row = 0;
  const int rc = cut_windows(st, m, rpA, P, s->window, 1, &s->cut, &row);
  if (rc == kWindowRowOverLimit) {
    release_windows(s, st);
    set_error("spgemm_symbolic (64-bit offsets): row %lld holds more than %lld entries or products (window limit)",
              (long long)row, (long long)s->window);
    return B200SP_ERR_OVERFLOW;
  }
  if (rc == kWindowsOverCap) {
    release_windows(s, st);
    set_error("spgemm_symbolic (64-bit offsets): more than %d windows of %lld products", kMaxWindows, (long long)s->window);
    return B200SP_ERR_OVERFLOW;
  }
  if (rc) return rc;
  B200SP_CUDA_TRY(s->rel_c.alloc((size_t)s->cut.rel_size, st));
  int64_t c_base = 0;
  int c_max = 0;
  for (const RowWindow& x : s->cut.win) {
    const int wm = x.r1 - x.r0;
    const int64_t count = (int64_t)wm + 1;
    s->plans.push_back(nullptr);
    if (int rc = b200sp_spgemm_plan_create(&s->plans.back())) return rc;
    int64_t w_nnz = 0;
    int w_max = 0;
    if (int rc = b200sp_spgemm_symbolic_i32(s->plans.back(), (void*)st, wm, n, k, s->cut.rel + x.rel_off, ciA + x.base, s->rp_b,
                                            ciB, s->rel_c + x.rel_off, &w_nnz, &w_max))
      return rc;
    s->c_base.push_back(c_base);
    win64_widen_kernel<<<grid_for(count), 256, 0, st>>>(x.r0, count, c_base, s->rel_c + x.rel_off, rpC);
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
  for (size_t w = 0; w < s->cut.win.size(); ++w) {
    const RowWindow& x = s->cut.win[w];
    if (int rc = call32(s->plans[w], stream, x.r1 - x.r0, n, k, s->cut.rel + x.rel_off, ciA + x.base, vA + x.base, s->rp_b, ciB,
                        vB, s->rel_c + x.rel_off, ciC + s->c_base[w], vC + s->c_base[w]))
      return rc;
  }
  return B200SP_OK;
}

}  // namespace

bool spgemm64_holds_product(const Spgemm64State* s) { return s && s->done; }

int spgemm64_window_count(const Spgemm64State* s) { return s ? (int)s->plans.size() : 0; }

const b200sp_spgemm_plan* spgemm64_window_plan(const Spgemm64State* s, int w) { return s->plans[(size_t)w]; }

void spgemm64_state_free(Spgemm64State* s, cudaStream_t st) {
  if (!s) return;
  release_windows(s, st);
  delete s;
}

}  // namespace b200sp

extern "C" {

int b200sp_spgemm_plan_set_window(b200sp_spgemm_plan* plan, int64_t max_entries) {
  B200SP_REQUIRE(plan != nullptr, "spgemm_plan_set_window: null plan");
  if (int rc = b200sp::check_window_limit("spgemm_plan_set_window", max_entries)) return rc;
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
  return s ? (int)s->cut.win.size() : 0;
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
