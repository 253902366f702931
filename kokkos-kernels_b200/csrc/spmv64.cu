// spmv64.cu -- SpMV on a CrsMatrix with 64-bit offsets (and 32- or 64-bit column indices): matrices past 2^31 entries.
//
// Replaces the (int64_t ordinal, size_t offset) instantiations of the reference's cuSPARSE SpMV slot
//   KOKKOSSPARSE_SPMV_CUSPARSE(double|float, int64_t, size_t, ...)   sparse/tpls/KokkosSparse_spmv_tpl_spec_decl.hpp:246-257
//   (availability: sparse/tpls/KokkosSparse_spmv_tpl_spec_avail.hpp:85-102)
// and also takes (int ordinal, 64-bit offset), which that slot cannot (":86 TODO: if Nvidia ever supports int/size_t").
//
// 180 GB of HBM3e hold about 15e9 fp64 entries with 32-bit columns: seven times what an int32 row map addresses.  A kernel
// that streamed the caller's 64-bit arrays would move 16 B per entry (8 B value + 8 B column) against the 12 B of the
// 32-bit path, i.e. run at 3/4 of its speed on an HBM-bound product.  So the 64-bit structure is read ONCE, at analysis:
//   * the rows are cut into windows of consecutive rows holding < 2^31 entries each (windows64.cuh);
//   * per window the plan keeps a 32-bit row map RELATIVE to the window's first (4-aligned) entry   -- 4 B per row;
//   * 64-bit columns are narrowed to 32 bits (the matrix must have < 2^31 columns)                  -- 4 B per entry,
//     32-bit columns are used where they lie (nothing copied);
//   * every product is then one launch sequence of the 32-bit kernels (spmv.cu: TMA-tiled kernel, long rows, self-tuning,
//     scatter kernel for the transposed modes) per window, on `values + base` and `columns + base`.
// Traffic per product: 12 B per entry (fp64), as for a 32-bit matrix; the results are those of the 32-bit path on each
// window, i.e. bit-identical to it on any matrix both can take.
#include <cstdlib>
#include <new>
#include <vector>

#include "common.cuh"
#include "windows64.cuh"

struct b200sp_spmv64_plan {
  int algo = 0;
  int64_t window_nnz = b200sp::kDefaultWindow;
  b200sp::PlanKey key;  // of the analysed matrix
  // analysis products: windows based on multiples of 4 entries (16-byte aligned bulk copies), one plan per window
  b200sp::RowWindows cut;
  std::vector<b200sp_spmv_plan*> plans;
  b200sp::DevArray<int> col32;  // narrowed columns (64-bit input only)
  char last_kernel[128] = "none";
};

namespace b200sp {
int spmv_lanes_per_row(int64_t m, int64_t nnz);  // spmv.cu
namespace {

void release(b200sp_spmv64_plan* p, cudaStream_t st) {
  for (b200sp_spmv_plan* pl : p->plans) b200sp_spmv_plan_destroy(pl, (void*)st);
  p->plans.clear();
  p->cut.release(st);
  p->col32.release(st);
  p->key = PlanKey();
}

int analyse(b200sp_spmv64_plan* p, cudaStream_t st, int64_t m, int64_t n, int64_t nnz, const int64_t* row_ptr,
            const void* col_idx, int col_bits) {
  const PlanKey key{row_ptr, col_idx, m, n, nnz, col_bits};
  if (p->key == key) return B200SP_OK;
  release(p, st);
  int64_t row = 0;
  int rc = cut_windows(st, m, row_ptr, nullptr, p->window_nnz, 4, &p->cut, &row);
  if (rc == kWindowRowOverLimit) {
    set_error("spmv (64-bit offsets): a row holds more than %lld entries (window limit)", (long long)p->window_nnz);
    return B200SP_ERR_OVERFLOW;
  }
  if (rc == kWindowsOverCap) {
    set_error("spmv (64-bit offsets): more than %d windows of %lld entries", kMaxWindows, (long long)p->window_nnz);
    return B200SP_ERR_OVERFLOW;
  }
  if (rc) return rc;
  if (col_bits == 64) {
    DevTmp tmp(st);
    int* d_bad = nullptr;
    int bad = 0;
    B200SP_CUDA_TRY(tmp.alloc(&d_bad, 1));
    B200SP_CUDA_TRY(cudaMemsetAsync(d_bad, 0, sizeof(int), st));
    B200SP_CUDA_TRY(p->col32.alloc((size_t)std::max<int64_t>(nnz, 1), st));
    win64_narrow_kernel<<<grid_for(nnz, 256, 16), 256, 0, st>>>(nnz, (const int64_t*)col_idx, p->col32, d_bad);
    B200SP_LAUNCH_CHECK();
    B200SP_CUDA_TRY(cudaMemcpyAsync(&bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost, st));
    B200SP_CUDA_TRY(cudaStreamSynchronize(st));
    if (bad) {
      release(p, st);
      set_error("spmv (64-bit columns): a column index does not fit 31 bits");
      return B200SP_ERR_OVERFLOW;
    }
  }
  p->plans.assign(p->cut.win.size(), nullptr);
  for (b200sp_spmv_plan*& pl : p->plans) {
    if ((rc = b200sp_spmv_plan_create(&pl, p->algo))) return rc;
    // lanes per row chosen once from the WHOLE matrix: the summation order of a row, hence the result, does not depend
    // on where the windows fall, and equals the 32-bit entry points' on a matrix both can take
    if ((rc = b200sp_spmv_plan_tune(pl, -1, spmv_lanes_per_row(m, nnz), -1))) return rc;
  }
  p->key = key;
  return B200SP_OK;
}

inline int call32(b200sp_spmv_plan* pl, void* st, char mode, int m, int n, int64_t nnz, double a, const int* rp, const int* ci,
                  const double* v, const double* x, double b, double* y) {
  return b200sp_spmv_f64_i32(pl, st, mode, m, n, nnz, a, rp, ci, v, x, b, y);
}
inline int call32(b200sp_spmv_plan* pl, void* st, char mode, int m, int n, int64_t nnz, float a, const int* rp, const int* ci,
                  const float* v, const float* x, float b, float* y) {
  return b200sp_spmv_f32_i32(pl, st, mode, m, n, nnz, a, rp, ci, v, x, b, y);
}

inline int call32mm(b200sp_spmv_plan* pl, void* st, char mode, int m, int n, int64_t nnz, int k, double a, const int* rp,
                    const int* ci, const double* v, const double* X, int64_t ldx, int xrm, double b, double* Y, int64_t ldy, int yrm) {
  return b200sp_spmm_f64_i32(pl, st, mode, m, n, nnz, k, a, rp, ci, v, X, ldx, xrm, b, Y, ldy, yrm);
}
inline int call32mm(b200sp_spmv_plan* pl, void* st, char mode, int m, int n, int64_t nnz, int k, float a, const int* rp,
                    const int* ci, const float* v, const float* X, int64_t ldx, int xrm, float b, float* Y, int64_t ldy, int yrm) {
  return b200sp_spmm_f32_i32(pl, st, mode, m, n, nnz, k, a, rp, ci, v, X, ldx, xrm, b, Y, ldy, yrm);
}

// rank 1 (k < 0) and rank 2 (k >= 0 columns) share the argument checks, the analysis and the loop over the windows
template <typename S>
int spmv64_impl(b200sp_spmv64_plan* p, void* stream, char mode, int64_t m, int64_t n, int64_t nnz, int k, S alpha,
                const int64_t* row_ptr, const void* col_idx, int col_bits, const S* vals, const S* x, int64_t ldx, int xrm,
                S beta, S* y, int64_t ldy, int yrm) {
  cudaStream_t st = (cudaStream_t)stream;
  const bool mv = k >= 0;
  B200SP_REQUIRE(p != nullptr, "spmv (64-bit offsets): a plan is required (it owns the 32-bit windows)");
  B200SP_REQUIRE(col_bits == 32 || col_bits == 64, "spmv (64-bit offsets): col_bits must be 32 or 64, got %d", col_bits);
  B200SP_REQUIRE(m >= 0 && n >= 0 && nnz >= 0, "spmv: negative dimension (m=%lld n=%lld nnz=%lld)", (long long)m,
                 (long long)n, (long long)nnz);
  if (m > INT32_MAX || n > INT32_MAX) {
    set_error("spmv (64-bit offsets): m=%lld / n=%lld: rows and columns must stay below 2^31 (only the offsets are 64-bit)",
              (long long)m, (long long)n);
    return B200SP_ERR_OVERFLOW;
  }
  bool trans;
  switch (mode) {
    case 'N': case 'n': case 'C': case 'c': trans = false; break;
    case 'T': case 't': case 'H': case 'h': trans = true; break;
    default:
      set_error("Invalid transpose mode %c for KokkosSparse::spmv()", mode);  // spmv_impl.hpp:537-541
      return B200SP_ERR_INVALID_ARGUMENT;
  }
  if (alpha == S(0) || m == 0 || n == 0 || nnz == 0) {  // y = beta*y, KokkosSparse_spmv.hpp:145-154
    snprintf(p->last_kernel, sizeof(p->last_kernel), "scale");
    if (mv) return call32mm(nullptr, stream, mode, (int)m, (int)n, 0, k, alpha, nullptr, nullptr, vals, x, ldx, xrm, beta, y, ldy, yrm);
    return call32(nullptr, stream, mode, (int)m, (int)n, 0, alpha, nullptr, nullptr, vals, x, beta, y);
  }
  B200SP_REQUIRE(row_ptr && col_idx && vals && x && y, "spmv: null pointer argument");
  int rc = analyse(p, st, m, n, nnz, row_ptr, col_idx, col_bits);
  if (rc) return rc;
  const int* cols = col_bits == 64 ? p->col32 : (const int*)col_idx;
  // row r of X / Y starts r*ld elements in when the rows are contiguous (LayoutRight), r elements in otherwise
  const int64_t xstep = mv ? (xrm ? ldx : 1) : 1, ystep = mv ? (yrm ? ldy : 1) : 1;
  const size_t nw = p->cut.win.size();
  for (size_t i = 0; i < nw; ++i) {
    const RowWindow& w = p->cut.win[i];
    const int wm = w.r1 - w.r0;
    const int64_t w_nnz = w.end - w.base;  // the window's entries counted from its base = its relative row map's last value
    const int* rp = p->cut.rel + w.rel_off;
    const S* xw = trans ? x + w.r0 * xstep : x;  // T / H: the window's rows of x, all of y (accumulated window by window)
    S* yw = trans ? y : y + w.r0 * ystep;        // N / C: all of x, the window's rows of y
    const S bw = (trans && i > 0) ? S(1) : beta;
    const char md = trans ? 'T' : 'N';
    b200sp_spmv_plan* pl = p->plans[i];
    if (mv) rc = call32mm(pl, stream, md, wm, (int)n, w_nnz, k, alpha, rp, cols + w.base, vals + w.base, xw, ldx, xrm, bw, yw, ldy, yrm);
    else rc = call32(pl, stream, md, wm, (int)n, w_nnz, alpha, rp, cols + w.base, vals + w.base, xw, bw, yw);
    if (rc) return rc;
  }
  snprintf(p->last_kernel, sizeof(p->last_kernel), "%d window%s x %.90s", (int)nw, nw == 1 ? "" : "s",
           nw == 0 ? "none" : b200sp_spmv_last_kernel(p->plans[0]));
  return B200SP_OK;
}

}  // namespace
}  // namespace b200sp

extern "C" {

int b200sp_spmv64_plan_create(b200sp_spmv64_plan** plan, int algo) {
  B200SP_REQUIRE(plan != nullptr, "spmv64_plan_create: null output pointer");
  B200SP_REQUIRE(algo >= 0 && algo <= 2, "spmv64_plan_create: unknown algorithm %d", algo);
  b200sp_spmv64_plan* p = new (std::nothrow) b200sp_spmv64_plan();
  if (!p) {
    b200sp::set_error("spmv64_plan_create: out of host memory");
    return B200SP_ERR_ALLOC;
  }
  p->algo = algo;
  *plan = p;
  return B200SP_OK;
}

int b200sp_spmv64_plan_destroy(b200sp_spmv64_plan* p, void* stream) {
  if (!p) return B200SP_OK;
  b200sp::release(p, (cudaStream_t)stream);
  delete p;
  return B200SP_OK;
}

int b200sp_spmv64_plan_set_window(b200sp_spmv64_plan* p, int64_t max_entries) {
  B200SP_REQUIRE(p != nullptr, "spmv64_plan_set_window: null plan");
  if (int rc = b200sp::check_window_limit("spmv64_plan_set_window", max_entries)) return rc;
  p->window_nnz = max_entries;
  p->key = b200sp::PlanKey();  // next call analyses again
  return B200SP_OK;
}

int b200sp_spmv64_plan_windows(const b200sp_spmv64_plan* p) { return p ? (int)p->cut.win.size() : 0; }
const char* b200sp_spmv64_last_kernel(const b200sp_spmv64_plan* p) { return p ? p->last_kernel : "none"; }

int b200sp_spmv_f64_i64(b200sp_spmv64_plan* plan, void* stream, char mode, int64_t m, int64_t n, int64_t nnz, double alpha,
                        const int64_t* row_ptr, const void* col_idx, int col_bits, const double* vals, const double* x,
                        double beta, double* y) {
  return b200sp::spmv64_impl<double>(plan, stream, mode, m, n, nnz, -1, alpha, row_ptr, col_idx, col_bits, vals, x, 0, 0, beta, y, 0, 0);
}

int b200sp_spmv_f32_i64(b200sp_spmv64_plan* plan, void* stream, char mode, int64_t m, int64_t n, int64_t nnz, float alpha,
                        const int64_t* row_ptr, const void* col_idx, int col_bits, const float* vals, const float* x,
                        float beta, float* y) {
  return b200sp::spmv64_impl<float>(plan, stream, mode, m, n, nnz, -1, alpha, row_ptr, col_idx, col_bits, vals, x, 0, 0, beta, y, 0, 0);
}

int b200sp_spmm_f64_i64(b200sp_spmv64_plan* plan, void* stream, char mode, int64_t m, int64_t n, int64_t nnz, int k, double alpha,
                        const int64_t* row_ptr, const void* col_idx, int col_bits, const double* vals, const double* X,
                        int64_t ldx, int x_row_major, double beta, double* Y, int64_t ldy, int y_row_major) {
  B200SP_REQUIRE(k >= 0, "spmm: negative number of columns %d", k);
  return b200sp::spmv64_impl<double>(plan, stream, mode, m, n, nnz, k, alpha, row_ptr, col_idx, col_bits, vals, X, ldx, x_row_major,
                                     beta, Y, ldy, y_row_major);
}

int b200sp_spmm_f32_i64(b200sp_spmv64_plan* plan, void* stream, char mode, int64_t m, int64_t n, int64_t nnz, int k, float alpha,
                        const int64_t* row_ptr, const void* col_idx, int col_bits, const float* vals, const float* X,
                        int64_t ldx, int x_row_major, float beta, float* Y, int64_t ldy, int y_row_major) {
  B200SP_REQUIRE(k >= 0, "spmm: negative number of columns %d", k);
  return b200sp::spmv64_impl<float>(plan, stream, mode, m, n, nnz, k, alpha, row_ptr, col_idx, col_bits, vals, X, ldx, x_row_major,
                                    beta, Y, ldy, y_row_major);
}

}  // extern "C"
