// gpu_check.cpp -- torch-free GPU validation + timing harness for libb200sparse (TEST INFRASTRUCTURE).
//
// Why: a fresh GPU box spends about a minute importing torch before the first test runs; this binary
// starts in milliseconds, so a short gpurun slot is enough to check new kernels against the oracle and
// to A/B-time kernel variants.  It links the product library (C ABI), the host matrix generators and
// the oracle (the checker -- never the thing measured).  Each suite runs in a forked child so that a
// faulting kernel cannot take the other suites down; every check appends one JSON line to --out.
//
//   gpu_check [--out FILE] [--suite NAME]... [--big]      suites: spgemm crs spgemm_c4 crs_big spmm spmv_t spmm_sweep jacobi spmv_longrows bsr cg solvers spmv64
//
// Exit code: number of failed suites.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <signal.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/wait.h>
#include <unistd.h>
#include <algorithm>
#include <chrono>
#include <cmath>
#include <functional>
#include <limits>
#include <numeric>
#include <string>
#include <vector>

#include "b200sparse.h"

extern "C" {
// oracle (oracle/kk_oracle.c, oracle/kk_oracle_crs.c)
int64_t okk_spgemm_symbolic(int m, int k, const int* rmA, const int* entA, const int* rmB, const int* entB, int* rmC);
void okk_spgemm_numeric_f64(int m, int k, const int* rmA, const int* entA, const double* valA, const int* rmB,
                            const int* entB, const double* valB, const int* rmC, int* entC, double* valC);
void okk_spgemm_numeric_f32(int m, int k, const int* rmA, const int* entA, const float* valA, const int* rmB,
                            const int* entB, const float* valB, const int* rmC, int* entC, float* valC);
void okk_sort_crs_f64(int m, const int* rm, int* ent, double* val);
void okk_sort_crs_f32(int m, const int* rm, int* ent, float* val);
void okk_sort_crs_stable_f64(int m, const int* rm, int* ent, double* val);
void okk_sort_crs_stable_f32(int m, const int* rm, int* ent, float* val);
int64_t okk_merged_rowmap(int m, const int* rm, const int* ent, int* rm_out);
void okk_merged_entries_f64(int m, const int* rm, const int* ent, const double* val, const int* rm_out, int* ent_out,
                            double* val_out);
void okk_merged_entries_f32(int m, const int* rm, const int* ent, const float* val, const int* rm_out, int* ent_out,
                            float* val_out);
int64_t okk_spadd_sorted_symbolic(int m, const int* rmA, const int* entA, const int* rmB, const int* entB, int* rmC);
void okk_spadd_sorted_numeric_f64(int m, const int* rmA, const int* entA, const double* valA, double alpha, const int* rmB,
                                  const int* entB, const double* valB, double beta, const int* rmC, int* entC, double* valC);
void okk_spadd_sorted_numeric_f32(int m, const int* rmA, const int* entA, const float* valA, float alpha, const int* rmB,
                                  const int* entB, const float* valB, float beta, const int* rmC, int* entC, float* valC);
int64_t okk_spadd_unsorted_symbolic(int m, const int* rmA, const int* entA, const int* rmB, const int* entB, int* rmC,
                                    int* apos, int* bpos);
void okk_spadd_unsorted_numeric_f64(int m, const int* rmA, const int* entA, const double* valA, double alpha,
                                    const int* rmB, const int* entB, const double* valB, double beta, const int* rmC,
                                    int* entC, double* valC, const int* apos, const int* bpos);
void okk_spadd_unsorted_numeric_f32(int m, const int* rmA, const int* entA, const float* valA, float alpha,
                                    const int* rmB, const int* entB, const float* valB, float beta, const int* rmC,
                                    int* entC, float* valC, const int* apos, const int* bpos);
void okk_transpose_f64(int nrow, int ncol, const int* rm, const int* ent, const double* val, int* trm, int* tent,
                       double* tval);
void okk_spmv_mv_f64(int nrow, int ncol, int nvec, const int* rm, const int* ci, const double* v, const double* X,
                     int64_t xr, int64_t xc, double* Y, int64_t yr, int64_t yc, double alpha, double beta, int threads);
void okk_spmv_mv_f32(int nrow, int ncol, int nvec, const int* rm, const int* ci, const float* v, const float* X,
                     int64_t xr, int64_t xc, float* Y, int64_t yr, int64_t yc, float alpha, float beta, int threads);
void okk_spmv_serial_f64(int nrow, const int* rm, const int* ci, const double* v, const double* x, double* y, double alpha,
                         double beta);
void okk_spmv_transpose_f64(int nrow, int ncol, const int* rm, const int* ci, const double* v, const double* x, double* y,
                            double alpha, double beta);
void okk_spgemm_jacobi_f64(int m, int k, const int* rmA, const int* entA, const double* valA, const int* rmB, const int* entB,
                           const double* valB, const int* rmC, int* entC, double* valC, double omega, const double* dinv);
void okk_bsr_spmv_v42_f64(int mb, int bs, int nvec, const int* rm, const int* ent, const double* val, const double* X, int64_t xr,
                          int64_t xc, double* Y, int64_t yr, int64_t yc, double alpha, double beta);
void okk_bsr_spmv_v41_f64(char mode, int mb, int ylen_b, int bs, int nvec, const int* rm, const int* ent, const double* val,
                          const double* X, int64_t xr, int64_t xc, double* Y, int64_t yr, int64_t yc, double alpha, double beta);
int okk_cg_f64(int n, const int* rm, const int* ci, const double* v, const double* b, double* x, int maximum_iteration, double tolerance,
               double* norm_res_out);
int okk_pcg_f64(int n, const int* rm, const int* ci, const double* v, const double* b, double* x, int maximum_iteration, double tolerance,
                double* norm_res_out, int ncolors, const int* color_ptr, const int* color_rows, const double* dinv);
int okk_pcg_gs2_f64(int n, const int* row_map, const int* col_idx, const double* values, const double* b, double* x, int maximum_iteration,
                    double tolerance, double* norm_res_out, int inner_sweeps, int compact);
int okk_gs2_apply_f64(int n, int ncols, const int* rm, const int* ci, const double* v, const double* given_inverse_diagonal, int compact,
                      int inner_sweeps, int outer_sweeps, double gamma, double* x, const double* b, int init_zero_x, double omega, int num_iter,
                      int direction);
void okk_gs_apply_f64(int n, const int* rm, const int* ci, const double* v, int ncolors, const int* color_ptr, const int* color_rows,
                      const double* dinv, const double* y, double* x, int init_zero_x, double omega, int sweeps, int direction);
int okk_gmres_f64(int n, const int* rm, const int* ci, const double* v, const int* prm, const int* pci, const double* pv, const double* B,
                  double* X, int m, double tol, int max_restart, int ortho, int* num_iters_out, double* end_rel_res_out, int* conv_flag_out);
int okk_num_threads(void);
// host generators (kokkos-kernels_b200/csrc/matgen.c)
void b200gen_fill_f64(int64_t n, double* v, double lo, double hi, uint64_t seed);
void b200gen_fill_f32(int64_t n, float* v, float lo, float hi, uint64_t seed);
int64_t b200gen_kk_rowptr(int nrows, int ncols, int64_t nnz_target, int row_size_variance, int* rowptr);
void b200gen_kk_colidx(int nrows, int ncols, int64_t nnz_target, int row_size_variance, int bandwidth, const int* rowptr,
                       int* colind);
int64_t b200gen_lap27_rows(int nx, int ny, int nz, int ndof, int64_t row_begin, int64_t row_end, int* rowptr, int* colidx,
                           double* vals, double noise, uint64_t seed);
void b200gen_uniform(int nrows, int ncols, int deg, uint64_t seed, int* rowptr, int* colidx);
void* b200gen_rmat_build(int scale, int edge_factor, double a, double b, double c, uint64_t seed, int64_t* nnz_out);
void b200gen_rmat_emit(void* h, int* rowptr, int* colidx);
}

// ------------------------------------------------------------------------------------------------
static std::string g_out = "gpurun_out/gpu_check.jsonl";
static const char* g_suite = "";
static int g_fail = 0;
static bool g_big = false;
static bool g_dry = false;  // --dry: no CUDA at all (device buffers live in host memory, C-ABI calls are skipped): exercises the
                            // generators, the oracle calls and the comparison code on a machine without a GPU

static double now_s() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

static void record(const char* name, bool ok, const char* fmt, ...) {
  char detail[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(detail, sizeof(detail), fmt, ap);
  va_end(ap);
  for (char* c = detail; *c; ++c)
    if (*c == '"' || *c == '\\' || *c == '\n') *c = ' ';
  FILE* f = fopen(g_out.c_str(), "a");
  if (f) {
    fprintf(f, "{\"suite\": \"%s\", \"check\": \"%s\", \"ok\": %s, \"detail\": \"%s\"}\n", g_suite, name, ok ? "true" : "false", detail);
    fclose(f);
  }
  fprintf(stderr, "[%s] %-44s %s  %s\n", g_suite, name, ok ? "ok  " : "FAIL", detail);
  if (!ok) ++g_fail;
}

#define CK(expr)                                                                                   \
  do {                                                                                             \
    if (g_dry) break;                                                                              \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess) {                                                                       \
      record("cuda", false, "%s -> %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      exit(3);                                                                                     \
    }                                                                                              \
  } while (0)
#define SP(expr)                                                                                    \
  do {                                                                                              \
    if (g_dry) break;                                                                               \
    int _rc = (expr);                                                                               \
    if (_rc != 0) {                                                                                 \
      record("cabi", false, "%s -> status %d: %s (%s:%d)", #expr, _rc, b200sp_last_error_string(), __FILE__, __LINE__); \
      exit(4);                                                                                      \
    }                                                                                               \
  } while (0)

template <typename T>
struct Dev {
  T* p = nullptr;
  size_t n = 0;
  Dev() {}
  explicit Dev(size_t count) { alloc(count); }
  explicit Dev(const std::vector<T>& h) {
    alloc(h.size());
    if (n && g_dry) memcpy(p, h.data(), n * sizeof(T));
    if (n) CK(cudaMemcpy(p, h.data(), n * sizeof(T), cudaMemcpyHostToDevice));
  }
  Dev(const Dev&) = delete;
  Dev& operator=(const Dev&) = delete;
  ~Dev() { release(); }
  void release() {
    if (p && g_dry) free(p);
    else if (p) cudaFree(p);
    p = nullptr;
  }
  void alloc(size_t count) {
    release();
    n = count;
    if (g_dry) p = (T*)calloc(std::max<size_t>(count, 1), sizeof(T));
    CK(cudaMalloc((void**)&p, std::max<size_t>(count, 1) * sizeof(T)));
  }
  void fill_bytes(int byte) {
    if (g_dry) memset(p, byte, std::max<size_t>(n, 1) * sizeof(T));
    CK(cudaMemset(p, byte, std::max<size_t>(n, 1) * sizeof(T)));
  }
  std::vector<T> host() const { return host(0, n); }
  std::vector<T> host(size_t off, size_t count) const {
    std::vector<T> h(count);
    if (count && g_dry) memcpy(h.data(), p + off, count * sizeof(T));
    if (count) CK(cudaMemcpy(h.data(), p + off, count * sizeof(T), cudaMemcpyDeviceToHost));
    return h;
  }
};

struct Rng {
  uint64_t s;
  explicit Rng(uint64_t seed) : s(seed * 0x9E3779B97F4A7C15ull + 0x1234567ull) {}
  uint64_t next() {
    s += 0x9E3779B97F4A7C15ull;
    uint64_t x = s;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
  }
  int below(int n) { return (int)(next() % (uint64_t)std::max(n, 1)); }
  double u01() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
};

template <typename S>
struct Csr {
  int m = 0, n = 0;
  std::vector<int> rp, ci;
  std::vector<S> v;
  int64_t nnz() const { return (int64_t)ci.size(); }
};

template <typename S>
static void fill_vals(std::vector<S>& v, double lo, double hi, uint64_t seed) {
  Rng r(seed);
  for (auto& x : v) x = (S)(lo + (hi - lo) * r.u01());
}

// kk_generate_sparse_matrix structure (unsorted rows, no duplicates)
template <typename S>
static Csr<S> gen_kk(int m, int n, int64_t nnz, int var, int bw, uint64_t seed) {
  Csr<S> A;
  A.m = m;
  A.n = n;
  A.rp.assign(m + 1, 0);
  const int64_t got = b200gen_kk_rowptr(m, n, nnz, var, A.rp.data());
  A.ci.resize(got);
  b200gen_kk_colidx(m, n, nnz, var, bw, A.rp.data(), A.ci.data());
  A.v.resize(got);
  fill_vals(A.v, 1.0, 50.0, seed);
  return A;
}

// arbitrary row lengths, columns uniform in [0, n) -- duplicates allowed unless `distinct`
template <typename S>
static Csr<S> gen_rows(const std::vector<int>& lens, int n, bool distinct, bool sorted, uint64_t seed) {
  Csr<S> A;
  A.m = (int)lens.size();
  A.n = n;
  A.rp.assign(A.m + 1, 0);
  for (int i = 0; i < A.m; ++i) A.rp[i + 1] = A.rp[i] + lens[i];
  A.ci.resize(A.rp[A.m]);
  Rng r(seed);
  std::vector<char> used;
  if (distinct) used.assign(n, 0);
  for (int i = 0; i < A.m; ++i) {
    int* c = A.ci.data() + A.rp[i];
    for (int j = 0; j < lens[i]; ++j) {
      int col;
      do col = r.below(n);
      while (distinct && used[col]);
      if (distinct) used[col] = 1;
      c[j] = col;
    }
    if (distinct)
      for (int j = 0; j < lens[i]; ++j) used[c[j]] = 0;
    if (sorted) std::sort(c, c + lens[i]);
  }
  A.v.resize(A.ci.size());
  fill_vals(A.v, 1.0, 50.0, seed + 17);
  return A;
}

template <typename S>
static Csr<S> gen_lap27(int g, int ndof) {
  Csr<S> A;
  A.m = A.n = g * g * g * ndof;
  A.rp.assign(A.m + 1, 0);
  const int64_t nnz = b200gen_lap27_rows(g, g, g, ndof, 0, A.m, A.rp.data(), nullptr, nullptr, 0.0, 0);
  A.ci.resize(nnz);
  std::vector<double> v(nnz);
  b200gen_lap27_rows(g, g, g, ndof, 0, A.m, A.rp.data(), A.ci.data(), v.data(), 0.5, 7);
  A.v.resize(nnz);
  for (int64_t i = 0; i < nnz; ++i) A.v[i] = (S)(std::fabs(v[i]) + 1.0);
  return A;
}

template <typename S>
static Csr<S> gen_uniform(int m, int n, int deg, uint64_t seed) {
  Csr<S> A;
  A.m = m;
  A.n = n;
  A.rp.resize(m + 1);
  A.ci.resize((size_t)m * deg);
  b200gen_uniform(m, n, deg, seed, A.rp.data(), A.ci.data());
  A.v.resize(A.ci.size());
  if (sizeof(S) == 8) b200gen_fill_f64((int64_t)A.v.size(), (double*)A.v.data(), 1.0, 50.0, seed);
  else b200gen_fill_f32((int64_t)A.v.size(), (float*)A.v.data(), 1.0f, 50.0f, seed);
  return A;
}

template <typename S>
static int64_t rel_mismatch(const std::vector<S>& a, const std::vector<S>& b, double eps) {
  // is_same_matrix value law (Test_Sparse_Utils.hpp:86-118)
  int64_t bad = 0;
  for (size_t i = 0; i < a.size(); ++i) {
    const double x = a[i], y = b[i], ax = std::fabs(x), ay = std::fabs(y);
    if (ax <= eps && ay <= eps) continue;
    if (!(std::fabs(x - y) / (ax + ay) <= eps)) ++bad;
  }
  return bad;
}

template <typename T>
static int64_t count_diff(const std::vector<T>& a, const std::vector<T>& b) {
  if (a.size() != b.size()) return -1;
  int64_t d = 0;
  for (size_t i = 0; i < a.size(); ++i) d += (memcmp(&a[i], &b[i], sizeof(T)) != 0);
  return d;
}

struct Timer {
  cudaEvent_t a, b;
  Timer() {
    CK(cudaEventCreate(&a));
    CK(cudaEventCreate(&b));
  }
  ~Timer() {
    if (g_dry) return;
    cudaEventDestroy(a);
    cudaEventDestroy(b);
  }
  void start() { CK(cudaEventRecord(a, 0)); }
  float stop_ms() {
    if (g_dry) return 1.0f;
    CK(cudaEventRecord(b, 0));
    CK(cudaEventSynchronize(b));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, a, b));
    return ms;
  }
};

// ------------------------------------------------------------------------------------------------
// suite: spgemm -- numeric variants 1/2/3 against the oracle (row_ptr / col_idx exact, values by the law)
// ------------------------------------------------------------------------------------------------
template <typename S>
struct OracleSpgemm {
  std::vector<int> rp, ci;
  std::vector<S> v;
};
static void oracle_numeric(int m, int k, const Csr<double>& A, const Csr<double>& B, const std::vector<int>& rp,
                           std::vector<int>& ci, std::vector<double>& v) {
  okk_spgemm_numeric_f64(m, k, A.rp.data(), A.ci.data(), A.v.data(), B.rp.data(), B.ci.data(), B.v.data(), rp.data(), ci.data(), v.data());
  okk_sort_crs_f64(m, rp.data(), ci.data(), v.data());
}
static void oracle_numeric(int m, int k, const Csr<float>& A, const Csr<float>& B, const std::vector<int>& rp,
                           std::vector<int>& ci, std::vector<float>& v) {
  okk_spgemm_numeric_f32(m, k, A.rp.data(), A.ci.data(), A.v.data(), B.rp.data(), B.ci.data(), B.v.data(), rp.data(), ci.data(), v.data());
  okk_sort_crs_f32(m, rp.data(), ci.data(), v.data());
}
static int numeric_call(b200sp_spgemm_plan* p, int m, int n, int k, const int* rpA, const int* ciA, const double* vA,
                        const int* rpB, const int* ciB, const double* vB, const int* rpC, int* ciC, double* vC) {
  return b200sp_spgemm_numeric_f64_i32(p, nullptr, m, n, k, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC);
}
static int numeric_call(b200sp_spgemm_plan* p, int m, int n, int k, const int* rpA, const int* ciA, const float* vA,
                        const int* rpB, const int* ciB, const float* vB, const int* rpC, int* ciC, float* vC) {
  return b200sp_spgemm_numeric_f32_i32(p, nullptr, m, n, k, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC);
}

template <typename S>
static void spgemm_case(const char* name, const Csr<S>& A, const Csr<S>& B) {
  const int m = A.m, n = A.n, k = B.n;
  OracleSpgemm<S> o;
  o.rp.assign(m + 1, 0);
  const int64_t onnz = okk_spgemm_symbolic(m, k, A.rp.data(), A.ci.data(), B.rp.data(), B.ci.data(), o.rp.data());
  o.ci.resize(onnz);
  o.v.resize(onnz);
  oracle_numeric(m, k, A, B, o.rp, o.ci, o.v);
  Dev<int> rpA(A.rp), ciA(A.ci), rpB(B.rp), ciB(B.ci), rpC((size_t)m + 1);
  Dev<S> vA(A.v), vB(B.v);
  rpC.fill_bytes(0x7b);
  b200sp_spgemm_plan* plan = nullptr;
  SP(b200sp_spgemm_plan_create(&plan));
  int64_t c_nnz = -1;
  int c_max = -1;
  SP(b200sp_spgemm_symbolic_i32(plan, nullptr, m, n, k, rpA.p, ciA.p, rpB.p, ciB.p, rpC.p, &c_nnz, &c_max));
  char nm[128];
  snprintf(nm, sizeof(nm), "%s/symbolic", name);
  const bool sym_ok = c_nnz == onnz && count_diff(rpC.host(), o.rp) == 0;
  record(nm, sym_ok, "m=%d nnzA=%lld c_nnz=%lld (oracle %lld) c_max=%d", m, (long long)A.nnz(), (long long)c_nnz, (long long)onnz, c_max);
  if (!sym_ok) {
    b200sp_spgemm_plan_destroy(plan, nullptr);
    return;
  }
  const double eps = sizeof(S) == 8 ? 1e-7 : 3.7e-3;
  for (int variant = 1; variant <= 6; ++variant) {
    char ev[8];
    snprintf(ev, sizeof(ev), "%d", variant);
    setenv("B200SP_SPGEMM_NUMERIC", ev, 1);
    Dev<int> ciC((size_t)c_nnz);
    Dev<S> vC((size_t)c_nnz);
    ciC.fill_bytes(0xff);
    vC.fill_bytes(0xff);
    Timer t;
    t.start();
    SP(numeric_call(plan, m, n, k, rpA.p, ciA.p, vA.p, rpB.p, ciB.p, vB.p, rpC.p, ciC.p, vC.p));
    const float ms = t.stop_ms();
    CK(cudaDeviceSynchronize());
    const int64_t dci = count_diff(ciC.host(), o.ci);
    const int64_t dv = rel_mismatch(vC.host(), o.v, eps);
    snprintf(nm, sizeof(nm), "%s/numeric_v%d", name, variant);
    record(nm, dci == 0 && dv == 0, "col_idx diffs=%lld value law violations=%lld of %lld, %.3f ms", (long long)dci, (long long)dv,
           (long long)c_nnz, ms);
  }
  unsetenv("B200SP_SPGEMM_NUMERIC");
  b200sp_spgemm_plan_destroy(plan, nullptr);
  {  // symbolic variant 2 (finer bins, tables of 2x the flop bound): same row map
    setenv("B200SP_SPGEMM_SYMBOLIC", "2", 1);
    b200sp_spgemm_plan* p2 = nullptr;
    SP(b200sp_spgemm_plan_create(&p2));
    Dev<int> rpC2((size_t)m + 1);
    rpC2.fill_bytes(0x7b);
    int64_t c2 = -1;
    int cm2 = -1;
    SP(b200sp_spgemm_symbolic_i32(p2, nullptr, m, n, k, rpA.p, ciA.p, rpB.p, ciB.p, rpC2.p, &c2, &cm2));
    snprintf(nm, sizeof(nm), "%s/symbolic_v2", name);
    record(nm, c2 == onnz && cm2 == c_max && count_diff(rpC2.host(), o.rp) == 0, "c_nnz=%lld c_max=%d", (long long)c2, cm2);
    b200sp_spgemm_plan_destroy(p2, nullptr);
    unsetenv("B200SP_SPGEMM_SYMBOLIC");
  }
}

static void suite_spgemm() {
  {
    auto A = gen_kk<double>(10000, 8000, 160000, 10, 500, 1), B = gen_kk<double>(8000, 6000, 160000, 10, 500, 2);
    okk_sort_crs_f64(A.m, A.rp.data(), A.ci.data(), A.v.data());
    okk_sort_crs_f64(B.m, B.rp.data(), B.ci.data(), B.v.data());
    spgemm_case("kk_10000x8000x6000_f64", A, B);
  }
  {
    auto A = gen_kk<float>(1000, 500, 20000, 10, 500, 1), B = gen_kk<float>(500, 1600, 20000, 10, 500, 2);
    spgemm_case("kk_unsorted_1000x500x1600_f32", A, B);
  }
  {
    Rng r(3);
    std::vector<int> lens(20000);
    for (auto& l : lens) l = r.below(12);
    lens[0] = 6000;
    lens[1] = 1200;
    lens[2] = 400;
    auto A = gen_rows<double>(lens, 20000, true, false, 3);
    spgemm_case("wide_rows_unsorted_20000_f64", A, A);
  }
  {
    auto A = gen_lap27<double>(12, 2);
    spgemm_case("lap27_12x2dof_dense_accumulator_f64", A, A);
  }
  {
    auto A = gen_uniform<double>(60000, 60000, 32, 4);
    spgemm_case("uniform32_60000_f64", A, A);
  }
  {
    auto A = gen_uniform<float>(40000, 40000, 32, 5);
    spgemm_case("uniform32_40000_f32", A, A);
  }
  {
    // duplicate columns inside rows of A and B (legal input: products just accumulate)
    Rng r(9);
    std::vector<int> lens(5000);
    for (auto& l : lens) l = r.below(20);
    auto A = gen_rows<double>(lens, 300, false, false, 11);
    auto B = gen_rows<double>(std::vector<int>(300, 9), 700, false, false, 12);
    spgemm_case("duplicate_entries_5000x300x700_f64", A, B);
  }
  {
    // medium rows: nnz(C_i) in the 64..4096 bins with products beyond the parking capacity
    Rng r(21);
    std::vector<int> lens(3000);
    for (auto& l : lens) l = 20 + r.below(100);
    auto A = gen_rows<double>(lens, 3000, true, true, 21);
    spgemm_case("medium_rows_3000_f64", A, A);
  }
}

// ------------------------------------------------------------------------------------------------
// suite: spgemm_c4 -- BASELINE.json config 4 timing of the numeric variants (+ sampled-row parity)
// ------------------------------------------------------------------------------------------------
static void suite_spgemm_c4() {
  const int n = g_big ? 2000000 : 500000, deg = 32;
  double t0 = now_s();
  auto A = gen_uniform<double>(n, n, deg, 4);
  record("generate", true, "n=%d deg=%d in %.1f s", n, deg, now_s() - t0);
  Dev<int> rp(A.rp), ci(A.ci), rpC((size_t)n + 1);
  Dev<double> v(A.v);
  b200sp_spgemm_plan* plan = nullptr;
  SP(b200sp_spgemm_plan_create(&plan));
  int64_t c_nnz = 0;
  int c_max = 0;
  t0 = now_s();
  SP(b200sp_spgemm_symbolic_i32(plan, nullptr, n, n, n, rp.p, ci.p, rp.p, ci.p, rpC.p, &c_nnz, &c_max));
  const double sym_s = now_s() - t0;
  record("symbolic", c_nnz > 0, "c_nnz=%lld c_max=%d wall %.2f ms (first call, includes allocation)", (long long)c_nnz, c_max, sym_s * 1e3);
  for (int sv = 1; sv <= 2; ++sv) {  // warm timings of the symbolic phase (wall clock: it synchronises by nature)
    char ev[8];
    snprintf(ev, sizeof(ev), "%d", sv);
    setenv("B200SP_SPGEMM_SYMBOLIC", ev, 1);
    double best = 1e30;
    int64_t cn = 0;
    for (int rep = 0; rep < 3; ++rep) {
      b200sp_spgemm_plan* p2 = nullptr;
      SP(b200sp_spgemm_plan_create(&p2));
      Dev<int> rpC2((size_t)n + 1);
      CK(cudaDeviceSynchronize());
      const double t1 = now_s();
      SP(b200sp_spgemm_symbolic_i32(p2, nullptr, n, n, n, rp.p, ci.p, rp.p, ci.p, rpC2.p, &cn, &c_max));
      best = std::min(best, now_s() - t1);
      b200sp_spgemm_plan_destroy(p2, nullptr);
    }
    char nm[64];
    snprintf(nm, sizeof(nm), "symbolic_v%d_warm", sv);
    record(nm, cn == c_nnz, "%.3f ms best of 3 (wall clock incl. its host synchronisations), c_nnz=%lld", best * 1e3, (long long)cn);
  }
  unsetenv("B200SP_SPGEMM_SYMBOLIC");
  Dev<int> ciC((size_t)c_nnz);
  Dev<double> vC((size_t)c_nnz);
  const double flops = (double)n * deg * deg;
  const double balg = 12.0 * 2 * A.nnz() + 4.0 * 3 * (n + 1) + 12.0 * (double)c_nnz;
  std::vector<int> hrpC = rpC.host();
  Rng r(0);
  for (int variant = 1; variant <= 6; ++variant) {
    char ev[8];
    snprintf(ev, sizeof(ev), "%d", variant);
    setenv("B200SP_SPGEMM_NUMERIC", ev, 1);
    float best = 1e30f;
    for (int rep = 0; rep < 3; ++rep) {
      Timer t;
      t.start();
      SP(b200sp_spgemm_numeric_f64_i32(plan, nullptr, n, n, n, rp.p, ci.p, v.p, rp.p, ci.p, v.p, rpC.p, ciC.p, vC.p));
      best = std::min(best, t.stop_ms());
    }
    // sampled rows against a host Gustavson product
    int bad = 0;
    for (int s = 0; s < 200; ++s) {
      const int row = r.below(n);
      std::vector<std::pair<int, double>> acc;
      for (int a = A.rp[row]; a < A.rp[row + 1]; ++a) {
        const int j = A.ci[a];
        for (int b = A.rp[j]; b < A.rp[j + 1]; ++b) acc.emplace_back(A.ci[b], A.v[b] * A.v[a]);
      }
      std::stable_sort(acc.begin(), acc.end(), [](auto& x, auto& y) { return x.first < y.first; });
      std::vector<int> ec;
      std::vector<double> evv;
      for (auto& pr : acc) {
        if (!ec.empty() && ec.back() == pr.first) evv.back() += pr.second;
        else {
          ec.push_back(pr.first);
          evv.push_back(pr.second);
        }
      }
      const int s0 = hrpC[row], s1 = hrpC[row + 1];
      if ((int)ec.size() != s1 - s0) {
        ++bad;
        continue;
      }
      auto gc = ciC.host(s0, s1 - s0);
      auto gv = vC.host(s0, s1 - s0);
      if (count_diff(gc, ec) != 0 || rel_mismatch(gv, evv, 1e-7) != 0) ++bad;
    }
    char nm[64];
    snprintf(nm, sizeof(nm), "numeric_v%d", variant);
    record(nm, bad == 0, "%.3f ms best of 3, %.1f GFLOP/s, %.0f GB/s algorithmic, sampled rows bad=%d", best,
           2.0 * flops / (best * 1e-3) / 1e9, balg / (best * 1e-3) / 1e9, bad);
  }
  unsetenv("B200SP_SPGEMM_NUMERIC");
  b200sp_spgemm_plan_destroy(plan, nullptr);
}

// ------------------------------------------------------------------------------------------------
// suite: crs -- sort / sort_and_merge / transpose / spadd, every output array bit-identical to the oracle
// ------------------------------------------------------------------------------------------------
static int sort_call(int m, const int* rp, int* ci, double* v) { return b200sp_sort_crs_f64_i32(nullptr, m, rp, ci, v); }
static int sort_call(int m, const int* rp, int* ci, float* v) { return b200sp_sort_crs_f32_i32(nullptr, m, rp, ci, v); }
static void osort(int m, const int* rp, int* ci, double* v) { okk_sort_crs_stable_f64(m, rp, ci, v); }
static void osort(int m, const int* rp, int* ci, float* v) { okk_sort_crs_stable_f32(m, rp, ci, v); }

template <typename S>
static void sort_case(const char* name, Csr<S> A) {
  Dev<int> rp(A.rp), ci(A.ci), g(A.ci);
  Dev<S> v(A.v);
  Timer t;
  t.start();
  SP(sort_call(A.m, rp.p, ci.p, v.p));
  const float ms = t.stop_ms();
  SP(b200sp_sort_crs_graph_i32(nullptr, A.m, rp.p, g.p));
  CK(cudaDeviceSynchronize());
  osort(A.m, A.rp.data(), A.ci.data(), A.v.data());
  const int64_t d1 = count_diff(ci.host(), A.ci), d2 = count_diff(v.host(), A.v), d3 = count_diff(g.host(), A.ci);
  // second call: already sorted -> no change
  SP(sort_call(A.m, rp.p, ci.p, v.p));
  CK(cudaDeviceSynchronize());
  const int64_t d4 = count_diff(ci.host(), A.ci) + count_diff(v.host(), A.v);
  record(name, d1 == 0 && d2 == 0 && d3 == 0 && d4 == 0, "m=%d nnz=%lld: entries diffs=%lld values diffs=%lld graph diffs=%lld resort diffs=%lld, %.3f ms",
         A.m, (long long)A.nnz(), (long long)d1, (long long)d2, (long long)d3, (long long)d4, ms);
}

template <typename S>
static void merge_case(const char* name, Csr<S> A);
template <>
void merge_case<double>(const char* name, Csr<double> A) {
  Dev<int> rp(A.rp), ci(A.ci), rpo((size_t)A.m + 1);
  Dev<double> v(A.v);
  int64_t merged = -1;
  SP(b200sp_sort_and_merge_count_f64_i32(nullptr, A.m, rp.p, ci.p, v.p, rpo.p, &merged));
  okk_sort_crs_stable_f64(A.m, A.rp.data(), A.ci.data(), A.v.data());
  std::vector<int> orp((size_t)A.m + 1, 0);
  const int64_t om = A.m > 0 ? okk_merged_rowmap(A.m, A.rp.data(), A.ci.data(), orp.data()) : 0;
  std::vector<int> oci(om);
  std::vector<double> ov(om);
  if (A.m > 0) okk_merged_entries_f64(A.m, A.rp.data(), A.ci.data(), A.v.data(), orp.data(), oci.data(), ov.data());
  Dev<int> cio((size_t)std::max<int64_t>(merged, 0));
  Dev<double> vo((size_t)std::max<int64_t>(merged, 0));
  SP(b200sp_sort_and_merge_fill_f64_i32(nullptr, A.m, rp.p, ci.p, v.p, rpo.p, cio.p, vo.p));
  CK(cudaDeviceSynchronize());
  const bool ok = merged == om && count_diff(rpo.host(), orp) == 0 && count_diff(cio.host(), oci) == 0 && count_diff(vo.host(), ov) == 0 &&
                  count_diff(ci.host(), A.ci) == 0;
  record(name, ok, "m=%d nnz=%lld merged=%lld (oracle %lld)", A.m, (long long)A.nnz(), (long long)merged, (long long)om);
}

static void transpose_case(const char* name, const Csr<double>& A) {
  Dev<int> rp(A.rp), ci(A.ci), trp((size_t)A.n + 1), tci((size_t)A.nnz());
  Dev<double> v(A.v), tv((size_t)A.nnz());
  trp.fill_bytes(0x55);
  Timer t;
  t.start();
  SP(b200sp_transpose_f64_i32(nullptr, A.m, A.n, rp.p, ci.p, v.p, trp.p, tci.p, tv.p));
  const float ms = t.stop_ms();
  CK(cudaDeviceSynchronize());
  std::vector<int> otrp((size_t)A.n + 1), otci(A.nnz());
  std::vector<double> otv(A.nnz());
  okk_transpose_f64(A.m, A.n, A.rp.data(), A.ci.data(), A.v.data(), otrp.data(), otci.data(), otv.data());
  const int64_t d1 = count_diff(trp.host(), otrp), d2 = count_diff(tci.host(), otci), d3 = count_diff(tv.host(), otv);
  record(name, d1 == 0 && d2 == 0 && d3 == 0, "%dx%d nnz=%lld: row map diffs=%lld entries diffs=%lld values diffs=%lld, %.3f ms", A.m, A.n,
         (long long)A.nnz(), (long long)d1, (long long)d2, (long long)d3, ms);
}

// randomMatrix of Test_Sparse_spadd.hpp:41-94
template <typename S>
static Csr<S> spadd_matrix(int m, int n, int lo, int hi, bool sorted, uint64_t seed) {
  Rng r(seed);
  std::vector<int> lens(m);
  int maxlen = 0;
  for (auto& l : lens) {
    l = lo + (hi > lo ? r.below(hi - lo + 1) : 0);
    maxlen = std::max(maxlen, l);
  }
  Csr<S> A;
  A.m = m;
  A.n = n;
  A.rp.assign(m + 1, 0);
  for (int i = 0; i < m; ++i) A.rp[i + 1] = A.rp[i] + lens[i];
  A.ci.resize(A.rp[m]);
  std::vector<int> idx(std::max(n, maxlen));
  for (int i = 0; i < m; ++i) {
    for (size_t j = 0; j < idx.size(); ++j) idx[j] = (int)(j % (size_t)std::max(n, 1));
    for (size_t j = idx.size(); j > 1; --j) std::swap(idx[j - 1], idx[r.below((int)j)]);
    if (sorted) std::sort(idx.begin(), idx.begin() + lens[i]);
    std::copy(idx.begin(), idx.begin() + lens[i], A.ci.begin() + A.rp[i]);
  }
  A.v.resize(A.ci.size());
  fill_vals(A.v, 0.0, 1.0, seed + 5);
  return A;
}

static int spadd_num(b200sp_spadd_plan* p, int m, int n, const int* ra, const int* ca, const double* va, double al, const int* rb,
                     const int* cb, const double* vb, double be, const int* rc, int* cc, double* vc) {
  return b200sp_spadd_numeric_f64_i32(p, nullptr, m, n, ra, ca, va, al, rb, cb, vb, be, rc, cc, vc);
}
static int spadd_num(b200sp_spadd_plan* p, int m, int n, const int* ra, const int* ca, const float* va, float al, const int* rb,
                     const int* cb, const float* vb, float be, const int* rc, int* cc, float* vc) {
  return b200sp_spadd_numeric_f32_i32(p, nullptr, m, n, ra, ca, va, al, rb, cb, vb, be, rc, cc, vc);
}
static void ospadd_sorted(int m, const Csr<double>& A, double al, const Csr<double>& B, double be, const std::vector<int>& rc,
                          std::vector<int>& cc, std::vector<double>& vc) {
  okk_spadd_sorted_numeric_f64(m, A.rp.data(), A.ci.data(), A.v.data(), al, B.rp.data(), B.ci.data(), B.v.data(), be, rc.data(), cc.data(), vc.data());
}
static void ospadd_sorted(int m, const Csr<float>& A, float al, const Csr<float>& B, float be, const std::vector<int>& rc,
                          std::vector<int>& cc, std::vector<float>& vc) {
  okk_spadd_sorted_numeric_f32(m, A.rp.data(), A.ci.data(), A.v.data(), al, B.rp.data(), B.ci.data(), B.v.data(), be, rc.data(), cc.data(), vc.data());
}
static void ospadd_unsorted(int m, const Csr<double>& A, double al, const Csr<double>& B, double be, const std::vector<int>& rc,
                            std::vector<int>& cc, std::vector<double>& vc, const std::vector<int>& ap, const std::vector<int>& bp) {
  okk_spadd_unsorted_numeric_f64(m, A.rp.data(), A.ci.data(), A.v.data(), al, B.rp.data(), B.ci.data(), B.v.data(), be, rc.data(), cc.data(),
                                 vc.data(), ap.data(), bp.data());
}
static void ospadd_unsorted(int m, const Csr<float>& A, float al, const Csr<float>& B, float be, const std::vector<int>& rc,
                            std::vector<int>& cc, std::vector<float>& vc, const std::vector<int>& ap, const std::vector<int>& bp) {
  okk_spadd_unsorted_numeric_f32(m, A.rp.data(), A.ci.data(), A.v.data(), al, B.rp.data(), B.ci.data(), B.v.data(), be, rc.data(), cc.data(),
                                 vc.data(), ap.data(), bp.data());
}

template <typename S>
static void spadd_case(const char* name, int m, int n, int lo, int hi, bool sorted) {
  auto A = spadd_matrix<S>(m, n, lo, hi, sorted, ((uint64_t)m << 1) ^ (uint64_t)n);
  auto B = spadd_matrix<S>(m, n, lo, hi, sorted, (((uint64_t)m << 1) ^ (uint64_t)n) + 1);
  std::vector<int> orc((size_t)m + 1, 0), ap(std::max<size_t>(A.ci.size(), 1)), bp(std::max<size_t>(B.ci.size(), 1));
  const int64_t onnz = sorted ? okk_spadd_sorted_symbolic(m, A.rp.data(), A.ci.data(), B.rp.data(), B.ci.data(), orc.data())
                              : okk_spadd_unsorted_symbolic(m, A.rp.data(), A.ci.data(), B.rp.data(), B.ci.data(), orc.data(), ap.data(), bp.data());
  std::vector<int> occ(onnz);
  std::vector<S> ovc(onnz);
  const S al = (S)0.3, be = (S)-1.7;  // not powers of two: the products round
  if (sorted) ospadd_sorted(m, A, al, B, be, orc, occ, ovc);
  else ospadd_unsorted(m, A, al, B, be, orc, occ, ovc, ap, bp);
  Dev<int> ra(A.rp), ca(A.ci), rb(B.rp), cb(B.ci), rc((size_t)m + 1);
  Dev<S> va(A.v), vb(B.v);
  rc.fill_bytes(0x05);
  b200sp_spadd_plan* plan = nullptr;
  SP(b200sp_spadd_plan_create(&plan, sorted ? 1 : 0, hi <= n ? 1 : 0));
  int64_t c_nnz = -1;
  Timer t;
  t.start();
  SP(b200sp_spadd_symbolic_i32(plan, nullptr, m, n, ra.p, ca.p, rb.p, cb.p, rc.p, &c_nnz));
  const float ms_sym = t.stop_ms();
  bool ok = c_nnz == onnz && count_diff(rc.host(), orc) == 0;
  int64_t d1 = -1, d2 = -1;
  float ms_num = 0;
  if (ok) {
    Dev<int> cc((size_t)c_nnz);
    Dev<S> vc((size_t)c_nnz);
    cc.fill_bytes(0x05);
    vc.fill_bytes(0x05);
    t.start();
    SP(spadd_num(plan, m, n, ra.p, ca.p, va.p, al, rb.p, cb.p, vb.p, be, rc.p, cc.p, vc.p));
    ms_num = t.stop_ms();
    CK(cudaDeviceSynchronize());
    d1 = count_diff(cc.host(), occ);
    d2 = count_diff(vc.host(), ovc);
    ok = d1 == 0 && d2 == 0;
  }
  b200sp_spadd_plan_destroy(plan, nullptr);
  record(name, ok, "%dx%d rows %d..%d %s: c_nnz=%lld (oracle %lld) entries diffs=%lld values diffs=%lld; symbolic %.3f ms numeric %.3f ms", m, n, lo,
         hi, sorted ? "sorted" : "unsorted", (long long)c_nnz, (long long)onnz, (long long)d1, (long long)d2, ms_sym, ms_num);
}

static void suite_crs() {
  sort_case("sort/kk_10x10_f64", gen_kk<double>(10, 10, 20, 2, 5, 1));
  sort_case("sort/kk_1000x1000_f64", gen_kk<double>(1000, 1000, 30000, 2, 500, 1));
  sort_case("sort/kk_20000x20000_f32", gen_kk<float>(20000, 20000, 600000, 2, 10000, 1));
  {
    Rng r(11);
    std::vector<int> lens(3000);
    for (auto& l : lens) l = r.below(40);
    const int special[] = {9000, 5000, 4097, 4096, 300, 257, 256, 255, 33, 32, 31, 2, 1, 0};
    for (size_t i = 0; i < sizeof(special) / sizeof(int); ++i) lens[i] = special[i];
    sort_case("sort/long_rows_with_ties_f64", gen_rows<double>(lens, 500, false, false, 11));
    merge_case<double>("merge/long_rows_60_columns", gen_rows<double>(lens, 60, false, false, 12));
  }
  {
    // golden case 0 of Test_Sparse_SortCrs.hpp:203-243
    Csr<double> A;
    A.m = 5;
    A.n = 7;
    A.rp = {0, 4, 4, 5, 7, 10};
    A.ci = {4, 3, 5, 3, 6, 2, 2, 0, 1, 2};
    A.v = {1.5, 4, 1, -3, 2, -1, -2, 0, 3.5, -2.25};
    merge_case<double>("merge/golden_case0", A);
    Csr<double> E;
    E.m = 5;
    E.n = 7;
    E.rp = {0, 0, 0, 0, 0, 0};
    merge_case<double>("merge/golden_case2_empty", E);
  }
  {
    Rng r(5);
    std::vector<int> lens(3000);
    for (auto& l : lens) l = r.below(60);
    transpose_case("transpose/3000x1000_with_duplicates", gen_rows<double>(lens, 1000, false, false, 5));
    transpose_case("transpose/1x5", gen_rows<double>(std::vector<int>{3}, 5, true, false, 6));
    transpose_case("transpose/lap27", gen_lap27<double>(10, 2));
  }
  for (int sorted = 1; sorted >= 0; --sorted) {
    const char* tag = sorted ? "sorted" : "unsorted";
    char nm[96];
    snprintf(nm, sizeof(nm), "spadd/%s_10x10_empty_f64", tag);
    spadd_case<double>(nm, 10, 10, 0, 0, sorted);
    snprintf(nm, sizeof(nm), "spadd/%s_10x10_0..2_f64", tag);
    spadd_case<double>(nm, 10, 10, 0, 2, sorted);
    snprintf(nm, sizeof(nm), "spadd/%s_100x100_50..100_f64", tag);
    spadd_case<double>(nm, 100, 100, 50, 100, sorted);
    snprintf(nm, sizeof(nm), "spadd/%s_50x50_75..100_duplicates_f64", tag);
    spadd_case<double>(nm, 50, 50, 75, 100, sorted);
    snprintf(nm, sizeof(nm), "spadd/%s_50x50_75..100_duplicates_f32", tag);
    spadd_case<float>(nm, 50, 50, 75, 100, sorted);
    snprintf(nm, sizeof(nm), "spadd/%s_20000x3000_0..60_f64", tag);
    spadd_case<double>(nm, 20000, 3000, 0, 60, sorted);
    snprintf(nm, sizeof(nm), "spadd/%s_20000x3000_0..60_f32", tag);
    spadd_case<float>(nm, 20000, 3000, 0, 60, sorted);
  }
}

// ------------------------------------------------------------------------------------------------
// suite: crs_big -- timings on a bench-sized matrix (27-point stencil x 2 dof, rows shuffled for the sort)
// ------------------------------------------------------------------------------------------------
static void suite_crs_big() {
  const int g = g_big ? 64 : 40;
  auto A = gen_lap27<double>(g, 2);
  Csr<double> U = A;  // rows reversed: every row needs sorting
  for (int i = 0; i < U.m; ++i) {
    std::reverse(U.ci.begin() + U.rp[i], U.ci.begin() + U.rp[i + 1]);
    std::reverse(U.v.begin() + U.rp[i], U.v.begin() + U.rp[i + 1]);
  }
  const double gb = 12.0 * A.nnz() / 1e9;
  {  // warm-up: first-use costs (module load, stream-ordered pool growth) stay out of the timings below
    auto W = gen_lap27<double>(8, 2);
    Dev<int> rp(W.rp), ci(W.ci), rc((size_t)W.m + 1), trp((size_t)W.n + 1), tci((size_t)W.nnz());
    Dev<double> v(W.v), tv((size_t)W.nnz());
    SP(b200sp_sort_crs_f64_i32(nullptr, W.m, rp.p, ci.p, v.p));
    SP(b200sp_transpose_f64_i32(nullptr, W.m, W.n, rp.p, ci.p, v.p, trp.p, tci.p, tv.p));
    for (int sorted = 0; sorted <= 1; ++sorted) {
      b200sp_spadd_plan* plan = nullptr;
      int64_t c = 0;
      SP(b200sp_spadd_plan_create(&plan, sorted, 1));
      SP(b200sp_spadd_symbolic_i32(plan, nullptr, W.m, W.n, rp.p, ci.p, rp.p, ci.p, rc.p, &c));
      b200sp_spadd_plan_destroy(plan, nullptr);
    }
    Dev<char> big((size_t)1 << 30);  // grow the default memory pool once
    CK(cudaDeviceSynchronize());
  }
  {
    Dev<int> rp(U.rp), ci(U.ci);
    Dev<double> v(U.v);
    Timer t;
    t.start();
    SP(b200sp_sort_crs_f64_i32(nullptr, U.m, rp.p, ci.p, v.p));
    const float ms = t.stop_ms();
    const bool ok = count_diff(ci.host(), A.ci) == 0 && count_diff(v.host(), A.v) == 0;
    record("sort_reversed_rows", ok, "m=%d nnz=%lld %.3f ms (%.0f GB/s read+write of 12 B/entry)", U.m, (long long)U.nnz(), ms, 2 * gb / (ms * 1e-3));
    t.start();
    SP(b200sp_sort_crs_f64_i32(nullptr, U.m, rp.p, ci.p, v.p));
    record("sort_already_sorted", true, "%.3f ms (classification pass only)", t.stop_ms());
  }
  {
    Dev<int> rp(A.rp), ci(A.ci), trp((size_t)A.n + 1), tci((size_t)A.nnz());
    Dev<double> v(A.v), tv((size_t)A.nnz());
    Timer t;
    t.start();
    SP(b200sp_transpose_f64_i32(nullptr, A.m, A.n, rp.p, ci.p, v.p, trp.p, tci.p, tv.p));
    const float ms = t.stop_ms();
    // the stencil matrix is structurally symmetric: the transpose has the same graph
    const bool ok = count_diff(trp.host(), A.rp) == 0 && count_diff(tci.host(), A.ci) == 0;
    record("transpose", ok, "%.3f ms (%.0f GB/s of 24 B/entry)", ms, 2 * gb / (ms * 1e-3));
  }
  for (int sorted = 1; sorted >= 0; --sorted) {
    Dev<int> rp(A.rp), ci(A.ci), rc((size_t)A.m + 1);
    Dev<double> v(A.v);
    b200sp_spadd_plan* plan = nullptr;
    SP(b200sp_spadd_plan_create(&plan, sorted, 1));
    int64_t c_nnz = 0;
    Timer t;
    t.start();
    SP(b200sp_spadd_symbolic_i32(plan, nullptr, A.m, A.n, rp.p, ci.p, rp.p, ci.p, rc.p, &c_nnz));
    const float ms_sym = t.stop_ms();
    Dev<int> cc((size_t)c_nnz);
    Dev<double> vc((size_t)c_nnz);
    t.start();
    SP(b200sp_spadd_numeric_f64_i32(plan, nullptr, A.m, A.n, rp.p, ci.p, v.p, 1.0, rp.p, ci.p, v.p, 1.0, rc.p, cc.p, vc.p));
    const float ms_num = t.stop_ms();
    auto hv = vc.host();
    bool ok = c_nnz == A.nnz() && count_diff(cc.host(), A.ci) == 0;
    for (size_t i = 0; ok && i < hv.size(); ++i) ok = hv[i] == 2.0 * A.v[i];
    b200sp_spadd_plan_destroy(plan, nullptr);
    record(sorted ? "spadd_sorted_A_plus_A" : "spadd_unsorted_A_plus_A", ok, "symbolic %.3f ms, numeric %.3f ms (%.0f GB/s of 36 B/entry)", ms_sym,
           ms_num, 3 * gb / (ms_num * 1e-3));
  }
}

// ------------------------------------------------------------------------------------------------
// suite: spmm -- kernel variants of the rank-2 product (B200SP_SPMM_KERNEL) against the oracle + timing
// ------------------------------------------------------------------------------------------------
static int g_timeout_scale = 1;  // --timeout-scale N: the emulated build is orders of magnitude slower
static int g_spmm_scale = 0;  // --spmm-scale N (default 18, 21 with --big; 23 = BASELINE.json config 3)

static void suite_spmm() {
  const int scale = g_spmm_scale > 0 ? g_spmm_scale : (g_big ? 21 : 18), k = 16;
  const bool full_check = scale <= 21;  // above: parity on sampled rows (the full-size case is covered at scale 21)
  int64_t nnz = 0;
  double t0 = now_s();
  void* h = b200gen_rmat_build(scale, 16, 0.57, 0.19, 0.19, 23, &nnz);
  const int n = 1 << scale;
  std::vector<int> rp((size_t)n + 1), ci((size_t)nnz);
  b200gen_rmat_emit(h, rp.data(), ci.data());
  std::vector<float> v((size_t)nnz), X((size_t)n * k), Y0((size_t)n * k);
  b200gen_fill_f32(nnz, v.data(), 0.f, 1.f, 3);
  b200gen_fill_f32((int64_t)X.size(), X.data(), -1.f, 1.f, 4);
  b200gen_fill_f32((int64_t)Y0.size(), Y0.data(), -1.f, 1.f, 5);
  int maxrow = 0;
  for (int i = 0; i < n; ++i) maxrow = std::max(maxrow, rp[i + 1] - rp[i]);
  record("generate", true, "R-MAT scale %d: n=%d nnz=%lld longest row %d, %.1f s", scale, n, (long long)nnz, maxrow, now_s() - t0);
  const float alpha = 1.5f, beta = 0.5f;
  std::vector<float> Yref, Ys;
  std::vector<int> sample;
  if (full_check) {
    Yref = Y0;
    okk_spmv_mv_f32(n, n, k, rp.data(), ci.data(), v.data(), X.data(), k, 1, Yref.data(), k, 1, alpha, beta, okk_num_threads());
    // row-scaled tolerance: |alpha| sum |a||x| + |beta||y0|
    std::vector<float> va(v), Xa(X);
    Ys = Y0;
    for (auto& x : va) x = std::fabs(x);
    for (auto& x : Xa) x = std::fabs(x);
    for (auto& x : Ys) x = std::fabs(x);
    okk_spmv_mv_f32(n, n, k, rp.data(), ci.data(), va.data(), Xa.data(), k, 1, Ys.data(), k, 1, alpha, beta, okk_num_threads());
  } else {
    Rng r(1);
    for (int i = 0; i < 3000; ++i) sample.push_back(r.below(n));
    // the longest rows (segment path) are part of the sample
    std::vector<int> order(n);
    std::iota(order.begin(), order.end(), 0);
    std::partial_sort(order.begin(), order.begin() + 40, order.end(), [&](int a, int b) { return rp[a + 1] - rp[a] > rp[b + 1] - rp[b]; });
    sample.insert(sample.end(), order.begin(), order.begin() + 40);
  }
  auto check = [&](const std::vector<float>& got) -> double {
    double worst = 0;
    if (full_check) {
      for (size_t i = 0; i < got.size(); ++i) worst = std::max(worst, (double)std::fabs(got[i] - Yref[i]) / std::max((double)Ys[i], 1e-30));
      return worst;
    }
    for (int row : sample) {
      for (int j = 0; j < k; ++j) {
        double acc = 0, sc = 0;
        for (int e = rp[row]; e < rp[row + 1]; ++e) {
          const double t = (double)v[e] * (double)X[(size_t)ci[e] * k + j];
          acc += t;
          sc += std::fabs(t);
        }
        const double want = beta * (double)Y0[(size_t)row * k + j] + alpha * acc;
        const double scale_r = std::fabs(alpha) * sc + std::fabs(beta * Y0[(size_t)row * k + j]);
        worst = std::max(worst, std::fabs((double)got[(size_t)row * k + j] - want) / std::max(scale_r, 1e-30));
      }
    }
    return worst;
  };
  Dev<int> drp(rp), dci(ci);
  Dev<float> dv(v), dX(X), dY((size_t)n * k);
  const double balg = 8.0 * nnz + 4.0 * (n + 1) + 4.0 * (double)n * k * 3;
  struct Var {
    const char* kernel;
    const char* lmax;
    const char* cfg;
  };
  const Var vars[] = {{"split", nullptr, nullptr}, {"tile", nullptr, nullptr},  {"tilev", nullptr, nullptr}, {"tilev", "64", nullptr},
                      {"tilev", "128", nullptr},   {"tilev", "512", nullptr},   {"tilev", nullptr, "1"},     {"tilev", nullptr, "2"},
                      {"tilev", nullptr, "3"},     {"tilev", "128", "1"},       {"tilev", "128", "2"},       {"tilev", "128", "segvec"},
                      {"tilev", "64", "segvec"},   {"row", nullptr, nullptr}};
  for (const Var& vr : vars) {
    if (!strcmp(vr.kernel, "row") && scale > 21) continue;  // far the slowest at scale 21: not worth the slot
    setenv("B200SP_SPMM_KERNEL", vr.kernel, 1);
    if (vr.lmax) setenv("B200SP_SPMM_LMAX", vr.lmax, 1);
    else unsetenv("B200SP_SPMM_LMAX");
    unsetenv("B200SP_SPMM_CFG");
    unsetenv("B200SP_SPMM_SEG");
    if (vr.cfg && !strcmp(vr.cfg, "segvec")) setenv("B200SP_SPMM_SEG", "vec", 1);
    else if (vr.cfg) setenv("B200SP_SPMM_CFG", vr.cfg, 1);
    b200sp_spmv_plan* plan = nullptr;
    SP(b200sp_spmv_plan_create(&plan, 0));
    float best = 1e30f;
    for (int rep = 0; rep < 5; ++rep) {
      CK(cudaMemcpy(dY.p, Y0.data(), Y0.size() * sizeof(float), cudaMemcpyHostToDevice));
      Timer t;
      t.start();
      SP(b200sp_spmm_f32_i32(plan, nullptr, 'N', n, n, nnz, k, alpha, drp.p, dci.p, dv.p, dX.p, k, 1, beta, dY.p, k, 1));
      const float ms = t.stop_ms();
      if (rep > 0) best = std::min(best, ms);
    }
    const double worst = check(dY.host());
    char nm[96];
    snprintf(nm, sizeof(nm), "rmat%d_k16_f32/%s%s%s%s%s", scale, vr.kernel, vr.lmax ? "_lmax" : "", vr.lmax ? vr.lmax : "", vr.cfg ? "_cfg" : "",
             vr.cfg ? vr.cfg : "");
    record(nm, worst <= 1e-4, "kernel=%s %.3f ms, %.0f GFLOP/s, %.0f GB/s algorithmic, max scaled err %.2e (%s)", b200sp_spmv_last_kernel(plan), best,
           2.0 * nnz * k / (best * 1e-3) / 1e9, balg / (best * 1e-3) / 1e9, worst, full_check ? "all rows" : "sampled + longest rows");
    b200sp_spmv_plan_destroy(plan, nullptr);
  }
  unsetenv("B200SP_SPMM_KERNEL");
  unsetenv("B200SP_SPMM_LMAX");
  unsetenv("B200SP_SPMM_CFG");
  unsetenv("B200SP_SPMM_SEG");
}

// ------------------------------------------------------------------------------------------------
// suite: spmv_t -- transposed SpMV: atomics path vs the cached-transpose option, against the oracle
// ------------------------------------------------------------------------------------------------
static void spmv_t_case(const char* name, const Csr<double>& A) {
  std::vector<double> x((size_t)A.m), y0((size_t)A.n), yref, scale;
  b200gen_fill_f64(A.m, x.data(), -1.0, 1.0, 1);
  b200gen_fill_f64(A.n, y0.data(), -1.0, 1.0, 2);
  const double alpha = 1.25, beta = -0.5;
  yref = y0;
  okk_spmv_transpose_f64(A.m, A.n, A.rp.data(), A.ci.data(), A.v.data(), x.data(), yref.data(), alpha, beta);
  std::vector<double> va(A.v), xa(x);
  scale = y0;
  for (auto& t : va) t = std::fabs(t);
  for (auto& t : xa) t = std::fabs(t);
  for (auto& t : scale) t = std::fabs(t);
  okk_spmv_transpose_f64(A.m, A.n, A.rp.data(), A.ci.data(), va.data(), xa.data(), scale.data(), std::fabs(alpha), std::fabs(beta));
  Dev<int> rp(A.rp), ci(A.ci);
  Dev<double> v(A.v), dx(x), dy((size_t)A.n);
  for (int cached = 0; cached <= 1; ++cached) {
    b200sp_spmv_plan* plan = nullptr;
    SP(b200sp_spmv_plan_create(&plan, 0));
    SP(b200sp_spmv_plan_set_option(plan, B200SP_SPMV_OPT_CACHE_TRANSPOSE, cached));
    float best = 1e30f;
    std::vector<double> got, first;
    for (int rep = 0; rep < 4; ++rep) {
      CK(cudaMemcpy(dy.p, y0.data(), y0.size() * sizeof(double), cudaMemcpyHostToDevice));
      Timer t;
      t.start();
      SP(b200sp_spmv_f64_i32(plan, nullptr, 'T', A.m, A.n, A.nnz(), alpha, rp.p, ci.p, v.p, dx.p, beta, dy.p));
      const float ms = t.stop_ms();
      if (rep > 0) best = std::min(best, ms);
      got = dy.host();
      if (rep == 0) first = got;
    }
    double worst = 0;
    for (size_t i = 0; i < got.size(); ++i) worst = std::max(worst, std::fabs(got[i] - yref[i]) / std::max(scale[i], 1e-300));
    const int64_t drift = count_diff(got, first);  // run-to-run bit differences (atomics reorder, the cached path must not)
    char nm[128];
    snprintf(nm, sizeof(nm), "%s/%s", name, cached ? "cached_transpose" : "atomics");
    record(nm, worst <= 1e-10 && (!cached || drift == 0), "kernel=%s %.3f ms, max scaled err %.2e, run-to-run differing entries %lld",
           b200sp_spmv_last_kernel(plan), best, worst, (long long)drift);
    b200sp_spmv_plan_destroy(plan, nullptr);
  }
}

static void suite_spmv_t() {
  spmv_t_case("lap27_40x2dof", gen_lap27<double>(g_big ? 100 : 40, 2));
  {
    Rng r(8);
    std::vector<int> lens(50000);
    for (auto& l : lens) l = r.below(30);
    lens[7] = 20000;
    spmv_t_case("random_50000x20000_rect", gen_rows<double>(lens, 20000, false, false, 8));
  }
}

// ------------------------------------------------------------------------------------------------
// suite: bsr -- BsrMatrix SpMV (N: TMA tile kernel and the per-row kernel; T: atomics) and SpMM against the oracle's
// restatement of the reference functors (oracle/kk_oracle_bsr.c), with the algorithmic bandwidth of the N kernel
// ------------------------------------------------------------------------------------------------
static void bsr_case(const char* name, const Csr<double>& G, int bs) {
  const int mb = G.m, nb = G.n;
  const int64_t nnzb = G.nnz();
  const int64_t np_r = (int64_t)mb * bs, np_c = (int64_t)nb * bs;
  std::vector<double> vals((size_t)nnzb * bs * bs), x((size_t)np_c), xt((size_t)np_r), y0((size_t)np_r), yt0((size_t)np_c);
  b200gen_fill_f64((int64_t)vals.size(), vals.data(), -1.0, 1.0, 11 + bs);
  b200gen_fill_f64(np_c, x.data(), -1.0, 1.0, 1);
  b200gen_fill_f64(np_r, xt.data(), -1.0, 1.0, 2);
  b200gen_fill_f64(np_r, y0.data(), -1.0, 1.0, 3);
  b200gen_fill_f64(np_c, yt0.data(), -1.0, 1.0, 4);
  const double alpha = 1.25, beta = -0.5;
  std::vector<double> va(vals), xa(x), xta(xt);
  for (auto& t : va) t = std::fabs(t);
  for (auto& t : xa) t = std::fabs(t);
  for (auto& t : xta) t = std::fabs(t);
  Dev<int> rp(G.rp), ci(G.ci);
  Dev<double> v(vals), dx(x), dxt(xt), dy((size_t)np_r), dyt((size_t)np_c);
  const double bytes = (double)nnzb * (bs * bs * 8.0 + 4.0) + (mb + 1) * 4.0 + (double)np_c * 8.0 + (double)np_r * 16.0;
  // ---- N: tile kernel (default) and the per-row kernel
  {
    std::vector<double> yref(y0), scale(y0);
    okk_bsr_spmv_v42_f64(mb, bs, 1, G.rp.data(), G.ci.data(), vals.data(), x.data(), 1, 0, yref.data(), 1, 0, alpha, beta);
    for (auto& t : scale) t = std::fabs(t);
    okk_bsr_spmv_v42_f64(mb, bs, 1, G.rp.data(), G.ci.data(), va.data(), xa.data(), 1, 0, scale.data(), 1, 0, std::fabs(alpha),
                         std::fabs(beta));
    for (int variant = 0; variant < 3; ++variant) {
      if (variant == 2 && bs > 5) continue;  // "walk" is already the default tile kernel beyond bs = 5
      if (variant) setenv("B200SP_BSR_KERNEL", variant == 1 ? "vector" : "walk", 1);
      else unsetenv("B200SP_BSR_KERNEL");
      b200sp_bsr_plan* plan = nullptr;
      SP(b200sp_bsr_plan_create(&plan));
      float best = 1e30f;
      std::vector<double> got;
      for (int rep = 0; rep < 4; ++rep) {
        CK(cudaMemcpy(dy.p, y0.data(), y0.size() * sizeof(double), cudaMemcpyHostToDevice));
        Timer t;
        t.start();
        SP(b200sp_bsr_spmv_f64_i32(plan, nullptr, 'N', mb, nb, nnzb, bs, alpha, rp.p, ci.p, v.p, dx.p, beta, dy.p));
        const float ms = t.stop_ms();
        if (rep > 0) best = std::min(best, ms);
        got = dy.host();
      }
      double worst = 0;
      for (size_t i = 0; i < got.size(); ++i) worst = std::max(worst, std::fabs(got[i] - yref[i]) / std::max(scale[i], 1e-300));
      char nm[160];
      snprintf(nm, sizeof(nm), "%s_bs%d/N_%s", name, bs, variant == 0 ? "default" : variant == 1 ? "vector" : "walk");
      record(nm, worst <= 1e-10, "mb=%d nnzb=%lld kernel=%s %.3f ms (%.0f GB/s algorithmic), max scaled err %.2e", mb, (long long)nnzb,
             b200sp_bsr_last_kernel(plan), best, bytes / (best * 1e-3) / 1e9, worst);
      b200sp_bsr_plan_destroy(plan, nullptr);
    }
    unsetenv("B200SP_BSR_KERNEL");
  }
  // ---- T (atomics) and a 5-column multivector in both modes
  {
    std::vector<double> yref(yt0), scale(yt0);
    okk_bsr_spmv_v41_f64('T', mb, nb, bs, 1, G.rp.data(), G.ci.data(), vals.data(), xt.data(), 1, 0, yref.data(), 1, 0, alpha, beta);
    for (auto& t : scale) t = std::fabs(t);
    okk_bsr_spmv_v41_f64('T', mb, nb, bs, 1, G.rp.data(), G.ci.data(), va.data(), xta.data(), 1, 0, scale.data(), 1, 0, std::fabs(alpha),
                         std::fabs(beta));
    b200sp_bsr_plan* plan = nullptr;
    SP(b200sp_bsr_plan_create(&plan));
    CK(cudaMemcpy(dyt.p, yt0.data(), yt0.size() * sizeof(double), cudaMemcpyHostToDevice));
    Timer t;
    t.start();
    SP(b200sp_bsr_spmv_f64_i32(plan, nullptr, 'T', mb, nb, nnzb, bs, alpha, rp.p, ci.p, v.p, dxt.p, beta, dyt.p));
    const float ms = t.stop_ms();
    auto got = dyt.host();
    double worst = 0;
    for (size_t i = 0; i < got.size(); ++i) worst = std::max(worst, std::fabs(got[i] - yref[i]) / std::max(scale[i], 1e-300));
    char nm[160];
    snprintf(nm, sizeof(nm), "%s_bs%d/T", name, bs);
    record(nm, worst <= 1e-10, "kernel=%s %.3f ms (first call), max scaled err %.2e", b200sp_bsr_last_kernel(plan), ms, worst);
    const int k = 5;
    for (int rm = 0; rm <= 1; ++rm) {
      const int64_t ldx = rm ? k + 1 : np_c + 3, ldy = rm ? k : np_r + 1;
      const int64_t xr = rm ? ldx : 1, xc = rm ? 1 : ldx, yr = rm ? ldy : 1, yc = rm ? 1 : ldy;
      std::vector<double> X((size_t)(rm ? np_c * ldx : ldx * k)), Y0((size_t)(rm ? np_r * ldy : ldy * k));
      fill_vals(X, -1.0, 1.0, 31);
      fill_vals(Y0, -1.0, 1.0, 32);
      std::vector<double> Yref(Y0), Xa(X), Ys(Y0);
      okk_bsr_spmv_v42_f64(mb, bs, k, G.rp.data(), G.ci.data(), vals.data(), X.data(), xr, xc, Yref.data(), yr, yc, alpha, beta);
      for (auto& q : Xa) q = std::fabs(q);
      for (auto& q : Ys) q = std::fabs(q);
      okk_bsr_spmv_v42_f64(mb, bs, k, G.rp.data(), G.ci.data(), va.data(), Xa.data(), xr, xc, Ys.data(), yr, yc, std::fabs(alpha),
                           std::fabs(beta));
      Dev<double> dX(X), dY(Y0);
      SP(b200sp_bsr_spmm_f64_i32(plan, nullptr, 'N', mb, nb, nnzb, bs, k, alpha, rp.p, ci.p, v.p, dX.p, ldx, rm, beta, dY.p, ldy, rm));
      CK(cudaDeviceSynchronize());
      auto gotm = dY.host();
      double w2 = 0;
      int64_t touched_pad = 0;
      for (size_t i = 0; i < gotm.size(); ++i) {
        const int64_t r = rm ? (int64_t)i / ldy : (int64_t)i % ldy, c = rm ? (int64_t)i % ldy : (int64_t)i / ldy;
        if (r >= np_r || c >= k) {
          if (gotm[i] != Y0[i]) ++touched_pad;
          continue;
        }
        w2 = std::max(w2, std::fabs(gotm[i] - Yref[i]) / std::max(Ys[i], 1e-300));
      }
      snprintf(nm, sizeof(nm), "%s_bs%d/N_x%d_%s", name, bs, k, rm ? "layoutright" : "layoutleft");
      record(nm, w2 <= 1e-10 && touched_pad == 0, "kernel=%s max scaled err %.2e, padding entries touched %lld", b200sp_bsr_last_kernel(plan),
             w2, (long long)touched_pad);
    }
    b200sp_bsr_plan_destroy(plan, nullptr);
  }
}

static void suite_bsr() {
  const Csr<double> G = gen_lap27<double>(g_big ? 64 : 24, 1);  // 27 blocks per block row
  for (int bs : {2, 3, 4, 5, 8, 16}) {
    if (g_big && bs > 8) continue;  // 7 M blocks x 256 values would not fit next to the oracle copies
    bsr_case("lap27", G, bs);
  }
  {  // skewed block rows: a few beyond the stage, many empty
    Rng r(5);
    std::vector<int> lens(20000);
    for (auto& l : lens) l = r.below(7);
    lens[3] = 900;
    lens[9000] = 2500;
    bsr_case("skewed", gen_rows<double>(lens, 20000, false, false, 6), 3);
  }
}

// ------------------------------------------------------------------------------------------------
// suite: cg -- the device-resident CG driver against the oracle's restatement of the reference's pcgsolve, with the time per
// iteration next to the time of the SpMV alone (what the three extra kernels and the polling cost)
// ------------------------------------------------------------------------------------------------
static void suite_cg() {
  Csr<double> A = gen_lap27<double>(g_big ? 128 : 20, 1);
  for (int r = 0; r < A.m; ++r)  // shift the diagonal: the 27-point operator alone has the constants in its null space
    for (int q = A.rp[r]; q < A.rp[r + 1]; ++q)
      if (A.ci[q] == r) A.v[q] += 0.5;
  const int n = A.m;
  std::vector<double> xs((size_t)n), b((size_t)n, 0.0), xo((size_t)n, 0.0);
  b200gen_fill_f64(n, xs.data(), -1.0, 1.0, 9);
  okk_spmv_serial_f64(n, A.rp.data(), A.ci.data(), A.v.data(), xs.data(), b.data(), 1.0, 0.0);
  double nr_o = 0;
  const int it_o = okk_cg_f64(n, A.rp.data(), A.ci.data(), A.v.data(), b.data(), xo.data(), 100000, 1e-7, &nr_o);
  Dev<int> rp(A.rp), ci(A.ci);
  Dev<double> v(A.v), db(b), dx((size_t)n), dy((size_t)n);
  b200sp_spmv_plan* plan = nullptr;
  SP(b200sp_spmv_plan_create(&plan, 0));
  float spmv_ms = 1e30f;
  for (int rep = 0; rep < 6; ++rep) {  // also lets the plan finish its self-tuning before the solve
    Timer t;
    t.start();
    SP(b200sp_spmv_f64_i32(plan, nullptr, 'N', n, n, A.nnz(), 1.0, rp.p, ci.p, v.p, db.p, 0.0, dy.p));
    spmv_ms = std::min(spmv_ms, t.stop_ms());
  }
  for (int check_every : {1, 8, 32}) {
    dx.fill_bytes(0);
    int it = 0;
    double nr = 0;
    const double t0 = now_s();
    SP(b200sp_cg_solve_f64_i32(plan, nullptr, n, A.nnz(), rp.p, ci.p, v.p, db.p, dx.p, 100000, 1e-7, check_every, &it, &nr));
    const double ms = (now_s() - t0) * 1e3;
    auto x = dx.host();
    double num = 0, den = 0;
    for (int i = 0; i < n; ++i) {
      num += (x[i] - xo[i]) * (x[i] - xo[i]);
      den += xo[i] * xo[i];
    }
    char nm[96];
    snprintf(nm, sizeof(nm), "lap27_shifted/check_every_%d", check_every);
    record(nm, std::abs(it - it_o) <= 2 && nr <= 1e-7 && std::sqrt(num / std::max(den, 1e-300)) < 1e-8,
           "n=%d nnz=%lld: %d iterations (oracle %d), norm_res %.2e, |x-x_oracle|/|x_oracle| %.1e; %.3f ms = %.4f ms/iteration (SpMV alone "
           "%.4f ms)",
           n, (long long)A.nnz(), it, it_o, nr, std::sqrt(num / std::max(den, 1e-300)), ms, ms / std::max(it, 1), spmv_ms);
  }
  b200sp_spmv_plan_destroy(plan, nullptr);
}

// ------------------------------------------------------------------------------------------------
// suite: solvers -- point Gauss-Seidel (colouring, sweeps), the SGS-preconditioned CG and GMRES against the oracle, with the times
// that matter next to the SpMV's: symbolic, one symmetric sweep, PCG and GMRES per iteration
// ------------------------------------------------------------------------------------------------
static void suite_solvers() {
  Csr<double> A = gen_lap27<double>(g_big ? 128 : 20, 1);
  for (int r = 0; r < A.m; ++r)
    for (int q = A.rp[r]; q < A.rp[r + 1]; ++q)
      if (A.ci[q] == r) A.v[q] += 0.5;
  const int n = A.m;
  std::vector<double> xs((size_t)n), b((size_t)n, 0.0), dinv((size_t)n, 1.0);
  b200gen_fill_f64(n, xs.data(), -1.0, 1.0, 9);
  okk_spmv_serial_f64(n, A.rp.data(), A.ci.data(), A.v.data(), xs.data(), b.data(), 1.0, 0.0);
  for (int r = 0; r < n; ++r)
    for (int q = A.rp[r]; q < A.rp[r + 1]; ++q)
      if (A.ci[q] == r) dinv[r] = 1.0 / A.v[q];
  Dev<int> rp(A.rp), ci(A.ci);
  Dev<double> v(A.v), db(b), dx((size_t)n);
  b200sp_spmv_plan* plan = nullptr;
  SP(b200sp_spmv_plan_create(&plan, 0));
  float spmv_ms = 1e30f;
  for (int rep = 0; rep < 6; ++rep) {
    Timer t;
    t.start();
    SP(b200sp_spmv_f64_i32(plan, nullptr, 'N', n, n, A.nnz(), 1.0, rp.p, ci.p, v.p, db.p, 0.0, dx.p));
    spmv_ms = std::min(spmv_ms, t.stop_ms());
  }
  // ---- Gauss-Seidel
  b200sp_gs_plan* gs = nullptr;
  SP(b200sp_gs_plan_create(&gs));
  double t0 = now_s();
  SP(b200sp_gs_symbolic_i32(gs, nullptr, n, rp.p, ci.p, 1));
  const double sym_ms = (now_s() - t0) * 1e3;
  SP(b200sp_gs_numeric_f64_i32(gs, nullptr, n, rp.p, ci.p, v.p));
  int nc = 0;
  SP(b200sp_gs_get_coloring(gs, &nc, nullptr, nullptr, nullptr));
  std::vector<int> colors((size_t)n), cptr((size_t)nc + 1), crows((size_t)n);
  SP(b200sp_gs_copy_coloring(gs, nullptr, colors.data(), cptr.data(), crows.data()));
  int64_t clashes = 0;
  for (int r = 0; r < n; ++r)
    for (int q = A.rp[r]; q < A.rp[r + 1]; ++q)
      if (A.ci[q] != r && colors[A.ci[q]] == colors[r]) ++clashes;
  for (int direction = 0; direction < 3; ++direction) {
    float best = 1e30f;
    for (int rep = 0; rep < 3; ++rep) {
      Timer t;
      t.start();
      SP(b200sp_gs_apply_f64_i32(gs, nullptr, n, rp.p, ci.p, v.p, dx.p, db.p, 1, 0.9, 2, direction));
      best = std::min(best, t.stop_ms());
    }
    auto x = dx.host();
    std::vector<double> xo((size_t)n, 0.0);
    okk_gs_apply_f64(n, A.rp.data(), A.ci.data(), A.v.data(), nc, cptr.data(), crows.data(), dinv.data(), b.data(), xo.data(), 1, 0.9, 2, direction);
    double worst = 0, err = 0, nrm = 0;
    for (int i = 0; i < n; ++i) {
      worst = std::max(worst, std::fabs(x[i] - xo[i]));
      err += (x[i] - xs[i]) * (x[i] - xs[i]);
      nrm += xs[i] * xs[i];
    }
    char nm[96];
    snprintf(nm, sizeof(nm), "gauss_seidel/%s", direction == 0 ? "symmetric" : direction == 1 ? "forward" : "backward");
    record(nm, clashes == 0 && worst <= 1e-12 && err < nrm,
           "n=%d: %d colours (%lld clashes), symbolic %.2f ms; 2 sweeps %.3f ms (SpMV %.4f ms), max |x - x_oracle| %.1e, error norm %.3f of the "
           "initial one",
           n, nc, (long long)clashes, sym_ms, best, spmv_ms, worst, std::sqrt(err / nrm));
  }
  // ---- two-stage Gauss-Seidel (every product the library's SpMV): classic and compact recurrence, 1 and 3 inner sweeps
  for (int compact = 0; compact <= 1; ++compact)
    for (int inner : {1, 3}) {
      b200sp_gs2_plan* g2 = nullptr;
      SP(b200sp_gs2_plan_create(&g2));
      SP(b200sp_gs2_plan_set(g2, B200SP_GS2_COMPACT_FORM, compact));
      SP(b200sp_gs2_plan_set(g2, B200SP_GS2_NUM_INNER_SWEEPS, inner));
      t0 = now_s();
      SP(b200sp_gs2_symbolic_i32(g2, nullptr, n, n, rp.p, ci.p));
      SP(b200sp_gs2_numeric_f64_i32(g2, nullptr, n, n, rp.p, ci.p, v.p, nullptr));
      CK(cudaDeviceSynchronize());
      const double setup_ms = (now_s() - t0) * 1e3;
      float best = 1e30f;
      for (int rep = 0; rep < 4; ++rep) {
        Timer t;
        t.start();
        SP(b200sp_gs2_apply_f64_i32(g2, nullptr, n, n, rp.p, ci.p, v.p, dx.p, n, db.p, n, 1, 1, 0.9, 2, 0));
        const float ms = t.stop_ms();
        if (rep > 0) best = std::min(best, ms);
      }
      auto x = dx.host();
      std::vector<double> xo((size_t)n, 0.0);
      okk_gs2_apply_f64(n, n, A.rp.data(), A.ci.data(), A.v.data(), nullptr, compact, inner, 1, 1.0, xo.data(), b.data(), 1, 0.9, 2, 0);
      double worst = 0, err = 0, nrm = 0;
      for (int i = 0; i < n; ++i) {
        worst = std::max(worst, std::fabs(x[i] - xo[i]));
        err += (x[i] - xs[i]) * (x[i] - xs[i]);
        nrm += xs[i] * xs[i];
      }
      char nm[96];
      snprintf(nm, sizeof(nm), "two_stage_gs/%s/inner%d", compact ? "compact" : "classic", inner);
      // 2 symmetric sweeps = 4 sweeps of (residual SpMV with A unless skipped) + `inner` SpMVs with L or U (half of A each)
      record(nm, g_dry || (worst <= 1e-12 && err < nrm),
             "symbolic + numeric %.2f ms; 2 symmetric sweeps %.3f ms = %.1f x the SpMV of A (%.4f ms), max |x - x_oracle| %.1e, error norm %.3f of the "
             "initial one",
             setup_ms, best, best / spmv_ms, spmv_ms, worst, std::sqrt(err / nrm));
      if (!g_dry) b200sp_gs2_plan_destroy(g2, nullptr);
    }
  // ---- PCG (symmetric Gauss-Seidel preconditioner) next to plain CG
  {
    std::vector<double> xo((size_t)n, 0.0), xc((size_t)n, 0.0);
    double nr_o = 0, nr_c = 0;
    const int it_o = okk_pcg_f64(n, A.rp.data(), A.ci.data(), A.v.data(), b.data(), xo.data(), 100000, 1e-7, &nr_o, nc, cptr.data(), crows.data(),
                                 dinv.data());
    const int it_c = okk_cg_f64(n, A.rp.data(), A.ci.data(), A.v.data(), b.data(), xc.data(), 100000, 1e-7, &nr_c);
    dx.fill_bytes(0);
    int it = 0;
    double nr = 0;
    t0 = now_s();
    SP(b200sp_pcg_solve_f64_i32(plan, gs, nullptr, n, A.nnz(), rp.p, ci.p, v.p, db.p, dx.p, 100000, 1e-7, 8, &it, &nr));
    const double ms = (now_s() - t0) * 1e3;
    auto x = dx.host();
    double num = 0, den = 0;
    for (int i = 0; i < n; ++i) {
      num += (x[i] - xo[i]) * (x[i] - xo[i]);
      den += xo[i] * xo[i];
    }
    record("pcg_sgs", std::abs(it - it_o) <= 1 && nr <= 1e-7 && std::sqrt(num / std::max(den, 1e-300)) < 1e-8,
           "%d iterations (oracle %d; plain CG %d), norm_res %.2e, |x-x_oracle|/|x_oracle| %.1e; %.3f ms = %.4f ms/iteration (SpMV %.4f ms)", it,
           it_o, it_c, nr, std::sqrt(num / std::max(den, 1e-300)), ms, ms / std::max(it, 1), spmv_ms);
  }
  // ---- PCG with the two-stage Gauss-Seidel as preconditioner (1 and 2 inner sweeps), next to plain CG.  The inner Jacobi-Richardson
  // sweeps need |D^-1 L| well below 1, which the stencil matrix above (positive off-diagonals summing to the diagonal) does not offer:
  // the same pattern with the diagonal raised to 1.5 x the off-diagonal row sum
  {
    Csr<double> A2 = A;
    for (int r = 0; r < n; ++r) {
      double off = 0;
      for (int q = A2.rp[r]; q < A2.rp[r + 1]; ++q)
        if (A2.ci[q] != r) off += std::fabs(A2.v[q]);
      for (int q = A2.rp[r]; q < A2.rp[r + 1]; ++q)
        if (A2.ci[q] == r) A2.v[q] = 1.5 * off + 1.0;
    }
    std::vector<double> b2((size_t)n, 0.0), xc((size_t)n, 0.0);
    okk_spmv_serial_f64(n, A2.rp.data(), A2.ci.data(), A2.v.data(), xs.data(), b2.data(), 1.0, 0.0);
    double nr_c = 0;
    const int it_c = okk_cg_f64(n, A2.rp.data(), A2.ci.data(), A2.v.data(), b2.data(), xc.data(), 500, 1e-7, &nr_c);
    Dev<double> v2(A2.v), db2(b2);
    b200sp_spmv_plan* plan2 = nullptr;
    SP(b200sp_spmv_plan_create(&plan2, 0));
    for (int inner : {1, 2}) {
      std::vector<double> xo((size_t)n, 0.0);
      double nr_o = 0;
      const int it_o = okk_pcg_gs2_f64(n, A2.rp.data(), A2.ci.data(), A2.v.data(), b2.data(), xo.data(), 500, 1e-7, &nr_o, inner, 0);
      b200sp_gs2_plan* g2 = nullptr;
      SP(b200sp_gs2_plan_create(&g2));
      SP(b200sp_gs2_plan_set(g2, B200SP_GS2_NUM_INNER_SWEEPS, inner));
      SP(b200sp_gs2_symbolic_i32(g2, nullptr, n, n, rp.p, ci.p));
      SP(b200sp_gs2_numeric_f64_i32(g2, nullptr, n, n, rp.p, ci.p, v2.p, nullptr));
      dx.fill_bytes(0);
      int it = 0;
      double nr = 0;
      t0 = now_s();
      SP(b200sp_pcg_solve_gs2_f64_i32(plan2, g2, nullptr, n, A2.nnz(), rp.p, ci.p, v2.p, db2.p, dx.p, 500, 1e-7, 8, &it, &nr));
      const double ms = (now_s() - t0) * 1e3;
      auto x = dx.host();
      double num = 0, den = 0;
      for (int i = 0; i < n; ++i) {
        num += (x[i] - xo[i]) * (x[i] - xo[i]);
        den += xo[i] * xo[i];
      }
      char nm[64];
      snprintf(nm, sizeof(nm), "pcg_two_stage_gs/inner%d", inner);
      record(nm, g_dry || (std::abs(it - it_o) <= 1 && it < it_c && nr <= 1e-7 && std::sqrt(num / std::max(den, 1e-300)) < 1e-7),
             "%d iterations (oracle %d; plain CG %d), norm_res %.2e, |x-x_oracle|/|x_oracle| %.1e; %.3f ms = %.4f ms/iteration (SpMV %.4f ms)", it,
             it_o, it_c, nr, std::sqrt(num / std::max(den, 1e-300)), ms, ms / std::max(it, 1), spmv_ms);
      if (!g_dry) b200sp_gs2_plan_destroy(g2, nullptr);
    }
    if (!g_dry) b200sp_spmv_plan_destroy(plan2, nullptr);
  }
  // ---- GMRES(15), CGS2 and MGS
  for (int ortho = 0; ortho < 2; ++ortho) {
    std::vector<double> xo((size_t)n, 0.0);
    int it_o = 0, flag_o = 0;
    double res_o = 0;
    okk_gmres_f64(n, A.rp.data(), A.ci.data(), A.v.data(), nullptr, nullptr, nullptr, b.data(), xo.data(), 15, 1e-8, 50, ortho, &it_o, &res_o,
                  &flag_o);
    dx.fill_bytes(0);
    int it = 0, flag = 0;
    double res = 0;
    t0 = now_s();
    SP(b200sp_gmres_f64_i32(plan, nullptr, n, A.nnz(), rp.p, ci.p, v.p, nullptr, 0, nullptr, nullptr, nullptr, db.p, dx.p, 15, 1e-8, 50, ortho, &it,
                            &res, &flag));
    const double ms = (now_s() - t0) * 1e3;
    record(ortho ? "gmres15/mgs" : "gmres15/cgs2", flag == 0 && flag_o == 0 && std::abs(it - it_o) <= 1 && res < 1e-8,
           "%d iterations (oracle %d), relative residual %.2e, flag %d; %.3f ms = %.4f ms/iteration (SpMV %.4f ms)", it, it_o, res, flag, ms,
           ms / std::max(it, 1), spmv_ms);
  }
  b200sp_gs_plan_destroy(gs, nullptr);
  b200sp_spmv_plan_destroy(plan, nullptr);
}

// ------------------------------------------------------------------------------------------------
// suite: spmm_sweep -- the rank-2 kernels over column counts / scalar types / leading dimensions / beta
// ------------------------------------------------------------------------------------------------
static void ospmm(int m, int n, int k, const Csr<double>& A, const double* X, int64_t ldx, double* Y, int64_t ldy, double al, double be) {
  okk_spmv_mv_f64(m, n, k, A.rp.data(), A.ci.data(), A.v.data(), X, ldx, 1, Y, ldy, 1, al, be, 1);
}
static void ospmm(int m, int n, int k, const Csr<float>& A, const float* X, int64_t ldx, float* Y, int64_t ldy, float al, float be) {
  okk_spmv_mv_f32(m, n, k, A.rp.data(), A.ci.data(), A.v.data(), X, ldx, 1, Y, ldy, 1, al, be, 1);
}
static int gspmm(b200sp_spmv_plan* p, int m, int n, int64_t nnz, int k, double al, const int* rp, const int* ci, const double* v,
                 const double* X, int64_t ldx, double be, double* Y, int64_t ldy) {
  return b200sp_spmm_f64_i32(p, nullptr, 'N', m, n, nnz, k, al, rp, ci, v, X, ldx, 1, be, Y, ldy, 1);
}
static int gspmm(b200sp_spmv_plan* p, int m, int n, int64_t nnz, int k, float al, const int* rp, const int* ci, const float* v,
                 const float* X, int64_t ldx, float be, float* Y, int64_t ldy) {
  return b200sp_spmm_f32_i32(p, nullptr, 'N', m, n, nnz, k, al, rp, ci, v, X, ldx, 1, be, Y, ldy, 1);
}

template <typename S>
static void spmm_sweep_matrix(const char* name, const Csr<S>& A) {
  const int ks[] = {1, 2, 3, 4, 5, 8, 10, 16, 17, 30, 32, 33, 64};
  Dev<int> rp(A.rp), ci(A.ci);
  Dev<S> v(A.v);
  Csr<S> Aabs = A;
  for (auto& t : Aabs.v) t = std::fabs(t);
  const double tol = sizeof(S) == 8 ? 1e-13 : 2e-5;
  for (const char* kern : {"tilev", "tile", "split", "tilev+segvec"}) {
    const bool segvec = strstr(kern, "segvec") != nullptr;
    setenv("B200SP_SPMM_KERNEL", segvec ? "tilev" : kern, 1);
    if (segvec) setenv("B200SP_SPMM_SEG", "vec", 1);
    else unsetenv("B200SP_SPMM_SEG");
    int bad = 0, runs = 0;
    double worst = 0;
    std::string last;
    for (int k : ks) {
      for (int pad = 0; pad <= 3; pad += 3) {
        for (int bz = 0; bz <= 1; ++bz) {
          const int64_t ldx = k + pad, ldy = k + (pad ? 1 : 0);
          const S al = (S)1.25, be = bz ? (S)0 : (S)-0.5;
          std::vector<S> X((size_t)A.n * ldx), Y0((size_t)A.m * ldy);
          fill_vals(X, -1.0, 1.0, 100 + k);
          fill_vals(Y0, -1.0, 1.0, 200 + k);
          std::vector<S> Yref = Y0, Xa = X, Ys = Y0;
          ospmm(A.m, A.n, k, A, X.data(), ldx, Yref.data(), ldy, al, be);
          for (auto& t : Xa) t = std::fabs(t);
          for (auto& t : Ys) t = std::fabs(t);
          ospmm(A.m, A.n, k, Aabs, Xa.data(), ldx, Ys.data(), ldy, (S)std::fabs(al), (S)std::fabs(be));
          std::vector<S> Yin = Y0;
          if (bz)  // beta == 0 must overwrite NaN (Test_Sparse_spmv.hpp:394-408)
            for (int r = 0; r < A.m; r += 19)
              for (int j = 0; j < k; ++j) Yin[(size_t)r * ldy + j] = std::numeric_limits<S>::quiet_NaN();
          Dev<S> dX(X), dY(Yin);
          b200sp_spmv_plan* plan = nullptr;
          SP(b200sp_spmv_plan_create(&plan, 0));
          SP(gspmm(plan, A.m, A.n, A.nnz(), k, al, rp.p, ci.p, v.p, dX.p, ldx, be, dY.p, ldy));
          CK(cudaDeviceSynchronize());
          last = b200sp_spmv_last_kernel(plan);
          b200sp_spmv_plan_destroy(plan, nullptr);
          auto got = dY.host();
          ++runs;
          bool ok = true;
          for (int r = 0; r < A.m && ok; ++r) {
            for (int j = 0; j < (int)ldy; ++j) {
              const size_t i = (size_t)r * ldy + j;
              if (j >= k) {  // padding columns must stay untouched
                if (memcmp(&got[i], &Yin[i], sizeof(S)) != 0) ok = false;
                continue;
              }
              const double err = std::fabs((double)got[i] - (double)Yref[i]) / std::max((double)Ys[i], 1e-300);
              if (!(err <= tol)) ok = false;
              if (err == err) worst = std::max(worst, err);
            }
          }
          if (!ok) {
            ++bad;
            fprintf(stderr, "    mismatch: %s kernel=%s k=%d ldx=%lld beta=%g\n", name, last.c_str(), k, (long long)ldx, (double)be);
          }
        }
      }
    }
    char nm[128];
    snprintf(nm, sizeof(nm), "%s/%s", name, kern);
    record(nm, bad == 0, "%d runs (13 column counts x 2 leading dimensions x beta in {0, -0.5}), %d bad, max scaled err %.2e, last kernel %s",
           runs, bad, worst, last.c_str());
  }
  unsetenv("B200SP_SPMM_KERNEL");
  unsetenv("B200SP_SPMM_SEG");
}

static void suite_spmm_sweep() {
  {
    auto A = gen_kk<double>(1000, 963, 20000, 5, 100, 3);
    for (auto& t : A.v) t = (t - 25.0) / 25.0;
    spmm_sweep_matrix("kk_1000x963_f64", A);
  }
  {
    auto A = gen_kk<float>(5000, 4963, 150000, 20, 400, 4);
    for (auto& t : A.v) t = (t - 25.0f) / 25.0f;
    spmm_sweep_matrix("kk_5000x4963_f32", A);
  }
  {
    // power-law rows incl. rows beyond the tile row limit (segment kernel, multi-segment atomics)
    int64_t nnz = 0;
    void* h = b200gen_rmat_build(13, 16, 0.57, 0.19, 0.19, 23, &nnz);
    Csr<float> A;
    A.m = A.n = 1 << 13;
    A.rp.resize((size_t)A.m + 1);
    A.ci.resize((size_t)nnz);
    b200gen_rmat_emit(h, A.rp.data(), A.ci.data());
    A.v.resize((size_t)nnz);
    fill_vals(A.v, -1.0, 1.0, 9);
    spmm_sweep_matrix("rmat13_f32", A);
  }
  {
    // very long rows (several segments each, combined with atomics), rows just around the tile row limit, empty rows
    Rng r(31);
    std::vector<int> lens(6000);
    for (auto& l : lens) l = r.below(25);
    const int special[] = {10000, 0, 0, 4097, 2049, 2048, 300, 257, 256, 255, 0, 1};
    for (size_t i = 0; i < sizeof(special) / sizeof(int); ++i) lens[100 + i] = special[i];
    auto B = gen_rows<double>(lens, 5000, false, false, 31);
    for (auto& t : B.v) t = (t - 25.0) / 25.0;
    spmm_sweep_matrix("long_rows_6000x5000_f64", B);
  }
}

// ------------------------------------------------------------------------------------------------
// suite: jacobi -- spgemm_jacobi (C = (I - omega D^-1 A) B) against the oracle's spgemm_jacobi_seq
// ------------------------------------------------------------------------------------------------
static void jacobi_case(const char* name, Csr<double> A, bool add_diagonal) {
  // diagonally dominant like the reference test: diagonal = 10 * sum |row| (+1), rows sorted
  if (add_diagonal) {
    Csr<double> D;
    D.m = A.m;
    D.n = A.n;
    D.rp.assign(A.m + 1, 0);
    for (int i = 0; i < A.m; ++i) {
      std::vector<std::pair<int, double>> row;
      double sum = 0;
      for (int j = A.rp[i]; j < A.rp[i + 1]; ++j)
        if (A.ci[j] != i) {
          const double v = (A.v[j] - 25.0) / 25.0;
          row.emplace_back(A.ci[j], v);
          sum += std::fabs(v);
        }
      row.emplace_back(i, 10.0 * sum + 1.0);
      std::sort(row.begin(), row.end());
      row.erase(std::unique(row.begin(), row.end(), [](auto& x, auto& y) { return x.first == y.first; }), row.end());
      for (auto& pr : row) {
        D.ci.push_back(pr.first);
        D.v.push_back(pr.second);
      }
      D.rp[i + 1] = (int)D.ci.size();
    }
    A = D;
  }
  const int m = A.m;
  const double omega = 3.0;
  std::vector<double> dinv((size_t)m, 2.0);
  std::vector<int> orp((size_t)m + 1, 0);
  const int64_t onnz = okk_spgemm_symbolic(m, m, A.rp.data(), A.ci.data(), A.rp.data(), A.ci.data(), orp.data());
  std::vector<int> oci(onnz);
  std::vector<double> ov(onnz);
  okk_spgemm_jacobi_f64(m, m, A.rp.data(), A.ci.data(), A.v.data(), A.rp.data(), A.ci.data(), A.v.data(), orp.data(), oci.data(), ov.data(),
                        omega, dinv.data());
  okk_sort_crs_f64(m, orp.data(), oci.data(), ov.data());
  Dev<int> rp(A.rp), ci(A.ci), rpC((size_t)m + 1);
  Dev<double> v(A.v), dd(dinv);
  b200sp_spgemm_plan* plan = nullptr;
  SP(b200sp_spgemm_plan_create(&plan));
  int64_t c_nnz = -1;
  int c_max = -1;
  SP(b200sp_spgemm_symbolic_i32(plan, nullptr, m, m, m, rp.p, ci.p, rp.p, ci.p, rpC.p, &c_nnz, &c_max));
  bool ok = c_nnz == onnz && count_diff(rpC.host(), orp) == 0;
  int64_t dci = -1, dv = -1;
  float ms = 0;
  if (ok) {
    Dev<int> ciC((size_t)c_nnz);
    Dev<double> vC((size_t)c_nnz);
    ciC.fill_bytes(0xff);
    vC.fill_bytes(0xff);
    Timer t;
    t.start();
    SP(b200sp_spgemm_jacobi_f64_i32(plan, nullptr, m, m, m, rp.p, ci.p, v.p, rp.p, ci.p, v.p, rpC.p, ciC.p, vC.p, omega, dd.p));
    ms = t.stop_ms();
    CK(cudaDeviceSynchronize());
    dci = count_diff(ciC.host(), oci);
    dv = rel_mismatch(vC.host(), ov, 1e-7);
    ok = dci == 0 && dv == 0;
  }
  b200sp_spgemm_plan_destroy(plan, nullptr);
  record(name, ok, "m=%d c_nnz=%lld (oracle %lld) col_idx diffs=%lld value law violations=%lld, %.3f ms", m, (long long)c_nnz, (long long)onnz,
         (long long)dci, (long long)dv, ms);
}

static void suite_jacobi() {
  jacobi_case("kk_1000_diag_dominant", gen_kk<double>(1000, 1000, 10000, 10, 50, 1), true);
  jacobi_case("kk_30000_diag_dominant", gen_kk<double>(30000, 30000, 240000, 6, 3000, 2), true);
  {
    Rng r(3);
    std::vector<int> lens(8000);
    for (auto& l : lens) l = r.below(12);
    lens[0] = 3000;  // rows in the large shared-memory bins and in the global fallback
    lens[1] = 700;
    jacobi_case("wide_rows_8000_diag_dominant", gen_rows<double>(lens, 8000, true, false, 3), true);
  }
  jacobi_case("lap27_10x2dof", gen_lap27<double>(10, 2), false);  // has its diagonal already
}

// ------------------------------------------------------------------------------------------------
// suite: spmv_longrows -- rank-1 SpMV on a power-law matrix: one CTA per long row (default) vs segments
// ------------------------------------------------------------------------------------------------
static void suite_spmv_longrows() {
  const int scale = g_big ? 22 : 18;
  int64_t nnz = 0;
  void* h = b200gen_rmat_build(scale, 16, 0.57, 0.19, 0.19, 23, &nnz);
  Csr<double> A;
  A.m = A.n = 1 << scale;
  A.rp.resize((size_t)A.m + 1);
  A.ci.resize((size_t)nnz);
  b200gen_rmat_emit(h, A.rp.data(), A.ci.data());
  A.v.resize((size_t)nnz);
  b200gen_fill_f64(nnz, A.v.data(), -1.0, 1.0, 3);
  std::vector<double> x((size_t)A.n), y0((size_t)A.m), yref, scale_v, va(A.v), xa;
  b200gen_fill_f64(A.n, x.data(), -1.0, 1.0, 4);
  b200gen_fill_f64(A.m, y0.data(), -1.0, 1.0, 5);
  const double alpha = 1.25, beta = -0.5;
  yref = y0;
  okk_spmv_serial_f64(A.m, A.rp.data(), A.ci.data(), A.v.data(), x.data(), yref.data(), alpha, beta);
  xa = x;
  scale_v = y0;
  for (auto& t : va) t = std::fabs(t);
  for (auto& t : xa) t = std::fabs(t);
  for (auto& t : scale_v) t = std::fabs(t);
  okk_spmv_serial_f64(A.m, A.rp.data(), A.ci.data(), va.data(), xa.data(), scale_v.data(), std::fabs(alpha), std::fabs(beta));
  int maxrow = 0;
  for (int i = 0; i < A.m; ++i) maxrow = std::max(maxrow, A.rp[i + 1] - A.rp[i]);
  Dev<int> rp(A.rp), ci(A.ci);
  Dev<double> v(A.v), dx(x), dy((size_t)A.m);
  setenv("B200SP_NO_AUTOTUNE", "1", 1);  // stay on the tiled kernel: the comparison is about its long-row path
  for (int seg = 0; seg <= 1; ++seg) {
    if (seg) setenv("B200SP_SPMV_LONGROWS", "seg", 1);
    else unsetenv("B200SP_SPMV_LONGROWS");
    b200sp_spmv_plan* plan = nullptr;
    SP(b200sp_spmv_plan_create(&plan, 0));
    float best = 1e30f;
    std::vector<double> got, first;
    for (int rep = 0; rep < 5; ++rep) {
      CK(cudaMemcpy(dy.p, y0.data(), y0.size() * sizeof(double), cudaMemcpyHostToDevice));
      Timer t;
      t.start();
      SP(b200sp_spmv_f64_i32(plan, nullptr, 'N', A.m, A.n, nnz, alpha, rp.p, ci.p, v.p, dx.p, beta, dy.p));
      const float ms = t.stop_ms();
      if (rep > 0) best = std::min(best, ms);
      got = dy.host();
      if (rep == 0) first = got;
    }
    double worst = 0;
    for (size_t i = 0; i < got.size(); ++i) worst = std::max(worst, std::fabs(got[i] - yref[i]) / std::max(scale_v[i], 1e-300));
    const double balg = 12.0 * nnz + 4.0 * (A.m + 1) + 8.0 * A.n + 16.0 * A.m;
    record(seg ? "rmat_f64/segments" : "rmat_f64/cta_per_row", worst <= 1e-10 && count_diff(got, first) == 0,
           "scale %d nnz=%lld longest row %d: kernel=%s %.3f ms (%.0f GB/s algorithmic), max scaled err %.2e, run-to-run differing entries %lld",
           scale, (long long)nnz, maxrow, b200sp_spmv_last_kernel(plan), best, balg / (best * 1e-3) / 1e9, worst,
           (long long)count_diff(got, first));
    b200sp_spmv_plan_destroy(plan, nullptr);
  }
  unsetenv("B200SP_SPMV_LONGROWS");
  unsetenv("B200SP_NO_AUTOTUNE");
}

// ------------------------------------------------------------------------------------------------
// suite: spmv64 -- SpMV on 64-bit offsets (spmv64.cu).  (1) a stencil matrix cut into many small windows and into one: equal
// bits to the 32-bit entry point, timings side by side (the windows must cost nothing but their launches); (2) with --big, a
// matrix PAST 2^31 entries: B = lap27(128) stacked K times (A = [B; B; ...], K*mB rows, same columns), entries and values
// replicated on the device, the int64 row map computed on the host; every block of y must equal, bit for bit, the 32-bit SpMV
// of B, which is checked against the oracle.  26 GB of matrix for fp64 + int32 columns.
// ------------------------------------------------------------------------------------------------
static void suite_spmv64() {
  // B200SP_SPMV64_SMALL=1: the --big logic on a small grid with a lowered window (what the CPU emulation can run)
  const bool small = getenv("B200SP_SPMV64_SMALL") != nullptr;
  {
    Csr<double> A = gen_lap27<double>(g_big && !small ? 100 : 30, 2);
    const int n = A.m;
    Rng r(77);
    std::vector<double> x((size_t)n), y0((size_t)n), yref;
    for (auto& t : x) t = 2 * r.u01() - 1;
    for (auto& t : y0) t = 2 * r.u01() - 1;
    const double alpha = 1.5, beta = -0.25;
    yref = y0;
    okk_spmv_serial_f64(A.m, A.rp.data(), A.ci.data(), A.v.data(), x.data(), yref.data(), alpha, beta);
    std::vector<int64_t> rp64(A.rp.begin(), A.rp.end()), ci64(A.ci.begin(), A.ci.end());
    Dev<int> rp(A.rp), ci(A.ci);
    Dev<int64_t> drp64(rp64), dci64(ci64);
    Dev<double> v(A.v), dx(x), dy((size_t)n);
    auto run = [&](const char* what, std::function<int()> call, std::vector<double>* out) {
      float best = 1e30f;
      for (int rep = 0; rep < 6; ++rep) {
        CK(cudaMemcpy(dy.p, y0.data(), y0.size() * sizeof(double), cudaMemcpyHostToDevice));
        Timer t;
        t.start();
        SP(call());
        const float ms = t.stop_ms();
        if (rep > 0) best = std::min(best, ms);
      }
      *out = dy.host();
      (void)what;
      return best;
    };
    b200sp_spmv_plan* p32 = nullptr;
    SP(b200sp_spmv_plan_create(&p32, 0));
    std::vector<double> g32;
    const float ms32 = run("i32", [&] { return b200sp_spmv_f64_i32(p32, nullptr, 'N', n, n, A.nnz(), alpha, rp.p, ci.p, v.p, dx.p, beta, dy.p); }, &g32);
    double worst = 0;
    for (size_t i = 0; i < g32.size(); ++i) worst = std::max(worst, std::fabs(g32[i] - yref[i]) / std::max(1.0, std::fabs(yref[i])));
    record("i32_vs_oracle", worst <= 1e-12, "lap27 x 2 dof, %d rows, %lld entries: %.3f ms, max rel err %.2e, kernel %s", n, (long long)A.nnz(), ms32,
           worst, g_dry ? "-" : b200sp_spmv_last_kernel(p32));
    for (int bits : {32, 64})
      for (int64_t window : {(int64_t)0, (int64_t)A.nnz() / 7 + 11}) {
        b200sp_spmv64_plan* p64 = nullptr;
        SP(b200sp_spmv64_plan_create(&p64, 0));
        if (window) SP(b200sp_spmv64_plan_set_window(p64, window));
        std::vector<double> g64;
        const void* cols = bits == 64 ? (const void*)dci64.p : (const void*)ci.p;
        const float ms64 = run("i64", [&] { return b200sp_spmv_f64_i64(p64, nullptr, 'N', n, n, A.nnz(), alpha, drp64.p, cols, bits, v.p, dx.p, beta, dy.p); }, &g64);
        const int64_t diff = g_dry ? 0 : count_diff(g64, g32);
        char nm[96];
        snprintf(nm, sizeof(nm), "cols%d/%s", bits, window ? "8_windows" : "1_window");
        record(nm, diff == 0 && (g_dry || b200sp_spmv64_plan_windows(p64) == (window ? 8 : 1)),
               "%d window(s), %.3f ms (32-bit entry %.3f ms), entries differing from the 32-bit result: %lld; %s", g_dry ? 0 : b200sp_spmv64_plan_windows(p64),
               ms64, ms32, (long long)diff, g_dry ? "-" : b200sp_spmv64_last_kernel(p64));
        // transposed: accumulated window by window
        std::vector<double> yt = y0;
        okk_spmv_transpose_f64(A.m, A.n, A.rp.data(), A.ci.data(), A.v.data(), x.data(), yt.data(), alpha, beta);
        CK(cudaMemcpy(dy.p, y0.data(), y0.size() * sizeof(double), cudaMemcpyHostToDevice));
        SP(b200sp_spmv_f64_i64(p64, nullptr, 'T', n, n, A.nnz(), alpha, drp64.p, cols, bits, v.p, dx.p, beta, dy.p));
        std::vector<double> gt = dy.host();
        double wt = 0;
        for (size_t i = 0; i < gt.size(); ++i) wt = std::max(wt, std::fabs(gt[i] - yt[i]) / std::max(1.0, std::fabs(yt[i])));
        snprintf(nm, sizeof(nm), "cols%d/%s/transposed", bits, window ? "8_windows" : "1_window");
        record(nm, g_dry || wt <= 1e-12, "max rel err vs the oracle %.2e", wt);
        if (!g_dry) b200sp_spmv64_plan_destroy(p64, nullptr);
      }
    if (!g_dry) b200sp_spmv_plan_destroy(p32, nullptr);
  }
  if (!g_big) {
    record("past_2^31_entries", true, "skipped (needs --big: 26 GB of matrix)");
    return;
  }
  // ---- past 2^31 entries
  Csr<double> B = gen_lap27<double>(small ? 12 : 128, 1);  // 2,097,152 rows, 55.7 M entries
  const int mB = B.m, nB = B.n;
  const int64_t nzB = B.nnz();
  const int K = small ? 5 : (int)(((int64_t)1 << 31) / nzB) + 2;
  const int64_t nnz = nzB * K;
  const int64_t m = (int64_t)mB * K;
  Rng r(5);
  std::vector<double> x((size_t)nB), yB((size_t)mB, 0.0);
  for (auto& t : x) t = 2 * r.u01() - 1;
  okk_spmv_serial_f64(mB, B.rp.data(), B.ci.data(), B.v.data(), x.data(), yB.data(), 1.0, 0.0);
  std::vector<int64_t> rp64((size_t)m + 1);
  for (int k = 0; k < K; ++k)
    for (int i = 0; i <= mB; ++i) rp64[(size_t)k * mB + i] = (int64_t)k * nzB + B.rp[(size_t)i];
  Dev<int> rpB(B.rp), ciB(B.ci);
  Dev<double> vB(B.v), dx(x), dyB((size_t)mB), dy((size_t)m);
  Dev<int64_t> drp64(rp64);
  Dev<int> ci((size_t)nnz);
  Dev<double> v((size_t)nnz);
  for (int k = 0; k < K; ++k) {
    CK(cudaMemcpy(ci.p + (size_t)k * nzB, ciB.p, sizeof(int) * (size_t)nzB, cudaMemcpyDeviceToDevice));
    CK(cudaMemcpy(v.p + (size_t)k * nzB, vB.p, sizeof(double) * (size_t)nzB, cudaMemcpyDeviceToDevice));
  }
  b200sp_spmv_plan* p32 = nullptr;
  SP(b200sp_spmv_plan_create(&p32, 0));
  float msB = 1e30f;
  for (int rep = 0; rep < 5; ++rep) {
    Timer t;
    t.start();
    SP(b200sp_spmv_f64_i32(p32, nullptr, 'N', mB, nB, nzB, 1.0, rpB.p, ciB.p, vB.p, dx.p, 0.0, dyB.p));
    const float ms = t.stop_ms();
    if (rep > 0) msB = std::min(msB, ms);
  }
  std::vector<double> gB = dyB.host();
  double worst = 0;
  for (size_t i = 0; i < gB.size(); ++i) worst = std::max(worst, std::fabs(gB[i] - yB[i]) / std::max(1.0, std::fabs(yB[i])));
  record("block_vs_oracle", worst <= 1e-12, "one block (lap27): %d rows, %lld entries, %.3f ms, max rel err %.2e", mB, (long long)nzB, msB, worst);
  b200sp_spmv64_plan* p64 = nullptr;
  SP(b200sp_spmv64_plan_create(&p64, 0));
  if (small) SP(b200sp_spmv64_plan_set_window(p64, nzB + nzB / 2));
  float ms64 = 1e30f;
  for (int rep = 0; rep < 5; ++rep) {
    dy.fill_bytes(0xFF);
    Timer t;
    t.start();
    SP(b200sp_spmv_f64_i64(p64, nullptr, 'N', m, nB, nnz, 1.0, drp64.p, ci.p, 32, v.p, dx.p, 0.0, dy.p));
    const float ms = t.stop_ms();
    if (rep > 0) ms64 = std::min(ms64, ms);
  }
  int64_t diff = 0;
  for (int k = 0; k < K; ++k) diff += count_diff(dy.host((size_t)k * mB, (size_t)mB), gB);
  const double gbs = ((double)nnz * 12 + (double)m * 12 + (double)nB * 8) / (ms64 * 1e-3) / 1e9;
  record("past_2^31_entries", diff == 0 && b200sp_spmv64_plan_windows(p64) >= 2,
         "%d stacked blocks: %lld rows, %lld entries (2^31 = 2147483648), %d windows, %.3f ms = %.0f GB/s algorithmic (%.2f x the block's %.3f ms x %d), "
         "entries differing from the block result: %lld; %s",
         K, (long long)m, (long long)nnz, b200sp_spmv64_plan_windows(p64), ms64, gbs, ms64 / (msB * K), msB, K, (long long)diff,
         b200sp_spmv64_last_kernel(p64));
  b200sp_spmv64_plan_destroy(p64, nullptr);
  b200sp_spmv_plan_destroy(p32, nullptr);
}

// ------------------------------------------------------------------------------------------------
struct Suite {
  const char* name;
  std::function<void()> fn;
  int timeout_s;
};

int main(int argc, char** argv) {
  std::vector<Suite> all = {{"spgemm", suite_spgemm, 60},       {"crs", suite_crs, 45},       {"spgemm_c4", suite_spgemm_c4, 60},
                            {"crs_big", suite_crs_big, 60},     {"spmv_t", suite_spmv_t, 45}, {"spmm", suite_spmm, 60},
                            {"spmm_sweep", suite_spmm_sweep, 60}, {"jacobi", suite_jacobi, 60}, {"spmv_longrows", suite_spmv_longrows, 60}, {"bsr", suite_bsr, 60}, {"cg", suite_cg, 60}, {"solvers", suite_solvers, 90}, {"spmv64", suite_spmv64, 300}};
  std::vector<std::string> pick;
  for (int i = 1; i < argc; ++i) {
    if (!strcmp(argv[i], "--out") && i + 1 < argc) g_out = argv[++i];
    else if (!strcmp(argv[i], "--suite") && i + 1 < argc) pick.push_back(argv[++i]);
    else if (!strcmp(argv[i], "--big")) g_big = true;
    else if (!strcmp(argv[i], "--dry")) g_dry = true;
    else if (!strcmp(argv[i], "--spmm-scale") && i + 1 < argc) g_spmm_scale = atoi(argv[++i]);
    else if (!strcmp(argv[i], "--timeout-scale") && i + 1 < argc) g_timeout_scale = std::max(1, atoi(argv[++i]));
    else {
      fprintf(stderr, "usage: gpu_check [--out FILE] [--suite NAME]... [--big] [--dry] [--spmm-scale N]\n");
      return 64;
    }
  }
  int failed = 0;
  for (auto& s : all) {
    if (!pick.empty() && std::find(pick.begin(), pick.end(), s.name) == pick.end()) continue;
    g_suite = s.name;
    const double t0 = now_s();
    fflush(nullptr);
    const pid_t pid = fork();  // the parent never touches CUDA
    if (pid == 0) {
      alarm((unsigned)(s.timeout_s * g_timeout_scale));
      int dev_count = 0;
      if (!g_dry && (cudaGetDeviceCount(&dev_count) != cudaSuccess || dev_count == 0 || b200sp_device_ok() != 1)) {
        record("device", false, "no compute-capability 10.x CUDA device");
        _exit(2);
      }
      s.fn();
      fflush(nullptr);
      _exit(g_fail ? 1 : 0);
    }
    int status = 0;
    waitpid(pid, &status, 0);
    const bool ok = WIFEXITED(status) && WEXITSTATUS(status) == 0;
    g_suite = "summary";
    record(s.name, ok, "exit=%d signal=%d %.1f s", WIFEXITED(status) ? WEXITSTATUS(status) : -1, WIFSIGNALED(status) ? WTERMSIG(status) : 0,
           now_s() - t0);
    g_fail = 0;
    if (!ok) ++failed;
  }
  return failed;
}
