// shim_driver.cpp -- instantiates the TPL_B200 specialisations exactly as KokkosSparse::spmv /
// spgemm_symbolic / spgemm_numeric would (Kokkos_Mock.hpp standing in for Kokkos), runs them on the
// GPU through libb200sparse and checks the results on the host.  Exit code 0 = all checks passed.
#define KOKKOSKERNELS_ENABLE_TPL_B200SPARSE
#include "Kokkos_Mock.hpp"
#include "KokkosSparse_spmv_b200_tpl_spec_avail.hpp"
#include "KokkosSparse_spmv_b200_tpl_spec_decl.hpp"
#include "KokkosSparse_spgemm_b200_tpl_spec_avail.hpp"
#include "KokkosSparse_spgemm_b200_tpl_spec_decl.hpp"
#include "KokkosSparse_spadd_b200_tpl_spec_avail.hpp"
#include "KokkosSparse_spadd_b200_tpl_spec_decl.hpp"
#include "KokkosSparse_spgemm_jacobi_b200_tpl_spec_avail.hpp"
#include "KokkosSparse_spgemm_jacobi_b200_tpl_spec_decl.hpp"
#include "KokkosSparse_gauss_seidel_b200_tpl_spec_avail.hpp"
#include "KokkosSparse_gauss_seidel_b200_tpl_spec_decl.hpp"
#include "KokkosSparse_spmv_bsrmatrix_b200_tpl_spec_avail.hpp"
#include "KokkosSparse_gmres_b200_tpl_spec_avail.hpp"
#include "KokkosSparse_gmres_b200_tpl_spec_decl.hpp"
#include "KokkosSparse_spmv_bsrmatrix_b200_tpl_spec_decl.hpp"
#include "KokkosSparse_sptrsv_b200_tpl_spec_avail.hpp"
#include "KokkosSparse_sptrsv_b200_tpl_spec_decl.hpp"

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

using namespace KokkosSparse;
using Dev   = Kokkos::Device<Kokkos::Cuda, Kokkos::CudaSpace>;
using UM    = Kokkos::MemoryTraits<Kokkos::Unmanaged>;
using UMRA  = Kokkos::MemoryTraits<Kokkos::Unmanaged | Kokkos::RandomAccess>;
using Hnd   = Impl::SPMVHandleImpl<Kokkos::Cuda, Kokkos::CudaSpace, double, int, int>;
using AMat  = CrsMatrix<const double, const int, Dev, UM, const int>;
using XVec  = Kokkos::View<const double*, Kokkos::LayoutLeft, Dev, UMRA>;
using YVec  = Kokkos::View<double*, Kokkos::LayoutLeft, Dev, UM>;
using XMV   = Kokkos::View<const double**, Kokkos::LayoutLeft, Dev, UMRA>;
using YMV   = Kokkos::View<double**, Kokkos::LayoutLeft, Dev, UM>;
using KH    = KokkosKernels::Experimental::KokkosKernelsHandle<const int, const int, const double, Kokkos::Cuda, Kokkos::CudaSpace, Kokkos::CudaSpace>;
using CIV   = Kokkos::View<const int*, KokkosKernels::default_layout, Dev, UM>;
using IV    = Kokkos::View<int*, KokkosKernels::default_layout, Dev, UM>;
using CSV   = Kokkos::View<const double*, KokkosKernels::default_layout, Dev, UM>;
using SV    = Kokkos::View<double*, KokkosKernels::default_layout, Dev, UM>;

static_assert(Impl::spmv_tpl_spec_avail<Kokkos::Cuda, Hnd, AMat, XVec, YVec>::value, "rank-1 specialisation must be available");
static_assert(Impl::spmv_mv_tpl_spec_avail<Kokkos::Cuda, Hnd, AMat, XMV, YMV>::value, "rank-2 specialisation must be available");
// 64-bit offsets: (int64_t, size_t) -- the cuSPARSE slot's other instantiation -- and (int, size_t)
using Hnd64  = Impl::SPMVHandleImpl<Kokkos::Cuda, Kokkos::CudaSpace, double, size_t, int64_t>;
using AMat64 = CrsMatrix<const double, const int64_t, Dev, UM, const size_t>;
using Hnd64i = Impl::SPMVHandleImpl<Kokkos::Cuda, Kokkos::CudaSpace, double, size_t, int>;
using AMat64i = CrsMatrix<const double, const int, Dev, UM, const size_t>;
static_assert(Impl::spmv_tpl_spec_avail<Kokkos::Cuda, Hnd64, AMat64, XVec, YVec>::value && Impl::spmv_mv_tpl_spec_avail<Kokkos::Cuda, Hnd64, AMat64, XMV, YMV>::value,
              "(int64_t, size_t) specialisations must be available");
static_assert(Impl::spmv_tpl_spec_avail<Kokkos::Cuda, Hnd64i, AMat64i, XVec, YVec>::value, "(int, size_t) specialisation must be available");
using DINV  = Kokkos::View<const double**, KokkosKernels::default_layout, Dev, UM>;
static_assert(Impl::spgemm_jacobi_tpl_spec_avail<KH, CIV, CIV, CSV, CIV, CIV, CSV, IV, IV, SV, DINV>::value, "spgemm_jacobi must be available");
using XGS   = Kokkos::View<double**, KokkosKernels::default_layout, Dev, UM>;
using YGS   = Kokkos::View<const double**, KokkosKernels::default_layout, Dev, UM>;
static_assert(Impl::gauss_seidel_symbolic_tpl_spec_avail<KH, CIV, CIV>::value && Impl::gauss_seidel_numeric_tpl_spec_avail<KH, CIV, CIV, CSV>::value &&
                  Impl::gauss_seidel_apply_tpl_spec_avail<KH, CIV, CIV, CSV, XGS, YGS>::value,
              "Gauss-Seidel symbolic / numeric / apply must be available");
using BMat  = Experimental::BsrMatrix<const double, const int, Dev, UM, const int>;
static_assert(Impl::spmv_bsrmatrix_tpl_spec_avail<Kokkos::Cuda, Hnd, BMat, XVec, YVec>::value, "BsrMatrix rank-1 must be available");
static_assert(Impl::spmv_mv_bsrmatrix_tpl_spec_avail<Kokkos::Cuda, Hnd, BMat, XMV, YMV>::value, "BsrMatrix rank-2 must be available");
static_assert(Impl::spgemm_symbolic_tpl_spec_avail<KH, CIV, CIV, CIV, CIV, IV>::value, "spgemm symbolic must be available");
static_assert(Impl::spgemm_numeric_tpl_spec_avail<KH, CIV, CIV, CSV, CIV, CIV, CSV, CIV, IV, SV>::value, "spgemm numeric");
static_assert(Impl::spadd_symbolic_tpl_spec_avail<Kokkos::Cuda, KH, CIV, CIV, CIV, CIV, IV>::value, "spadd symbolic must be available");
static_assert(Impl::spadd_numeric_tpl_spec_avail<Kokkos::Cuda, KH, CIV, CIV, CSV, CIV, CIV, CSV, CIV, IV, SV>::value, "spadd numeric");

template <class T>
T* to_dev(const std::vector<T>& h) {
  T* d = nullptr;
  cudaMalloc(&d, sizeof(T) * (h.size() ? h.size() : 1));
  cudaMemcpy(d, h.data(), sizeof(T) * h.size(), cudaMemcpyHostToDevice);
  return d;
}

int main(int argc, char** argv) {
  // --bsr: also run the BsrMatrix specialisations (not part of the default run)
  bool with_bsr = false, with_jacobi = false, with_gs = false, with_gmres = false;  // --jacobi, --gs: likewise for spgemm_jacobi / Gauss-Seidel
  int n_arg = 50000;                                                                 // --n N: rows of the test matrix (the CPU emulation runs a smaller one)
  bool with_sptrsv = false;                                                          // --sptrsv: SPTRSV_SYMBOLIC / SPTRSV_SOLVE
  bool with_spmv64 = false;                                                          // --spmv64: the 64-bit-offset specialisations
  for (int a = 1; a < argc; ++a) {
    with_bsr |= std::string(argv[a]) == "--bsr";
    with_jacobi |= std::string(argv[a]) == "--jacobi";
    with_gs |= std::string(argv[a]) == "--gs";
    with_gmres |= std::string(argv[a]) == "--gmres";
    with_spmv64 |= std::string(argv[a]) == "--spmv64";
    with_sptrsv |= std::string(argv[a]) == "--sptrsv";
    if (std::string(argv[a]) == "--n" && a + 1 < argc) n_arg = std::atoi(argv[a + 1]);
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    std::printf("no CUDA device\n");
    return 77;
  }
  // tridiagonal-ish n x n matrix with rows of 3 (ragged at the ends), values depend on (i,j)
  const int n = n_arg >= 8000 ? n_arg : 8000;
  std::vector<int> rp(n + 1, 0), ci;
  std::vector<double> va, x(n), y0(n);
  for (int i = 0; i < n; ++i) {
    for (int j = i - 1; j <= i + 1; ++j)
      if (j >= 0 && j < n) {
        ci.push_back(j);
        va.push_back(1.0 + 0.001 * ((i * 7 + j * 3) % 11));
      }
    rp[i + 1] = (int)ci.size();
    x[i]  = 0.5 + 0.25 * std::sin(0.01 * i);
    y0[i] = 1.0 + 0.001 * i;
  }
  int *d_rp = to_dev(rp), *d_ci = to_dev(ci);
  double *d_va = to_dev(va), *d_x = to_dev(x), *d_y = to_dev(y0);
  cudaStream_t stream;
  cudaStreamCreate(&stream);
  Kokkos::Cuda exec(stream);
  int failures = 0;
  {
    Hnd handle(SPMV_DEFAULT);
    AMat A(n, n, ci.size(), d_va, d_rp, d_ci);
    Impl::SPMV<Kokkos::Cuda, Hnd, AMat, XVec, YVec>::spmv(exec, &handle, "N", 2.0, A, XVec(d_x, n), 0.5, YVec(d_y, n));
    exec.fence();
    std::vector<double> y(n);
    cudaMemcpy(y.data(), d_y, sizeof(double) * n, cudaMemcpyDeviceToHost);
    for (int i = 0; i < n; ++i) {
      double s = 0;
      for (int k = rp[i]; k < rp[i + 1]; ++k) s += va[k] * x[ci[k]];
      const double e = 0.5 * y0[i] + 2.0 * s;
      if (std::fabs(y[i] - e) > 1e-12 * (1 + std::fabs(e))) ++failures;
    }
    std::printf("spmv rank-1 through SPMV<...,true>::spmv : %d mismatches\n", failures);
    // rank-2, 3 columns, LayoutLeft, transpose mode
    const int k = 3;
    std::vector<double> X(n * k), Y(n * k, 0.0);
    for (int j = 0; j < k; ++j)
      for (int i = 0; i < n; ++i) X[j * n + i] = x[i] * (j + 1);
    double *d_X = to_dev(X), *d_Y = to_dev(Y);
    Impl::SPMV_MV<Kokkos::Cuda, Hnd, AMat, XMV, YMV>::spmv_mv(exec, &handle, "T", 1.0, A, XMV(d_X, n, k), 0.0, YMV(d_Y, n, k));
    exec.fence();
    cudaMemcpy(Y.data(), d_Y, sizeof(double) * n * k, cudaMemcpyDeviceToHost);
    std::vector<double> E(n * k, 0.0);
    for (int i = 0; i < n; ++i)
      for (int q = rp[i]; q < rp[i + 1]; ++q)
        for (int j = 0; j < k; ++j) E[j * n + ci[q]] += va[q] * X[j * n + i];
    int f2 = 0;
    for (int i = 0; i < n * k; ++i)
      if (std::fabs(Y[i] - E[i]) > 1e-12 * (1 + std::fabs(E[i]))) ++f2;
    std::printf("spmv rank-2 'T' through SPMV_MV<...,false,true>::spmv_mv : %d mismatches\n", f2);
    failures += f2;
    cudaFree(d_X);
    cudaFree(d_Y);
  }  // handle destructor frees the plan stream-ordered
  if (with_spmv64) {
    // the same matrix with size_t offsets and int64_t (then int) ordinals, through the 64-bit specialisations
    std::vector<size_t> rp64(rp.begin(), rp.end());
    std::vector<int64_t> ci64(ci.begin(), ci.end());
    size_t* d_rp64  = to_dev(rp64);
    int64_t* d_ci64 = to_dev(ci64);
    int f64m = 0;
    auto check = [&](const char* what) {
      exec.fence();
      std::vector<double> y(n);
      cudaMemcpy(y.data(), d_y, sizeof(double) * n, cudaMemcpyDeviceToHost);
      int bad = 0;
      for (int i = 0; i < n; ++i) {
        double s = 0;
        for (int k = rp[i]; k < rp[i + 1]; ++k) s += va[k] * x[ci[k]];
        const double e = 0.5 * y0[i] + 2.0 * s;
        if (std::fabs(y[i] - e) > 1e-12 * (1 + std::fabs(e))) ++bad;
      }
      std::printf("spmv rank-1 %s : %d mismatches\n", what, bad);
      f64m += bad;
    };
    {
      Hnd64 handle(SPMV_DEFAULT);
      AMat64 A(n, n, ci.size(), d_va, d_rp64, d_ci64);
      cudaMemcpy(d_y, y0.data(), sizeof(double) * n, cudaMemcpyHostToDevice);
      Impl::SPMV<Kokkos::Cuda, Hnd64, AMat64, XVec, YVec>::spmv(exec, &handle, "N", 2.0, A, XVec(d_x, n), 0.5, YVec(d_y, n));
      check("(int64_t, size_t) through SPMV<...,true>::spmv");
      // rank 2, LayoutLeft, 'T', on the same handle's second slot
      const int k = 2;
      std::vector<double> X(n * k), Y(n * k, 0.0), E(n * k, 0.0);
      for (int j = 0; j < k; ++j)
        for (int i = 0; i < n; ++i) X[j * n + i] = x[i] * (j + 2);
      double *d_X = to_dev(X), *d_Y = to_dev(Y);
      Impl::SPMV_MV<Kokkos::Cuda, Hnd64, AMat64, XMV, YMV>::spmv_mv(exec, &handle, "T", 1.0, A, XMV(d_X, n, k), 0.0, YMV(d_Y, n, k));
      exec.fence();
      cudaMemcpy(Y.data(), d_Y, sizeof(double) * n * k, cudaMemcpyDeviceToHost);
      for (int i = 0; i < n; ++i)
        for (int q = rp[i]; q < rp[i + 1]; ++q)
          for (int j = 0; j < k; ++j) E[j * n + ci[q]] += va[q] * X[j * n + i];
      int bad = 0;
      for (int i = 0; i < n * k; ++i)
        if (std::fabs(Y[i] - E[i]) > 1e-12 * (1 + std::fabs(E[i]))) ++bad;
      std::printf("spmv rank-2 'T' (int64_t, size_t) through SPMV_MV<...,false,true>::spmv_mv : %d mismatches\n", bad);
      f64m += bad;
      cudaFree(d_X);
      cudaFree(d_Y);
    }
    {
      Hnd64i handle(SPMV_DEFAULT);
      AMat64i A(n, n, ci.size(), d_va, d_rp64, d_ci);
      cudaMemcpy(d_y, y0.data(), sizeof(double) * n, cudaMemcpyHostToDevice);
      Impl::SPMV<Kokkos::Cuda, Hnd64i, AMat64i, XVec, YVec>::spmv(exec, &handle, "N", 2.0, A, XVec(d_x, n), 0.5, YVec(d_y, n));
      check("(int, size_t) through SPMV<...,true>::spmv");
    }
    failures += f64m;
    cudaFree(d_rp64);
    cudaFree(d_ci64);
  }
  {
    // C = A*A through the SpGEMM specialisations; check against a host Gustavson product
    KH kh;
    kh.create_spgemm_handle();
    int* d_rpC = nullptr;
    cudaMalloc(&d_rpC, sizeof(int) * (n + 1));
    using SYM = Impl::SPGEMM_SYMBOLIC<KH, CIV, CIV, CIV, CIV, IV, true, true>;
    using NUM = Impl::SPGEMM_NUMERIC<KH, CIV, CIV, CSV, CIV, CIV, CSV, CIV, IV, SV, true, true>;
    CIV vrp(d_rp, n + 1), vci(d_ci, ci.size());
    CSV vva(d_va, va.size());
    SYM::spgemm_symbolic(&kh, n, n, n, vrp, vci, false, vrp, vci, false, IV(d_rpC, n + 1), false);
    const size_t cnnz = kh.get_spgemm_handle()->get_c_nnz();
    int* d_ciC = nullptr;
    double* d_vC = nullptr;
    cudaMalloc(&d_ciC, sizeof(int) * cnnz);
    cudaMalloc(&d_vC, sizeof(double) * cnnz);
    NUM::spgemm_numeric(&kh, n, n, n, vrp, vci, vva, false, vrp, vci, vva, false, CIV(d_rpC, n + 1), IV(d_ciC, cnnz), SV(d_vC, cnnz));
    cudaDeviceSynchronize();
    std::vector<int> rpC(n + 1), ciC(cnnz);
    std::vector<double> vC(cnnz);
    cudaMemcpy(rpC.data(), d_rpC, sizeof(int) * (n + 1), cudaMemcpyDeviceToHost);
    cudaMemcpy(ciC.data(), d_ciC, sizeof(int) * cnnz, cudaMemcpyDeviceToHost);
    cudaMemcpy(vC.data(), d_vC, sizeof(double) * cnnz, cudaMemcpyDeviceToHost);
    int f3 = 0;
    std::vector<double> acc(n, 0.0);
    std::vector<char> flag(n, 0);
    for (int i = 0; i < n; ++i) {
      std::vector<int> cols;
      for (int a = rp[i]; a < rp[i + 1]; ++a)
        for (int b = rp[ci[a]]; b < rp[ci[a] + 1]; ++b) {
          if (!flag[ci[b]]) {
            flag[ci[b]] = 1;
            cols.push_back(ci[b]);
          }
          acc[ci[b]] += va[b] * va[a];
        }
      if (rpC[i + 1] - rpC[i] != (int)cols.size()) ++f3;
      for (int q = rpC[i]; q < rpC[i + 1] && q < (int)cnnz; ++q) {
        if (q > rpC[i] && ciC[q] <= ciC[q - 1]) ++f3;  // sorted, no duplicates
        if (!flag[ciC[q]] || std::fabs(vC[q] - acc[ciC[q]]) > 1e-12 * std::fabs(acc[ciC[q]])) ++f3;
      }
      for (int c : cols) {
        flag[c] = 0;
        acc[c]  = 0;
      }
    }
    auto sh = kh.get_spgemm_handle();
    if (!sh->is_symbolic_called() || !sh->is_numeric_called() || !sh->are_rowptrs_computed() || !sh->are_entries_computed()) ++f3;
    std::printf("spgemm through SPGEMM_SYMBOLIC/NUMERIC<...,true,true> : c_nnz=%zu, %d mismatches\n", cnnz, f3);
    failures += f3;
    if (with_jacobi) {
      // C = (I - omega*diag(dinv)*A)*A on the structure just computed, through SPGEMM_JACOBI<...,true,true>
      using JAC = Impl::SPGEMM_JACOBI<KH, CIV, CIV, CSV, CIV, CIV, CSV, IV, IV, SV, DINV, true, true>;
      const double omega = 0.75;
      std::vector<double> dinv(n);
      for (int i = 0; i < n; ++i) dinv[i] = 0.5 + 0.001 * (i % 97);
      double* d_dinv = to_dev(dinv);
      IV vciC(d_ciC, cnnz);
      SV vvC(d_vC, cnnz);
      JAC::spgemm_jacobi(&kh, n, n, n, vrp, vci, vva, false, vrp, vci, vva, false, IV(d_rpC, n + 1), vciC, vvC, omega, DINV(d_dinv, n, 1));
      cudaDeviceSynchronize();
      cudaMemcpy(ciC.data(), d_ciC, sizeof(int) * cnnz, cudaMemcpyDeviceToHost);
      cudaMemcpy(vC.data(), d_vC, sizeof(double) * cnnz, cudaMemcpyDeviceToHost);
      int f7 = 0;
      for (int i = 0; i < n; ++i) {
        std::vector<int> cols;
        for (int a = rp[i]; a < rp[i + 1]; ++a)
          for (int b = rp[ci[a]]; b < rp[ci[a] + 1]; ++b) {
            if (!flag[ci[b]]) {
              flag[ci[b]] = 1;
              cols.push_back(ci[b]);
            }
            acc[ci[b]] += va[b] * va[a];
          }
        for (int c : cols) acc[c] *= -omega * dinv[i];
        for (int b = rp[i]; b < rp[i + 1]; ++b) acc[ci[b]] += va[b];  // + row i of B (= A here)
        for (int q = rpC[i]; q < rpC[i + 1]; ++q) {
          if (q > rpC[i] && ciC[q] <= ciC[q - 1]) ++f7;
          if (!flag[ciC[q]] || std::fabs(vC[q] - acc[ciC[q]]) > 1e-12 * (1 + std::fabs(acc[ciC[q]]))) ++f7;
        }
        for (int c : cols) {
          flag[c] = 0;
          acc[c]  = 0;
        }
      }
      std::printf("spgemm_jacobi through SPGEMM_JACOBI<...,true,true> : %d mismatches\n", f7);
      failures += f7;
      cudaFree(d_dinv);
    }
    kh.destroy_spgemm_handle();
  }
  {
    // C = 2*A - 0.5*A through the spadd specialisations (strict CRS input, the only case that reaches a TPL)
    KH kh;
    kh.create_spadd_handle(true, true);
    int* d_rpC = nullptr;
    cudaMalloc(&d_rpC, sizeof(int) * (n + 1));
    using ASYM = Impl::SPADD_SYMBOLIC<Kokkos::Cuda, KH, CIV, CIV, CIV, CIV, IV, true, true>;
    using ANUM = Impl::SPADD_NUMERIC<Kokkos::Cuda, KH, CIV, CIV, CSV, CIV, CIV, CSV, CIV, IV, SV, true, true>;
    CIV vrp(d_rp, n + 1), vci(d_ci, ci.size());
    CSV vva(d_va, va.size());
    ASYM::spadd_symbolic(exec, &kh, n, n, vrp, vci, vrp, vci, IV(d_rpC, n + 1));
    const size_t cnnz = kh.get_spadd_handle()->get_c_nnz();
    int* d_ciC = nullptr;
    double* d_vC = nullptr;
    cudaMalloc(&d_ciC, sizeof(int) * (cnnz ? cnnz : 1));
    cudaMalloc(&d_vC, sizeof(double) * (cnnz ? cnnz : 1));
    ANUM::spadd_numeric(exec, &kh, n, n, 2.0, vrp, vci, vva, -0.5, vrp, vci, vva, CIV(d_rpC, n + 1), IV(d_ciC, cnnz), SV(d_vC, cnnz));
    exec.fence();
    std::vector<int> rpC(n + 1), ciC(cnnz);
    std::vector<double> vC(cnnz);
    cudaMemcpy(rpC.data(), d_rpC, sizeof(int) * (n + 1), cudaMemcpyDeviceToHost);
    cudaMemcpy(ciC.data(), d_ciC, sizeof(int) * cnnz, cudaMemcpyDeviceToHost);
    cudaMemcpy(vC.data(), d_vC, sizeof(double) * cnnz, cudaMemcpyDeviceToHost);
    int f4 = (cnnz == ci.size()) ? 0 : 1;
    for (int i = 0; i <= n && !f4; ++i)
      if (rpC[i] != rp[i]) ++f4;
    for (size_t q = 0; q < cnnz && !f4; ++q)
      if (ciC[q] != ci[q] || vC[q] != 2.0 * va[q] + -0.5 * va[q]) ++f4;
    auto ah = kh.get_spadd_handle();
    if (!ah->is_symbolic_called() || !ah->is_numeric_called()) ++f4;
    std::printf("spadd through SPADD_SYMBOLIC/NUMERIC<...,true,true> : c_nnz=%zu, %d mismatches\n", cnnz, f4);
    failures += f4;
    kh.destroy_spadd_handle();
    cudaFree(d_rpC);
    cudaFree(d_ciC);
    cudaFree(d_vC);
  }
  if (with_gs) {
    // Gauss-Seidel through GAUSS_SEIDEL_SYMBOLIC / NUMERIC / APPLY<Kokkos::Cuda, ..., true, true>: the tridiagonal-ish matrix made
    // diagonally dominant, two columns of right-hand sides, 12 symmetric sweeps from x = 0 must reach the solution
    std::vector<double> vd(va);
    for (int i = 0; i < n; ++i)
      for (int q = rp[i]; q < rp[i + 1]; ++q)
        if (ci[q] == i) vd[q] = 4.0;
    double* d_vd = to_dev(vd);
    const int k = 2;
    std::vector<double> xs(n * k), yy(n * k, 0.0), x0(n * k, 7.0);
    for (int j = 0; j < k; ++j)
      for (int i = 0; i < n; ++i) xs[j * n + i] = std::sin(0.01 * i + j);
    for (int j = 0; j < k; ++j)
      for (int i = 0; i < n; ++i)
        for (int q = rp[i]; q < rp[i + 1]; ++q) yy[j * n + i] += vd[q] * xs[j * n + ci[q]];
    double *d_xg = to_dev(x0), *d_yg = to_dev(yy);
    KH kh;
    kh.create_gs_handle();
    CIV vrp(d_rp, n + 1), vci(d_ci, ci.size());
    CSV vvd(d_vd, vd.size());
    using GSS = Impl::GAUSS_SEIDEL_SYMBOLIC<Kokkos::Cuda, KH, CIV, CIV, true, true>;
    using GSN = Impl::GAUSS_SEIDEL_NUMERIC<Kokkos::Cuda, KH, SparseMatrixFormat::CRS, CIV, CIV, CSV, true, true>;
    using GSA = Impl::GAUSS_SEIDEL_APPLY<Kokkos::Cuda, KH, SparseMatrixFormat::CRS, CIV, CIV, CSV, XGS, YGS, true, true>;
    GSS::gauss_seidel_symbolic(exec, &kh, n, n, vrp, vci, true);
    GSN::gauss_seidel_numeric(exec, &kh, n, n, vrp, vci, vvd, true);
    GSA::gauss_seidel_apply(exec, &kh, n, n, vrp, vci, vvd, XGS(d_xg, n, k), YGS(d_yg, n, k), true, true, 1.0, 12, true, true);
    exec.fence();
    std::vector<double> xg(n * k);
    cudaMemcpy(xg.data(), d_xg, sizeof(double) * n * k, cudaMemcpyDeviceToHost);
    int f8 = 0;
    for (int i = 0; i < n * k; ++i)
      if (std::fabs(xg[i] - xs[i]) > 1e-6) ++f8;
    if (!kh.get_point_gs_handle()->is_symbolic_called() || !kh.get_point_gs_handle()->is_numeric_called()) ++f8;
    std::printf("Gauss-Seidel through GAUSS_SEIDEL_SYMBOLIC/NUMERIC/APPLY<...,true,true> : %d mismatches\n", f8);
    failures += f8;
    kh.destroy_gs_handle();
    // the same structs with a GS_TWOSTAGE handle: compact recurrence, 20 symmetric sweeps.  (The compact form iterates on x itself,
    // so a truncated inner solve biases its fixed point: 14 inner Jacobi-Richardson sweeps, |D^-1 L| = 1/4, leave 4^-14.)
    kh.create_gs_handle(GS_TWOSTAGE);
    kh.set_gs_twostage(true, n);
    kh.set_gs_set_num_inner_sweeps(14);
    kh.set_gs_twostage_compact_form(true);
    cudaMemcpy(d_xg, x0.data(), sizeof(double) * n * k, cudaMemcpyHostToDevice);
    GSS::gauss_seidel_symbolic(exec, &kh, n, n, vrp, vci, true);
    GSN::gauss_seidel_numeric(exec, &kh, n, n, vrp, vci, vvd, true);
    GSA::gauss_seidel_apply(exec, &kh, n, n, vrp, vci, vvd, XGS(d_xg, n, k), YGS(d_yg, n, k), true, true, 1.0, 20, true, true);
    exec.fence();
    cudaMemcpy(xg.data(), d_xg, sizeof(double) * n * k, cudaMemcpyDeviceToHost);
    int f9 = 0;
    for (int i = 0; i < n * k; ++i)
      if (std::fabs(xg[i] - xs[i]) > 1e-6) ++f9;
    if (!kh.get_twostage_gs_handle()->is_symbolic_called() || !kh.get_twostage_gs_handle()->is_numeric_called()) ++f9;
    if (Impl::mock_native_gs_calls() != 0) ++f9;  // nothing went to the native path so far
    // the classic form (set_gs_twostage(false): triangular solves instead of inner sweeps) through the same structs
    kh.set_gs_twostage(false, n);
    kh.set_gs_twostage_compact_form(false);
    cudaMemcpy(d_xg, x0.data(), sizeof(double) * n * k, cudaMemcpyHostToDevice);
    GSS::gauss_seidel_symbolic(exec, &kh, n, n, vrp, vci, true);
    GSN::gauss_seidel_numeric(exec, &kh, n, n, vrp, vci, vvd, true);
    // (exact triangular solves: a symmetric sweep contracts the error by ~(1/2)^4 on this matrix, 8 sweeps leave < 1e-8;
    //  every row is its own level here, so a sweep is 2 x n dependent steps)
    GSA::gauss_seidel_apply(exec, &kh, n, n, vrp, vci, vvd, XGS(d_xg, n, k), YGS(d_yg, n, k), true, true, 1.0, 8, true, true);
    exec.fence();
    cudaMemcpy(xg.data(), d_xg, sizeof(double) * n * k, cudaMemcpyDeviceToHost);
    for (int i = 0; i < n * k; ++i)
      if (std::fabs(xg[i] - xs[i]) > 1e-6) ++f9;
    if (Impl::mock_native_gs_calls() != 0) ++f9;
    // what the TPL does not serve is forwarded to the native specialisation: cluster Gauss-Seidel
    kh.create_gs_handle(GS_CLUSTER);
    GSS::gauss_seidel_symbolic(exec, &kh, n, n, vrp, vci, true);
    GSN::gauss_seidel_numeric(exec, &kh, n, n, vrp, vci, vvd, true);
    GSA::gauss_seidel_apply(exec, &kh, n, n, vrp, vci, vvd, XGS(d_xg, n, k), YGS(d_yg, n, k), true, true, 1.0, 1, true, true);
    if (Impl::mock_native_gs_calls() != 3) ++f9;
    std::printf("two-stage Gauss-Seidel through the same structs (GS_TWOSTAGE handle: inner sweeps and the sptrsv form), cluster forwarded : %d mismatches\n", f9);
    failures += f9;
    kh.destroy_gs_handle();
    cudaFree(d_vd);
    cudaFree(d_xg);
    cudaFree(d_yg);
  }
  if (with_gmres) {
    // gmres through GMRES<KH, ..., true, true>::gmres (CrsMatrix, no preconditioner -> the library; with one -> the native GmresWrap)
    using UMRAV = Kokkos::MemoryTraits<Kokkos::Unmanaged | Kokkos::RandomAccess>;
    using GB    = Kokkos::View<const double*, KokkosKernels::default_layout, Dev, UMRAV>;
    using GX    = Kokkos::View<double*, KokkosKernels::default_layout, Dev, UMRAV>;
    using GM    = Impl::GMRES<KH, const double, const int, Dev, UM, const int, GB, GX, true, true>;
    static_assert(Impl::gmres_tpl_spec_avail<KH, const double, const int, Dev, UM, const int, GB, GX>::value, "gmres must be available");
    std::vector<double> vd(va);
    for (int i = 0; i < n; ++i)
      for (int q = rp[i]; q < rp[i + 1]; ++q)
        if (ci[q] == i) vd[q] = 3.0;
    double* d_vd = to_dev(vd);
    std::vector<double> ones(n, 1.0), zeros(n, 0.0);
    double *d_b = to_dev(ones), *d_xx = to_dev(zeros);
    KH kh;
    kh.create_gmres_handle(15, 1e-8);
    AMat A(n, n, ci.size(), d_vd, d_rp, d_ci);
    GB Bv(d_b, n);
    GX Xv(d_xx, n);
    GM::gmres(&kh, A, Bv, Xv);
    cudaDeviceSynchronize();
    std::vector<double> xg(n);
    cudaMemcpy(xg.data(), d_xx, sizeof(double) * n, cudaMemcpyDeviceToHost);
    double rr = 0, bb = 0;
    for (int i = 0; i < n; ++i) {
      double s = 0;
      for (int q = rp[i]; q < rp[i + 1]; ++q) s += vd[q] * xg[ci[q]];
      rr += (1.0 - s) * (1.0 - s);
      bb += 1.0;
    }
    auto gh = kh.get_gmres_handle();
    int f9  = (std::sqrt(rr / bb) < 1e-8 && gh->conv_flag_val == GMRESHandleMock::Conv && gh->num_iters > 0) ? 0 : 1;
    Experimental::Preconditioner<AMat> prec;
    using Wrap = Impl::Experimental::GmresWrap<GMRESHandleMock>;
    const int before = Wrap::calls();
    GM::gmres(&kh, A, Bv, Xv, &prec);
    if (Wrap::calls() != before + 1) ++f9;  // a preconditioner routes to the native implementation
    std::printf("gmres through GMRES<...,true,true>::gmres : rel. residual %.2e after %d iterations, %d mismatches\n", std::sqrt(rr / bb),
                gh->num_iters, f9);
    failures += f9;
    kh.destroy_gmres_handle();
    cudaFree(d_vd);
    cudaFree(d_b);
    cudaFree(d_xx);
  }
  if (with_sptrsv) {
    // sptrsv through SPTRSV_SYMBOLIC / SPTRSV_SOLVE<...,true,true>: the lower and the upper triangle (diagonal 3) of the matrix above,
    // against the serial substitution loop (bit for bit: the library computes every row in storage order with unfused operations)
    using UMRAV = Kokkos::MemoryTraits<Kokkos::Unmanaged | Kokkos::RandomAccess>;
    using TRI   = Kokkos::View<const int*, KokkosKernels::default_layout, Dev, UMRAV>;
    using TRS   = Kokkos::View<const double*, KokkosKernels::default_layout, Dev, UMRAV>;
    using TRX   = Kokkos::View<double*, KokkosKernels::default_layout, Dev, UM>;
    using TSY   = Impl::SPTRSV_SYMBOLIC<Kokkos::Cuda, KH, TRI, TRI, true, true>;
    using TSO   = Impl::SPTRSV_SOLVE<Kokkos::Cuda, KH, TRI, TRI, TRS, TRS, TRX, true, true>;
    static_assert(Impl::sptrsv_symbolic_tpl_spec_avail<KH, TRI, TRI>::value, "sptrsv_symbolic must be available");
    static_assert(Impl::sptrsv_solve_tpl_spec_avail<Kokkos::Cuda, KH, TRI, TRI, TRS, TRS, TRX>::value, "sptrsv_solve must be available");
    int f10 = 0;
    const int nt = 6000;  // the leading nt x nt block: a tridiagonal matrix has as many levels as rows, and symbolic sweeps once per level
    for (int lower = 1; lower >= 0; --lower) {
      std::vector<int> trp(nt + 1, 0), tci;
      std::vector<double> tva, bh(nt), xr(nt), xg(nt);
      for (int i = 0; i < nt; ++i) {
        for (int q = rp[i]; q < rp[i + 1]; ++q)
          if (ci[q] < nt && (lower ? ci[q] <= i : ci[q] >= i)) {
            tci.push_back(ci[q]);
            tva.push_back(ci[q] == i ? 3.0 : va[q]);
          }
        trp[i + 1] = (int)tci.size();
        bh[i]      = 1.0 + 0.5 * std::cos(0.02 * i);
      }
      for (int t = 0; t < nt; ++t) {
        const int i = lower ? t : nt - 1 - t;
        volatile double acc = bh[i];  // volatile: no contraction of the multiply and the subtract
        double d            = 1.0;
        for (int q = trp[i]; q < trp[i + 1]; ++q) {
          if (tci[q] == i) d = tva[q];
          else {
            volatile double prod = tva[q] * xr[tci[q]];
            acc                  = acc - prod;
          }
        }
        xr[i] = acc / d;
      }
      int *d_trp = to_dev(trp), *d_tci = to_dev(tci);
      double *d_tva = to_dev(tva), *d_b = to_dev(bh), *d_xx = to_dev(xg);
      KH kh;
      kh.create_sptrsv_handle(Experimental::SPTRSVAlgorithm::SEQLVLSCHD_TP1, nt, lower != 0);
      TRI vrp(d_trp, nt + 1), vci(d_tci, tci.size());
      bool threw = false;
      try {
        TSO::sptrsv_solve(exec, &kh, vrp, vci, TRS(d_tva, tva.size()), TRS(d_b, nt), TRX(d_xx, nt));
      } catch (const std::runtime_error&) { threw = true; }
      if (!threw) ++f10;  // solve before symbolic is an error, as in the front end (sparse/src/KokkosSparse_sptrsv.hpp:300-310)
      TSY::sptrsv_symbolic(exec, &kh, vrp, vci);
      if (!kh.get_sptrsv_handle()->is_symbolic_complete()) ++f10;
      TSO::sptrsv_solve(exec, &kh, vrp, vci, TRS(d_tva, tva.size()), TRS(d_b, nt), TRX(d_xx, nt));
      exec.fence();
      cudaMemcpy(xg.data(), d_xx, sizeof(double) * nt, cudaMemcpyDeviceToHost);
      for (int i = 0; i < nt; ++i)
        if (std::memcmp(&xg[i], &xr[i], sizeof(double)) != 0) ++f10;
      kh.destroy_sptrsv_handle();
      cudaFree(d_trp);
      cudaFree(d_tci);
      cudaFree(d_tva);
      cudaFree(d_b);
      cudaFree(d_xx);
    }
    std::printf("sptrsv through SPTRSV_SYMBOLIC / SPTRSV_SOLVE<...,true,true> (lower and upper) : %d mismatches\n", f10);
    failures += f10;
  }
  if (with_bsr) {
    // BsrMatrix: block-tridiagonal, 3 x 3 blocks, through SPMV_BSRMATRIX<...,true,true> (N) and
    // SPMV_MV_BSRMATRIX<...,false,true,true> ('T', 2 columns)
    const int mb = 20000, bs = 3;
    std::vector<int> brp(mb + 1, 0), bci;
    std::vector<double> bva;
    for (int i = 0; i < mb; ++i) {
      for (int j = i - 1; j <= i + 1; ++j)
        if (j >= 0 && j < mb) {
          bci.push_back(j);
          for (int q = 0; q < bs * bs; ++q) bva.push_back(0.5 + 0.01 * ((i * 5 + j * 3 + q) % 13));
        }
      brp[i + 1] = (int)bci.size();
    }
    const int np = mb * bs;
    std::vector<double> bx(np), by0(np);
    for (int i = 0; i < np; ++i) {
      bx[i]  = 0.5 + 0.25 * std::cos(0.01 * i);
      by0[i] = 1.0 + 0.001 * (i % 977);
    }
    int *d_brp = to_dev(brp), *d_bci = to_dev(bci);
    double *d_bva = to_dev(bva), *d_bx = to_dev(bx), *d_by = to_dev(by0);
    Hnd handle(SPMV_DEFAULT);
    BMat A(mb, mb, bci.size(), d_bva, d_brp, d_bci, bs);
    Impl::SPMV_BSRMATRIX<Kokkos::Cuda, Hnd, BMat, XVec, YVec>::spmv_bsrmatrix(exec, &handle, "N", 2.0, A, XVec(d_bx, np), 0.5,
                                                                              YVec(d_by, np));
    exec.fence();
    std::vector<double> y(np);
    cudaMemcpy(y.data(), d_by, sizeof(double) * np, cudaMemcpyDeviceToHost);
    int f5 = 0;
    for (int i = 0; i < mb; ++i)
      for (int lr = 0; lr < bs; ++lr) {
        double s = 0;
        for (int q = brp[i]; q < brp[i + 1]; ++q)
          for (int c = 0; c < bs; ++c) s += bva[(size_t)q * bs * bs + lr * bs + c] * bx[bci[q] * bs + c];
        const double e = 0.5 * by0[i * bs + lr] + 2.0 * s;
        if (std::fabs(y[i * bs + lr] - e) > 1e-12 * (1 + std::fabs(e))) ++f5;
      }
    std::printf("BsrMatrix spmv through SPMV_BSRMATRIX<...,true,true>::spmv_bsrmatrix : %d mismatches\n", f5);
    const int k = 2;
    std::vector<double> X(np * k), Y(np * k, 0.0), E(np * k, 0.0);
    for (int j = 0; j < k; ++j)
      for (int i = 0; i < np; ++i) X[j * np + i] = bx[i] * (j + 1);
    double *d_X = to_dev(X), *d_Y = to_dev(Y);
    Impl::SPMV_MV_BSRMATRIX<Kokkos::Cuda, Hnd, BMat, XMV, YMV>::spmv_mv_bsrmatrix(exec, &handle, "T", 1.0, A, XMV(d_X, np, k), 0.0,
                                                                                  YMV(d_Y, np, k));
    exec.fence();
    cudaMemcpy(Y.data(), d_Y, sizeof(double) * np * k, cudaMemcpyDeviceToHost);
    for (int i = 0; i < mb; ++i)
      for (int q = brp[i]; q < brp[i + 1]; ++q)
        for (int lr = 0; lr < bs; ++lr)
          for (int c = 0; c < bs; ++c)
            for (int j = 0; j < k; ++j) E[j * np + bci[q] * bs + c] += bva[(size_t)q * bs * bs + lr * bs + c] * X[j * np + i * bs + lr];
    int f6 = 0;
    for (int i = 0; i < np * k; ++i)
      if (std::fabs(Y[i] - E[i]) > 1e-12 * (1 + std::fabs(E[i]))) ++f6;
    std::printf("BsrMatrix spmv 'T' rank-2 through SPMV_MV_BSRMATRIX<...,false,true,true>::spmv_mv_bsrmatrix : %d mismatches\n", f6);
    failures += f5 + f6;
    cudaFree(d_X);
    cudaFree(d_Y);
    cudaFree(d_brp);
    cudaFree(d_bci);
    cudaFree(d_bva);
    cudaFree(d_bx);
    cudaFree(d_by);
  }
  std::printf(failures ? "SHIM DRIVER FAILED\n" : "SHIM DRIVER OK\n");
  return failures ? 1 : 0;
}
