// shim_bspgemm_driver.cpp -- the block SpGEMM path of the TPL_B200 shim, instantiated the way Kokkos'
// block_spgemm_symbolic / block_spgemm_numeric reach it (sparse/src/KokkosSparse_spgemm.hpp:77-103,145-156): the point
// SPGEMM_SYMBOLIC slot on the block graphs, then BSPGEMM_NUMERIC named with its defaulted tpl_spec_avail argument, so an
// unavailable combination would land in the native stand-in (which only counts its calls).  On a GPU it multiplies a
// block-tridiagonal BsrMatrix (bs = 3, fp64 and fp32) by itself, compares the result bit for bit with direct C ABI calls and
// checks the "must first call spgemm_symbolic" throw.  Without a device it exits 77 after its static_asserts were compiled
// in.  Exit code 0 = all checks passed.
#define KOKKOSKERNELS_ENABLE_TPL_B200SPARSE
#include "Kokkos_Mock.hpp"
#include "Kokkos_Mock_Bspgemm.hpp"
#include "KokkosSparse_spgemm_b200_tpl_spec_avail.hpp"
#include "KokkosSparse_spgemm_b200_tpl_spec_decl.hpp"
#include "KokkosSparse_bspgemm_b200_tpl_spec_avail.hpp"
#include "KokkosSparse_bspgemm_b200_tpl_spec_decl.hpp"

#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

using namespace KokkosSparse;
using Dev = Kokkos::Device<Kokkos::Cuda, Kokkos::CudaSpace>;
using UM  = Kokkos::MemoryTraits<Kokkos::Unmanaged>;
template <class S>
using KH = KokkosKernels::Experimental::KokkosKernelsHandle<const int, const int, const S, Kokkos::Cuda, Kokkos::CudaSpace, Kokkos::CudaSpace>;
using CIV = Kokkos::View<const int*, KokkosKernels::default_layout, Dev, UM>;
using IV  = Kokkos::View<int*, KokkosKernels::default_layout, Dev, UM>;
template <class S>
using CSV = Kokkos::View<const S*, KokkosKernels::default_layout, Dev, UM>;
template <class S>
using SV = Kokkos::View<S*, KokkosKernels::default_layout, Dev, UM>;

static_assert(Impl::bspgemm_numeric_tpl_spec_avail<KH<double>, CIV, CIV, CSV<double>, CIV, CIV, CSV<double>, CIV, IV, SV<double>>::value,
              "block spgemm numeric (double) must be available");
static_assert(Impl::bspgemm_numeric_tpl_spec_avail<KH<float>, CIV, CIV, CSV<float>, CIV, CIV, CSV<float>, CIV, IV, SV<float>>::value,
              "block spgemm numeric (float) must be available");

template <class T>
static T* to_dev(const std::vector<T>& h) {
  T* d = nullptr;
  cudaMalloc(&d, sizeof(T) * (h.size() ? h.size() : 1));
  cudaMemcpy(d, h.data(), sizeof(T) * h.size(), cudaMemcpyHostToDevice);
  return d;
}
template <class T>
static std::vector<T> to_host(const T* d, size_t n) {
  std::vector<T> h(n);
  cudaMemcpy(h.data(), d, sizeof(T) * n, cudaMemcpyDeviceToHost);
  return h;
}

template <class S>
static int run(const char* name) {
  using SYM = Impl::SPGEMM_SYMBOLIC<KH<S>, CIV, CIV, CIV, CIV, IV, true, true>;
  using NUM = Impl::BSPGEMM_NUMERIC<KH<S>, CIV, CIV, CSV<S>, CIV, CIV, CSV<S>, CIV, IV, SV<S>>;  // tpl argument defaulted
  const int mb = 3000, bs = 3, bb = bs * bs;
  std::vector<int> rp(mb + 1, 0), ci;
  std::vector<S> va;
  for (int i = 0; i < mb; ++i) {
    for (int j = i + 1; j >= i - 1; --j)  // unsorted rows
      if (j >= 0 && j < mb) {
        ci.push_back(j);
        for (int e = 0; e < bb; ++e) va.push_back(S(0.25) + S(0.001) * S((i * 7 + j * 3 + e * 5) % 13) - S(e % 2 ? 0.5 : 0.0));
      }
    rp[i + 1] = (int)ci.size();
  }
  int *d_rp = to_dev(rp), *d_ci = to_dev(ci);
  S* d_va = to_dev(va);
  CIV vrp(d_rp, mb + 1), vci(d_ci, ci.size());
  CSV<S> vva(d_va, va.size());
  int failures = 0;

  // numeric before symbolic: the native struct's check (bspgemm_numeric_spec.hpp:143-147)
  {
    KH<S> kh;
    kh.create_spgemm_handle();
    bool threw = false;
    try {
      IV e0(nullptr, 0);
      SV<S> v0(nullptr, 0);
      NUM::bspgemm_numeric(&kh, mb, mb, mb, bs, vrp, vci, vva, false, vrp, vci, vva, false, vrp, e0, v0);
    } catch (const std::runtime_error& e) {
      threw = std::string(e.what()).find("must first call spgemm_symbolic with the same handle") != std::string::npos;
    }
    if (!threw) ++failures;
    std::printf("%s numeric before symbolic throws: %s\n", name, threw ? "ok" : "FAILED");
    kh.destroy_spgemm_handle();
  }

  KH<S> kh;
  kh.create_spgemm_handle();
  int* d_rpC = nullptr;
  cudaMalloc(&d_rpC, sizeof(int) * (mb + 1));
  SYM::spgemm_symbolic(&kh, mb, mb, mb, vrp, vci, false, vrp, vci, false, IV(d_rpC, mb + 1), false);
  const size_t cnnz = kh.get_spgemm_handle()->get_c_nnz();
  int* d_ciC = nullptr;
  S* d_vC    = nullptr;
  cudaMalloc(&d_ciC, sizeof(int) * cnnz);
  cudaMalloc(&d_vC, sizeof(S) * cnnz * bb);
  IV eC(d_ciC, cnnz);
  SV<S> vC(d_vC, cnnz * bb);
  NUM::bspgemm_numeric(&kh, mb, mb, mb, bs, vrp, vci, vva, false, vrp, vci, vva, false, CIV(d_rpC, mb + 1), eC, vC);
  cudaDeviceSynchronize();
  auto sh = kh.get_spgemm_handle();
  if (!sh->is_numeric_called() || !sh->are_entries_computed()) ++failures;

  // the same product through the C ABI on a fresh plan
  b200sp_spgemm_plan* plan = nullptr;
  b200sp_spgemm_plan_create(&plan);
  int* d_rpC2 = nullptr;
  int* d_ciC2 = nullptr;
  S* d_vC2    = nullptr;
  cudaMalloc(&d_rpC2, sizeof(int) * (mb + 1));
  int64_t cnnz2 = 0;
  int cmax      = 0;
  b200sp_spgemm_symbolic_i32(plan, nullptr, mb, mb, mb, d_rp, d_ci, d_rp, d_ci, d_rpC2, &cnnz2, &cmax);
  cudaMalloc(&d_ciC2, sizeof(int) * cnnz2);
  cudaMalloc(&d_vC2, sizeof(S) * cnnz2 * bb);
  Impl::b200_call_bspgemm_numeric(plan, nullptr, mb, mb, mb, bs, d_rp, d_ci, d_va, d_rp, d_ci, d_va, d_rpC2, d_ciC2, d_vC2);
  cudaDeviceSynchronize();
  b200sp_spgemm_plan_destroy(plan, nullptr);
  const bool same = (size_t)cnnz2 == cnnz && to_host(d_rpC, mb + 1) == to_host(d_rpC2, mb + 1) && to_host(d_ciC, cnnz) == to_host(d_ciC2, cnnz) &&
                    [&] {
                      auto a = to_host(d_vC, cnnz * bb), b = to_host(d_vC2, cnnz * bb);
                      return std::memcmp(a.data(), b.data(), sizeof(S) * a.size()) == 0;
                    }();
  if (!same) ++failures;
  std::printf("%s block spgemm through SPGEMM_SYMBOLIC + BSPGEMM_NUMERIC<...,true,true> : c_nnz=%zu, C ABI bits %s\n", name, cnnz,
              same ? "identical" : "DIFFER");
  kh.destroy_spgemm_handle();
  cudaFree(d_rp);
  cudaFree(d_ci);
  cudaFree(d_va);
  cudaFree(d_rpC);
  cudaFree(d_ciC);
  cudaFree(d_vC);
  cudaFree(d_rpC2);
  cudaFree(d_ciC2);
  cudaFree(d_vC2);
  return failures;
}

int main() {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    std::printf("no CUDA device\n");
    return 77;
  }
  int failures = run<double>("f64") + run<float>("f32");
  std::printf("native BSPGEMM_NUMERIC calls: %d\n", Impl::native_bspgemm_calls());
  failures += Impl::native_bspgemm_calls();
  if (failures == 0) std::printf("SHIM BSPGEMM DRIVER OK\n");
  return failures == 0 ? 0 : 1;
}
