// shim_spgemm64_driver.cpp -- the (int, size_t) SPGEMM_SYMBOLIC / SPGEMM_NUMERIC specialisations of the TPL_B200 shim
// (64-bit offsets, 32-bit ordinals: Kokkos' default offsets in a Trilinos build), instantiated the way
// KokkosSparse::spgemm_symbolic / spgemm_numeric pick them: the dispatch below names the slot with the value of
// spgemm_{symbolic,numeric}_tpl_spec_avail, so an unavailable combination would land in the native stand-ins (which only
// count their calls).  On a GPU it multiplies a random matrix with size_t row maps by itself (fp64 and fp32), runs numeric
// twice on the handle's plan, and compares row map, entries and values bit for bit with direct b200sp_spgemm_*_i64 calls on
// a plan of its own.  Without a device it exits 77 after its static_asserts were compiled in.  Exit code 0 = all checks
// passed.
#define KOKKOSKERNELS_ENABLE_TPL_B200SPARSE
#include "Kokkos_Mock.hpp"
#include "KokkosSparse_spgemm_b200_tpl_spec_avail.hpp"
#include "KokkosSparse_spgemm_b200_tpl_spec_decl.hpp"

#include <cstdio>
#include <cstring>
#include <vector>

using namespace KokkosSparse;
using UM = Kokkos::MemoryTraits<Kokkos::Unmanaged>;
template <class S, class Mem = Kokkos::CudaSpace>
using KH = KokkosKernels::Experimental::KokkosKernelsHandle<const size_t, const int, const S, Kokkos::Cuda, Mem, Mem>;
template <class T, class Mem = Kokkos::CudaSpace>
using V = Kokkos::View<T*, KokkosKernels::default_layout, Kokkos::Device<Kokkos::Cuda, Mem>, UM>;

template <class S, class Mem = Kokkos::CudaSpace>
constexpr bool sym_avail = Impl::spgemm_symbolic_tpl_spec_avail<KH<S, Mem>, V<const size_t, Mem>, V<const int, Mem>,
                                                                V<const size_t, Mem>, V<const int, Mem>, V<size_t, Mem>>::value;
template <class S, class Mem = Kokkos::CudaSpace>
constexpr bool num_avail =
    Impl::spgemm_numeric_tpl_spec_avail<KH<S, Mem>, V<const size_t, Mem>, V<const int, Mem>, V<const S, Mem>, V<const size_t, Mem>,
                                        V<const int, Mem>, V<const S, Mem>, V<const size_t, Mem>, V<int, Mem>, V<S, Mem>>::value;
static_assert(sym_avail<double> && num_avail<double>, "(int, size_t) spgemm (double, CudaSpace) must be available");
static_assert(sym_avail<float> && num_avail<float>, "(int, size_t) spgemm (float, CudaSpace) must be available");
static_assert(sym_avail<double, Kokkos::CudaUVMSpace> && num_avail<double, Kokkos::CudaUVMSpace>, "(int, size_t) double UVM");
static_assert(sym_avail<float, Kokkos::CudaUVMSpace> && num_avail<float, Kokkos::CudaUVMSpace>, "(int, size_t) float UVM");
// 64-bit ordinals stay with the native path
static_assert(!Impl::spgemm_symbolic_tpl_spec_avail<
                  KokkosKernels::Experimental::KokkosKernelsHandle<const size_t, const int64_t, const double, Kokkos::Cuda,
                                                                   Kokkos::CudaSpace, Kokkos::CudaSpace>,
                  V<const size_t>, V<const int64_t>, V<const size_t>, V<const int64_t>, V<size_t>>::value,
              "(int64_t, size_t) is not provided");

namespace KokkosSparse {
namespace Impl {
// the native SPGEMM_SYMBOLIC / SPGEMM_NUMERIC (sparse/impl/KokkosSparse_spgemm_{symbolic,numeric}_spec.hpp, tpl = false):
// stand-ins that count their calls
inline int& native_spgemm_calls() {
  static int n = 0;
  return n;
}
template <class KHT, class a_r, class a_e, class b_r, class b_e, class c_r, bool eti>
struct SPGEMM_SYMBOLIC<KHT, a_r, a_e, b_r, b_e, c_r, false, eti> {
  template <class... Args>
  static void spgemm_symbolic(Args&&...) {
    ++native_spgemm_calls();
  }
};
template <class KHT, class a_r, class a_e, class a_v, class b_r, class b_e, class b_v, class c_r, class c_e, class c_v, bool eti>
struct SPGEMM_NUMERIC<KHT, a_r, a_e, a_v, b_r, b_e, b_v, c_r, c_e, c_v, false, eti> {
  template <class... Args>
  static void spgemm_numeric(Args&&...) {
    ++native_spgemm_calls();
  }
};
}  // namespace Impl
}  // namespace KokkosSparse

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
  using SYM = Impl::SPGEMM_SYMBOLIC<KH<S>, V<const size_t>, V<const int>, V<const size_t>, V<const int>, V<size_t>, sym_avail<S>, true>;
  using NUM = Impl::SPGEMM_NUMERIC<KH<S>, V<const size_t>, V<const int>, V<const S>, V<const size_t>, V<const int>, V<const S>,
                                   V<const size_t>, V<int>, V<S>, num_avail<S>, true>;
  const int n = 4000;
  std::vector<size_t> rp(n + 1, 0);
  std::vector<int> ci;
  std::vector<S> va;
  unsigned s = 2024u;
  auto rnd = [&s]() { return (s = s * 1664525u + 1013904223u) >> 8; };
  for (int i = 0; i < n; ++i) {
    const int len = (i % 251 == 0) ? 200 : (int)(rnd() % 14);  // a few rows past the shared-memory bins' reach of C
    for (int e = 0; e < len; ++e) {
      ci.push_back((int)(rnd() % n));
      va.push_back(S(((int)(rnd() % 2001) - 1000) / 256.0));
    }
    rp[i + 1] = ci.size();
  }
  size_t* d_rp = to_dev(rp);
  int* d_ci    = to_dev(ci);
  S* d_va      = to_dev(va);
  V<const size_t> vrp(d_rp, n + 1);
  V<const int> vci(d_ci, ci.size());
  V<const S> vva(d_va, va.size());
  int failures = 0;

  KH<S> kh;
  kh.create_spgemm_handle();
  size_t* d_rpC = nullptr;
  cudaMalloc(&d_rpC, sizeof(size_t) * (n + 1));
  SYM::spgemm_symbolic(&kh, n, n, n, vrp, vci, false, vrp, vci, false, V<size_t>(d_rpC, n + 1), false);
  const size_t cnnz = kh.get_spgemm_handle()->get_c_nnz();
  int* d_ciC = nullptr;
  S* d_vC    = nullptr;
  cudaMalloc(&d_ciC, sizeof(int) * (cnnz ? cnnz : 1));
  cudaMalloc(&d_vC, sizeof(S) * (cnnz ? cnnz : 1));
  for (int rep = 0; rep < 2; ++rep)  // numeric again on the same structure
    NUM::spgemm_numeric(&kh, n, n, n, vrp, vci, vva, false, vrp, vci, vva, false, V<const size_t>(d_rpC, n + 1), V<int>(d_ciC, cnnz),
                        V<S>(d_vC, cnnz));
  cudaDeviceSynchronize();
  auto sh = kh.get_spgemm_handle();
  if (!sh->is_symbolic_called() || !sh->are_rowptrs_computed() || !sh->is_numeric_called() || !sh->are_entries_computed())
    ++failures;

  // the same product through the C ABI on a fresh plan
  b200sp_spgemm_plan* plan = nullptr;
  b200sp_spgemm_plan_create(&plan);
  int64_t* d_rpC2 = nullptr;
  cudaMalloc(&d_rpC2, sizeof(int64_t) * (n + 1));
  int64_t cnnz2 = 0;
  int cmax      = 0;
  int rc = b200sp_spgemm_symbolic_i64(plan, nullptr, n, n, n, (const int64_t*)d_rp, d_ci, (const int64_t*)d_rp, d_ci, d_rpC2, &cnnz2, &cmax);
  int* d_ciC2 = nullptr;
  S* d_vC2    = nullptr;
  cudaMalloc(&d_ciC2, sizeof(int) * (cnnz2 ? cnnz2 : 1));
  cudaMalloc(&d_vC2, sizeof(S) * (cnnz2 ? cnnz2 : 1));
  rc |= Impl::b200_call_numeric(plan, nullptr, n, n, n, d_rp, d_ci, d_va, d_rp, d_ci, d_va, (const size_t*)d_rpC2, d_ciC2, d_vC2);
  cudaDeviceSynchronize();
  b200sp_spgemm_plan_destroy(plan, nullptr);
  const std::vector<size_t> rpC = to_host(d_rpC, n + 1);
  const std::vector<int64_t> rpC2 = to_host(d_rpC2, n + 1);
  const std::vector<S> vC = to_host(d_vC, cnnz), vC2 = to_host(d_vC2, cnnz);
  const bool same = rc == 0 && (size_t)cnnz2 == cnnz && cnnz > 0 && std::memcmp(rpC.data(), rpC2.data(), sizeof(size_t) * (n + 1)) == 0 &&
                    to_host(d_ciC, cnnz) == to_host(d_ciC2, cnnz) && std::memcmp(vC.data(), vC2.data(), sizeof(S) * cnnz) == 0;
  if (!same) ++failures;
  std::printf("%s (int, size_t) spgemm through SPGEMM_SYMBOLIC/NUMERIC<...,true,true> : c_nnz=%zu, C ABI bits %s\n", name, cnnz,
              same ? "identical" : "DIFFER");
  kh.destroy_spgemm_handle();
  for (void* p : {(void*)d_rp, (void*)d_ci, (void*)d_va, (void*)d_rpC, (void*)d_ciC, (void*)d_vC, (void*)d_rpC2, (void*)d_ciC2, (void*)d_vC2})
    cudaFree(p);
  return failures;
}

int main() {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    std::printf("no CUDA device\n");
    return 77;
  }
  int failures = run<double>("f64") + run<float>("f32");
  std::printf("native SPGEMM_SYMBOLIC/NUMERIC calls: %d\n", Impl::native_spgemm_calls());
  failures += Impl::native_spgemm_calls();
  if (failures == 0) std::printf("SHIM SPGEMM64 DRIVER OK\n");
  return failures == 0 ? 0 : 1;
}
