// shim_half_driver.cpp -- the half_t SPMV_MV specialisations of the TPL_B200 shim, instantiated the way KokkosSparse::spmv
// picks them: the dispatch below names SPMV_MV with its defaulted tpl_spec_avail argument, so an unavailable combination
// would land in the native stand-in (which only counts its calls).  On a GPU it runs every layout pair on half LayoutLeft /
// LayoutRight views, compares the result bit for bit with a direct b200sp_spmm_f16_i32 call and checks it against a host
// reference.  Without a device it exits 77 after its static_asserts were compiled in.  Exit code 0 = all checks passed.
#define KOKKOSKERNELS_ENABLE_TPL_B200SPARSE
#define KOKKOS_HALF_T_IS_FLOAT 0
#include "Kokkos_Mock.hpp"
#include "Kokkos_Mock_Half.hpp"
#include "KokkosSparse_spmv_b200_tpl_spec_avail.hpp"
#include "KokkosSparse_spmv_b200_tpl_spec_decl.hpp"

#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

using half_t = Kokkos::Experimental::half_t;
using Dev    = Kokkos::Device<Kokkos::Cuda, Kokkos::CudaSpace>;
using UVM    = Kokkos::Device<Kokkos::Cuda, Kokkos::CudaUVMSpace>;
using UM     = Kokkos::MemoryTraits<Kokkos::Unmanaged>;
using UMRA   = Kokkos::MemoryTraits<Kokkos::Unmanaged | Kokkos::RandomAccess>;
using Hnd    = KokkosSparse::Impl::SPMVHandleImpl<Kokkos::Cuda, Kokkos::CudaSpace, half_t, int, int>;
using HndU   = KokkosSparse::Impl::SPMVHandleImpl<Kokkos::Cuda, Kokkos::CudaUVMSpace, half_t, int, int>;
using AMat   = KokkosSparse::CrsMatrix<const half_t, const int, Dev, UM, const int>;
using AMatU  = KokkosSparse::CrsMatrix<const half_t, const int, UVM, UM, const int>;
template <class L, class D = Dev> using XMV = Kokkos::View<const half_t**, L, D, UMRA>;
template <class L, class D = Dev> using YMV = Kokkos::View<half_t**, L, D, UM>;

namespace KokkosSparse {
namespace Impl {
// the native SPMV_MV (sparse/impl/KokkosSparse_spmv_spec.hpp:126-135, tpl = false): a stand-in that counts its calls
inline int& native_spmv_mv_calls() {
  static int n = 0;
  return n;
}
template <class ExecutionSpace, class Handle, class AMatrix, class XVector, class YVector>
struct SPMV_MV<ExecutionSpace, Handle, AMatrix, XVector, YVector, false, false> {
  template <class... Args>
  static void spmv_mv(Args&&...) {
    ++native_spmv_mv_calls();
  }
};
}  // namespace Impl
}  // namespace KokkosSparse

using KokkosSparse::Impl::spmv_mv_tpl_spec_avail;
using Kokkos::LayoutLeft;
using Kokkos::LayoutRight;
static_assert(spmv_mv_tpl_spec_avail<Kokkos::Cuda, Hnd, AMat, XMV<LayoutLeft>, YMV<LayoutLeft>>::value, "half LL");
static_assert(spmv_mv_tpl_spec_avail<Kokkos::Cuda, Hnd, AMat, XMV<LayoutRight>, YMV<LayoutLeft>>::value, "half RL");
static_assert(spmv_mv_tpl_spec_avail<Kokkos::Cuda, Hnd, AMat, XMV<LayoutLeft>, YMV<LayoutRight>>::value, "half LR");
static_assert(spmv_mv_tpl_spec_avail<Kokkos::Cuda, Hnd, AMat, XMV<LayoutRight>, YMV<LayoutRight>>::value, "half RR");
static_assert(spmv_mv_tpl_spec_avail<Kokkos::Cuda, HndU, AMatU, XMV<LayoutLeft, UVM>, YMV<LayoutLeft, UVM>>::value, "half UVM");
static_assert(spmv_mv_tpl_spec_avail<Kokkos::Cuda, HndU, AMatU, XMV<LayoutRight, UVM>, YMV<LayoutRight, UVM>>::value, "half UVM");
// rank 1 stays unavailable for half_t (no such cuSPARSE slot)
static_assert(!KokkosSparse::Impl::spmv_tpl_spec_avail<Kokkos::Cuda, Hnd, AMat, Kokkos::View<const half_t*, LayoutLeft, Dev, UMRA>,
                                                       Kokkos::View<half_t*, LayoutLeft, Dev, UM>>::value,
              "no rank-1 half");

// KokkosSparse::spmv's rank-2 dispatch: SPMV_MV with the defaulted availability argument
template <class XL, class YL>
void kk_spmv(const Kokkos::Cuda& exec, Hnd* h, const char* mode, half_t alpha, const AMat& A, const XMV<XL>& X, half_t beta,
             const YMV<YL>& Y) {
  KokkosSparse::Impl::SPMV_MV<Kokkos::Cuda, Hnd, AMat, XMV<XL>, YMV<YL>>::spmv_mv(exec, h, mode, alpha, A, X, beta, Y);
}

template <class T>
static T* to_dev(const std::vector<T>& h) {
  T* d = nullptr;
  cudaMalloc(&d, sizeof(T) * (h.size() ? h.size() : 1));
  cudaMemcpy(d, h.data(), sizeof(T) * h.size(), cudaMemcpyHostToDevice);
  return d;
}

static float h2f(half_t h) { return static_cast<float>(h); }

struct Case {
  int m, n, k;
  std::vector<int> rp, ci;
  std::vector<half_t> va, X, Y0;  // X and Y0 row-major
};

// one layout pair: the shim's result against a direct C ABI call on a second plan (same kernels: the same bits) and against a
// double-precision host reference (fp32 accumulation: a loose relative bound)
template <class XL, class YL>
static int run_pair(const Case& c, const char* name, cudaStream_t stream, const int* d_rp, const int* d_ci, const half_t* d_va) {
  constexpr bool xr = std::is_same<XL, LayoutRight>::value, yr = std::is_same<YL, LayoutRight>::value;
  const int m = c.m, n = c.n, k = c.k;
  std::vector<half_t> Xl(n * k), Yl(m * k);
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < k; ++j) Xl[xr ? i * k + j : j * n + i] = c.X[i * k + j];
  for (int i = 0; i < m; ++i)
    for (int j = 0; j < k; ++j) Yl[yr ? i * k + j : j * m + i] = c.Y0[i * k + j];
  half_t *d_X = to_dev(Xl), *d_Y = to_dev(Yl), *d_Yc = to_dev(Yl);
  const half_t alpha(1.5f), beta(-0.5f);
  Kokkos::Cuda exec(stream);
  Hnd handle(KokkosSparse::SPMV_DEFAULT);
  AMat A(m, n, c.ci.size(), d_va, const_cast<int*>(d_rp), const_cast<int*>(d_ci));
  for (int rep = 0; rep < 2; ++rep) {  // the second call reuses the plan's analysis
    cudaMemcpy(d_Y, Yl.data(), sizeof(half_t) * Yl.size(), cudaMemcpyHostToDevice);
    kk_spmv<XL, YL>(exec, &handle, "N", alpha, A, XMV<XL>(d_X, n, k), beta, YMV<YL>(d_Y, m, k));
  }
  b200sp_spmv_plan* plan = nullptr;
  b200sp_spmv_plan_create(&plan, 0);
  int rc = b200sp_spmm_f16_i32(plan, stream, 'N', m, n, (int64_t)c.ci.size(), k, 1.5f, d_rp, d_ci, (const uint16_t*)d_va,
                               (const uint16_t*)d_X, xr ? k : n, xr, -0.5f, (uint16_t*)d_Yc, yr ? k : m, yr);
  cudaStreamSynchronize(stream);
  b200sp_spmv_plan_destroy(plan, stream);
  std::vector<half_t> got(m * k), ref(m * k);
  cudaMemcpy(got.data(), d_Y, sizeof(half_t) * got.size(), cudaMemcpyDeviceToHost);
  cudaMemcpy(ref.data(), d_Yc, sizeof(half_t) * ref.size(), cudaMemcpyDeviceToHost);
  int bad = rc != 0 ? 1 : 0;
  if (std::memcmp(got.data(), ref.data(), sizeof(half_t) * got.size()) != 0) ++bad;
  for (int i = 0; i < m; ++i)
    for (int j = 0; j < k; ++j) {
      double s = 0, a = 0;
      for (int e = c.rp[i]; e < c.rp[i + 1]; ++e) {
        s += (double)h2f(c.va[e]) * h2f(c.X[c.ci[e] * k + j]);
        a += std::fabs((double)h2f(c.va[e]) * h2f(c.X[c.ci[e] * k + j]));
      }
      const double y0 = h2f(c.Y0[i * k + j]);
      const double e = 1.5 * s - 0.5 * y0, g = h2f(got[yr ? i * k + j : j * m + i]);
      if (!(std::fabs(g - e) <= 1e-3 * std::fabs(e) + 1e-5 * (1.5 * a + 0.5 * std::fabs(y0)) + 1e-7)) ++bad;
    }
  std::printf("half spmv_mv %s through SPMV_MV<...,false,true>::spmv_mv : %s\n", name, bad ? "MISMATCH" : "ok");
  cudaFree(d_X);
  cudaFree(d_Y);
  cudaFree(d_Yc);
  return bad;
}

int main() {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    std::printf("no CUDA device\n");
    return 77;
  }
  Case c;
  c.m = 3000, c.n = 2500, c.k = 16;
  c.rp.assign(c.m + 1, 0);
  unsigned s = 12345u;
  auto rnd = [&s]() { return (s = s * 1664525u + 1013904223u) >> 8; };
  for (int i = 0; i < c.m; ++i) {
    const int len = (i % 97 == 0) ? 300 : (int)(rnd() % 40);  // a few rows of several items
    for (int e = 0; e < len; ++e) {
      c.ci.push_back((int)(rnd() % c.n));
      c.va.push_back(half_t(((int)(rnd() % 2001) - 1000) / 512.0f));
    }
    c.rp[i + 1] = (int)c.ci.size();
  }
  for (int i = 0; i < c.n * c.k; ++i) c.X.push_back(half_t(((int)(rnd() % 2001) - 1000) / 256.0f));
  for (int i = 0; i < c.m * c.k; ++i) c.Y0.push_back(half_t(((int)(rnd() % 2001) - 1000) / 128.0f));
  int *d_rp = to_dev(c.rp), *d_ci = to_dev(c.ci);
  half_t* d_va = to_dev(c.va);
  cudaStream_t stream;
  cudaStreamCreate(&stream);
  int failures = 0;
  failures += run_pair<LayoutLeft, LayoutLeft>(c, "LL", stream, d_rp, d_ci, d_va);
  failures += run_pair<LayoutRight, LayoutLeft>(c, "RL", stream, d_rp, d_ci, d_va);
  failures += run_pair<LayoutLeft, LayoutRight>(c, "LR", stream, d_rp, d_ci, d_va);
  failures += run_pair<LayoutRight, LayoutRight>(c, "RR", stream, d_rp, d_ci, d_va);
  const int native = KokkosSparse::Impl::native_spmv_mv_calls();
  std::printf("native SPMV_MV calls: %d\n", native);
  failures += native;
  cudaFree(d_rp);
  cudaFree(d_ci);
  cudaFree(d_va);
  cudaStreamDestroy(stream);
  if (failures) {
    std::printf("SHIM HALF DRIVER FAILED (%d)\n", failures);
    return 1;
  }
  std::printf("SHIM HALF DRIVER OK\n");
  return 0;
}
