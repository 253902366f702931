// Full specialisations of SPGEMM_JACOBI for Kokkos::Cuda that forward to libb200sparse.  Generic declaration:
// sparse/impl/KokkosSparse_spgemm_jacobi_spec.hpp:83-107; the native body being replaced: :113-166 (symbolic check,
// row flops, KokkosSPGEMM_jacobi_sparseacc, then sort_crs_matrix -- the library's rows come out sorted, no sort pass).
// Reuses the plan SPGEMM_SYMBOLIC's B200 specialisation left on the SPGEMMHandle (b200_spgemm_plan): spgemm_jacobi
// must follow spgemm_symbolic on the same handle, as in the reference (:118-122).
#ifndef KOKKOSSPARSE_SPGEMM_JACOBI_B200_TPL_SPEC_DECL_HPP_
#define KOKKOSSPARSE_SPGEMM_JACOBI_B200_TPL_SPEC_DECL_HPP_
#ifdef KOKKOSKERNELS_ENABLE_TPL_B200SPARSE

#include "KokkosSparse_b200_utils.hpp"

namespace KokkosSparse {
namespace Impl {

inline int b200_call_jacobi(b200sp_spgemm_plan* p, void* s, int m, int n, int k, const int* rA, const int* cA, const double* vA,
                            const int* rB, const int* cB, const double* vB, const int* rC, int* cC, double* vC, double omega,
                            const double* dinv) {
  return b200sp_spgemm_jacobi_f64_i32(p, s, m, n, k, rA, cA, vA, rB, cB, vB, rC, cC, vC, omega, dinv);
}
inline int b200_call_jacobi(b200sp_spgemm_plan* p, void* s, int m, int n, int k, const int* rA, const int* cA, const float* vA,
                            const int* rB, const int* cB, const float* vB, const int* rC, int* cC, float* vC, float omega,
                            const float* dinv) {
  return b200sp_spgemm_jacobi_f32_i32(p, s, m, n, k, rA, cA, vA, rB, cB, vB, rC, cC, vC, omega, dinv);
}

#define KOKKOSSPARSE_B200_SPGEMM_JACOBI_DECL(SCALAR, MEMSPACE, ETI_AVAIL)                                              \
  template <>                                                                                                          \
  struct SPGEMM_JACOBI<KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE),              \
                       KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE),        \
                       KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE),           \
                       KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE), KOKKOSSPARSE_B200_IV(int, MEMSPACE),              \
                       KOKKOSSPARSE_B200_IV(int, MEMSPACE), KOKKOSSPARSE_B200_IV(SCALAR, MEMSPACE),                    \
                       KOKKOSSPARSE_B200_DINV(SCALAR, MEMSPACE), true, ETI_AVAIL> {                                    \
    using KernelHandle    = KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE);                                                    \
    using c_int_view_t    = KOKKOSSPARSE_B200_IV(const int, MEMSPACE);                                                 \
    using int_view_t      = KOKKOSSPARSE_B200_IV(int, MEMSPACE);                                                       \
    using c_scalar_view_t = KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE);                                              \
    using scalar_view_t   = KOKKOSSPARSE_B200_IV(SCALAR, MEMSPACE);                                                    \
    using dinv_view_t     = KOKKOSSPARSE_B200_DINV(SCALAR, MEMSPACE);                                                  \
    static void spgemm_jacobi(KernelHandle* handle, typename KernelHandle::nnz_lno_t m,                                \
                              typename KernelHandle::nnz_lno_t n, typename KernelHandle::nnz_lno_t k,                  \
                              c_int_view_t row_mapA, c_int_view_t entriesA, c_scalar_view_t valuesA, bool,             \
                              c_int_view_t row_mapB, c_int_view_t entriesB, c_scalar_view_t valuesB, bool,             \
                              int_view_t row_mapC, int_view_t& entriesC, scalar_view_t& valuesC, const SCALAR omega,   \
                              dinv_view_t dinv) {                                                                      \
      auto* sh = handle->get_spgemm_handle();                                                                          \
      if (!sh->is_symbolic_called() || !sh->b200_spgemm_plan)                                                          \
        throw std::runtime_error("KokkosSparse::spgemm_jacobi: must first call spgemm_symbolic with the same handle."); \
      Kokkos::Profiling::pushRegion("KokkosSparse::spgemm_jacobi[TPL_B200," + Kokkos::ArithTraits<SCALAR>::name() + "]"); \
      void* stream = (void*)Kokkos::Cuda().cuda_stream();                                                              \
      KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200_call_jacobi(sh->b200_spgemm_plan, stream, m, n, k, row_mapA.data(),        \
                                                        entriesA.data(), valuesA.data(), row_mapB.data(),              \
                                                        entriesB.data(), valuesB.data(), row_mapC.data(),              \
                                                        entriesC.data(), valuesC.data(), omega, dinv.data()));         \
      Kokkos::Profiling::popRegion();                                                                                  \
    }                                                                                                                  \
  };

#define KOKKOSSPARSE_B200_SPGEMM_JACOBI_DECL_S(SCALAR, ETI_AVAIL)              \
  KOKKOSSPARSE_B200_SPGEMM_JACOBI_DECL(SCALAR, Kokkos::CudaSpace, ETI_AVAIL)   \
  KOKKOSSPARSE_B200_SPGEMM_JACOBI_DECL(SCALAR, Kokkos::CudaUVMSpace, ETI_AVAIL)

KOKKOSSPARSE_B200_SPGEMM_JACOBI_DECL_S(double, true)
KOKKOSSPARSE_B200_SPGEMM_JACOBI_DECL_S(float, true)
KOKKOSSPARSE_B200_SPGEMM_JACOBI_DECL_S(double, false)
KOKKOSSPARSE_B200_SPGEMM_JACOBI_DECL_S(float, false)

}  // namespace Impl
}  // namespace KokkosSparse
#endif
#endif
