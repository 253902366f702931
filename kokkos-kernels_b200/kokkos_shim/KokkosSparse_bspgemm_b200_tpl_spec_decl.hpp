// BSPGEMM_NUMERIC<..., true, *> for Kokkos::Cuda: forwards the block SpGEMM numeric phase to libb200sparse
// (b200sp_bspgemm_numeric_*) on the plan the point SPGEMM_SYMBOLIC specialisation created for the block graphs
// (KokkosSparse_spgemm_b200_tpl_spec_decl.hpp).  Generic declaration and the native struct's checks:
// sparse/impl/KokkosSparse_bspgemm_numeric_spec.hpp:113-191.  C's block rows come out sorted, so the native path's
// trailing sort_bsr_matrix (:187-189) has no counterpart.
#ifndef KOKKOSSPARSE_BSPGEMM_B200_TPL_SPEC_DECL_HPP_
#define KOKKOSSPARSE_BSPGEMM_B200_TPL_SPEC_DECL_HPP_
#ifdef KOKKOSKERNELS_ENABLE_TPL_B200SPARSE

#include "KokkosSparse_b200_utils.hpp"
#include "KokkosSparse_spgemm_b200_tpl_spec_decl.hpp"

namespace KokkosSparse {
namespace Impl {

inline int b200_call_bspgemm_numeric(b200sp_spgemm_plan* p, void* s, int m, int n, int k, int bs, const int* rA, const int* cA,
                                     const double* vA, const int* rB, const int* cB, const double* vB, const int* rC, int* cC,
                                     double* vC) {
  return b200sp_bspgemm_numeric_f64_i32(p, s, m, n, k, bs, rA, cA, vA, rB, cB, vB, rC, cC, vC);
}
inline int b200_call_bspgemm_numeric(b200sp_spgemm_plan* p, void* s, int m, int n, int k, int bs, const int* rA, const int* cA,
                                     const float* vA, const int* rB, const int* cB, const float* vB, const int* rC, int* cC,
                                     float* vC) {
  return b200sp_bspgemm_numeric_f32_i32(p, s, m, n, k, bs, rA, cA, vA, rB, cB, vB, rC, cC, vC);
}

template <class SpgemmHandle, class CIV, class CSV, class IV, class SV>
void bspgemm_numeric_b200(SpgemmHandle* sh, int m, int n, int k, int bs, const CIV& rowmapA, const CIV& entriesA,
                          const CSV& valuesA, bool transposeA, const CIV& rowmapB, const CIV& entriesB, const CSV& valuesB,
                          bool transposeB, const CIV& rowmapC, IV& entriesC, SV& valuesC) {
  if (transposeA || transposeB) throw std::runtime_error("KokkosSparse::bspgemm_numeric: transposing A or B is not supported");
  if (!sh->is_symbolic_called() || !sh->b200_spgemm_plan)  // bspgemm_numeric_spec.hpp:143-147
    throw std::runtime_error("KokkosSparse::bspgemm_numeric: must first call spgemm_symbolic with the same handle.");
  void* stream = (void*)Kokkos::Cuda().cuda_stream();  // as the point SpGEMM: the default instance
  KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200_call_bspgemm_numeric(sh->b200_spgemm_plan, stream, m, n, k, bs, rowmapA.data(),
                                                             entriesA.data(), valuesA.data(), rowmapB.data(), entriesB.data(),
                                                             valuesB.data(), rowmapC.data(), entriesC.data(), valuesC.data()));
  sh->set_computed_entries();
  sh->set_call_numeric();
}

#define KOKKOSSPARSE_B200_BSPGEMM_DECL(SCALAR, MEMSPACE, ETI_AVAIL)                                                           \
  template <>                                                                                                                \
  struct BSPGEMM_NUMERIC<KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE),                  \
                         KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE),            \
                         KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE),               \
                         KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE),            \
                         KOKKOSSPARSE_B200_IV(int, MEMSPACE), KOKKOSSPARSE_B200_IV(SCALAR, MEMSPACE), true, ETI_AVAIL> {     \
    using KernelHandle    = KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE);                                                          \
    using c_int_view_t    = KOKKOSSPARSE_B200_IV(const int, MEMSPACE);                                                       \
    using int_view_t      = KOKKOSSPARSE_B200_IV(int, MEMSPACE);                                                             \
    using c_scalar_view_t = KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE);                                                    \
    using scalar_view_t   = KOKKOSSPARSE_B200_IV(SCALAR, MEMSPACE);                                                          \
    static void bspgemm_numeric(KernelHandle* handle, typename KernelHandle::const_nnz_lno_t m,                              \
                                typename KernelHandle::const_nnz_lno_t n, typename KernelHandle::const_nnz_lno_t k,          \
                                typename KernelHandle::const_nnz_lno_t blockDim, c_int_view_t row_mapA,                      \
                                c_int_view_t entriesA, c_scalar_view_t valuesA, bool transposeA, c_int_view_t row_mapB,      \
                                c_int_view_t entriesB, c_scalar_view_t valuesB, bool transposeB, c_int_view_t row_mapC,      \
                                int_view_t& entriesC, scalar_view_t& valuesC) {                                              \
      Kokkos::Profiling::pushRegion("KokkosSparse::bspgemm_numeric[TPL_B200," + Kokkos::ArithTraits<SCALAR>::name() + "]"); \
      bspgemm_numeric_b200(handle->get_spgemm_handle(), m, n, k, blockDim, row_mapA, entriesA, valuesA, transposeA,         \
                           row_mapB, entriesB, valuesB, transposeB, row_mapC, entriesC, valuesC);                            \
      Kokkos::Profiling::popRegion();                                                                                        \
    }                                                                                                                        \
  };

#define KOKKOSSPARSE_B200_BSPGEMM_DECL_S(SCALAR, ETI_AVAIL)                  \
  KOKKOSSPARSE_B200_BSPGEMM_DECL(SCALAR, Kokkos::CudaSpace, ETI_AVAIL)       \
  KOKKOSSPARSE_B200_BSPGEMM_DECL(SCALAR, Kokkos::CudaUVMSpace, ETI_AVAIL)

KOKKOSSPARSE_B200_BSPGEMM_DECL_S(double, true)
KOKKOSSPARSE_B200_BSPGEMM_DECL_S(float, true)
KOKKOSSPARSE_B200_BSPGEMM_DECL_S(double, false)
KOKKOSSPARSE_B200_BSPGEMM_DECL_S(float, false)

}  // namespace Impl
}  // namespace KokkosSparse
#endif
#endif
