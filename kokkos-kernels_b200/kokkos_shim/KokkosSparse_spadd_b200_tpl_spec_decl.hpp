// Full specialisations of SPADD_SYMBOLIC / SPADD_NUMERIC for Kokkos::Cuda that forward to libb200sparse --
// the slot of the cuSPARSE csrgeam2 leg (sparse/tpls/KokkosSparse_spadd_symbolic_tpl_spec_decl.hpp:25-119,
// sparse/tpls/KokkosSparse_spadd_numeric_tpl_spec_decl.hpp:25-127).  Generic declarations:
// sparse/impl/KokkosSparse_spadd_symbolic_spec.hpp:70-80, ..._numeric_spec.hpp.
//
// Needs one member on SPADDHandle (sparse/src/KokkosSparse_spadd_handle.hpp, next to cusparseData at :107):
//   #ifdef KOKKOSKERNELS_ENABLE_TPL_B200SPARSE
//   struct SpaddB200Data { b200sp_spadd_plan* plan = nullptr; ~SpaddB200Data() { b200sp_spadd_plan_destroy(plan, nullptr); } };
//   SpaddB200Data b200Data;
//   #endif
// (INTEGRATION.md shows the patch).
#ifndef KOKKOSSPARSE_SPADD_B200_TPL_SPEC_DECL_HPP_
#define KOKKOSSPARSE_SPADD_B200_TPL_SPEC_DECL_HPP_
#ifdef KOKKOSKERNELS_ENABLE_TPL_B200SPARSE

#include "KokkosSparse_b200_utils.hpp"

namespace KokkosSparse {
namespace Impl {

inline int b200_call_spadd_numeric(b200sp_spadd_plan* p, void* s, int m, int n, const int* rA, const int* cA, const double* vA,
                                   double alpha, const int* rB, const int* cB, const double* vB, double beta, const int* rC,
                                   int* cC, double* vC) {
  return b200sp_spadd_numeric_f64_i32(p, s, m, n, rA, cA, vA, alpha, rB, cB, vB, beta, rC, cC, vC);
}
inline int b200_call_spadd_numeric(b200sp_spadd_plan* p, void* s, int m, int n, const int* rA, const int* cA, const float* vA,
                                   float alpha, const int* rB, const int* cB, const float* vB, float beta, const int* rC,
                                   int* cC, float* vC) {
  return b200sp_spadd_numeric_f32_i32(p, s, m, n, rA, cA, vA, alpha, rB, cB, vB, beta, rC, cC, vC);
}

#define KOKKOSSPARSE_B200_SPADD_DECL(SCALAR, ETI_SPEC_AVAIL)                                                           \
  template <>                                                                                                          \
  struct SPADD_SYMBOLIC<Kokkos::Cuda, KOKKOSSPARSE_B200_AKH(SCALAR), KOKKOSSPARSE_B200_AV(const int),                  \
                        KOKKOSSPARSE_B200_AV(const int), KOKKOSSPARSE_B200_AV(const int),                              \
                        KOKKOSSPARSE_B200_AV(const int), KOKKOSSPARSE_B200_AV(int), true, ETI_SPEC_AVAIL> {            \
    using kernelhandle_t          = KOKKOSSPARSE_B200_AKH(SCALAR);                                                     \
    using rowmap_view_t           = KOKKOSSPARSE_B200_AV(const int);                                                   \
    using non_const_rowmap_view_t = KOKKOSSPARSE_B200_AV(int);                                                         \
    using colidx_view_t           = KOKKOSSPARSE_B200_AV(const int);                                                   \
    static void spadd_symbolic(const Kokkos::Cuda& exec, kernelhandle_t* handle, const int m, const int n,             \
                               rowmap_view_t rowmapA, colidx_view_t colidxA, rowmap_view_t rowmapB,                    \
                               colidx_view_t colidxB, non_const_rowmap_view_t rowmapC) {                               \
      Kokkos::Profiling::pushRegion("KokkosSparse::spadd_symbolic[TPL_B200," + Kokkos::ArithTraits<SCALAR>::name() + "]"); \
      auto addHandle = handle->get_spadd_handle();                                                                     \
      auto& data     = addHandle->b200Data;                                                                            \
      if (data.plan) {                                                                                                 \
        b200sp_spadd_plan_destroy(data.plan, (void*)exec.cuda_stream());                                               \
        data.plan = nullptr;                                                                                           \
      }                                                                                                                \
      KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200sp_spadd_plan_create(&data.plan, addHandle->is_input_sorted() ? 1 : 0,      \
                                                                addHandle->is_input_merged() ? 1 : 0));                \
      int64_t c_nnz = 0;                                                                                               \
      KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200sp_spadd_symbolic_i32(data.plan, (void*)exec.cuda_stream(), m, n,           \
                                                                 rowmapA.data(), colidxA.data(), rowmapB.data(),       \
                                                                 colidxB.data(), rowmapC.data(), &c_nnz));             \
      addHandle->set_c_nnz(c_nnz);                                                                                     \
      addHandle->set_call_symbolic();                                                                                  \
      addHandle->set_call_numeric(false);                                                                              \
      Kokkos::Profiling::popRegion();                                                                                  \
    }                                                                                                                  \
  };                                                                                                                   \
  template <>                                                                                                          \
  struct SPADD_NUMERIC<Kokkos::Cuda, KOKKOSSPARSE_B200_AKH(SCALAR), KOKKOSSPARSE_B200_AV(const int),                   \
                       KOKKOSSPARSE_B200_AV(const int), KOKKOSSPARSE_B200_AV(const SCALAR),                            \
                       KOKKOSSPARSE_B200_AV(const int), KOKKOSSPARSE_B200_AV(const int),                               \
                       KOKKOSSPARSE_B200_AV(const SCALAR), KOKKOSSPARSE_B200_AV(const int), KOKKOSSPARSE_B200_AV(int), \
                       KOKKOSSPARSE_B200_AV(SCALAR), true, ETI_SPEC_AVAIL> {                                           \
    using kernelhandle_t           = KOKKOSSPARSE_B200_AKH(SCALAR);                                                    \
    using rowmap_view_t            = KOKKOSSPARSE_B200_AV(const int);                                                  \
    using colidx_view_t            = KOKKOSSPARSE_B200_AV(const int);                                                  \
    using non_const_colidx_view_t  = KOKKOSSPARSE_B200_AV(int);                                                        \
    using scalar_view_t            = KOKKOSSPARSE_B200_AV(const SCALAR);                                               \
    using non_const_scalar_view_t  = KOKKOSSPARSE_B200_AV(SCALAR);                                                     \
    static void spadd_numeric(const Kokkos::Cuda& exec, kernelhandle_t* handle, const int m, const int n,              \
                              const SCALAR alpha, rowmap_view_t rowmapA, colidx_view_t colidxA, scalar_view_t valuesA, \
                              const SCALAR beta, rowmap_view_t rowmapB, colidx_view_t colidxB, scalar_view_t valuesB,  \
                              rowmap_view_t rowmapC, non_const_colidx_view_t colidxC,                                  \
                              non_const_scalar_view_t valuesC) {                                                       \
      Kokkos::Profiling::pushRegion("KokkosSparse::spadd_numeric[TPL_B200," + Kokkos::ArithTraits<SCALAR>::name() + "]"); \
      auto addHandle = handle->get_spadd_handle();                                                                     \
      if (!addHandle->b200Data.plan) throw std::invalid_argument("spadd_numeric: call spadd_symbolic first");          \
      KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200_call_spadd_numeric(                                                        \
          addHandle->b200Data.plan, (void*)exec.cuda_stream(), m, n, rowmapA.data(), colidxA.data(), valuesA.data(),   \
          alpha, rowmapB.data(), colidxB.data(), valuesB.data(), beta, rowmapC.data(), colidxC.data(),                 \
          valuesC.data()));                                                                                            \
      addHandle->set_call_numeric();                                                                                   \
      Kokkos::Profiling::popRegion();                                                                                  \
    }                                                                                                                  \
  };

// both ETI flavours, like the cuSPARSE file (spadd_symbolic_tpl_spec_decl.hpp:121-160)
KOKKOSSPARSE_B200_SPADD_DECL(double, true)
KOKKOSSPARSE_B200_SPADD_DECL(float, true)
KOKKOSSPARSE_B200_SPADD_DECL(double, false)
KOKKOSSPARSE_B200_SPADD_DECL(float, false)

}  // namespace Impl
}  // namespace KokkosSparse
#endif
#endif
