// Full specialisations of GAUSS_SEIDEL_SYMBOLIC / GAUSS_SEIDEL_NUMERIC / GAUSS_SEIDEL_APPLY (CRS format) for Kokkos::Cuda that
// forward to libb200sparse.  Generic declarations: sparse/impl/KokkosSparse_gauss_seidel_spec.hpp:105-151; the native bodies
// being replaced (PointGaussSeidel through the handle's algorithm): :153-262.
//
// Needs one member on PointGaussSeidelHandle (sparse/src/KokkosSparse_gauss_seidel_handle.hpp, next to the colour views) and one
// on TwoStageGaussSeidelHandle (:513-673):
//   b200sp_gs_plan*  b200_gs_plan  = nullptr;   // released in the destructor with b200sp_gs_plan_destroy
//   b200sp_gs2_plan* b200_gs2_plan = nullptr;   // ... b200sp_gs2_plan_destroy
// and the usual called-flags (set_call_symbolic / set_call_numeric, :150-160).  The bodies dispatch on
// handle->get_gs_handle()->get_algorithm_type() as the native ones do (sparse/impl/KokkosSparse_gauss_seidel_spec.hpp:153-262):
//   GS_DEFAULT / GS_PERMUTED / GS_TEAM -> the point multicolour kernels (b200sp_gs_*);
//   GS_TWOSTAGE with inner Jacobi-Richardson sweeps -> b200sp_gs2_* (every product the library's SpMV), options read from the
//     handle (isCompactForm, getNumInnerSweeps, getNumOuterSweeps, getInnerDampFactor) at symbolic / apply time;
//   GS_CLUSTER and point numeric with a given inverse diagonal -> forwarded to
//     the native specialisation (tpl_spec_avail = false) of the same struct, i.e. unchanged behaviour.
// x / y with several columns: point sweeps column by column (independent systems), two-stage through nrhs.
#ifndef KOKKOSSPARSE_GAUSS_SEIDEL_B200_TPL_SPEC_DECL_HPP_
#define KOKKOSSPARSE_GAUSS_SEIDEL_B200_TPL_SPEC_DECL_HPP_
#ifdef KOKKOSKERNELS_ENABLE_TPL_B200SPARSE

#include "KokkosSparse_b200_utils.hpp"

namespace KokkosSparse {
namespace Impl {

inline int b200_call_gs_numeric(b200sp_gs_plan* p, void* s, int n, const int* rp, const int* ci, const double* v) {
  return b200sp_gs_numeric_f64_i32(p, s, n, rp, ci, v);
}
inline int b200_call_gs_numeric(b200sp_gs_plan* p, void* s, int n, const int* rp, const int* ci, const float* v) {
  return b200sp_gs_numeric_f32_i32(p, s, n, rp, ci, v);
}
inline int b200_call_gs_apply(b200sp_gs_plan* p, void* s, int n, const int* rp, const int* ci, const double* v, double* x, const double* y,
                              int zero, double omega, int sweeps, int dir) {
  return b200sp_gs_apply_f64_i32(p, s, n, rp, ci, v, x, y, zero, omega, sweeps, dir);
}
inline int b200_call_gs_apply(b200sp_gs_plan* p, void* s, int n, const int* rp, const int* ci, const float* v, float* x, const float* y,
                              int zero, float omega, int sweeps, int dir) {
  return b200sp_gs_apply_f32_i32(p, s, n, rp, ci, v, x, y, zero, omega, sweeps, dir);
}

template <class GsHandle>
inline b200sp_gs_plan* b200_gs_plan_of(GsHandle* gsh) {
  if (!gsh->b200_gs_plan) KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200sp_gs_plan_create(&gsh->b200_gs_plan));
  return gsh->b200_gs_plan;
}
// two-stage: the plan, with the handle's options pushed into it (the compact flag must be known before symbolic)
template <class Gs2Handle>
inline b200sp_gs2_plan* b200_gs2_plan_of(Gs2Handle* gs2) {
  if (!gs2->b200_gs2_plan) KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200sp_gs2_plan_create(&gs2->b200_gs2_plan));
  b200sp_gs2_plan* p = gs2->b200_gs2_plan;
  KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200sp_gs2_plan_set(p, B200SP_GS2_NUM_INNER_SWEEPS, (double)gs2->getNumInnerSweeps()));
  KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200sp_gs2_plan_set(p, B200SP_GS2_NUM_OUTER_SWEEPS, (double)gs2->getNumOuterSweeps()));
  KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200sp_gs2_plan_set(p, B200SP_GS2_INNER_DAMP_FACTOR, (double)gs2->getInnerDampFactor()));
  return p;
}
inline int b200_call_gs2_numeric(b200sp_gs2_plan* p, void* s, int n, int nc, const int* rp, const int* ci, const double* v, const double* d) {
  return b200sp_gs2_numeric_f64_i32(p, s, n, nc, rp, ci, v, d);
}
inline int b200_call_gs2_numeric(b200sp_gs2_plan* p, void* s, int n, int nc, const int* rp, const int* ci, const float* v, const float* d) {
  return b200sp_gs2_numeric_f32_i32(p, s, n, nc, rp, ci, v, d);
}
inline int b200_call_gs2_apply(b200sp_gs2_plan* p, void* s, int n, int nc, const int* rp, const int* ci, const double* v, double* x, int64_t ldx,
                               const double* y, int64_t ldy, int nrhs, int zero, double omega, int it, int dir) {
  return b200sp_gs2_apply_f64_i32(p, s, n, nc, rp, ci, v, x, ldx, y, ldy, nrhs, zero, omega, it, dir);
}
inline int b200_call_gs2_apply(b200sp_gs2_plan* p, void* s, int n, int nc, const int* rp, const int* ci, const float* v, float* x, int64_t ldx,
                               const float* y, int64_t ldy, int nrhs, int zero, float omega, int it, int dir) {
  return b200sp_gs2_apply_f32_i32(p, s, n, nc, rp, ci, v, x, ldx, y, ldy, nrhs, zero, omega, it, dir);
}
// what this TPL serves; everything else goes to the native specialisation
template <class KernelHandle>
inline int b200_gs_kind(KernelHandle* handle) {  // 0 point, 1 two-stage (inner sweeps or triangular solves), -1 native
  const auto a = handle->get_gs_handle()->get_algorithm_type();
  if (a == GS_CLUSTER) return -1;
  if (a == GS_TWOSTAGE) return 1;  // both forms: inner Jacobi-Richardson sweeps and the classic one (sptrsv; isTwoStage() == false)
  return 0;
}

#define KOKKOSSPARSE_B200_GS_DECL(SCALAR, MEMSPACE, ETI_AVAIL)                                                          \
  template <>                                                                                                          \
  struct GAUSS_SEIDEL_SYMBOLIC<Kokkos::Cuda, KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE), \
                               KOKKOSSPARSE_B200_IV(const int, MEMSPACE), true, ETI_AVAIL> {                           \
    using KernelHandle = KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE);                                                       \
    using c_int_view_t = KOKKOSSPARSE_B200_IV(const int, MEMSPACE);                                                    \
    static void gauss_seidel_symbolic(const Kokkos::Cuda& exec, KernelHandle* handle, typename KernelHandle::const_nnz_lno_t num_rows, \
                                      typename KernelHandle::const_nnz_lno_t num_cols, c_int_view_t row_map, c_int_view_t entries, \
                                      bool is_graph_symmetric) {                                                       \
      const int kind = b200_gs_kind(handle);                                                                           \
      if (kind < 0) {                                                                                                  \
        GAUSS_SEIDEL_SYMBOLIC<Kokkos::Cuda, KernelHandle, c_int_view_t, c_int_view_t, false, ETI_AVAIL>::gauss_seidel_symbolic( \
            exec, handle, num_rows, num_cols, row_map, entries, is_graph_symmetric);                                   \
        return;                                                                                                        \
      }                                                                                                                \
      if (kind == 1) {                                                                                                 \
        auto* gs2 = handle->get_twostage_gs_handle();                                                                  \
        b200sp_gs2_plan* p2 = b200_gs2_plan_of(gs2);                                                                   \
        KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200sp_gs2_plan_set(p2, B200SP_GS2_COMPACT_FORM, gs2->isCompactForm() ? 1.0 : 0.0)); \
        KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200sp_gs2_plan_set(p2, B200SP_GS2_TWO_STAGE, gs2->isTwoStage() ? 1.0 : 0.0));     \
        KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200sp_gs2_symbolic_i32(p2, (void*)exec.cuda_stream(), num_rows, num_cols, row_map.data(), \
                                                                 entries.data()));                                     \
        gs2->set_call_symbolic(true);                                                                                  \
        gs2->set_call_numeric(false);                                                                                  \
        return;                                                                                                        \
      }                                                                                                                \
      auto* gsh = handle->get_point_gs_handle();                                                                       \
      KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200sp_gs_symbolic_nc_i32(b200_gs_plan_of(gsh), (void*)exec.cuda_stream(), num_rows, num_cols, \
                                                                 row_map.data(), entries.data(), is_graph_symmetric ? 1 : 0)); \
      gsh->set_call_symbolic(true);                                                                                    \
      gsh->set_call_numeric(false);                                                                                    \
    }                                                                                                                  \
  };                                                                                                                   \
  template <>                                                                                                          \
  struct GAUSS_SEIDEL_NUMERIC<Kokkos::Cuda, KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE), KokkosSparse::SparseMatrixFormat::CRS, \
                              KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE),   \
                              KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE), true, ETI_AVAIL> {                         \
    using KernelHandle    = KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE);                                                    \
    using c_int_view_t    = KOKKOSSPARSE_B200_IV(const int, MEMSPACE);                                                 \
    using c_scalar_view_t = KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE);                                              \
    using Native = GAUSS_SEIDEL_NUMERIC<Kokkos::Cuda, KernelHandle, KokkosSparse::SparseMatrixFormat::CRS, c_int_view_t, c_int_view_t, \
                                        c_scalar_view_t, false, ETI_AVAIL>;                                           \
    static void two_stage_numeric(const Kokkos::Cuda& exec, KernelHandle* handle, int num_rows, int num_cols, c_int_view_t row_map, \
                                  c_int_view_t entries, c_scalar_view_t values, const SCALAR* given_inverse_diagonal) {  \
      auto* gs2 = handle->get_twostage_gs_handle();                                                                    \
      if (!gs2->is_symbolic_called()) throw std::runtime_error("KokkosSparse::gauss_seidel_numeric: call gauss_seidel_symbolic first"); \
      KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200_call_gs2_numeric(b200_gs2_plan_of(gs2), (void*)exec.cuda_stream(), num_rows, num_cols, \
                                                             row_map.data(), entries.data(), values.data(), given_inverse_diagonal)); \
      gs2->set_call_numeric(true);                                                                                     \
    }                                                                                                                  \
    static void gauss_seidel_numeric(const Kokkos::Cuda& exec, KernelHandle* handle, typename KernelHandle::const_nnz_lno_t num_rows, \
                                     typename KernelHandle::const_nnz_lno_t num_cols, c_int_view_t row_map, c_int_view_t entries, \
                                     c_scalar_view_t values, bool is_graph_symmetric) {                                \
      const int kind = b200_gs_kind(handle);                                                                           \
      if (kind < 0) return Native::gauss_seidel_numeric(exec, handle, num_rows, num_cols, row_map, entries, values, is_graph_symmetric); \
      if (kind == 1) return two_stage_numeric(exec, handle, num_rows, num_cols, row_map, entries, values, nullptr);    \
      auto* gsh = handle->get_point_gs_handle();                                                                       \
      if (!gsh->is_symbolic_called()) throw std::runtime_error("KokkosSparse::gauss_seidel_numeric: call gauss_seidel_symbolic first"); \
      KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200_call_gs_numeric(b200_gs_plan_of(gsh), (void*)exec.cuda_stream(), num_rows, row_map.data(), \
                                                            entries.data(), values.data()));                           \
      gsh->set_call_numeric(true);                                                                                     \
    }                                                                                                                  \
    static void gauss_seidel_numeric(const Kokkos::Cuda& exec, KernelHandle* handle, typename KernelHandle::const_nnz_lno_t num_rows, \
                                     typename KernelHandle::const_nnz_lno_t num_cols, c_int_view_t row_map, c_int_view_t entries, \
                                     c_scalar_view_t values, c_scalar_view_t given_inverse_diagonal, bool is_graph_symmetric) { \
      if (b200_gs_kind(handle) == 1)                                                                                   \
        return two_stage_numeric(exec, handle, num_rows, num_cols, row_map, entries, values, given_inverse_diagonal.data()); \
      /* point and cluster handles with a caller-supplied inverse diagonal keep the native path */                    \
      Native::gauss_seidel_numeric(exec, handle, num_rows, num_cols, row_map, entries, values, given_inverse_diagonal, is_graph_symmetric); \
    }                                                                                                                  \
  };                                                                                                                   \
  template <>                                                                                                          \
  struct GAUSS_SEIDEL_APPLY<Kokkos::Cuda, KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE), KokkosSparse::SparseMatrixFormat::CRS,  \
                            KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE),     \
                            KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE), KOKKOSSPARSE_B200_MV(SCALAR, MEMSPACE),     \
                            KOKKOSSPARSE_B200_MV(const SCALAR, MEMSPACE), true, ETI_AVAIL> {                           \
    using KernelHandle    = KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE);                                                    \
    using c_int_view_t    = KOKKOSSPARSE_B200_IV(const int, MEMSPACE);                                                 \
    using c_scalar_view_t = KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE);                                              \
    using x_view_t        = KOKKOSSPARSE_B200_MV(SCALAR, MEMSPACE);                                                    \
    using y_view_t        = KOKKOSSPARSE_B200_MV(const SCALAR, MEMSPACE);                                              \
    static void gauss_seidel_apply(const Kokkos::Cuda& exec, KernelHandle* handle, typename KernelHandle::const_nnz_lno_t num_rows, \
                                   typename KernelHandle::const_nnz_lno_t num_cols, c_int_view_t row_map, c_int_view_t entries, \
                                   c_scalar_view_t values, x_view_t x_lhs_output_vec, y_view_t y_rhs_input_vec,        \
                                   bool init_zero_x_vector, bool update_y_vector, typename KernelHandle::nnz_scalar_t omega, \
                                   int numIter, bool apply_forward, bool apply_backward) {                            \
      const int kind = b200_gs_kind(handle);                                                                           \
      if (kind < 0) {                                                                                                  \
        GAUSS_SEIDEL_APPLY<Kokkos::Cuda, KernelHandle, KokkosSparse::SparseMatrixFormat::CRS, c_int_view_t, c_int_view_t, c_scalar_view_t, \
                           x_view_t, y_view_t, false, ETI_AVAIL>::gauss_seidel_apply(exec, handle, num_rows, num_cols, row_map, entries, values, \
                                                                                     x_lhs_output_vec, y_rhs_input_vec, init_zero_x_vector, \
                                                                                     update_y_vector, omega, numIter, apply_forward,    \
                                                                                     apply_backward);                                 \
        return;                                                                                                        \
      }                                                                                                                \
      if (!apply_forward && !apply_backward) return;                                                                   \
      const int dir = (apply_forward && apply_backward) ? 0 : (apply_forward ? 1 : 2);                                 \
      if (kind == 1) {                                                                                                 \
        auto* gs2 = handle->get_twostage_gs_handle();                                                                  \
        if (!gs2->is_numeric_called()) throw std::runtime_error("KokkosSparse::gauss_seidel_apply: call gauss_seidel_numeric first"); \
        KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200_call_gs2_apply(                                                          \
            b200_gs2_plan_of(gs2), (void*)exec.cuda_stream(), num_rows, num_cols, row_map.data(), entries.data(), values.data(), \
            x_lhs_output_vec.data(), (int64_t)x_lhs_output_vec.stride(1), y_rhs_input_vec.data(), (int64_t)y_rhs_input_vec.stride(1), \
            (int)x_lhs_output_vec.extent(1), init_zero_x_vector ? 1 : 0, omega, numIter, dir));                        \
        return;                                                                                                        \
      }                                                                                                                \
      auto* gsh = handle->get_point_gs_handle();                                                                       \
      if (!gsh->is_numeric_called()) throw std::runtime_error("KokkosSparse::gauss_seidel_apply: call gauss_seidel_numeric first"); \
      for (size_t col = 0; col < x_lhs_output_vec.extent(1); ++col) /* LayoutLeft: a column is contiguous */           \
        KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200_call_gs_apply(                                                           \
            b200_gs_plan_of(gsh), (void*)exec.cuda_stream(), num_rows, row_map.data(), entries.data(), values.data(),  \
            x_lhs_output_vec.data() + col * x_lhs_output_vec.stride(1), y_rhs_input_vec.data() + col * y_rhs_input_vec.stride(1), \
            init_zero_x_vector ? 1 : 0, omega, numIter, dir));                                                         \
    }                                                                                                                  \
  };

#define KOKKOSSPARSE_B200_GS_DECL_S(SCALAR, ETI_AVAIL)              \
  KOKKOSSPARSE_B200_GS_DECL(SCALAR, Kokkos::CudaSpace, ETI_AVAIL)   \
  KOKKOSSPARSE_B200_GS_DECL(SCALAR, Kokkos::CudaUVMSpace, ETI_AVAIL)

KOKKOSSPARSE_B200_GS_DECL_S(double, true)
KOKKOSSPARSE_B200_GS_DECL_S(float, true)
KOKKOSSPARSE_B200_GS_DECL_S(double, false)
KOKKOSSPARSE_B200_GS_DECL_S(float, false)

}  // namespace Impl
}  // namespace KokkosSparse
#endif
#endif
