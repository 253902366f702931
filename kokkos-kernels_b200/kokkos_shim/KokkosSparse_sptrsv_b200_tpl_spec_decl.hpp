// Full specialisations of SPTRSV_SYMBOLIC / SPTRSV_SOLVE for Kokkos::Cuda that forward to libb200sparse (b200sp_sptrsv_*: level
// sets).  Generic declarations: sparse/impl/KokkosSparse_sptrsv_symbolic_spec.hpp:63-70, sparse/impl/KokkosSparse_sptrsv_solve_spec.hpp:
// 79-93; the native bodies being replaced: :77-108 (lower_tri_symbolic / upper_tri_symbolic) and :99-210 (the per-algorithm solves).
// The plan hangs off the SPTRSVHandle (member `b200_sptrsv_plan`, INTEGRATION.md), which also says which triangle it is
// (is_lower_tri(), sparse/src/KokkosSparse_sptrsv_handle.hpp).  sptrsv_solve_streams runs the solves one after the other on their
// execution spaces' streams.
#ifndef KOKKOSSPARSE_SPTRSV_B200_TPL_SPEC_DECL_HPP_
#define KOKKOSSPARSE_SPTRSV_B200_TPL_SPEC_DECL_HPP_
#ifdef KOKKOSKERNELS_ENABLE_TPL_B200SPARSE

#include <vector>

#include "KokkosSparse_b200_utils.hpp"

namespace KokkosSparse {
namespace Impl {

inline int b200_call_sptrsv_solve(b200sp_sptrsv_plan* p, void* s, int n, const int* rp, const int* ci, const double* v, const double* b,
                                  double* x) {
  return b200sp_sptrsv_solve_f64_i32(p, s, n, rp, ci, v, b, x);
}
inline int b200_call_sptrsv_solve(b200sp_sptrsv_plan* p, void* s, int n, const int* rp, const int* ci, const float* v, const float* b,
                                  float* x) {
  return b200sp_sptrsv_solve_f32_i32(p, s, n, rp, ci, v, b, x);
}

#define KOKKOSSPARSE_B200_SPTRSV_DECL(SCALAR, MEMSPACE, ETI_AVAIL)                                                     \
  template <>                                                                                                          \
  struct SPTRSV_SYMBOLIC<Kokkos::Cuda, KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE), KOKKOSSPARSE_B200_RAV(const int, MEMSPACE), \
                         KOKKOSSPARSE_B200_RAV(const int, MEMSPACE), true, ETI_AVAIL> {                                \
    using KernelHandle = KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE);                                                       \
    using c_int_view_t = KOKKOSSPARSE_B200_RAV(const int, MEMSPACE);                                                   \
    static void sptrsv_symbolic(const Kokkos::Cuda& space, KernelHandle* handle, const c_int_view_t row_map,           \
                                const c_int_view_t entries) {                                                          \
      auto* sh = handle->get_sptrsv_handle();                                                                          \
      if (!sh->b200_sptrsv_plan) KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200sp_sptrsv_plan_create(&sh->b200_sptrsv_plan));   \
      KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200sp_sptrsv_symbolic_i32(sh->b200_sptrsv_plan, (void*)space.cuda_stream(),    \
                                                                  (int)row_map.extent(0) - 1, row_map.data(), entries.data(), \
                                                                  sh->is_lower_tri() ? 1 : 0));                        \
      sh->set_symbolic_complete();                                                                                     \
    }                                                                                                                  \
  };                                                                                                                   \
  template <>                                                                                                          \
  struct SPTRSV_SOLVE<Kokkos::Cuda, KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE), KOKKOSSPARSE_B200_RAV(const int, MEMSPACE), \
                      KOKKOSSPARSE_B200_RAV(const int, MEMSPACE), KOKKOSSPARSE_B200_RAV(const SCALAR, MEMSPACE),       \
                      KOKKOSSPARSE_B200_RAV(const SCALAR, MEMSPACE), KOKKOSSPARSE_B200_IV(SCALAR, MEMSPACE), true, ETI_AVAIL> { \
    using KernelHandle    = KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE);                                                    \
    using c_int_view_t    = KOKKOSSPARSE_B200_RAV(const int, MEMSPACE);                                                \
    using c_scalar_view_t = KOKKOSSPARSE_B200_RAV(const SCALAR, MEMSPACE);                                             \
    using scalar_view_t   = KOKKOSSPARSE_B200_IV(SCALAR, MEMSPACE);                                                    \
    static void sptrsv_solve(Kokkos::Cuda& space, KernelHandle* handle, const c_int_view_t row_map, const c_int_view_t entries, \
                             const c_scalar_view_t values, c_scalar_view_t b, scalar_view_t x) {                       \
      auto* sh = handle->get_sptrsv_handle();                                                                          \
      if (!sh->is_symbolic_complete() || !sh->b200_sptrsv_plan)                                                        \
        throw std::runtime_error("KokkosSparse::sptrsv_solve: sptrsv_symbolic was not called on this handle");         \
      Kokkos::Profiling::pushRegion("KokkosSparse::sptrsv_solve[TPL_B200," + Kokkos::ArithTraits<SCALAR>::name() + "]"); \
      KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200_call_sptrsv_solve(sh->b200_sptrsv_plan, (void*)space.cuda_stream(), (int)row_map.extent(0) - 1, \
                                                              row_map.data(), entries.data(), values.data(), b.data(), x.data())); \
      Kokkos::Profiling::popRegion();                                                                                  \
    }                                                                                                                  \
    static void sptrsv_solve_streams(const std::vector<Kokkos::Cuda>& execspace_v, std::vector<KernelHandle>& handle_v, \
                                     const std::vector<c_int_view_t>& row_map_v, const std::vector<c_int_view_t>& entries_v, \
                                     const std::vector<c_scalar_view_t>& values_v, const std::vector<c_scalar_view_t>& b_v, \
                                     std::vector<scalar_view_t>& x_v) {                                                \
      for (size_t i = 0; i < execspace_v.size(); ++i) {                                                                \
        Kokkos::Cuda space = execspace_v[i];                                                                           \
        sptrsv_solve(space, &handle_v[i], row_map_v[i], entries_v[i], values_v[i], b_v[i], x_v[i]);                    \
      }                                                                                                                \
    }                                                                                                                  \
  };

#define KOKKOSSPARSE_B200_SPTRSV_DECL_S(SCALAR, ETI_AVAIL)              \
  KOKKOSSPARSE_B200_SPTRSV_DECL(SCALAR, Kokkos::CudaSpace, ETI_AVAIL)   \
  KOKKOSSPARSE_B200_SPTRSV_DECL(SCALAR, Kokkos::CudaUVMSpace, ETI_AVAIL)

KOKKOSSPARSE_B200_SPTRSV_DECL_S(double, true)
KOKKOSSPARSE_B200_SPTRSV_DECL_S(float, true)
KOKKOSSPARSE_B200_SPTRSV_DECL_S(double, false)
KOKKOSSPARSE_B200_SPTRSV_DECL_S(float, false)

}  // namespace Impl
}  // namespace KokkosSparse
#endif
#endif
