// Full specialisations of KokkosSparse::Impl::GMRES for Kokkos::Cuda that forward to libb200sparse.  Generic declaration:
// sparse/impl/KokkosSparse_gmres_spec.hpp:69-82 (one struct, a CrsMatrix and a BsrMatrix overload); the native body being
// replaced: :86-107 (GmresWrap<GMRESHandle>::gmres).
//
// Without a preconditioner the solve runs in the library (b200sp_gmres_* / b200sp_gmres_bsr_*) with the handle's m, tol,
// max_restart, ortho; the statistics go back through set_stats.  WITH a preconditioner the body calls the native GmresWrap, as the
// generic specialisation does: the front end hands the preconditioner over through a reinterpret_cast between two
// Preconditioner<> instantiations (sparse/src/KokkosSparse_gmres.hpp:150), so its dynamic type (MatrixPrec or a user class) cannot
// be recovered here.  (A maintainer who wants MatrixPrec on this path too intercepts in KokkosSparse::gmres itself, before
// that cast, with an accessor for MatrixPrec's private matrix -- INTEGRATION.md.)
// The plans live on the GMRESHandle: `b200sp_spmv_plan* b200_spmv_plan` / `b200sp_bsr_plan* b200_bsr_plan` (INTEGRATION.md).
#ifndef KOKKOSSPARSE_GMRES_B200_TPL_SPEC_DECL_HPP_
#define KOKKOSSPARSE_GMRES_B200_TPL_SPEC_DECL_HPP_
#ifdef KOKKOSKERNELS_ENABLE_TPL_B200SPARSE

#include "KokkosSparse_b200_utils.hpp"

namespace KokkosSparse {
namespace Impl {

inline int b200_call_gmres(b200sp_spmv_plan* p, void* s, int n, int64_t nnz, const int* rp, const int* ci, const double* v, const double* b,
                           double* x, int m, double tol, int mr, int ortho, int* it, double* res, int* flag) {
  return b200sp_gmres_f64_i32(p, s, n, nnz, rp, ci, v, nullptr, 0, nullptr, nullptr, nullptr, b, x, m, tol, mr, ortho, it, res, flag);
}
inline int b200_call_gmres(b200sp_spmv_plan* p, void* s, int n, int64_t nnz, const int* rp, const int* ci, const float* v, const float* b,
                           float* x, int m, float tol, int mr, int ortho, int* it, float* res, int* flag) {
  return b200sp_gmres_f32_i32(p, s, n, nnz, rp, ci, v, nullptr, 0, nullptr, nullptr, nullptr, b, x, m, tol, mr, ortho, it, res, flag);
}
inline int b200_call_gmres_bsr(b200sp_bsr_plan* p, void* s, int mb, int64_t nnzb, int bs, const int* rp, const int* ci, const double* v,
                               const double* b, double* x, int m, double tol, int mr, int ortho, int* it, double* res, int* flag) {
  return b200sp_gmres_bsr_f64_i32(p, s, mb, nnzb, bs, rp, ci, v, nullptr, 0, nullptr, nullptr, nullptr, b, x, m, tol, mr, ortho, it, res, flag);
}
inline int b200_call_gmres_bsr(b200sp_bsr_plan* p, void* s, int mb, int64_t nnzb, int bs, const int* rp, const int* ci, const float* v,
                               const float* b, float* x, int m, float tol, int mr, int ortho, int* it, float* res, int* flag) {
  return b200sp_gmres_bsr_f32_i32(p, s, mb, nnzb, bs, rp, ci, v, nullptr, 0, nullptr, nullptr, nullptr, b, x, m, tol, mr, ortho, it, res, flag);
}

#define KOKKOSSPARSE_B200_GMRES_DECL(SCALAR, MEMSPACE, ETI_AVAIL)                                                      \
  template <>                                                                                                          \
  struct GMRES<KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE), const SCALAR, const int, Kokkos::Device<Kokkos::Cuda, MEMSPACE>, \
               Kokkos::MemoryTraits<Kokkos::Unmanaged>, const int, KOKKOSSPARSE_B200_GMRES_VEC(const SCALAR, MEMSPACE), \
               KOKKOSSPARSE_B200_GMRES_VEC(SCALAR, MEMSPACE), true, ETI_AVAIL> {                                       \
    using KernelHandle = KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE);                                                       \
    using device_type  = Kokkos::Device<Kokkos::Cuda, MEMSPACE>;                                                       \
    using AMatrix  = CrsMatrix<const SCALAR, const int, device_type, Kokkos::MemoryTraits<Kokkos::Unmanaged>, const int>; \
    using BAMatrix = KokkosSparse::Experimental::BsrMatrix<const SCALAR, const int, device_type,                       \
                                                           Kokkos::MemoryTraits<Kokkos::Unmanaged>, const int>;        \
    using BType = KOKKOSSPARSE_B200_GMRES_VEC(const SCALAR, MEMSPACE);                                                 \
    using XType = KOKKOSSPARSE_B200_GMRES_VEC(SCALAR, MEMSPACE);                                                       \
    template <class GH>                                                                                                \
    static void finish(GH* gh, int it, SCALAR res, int flag) {                                                         \
      gh->set_stats(it, res, flag == 0 ? GH::Flag::Conv : (flag == 2 ? GH::Flag::LOA : GH::Flag::NoConv));             \
    }                                                                                                                  \
    static void gmres(KernelHandle* handle, const AMatrix& A, const BType& B, XType& X,                                \
                      KokkosSparse::Experimental::Preconditioner<AMatrix>* precond = nullptr) {                       \
      auto gh = handle->get_gmres_handle();                                                                            \
      using GH = typename std::remove_pointer<decltype(gh)>::type;                                                     \
      if (precond) return Experimental::GmresWrap<GH>::gmres(*gh, A, B, X, precond);                                   \
      if (!gh->b200_spmv_plan) KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200sp_spmv_plan_create(&gh->b200_spmv_plan, B200SP_SPMV_DEFAULT)); \
      int it = 0, flag = 0;                                                                                            \
      SCALAR res = 0;                                                                                                  \
      KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200_call_gmres(                                                                \
          gh->b200_spmv_plan, (void*)Kokkos::Cuda().cuda_stream(), A.numRows(), (int64_t)A.nnz(), A.graph.row_map.data(), \
          A.graph.entries.data(), A.values.data(), B.data(), X.data(), (int)gh->get_m(), (SCALAR)gh->get_tol(),        \
          (int)gh->get_max_restart(), gh->get_ortho() == GH::Ortho::MGS ? 1 : 0, &it, &res, &flag));                   \
      finish(gh, it, res, flag);                                                                                       \
    }                                                                                                                  \
    static void gmres(KernelHandle* handle, const BAMatrix& A, const BType& B, XType& X,                               \
                      KokkosSparse::Experimental::Preconditioner<BAMatrix>* precond = nullptr) {                      \
      auto gh = handle->get_gmres_handle();                                                                            \
      using GH = typename std::remove_pointer<decltype(gh)>::type;                                                     \
      if (precond) return Experimental::GmresWrap<GH>::gmres(*gh, A, B, X, precond);                                   \
      if (!gh->b200_bsr_plan) KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200sp_bsr_plan_create(&gh->b200_bsr_plan));            \
      int it = 0, flag = 0;                                                                                            \
      SCALAR res = 0;                                                                                                  \
      KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200_call_gmres_bsr(                                                            \
          gh->b200_bsr_plan, (void*)Kokkos::Cuda().cuda_stream(), A.numRows(), (int64_t)A.nnz(), A.blockDim(),         \
          A.graph.row_map.data(), A.graph.entries.data(), A.values.data(), B.data(), X.data(), (int)gh->get_m(),       \
          (SCALAR)gh->get_tol(), (int)gh->get_max_restart(), gh->get_ortho() == GH::Ortho::MGS ? 1 : 0, &it, &res, &flag)); \
      finish(gh, it, res, flag);                                                                                       \
    }                                                                                                                  \
  };

#define KOKKOSSPARSE_B200_GMRES_DECL_S(SCALAR, ETI_AVAIL)              \
  KOKKOSSPARSE_B200_GMRES_DECL(SCALAR, Kokkos::CudaSpace, ETI_AVAIL)   \
  KOKKOSSPARSE_B200_GMRES_DECL(SCALAR, Kokkos::CudaUVMSpace, ETI_AVAIL)

KOKKOSSPARSE_B200_GMRES_DECL_S(double, true)
KOKKOSSPARSE_B200_GMRES_DECL_S(float, true)
KOKKOSSPARSE_B200_GMRES_DECL_S(double, false)
KOKKOSSPARSE_B200_GMRES_DECL_S(float, false)

}  // namespace Impl
}  // namespace KokkosSparse
#endif
#endif
