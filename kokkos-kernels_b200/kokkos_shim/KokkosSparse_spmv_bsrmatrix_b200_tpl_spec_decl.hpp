// Full specialisations of KokkosSparse::Impl::SPMV_BSRMATRIX / SPMV_MV_BSRMATRIX for Kokkos::Cuda that forward to
// libb200sparse -- the slot spmv_bsr_cusparse / spmv_mv_bsr_cusparse occupy
// (sparse/tpls/KokkosSparse_spmv_bsrmatrix_tpl_spec_decl.hpp:463-493,516-546).  Generic declarations being
// specialised: sparse/impl/KokkosSparse_spmv_bsrmatrix_spec.hpp:89-112 (rank 1: <..., tpl, eti>; rank 2:
// <..., integerScalarType, tpl, eti>).
//
// The cuSPARSE bodies throw for every mode but N (decl:294-300,387-393) and the front end routes T/C/H around
// them (KokkosSparse_spmv.hpp:322-360 leaves `useNative` for rank 1 as the algorithm says, so 'T' with a cuSPARSE
// build reaches that throw); these bodies accept N, C, T, H.  blockDim() == 1 never arrives here
// (KokkosSparse_spmv.hpp:169-185) but is accepted as well.
#ifndef KOKKOSSPARSE_SPMV_BSRMATRIX_B200_TPL_SPEC_DECL_HPP_
#define KOKKOSSPARSE_SPMV_BSRMATRIX_B200_TPL_SPEC_DECL_HPP_
#ifdef KOKKOSKERNELS_ENABLE_TPL_B200SPARSE

#include "KokkosSparse_b200_utils.hpp"

namespace KokkosSparse {
namespace Impl {

// Per-matrix state hung off SPMVHandleImpl::tpl_rank1 / tpl_rank2 (CuSparse9_SpMV_Data's place,
// sparse/src/KokkosSparse_spmv_handle.hpp:137-160)
struct B200_BsrSpMV_Data : public TPL_SpMV_Data<Kokkos::Cuda> {
  B200_BsrSpMV_Data(const Kokkos::Cuda& exec_) : TPL_SpMV_Data(exec_) {
    KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200sp_bsr_plan_create(&plan));
  }
  ~B200_BsrSpMV_Data() { b200sp_bsr_plan_destroy(plan, (void*)exec.cuda_stream()); }
  b200sp_bsr_plan* plan = nullptr;
};

inline b200sp_bsr_plan* b200_bsr_plan_of(TPL_SpMV_Data<Kokkos::Cuda>*& slot, const Kokkos::Cuda& exec) {
  B200_BsrSpMV_Data* sub;
  if (slot) {
    sub = dynamic_cast<B200_BsrSpMV_Data*>(slot);
    if (!sub) throw std::runtime_error("KokkosSparse::spmv: subhandle is not set up for b200sparse (BsrMatrix)");
    sub->set_exec_space(exec);
  } else {
    sub  = new B200_BsrSpMV_Data(exec);
    slot = sub;
  }
  return sub->plan;
}

inline int b200_call_bsr_spmv(b200sp_bsr_plan* p, void* s, char mode, int mb, int nb, int64_t nnzb, int bs, double alpha,
                              const int* rp, const int* ci, const double* v, const double* x, double beta, double* y) {
  return b200sp_bsr_spmv_f64_i32(p, s, mode, mb, nb, nnzb, bs, alpha, rp, ci, v, x, beta, y);
}
inline int b200_call_bsr_spmv(b200sp_bsr_plan* p, void* s, char mode, int mb, int nb, int64_t nnzb, int bs, float alpha,
                              const int* rp, const int* ci, const float* v, const float* x, float beta, float* y) {
  return b200sp_bsr_spmv_f32_i32(p, s, mode, mb, nb, nnzb, bs, alpha, rp, ci, v, x, beta, y);
}
inline int b200_call_bsr_spmm(b200sp_bsr_plan* p, void* s, char mode, int mb, int nb, int64_t nnzb, int bs, int k,
                              double alpha, const int* rp, const int* ci, const double* v, const double* X, int64_t ldx,
                              int xrm, double beta, double* Y, int64_t ldy, int yrm) {
  return b200sp_bsr_spmm_f64_i32(p, s, mode, mb, nb, nnzb, bs, k, alpha, rp, ci, v, X, ldx, xrm, beta, Y, ldy, yrm);
}
inline int b200_call_bsr_spmm(b200sp_bsr_plan* p, void* s, char mode, int mb, int nb, int64_t nnzb, int bs, int k,
                              float alpha, const int* rp, const int* ci, const float* v, const float* X, int64_t ldx, int xrm,
                              float beta, float* Y, int64_t ldy, int yrm) {
  return b200sp_bsr_spmm_f32_i32(p, s, mode, mb, nb, nnzb, bs, k, alpha, rp, ci, v, X, ldx, xrm, beta, Y, ldy, yrm);
}

#define KOKKOSSPARSE_B200_SPMV_BSR_DECL(SCALAR, LAYOUT, MEMSPACE)                                                     \
  template <>                                                                                                         \
  struct SPMV_BSRMATRIX<                                                                                              \
      Kokkos::Cuda, SPMVHandleImpl<Kokkos::Cuda, MEMSPACE, SCALAR, int, int>,                                         \
      ::KokkosSparse::Experimental::BsrMatrix<SCALAR const, int const, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,        \
                                              Kokkos::MemoryTraits<Kokkos::Unmanaged>, int const>,                    \
      Kokkos::View<SCALAR const*, LAYOUT, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                                     \
                   Kokkos::MemoryTraits<Kokkos::Unmanaged | Kokkos::RandomAccess>>,                                   \
      Kokkos::View<SCALAR*, LAYOUT, Kokkos::Device<Kokkos::Cuda, MEMSPACE>, Kokkos::MemoryTraits<Kokkos::Unmanaged>>, \
      true> { /* eti: the default argument, as the cuSPARSE specialisation leaves it (tpl_spec_decl.hpp:470) */     \
    using device_type = Kokkos::Device<Kokkos::Cuda, MEMSPACE>;                                                       \
    using Handle      = SPMVHandleImpl<Kokkos::Cuda, MEMSPACE, SCALAR, int, int>;                                     \
    using AMatrix     = ::KokkosSparse::Experimental::BsrMatrix<SCALAR const, int const, device_type,                 \
                                                            Kokkos::MemoryTraits<Kokkos::Unmanaged>, int const>;      \
    using XVector = Kokkos::View<SCALAR const*, LAYOUT, device_type,                                                  \
                                 Kokkos::MemoryTraits<Kokkos::Unmanaged | Kokkos::RandomAccess>>;                     \
    using YVector = Kokkos::View<SCALAR*, LAYOUT, device_type, Kokkos::MemoryTraits<Kokkos::Unmanaged>>;              \
    using coefficient_type = typename YVector::non_const_value_type;                                                  \
    static void spmv_bsrmatrix(const Kokkos::Cuda& exec, Handle* handle, const char mode[],                           \
                               const coefficient_type& alpha, const AMatrix& A, const XVector& x,                     \
                               const coefficient_type& beta, const YVector& y) {                                      \
      Kokkos::Profiling::pushRegion("KokkosSparse::spmv[TPL_B200,BSRMATRIX," + Kokkos::ArithTraits<SCALAR>::name() + "]"); \
      b200sp_bsr_plan* plan = b200_bsr_plan_of(handle->tpl_rank1, exec);                                              \
      KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200_call_bsr_spmv(                                                            \
          plan, (void*)exec.cuda_stream(), mode[0], A.numRows(), A.numCols(), (int64_t)A.nnz(), A.blockDim(), alpha,  \
          A.graph.row_map.data(), A.graph.entries.data(), A.values.data(), x.data(), beta, y.data()));                \
      Kokkos::Profiling::popRegion();                                                                                 \
    }                                                                                                                 \
  };                                                                                                                  \
  template <>                                                                                                         \
  struct SPMV_MV_BSRMATRIX<                                                                                           \
      Kokkos::Cuda, SPMVHandleImpl<Kokkos::Cuda, MEMSPACE, SCALAR, int, int>,                                         \
      ::KokkosSparse::Experimental::BsrMatrix<SCALAR const, int const, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,        \
                                              Kokkos::MemoryTraits<Kokkos::Unmanaged>, int const>,                    \
      Kokkos::View<SCALAR const**, LAYOUT, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                                    \
                   Kokkos::MemoryTraits<Kokkos::Unmanaged | Kokkos::RandomAccess>>,                                   \
      Kokkos::View<SCALAR**, LAYOUT, Kokkos::Device<Kokkos::Cuda, MEMSPACE>, Kokkos::MemoryTraits<Kokkos::Unmanaged>>, \
      false, true> { /* eti: the default argument */                                                                  \
    using device_type = Kokkos::Device<Kokkos::Cuda, MEMSPACE>;                                                       \
    using Handle      = SPMVHandleImpl<Kokkos::Cuda, MEMSPACE, SCALAR, int, int>;                                     \
    using AMatrix     = ::KokkosSparse::Experimental::BsrMatrix<SCALAR const, int const, device_type,                 \
                                                            Kokkos::MemoryTraits<Kokkos::Unmanaged>, int const>;      \
    using XVector = Kokkos::View<SCALAR const**, LAYOUT, device_type,                                                 \
                                 Kokkos::MemoryTraits<Kokkos::Unmanaged | Kokkos::RandomAccess>>;                     \
    using YVector = Kokkos::View<SCALAR**, LAYOUT, device_type, Kokkos::MemoryTraits<Kokkos::Unmanaged>>;             \
    using coefficient_type = typename YVector::non_const_value_type;                                                  \
    static void spmv_mv_bsrmatrix(const Kokkos::Cuda& exec, Handle* handle, const char mode[],                        \
                                  const coefficient_type& alpha, const AMatrix& A, const XVector& X,                  \
                                  const coefficient_type& beta, const YVector& Y) {                                   \
      Kokkos::Profiling::pushRegion("KokkosSparse::spmv[TPL_B200,BSRMATRIX," + Kokkos::ArithTraits<SCALAR>::name() + "]"); \
      b200sp_bsr_plan* plan = b200_bsr_plan_of(handle->tpl_rank2, exec);                                              \
      /* SPMV_BSR_TC: the handle asks for tensor cores (spmv_bsrmatrix_spec.hpp:176-177) */                           \
      KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200sp_bsr_plan_set_algorithm(                                                 \
          plan, handle->algo == SPMV_BSR_TC ? B200SP_BSR_ALGO_TENSOR_CORES : B200SP_BSR_ALGO_DEFAULT));               \
      constexpr int rm  = std::is_same<LAYOUT, Kokkos::LayoutRight>::value ? 1 : 0;                                   \
      const int64_t ldx = rm ? (int64_t)X.stride(0) : (int64_t)X.stride(1);                                           \
      const int64_t ldy = rm ? (int64_t)Y.stride(0) : (int64_t)Y.stride(1);                                           \
      KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200_call_bsr_spmm(                                                            \
          plan, (void*)exec.cuda_stream(), mode[0], A.numRows(), A.numCols(), (int64_t)A.nnz(), A.blockDim(),         \
          (int)X.extent(1), alpha, A.graph.row_map.data(), A.graph.entries.data(), A.values.data(), X.data(), ldx, rm, \
          beta, Y.data(), ldy, rm));                                                                                  \
      Kokkos::Profiling::popRegion();                                                                                 \
    }                                                                                                                 \
  };

#define KOKKOSSPARSE_B200_SPMV_BSR_DECL_ALL(SCALAR, MEMSPACE)            \
  KOKKOSSPARSE_B200_SPMV_BSR_DECL(SCALAR, Kokkos::LayoutLeft, MEMSPACE)  \
  KOKKOSSPARSE_B200_SPMV_BSR_DECL(SCALAR, Kokkos::LayoutRight, MEMSPACE)

KOKKOSSPARSE_B200_SPMV_BSR_DECL_ALL(double, Kokkos::CudaSpace)
KOKKOSSPARSE_B200_SPMV_BSR_DECL_ALL(float, Kokkos::CudaSpace)
KOKKOSSPARSE_B200_SPMV_BSR_DECL_ALL(double, Kokkos::CudaUVMSpace)
KOKKOSSPARSE_B200_SPMV_BSR_DECL_ALL(float, Kokkos::CudaUVMSpace)

#undef KOKKOSSPARSE_B200_SPMV_BSR_DECL_ALL
}  // namespace Impl
}  // namespace KokkosSparse
#endif
#endif
