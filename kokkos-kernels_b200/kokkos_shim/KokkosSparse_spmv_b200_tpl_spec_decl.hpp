// Full specialisations of KokkosSparse::Impl::SPMV / SPMV_MV for Kokkos::Cuda that forward to
// libb200sparse -- the slot spmv_cusparse / spmm_cusparse occupy
// (sparse/tpls/KokkosSparse_spmv_tpl_spec_decl.hpp:199-225,
//  sparse/tpls/KokkosSparse_spmv_mv_tpl_spec_decl.hpp:198-225).  Generic declarations being
// specialised: sparse/impl/KokkosSparse_spmv_spec.hpp:92-100,126-135.
#ifndef KOKKOSSPARSE_SPMV_B200_TPL_SPEC_DECL_HPP_
#define KOKKOSSPARSE_SPMV_B200_TPL_SPEC_DECL_HPP_
#ifdef KOKKOSKERNELS_ENABLE_TPL_B200SPARSE

#include "KokkosSparse_b200_utils.hpp"

namespace KokkosSparse {
namespace Impl {

inline b200sp_spmv_plan* b200_plan_of(TPL_SpMV_Data<Kokkos::Cuda>*& slot, const Kokkos::Cuda& exec, int algo) {
  B200_SpMV_Data* sub;
  if (slot) {
    sub = dynamic_cast<B200_SpMV_Data*>(slot);
    if (!sub) throw std::runtime_error("KokkosSparse::spmv: subhandle is not set up for b200sparse");
    sub->set_exec_space(exec);  // fences the old stream when the instance changes (spmv_handle.hpp:95-104)
  } else {
    sub  = new B200_SpMV_Data(exec, algo);
    slot = sub;
  }
  return sub->plan;
}

inline int b200_call_spmv(b200sp_spmv_plan* p, void* s, char mode, int m, int n, int64_t nnz, double alpha, const int* rp,
                          const int* ci, const double* v, const double* x, double beta, double* y) {
  return b200sp_spmv_f64_i32(p, s, mode, m, n, nnz, alpha, rp, ci, v, x, beta, y);
}
inline int b200_call_spmv(b200sp_spmv_plan* p, void* s, char mode, int m, int n, int64_t nnz, float alpha, const int* rp,
                          const int* ci, const float* v, const float* x, float beta, float* y) {
  return b200sp_spmv_f32_i32(p, s, mode, m, n, nnz, alpha, rp, ci, v, x, beta, y);
}
inline int b200_call_spmm(b200sp_spmv_plan* p, void* s, char mode, int m, int n, int64_t nnz, int k, double alpha,
                          const int* rp, const int* ci, const double* v, const double* X, int64_t ldx, int xrm, double beta,
                          double* Y, int64_t ldy, int yrm) {
  return b200sp_spmm_f64_i32(p, s, mode, m, n, nnz, k, alpha, rp, ci, v, X, ldx, xrm, beta, Y, ldy, yrm);
}
inline int b200_call_spmm(b200sp_spmv_plan* p, void* s, char mode, int m, int n, int64_t nnz, int k, float alpha,
                          const int* rp, const int* ci, const float* v, const float* X, int64_t ldx, int xrm, float beta,
                          float* Y, int64_t ldy, int yrm) {
  return b200sp_spmm_f32_i32(p, s, mode, m, n, nnz, k, alpha, rp, ci, v, X, ldx, xrm, beta, Y, ldy, yrm);
}

#define KOKKOSSPARSE_B200_SPMV_DECL(SCALAR, LAYOUT, MEMSPACE)                                                        \
  template <>                                                                                                        \
  struct SPMV<Kokkos::Cuda, SPMVHandleImpl<Kokkos::Cuda, MEMSPACE, SCALAR, int, int>,                                \
              CrsMatrix<SCALAR const, int const, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                             \
                        Kokkos::MemoryTraits<Kokkos::Unmanaged>, int const>,                                         \
              Kokkos::View<SCALAR const*, LAYOUT, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                            \
                           Kokkos::MemoryTraits<Kokkos::Unmanaged | Kokkos::RandomAccess>>,                          \
              Kokkos::View<SCALAR*, LAYOUT, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                                  \
                           Kokkos::MemoryTraits<Kokkos::Unmanaged>>,                                                 \
              true> {                                                                                                \
    using device_type = Kokkos::Device<Kokkos::Cuda, MEMSPACE>;                                                      \
    using Handle      = SPMVHandleImpl<Kokkos::Cuda, MEMSPACE, SCALAR, int, int>;                                    \
    using AMatrix = CrsMatrix<SCALAR const, int const, device_type, Kokkos::MemoryTraits<Kokkos::Unmanaged>, int const>; \
    using XVector = Kokkos::View<SCALAR const*, LAYOUT, device_type,                                                 \
                                 Kokkos::MemoryTraits<Kokkos::Unmanaged | Kokkos::RandomAccess>>;                    \
    using YVector = Kokkos::View<SCALAR*, LAYOUT, device_type, Kokkos::MemoryTraits<Kokkos::Unmanaged>>;             \
    using coefficient_type = typename YVector::non_const_value_type;                                                 \
    static void spmv(const Kokkos::Cuda& exec, Handle* handle, const char mode[], const coefficient_type& alpha,     \
                     const AMatrix& A, const XVector& x, const coefficient_type& beta, const YVector& y) {           \
      Kokkos::Profiling::pushRegion("KokkosSparse::spmv[TPL_B200," + Kokkos::ArithTraits<SCALAR>::name() + "]");     \
      b200sp_spmv_plan* plan = b200_plan_of(handle->tpl_rank1, exec, b200_spmv_algo(handle->get_algorithm()));       \
      KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200_call_spmv(                                                               \
          plan, (void*)exec.cuda_stream(), mode[0], A.numRows(), A.numCols(), (int64_t)A.nnz(), alpha,               \
          A.graph.row_map.data(), A.graph.entries.data(), A.values.data(), x.data(), beta, y.data()));               \
      Kokkos::Profiling::popRegion();                                                                                \
    }                                                                                                                \
  };

#define KOKKOSSPARSE_B200_SPMV_MV_DECL(SCALAR, XL, YL, MEMSPACE)                                                     \
  template <>                                                                                                        \
  struct SPMV_MV<Kokkos::Cuda, SPMVHandleImpl<Kokkos::Cuda, MEMSPACE, SCALAR, int, int>,                             \
                 CrsMatrix<SCALAR const, int const, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                          \
                           Kokkos::MemoryTraits<Kokkos::Unmanaged>, int const>,                                      \
                 Kokkos::View<SCALAR const**, XL, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                            \
                              Kokkos::MemoryTraits<Kokkos::Unmanaged | Kokkos::RandomAccess>>,                       \
                 Kokkos::View<SCALAR**, YL, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                                  \
                              Kokkos::MemoryTraits<Kokkos::Unmanaged>>,                                              \
                 false, true> {                                                                                      \
    using device_type = Kokkos::Device<Kokkos::Cuda, MEMSPACE>;                                                      \
    using Handle      = SPMVHandleImpl<Kokkos::Cuda, MEMSPACE, SCALAR, int, int>;                                    \
    using AMatrix = CrsMatrix<SCALAR const, int const, device_type, Kokkos::MemoryTraits<Kokkos::Unmanaged>, int const>; \
    using XVector = Kokkos::View<SCALAR const**, XL, device_type,                                                    \
                                 Kokkos::MemoryTraits<Kokkos::Unmanaged | Kokkos::RandomAccess>>;                    \
    using YVector = Kokkos::View<SCALAR**, YL, device_type, Kokkos::MemoryTraits<Kokkos::Unmanaged>>;                \
    using coefficient_type = typename YVector::non_const_value_type;                                                 \
    static void spmv_mv(const Kokkos::Cuda& exec, Handle* handle, const char mode[], const coefficient_type& alpha,  \
                        const AMatrix& A, const XVector& X, const coefficient_type& beta, const YVector& Y) {        \
      Kokkos::Profiling::pushRegion("KokkosSparse::spmv[TPL_B200," + Kokkos::ArithTraits<SCALAR>::name() + "]");     \
      b200sp_spmv_plan* plan = b200_plan_of(handle->tpl_rank2, exec, b200_spmv_algo(handle->get_algorithm()));       \
      constexpr int xrm = std::is_same<XL, Kokkos::LayoutRight>::value ? 1 : 0;                                      \
      constexpr int yrm = std::is_same<YL, Kokkos::LayoutRight>::value ? 1 : 0;                                      \
      const int64_t ldx = xrm ? (int64_t)X.stride(0) : (int64_t)X.stride(1);                                         \
      const int64_t ldy = yrm ? (int64_t)Y.stride(0) : (int64_t)Y.stride(1);                                         \
      KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200_call_spmm(                                                               \
          plan, (void*)exec.cuda_stream(), mode[0], A.numRows(), A.numCols(), (int64_t)A.nnz(), (int)X.extent(1),    \
          alpha, A.graph.row_map.data(), A.graph.entries.data(), A.values.data(), X.data(), ldx, xrm, beta,          \
          Y.data(), ldy, yrm));                                                                                      \
      Kokkos::Profiling::popRegion();                                                                                \
    }                                                                                                                \
  };

#define KOKKOSSPARSE_B200_SPMV_DECL_ALL(SCALAR, MEMSPACE)                                   \
  KOKKOSSPARSE_B200_SPMV_DECL(SCALAR, Kokkos::LayoutLeft, MEMSPACE)                         \
  KOKKOSSPARSE_B200_SPMV_DECL(SCALAR, Kokkos::LayoutRight, MEMSPACE)                        \
  KOKKOSSPARSE_B200_SPMV_MV_DECL(SCALAR, Kokkos::LayoutLeft, Kokkos::LayoutLeft, MEMSPACE)  \
  KOKKOSSPARSE_B200_SPMV_MV_DECL(SCALAR, Kokkos::LayoutRight, Kokkos::LayoutLeft, MEMSPACE) \
  KOKKOSSPARSE_B200_SPMV_MV_DECL(SCALAR, Kokkos::LayoutLeft, Kokkos::LayoutRight, MEMSPACE) \
  KOKKOSSPARSE_B200_SPMV_MV_DECL(SCALAR, Kokkos::LayoutRight, Kokkos::LayoutRight, MEMSPACE)

KOKKOSSPARSE_B200_SPMV_DECL_ALL(double, Kokkos::CudaSpace)
KOKKOSSPARSE_B200_SPMV_DECL_ALL(float, Kokkos::CudaSpace)
KOKKOSSPARSE_B200_SPMV_DECL_ALL(double, Kokkos::CudaUVMSpace)
KOKKOSSPARSE_B200_SPMV_DECL_ALL(float, Kokkos::CudaUVMSpace)

#undef KOKKOSSPARSE_B200_SPMV_DECL_ALL

// ---- half_t, rank 2 (guard as in the avail header): binary16 data, alpha and beta converted to float exactly ----------
#if defined(KOKKOS_HALF_T_IS_FLOAT) && !KOKKOS_HALF_T_IS_FLOAT
static_assert(sizeof(Kokkos::Experimental::half_t) == sizeof(uint16_t), "half_t is passed as binary16 bit patterns");
inline int b200_call_spmm(b200sp_spmv_plan* p, void* s, char mode, int m, int n, int64_t nnz, int k,
                          Kokkos::Experimental::half_t alpha, const int* rp, const int* ci, const Kokkos::Experimental::half_t* v,
                          const Kokkos::Experimental::half_t* X, int64_t ldx, int xrm, Kokkos::Experimental::half_t beta,
                          Kokkos::Experimental::half_t* Y, int64_t ldy, int yrm) {
  return b200sp_spmm_f16_i32(p, s, mode, m, n, nnz, k, static_cast<float>(alpha), rp, ci, reinterpret_cast<const uint16_t*>(v),
                             reinterpret_cast<const uint16_t*>(X), ldx, xrm, static_cast<float>(beta),
                             reinterpret_cast<uint16_t*>(Y), ldy, yrm);
}
#define KOKKOSSPARSE_B200_SPMV_MV_HALF_DECL_ALL(MEMSPACE)                                                                          \
  KOKKOSSPARSE_B200_SPMV_MV_DECL(Kokkos::Experimental::half_t, Kokkos::LayoutLeft, Kokkos::LayoutLeft, MEMSPACE)                   \
  KOKKOSSPARSE_B200_SPMV_MV_DECL(Kokkos::Experimental::half_t, Kokkos::LayoutRight, Kokkos::LayoutLeft, MEMSPACE)                  \
  KOKKOSSPARSE_B200_SPMV_MV_DECL(Kokkos::Experimental::half_t, Kokkos::LayoutLeft, Kokkos::LayoutRight, MEMSPACE)                  \
  KOKKOSSPARSE_B200_SPMV_MV_DECL(Kokkos::Experimental::half_t, Kokkos::LayoutRight, Kokkos::LayoutRight, MEMSPACE)
KOKKOSSPARSE_B200_SPMV_MV_HALF_DECL_ALL(Kokkos::CudaSpace)
KOKKOSSPARSE_B200_SPMV_MV_HALF_DECL_ALL(Kokkos::CudaUVMSpace)
#undef KOKKOSSPARSE_B200_SPMV_MV_HALF_DECL_ALL
#endif

// ---- 64-bit offsets -----------------------------------------------------------------------------------------------
inline b200sp_spmv64_plan* b200_plan64_of(TPL_SpMV_Data<Kokkos::Cuda>*& slot, const Kokkos::Cuda& exec, int algo) {
  B200_SpMV64_Data* sub;
  if (slot) {
    sub = dynamic_cast<B200_SpMV64_Data*>(slot);
    if (!sub) throw std::runtime_error("KokkosSparse::spmv: subhandle is not set up for b200sparse (64-bit offsets)");
    sub->set_exec_space(exec);
  } else {
    sub  = new B200_SpMV64_Data(exec, algo);
    slot = sub;
  }
  return sub->plan;
}
static_assert(sizeof(size_t) == sizeof(int64_t), "size_t offsets are read as int64_t (values below 2^63)");
inline int b200_call_spmv64(b200sp_spmv64_plan* p, void* s, char mode, int64_t m, int64_t n, int64_t nnz, double alpha,
                            const void* rp, const void* ci, int bits, const double* v, const double* x, double beta, double* y) {
  return b200sp_spmv_f64_i64(p, s, mode, m, n, nnz, alpha, (const int64_t*)rp, ci, bits, v, x, beta, y);
}
inline int b200_call_spmv64(b200sp_spmv64_plan* p, void* s, char mode, int64_t m, int64_t n, int64_t nnz, float alpha,
                            const void* rp, const void* ci, int bits, const float* v, const float* x, float beta, float* y) {
  return b200sp_spmv_f32_i64(p, s, mode, m, n, nnz, alpha, (const int64_t*)rp, ci, bits, v, x, beta, y);
}
inline int b200_call_spmm64(b200sp_spmv64_plan* p, void* s, char mode, int64_t m, int64_t n, int64_t nnz, int k, double alpha,
                            const void* rp, const void* ci, int bits, const double* v, const double* X, int64_t ldx, int xrm,
                            double beta, double* Y, int64_t ldy, int yrm) {
  return b200sp_spmm_f64_i64(p, s, mode, m, n, nnz, k, alpha, (const int64_t*)rp, ci, bits, v, X, ldx, xrm, beta, Y, ldy, yrm);
}
inline int b200_call_spmm64(b200sp_spmv64_plan* p, void* s, char mode, int64_t m, int64_t n, int64_t nnz, int k, float alpha,
                            const void* rp, const void* ci, int bits, const float* v, const float* X, int64_t ldx, int xrm,
                            float beta, float* Y, int64_t ldy, int yrm) {
  return b200sp_spmm_f32_i64(p, s, mode, m, n, nnz, k, alpha, (const int64_t*)rp, ci, bits, v, X, ldx, xrm, beta, Y, ldy, yrm);
}

#define KOKKOSSPARSE_B200_SPMV64_DECL(SCALAR, ORDINAL, OFFSET, LAYOUT, MEMSPACE)                                     \
  template <>                                                                                                        \
  struct SPMV<Kokkos::Cuda, SPMVHandleImpl<Kokkos::Cuda, MEMSPACE, SCALAR, OFFSET, ORDINAL>,                         \
              CrsMatrix<SCALAR const, ORDINAL const, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                         \
                        Kokkos::MemoryTraits<Kokkos::Unmanaged>, OFFSET const>,                                      \
              Kokkos::View<SCALAR const*, LAYOUT, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                            \
                           Kokkos::MemoryTraits<Kokkos::Unmanaged | Kokkos::RandomAccess>>,                          \
              Kokkos::View<SCALAR*, LAYOUT, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                                  \
                           Kokkos::MemoryTraits<Kokkos::Unmanaged>>,                                                 \
              true> {                                                                                                \
    using device_type = Kokkos::Device<Kokkos::Cuda, MEMSPACE>;                                                      \
    using Handle      = SPMVHandleImpl<Kokkos::Cuda, MEMSPACE, SCALAR, OFFSET, ORDINAL>;                             \
    using AMatrix =                                                                                                  \
        CrsMatrix<SCALAR const, ORDINAL const, device_type, Kokkos::MemoryTraits<Kokkos::Unmanaged>, OFFSET const>;  \
    using XVector = Kokkos::View<SCALAR const*, LAYOUT, device_type,                                                 \
                                 Kokkos::MemoryTraits<Kokkos::Unmanaged | Kokkos::RandomAccess>>;                    \
    using YVector = Kokkos::View<SCALAR*, LAYOUT, device_type, Kokkos::MemoryTraits<Kokkos::Unmanaged>>;             \
    using coefficient_type = typename YVector::non_const_value_type;                                                 \
    static void spmv(const Kokkos::Cuda& exec, Handle* handle, const char mode[], const coefficient_type& alpha,     \
                     const AMatrix& A, const XVector& x, const coefficient_type& beta, const YVector& y) {           \
      Kokkos::Profiling::pushRegion("KokkosSparse::spmv[TPL_B200," + Kokkos::ArithTraits<SCALAR>::name() + "]");     \
      b200sp_spmv64_plan* plan = b200_plan64_of(handle->tpl_rank1, exec, b200_spmv_algo(handle->get_algorithm()));   \
      KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200_call_spmv64(                                                             \
          plan, (void*)exec.cuda_stream(), mode[0], (int64_t)A.numRows(), (int64_t)A.numCols(), (int64_t)A.nnz(),    \
          alpha, A.graph.row_map.data(), A.graph.entries.data(), (int)(8 * sizeof(ORDINAL)), A.values.data(),        \
          x.data(), beta, y.data()));                                                                                \
      Kokkos::Profiling::popRegion();                                                                                \
    }                                                                                                                \
  };

#define KOKKOSSPARSE_B200_SPMV64_MV_DECL(SCALAR, ORDINAL, OFFSET, XL, YL, MEMSPACE)                                  \
  template <>                                                                                                        \
  struct SPMV_MV<Kokkos::Cuda, SPMVHandleImpl<Kokkos::Cuda, MEMSPACE, SCALAR, OFFSET, ORDINAL>,                      \
                 CrsMatrix<SCALAR const, ORDINAL const, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                      \
                           Kokkos::MemoryTraits<Kokkos::Unmanaged>, OFFSET const>,                                   \
                 Kokkos::View<SCALAR const**, XL, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                            \
                              Kokkos::MemoryTraits<Kokkos::Unmanaged | Kokkos::RandomAccess>>,                       \
                 Kokkos::View<SCALAR**, YL, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                                  \
                              Kokkos::MemoryTraits<Kokkos::Unmanaged>>,                                              \
                 false, true> {                                                                                      \
    using device_type = Kokkos::Device<Kokkos::Cuda, MEMSPACE>;                                                      \
    using Handle      = SPMVHandleImpl<Kokkos::Cuda, MEMSPACE, SCALAR, OFFSET, ORDINAL>;                             \
    using AMatrix =                                                                                                  \
        CrsMatrix<SCALAR const, ORDINAL const, device_type, Kokkos::MemoryTraits<Kokkos::Unmanaged>, OFFSET const>;  \
    using XVector = Kokkos::View<SCALAR const**, XL, device_type,                                                    \
                                 Kokkos::MemoryTraits<Kokkos::Unmanaged | Kokkos::RandomAccess>>;                    \
    using YVector = Kokkos::View<SCALAR**, YL, device_type, Kokkos::MemoryTraits<Kokkos::Unmanaged>>;                \
    using coefficient_type = typename YVector::non_const_value_type;                                                 \
    static void spmv_mv(const Kokkos::Cuda& exec, Handle* handle, const char mode[], const coefficient_type& alpha,  \
                        const AMatrix& A, const XVector& X, const coefficient_type& beta, const YVector& Y) {        \
      Kokkos::Profiling::pushRegion("KokkosSparse::spmv[TPL_B200," + Kokkos::ArithTraits<SCALAR>::name() + "]");     \
      b200sp_spmv64_plan* plan = b200_plan64_of(handle->tpl_rank2, exec, b200_spmv_algo(handle->get_algorithm()));   \
      constexpr int xrm = std::is_same<XL, Kokkos::LayoutRight>::value ? 1 : 0;                                      \
      constexpr int yrm = std::is_same<YL, Kokkos::LayoutRight>::value ? 1 : 0;                                      \
      const int64_t ldx = xrm ? (int64_t)X.stride(0) : (int64_t)X.stride(1);                                         \
      const int64_t ldy = yrm ? (int64_t)Y.stride(0) : (int64_t)Y.stride(1);                                         \
      KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200_call_spmm64(                                                             \
          plan, (void*)exec.cuda_stream(), mode[0], (int64_t)A.numRows(), (int64_t)A.numCols(), (int64_t)A.nnz(),    \
          (int)X.extent(1), alpha, A.graph.row_map.data(), A.graph.entries.data(), (int)(8 * sizeof(ORDINAL)),       \
          A.values.data(), X.data(), ldx, xrm, beta, Y.data(), ldy, yrm));                                           \
      Kokkos::Profiling::popRegion();                                                                                \
    }                                                                                                                \
  };

#define KOKKOSSPARSE_B200_SPMV64_DECL_ALL(SCALAR, ORDINAL, OFFSET, MEMSPACE)                                   \
  KOKKOSSPARSE_B200_SPMV64_DECL(SCALAR, ORDINAL, OFFSET, Kokkos::LayoutLeft, MEMSPACE)                         \
  KOKKOSSPARSE_B200_SPMV64_DECL(SCALAR, ORDINAL, OFFSET, Kokkos::LayoutRight, MEMSPACE)                        \
  KOKKOSSPARSE_B200_SPMV64_MV_DECL(SCALAR, ORDINAL, OFFSET, Kokkos::LayoutLeft, Kokkos::LayoutLeft, MEMSPACE)  \
  KOKKOSSPARSE_B200_SPMV64_MV_DECL(SCALAR, ORDINAL, OFFSET, Kokkos::LayoutRight, Kokkos::LayoutRight, MEMSPACE)

KOKKOSSPARSE_B200_SPMV64_DECL_ALL(double, int64_t, size_t, Kokkos::CudaSpace)
KOKKOSSPARSE_B200_SPMV64_DECL_ALL(float, int64_t, size_t, Kokkos::CudaSpace)
KOKKOSSPARSE_B200_SPMV64_DECL_ALL(double, int, size_t, Kokkos::CudaSpace)
KOKKOSSPARSE_B200_SPMV64_DECL_ALL(float, int, size_t, Kokkos::CudaSpace)
KOKKOSSPARSE_B200_SPMV64_DECL_ALL(double, int64_t, size_t, Kokkos::CudaUVMSpace)
KOKKOSSPARSE_B200_SPMV64_DECL_ALL(float, int64_t, size_t, Kokkos::CudaUVMSpace)
KOKKOSSPARSE_B200_SPMV64_DECL_ALL(double, int, size_t, Kokkos::CudaUVMSpace)
KOKKOSSPARSE_B200_SPMV64_DECL_ALL(float, int, size_t, Kokkos::CudaUVMSpace)
#undef KOKKOSSPARSE_B200_SPMV64_DECL_ALL
}  // namespace Impl
}  // namespace KokkosSparse
#endif
#endif
