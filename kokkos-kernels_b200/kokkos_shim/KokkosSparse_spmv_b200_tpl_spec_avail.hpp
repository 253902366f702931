// Marks the (Kokkos::Cuda, int, int, {double,float}) SpMV instantiations as served by
// libb200sparse -- the pattern of sparse/tpls/KokkosSparse_spmv_tpl_spec_avail.hpp:38-71;
// include it from that file inside namespace KokkosSparse::Impl, after the generic
// spmv_tpl_spec_avail / spmv_mv_tpl_spec_avail declarations.
#ifndef KOKKOSSPARSE_SPMV_B200_TPL_SPEC_AVAIL_HPP_
#define KOKKOSSPARSE_SPMV_B200_TPL_SPEC_AVAIL_HPP_
#ifdef KOKKOSKERNELS_ENABLE_TPL_B200SPARSE

namespace KokkosSparse {
namespace Impl {

#define KOKKOSSPARSE_B200_SPMV_AVAIL(SCALAR, LAYOUT, MEMSPACE)                                                      \
  template <>                                                                                                       \
  struct spmv_tpl_spec_avail<                                                                                       \
      Kokkos::Cuda, SPMVHandleImpl<Kokkos::Cuda, MEMSPACE, SCALAR, int, int>,                                       \
      CrsMatrix<const SCALAR, const int, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                                    \
                Kokkos::MemoryTraits<Kokkos::Unmanaged>, const int>,                                                \
      Kokkos::View<const SCALAR*, LAYOUT, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                                   \
                   Kokkos::MemoryTraits<Kokkos::Unmanaged | Kokkos::RandomAccess>>,                                 \
      Kokkos::View<SCALAR*, LAYOUT, Kokkos::Device<Kokkos::Cuda, MEMSPACE>, Kokkos::MemoryTraits<Kokkos::Unmanaged>>> { \
    enum : bool { value = true };                                                                                   \
  };

// rank-2: X may be LayoutLeft or LayoutRight, Y likewise (libb200sparse takes any mix)
#define KOKKOSSPARSE_B200_SPMV_MV_AVAIL(SCALAR, XL, YL, MEMSPACE)                                                   \
  template <>                                                                                                       \
  struct spmv_mv_tpl_spec_avail<                                                                                    \
      Kokkos::Cuda, SPMVHandleImpl<Kokkos::Cuda, MEMSPACE, SCALAR, int, int>,                                       \
      CrsMatrix<const SCALAR, const int, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                                    \
                Kokkos::MemoryTraits<Kokkos::Unmanaged>, const int>,                                                \
      Kokkos::View<const SCALAR**, XL, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                                      \
                   Kokkos::MemoryTraits<Kokkos::Unmanaged | Kokkos::RandomAccess>>,                                 \
      Kokkos::View<SCALAR**, YL, Kokkos::Device<Kokkos::Cuda, MEMSPACE>, Kokkos::MemoryTraits<Kokkos::Unmanaged>>> { \
    enum : bool { value = true };                                                                                   \
  };

#define KOKKOSSPARSE_B200_SPMV_AVAIL_ALL(SCALAR, MEMSPACE)                                   \
  KOKKOSSPARSE_B200_SPMV_AVAIL(SCALAR, Kokkos::LayoutLeft, MEMSPACE)                         \
  KOKKOSSPARSE_B200_SPMV_AVAIL(SCALAR, Kokkos::LayoutRight, MEMSPACE)                        \
  KOKKOSSPARSE_B200_SPMV_MV_AVAIL(SCALAR, Kokkos::LayoutLeft, Kokkos::LayoutLeft, MEMSPACE)  \
  KOKKOSSPARSE_B200_SPMV_MV_AVAIL(SCALAR, Kokkos::LayoutRight, Kokkos::LayoutLeft, MEMSPACE) \
  KOKKOSSPARSE_B200_SPMV_MV_AVAIL(SCALAR, Kokkos::LayoutLeft, Kokkos::LayoutRight, MEMSPACE) \
  KOKKOSSPARSE_B200_SPMV_MV_AVAIL(SCALAR, Kokkos::LayoutRight, Kokkos::LayoutRight, MEMSPACE)

KOKKOSSPARSE_B200_SPMV_AVAIL_ALL(double, Kokkos::CudaSpace)
KOKKOSSPARSE_B200_SPMV_AVAIL_ALL(float, Kokkos::CudaSpace)
KOKKOSSPARSE_B200_SPMV_AVAIL_ALL(double, Kokkos::CudaUVMSpace)
KOKKOSSPARSE_B200_SPMV_AVAIL_ALL(float, Kokkos::CudaUVMSpace)

#undef KOKKOSSPARSE_B200_SPMV_AVAIL_ALL

// half_t, rank 2 only, where half_t is a real 16-bit type (the guard of the reference's cuSPARSE slot,
// sparse/tpls/KokkosSparse_spmv_mv_tpl_spec_avail.hpp:93-104); fp32 products and sums, every layout pair
#if defined(KOKKOS_HALF_T_IS_FLOAT) && !KOKKOS_HALF_T_IS_FLOAT
#define KOKKOSSPARSE_B200_SPMV_MV_HALF_AVAIL_ALL(MEMSPACE)                                                                          \
  KOKKOSSPARSE_B200_SPMV_MV_AVAIL(Kokkos::Experimental::half_t, Kokkos::LayoutLeft, Kokkos::LayoutLeft, MEMSPACE)                   \
  KOKKOSSPARSE_B200_SPMV_MV_AVAIL(Kokkos::Experimental::half_t, Kokkos::LayoutRight, Kokkos::LayoutLeft, MEMSPACE)                  \
  KOKKOSSPARSE_B200_SPMV_MV_AVAIL(Kokkos::Experimental::half_t, Kokkos::LayoutLeft, Kokkos::LayoutRight, MEMSPACE)                  \
  KOKKOSSPARSE_B200_SPMV_MV_AVAIL(Kokkos::Experimental::half_t, Kokkos::LayoutRight, Kokkos::LayoutRight, MEMSPACE)
KOKKOSSPARSE_B200_SPMV_MV_HALF_AVAIL_ALL(Kokkos::CudaSpace)
KOKKOSSPARSE_B200_SPMV_MV_HALF_AVAIL_ALL(Kokkos::CudaUVMSpace)
#undef KOKKOSSPARSE_B200_SPMV_MV_HALF_AVAIL_ALL
#endif

// 64-bit offsets: (int64_t, size_t) -- the instantiation of the cuSPARSE slot (..._tpl_spec_avail.hpp:85-102) -- and
// (int, size_t), which cuSPARSE does not take (:86); rank 1 and rank 2
#define KOKKOSSPARSE_B200_SPMV64_AVAIL(SCALAR, ORDINAL, OFFSET, LAYOUT, MEMSPACE)                                   \
  template <>                                                                                                       \
  struct spmv_tpl_spec_avail<                                                                                       \
      Kokkos::Cuda, SPMVHandleImpl<Kokkos::Cuda, MEMSPACE, SCALAR, OFFSET, ORDINAL>,                                \
      CrsMatrix<const SCALAR, const ORDINAL, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                                \
                Kokkos::MemoryTraits<Kokkos::Unmanaged>, const OFFSET>,                                             \
      Kokkos::View<const SCALAR*, LAYOUT, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                                   \
                   Kokkos::MemoryTraits<Kokkos::Unmanaged | Kokkos::RandomAccess>>,                                 \
      Kokkos::View<SCALAR*, LAYOUT, Kokkos::Device<Kokkos::Cuda, MEMSPACE>, Kokkos::MemoryTraits<Kokkos::Unmanaged>>> { \
    enum : bool { value = true };                                                                                   \
  };
#define KOKKOSSPARSE_B200_SPMV64_MV_AVAIL(SCALAR, ORDINAL, OFFSET, XL, YL, MEMSPACE)                                \
  template <>                                                                                                       \
  struct spmv_mv_tpl_spec_avail<                                                                                    \
      Kokkos::Cuda, SPMVHandleImpl<Kokkos::Cuda, MEMSPACE, SCALAR, OFFSET, ORDINAL>,                                \
      CrsMatrix<const SCALAR, const ORDINAL, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                                \
                Kokkos::MemoryTraits<Kokkos::Unmanaged>, const OFFSET>,                                             \
      Kokkos::View<const SCALAR**, XL, Kokkos::Device<Kokkos::Cuda, MEMSPACE>,                                      \
                   Kokkos::MemoryTraits<Kokkos::Unmanaged | Kokkos::RandomAccess>>,                                 \
      Kokkos::View<SCALAR**, YL, Kokkos::Device<Kokkos::Cuda, MEMSPACE>, Kokkos::MemoryTraits<Kokkos::Unmanaged>>> { \
    enum : bool { value = true };                                                                                   \
  };
#define KOKKOSSPARSE_B200_SPMV64_AVAIL_ALL(SCALAR, ORDINAL, OFFSET, MEMSPACE)                                   \
  KOKKOSSPARSE_B200_SPMV64_AVAIL(SCALAR, ORDINAL, OFFSET, Kokkos::LayoutLeft, MEMSPACE)                         \
  KOKKOSSPARSE_B200_SPMV64_AVAIL(SCALAR, ORDINAL, OFFSET, Kokkos::LayoutRight, MEMSPACE)                        \
  KOKKOSSPARSE_B200_SPMV64_MV_AVAIL(SCALAR, ORDINAL, OFFSET, Kokkos::LayoutLeft, Kokkos::LayoutLeft, MEMSPACE)  \
  KOKKOSSPARSE_B200_SPMV64_MV_AVAIL(SCALAR, ORDINAL, OFFSET, Kokkos::LayoutRight, Kokkos::LayoutRight, MEMSPACE)

KOKKOSSPARSE_B200_SPMV64_AVAIL_ALL(double, int64_t, size_t, Kokkos::CudaSpace)
KOKKOSSPARSE_B200_SPMV64_AVAIL_ALL(float, int64_t, size_t, Kokkos::CudaSpace)
KOKKOSSPARSE_B200_SPMV64_AVAIL_ALL(double, int, size_t, Kokkos::CudaSpace)
KOKKOSSPARSE_B200_SPMV64_AVAIL_ALL(float, int, size_t, Kokkos::CudaSpace)
KOKKOSSPARSE_B200_SPMV64_AVAIL_ALL(double, int64_t, size_t, Kokkos::CudaUVMSpace)
KOKKOSSPARSE_B200_SPMV64_AVAIL_ALL(float, int64_t, size_t, Kokkos::CudaUVMSpace)
KOKKOSSPARSE_B200_SPMV64_AVAIL_ALL(double, int, size_t, Kokkos::CudaUVMSpace)
KOKKOSSPARSE_B200_SPMV64_AVAIL_ALL(float, int, size_t, Kokkos::CudaUVMSpace)
#undef KOKKOSSPARSE_B200_SPMV64_AVAIL_ALL
}  // namespace Impl
}  // namespace KokkosSparse
#endif
#endif
