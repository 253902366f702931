// Marks Kokkos::Cuda / int / int and int / size_t SpGEMM symbolic + numeric as served by libb200sparse -- the
// pattern of sparse/tpls/KokkosSparse_spgemm_symbolic_tpl_spec_avail.hpp:29-69 and
// ..._numeric_tpl_spec_avail.hpp; include from those files.
#ifndef KOKKOSSPARSE_SPGEMM_B200_TPL_SPEC_AVAIL_HPP_
#define KOKKOSSPARSE_SPGEMM_B200_TPL_SPEC_AVAIL_HPP_
#ifdef KOKKOSKERNELS_ENABLE_TPL_B200SPARSE

namespace KokkosSparse {
namespace Impl {

#define KOKKOSSPARSE_B200_IV(T, MEMSPACE) \
  Kokkos::View<T*, KokkosKernels::default_layout, Kokkos::Device<Kokkos::Cuda, MEMSPACE>, Kokkos::MemoryTraits<Kokkos::Unmanaged>>
#define KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE) \
  KokkosKernels::Experimental::KokkosKernelsHandle<const int, const int, const SCALAR, Kokkos::Cuda, MEMSPACE, MEMSPACE>

#define KOKKOSSPARSE_B200_SPGEMM_AVAIL(SCALAR, MEMSPACE)                                                               \
  template <>                                                                                                          \
  struct spgemm_symbolic_tpl_spec_avail<KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE), \
                                        KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE), \
                                        KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(int, MEMSPACE)> { \
    enum : bool { value = true };                                                                                      \
  };                                                                                                                   \
  template <>                                                                                                          \
  struct spgemm_numeric_tpl_spec_avail<                                                                                \
      KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE),                               \
      KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE),                         \
      KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE),                            \
      KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE),                         \
      KOKKOSSPARSE_B200_IV(int, MEMSPACE), KOKKOSSPARSE_B200_IV(SCALAR, MEMSPACE)> {                                   \
    enum : bool { value = true };                                                                                      \
  };

KOKKOSSPARSE_B200_SPGEMM_AVAIL(double, Kokkos::CudaSpace)
KOKKOSSPARSE_B200_SPGEMM_AVAIL(float, Kokkos::CudaSpace)
KOKKOSSPARSE_B200_SPGEMM_AVAIL(double, Kokkos::CudaUVMSpace)
KOKKOSSPARSE_B200_SPGEMM_AVAIL(float, Kokkos::CudaUVMSpace)

// 64-bit offsets with 32-bit ordinals, Kokkos' (int, size_t) -- the default offsets of a Trilinos build
// (cmake/kokkoskernels_eti_offsets.cmake:1-11), which the cuSPARSE slot cannot take
// (sparse/tpls/KokkosSparse_spgemm_numeric_tpl_spec_avail.hpp:38-41): libb200sparse's _i64 entries
#define KOKKOSSPARSE_B200_KH64(SCALAR, MEMSPACE) \
  KokkosKernels::Experimental::KokkosKernelsHandle<const size_t, const int, const SCALAR, Kokkos::Cuda, MEMSPACE, MEMSPACE>

#define KOKKOSSPARSE_B200_SPGEMM64_AVAIL(SCALAR, MEMSPACE)                                                             \
  template <>                                                                                                          \
  struct spgemm_symbolic_tpl_spec_avail<                                                                               \
      KOKKOSSPARSE_B200_KH64(SCALAR, MEMSPACE), KOKKOSSPARSE_B200_IV(const size_t, MEMSPACE),                          \
      KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(const size_t, MEMSPACE),                         \
      KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(size_t, MEMSPACE)> {                             \
    enum : bool { value = true };                                                                                      \
  };                                                                                                                   \
  template <>                                                                                                          \
  struct spgemm_numeric_tpl_spec_avail<                                                                                \
      KOKKOSSPARSE_B200_KH64(SCALAR, MEMSPACE), KOKKOSSPARSE_B200_IV(const size_t, MEMSPACE),                          \
      KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE),                         \
      KOKKOSSPARSE_B200_IV(const size_t, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE),                         \
      KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE), KOKKOSSPARSE_B200_IV(const size_t, MEMSPACE),                      \
      KOKKOSSPARSE_B200_IV(int, MEMSPACE), KOKKOSSPARSE_B200_IV(SCALAR, MEMSPACE)> {                                   \
    enum : bool { value = true };                                                                                      \
  };

KOKKOSSPARSE_B200_SPGEMM64_AVAIL(double, Kokkos::CudaSpace)
KOKKOSSPARSE_B200_SPGEMM64_AVAIL(float, Kokkos::CudaSpace)
KOKKOSSPARSE_B200_SPGEMM64_AVAIL(double, Kokkos::CudaUVMSpace)
KOKKOSSPARSE_B200_SPGEMM64_AVAIL(float, Kokkos::CudaUVMSpace)

}  // namespace Impl
}  // namespace KokkosSparse
#endif
#endif
