// Marks Kokkos::Cuda / int / int block SpGEMM numeric (double, float; CudaSpace, CudaUVMSpace) as served by libb200sparse:
// bspgemm_numeric_tpl_spec_avail, the switch the reference keeps "for future use" and false for every type
// (sparse/impl/KokkosSparse_bspgemm_numeric_spec.hpp:103-108).  Its include of the avail header is commented out there
// (:97); INTEGRATION.md shows the line to add.  Block symbolic is the point SPGEMM_SYMBOLIC slot
// (KokkosSparse_spgemm_b200_tpl_spec_avail.hpp).
#ifndef KOKKOSSPARSE_BSPGEMM_B200_TPL_SPEC_AVAIL_HPP_
#define KOKKOSSPARSE_BSPGEMM_B200_TPL_SPEC_AVAIL_HPP_
#ifdef KOKKOSKERNELS_ENABLE_TPL_B200SPARSE

#include "KokkosSparse_spgemm_b200_tpl_spec_avail.hpp"  // KOKKOSSPARSE_B200_IV / _KH

namespace KokkosSparse {
namespace Impl {

#define KOKKOSSPARSE_B200_BSPGEMM_AVAIL(SCALAR, MEMSPACE)                                                                    \
  template <>                                                                                                               \
  struct bspgemm_numeric_tpl_spec_avail<                                                                                    \
      KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE),                                    \
      KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE),                              \
      KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE),                                 \
      KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE),                              \
      KOKKOSSPARSE_B200_IV(int, MEMSPACE), KOKKOSSPARSE_B200_IV(SCALAR, MEMSPACE)> {                                        \
    enum : bool { value = true };                                                                                           \
  };

KOKKOSSPARSE_B200_BSPGEMM_AVAIL(double, Kokkos::CudaSpace)
KOKKOSSPARSE_B200_BSPGEMM_AVAIL(float, Kokkos::CudaSpace)
KOKKOSSPARSE_B200_BSPGEMM_AVAIL(double, Kokkos::CudaUVMSpace)
KOKKOSSPARSE_B200_BSPGEMM_AVAIL(float, Kokkos::CudaUVMSpace)

}  // namespace Impl
}  // namespace KokkosSparse
#endif
#endif
