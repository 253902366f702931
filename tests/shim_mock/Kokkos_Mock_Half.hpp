// Kokkos_Mock_Half.hpp -- Kokkos::Experimental::half_t for the View mock (Kokkos_Mock.hpp), where it is a real 16-bit type:
// core/src/Kokkos_Half_FloatingPointWrapper.hpp defines KOKKOS_HALF_T_IS_FLOAT to 0 then.  2 bytes wrapping __half, float
// conversions both ways, and its ArithTraits name.  Included after Kokkos_Mock.hpp by the translation units that exercise the
// half_t specialisations of the shim (shim_half_driver.cpp); the other drivers never see it.
// TEST INFRASTRUCTURE ONLY.
#pragma once
#include "Kokkos_Mock.hpp"

#if defined(KOKKOS_HALF_T_IS_FLOAT) && !KOKKOS_HALF_T_IS_FLOAT
#include <cuda_fp16.h>
namespace Kokkos {
namespace Experimental {
struct half_t {
  __half val;
  half_t() = default;
  half_t(float f) : val(__float2half_rn(f)) {}
  operator float() const { return __half2float(val); }
};
}  // namespace Experimental
template <>
struct ArithTraits<Experimental::half_t> {
  static std::string name() { return "half"; }
};
}  // namespace Kokkos
#endif
