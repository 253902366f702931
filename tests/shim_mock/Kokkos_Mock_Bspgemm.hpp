// Kokkos_Mock_Bspgemm.hpp -- what the block SpGEMM shim needs beyond Kokkos_Mock.hpp (TEST INFRASTRUCTURE ONLY):
//   bspgemm_numeric_tpl_spec_avail   false by default (sparse/impl/KokkosSparse_bspgemm_numeric_spec.hpp:103-108)
//   BSPGEMM_NUMERIC                  the unification layer's declaration with its defaulted tpl argument (:113-127), and a
//                                    stand-in for the native struct (tpl = false, :132-191) that only counts its calls
#pragma once
#include "Kokkos_Mock.hpp"

namespace KokkosSparse {
namespace Impl {
template <class KH, class a_r, class a_e, class a_v, class b_r, class b_e, class b_v, class c_r, class c_e, class c_v>
struct bspgemm_numeric_tpl_spec_avail {
  enum : bool { value = false };
};
template <class KH, class a_r, class a_e, class a_v, class b_r, class b_e, class b_v, class c_r, class c_e, class c_v,
          bool tpl = bspgemm_numeric_tpl_spec_avail<KH, a_r, a_e, a_v, b_r, b_e, b_v, c_r, c_e, c_v>::value, bool eti = true>
struct BSPGEMM_NUMERIC;

inline int& native_bspgemm_calls() {
  static int n = 0;
  return n;
}
template <class KH, class a_r, class a_e, class a_v, class b_r, class b_e, class b_v, class c_r, class c_e, class c_v, bool eti>
struct BSPGEMM_NUMERIC<KH, a_r, a_e, a_v, b_r, b_e, b_v, c_r, c_e, c_v, false, eti> {
  template <class... Args>
  static void bspgemm_numeric(Args&&...) {
    ++native_bspgemm_calls();
  }
};
}  // namespace Impl
}  // namespace KokkosSparse
