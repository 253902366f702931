// Stand-in for the reference's batched/KokkosBatched_Util.hpp: the algorithm tags the serial GEMM is specialised on,
// and a declaration of the blocked inner kernel its Blocked variant names (the block SpGEMM uses Unblocked only; the
// reference's InnerGemmFixC serial implementation is skipped through its include guard).  TEST INFRASTRUCTURE ONLY.
#pragma once
#include "KokkosKernels_helpers.hpp"

namespace KokkosBatched {
namespace Algo {
namespace Gemm {
struct Unblocked {};
struct Blocked {
  static constexpr int mb() { return 4; }
};
}  // namespace Gemm
}  // namespace Algo

template <int MB, int NB>
struct InnerGemmFixC {
  InnerGemmFixC(int, int, int, int, int, int) {}
  template <class OpA, class OpB, class S, class V>
  int serial_invoke(OpA, OpB, const S, const V*, const V*, int, int, int, V*) {
    return -1;  // never called
  }
};
}  // namespace KokkosBatched
