// KokkosSparse_b200_utils.hpp -- glue between Kokkos Kernels' TPL layer and libb200sparse.
//
// Install: copy this directory into kokkos-kernels/sparse/tpls/, add
// KOKKOSKERNELS_ENABLE_TPL_B200SPARSE to KokkosKernels_config.h.in, include the
// *_avail.hpp / *_decl.hpp files next to the cuSPARSE ones (INTEGRATION.md lists
// the exact lines), link -lb200sparse.  The TPL_B200 specialisations occupy the slot
// of the cuSPARSE ones (same template arguments), so build with
// KokkosKernels_ENABLE_TPL_CUSPARSE=OFF.
#ifndef KOKKOSSPARSE_B200_UTILS_HPP_
#define KOKKOSSPARSE_B200_UTILS_HPP_
#ifdef KOKKOSKERNELS_ENABLE_TPL_B200SPARSE

#include <sstream>
#include <stdexcept>
#include "b200sparse.h"

namespace KokkosSparse {
namespace Impl {

// status -> exception, the analogue of KOKKOSSPARSE_IMPL_CUSPARSE_SAFE_CALL
// (sparse/src/KokkosSparse_Utils_cusparse.hpp:28-67)
inline void b200sparse_internal_safe_call(int status, const char* name, const char* file, int line) {
  if (status == B200SP_OK) return;
  std::ostringstream out;
  out << name << " failed with status " << status << " (" << b200sp_last_error_string() << ") at " << file << ":"
      << line;
  if (status == B200SP_ERR_STATE) throw std::invalid_argument(out.str());
  throw std::runtime_error(out.str());
}
#define KOKKOSSPARSE_IMPL_B200_SAFE_CALL(call) \
  KokkosSparse::Impl::b200sparse_internal_safe_call(call, #call, __FILE__, __LINE__)

// SPMVAlgorithm -> b200sp_spmv_algo.  Only DEFAULT / FAST_SETUP / MERGE_PATH reach a TPL;
// the NATIVE algorithms are routed around it by KokkosSparse::spmv (KokkosSparse_spmv.hpp:222,264).
inline int b200_spmv_algo(SPMVAlgorithm a) {
  switch (a) {
    case SPMV_FAST_SETUP: return B200SP_SPMV_FAST_SETUP;
    case SPMV_MERGE_PATH: return B200SP_SPMV_MERGE_PATH;
    default: return B200SP_SPMV_DEFAULT;
  }
}

// Per-matrix state hung off SPMVHandleImpl::tpl_rank1 / tpl_rank2, the way
// CuSparse10_SpMV_Data is (sparse/src/KokkosSparse_spmv_handle.hpp:112-135).
struct B200_SpMV_Data : public TPL_SpMV_Data<Kokkos::Cuda> {
  B200_SpMV_Data(const Kokkos::Cuda& exec_, int algo) : TPL_SpMV_Data(exec_) {
    KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200sp_spmv_plan_create(&plan, algo));
  }
  ~B200_SpMV_Data() {
    // stream-ordered frees on the last stream used: safe without a user fence
    b200sp_spmv_plan_destroy(plan, (void*)exec.cuda_stream());
  }
  b200sp_spmv_plan* plan = nullptr;
};

// Same for matrices with 64-bit offsets (the (int64_t, size_t) instantiation cuSPARSE serves,
// sparse/tpls/KokkosSparse_spmv_tpl_spec_decl.hpp:246-257): the plan owns the 32-bit row windows.
struct B200_SpMV64_Data : public TPL_SpMV_Data<Kokkos::Cuda> {
  B200_SpMV64_Data(const Kokkos::Cuda& exec_, int algo) : TPL_SpMV_Data(exec_) {
    KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200sp_spmv64_plan_create(&plan, algo));
  }
  ~B200_SpMV64_Data() { b200sp_spmv64_plan_destroy(plan, (void*)exec.cuda_stream()); }
  b200sp_spmv64_plan* plan = nullptr;
};

}  // namespace Impl
}  // namespace KokkosSparse
#endif
#endif
