// Full specialisations of SPGEMM_SYMBOLIC / SPGEMM_NUMERIC for Kokkos::Cuda that forward to
// libb200sparse -- the slot of spgemm_symbolic_cusparse / spgemm_numeric_cusparse
// (sparse/tpls/KokkosSparse_spgemm_symbolic_tpl_spec_decl.hpp:316-363,
//  sparse/tpls/KokkosSparse_spgemm_numeric_tpl_spec_decl.hpp:195-256).  Generic declarations:
// sparse/impl/KokkosSparse_spgemm_symbolic_spec.hpp:72-83, ..._numeric_spec.hpp:84-98.
//
// Needs one member on SPGEMMHandle (sparse/src/KokkosSparse_spgemm_handle.hpp, next to
// cusparse_spgemm_handle at :328): `b200sp_spgemm_plan* b200_spgemm_plan = nullptr;` released in
// the destructor with b200sp_spgemm_plan_destroy (INTEGRATION.md shows the patch).
#ifndef KOKKOSSPARSE_SPGEMM_B200_TPL_SPEC_DECL_HPP_
#define KOKKOSSPARSE_SPGEMM_B200_TPL_SPEC_DECL_HPP_
#ifdef KOKKOSKERNELS_ENABLE_TPL_B200SPARSE

#include "KokkosSparse_b200_utils.hpp"

namespace KokkosSparse {
namespace Impl {

// (int, size_t) handles pass their size_t row maps to the _i64 entries as int64_t
static_assert(sizeof(size_t) == sizeof(int64_t), "the 64-bit SpGEMM entries read size_t row maps as int64_t");

inline int b200_call_symbolic(b200sp_spgemm_plan* p, void* s, int m, int n, int k, const int* rA, const int* cA, const int* rB,
                              const int* cB, int* rC, int64_t* c_nnz, int* c_max) {
  return b200sp_spgemm_symbolic_i32(p, s, m, n, k, rA, cA, rB, cB, rC, c_nnz, c_max);
}
inline int b200_call_symbolic(b200sp_spgemm_plan* p, void* s, int m, int n, int k, const size_t* rA, const int* cA,
                              const size_t* rB, const int* cB, size_t* rC, int64_t* c_nnz, int* c_max) {
  return b200sp_spgemm_symbolic_i64(p, s, m, n, k, (const int64_t*)rA, cA, (const int64_t*)rB, cB, (int64_t*)rC, c_nnz, c_max);
}

inline int b200_call_numeric(b200sp_spgemm_plan* p, void* s, int m, int n, int k, const int* rA, const int* cA,
                             const double* vA, const int* rB, const int* cB, const double* vB, const int* rC, int* cC,
                             double* vC) {
  return b200sp_spgemm_numeric_f64_i32(p, s, m, n, k, rA, cA, vA, rB, cB, vB, rC, cC, vC);
}
inline int b200_call_numeric(b200sp_spgemm_plan* p, void* s, int m, int n, int k, const int* rA, const int* cA,
                             const float* vA, const int* rB, const int* cB, const float* vB, const int* rC, int* cC,
                             float* vC) {
  return b200sp_spgemm_numeric_f32_i32(p, s, m, n, k, rA, cA, vA, rB, cB, vB, rC, cC, vC);
}
inline int b200_call_numeric(b200sp_spgemm_plan* p, void* s, int m, int n, int k, const size_t* rA, const int* cA,
                             const double* vA, const size_t* rB, const int* cB, const double* vB, const size_t* rC, int* cC,
                             double* vC) {
  return b200sp_spgemm_numeric_f64_i64(p, s, m, n, k, (const int64_t*)rA, cA, vA, (const int64_t*)rB, cB, vB, (const int64_t*)rC,
                                       cC, vC);
}
inline int b200_call_numeric(b200sp_spgemm_plan* p, void* s, int m, int n, int k, const size_t* rA, const int* cA,
                             const float* vA, const size_t* rB, const int* cB, const float* vB, const size_t* rC, int* cC,
                             float* vC) {
  return b200sp_spgemm_numeric_f32_i64(p, s, m, n, k, (const int64_t*)rA, cA, vA, (const int64_t*)rB, cB, vB, (const int64_t*)rC,
                                       cC, vC);
}

// CSV: the row maps (const int or const size_t), CIV: the entries (const int), SV: row_mapC
template <class SpgemmHandle, class CSV, class CIV, class SV>
void spgemm_symbolic_b200(SpgemmHandle* sh, int m, int n, int k, const CSV& rowmapA, const CIV& entriesA,
                          const CSV& rowmapB, const CIV& entriesB, const SV& rowmapC, bool /*computeRowptrs*/) {
  // second call on the same handle is a no-op (symbolic_spec.hpp:99; cuSPARSE leg :69-77)
  if (sh->is_symbolic_called() && sh->are_rowptrs_computed()) return;
  if (!sh->b200_spgemm_plan) KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200sp_spgemm_plan_create(&sh->b200_spgemm_plan));
  int64_t c_nnz = 0;
  int c_max     = 0;
  void* stream  = (void*)Kokkos::Cuda().cuda_stream();  // SpGEMM has no exec-instance overload: default instance
  KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200_call_symbolic(sh->b200_spgemm_plan, stream, m, n, k, rowmapA.data(), entriesA.data(),
                                                      rowmapB.data(), entriesB.data(), rowmapC.data(), &c_nnz, &c_max));
  sh->set_c_nnz(c_nnz);
  sh->set_max_result_nnz(c_max);
  sh->set_call_symbolic();
  sh->set_computed_rowptrs();  // always written, also without computeRowptrs
}

// CRV: the row maps (const int or const size_t), CIV: the entries (const int)
template <class SpgemmHandle, class CRV, class CIV, class CSV, class IV, class SV>
void spgemm_numeric_b200(SpgemmHandle* sh, int m, int n, int k, const CRV& rowmapA, const CIV& entriesA, const CSV& valuesA,
                         const CRV& rowmapB, const CIV& entriesB, const CSV& valuesB, const CRV& rowmapC,
                         const IV& entriesC, const SV& valuesC) {
  if (!sh->b200_spgemm_plan) throw std::invalid_argument("Call spgemm symbolic before spgemm numeric");
  void* stream = (void*)Kokkos::Cuda().cuda_stream();
  KOKKOSSPARSE_IMPL_B200_SAFE_CALL(b200_call_numeric(sh->b200_spgemm_plan, stream, m, n, k, rowmapA.data(), entriesA.data(),
                                                     valuesA.data(), rowmapB.data(), entriesB.data(), valuesB.data(),
                                                     rowmapC.data(), entriesC.data(), valuesC.data()));
  sh->set_computed_entries();
  sh->set_call_numeric();
}

#define KOKKOSSPARSE_B200_SPGEMM_DECL(SCALAR, MEMSPACE, TPL_AVAIL)                                                     \
  template <>                                                                                                          \
  struct SPGEMM_SYMBOLIC<KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE),            \
                         KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE),         \
                         KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(int, MEMSPACE), true,         \
                         TPL_AVAIL> {                                                                                  \
    using KernelHandle = KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE);                                                       \
    using c_int_view_t = KOKKOSSPARSE_B200_IV(const int, MEMSPACE);                                                    \
    using int_view_t   = KOKKOSSPARSE_B200_IV(int, MEMSPACE);                                                          \
    static void spgemm_symbolic(KernelHandle* handle, typename KernelHandle::nnz_lno_t m,                              \
                                typename KernelHandle::nnz_lno_t n, typename KernelHandle::nnz_lno_t k,                \
                                c_int_view_t row_mapA, c_int_view_t entriesA, bool, c_int_view_t row_mapB,             \
                                c_int_view_t entriesB, bool, int_view_t row_mapC, bool computeRowptrs) {               \
      Kokkos::Profiling::pushRegion("KokkosSparse::spgemm_symbolic[TPL_B200," + Kokkos::ArithTraits<SCALAR>::name() + "]"); \
      spgemm_symbolic_b200(handle->get_spgemm_handle(), m, n, k, row_mapA, entriesA, row_mapB, entriesB, row_mapC,     \
                           computeRowptrs);                                                                            \
      Kokkos::Profiling::popRegion();                                                                                  \
    }                                                                                                                  \
  };                                                                                                                   \
  template <>                                                                                                          \
  struct SPGEMM_NUMERIC<KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE),             \
                        KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE),       \
                        KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE),          \
                        KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE),       \
                        KOKKOSSPARSE_B200_IV(int, MEMSPACE), KOKKOSSPARSE_B200_IV(SCALAR, MEMSPACE), true, TPL_AVAIL> { \
    using KernelHandle    = KOKKOSSPARSE_B200_KH(SCALAR, MEMSPACE);                                                    \
    using c_int_view_t    = KOKKOSSPARSE_B200_IV(const int, MEMSPACE);                                                 \
    using int_view_t      = KOKKOSSPARSE_B200_IV(int, MEMSPACE);                                                       \
    using c_scalar_view_t = KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE);                                              \
    using scalar_view_t   = KOKKOSSPARSE_B200_IV(SCALAR, MEMSPACE);                                                    \
    static void spgemm_numeric(KernelHandle* handle, typename KernelHandle::nnz_lno_t m,                               \
                               typename KernelHandle::nnz_lno_t n, typename KernelHandle::nnz_lno_t k,                 \
                               c_int_view_t row_mapA, c_int_view_t entriesA, c_scalar_view_t valuesA, bool,            \
                               c_int_view_t row_mapB, c_int_view_t entriesB, c_scalar_view_t valuesB, bool,            \
                               c_int_view_t row_mapC, int_view_t entriesC, scalar_view_t valuesC) {                    \
      Kokkos::Profiling::pushRegion("KokkosSparse::spgemm_numeric[TPL_B200," + Kokkos::ArithTraits<SCALAR>::name() + "]"); \
      spgemm_numeric_b200(handle->get_spgemm_handle(), m, n, k, row_mapA, entriesA, valuesA, row_mapB, entriesB,       \
                          valuesB, row_mapC, entriesC, valuesC);                                                       \
      Kokkos::Profiling::popRegion();                                                                                  \
    }                                                                                                                  \
  };

// (int, size_t): the same bodies on size_t row maps, forwarded to the _i64 entries (64-bit offsets, products past 2^31 entries)
#define KOKKOSSPARSE_B200_SPGEMM64_DECL(SCALAR, MEMSPACE, TPL_AVAIL)                                                   \
  template <>                                                                                                          \
  struct SPGEMM_SYMBOLIC<KOKKOSSPARSE_B200_KH64(SCALAR, MEMSPACE), KOKKOSSPARSE_B200_IV(const size_t, MEMSPACE),       \
                         KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(const size_t, MEMSPACE),      \
                         KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(size_t, MEMSPACE), true,      \
                         TPL_AVAIL> {                                                                                  \
    using KernelHandle    = KOKKOSSPARSE_B200_KH64(SCALAR, MEMSPACE);                                                  \
    using c_size_view_t   = KOKKOSSPARSE_B200_IV(const size_t, MEMSPACE);                                              \
    using size_view_t     = KOKKOSSPARSE_B200_IV(size_t, MEMSPACE);                                                    \
    using c_int_view_t    = KOKKOSSPARSE_B200_IV(const int, MEMSPACE);                                                 \
    static void spgemm_symbolic(KernelHandle* handle, typename KernelHandle::nnz_lno_t m,                              \
                                typename KernelHandle::nnz_lno_t n, typename KernelHandle::nnz_lno_t k,                \
                                c_size_view_t row_mapA, c_int_view_t entriesA, bool, c_size_view_t row_mapB,           \
                                c_int_view_t entriesB, bool, size_view_t row_mapC, bool computeRowptrs) {              \
      Kokkos::Profiling::pushRegion("KokkosSparse::spgemm_symbolic[TPL_B200," + Kokkos::ArithTraits<SCALAR>::name() + "]"); \
      spgemm_symbolic_b200(handle->get_spgemm_handle(), m, n, k, row_mapA, entriesA, row_mapB, entriesB, row_mapC,     \
                           computeRowptrs);                                                                            \
      Kokkos::Profiling::popRegion();                                                                                  \
    }                                                                                                                  \
  };                                                                                                                   \
  template <>                                                                                                          \
  struct SPGEMM_NUMERIC<KOKKOSSPARSE_B200_KH64(SCALAR, MEMSPACE), KOKKOSSPARSE_B200_IV(const size_t, MEMSPACE),        \
                        KOKKOSSPARSE_B200_IV(const int, MEMSPACE), KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE),       \
                        KOKKOSSPARSE_B200_IV(const size_t, MEMSPACE), KOKKOSSPARSE_B200_IV(const int, MEMSPACE),       \
                        KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE), KOKKOSSPARSE_B200_IV(const size_t, MEMSPACE),    \
                        KOKKOSSPARSE_B200_IV(int, MEMSPACE), KOKKOSSPARSE_B200_IV(SCALAR, MEMSPACE), true, TPL_AVAIL> { \
    using KernelHandle    = KOKKOSSPARSE_B200_KH64(SCALAR, MEMSPACE);                                                  \
    using c_size_view_t   = KOKKOSSPARSE_B200_IV(const size_t, MEMSPACE);                                              \
    using c_int_view_t    = KOKKOSSPARSE_B200_IV(const int, MEMSPACE);                                                 \
    using int_view_t      = KOKKOSSPARSE_B200_IV(int, MEMSPACE);                                                       \
    using c_scalar_view_t = KOKKOSSPARSE_B200_IV(const SCALAR, MEMSPACE);                                              \
    using scalar_view_t   = KOKKOSSPARSE_B200_IV(SCALAR, MEMSPACE);                                                    \
    static void spgemm_numeric(KernelHandle* handle, typename KernelHandle::nnz_lno_t m,                               \
                               typename KernelHandle::nnz_lno_t n, typename KernelHandle::nnz_lno_t k,                 \
                               c_size_view_t row_mapA, c_int_view_t entriesA, c_scalar_view_t valuesA, bool,           \
                               c_size_view_t row_mapB, c_int_view_t entriesB, c_scalar_view_t valuesB, bool,           \
                               c_size_view_t row_mapC, int_view_t entriesC, scalar_view_t valuesC) {                   \
      Kokkos::Profiling::pushRegion("KokkosSparse::spgemm_numeric[TPL_B200," + Kokkos::ArithTraits<SCALAR>::name() + "]"); \
      spgemm_numeric_b200(handle->get_spgemm_handle(), m, n, k, row_mapA, entriesA, valuesA, row_mapB, entriesB,       \
                          valuesB, row_mapC, entriesC, valuesC);                                                       \
      Kokkos::Profiling::popRegion();                                                                                  \
    }                                                                                                                  \
  };

#define KOKKOSSPARSE_B200_SPGEMM_DECL_S(SCALAR, TPL_AVAIL)                  \
  KOKKOSSPARSE_B200_SPGEMM_DECL(SCALAR, Kokkos::CudaSpace, TPL_AVAIL)       \
  KOKKOSSPARSE_B200_SPGEMM_DECL(SCALAR, Kokkos::CudaUVMSpace, TPL_AVAIL)       \
  KOKKOSSPARSE_B200_SPGEMM64_DECL(SCALAR, Kokkos::CudaSpace, TPL_AVAIL)     \
  KOKKOSSPARSE_B200_SPGEMM64_DECL(SCALAR, Kokkos::CudaUVMSpace, TPL_AVAIL)

// both ETI flavours, as the cuSPARSE file declares (symbolic_tpl_spec_decl.hpp:355-363)
KOKKOSSPARSE_B200_SPGEMM_DECL_S(double, true)
KOKKOSSPARSE_B200_SPGEMM_DECL_S(float, true)
KOKKOSSPARSE_B200_SPGEMM_DECL_S(double, false)
KOKKOSSPARSE_B200_SPGEMM_DECL_S(float, false)

}  // namespace Impl
}  // namespace KokkosSparse
#endif
#endif
