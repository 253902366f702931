// oracle/_ref/libkkref_bspgemm.so: the reference's own block SpGEMM host path, bspgemm_debug_numeric
// (sparse/impl/KokkosSparse_bspgemm_impl_seq.hpp:39-130) with its GEMM, SerialGemmInternal<Unblocked>
// (batched/dense/impl/KokkosBatched_Gemm_Serial_Internal.hpp:45-76), both compiled from the reference tree in place
// (paths injected by oracle/bspgemm.mk) over the stand-ins in oracle/kokkos_mock/bspgemm.  No reference source is
// copied into this repository.  TEST INFRASTRUCTURE ONLY: pins oracle/kk_oracle_bspgemm.c's restatement bit for bit
// (tests/test_oracle_bspgemm.py).
//
// The reference writes each C row's columns in first-touch order (its spec layer runs sort_bsr_matrix afterwards,
// bspgemm_numeric_spec.hpp:187-189); the caller sorts.
#include <cstdint>
#include "KokkosKernels_helpers.hpp"
#include KKREF_BSPGEMM_SEQ

namespace {
template <class Scalar>
struct KernelHandleMock {
  using nnz_lno_t    = int;
  using size_type    = int;
  using nnz_scalar_t = Scalar;
};

template <class S>
void run(int m, int n, int k, int bs, int* rmA, int nnzA, int* entA, S* valA, int* rmB, int nnzB, int* entB, S* valB,
         int* rmC, int nnzC, int* entC, S* valC) {
  KernelHandleMock<S> kh;
  const size_t bb = (size_t)bs * bs;
  Kokkos::View<int> vrmA(rmA, (size_t)m + 1), ventA(entA, (size_t)nnzA), vrmB(rmB, (size_t)n + 1), ventB(entB, (size_t)nnzB),
      vrmC(rmC, (size_t)m + 1), ventC(entC, (size_t)nnzC);
  Kokkos::View<S> vvalA(valA, nnzA * bb), vvalB(valB, nnzB * bb), vvalC(valC, nnzC * bb);
  KokkosSparse::Impl::bspgemm_debug_numeric(&kh, m, n, k, bs, vrmA, ventA, vvalA, false, vrmB, ventB, vvalB, false, vrmC, ventC,
                                            vvalC);
}
}  // namespace

extern "C" {
__attribute__((visibility("default"))) void kkref_bspgemm_numeric_f64(int m, int n, int k, int bs, int* rmA, int nnzA, int* entA,
                                                                       double* valA, int* rmB, int nnzB, int* entB, double* valB,
                                                                       int* rmC, int nnzC, int* entC, double* valC) {
  run<double>(m, n, k, bs, rmA, nnzA, entA, valA, rmB, nnzB, entB, valB, rmC, nnzC, entC, valC);
}
__attribute__((visibility("default"))) void kkref_bspgemm_numeric_f32(int m, int n, int k, int bs, int* rmA, int nnzA, int* entA,
                                                                       float* valA, int* rmB, int nnzB, int* entB, float* valB,
                                                                       int* rmC, int nnzC, int* entC, float* valC) {
  run<float>(m, n, k, bs, rmA, nnzA, entA, valA, rmB, nnzB, entB, valB, rmC, nnzC, entC, valC);
}
}
