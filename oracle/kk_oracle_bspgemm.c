/* oracle/libkkoracle_bspgemm.so: restatement of the reference's block SpGEMM host path (TEST INFRASTRUCTURE ONLY).
 *
 * bspgemm_debug_numeric (sparse/impl/KokkosSparse_bspgemm_impl_seq.hpp:39-130) with SerialGemmInternal<Unblocked>
 * (batched/dense/impl/KokkosBatched_Gemm_Serial_Internal.hpp:45-76, alpha = beta = 1): a dense accumulator of k blocks
 * per row, zeroed to +0.0; for every product of the row in ordinal order (A's row in storage order, each B row in
 * storage order) and p = 0..bs-1, acc(r, c) += (1 * a(r, p)) * b(p, c).  Built with -ffp-contract=off, so every
 * multiply and add is rounded on its own.  Unlike the reference, each C row's blocks are written SORTED by column
 * (the reference sorts afterwards with sort_bsr_matrix, bspgemm_numeric_spec.hpp:187-189).
 * Pinned bit for bit on the reference compiled in place (oracle/kkref_bspgemm.cpp, tests/test_oracle_bspgemm.py). */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define API __attribute__((visibility("default")))

/* distinct columns of every row of the block graph product (point symbolic on the block graphs); rmC: m + 1 */
API int64_t kko_bspgemm_symbolic(int m, int n, int k, const int* rmA, const int* entA, const int* rmB, const int* entB, int* rmC) {
  (void)n;
  char* flag = (char*)calloc((size_t)(k > 0 ? k : 1), 1);
  int* touched = (int*)malloc(sizeof(int) * (size_t)(k > 0 ? k : 1));
  int64_t nnz = 0;
  rmC[0] = 0;
  for (int i = 0; i < m; ++i) {
    int nt = 0;
    for (int a = rmA[i]; a < rmA[i + 1]; ++a) {
      const int col = entA[a];
      for (int b = rmB[col]; b < rmB[col + 1]; ++b) {
        const int c = entB[b];
        if (!flag[c]) {
          flag[c] = 1;
          touched[nt++] = c;
        }
      }
    }
    for (int t = 0; t < nt; ++t) flag[touched[t]] = 0;
    nnz += nt;
    rmC[i + 1] = (int)nnz;
  }
  free(flag);
  free(touched);
  return nnz;
}

static int cmp_int(const void* x, const void* y) {
  const int a = *(const int*)x, b = *(const int*)y;
  return (a > b) - (a < b);
}

#define BSPGEMM_NUMERIC(SFX, S)                                                                                                    \
  API void kko_bspgemm_numeric_##SFX(int m, int n, int k, int bs, const int* rmA, const int* entA, const S* valA, const int* rmB,  \
                                     const int* entB, const S* valB, const int* rmC, int* entC, S* valC) {                         \
    (void)n;                                                                                                                       \
    const size_t bb = (size_t)bs * (size_t)bs;                                                                                     \
    S* acc = (S*)malloc(sizeof(S) * (size_t)(k > 0 ? k : 1) * bb);                                                                 \
    char* flag = (char*)calloc((size_t)(k > 0 ? k : 1), 1);                                                                        \
    for (size_t e = 0; e < (size_t)k * bb; ++e) acc[e] = (S)0;                                                                     \
    for (int i = 0; i < m; ++i) {                                                                                                  \
      const int c0 = rmC[i];                                                                                                       \
      int nt = 0;                                                                                                                  \
      for (int a = rmA[i]; a < rmA[i + 1]; ++a) {                                                                                  \
        const S* av = valA + (size_t)a * bb;                                                                                       \
        const int col = entA[a];                                                                                                   \
        for (int b = rmB[col]; b < rmB[col + 1]; ++b) {                                                                            \
          const int c = entB[b];                                                                                                   \
          const S* bv = valB + (size_t)b * bb;                                                                                     \
          S* cv = acc + (size_t)c * bb;                                                                                            \
          if (!flag[c]) {                                                                                                          \
            flag[c] = 1;                                                                                                           \
            entC[c0 + nt++] = c;                                                                                                   \
          }                                                                                                                        \
          for (int p = 0; p < bs; ++p)                                                                                             \
            for (int r = 0; r < bs; ++r) {                                                                                         \
              const S ta = (S)1 * av[(size_t)r * bs + p];                                                                          \
              for (int q = 0; q < bs; ++q) cv[(size_t)r * bs + q] += ta * bv[(size_t)p * bs + q];                                 \
            }                                                                                                                      \
        }                                                                                                                          \
      }                                                                                                                            \
      qsort(entC + c0, (size_t)nt, sizeof(int), cmp_int);                                                                          \
      for (int t = 0; t < nt; ++t) {                                                                                               \
        const int c = entC[c0 + t];                                                                                                \
        memcpy(valC + (size_t)(c0 + t) * bb, acc + (size_t)c * bb, sizeof(S) * bb);                                               \
        for (size_t e = 0; e < bb; ++e) acc[(size_t)c * bb + e] = (S)0;                                                            \
        flag[c] = 0;                                                                                                               \
      }                                                                                                                            \
    }                                                                                                                              \
    free(acc);                                                                                                                     \
    free(flag);                                                                                                                    \
  }

BSPGEMM_NUMERIC(f64, double)
BSPGEMM_NUMERIC(f32, float)
