// gs2.cu -- two-stage Gauss-Seidel (GS_TWOSTAGE with inner Jacobi-Richardson sweeps): the Gauss-Seidel variant that is a loop
// of SpMVs (SURVEY.md section 8f rank 4: "Gauss-Seidel ... drivers that call spmv in a loop").
//
// Replaces, behind the C ABI (b200sp_gs2_*), TwostageGaussSeidel of
//   sparse/impl/KokkosSparse_twostage_gauss_seidel_impl.hpp   symbolic :544-697, numeric :700-772, apply :778-1035
// reached through gauss_seidel_symbolic / numeric / apply with a handle created as GS_TWOSTAGE
// (sparse/src/KokkosSparse_gauss_seidel_handle.hpp:513-673; options set_gs_set_num_inner_sweeps / _outer_sweeps /
// _inner_damp_factor / set_gs_twostage_compact_form, sparse/src/KokkosKernels_Handle.hpp:639-683).
//
// A = L + D + U on the square part (columns >= num_rows belong to ghost entries of x: read, never written).
//   symbolic: row maps and entries of L (strictly lower) and U (strictly upper, column < num_rows), storage order of A kept;
//             compact form also La (lower entries + ghost columns) and Ua (upper entries, ghost columns included)
//   numeric : D = 1 / a_ii (or the caller's inverse diagonal), values of L and U scaled by D (row scaling); La / Ua unscaled, Da = a_ii
//   apply   : per sweep  R = B - A x  (compact: R = B - (Ua or La) x + (1/omega - 1) Da.*x);  T = D.*R;  R = gamma T;
//             inner sweeps: Z = T - omega (L or U) R;  Z = gamma Z + (1 - gamma) R;  R = Z;  then x += omega Z (compact: x = omega Z)
// Every product is the library's own SpMV (spmv.cu: the TMA-tiled kernel with its plan, one plan per matrix A, L, U, La, Ua);
// the vector updates in between are fused into one kernel per step, each computing exactly the expression the reference's
// KokkosBlas call sequence computes (mult with beta = 0, scal, axpy), so the only difference to the reference is the summation
// order inside the SpMVs.  No colouring, no atomics: deterministic and independent of the row order.  Several right-hand sides go
// through the multivector products (spmm.cu), so a sweep reads the matrix once for all of them.
// The sptrsv variant (two_stage = false, "classic" in the reference's unit test; B200SP_GS2_TWO_STAGE = 0): Z = (L + D)^{-1} R is a
// level-set triangular solve on the lower (upper) triangle of A itself (sptrsv.cu, no copy of the triangle), then x += Z; omega
// must be 1, as in the reference (:886-893).
#include <algorithm>
#include <new>

#include "common.cuh"
#include "scan.cuh"

struct b200sp_sptrsv_plan;
extern "C" int b200sp_sptrsv_plan_create(b200sp_sptrsv_plan** plan);
extern "C" int b200sp_sptrsv_plan_destroy(b200sp_sptrsv_plan* plan, void* stream);
namespace b200sp {
int sptrsv_symbolic_impl(b200sp_sptrsv_plan* p, cudaStream_t st, int n, const int* rp, const int* ci, bool lower, bool filter);
template <typename S>
int sptrsv_solve_impl(b200sp_sptrsv_plan* p, cudaStream_t st, int n, const int* rp, const int* ci, const S* v, const S* b, S* x,
                      const S* dinv);
}  // namespace b200sp

struct b200sp_gs2_plan {
  bool compact = false;
  bool two_stage = true;      // false: the classic form, triangular solves instead of inner Jacobi-Richardson sweeps
  bool given_dinv = false;    // numeric was handed an inverse diagonal
  b200sp_sptrsv_plan* tr[2] = {nullptr, nullptr};  // level sets of the lower / upper triangle of A (classic form)
  int inner = 1, outer = 1;
  double gamma = 1.0;
  bool symbolic = false, numeric = false;
  int n = 0, ncols = 0;
  int64_t nnz = 0;
  const int *key_rp = nullptr, *key_ci = nullptr;
  int scalar_bytes = 0;
  b200sp::DevArray<int> rp[4];  // L, U, La, Ua
  b200sp::DevArray<int> ci[4];
  b200sp::DevArray<char> v[4];  // values and vectors below: scalars of the numeric call's type
  int64_t cnt[4] = {0, 0, 0, 0};
  b200sp::DevArray<char> D, Da;
  b200sp::DevArray<char> R, T, Z;
  int work_cols = 0;  // right-hand sides R, T, Z are sized for
  b200sp_spmv_plan* plan[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};  // L, U, La, Ua, A
};

namespace b200sp {
namespace {

enum { kL = 0, kU = 1, kLa = 2, kUa = 3, kA = 4 };

// entries of row i per part; missing diagonal -> *nodiag = 1 + smallest such row
__global__ void __launch_bounds__(256) gs2_count_kernel(int n, const int* __restrict__ rp, const int* __restrict__ ci, int* __restrict__ cL,
                                                        int* __restrict__ cU, int* __restrict__ cLa, int* __restrict__ cUa, int compact,
                                                        int* __restrict__ nodiag) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    int l = 0, u = 0, g = 0, d = 0;
    for (int k = rp[i]; k < rp[i + 1]; ++k) {
      const int c = ci[k];
      if (c < i) ++l;
      else if (c == i) d = 1;
      else if (c < n) ++u;
      else ++g;
    }
    cL[i] = l;
    cU[i] = u;
    if (compact) {
      cLa[i] = l + g;
      cUa[i] = u + g;
    }
    if (!d) atomicMin(nodiag, i);
  }
}

__global__ void __launch_bounds__(256) gs2_entries_kernel(int n, const int* __restrict__ rp, const int* __restrict__ ci, const int* __restrict__ rL,
                                                          int* __restrict__ eL, const int* __restrict__ rU, int* __restrict__ eU,
                                                          const int* __restrict__ rLa, int* __restrict__ eLa, const int* __restrict__ rUa,
                                                          int* __restrict__ eUa, int compact) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    int pl = rL[i], pu = rU[i], pla = compact ? rLa[i] : 0, pua = compact ? rUa[i] : 0;
    for (int k = rp[i]; k < rp[i + 1]; ++k) {
      const int c = ci[k];
      if (c < i) {
        eL[pl++] = c;
        if (compact) eLa[pla++] = c;
      } else if (c > i) {
        if (c < n) {
          eU[pu++] = c;
          if (compact) eUa[pua++] = c;
        } else if (compact) {
          eLa[pla++] = c;
          eUa[pua++] = c;
        }
      }
    }
  }
}

// values of the parts + the diagonal (Tag_valuesLU, :385-470); L and U leave here already scaled by D
template <typename S>
__global__ void __launch_bounds__(256) gs2_values_kernel(int n, const int* __restrict__ rp, const int* __restrict__ ci, const S* __restrict__ v,
                                                         const S* __restrict__ given_dinv, const int* __restrict__ rL, S* __restrict__ vL,
                                                         const int* __restrict__ rU, S* __restrict__ vU, const int* __restrict__ rLa,
                                                         S* __restrict__ vLa, const int* __restrict__ rUa, S* __restrict__ vUa,
                                                         S* __restrict__ D, S* __restrict__ Da, int compact) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    S d = S(0), da = S(0);
    for (int k = rp[i]; k < rp[i + 1]; ++k)
      if (ci[k] == i) {
        d = given_dinv ? given_dinv[i] : v[k];
        da = v[k];
      }
    if (!given_dinv) d = S(1) / d;
    D[i] = d;
    if (compact) Da[i] = da;
    int pl = rL[i], pu = rU[i], pla = compact ? rLa[i] : 0, pua = compact ? rUa[i] : 0;
    for (int k = rp[i]; k < rp[i + 1]; ++k) {
      const int c = ci[k];
      const S a = v[k];
      if (c < i) {
        vL[pl++] = a * d;
        if (compact) vLa[pla++] = a;
      } else if (c > i) {
        if (c < n) {
          vU[pu++] = a * d;
          if (compact) vUa[pua++] = a;
        } else if (compact) {
          vLa[pla++] = a;
          vUa[pua++] = a;
        }
      }
    }
  }
}

// the vector steps between the SpMVs; every expression is the one the reference's KokkosBlas sequence evaluates.  All of them
// run over an n x k block (k right-hand sides, column-major): blockIdx.y is the column, so no index is ever divided; the work
// vectors R, T, Z have leading dimension n, x and b the caller's.
#define GS2_ROWS(i) for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
template <typename S>
__global__ void __launch_bounds__(256) gs2_copy_kernel(int n, const S* __restrict__ a, int64_t lda, S* __restrict__ out,
                                                       int64_t ldo) {  // scal(out, one, a)
  a += blockIdx.y * lda;
  out += blockIdx.y * ldo;
  GS2_ROWS(i) out[i] = S(1) * a[i];
}
template <typename S>
__global__ void __launch_bounds__(256) gs2_diag_term_kernel(int n, const S* __restrict__ Da, const S* __restrict__ x, int64_t ldx, S omega2,
                                                            S* __restrict__ Z, S* __restrict__ R) {  // Z = Da.*x;  R += omega2 Z
  x += blockIdx.y * ldx;
  Z += (int64_t)blockIdx.y * n;
  R += (int64_t)blockIdx.y * n;
  GS2_ROWS(i) {
    const S z = S(1) * Da[i] * x[i];
    Z[i] = z;
    R[i] += omega2 * z;
  }
}
// inner == 0:  Z = D.*R (times gamma);  else  T = D.*R, R = T (times gamma)
template <typename S>
__global__ void __launch_bounds__(256) gs2_start_kernel(int n, const S* __restrict__ D, S* __restrict__ R, S* __restrict__ T, S* __restrict__ Z,
                                                        S gamma, int inner) {
  const int64_t off = (int64_t)blockIdx.y * n;
  R += off;
  T += off;
  Z += off;
  GS2_ROWS(i) {
    const S t = S(1) * D[i] * R[i];
    if (inner == 0) {
      Z[i] = (gamma != S(1)) ? gamma * t : t;
    } else {
      T[i] = t;
      const S r = S(1) * t;
      R[i] = (gamma != S(1)) ? gamma * r : r;
    }
  }
}
// after Z = T - omega M R:  gamma != 1: Z = gamma Z + (1 - gamma) R;  not the last inner sweep: R = Z
template <typename S>
__global__ void __launch_bounds__(256) gs2_inner_kernel(int n, S* __restrict__ Z, S* __restrict__ R, S gamma, int copy_back) {
  Z += (int64_t)blockIdx.y * n;
  R += (int64_t)blockIdx.y * n;
  GS2_ROWS(i) {
    S z = Z[i];
    if (gamma != S(1)) {
      z = gamma * z;
      z += (S(1) - gamma) * R[i];
      Z[i] = z;
    }
    if (copy_back) R[i] = S(1) * z;
  }
}
template <typename S>
__global__ void __launch_bounds__(256) gs2_update_kernel(int n, const S* __restrict__ Z, S omega, S* __restrict__ x, int64_t ldx, int compact) {
  Z += (int64_t)blockIdx.y * n;
  x += blockIdx.y * ldx;
  GS2_ROWS(i) {
    if (compact) x[i] = omega * Z[i];
    else x[i] += omega * Z[i];
  }
}
#undef GS2_ROWS

void release_parts(b200sp_gs2_plan* p, cudaStream_t st) {
  for (int q = 0; q < 4; ++q) {
    p->rp[q].release(st);
    p->ci[q].release(st);
    p->v[q].release(st);
    p->cnt[q] = 0;
  }
  for (DevArray<char>* q : {&p->D, &p->Da, &p->R, &p->T, &p->Z}) q->release(st);
  p->symbolic = p->numeric = false;
  p->scalar_bytes = 0;
  p->work_cols = 0;
}

inline int spmv32(b200sp_spmv_plan* pl, void* st, int m, int n, int64_t nnz, double a, const int* rp, const int* ci, const double* v,
                  const double* x, double b, double* y) {
  return b200sp_spmv_f64_i32(pl, st, 'N', m, n, nnz, a, rp, ci, v, x, b, y);
}
inline int spmv32(b200sp_spmv_plan* pl, void* st, int m, int n, int64_t nnz, float a, const int* rp, const int* ci, const float* v,
                  const float* x, float b, float* y) {
  return b200sp_spmv_f32_i32(pl, st, 'N', m, n, nnz, a, rp, ci, v, x, b, y);
}

inline int spmm32(b200sp_spmv_plan* pl, void* st, int m, int n, int64_t nnz, int k, double a, const int* rp, const int* ci, const double* v,
                  const double* X, int64_t ldx, double b, double* Y, int64_t ldy) {
  return b200sp_spmm_f64_i32(pl, st, 'N', m, n, nnz, k, a, rp, ci, v, X, ldx, 0, b, Y, ldy, 0);
}
inline int spmm32(b200sp_spmv_plan* pl, void* st, int m, int n, int64_t nnz, int k, float a, const int* rp, const int* ci, const float* v,
                  const float* X, int64_t ldx, float b, float* Y, int64_t ldy) {
  return b200sp_spmm_f32_i32(pl, st, 'N', m, n, nnz, k, a, rp, ci, v, X, ldx, 0, b, Y, ldy, 0);
}
// Y = beta Y + alpha M X for k columns (column-major): the rank-1 kernels for one column, the multivector kernels otherwise --
// the matrix is read once for all right-hand sides
template <typename S>
inline int product(b200sp_spmv_plan* pl, void* st, int m, int n, int64_t nnz, int k, S a, const int* rp, const int* ci, const S* v, const S* X,
                   int64_t ldx, S b, S* Y, int64_t ldy) {
  if (k == 1) return spmv32(pl, st, m, n, nnz, a, rp, ci, v, X, b, Y);
  return spmm32(pl, st, m, n, nnz, k, a, rp, ci, v, X, ldx, b, Y, ldy);
}

template <typename S>
int numeric_impl(b200sp_gs2_plan* p, cudaStream_t st, int n, int ncols, const int* row_ptr, const int* col_idx, const S* vals,
                 const S* given_dinv) {
  B200SP_REQUIRE(p != nullptr, "gs2_numeric: null plan");
  if (!p->symbolic || p->n != n || p->ncols != ncols || p->key_rp != row_ptr || p->key_ci != col_idx) {
    set_error("gs2_numeric: symbolic was not called on this plan with this matrix");
    return B200SP_ERR_STATE;
  }
  if (p->scalar_bytes != (int)sizeof(S)) {
    for (int q = 0; q < 4; ++q)
      if (q < 2 || p->compact) B200SP_CUDA_TRY(p->v[q].grow(sizeof(S) * (size_t)std::max<int64_t>(p->cnt[q], 1), st));
    for (DevArray<char>* q : {&p->D, &p->Da, &p->R, &p->T, &p->Z}) B200SP_CUDA_TRY(q->grow(sizeof(S) * (size_t)std::max(n, 1), st));
    p->scalar_bytes = (int)sizeof(S);
    p->work_cols = 1;
  }
  if (n > 0) {
    B200SP_REQUIRE(vals != nullptr, "gs2_numeric: null values");
    gs2_values_kernel<S><<<grid_for(n), 256, 0, st>>>(n, row_ptr, col_idx, vals, given_dinv, p->rp[kL], p->v[kL].as<S>(), p->rp[kU], p->v[kU].as<S>(),
                                                         p->rp[kLa], p->v[kLa].as<S>(), p->rp[kUa], p->v[kUa].as<S>(), p->D.as<S>(), p->Da.as<S>(),
                                                         p->compact ? 1 : 0);
    B200SP_LAUNCH_CHECK();
  }
  p->given_dinv = given_dinv != nullptr;
  p->numeric = true;
  return B200SP_OK;
}

template <typename S>
int apply_impl(b200sp_gs2_plan* p, void* stream, int n, int ncols, const int* row_ptr, const int* col_idx, const S* vals, S* x, int64_t ldx,
               const S* b, int64_t ldb, int nrhs, int init_zero_x, S omega, int num_iter, int direction) {
  cudaStream_t st = (cudaStream_t)stream;
  B200SP_REQUIRE(p != nullptr, "gs2_apply: null plan");
  B200SP_REQUIRE(direction >= 0 && direction <= 2, "gs2_apply: direction %d not in {0 symmetric, 1 forward, 2 backward}", direction);
  B200SP_REQUIRE(nrhs <= 65535, "gs2_apply: at most 65535 right-hand sides per call (got %d)", nrhs);
  B200SP_REQUIRE(nrhs >= 0 && num_iter >= 0, "gs2_apply: negative count (nrhs=%d numIter=%d)", nrhs, num_iter);
  if (!p->numeric || p->n != n || p->ncols != ncols || p->key_rp != row_ptr || p->key_ci != col_idx || p->scalar_bytes != (int)sizeof(S)) {
    set_error("gs2_apply: numeric was not called on this plan with this matrix and scalar type");
    return B200SP_ERR_STATE;
  }
  if (n == 0 || nrhs == 0) return B200SP_OK;
  B200SP_REQUIRE(x && b && vals, "gs2_apply: null pointer argument");
  B200SP_REQUIRE(nrhs == 1 || (ldx >= ncols && ldb >= n), "gs2_apply: leading dimensions too small (ldx=%lld ldb=%lld)", (long long)ldx,
                 (long long)ldb);
  const S one = S(1), gamma = (S)p->gamma;
  if (!p->two_stage && omega != one) {  // the reference throws std::invalid_argument here (:886-893)
    set_error("gs2_apply: omega != 1 is not supported by the classic (sptrsv) form");
    return B200SP_ERR_INVALID_ARGUMENT;
  }
  const int k = nrhs;
  const int64_t total = (int64_t)n * k;
  if (k > p->work_cols) {  // work vectors for k right-hand sides (numeric sizes them for one)
    p->work_cols = 0;
    for (DevArray<char>* q : {&p->R, &p->T, &p->Z}) B200SP_CUDA_TRY(q->grow(sizeof(S) * (size_t)total, st));
    p->work_cols = k;
  }
  S *R = p->R.as<S>(), *T = p->T.as<S>(), *Z = p->Z.as<S>();
  const S *D = p->D.as<const S>(), *Da = p->Da.as<const S>();
  const dim3 nb((unsigned)grid_for(n), (unsigned)k);  // blockIdx.y = right-hand side
  if (k == 1) {
    ldx = ncols;
    ldb = n;
  }
  int sweeps = std::max(p->outer, num_iter);
  if (direction == 0) sweeps *= 2;
  if (init_zero_x)
    for (int j = 0; j < k; ++j) B200SP_CUDA_TRY(cudaMemsetAsync(x + (int64_t)j * ldx, 0, sizeof(S) * (size_t)ncols, st));
  for (int sweep = 0; sweep < sweeps; ++sweep) {
    const bool forward = direction == 1 || (direction == 0 && sweep % 2 == 0);
    gs2_copy_kernel<S><<<nb, 256, 0, st>>>(n, b, ldb, R, (int64_t)n);
    B200SP_LAUNCH_CHECK();
    int rc = B200SP_OK;
    if (sweep > 0 || !init_zero_x) {
      if (p->compact) {
        const int q = forward ? kUa : kLa;
        rc = product<S>(p->plan[q], stream, n, ncols, p->cnt[q], k, -one, p->rp[q], p->ci[q], p->v[q].as<const S>(), x, ldx, one, R, n);
        if (rc) return rc;
        if (omega != one) {
          gs2_diag_term_kernel<S><<<nb, 256, 0, st>>>(n, Da, x, ldx, one / omega - one, Z, R);
          B200SP_LAUNCH_CHECK();
        }
      } else {
        rc = product<S>(p->plan[kA], stream, n, ncols, p->nnz, k, -one, row_ptr, col_idx, vals, x, ldx, one, R, n);
        if (rc) return rc;
      }
    }
    if (!p->two_stage) {
      // ===== classic form: Z = (L + D)^{-1} R  or  (U + D)^{-1} R, one right-hand side at a time (:894-915), then x (+)= Z
      for (int j = 0; j < k; ++j) {
        rc = sptrsv_solve_impl<S>(p->tr[forward ? 0 : 1], st, n, row_ptr, col_idx, vals, R + (int64_t)j * n, Z + (int64_t)j * n,
                                  p->given_dinv ? D : (const S*)nullptr);
        if (rc) return rc;
      }
      gs2_update_kernel<S><<<nb, 256, 0, st>>>(n, Z, one, x, ldx, p->compact ? 1 : 0);
      B200SP_LAUNCH_CHECK();
      continue;
    }
    gs2_start_kernel<S><<<nb, 256, 0, st>>>(n, D, R, T, Z, gamma, p->inner);
    B200SP_LAUNCH_CHECK();
    for (int ii = 0; ii < p->inner; ++ii) {
      gs2_copy_kernel<S><<<nb, 256, 0, st>>>(n, T, (int64_t)n, Z, (int64_t)n);
      B200SP_LAUNCH_CHECK();
      const int q = forward ? kL : kU;
      rc = product<S>(p->plan[q], stream, n, n, p->cnt[q], k, -omega, p->rp[q], p->ci[q], p->v[q].as<const S>(), R, n, one, Z, n);
      if (rc) return rc;
      const int copy_back = ii + 1 < p->inner;
      if (gamma != one) {
        gs2_inner_kernel<S><<<nb, 256, 0, st>>>(n, Z, R, gamma, copy_back);
        B200SP_LAUNCH_CHECK();
      } else if (copy_back) {
        std::swap(R, Z);  // R = 1 * Z is exact: the next inner sweep reads the buffer just written, no copy
      }
    }
    gs2_update_kernel<S><<<nb, 256, 0, st>>>(n, Z, omega, x, ldx, p->compact ? 1 : 0);
    B200SP_LAUNCH_CHECK();
  }
  return B200SP_OK;
}

}  // namespace
}  // namespace b200sp

extern "C" {

int b200sp_gs2_plan_create(b200sp_gs2_plan** plan) {
  B200SP_REQUIRE(plan != nullptr, "gs2_plan_create: null output pointer");
  b200sp_gs2_plan* p = new (std::nothrow) b200sp_gs2_plan();
  if (!p) {
    b200sp::set_error("gs2_plan_create: out of host memory");
    return B200SP_ERR_ALLOC;
  }
  for (int q = 0; q < 5; ++q) {
    const int rc = b200sp_spmv_plan_create(&p->plan[q], B200SP_SPMV_DEFAULT);
    if (rc) {
      b200sp_gs2_plan_destroy(p, nullptr);
      return rc;
    }
  }
  *plan = p;
  return B200SP_OK;
}

int b200sp_gs2_plan_destroy(b200sp_gs2_plan* p, void* stream) {
  if (!p) return B200SP_OK;
  b200sp::release_parts(p, (cudaStream_t)stream);
  for (int q = 0; q < 2; ++q) b200sp_sptrsv_plan_destroy(p->tr[q], stream);
  for (int q = 0; q < 5; ++q)
    if (p->plan[q]) b200sp_spmv_plan_destroy(p->plan[q], stream);
  delete p;
  return B200SP_OK;
}

int b200sp_gs2_plan_set(b200sp_gs2_plan* p, int option, double value) {
  B200SP_REQUIRE(p != nullptr, "gs2_plan_set: null plan");
  switch (option) {
    case B200SP_GS2_COMPACT_FORM:
      if ((value != 0.0) != p->compact) p->symbolic = p->numeric = false;  // La / Ua are built by symbolic
      p->compact = value != 0.0;
      return B200SP_OK;
    case B200SP_GS2_NUM_INNER_SWEEPS:
      B200SP_REQUIRE(value >= 0, "gs2_plan_set: negative number of inner sweeps");
      p->inner = (int)value;
      return B200SP_OK;
    case B200SP_GS2_NUM_OUTER_SWEEPS:
      B200SP_REQUIRE(value >= 0, "gs2_plan_set: negative number of outer sweeps");
      p->outer = (int)value;
      return B200SP_OK;
    case B200SP_GS2_INNER_DAMP_FACTOR: p->gamma = value; return B200SP_OK;
    case B200SP_GS2_TWO_STAGE:
      if ((value != 0.0) != p->two_stage) p->symbolic = p->numeric = false;  // the level sets are built by symbolic
      p->two_stage = value != 0.0;
      return B200SP_OK;
  }
  b200sp::set_error("gs2_plan_set: unknown option %d", option);
  return B200SP_ERR_INVALID_ARGUMENT;
}

int b200sp_gs2_symbolic_i32(b200sp_gs2_plan* p, void* stream, int n, int ncols, const int* row_ptr, const int* col_idx) {
  using namespace b200sp;
  cudaStream_t st = (cudaStream_t)stream;
  B200SP_REQUIRE(p != nullptr, "gs2_symbolic: null plan");
  B200SP_REQUIRE(n >= 0 && ncols >= n, "gs2_symbolic: needs 0 <= num_rows <= num_cols (got %d x %d)", n, ncols);
  const bool compact = p->compact;
  release_parts(p, st);
  p->n = n;
  p->ncols = ncols;
  p->key_rp = row_ptr;
  p->key_ci = col_idx;
  p->nnz = 0;
  if (n == 0) {
    p->symbolic = true;
    return B200SP_OK;
  }
  B200SP_REQUIRE(row_ptr != nullptr, "gs2_symbolic: null row map");
  const int parts = compact ? 4 : 2;
  DevTmp tmp(st);
  int* cnt[4] = {nullptr, nullptr, nullptr, nullptr};
  for (int q = 0; q < parts; ++q) B200SP_CUDA_TRY(tmp.alloc(&cnt[q], (size_t)n));
  int *nodiag = nullptr, *dmax = nullptr, *bmax = nullptr;
  long long *bsum = nullptr, *dtotal = nullptr;
  B200SP_CUDA_TRY(tmp.alloc(&nodiag, 1));
  B200SP_CUDA_TRY(tmp.alloc(&dmax, 1));
  B200SP_CUDA_TRY(tmp.alloc(&bmax, (size_t)scan_blocks(n)));
  B200SP_CUDA_TRY(tmp.alloc(&bsum, (size_t)scan_blocks(n)));
  B200SP_CUDA_TRY(tmp.alloc(&dtotal, 4));
  B200SP_CUDA_TRY(cudaMemsetAsync(nodiag, 0x7F, sizeof(int), st));
  gs2_count_kernel<<<grid_for(n), 256, 0, st>>>(n, row_ptr, col_idx, cnt[0], cnt[1], cnt[2], cnt[3], compact ? 1 : 0, nodiag);
  B200SP_LAUNCH_CHECK();
  for (int q = 0; q < parts; ++q) {
    B200SP_CUDA_TRY(p->rp[q].alloc((size_t)n + 4, st));
    const int rc = launch_exclusive_scan(st, n, cnt[q], p->rp[q], bsum, bmax, dtotal + q, dmax);
    if (rc) return rc;
  }
  long long h_total[4] = {0, 0, 0, 0};
  int h_nodiag = 0, h_last[2] = {0, 0};
  B200SP_CUDA_TRY(cudaMemcpyAsync(h_total, dtotal, sizeof(long long) * parts, cudaMemcpyDeviceToHost, st));
  B200SP_CUDA_TRY(cudaMemcpyAsync(&h_nodiag, nodiag, sizeof(int), cudaMemcpyDeviceToHost, st));
  B200SP_CUDA_TRY(cudaMemcpyAsync(h_last, row_ptr + n, sizeof(int), cudaMemcpyDeviceToHost, st));
  B200SP_CUDA_TRY(cudaStreamSynchronize(st));
  if (h_nodiag < n) {
    release_parts(p, st);
    set_error("gs2_symbolic: row %d has no diagonal entry", h_nodiag);
    return B200SP_ERR_INVALID_ARGUMENT;
  }
  p->nnz = h_last[0];
  for (int q = 0; q < parts; ++q) {
    p->cnt[q] = h_total[q];
    B200SP_CUDA_TRY(p->ci[q].alloc((size_t)std::max<int64_t>(p->cnt[q], 1), st));
  }
  gs2_entries_kernel<<<grid_for(n), 256, 0, st>>>(n, row_ptr, col_idx, p->rp[kL], p->ci[kL], p->rp[kU], p->ci[kU], p->rp[kLa], p->ci[kLa],
                                                    p->rp[kUa], p->ci[kUa], compact ? 1 : 0);
  B200SP_LAUNCH_CHECK();
  if (!p->two_stage) {  // classic form: level sets of the lower and the upper triangle of A (sptrsv_symbolic, :685-697)
    for (int q = 0; q < 2; ++q) {
      if (!p->tr[q]) {
        const int rc = b200sp_sptrsv_plan_create(&p->tr[q]);
        if (rc) return rc;
      }
      const int rc = sptrsv_symbolic_impl(p->tr[q], st, n, row_ptr, col_idx, q == 0, true);
      if (rc) return rc;
    }
  }
  p->symbolic = true;
  return B200SP_OK;
}

int b200sp_gs2_numeric_f64_i32(b200sp_gs2_plan* p, void* stream, int n, int ncols, const int* row_ptr, const int* col_idx, const double* vals,
                               const double* given_inverse_diagonal) {
  return b200sp::numeric_impl<double>(p, (cudaStream_t)stream, n, ncols, row_ptr, col_idx, vals, given_inverse_diagonal);
}
int b200sp_gs2_numeric_f32_i32(b200sp_gs2_plan* p, void* stream, int n, int ncols, const int* row_ptr, const int* col_idx, const float* vals,
                               const float* given_inverse_diagonal) {
  return b200sp::numeric_impl<float>(p, (cudaStream_t)stream, n, ncols, row_ptr, col_idx, vals, given_inverse_diagonal);
}

int b200sp_gs2_apply_f64_i32(b200sp_gs2_plan* p, void* stream, int n, int ncols, const int* row_ptr, const int* col_idx, const double* vals,
                             double* x, int64_t ldx, const double* b, int64_t ldb, int nrhs, int init_zero_x, double omega, int num_iter,
                             int direction) {
  return b200sp::apply_impl<double>(p, stream, n, ncols, row_ptr, col_idx, vals, x, ldx, b, ldb, nrhs, init_zero_x, omega, num_iter, direction);
}
int b200sp_gs2_apply_f32_i32(b200sp_gs2_plan* p, void* stream, int n, int ncols, const int* row_ptr, const int* col_idx, const float* vals,
                             float* x, int64_t ldx, const float* b, int64_t ldb, int nrhs, int init_zero_x, float omega, int num_iter,
                             int direction) {
  return b200sp::apply_impl<float>(p, stream, n, ncols, row_ptr, col_idx, vals, x, ldx, b, ldb, nrhs, init_zero_x, omega, num_iter, direction);
}

}  // extern "C"
