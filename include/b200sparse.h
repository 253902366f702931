/*
 * b200sparse.h -- C ABI of libb200sparse: H100 (sm_90a) SpMV / SpMM / SpGEMM
 * for CrsMatrix data, the drop-in behind Kokkos Kernels' TPL slot for
 * Kokkos::Cuda (SURVEY.md section 8b).
 *
 * Conventions
 *  - plain C, opaque plans, caller-owned DEVICE pointers, explicit stream
 *    (a cudaStream_t passed as void*), 0-based int32 row offsets ("Offset")
 *    and column indices ("Ordinal") -- Kokkos Kernels' default_types
 *    (reference common/src/KokkosKernels_default_types.hpp:41-58) and the
 *    only combination its cuSPARSE SpMM/SpGEMM specialisations accept
 *    (sparse/tpls/KokkosSparse_spgemm_symbolic_tpl_spec_avail.hpp:36-40).
 *  - every entry point returns a b200sp_status; on failure
 *    b200sp_last_error_string() describes it (thread-local).  The Kokkos shim
 *    turns non-zero into std::runtime_error / std::invalid_argument like
 *    KOKKOSSPARSE_IMPL_CUSPARSE_SAFE_CALL does
 *    (sparse/src/KokkosSparse_Utils_cusparse.hpp:28-67).
 *  - SpMV/SpMM are asynchronous on `stream`: no host synchronisation, no
 *    device->host reads (reference contract: spmv never fences,
 *    sparse/unit_test/Test_Sparse_spmv.hpp:193-194).  SpGEMM symbolic is
 *    synchronous by nature (the caller needs c_nnz to allocate C).
 *  - A plan belongs to ONE matrix (same rule as SPMVHandle,
 *    sparse/src/KokkosSparse_spmv_handle.hpp:276-277) and is not thread-safe;
 *    distinct plans on distinct streams may run concurrently.
 */
#ifndef B200SPARSE_H_
#define B200SPARSE_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  B200SP_OK = 0,
  B200SP_ERR_INVALID_ARGUMENT = 1, /* bad mode / negative size / null pointer    */
  B200SP_ERR_CUDA = 2,             /* a CUDA runtime call failed                  */
  B200SP_ERR_STATE = 3,            /* numeric before symbolic, plan/matrix mismatch */
  B200SP_ERR_OVERFLOW = 4,         /* nnz(C) does not fit int32 offsets           */
  B200SP_ERR_ALLOC = 5
} b200sp_status;

/* Mirrors KokkosSparse::SPMVAlgorithm for the values that reach a TPL
 * (sparse/src/KokkosSparse_spmv_handle.hpp:32-47,76-86); SPMV_NATIVE* never
 * get here. */
typedef enum {
  B200SP_SPMV_DEFAULT = 0,    /* SPMV_DEFAULT: analyse once, TMA-tiled kernel        */
  B200SP_SPMV_FAST_SETUP = 1, /* SPMV_FAST_SETUP: no analysis, row-vector kernel     */
  B200SP_SPMV_MERGE_PATH = 2  /* SPMV_MERGE_PATH: same kernels as DEFAULT (tiles are nnz-balanced; rows beyond the tile
                                 row limit go to a long-row kernel, optionally split into segments)        */
} b200sp_spmv_algo;

typedef struct b200sp_spmv_plan b200sp_spmv_plan;     /* lives in SPMVHandle::tpl_rank1 / tpl_rank2 */
typedef struct b200sp_spgemm_plan b200sp_spgemm_plan; /* lives in SPGEMMHandle (like cuSparseSpgemmHandleType,
                                                         sparse/src/KokkosSparse_spgemm_handle.hpp:161-198) */

const char* b200sp_last_error_string(void);
int b200sp_version(void);
/* 1 when a CUDA device of compute capability 9.x (H100, sm_90a) is current, else 0. */
int b200sp_device_ok(void);

/* ---- SpMV plan ---------------------------------------------------------- */
/* Replaces CuSparse10_SpMV_Data creation
 * (sparse/tpls/KokkosSparse_spmv_tpl_spec_decl.hpp:107-133).  The analysis
 * itself happens lazily, stream-ordered, on the first spmv call. */
int b200sp_spmv_plan_create(b200sp_spmv_plan** plan, int algo);
/* Frees device state with cudaFreeAsync on `stream` (safe without a user
 * fence, like TPL_SpMV_Data's destructor, spmv_handle.hpp:116-128). */
int b200sp_spmv_plan_destroy(b200sp_spmv_plan* plan, void* stream);

/* Plan options.  B200SP_SPMV_OPT_CACHE_TRANSPOSE (default 0): modes T / H run through an explicit
 * transpose kept in the plan (structure built once per matrix with b200sp_transpose's kernels, values
 * re-gathered on every call, then the non-transposed kernel): deterministic, no atomics, at the price
 * of 8 bytes/entry of structure + sizeof(S) bytes/entry of values.  Without it T / H use atomicAdd
 * scatters like the reference's GPU path (sparse/impl/KokkosSparse_spmv_impl.hpp:36-84). */
#define B200SP_SPMV_OPT_CACHE_TRANSPOSE 1
/* B200SP_SPMV_OPT_HOSTVEC_DEFER (default 0), for b200sp_spmv_hostvec_*: a call no longer makes `stream` wait for its own
 * download of y, so the next call's kernel runs while this call's y is still on its way to the host (upload of call k+1,
 * compute of call k+1 and download of call k all overlap: the step time tends to the slowest of the three instead of
 * compute + download).  The price is the completion rule: y_host of ALL calls issued so far is valid only after
 * b200sp_spmv_hostvec_flush(plan, stream) followed by a synchronisation of `stream`; calls in flight must not depend on
 * each other's y_host (beta != 0 reads y_host at call time). */
#define B200SP_SPMV_OPT_HOSTVEC_DEFER 2
int b200sp_spmv_plan_set_option(b200sp_spmv_plan* plan, int option, int value);

/* ---- SpMV rank-1: y = beta*y + alpha*op(A)*x ---------------------------- */
/* Replaces SPMV<Kokkos::Cuda,...,true>::spmv -> spmv_cusparse
 * (sparse/tpls/KokkosSparse_spmv_tpl_spec_decl.hpp:31-225) and, without the
 * cuSPARSE guards of sparse/src/KokkosSparse_spmv.hpp:230-241, accepts all four
 * modes: 'N','C' (== N for real scalars), 'T','H' (== T).  m x n is A's shape;
 * x has n (N/C) or m (T/H) entries, y the other.  beta == 0 never reads y
 * (NaN in y is overwritten, Test_Sparse_spmv.hpp:394-408).  alpha == 0 or an
 * empty A reduces to y = beta*y (KokkosSparse_spmv.hpp:145-154).
 * plan may be NULL (row-vector kernel, nothing cached). */
int b200sp_spmv_f64_i32(b200sp_spmv_plan* plan, void* stream, char mode, int m, int n, int64_t nnz,
                        double alpha, const int* row_ptr, const int* col_idx, const double* vals,
                        const double* x, double beta, double* y);
int b200sp_spmv_f32_i32(b200sp_spmv_plan* plan, void* stream, char mode, int m, int n, int64_t nnz,
                        float alpha, const int* row_ptr, const int* col_idx, const float* vals,
                        const float* x, float beta, float* y);

/* ---- SpMV on 64-bit offsets (matrices past 2^31 entries) ----------------- */
/* Replaces the (int64_t ordinal, size_t offset) instantiations of the cuSPARSE SpMV slot,
 * KOKKOSSPARSE_SPMV_CUSPARSE(double|float, int64_t, size_t, ...)
 * (sparse/tpls/KokkosSparse_spmv_tpl_spec_decl.hpp:246-257, availability ..._spec_avail.hpp:85-102), and also takes
 * 32-bit columns under 64-bit offsets (col_bits = 32), which that slot cannot (:86).  row_ptr has m+1 int64 entries
 * (size_t offsets below 2^63 read the same); col_idx is const int32_t* or const int64_t* by col_bits.  m and n must
 * stay below 2^31 and no row may hold more than the window limit (about 2^31 entries): B200SP_ERR_OVERFLOW otherwise,
 * also when a 64-bit column index does not fit 31 bits.  Semantics of mode / alpha / beta as b200sp_spmv_f64_i32.
 * The plan is required: on the first call with a matrix (keyed on the array pointers, m, n, nnz) it reads the 64-bit
 * structure ONCE -- rows are cut into windows of < 2^31 entries, each with a 32-bit row map relative to its first entry
 * (4 B per row), 64-bit columns are narrowed to 32 bits (4 B per entry; 32-bit columns are used in place) -- and every
 * product then runs the 32-bit kernels window by window: 12 B of HBM traffic per fp64 entry instead of the 16 B a kernel
 * reading 64-bit columns would move, results bit-identical to the 32-bit entry points' on each window.  The analysis
 * synchronises `stream` once. */
typedef struct b200sp_spmv64_plan b200sp_spmv64_plan;
int b200sp_spmv64_plan_create(b200sp_spmv64_plan** plan, int algo);
int b200sp_spmv64_plan_destroy(b200sp_spmv64_plan* plan, void* stream);
/* Entries per window, 8 .. 2^31-65537 (the default); smaller windows only make sense for tests. */
int b200sp_spmv64_plan_set_window(b200sp_spmv64_plan* plan, int64_t max_entries);
int b200sp_spmv64_plan_windows(const b200sp_spmv64_plan* plan);
const char* b200sp_spmv64_last_kernel(const b200sp_spmv64_plan* plan);
int b200sp_spmv_f64_i64(b200sp_spmv64_plan* plan, void* stream, char mode, int64_t m, int64_t n, int64_t nnz,
                        double alpha, const int64_t* row_ptr, const void* col_idx, int col_bits, const double* vals,
                        const double* x, double beta, double* y);
int b200sp_spmv_f32_i64(b200sp_spmv64_plan* plan, void* stream, char mode, int64_t m, int64_t n, int64_t nnz,
                        float alpha, const int64_t* row_ptr, const void* col_idx, int col_bits, const float* vals,
                        const float* x, float beta, float* y);

/* Rank 2 on the same plan and windows (arguments as b200sp_spmm_f64_i32, declared below). */
int b200sp_spmm_f64_i64(b200sp_spmv64_plan* plan, void* stream, char mode, int64_t m, int64_t n, int64_t nnz, int k,
                        double alpha, const int64_t* row_ptr, const void* col_idx, int col_bits, const double* vals,
                        const double* X, int64_t ldx, int x_row_major, double beta, double* Y, int64_t ldy,
                        int y_row_major);
int b200sp_spmm_f32_i64(b200sp_spmv64_plan* plan, void* stream, char mode, int64_t m, int64_t n, int64_t nnz, int k,
                        float alpha, const int64_t* row_ptr, const void* col_idx, int col_bits, const float* vals,
                        const float* X, int64_t ldx, int x_row_major, float beta, float* Y, int64_t ldy,
                        int y_row_major);

/* Same call with HOST x / y (pinned or pageable): x is copied to the device,
 * y (when beta != 0) too, the kernel runs, y is copied back; all on `stream`.
 * The matrix arrays stay device-resident.  Requires a plan (owns the device
 * staging vectors).  This is the end-to-end path bench.py times as `e2e`. */
int b200sp_spmv_hostvec_f64_i32(b200sp_spmv_plan* plan, void* stream, char mode, int m, int n,
                                int64_t nnz, double alpha, const int* row_ptr, const int* col_idx,
                                const double* vals, const double* x_host, double beta,
                                double* y_host);

/* Deferred mode (B200SP_SPMV_OPT_HOSTVEC_DEFER) only: makes `stream` wait for every download issued so far. */
int b200sp_spmv_hostvec_flush(b200sp_spmv_plan* plan, void* stream);

/* Row-block-partitioned SpMV with the all-gather of y fused into the kernel (multi-GPU, config 5):
 * y = alpha*A*x for this rank's row block is stored to `y` AND to `n_extra` (<= 7) further device
 * pointers -- the slots of this row block inside the peers' next-x buffers, mapped into this process
 * (CUDA IPC / symmetric memory) -- with plain P2P stores from the SpMV kernel itself, so the NVLink
 * transfer overlaps the compute row by row.  No reference counterpart (the reference is single-process,
 * README.md:12-16); result identical to b200sp_spmv_f64_i32 + all-gather.  beta is 0.  The caller
 * synchronises the ranks between steps (bench.py uses the symmetric-memory barrier). */
int b200sp_spmv_scatter_f64_i32(b200sp_spmv_plan* plan, void* stream, int m, int n, int64_t nnz, double alpha,
                                const int* row_ptr, const int* col_idx, const double* vals, const double* x,
                                double* y, int n_extra, void* const* y_extra);

/* The same product with ONE further destination fed tile by tile: the kernel's producer warp (the one that streams the matrix
 * with TMA) copies every finished tile of y from the local slice to `y_forward` (same indexing as y) with coalesced stores --
 * 256 contiguous bytes per instruction instead of one 8-byte store per row.  Meant for the NVSwitch multicast mapping of the
 * symmetric next-x buffer: every y value leaves the GPU once, in whole 128-byte NVLink writes, while the rest of the shard is
 * still being computed (multigpu.py mode "multicast_fwd").  Rows the tiled kernel leaves to its helper kernels are stored to
 * y_forward by those.  Results identical to b200sp_spmv_f64_i32. */
int b200sp_spmv_forward_f64_i32(b200sp_spmv_plan* plan, void* stream, int m, int n, int64_t nnz, double alpha,
                                const int* row_ptr, const int* col_idx, const double* vals, const double* x,
                                double* y, void* y_forward);

/* Copy `bytes` from device pointer src to n_dst device pointers (peer GPUs' buffers mapped into this
 * process) with copy-engine transfers on `stream` -- the push half of the pipelined row-block SpMV
 * (kokkos-kernels_b200/multigpu.py): chunk c of y is pushed over NVLink while chunk c+1 is computed. */
int b200sp_peer_push(void* stream, const void* src, int64_t bytes, int n_dst, void* const* dsts);
/* Same, one copy per communication stream (n_dst streams), each ordered after everything enqueued on
 * compute_stream so far; b200sp_peer_join makes compute_stream wait for all of them. */
int b200sp_peer_push_async(void* compute_stream, void* const* comm_streams, int n_dst, void* const* dsts,
                           const void* src, int64_t bytes);
int b200sp_peer_join(void* compute_stream, void* const* comm_streams, int n);

/* Copy `bytes` (multiple of 8) from src to the NVSwitch multicast mapping `mc_dst` of a symmetric buffer with
 * 16-byte stores from `ctas` CTAs (default 16) on `stream`: the switch replicates every store into all
 * participating GPUs' copies, so a row block's y leaves its GPU once instead of once per peer.  src and mc_dst
 * must share their 16-byte phase.  The SM-driven counterpart of b200sp_peer_push_async for the pipelined
 * row-block SpMV (multigpu.py mode "pipelined_mc"); no reference counterpart. */
int b200sp_multicast_push(void* stream, const void* src, void* mc_dst, int64_t bytes, int ctas);
/* ctas > 0: multimem.st (16-byte) from `ctas` CTAs of 128 threads (0: 32); ctas < 0: plain stores from |ctas| CTAs. */

/* SM-driven unicast push: `bytes` (multiple of 8) from src to the same offset of n_dst (<= 8) peer buffers with 16-byte P2P
 * stores from `ctas` small CTAs (default 32) on `stream`; every 16 bytes are read once.  The SM counterpart of the copy-engine
 * b200sp_peer_push_async (multigpu.py mode "pipelined_sm"); src and the destinations share their 16-byte phase. */
int b200sp_peer_push_sm(void* stream, const void* src, int64_t bytes, int n_dst, void* const* dsts, int ctas);

/* ---- SpMV rank-2 (multivector): Y = beta*Y + alpha*op(A)*X, k columns --- */
/* Replaces SPMV_MV<Kokkos::Cuda,...,false,true>::spmv_mv -> cusparseSpMM
 * (sparse/tpls/KokkosSparse_spmv_mv_tpl_spec_decl.hpp:97-225).
 * X(i,j) = X[i*ldx + j] when x_row_major (Kokkos::LayoutRight) else
 * X[i + j*ldx] (LayoutLeft); same for Y.  Any mix of layouts is accepted. */
int b200sp_spmm_f64_i32(b200sp_spmv_plan* plan, void* stream, char mode, int m, int n, int64_t nnz,
                        int k, double alpha, const int* row_ptr, const int* col_idx,
                        const double* vals, const double* X, int64_t ldx, int x_row_major,
                        double beta, double* Y, int64_t ldy, int y_row_major);
int b200sp_spmm_f32_i32(b200sp_spmv_plan* plan, void* stream, char mode, int m, int n, int64_t nnz,
                        int k, float alpha, const int* row_ptr, const int* col_idx,
                        const float* vals, const float* X, int64_t ldx, int x_row_major,
                        float beta, float* Y, int64_t ldy, int y_row_major);
/* Half precision (Kokkos::Experimental::half_t, the reference's cusparseSpMM slot with an fp32 compute type,
 * sparse/tpls/KokkosSparse_spmv_mv_tpl_spec_decl.hpp:47-61): vals, X and Y hold IEEE binary16 bit patterns.
 *  - Every product a*x is formed in fp32, where it is exact (two 11-bit significands; even 2^-24 * 2^-24 is an fp32
 *    normal).  Products are accumulated in fp32; rows cut into several pieces keep their partial sums in fp32.
 *  - The epilogue beta*y + alpha*acc is evaluated in fp32 and rounded ONCE to binary16, to nearest even; a result
 *    beyond +-65504 becomes +-inf.  Intermediate sums may exceed the fp16 range without harm.
 *  - alpha and beta are used as given (the Kokkos shim converts half_t to float exactly).
 *  - Modes N == C, T == H.  beta == 0 never reads Y (NaN in Y is overwritten); alpha == 0 or an empty A gives
 *    Y = beta*Y.  Any mix of layouts is accepted.
 * Mode N with a plan and row-major X and Y runs the item kernels (16-byte loads of 8 halves when k, ldx and ldy are
 * multiples of 8 and X and Y are 16-byte aligned); LayoutLeft operands with a plan and k >= 4 go through row-major
 * copies; without a plan, or LayoutLeft with k < 4, one thread per (row, column) computes the entry.  On those item paths
 * the result has the same bits as b200sp_spmm_f32_i32 on the widened inputs, rounded to binary16.  T / H add the exact
 * products into a zeroed fp32 scratch (the plan's, or a stream-ordered temporary without a plan) with atomics and round
 * each entry once.  B200SP_SPMM_KERNEL (row / split / tile) does not apply to this entry point. */
int b200sp_spmm_f16_i32(b200sp_spmv_plan* plan, void* stream, char mode, int m, int n, int64_t nnz, int k, float alpha,
                        const int* row_ptr, const int* col_idx, const uint16_t* vals, const uint16_t* X, int64_t ldx,
                        int x_row_major, float beta, uint16_t* Y, int64_t ldy, int y_row_major);

/* ---- SpGEMM: C = A*B, A is m x n, B is n x k ---------------------------- */
int b200sp_spgemm_plan_create(b200sp_spgemm_plan** plan);
int b200sp_spgemm_plan_destroy(b200sp_spgemm_plan* plan, void* stream);

/* Replaces SPGEMM_SYMBOLIC<...,true,*>::spgemm_symbolic -> spgemm_symbolic_cusparse
 * (sparse/tpls/KokkosSparse_spgemm_symbolic_tpl_spec_decl.hpp:51-167,316-363).
 * Always writes all m+1 entries of row_ptr_C (it arrives uninitialised,
 * sparse/src/KokkosSparse_spgemm.hpp:47), returns nnz(C) and the longest C row
 * (SPGEMMHandle::set_c_nnz / set_max_result_nnz).  Rows of A and B need not be
 * sorted.  Structure is purely symbolic: explicit zeros are kept.  Calling it
 * again on the same plan is idempotent (symbolic_spec.hpp:99).  Synchronises
 * `stream` (c_nnz is returned to the host).  B200SP_ERR_OVERFLOW when
 * nnz(C) > INT32_MAX (symbolic_tpl_spec_decl.hpp:131-133). */
int b200sp_spgemm_symbolic_i32(b200sp_spgemm_plan* plan, void* stream, int m, int n, int k,
                               const int* row_ptr_A, const int* col_idx_A, const int* row_ptr_B,
                               const int* col_idx_B, int* row_ptr_C, int64_t* c_nnz,
                               int* c_max_row_nnz);

/* Replaces SPGEMM_NUMERIC<...,true,*>::spgemm_numeric -> spgemm_numeric_cusparse
 * (sparse/tpls/KokkosSparse_spgemm_numeric_tpl_spec_decl.hpp:44-256).
 * Fills col_idx_C / vals_C for the row_ptr_C symbolic produced; every C row
 * comes out SORTED by column (TPL contract; the native path sorts afterwards,
 * sparse/impl/KokkosSparse_spgemm_numeric_spec.hpp:138-140).  Re-runnable with
 * new value pointers on the same structure (Test_Sparse_spgemm.hpp:112-122).
 * B200SP_ERR_STATE when symbolic was not called on this plan
 * (numeric_spec.hpp:116-118).  Asynchronous on `stream`. */
int b200sp_spgemm_numeric_f64_i32(b200sp_spgemm_plan* plan, void* stream, int m, int n, int k,
                                  const int* row_ptr_A, const int* col_idx_A, const double* vals_A,
                                  const int* row_ptr_B, const int* col_idx_B, const double* vals_B,
                                  const int* row_ptr_C, int* col_idx_C, double* vals_C);
int b200sp_spgemm_numeric_f32_i32(b200sp_spgemm_plan* plan, void* stream, int m, int n, int k,
                                  const int* row_ptr_A, const int* col_idx_A, const float* vals_A,
                                  const int* row_ptr_B, const int* col_idx_B, const float* vals_B,
                                  const int* row_ptr_C, int* col_idx_C, float* vals_C);

/* spgemm_jacobi (sparse/src/KokkosSparse_spgemm_jacobi.hpp:25-190; native kernels
 * sparse/impl/KokkosSparse_spgemm_jacobi_{sparseacc,denseacc,seq}_impl.hpp): C = (I - omega * diag(dinv) * A) * B
 * = B - omega*dinv_i*(A*B)_i row by row, on the structure spgemm_symbolic computed for A*B with the same plan (A is
 * square and holds its diagonal, so that row i of B lies inside the pattern of row i of A*B -- the reference's
 * kernels assume the same; rows that violate it are completed without writing past their extent).  dinv has m
 * entries (the reference passes an m x 1 view).  C rows come out sorted.  B200SP_ERR_STATE without a prior
 * symbolic.  Asynchronous on `stream`. */
int b200sp_spgemm_jacobi_f64_i32(b200sp_spgemm_plan* plan, void* stream, int m, int n, int k,
                                 const int* row_ptr_A, const int* col_idx_A, const double* vals_A,
                                 const int* row_ptr_B, const int* col_idx_B, const double* vals_B,
                                 const int* row_ptr_C, int* col_idx_C, double* vals_C, double omega,
                                 const double* dinv);
int b200sp_spgemm_jacobi_f32_i32(b200sp_spgemm_plan* plan, void* stream, int m, int n, int k,
                                 const int* row_ptr_A, const int* col_idx_A, const float* vals_A,
                                 const int* row_ptr_B, const int* col_idx_B, const float* vals_B,
                                 const int* row_ptr_C, int* col_idx_C, float* vals_C, float omega,
                                 const float* dinv);

/* Block SpGEMM numeric: replaces Impl::BSPGEMM_NUMERIC (native KokkosBSPGEMM + sort_bsr_matrix,
 * sparse/impl/KokkosSparse_bspgemm_numeric_spec.hpp:113-191).  A is mb x nb blocks, B is nb x kb blocks, all
 * bs x bs and row-major within the block; row_ptr_C is what b200sp_spgemm_symbolic_i32 wrote on the same plan for
 * the BLOCK graphs (block symbolic is point symbolic, sparse/src/KokkosSparse_spgemm.hpp:77-103).  col_idx_C comes
 * out sorted in every block row; vals_C holds nnz(C) * bs * bs values.  Entry (r, c) of block C(i, j) is one chain
 * from +0.0 over the products of block row i in ordinal order (A's row in storage order, each B row in storage
 * order) and, within a product, over p = 0..bs-1: acc = acc + a(r,p) * b(p,c), every multiply and add rounded on
 * its own -- bit-identical to bspgemm_debug_numeric (sparse/impl/KokkosSparse_bspgemm_impl_seq.hpp:39-130) built
 * without FMA contraction.  Rows need not be sorted; explicit zero blocks are kept.  bs == 1 forwards to
 * b200sp_spgemm_numeric_*.  B200SP_ERR_INVALID_ARGUMENT for bs < 1, negative sizes or null arrays;
 * B200SP_ERR_STATE without a prior symbolic.  The first call on a plan groups the block rows by product count
 * (synchronises once); later calls with new value pointers on the same structure are asynchronous on `stream`. */
int b200sp_bspgemm_numeric_f64_i32(b200sp_spgemm_plan* plan, void* stream, int mb, int nb, int kb, int bs,
                                   const int* row_ptr_A, const int* col_idx_A, const double* vals_A,
                                   const int* row_ptr_B, const int* col_idx_B, const double* vals_B,
                                   const int* row_ptr_C, int* col_idx_C, double* vals_C);
int b200sp_bspgemm_numeric_f32_i32(b200sp_spgemm_plan* plan, void* stream, int mb, int nb, int kb, int bs,
                                   const int* row_ptr_A, const int* col_idx_A, const float* vals_A,
                                   const int* row_ptr_B, const int* col_idx_B, const float* vals_B,
                                   const int* row_ptr_C, int* col_idx_C, float* vals_C);

/* ---- SpGEMM on 64-bit offsets (products past 2^31 entries) -------------- */
/* Replaces the (int ordinal, size_t offset) instantiations of SPGEMM_SYMBOLIC / SPGEMM_NUMERIC, Kokkos' default offsets
 * in a Trilinos build (cmake/kokkoskernels_eti_offsets.cmake:1-11), which the cuSPARSE slot cannot take
 * (sparse/tpls/KokkosSparse_spgemm_numeric_tpl_spec_avail.hpp:38-41).  row_ptr_A / row_ptr_B / row_ptr_C have m+1 /
 * n+1 / m+1 int64 entries (size_t offsets below 2^63 read the same); column indices stay int32.  Any nnz(A) and nnz(C);
 * nnz(B) must not exceed 2^31-65537 (every window reads all of B; B200SP_ERR_OVERFLOW, naming B), nor may one row of A
 * hold more entries or products than the window limit (B200SP_ERR_OVERFLOW).  m, n, k and each row's entries stay below 2^31, as on the 32-bit path.
 * Symbolic reads the 64-bit structure once: B's row map is narrowed to int32 (4 B per row of B), the rows of A are cut
 * into at most 4096 windows of consecutive rows holding at most `limit` products and entries (an int64 scan and a
 * search), and every window runs b200sp_spgemm_symbolic_i32 on a child plan with a row map relative to its first entry
 * (4 B per row of A) and keeps its relative C row map (4 B per row of C).  Otherwise the contract is that of
 * b200sp_spgemm_symbolic_i32: all m+1 entries of row_ptr_C are written, c_nnz is the sum over the windows and
 * c_max_row_nnz the maximum, one handle serves one product (B200SP_ERR_STATE for another, also for a plan whose
 * symbolic had 32-bit offsets; the same product again is idempotent), synchronises `stream`. */
int b200sp_spgemm_symbolic_i64(b200sp_spgemm_plan* plan, void* stream, int m, int n, int k,
                               const int64_t* row_ptr_A, const int* col_idx_A, const int64_t* row_ptr_B,
                               const int* col_idx_B, int64_t* row_ptr_C, int64_t* c_nnz, int* c_max_row_nnz);
/* Numeric on the windows symbolic cut: b200sp_spgemm_numeric_*_i32 per window on the relative row maps and on
 * col_idx / vals of A and C shifted by the window's first entry.  Each row runs the kernel the 32-bit entry points run it
 * on: row map and columns equal theirs, and so do the values, bit for bit, of every row of at most 8192 products (and
 * 4096 entries of A).  Longer rows go to hash kernels that add with atomics on the GPU, so their values may differ in
 * the last bits from one run to the next, on either path.  Asynchronous on `stream`, re-runnable with new value
 * pointers.  B200SP_ERR_STATE when the plan's symbolic had 32-bit offsets or was not called; conversely the 32-bit
 * numeric, spgemm_jacobi and block numeric entries return B200SP_ERR_STATE on a plan whose symbolic had 64-bit offsets
 * (spgemm_jacobi and block SpGEMM are not provided on 64-bit offsets). */
int b200sp_spgemm_numeric_f64_i64(b200sp_spgemm_plan* plan, void* stream, int m, int n, int k,
                                  const int64_t* row_ptr_A, const int* col_idx_A, const double* vals_A,
                                  const int64_t* row_ptr_B, const int* col_idx_B, const double* vals_B,
                                  const int64_t* row_ptr_C, int* col_idx_C, double* vals_C);
int b200sp_spgemm_numeric_f32_i64(b200sp_spgemm_plan* plan, void* stream, int m, int n, int k,
                                  const int64_t* row_ptr_A, const int* col_idx_A, const float* vals_A,
                                  const int64_t* row_ptr_B, const int* col_idx_B, const float* vals_B,
                                  const int64_t* row_ptr_C, int* col_idx_C, float* vals_C);
/* Window limit of the next 64-bit symbolic on this plan: products and entries of A per window, 8 .. 2^31-65537 (the
 * default); smaller limits only make sense for tests.  _windows: the windows of the last 64-bit symbolic (0 for none). */
int b200sp_spgemm_plan_set_window(b200sp_spgemm_plan* plan, int64_t max_entries);
int b200sp_spgemm_plan_windows(const b200sp_spgemm_plan* plan);

/* ---- CrsMatrix utilities either side of the hot path (SURVEY.md section 8f) ----------------- */
/* sort_crs_matrix / sort_crs_graph (sparse/src/KokkosSparse_SortCrs.hpp:43-120,209-270): every row
 * sorted ascending by column, values permuted along, IN PLACE.  The sort is stable (entries with the
 * same column keep their order), which is what the reference's Serial/OpenMP path -- a per-row LSD
 * radix sort, common/src/KokkosKernels_Sorting.hpp:301-380 -- produces.  vals may be NULL (graph).
 * Rows that are already sorted are only read.  Synchronises `stream` once. */
int b200sp_sort_crs_f64_i32(void* stream, int m, const int* row_ptr, int* col_idx, double* vals);
int b200sp_sort_crs_f32_i32(void* stream, int m, const int* row_ptr, int* col_idx, float* vals);
int b200sp_sort_crs_graph_i32(void* stream, int m, const int* row_ptr, int* col_idx);

/* sort_and_merge_matrix / _graph (SortCrs.hpp:303-380,426-491) in two calls because the caller owns
 * the output: _count sorts the input in place (as the reference does, :336), writes the merged row
 * map (m+1 entries; for m == 0 a single 0 when row_ptr_out is non-NULL) and returns the merged
 * nnz; if that equals nnz(in) nothing is merged and the caller may alias the input (:346-360).
 * _fill writes merged entries / values; duplicates are summed in storage order of the sorted row
 * (MatrixMergedEntriesFunctor, sparse/impl/KokkosSparse_sort_crs_impl.hpp:163-205).  vals NULL = graph. */
int b200sp_sort_and_merge_count_f64_i32(void* stream, int m, const int* row_ptr, int* col_idx, double* vals,
                                        int* row_ptr_out, int64_t* merged_nnz);
int b200sp_sort_and_merge_count_f32_i32(void* stream, int m, const int* row_ptr, int* col_idx, float* vals,
                                        int* row_ptr_out, int64_t* merged_nnz);
int b200sp_sort_and_merge_fill_f64_i32(void* stream, int m, const int* row_ptr, const int* col_idx,
                                       const double* vals, const int* row_ptr_out, int* col_idx_out,
                                       double* vals_out);
int b200sp_sort_and_merge_fill_f32_i32(void* stream, int m, const int* row_ptr, const int* col_idx,
                                       const float* vals, const int* row_ptr_out, int* col_idx_out,
                                       float* vals_out);

/* transpose_matrix / transpose_graph (sparse/src/KokkosSparse_Utils.hpp:245-450): A is m x n, the
 * transpose n x m; t_row_ptr has n+1 entries and is fully written.  Every transposed row lists its
 * entries in (row of A, position in that row) order -- the order of the reference's Serial loop; its
 * parallel back ends fill with atomics and leave the order unspecified.  vals / t_vals NULL = graph.
 * Synchronises `stream`. */
int b200sp_transpose_f64_i32(void* stream, int m, int n, const int* row_ptr, const int* col_idx,
                             const double* vals, int* t_row_ptr, int* t_col_idx, double* t_vals);
int b200sp_transpose_f32_i32(void* stream, int m, int n, const int* row_ptr, const int* col_idx,
                             const float* vals, int* t_row_ptr, int* t_col_idx, float* t_vals);

/* spadd: C = alpha*A + beta*B, A, B, C all m x n (sparse/src/KokkosSparse_spadd.hpp:29-319).
 * The plan is the SPADDHandle (sparse/src/KokkosSparse_spadd_handle.hpp:24-137): input_sorted /
 * input_merged as given to create_spadd_handle; for unsorted input it keeps a_pos / b_pos between the
 * two phases (:73-84).  Symbolic fills row_ptr_C (m+1 entries, arrives uninitialised) and returns
 * nnz(C) (synchronous); numeric fills col_idx_C / vals_C: sorted input -> merged, sorted rows
 * (SortedNumericSumFunctor, spadd_numeric_impl.hpp:27-107); unsorted input -> rows in the order of
 * the sorted union, values accumulated A first then B (UnsortedNumericSumFunctor, :109-171).  Same
 * operation order as the reference's one-thread-per-row functors: results are bit-identical to its
 * Serial path.  B200SP_ERR_STATE when numeric precedes symbolic. */
typedef struct b200sp_spadd_plan b200sp_spadd_plan;
int b200sp_spadd_plan_create(b200sp_spadd_plan** plan, int input_sorted, int input_merged);
int b200sp_spadd_plan_destroy(b200sp_spadd_plan* plan, void* stream);
int b200sp_spadd_symbolic_i32(b200sp_spadd_plan* plan, void* stream, int m, int n, const int* row_ptr_A,
                              const int* col_idx_A, const int* row_ptr_B, const int* col_idx_B,
                              int* row_ptr_C, int64_t* c_nnz);
int b200sp_spadd_numeric_f64_i32(b200sp_spadd_plan* plan, void* stream, int m, int n, const int* row_ptr_A,
                                 const int* col_idx_A, const double* vals_A, double alpha,
                                 const int* row_ptr_B, const int* col_idx_B, const double* vals_B,
                                 double beta, const int* row_ptr_C, int* col_idx_C, double* vals_C);
int b200sp_spadd_numeric_f32_i32(b200sp_spadd_plan* plan, void* stream, int m, int n, const int* row_ptr_A,
                                 const int* col_idx_A, const float* vals_A, float alpha,
                                 const int* row_ptr_B, const int* col_idx_B, const float* vals_B,
                                 float beta, const int* row_ptr_C, int* col_idx_C, float* vals_C);

/* ---- matrix files (host side; SURVEY.md section 8f rank 2) ---------------------------------- */
/* read_kokkos_crst_matrix (sparse/src/KokkosSparse_IOUtils.hpp:1237-1290): MatrixMarket (.mtx, .mm;
 * read_mtx with symmetrize = remove_diagonal = transpose = false, :784-996 -- coordinate or array,
 * real / integer / pattern, general / symmetric / skew-symmetric / hermitian; rows come out sorted,
 * symmetric files are expanded) or the raw binary CRS dump (.bin, read_graph_bin :680-695; no column
 * count in the file: ncols = largest column + 1).  The three arrays are HOST memory allocated by the
 * library: release each with b200sp_host_free.  Harwell-Boeing files are not supported. */
int b200sp_read_crs_f64(const char* path, int* m, int* n, int64_t* nnz, int** row_ptr, int** col_idx, double** vals);
int b200sp_read_crs_f32(const char* path, int* m, int* n, int64_t* nnz, int** row_ptr, int** col_idx, float** vals);
/* read_mtx with its three options (IOUtils.hpp:785-786). */
int b200sp_read_mtx_f64(const char* path, int symmetrize, int remove_diagonal, int transpose, int* m, int* n,
                        int64_t* nnz, int** row_ptr, int** col_idx, double** vals);
int b200sp_read_mtx_f32(const char* path, int symmetrize, int remove_diagonal, int transpose, int* m, int* n,
                        int64_t* nnz, int** row_ptr, int** col_idx, float** vals);
/* write_kokkos_crst_matrix (IOUtils.hpp:740-782): .mtx / .mm (write_matrix_mtx, 17 significant digits) or
 * .bin (write_graph_bin; square matrices only, like the reference).  HOST arrays. */
int b200sp_write_crs_f64(const char* path, int m, int n, int64_t nnz, const int* row_ptr, const int* col_idx,
                         const double* vals);
int b200sp_write_crs_f32(const char* path, int m, int n, int64_t nnz, const int* row_ptr, const int* col_idx,
                         const float* vals);
void b200sp_host_free(void* p);

/* ---- BsrMatrix SpMV / SpMM (SURVEY.md 8f rank 3) --------------------------------------------------
 * Replaces SPMV_BSRMATRIX<Kokkos::Cuda, ..., tpl = true>::spmv_bsrmatrix -> spmv_bsr_cusparse
 * (sparse/tpls/KokkosSparse_spmv_bsrmatrix_tpl_spec_decl.hpp:279-352,469-493) and
 * SPMV_MV_BSRMATRIX<...>::spmv_mv_bsrmatrix -> spmv_mv_bsr_cusparse (:372-455,522-546), plus the native
 * functors the front end falls back to for the modes cuSPARSE lacks (KokkosSparse_spmv.hpp:322-375;
 * sparse/impl/KokkosSparse_spmv_bsrmatrix_impl_v42.hpp, ..._impl.hpp:707-834).
 *
 * A is mb x nb blocks of bs x bs (BsrMatrix, sparse/src/KokkosSparse_BsrMatrix.hpp:355-370): row_ptr has
 * mb+1 entries, col_idx nnzb block columns, vals nnzb*bs*bs values with every block row-major.
 * y = beta*y + alpha*op(A)*x, op by mode 'N','C' (= N for real scalars),'T','H' (= T); beta == 0 overwrites y
 * (NaN-safe), alpha == 0 only scales.  Unlike the cuSPARSE leg every mode and bs == 1 are accepted (bs == 1 is
 * forwarded to the CrsMatrix path as the reference's front end does, KokkosSparse_spmv.hpp:169-185).
 * The plan caches the tile analysis of the last block structure (keyed on row_ptr, mb, nnzb, bs), i.e. what
 * SPMVHandle::tpl_rank1 / tpl_rank2 hold for cuSPARSE; one plan per matrix, like the handle.
 * Errors: B200SP_ERR_INVALID_ARGUMENT for bs < 1 (BsrMatrix.hpp:429-433), an unknown mode, null arrays,
 * dimensions beyond int32.  Asynchronous on `stream`. */
typedef struct b200sp_bsr_plan b200sp_bsr_plan;
int b200sp_bsr_plan_create(b200sp_bsr_plan** plan);
int b200sp_bsr_plan_destroy(b200sp_bsr_plan* plan, void* stream);
int b200sp_bsr_spmv_f64_i32(b200sp_bsr_plan* plan, void* stream, char mode, int mb, int nb, int64_t nnzb, int bs,
                            double alpha, const int* row_ptr, const int* col_idx, const double* vals,
                            const double* x, double beta, double* y);
int b200sp_bsr_spmv_f32_i32(b200sp_bsr_plan* plan, void* stream, char mode, int mb, int nb, int64_t nnzb, int bs,
                            float alpha, const int* row_ptr, const int* col_idx, const float* vals,
                            const float* x, float beta, float* y);
/* k columns; X is (cols of op(A)) x k, Y is (rows of op(A)) x k; ld* = leading dimension in elements, *_row_major
 * as for b200sp_spmm_* (LayoutRight = 1, LayoutLeft = 0; the cuSPARSE leg takes LayoutLeft only, decl:365-371). */
int b200sp_bsr_spmm_f64_i32(b200sp_bsr_plan* plan, void* stream, char mode, int mb, int nb, int64_t nnzb, int bs, int k,
                            double alpha, const int* row_ptr, const int* col_idx, const double* vals,
                            const double* X, int64_t ldx, int x_row_major, double beta, double* Y, int64_t ldy,
                            int y_row_major);
int b200sp_bsr_spmm_f32_i32(b200sp_bsr_plan* plan, void* stream, char mode, int mb, int nb, int64_t nnzb, int bs, int k,
                            float alpha, const int* row_ptr, const int* col_idx, const float* vals, const float* X,
                            int64_t ldx, int x_row_major, float beta, float* Y, int64_t ldy, int y_row_major);
/* Name of the kernel the plan's last call used; static storage (tests / bench). */
const char* b200sp_bsr_last_kernel(const b200sp_bsr_plan* plan);
/* The handle's algorithm (sparse/src/KokkosSparse_spmv_handle.hpp: SPMV_BSR_V41 / V42 / TC).  For no-transpose multivector
 * products in double with 2 <= bs <= 16 there are two kernels: the mma.sync m8n8k4 kernel -- what SPMV_BSR_TC selects in the
 * reference (sparse/impl/KokkosSparse_spmv_bsrmatrix_spec.hpp:165-245, ..._impl.hpp:74-459: wmma fragments of the same
 * shape) -- and a scalar one.  DEFAULT picks the tensor-core kernel from 4 columns on (several times faster where measured),
 * TENSOR_CORES always, SCALAR never (SPMV_BSR_V41 / V42 requests); every other call takes the default kernels, as the
 * reference falls back when its functor is unavailable. */
#define B200SP_BSR_ALGO_DEFAULT 0
#define B200SP_BSR_ALGO_TENSOR_CORES 1
#define B200SP_BSR_ALGO_SCALAR 2
int b200sp_bsr_plan_set_algorithm(b200sp_bsr_plan* plan, int algo);

/* ---- point Gauss-Seidel (SURVEY.md 8f rank 4: the preconditioner of the reference's CG driver) ---------------------
 * gauss_seidel_symbolic / gauss_seidel_numeric / {symmetric_,forward_sweep_,backward_sweep_}gauss_seidel_apply for the point
 * (multicolour) algorithm (sparse/src/KokkosSparse_gauss_seidel.hpp:49-1100 -> PointGaussSeidel,
 * sparse/impl/KokkosSparse_gauss_seidel_impl.hpp; GS_DEFAULT of every execution space).  symbolic colours the graph of the
 * n x n matrix (is_graph_symmetric = 0: on pattern(A) + pattern(A^T)) and builds the row list of every colour set -- the
 * matrix is NOT permuted or copied; numeric extracts 1 / a_ii (B200SP_ERR_INVALID_ARGUMENT when a row has no or a zero
 * diagonal); apply runs `sweeps` sweeps over the colour sets: direction 0 = symmetric (forward then backward), 1 = forward,
 * 2 = backward; per row  sum = y_i - sum_j a_ij x_j,  x_i += omega * sum / a_ii  (PSGS::operator(), impl.hpp:159-179);
 * init_zero_x != 0 zeroes x first.  The plan is the GaussSeidelHandle's device state; B200SP_ERR_STATE when a phase is
 * called before its predecessor.  symbolic / numeric synchronise; apply is asynchronous on `stream`. */
typedef struct b200sp_gs_plan b200sp_gs_plan;
int b200sp_gs_plan_create(b200sp_gs_plan** plan);
int b200sp_gs_plan_destroy(b200sp_gs_plan* plan, void* stream);
int b200sp_gs_symbolic_i32(b200sp_gs_plan* plan, void* stream, int n, const int* row_ptr, const int* col_idx,
                           int is_graph_symmetric);
/* Same for a matrix with num_cols >= num_rows -- the local part of a distributed matrix, as Ifpack2 / MueLu hand it over:
 * columns >= num_rows address ghost entries of x, which the sweeps read and never write and which take no part in the
 * colouring (x then has num_cols entries; numeric / apply keep their signatures). */
int b200sp_gs_symbolic_nc_i32(b200sp_gs_plan* plan, void* stream, int n, int ncols, const int* row_ptr,
                              const int* col_idx, int is_graph_symmetric);
int b200sp_gs_numeric_f64_i32(b200sp_gs_plan* plan, void* stream, int n, const int* row_ptr, const int* col_idx,
                              const double* vals);
int b200sp_gs_numeric_f32_i32(b200sp_gs_plan* plan, void* stream, int n, const int* row_ptr, const int* col_idx,
                              const float* vals);
int b200sp_gs_apply_f64_i32(b200sp_gs_plan* plan, void* stream, int n, const int* row_ptr, const int* col_idx,
                            const double* vals, double* x, const double* y, int init_zero_x, double omega, int sweeps,
                            int direction);
int b200sp_gs_apply_f32_i32(b200sp_gs_plan* plan, void* stream, int n, const int* row_ptr, const int* col_idx,
                            const float* vals, float* x, const float* y, int init_zero_x, float omega, int sweeps,
                            int direction);
/* The colouring symbolic produced (device pointers owned by the plan): colour of every row, and the rows of colour c at
 * color_rows[color_ptr[c] .. color_ptr[c+1]), ascending. */
int b200sp_gs_get_coloring(const b200sp_gs_plan* plan, int* num_colors, const int** colors, const int** color_ptr,
                           const int** color_rows);
/* The same copied to host arrays of n, num_colors + 1 and n entries (NULL: skipped); synchronises `stream`. */
int b200sp_gs_copy_coloring(const b200sp_gs_plan* plan, void* stream, int* colors_host, int* color_ptr_host,
                            int* color_rows_host);

/* ---- Two-stage Gauss-Seidel (SURVEY.md 8f rank 4: the Gauss-Seidel that is a loop of SpMVs) -------------------------
 * gauss_seidel_symbolic / numeric / apply with a handle created as GS_TWOSTAGE and inner Jacobi-Richardson sweeps
 * (TwostageGaussSeidel, sparse/impl/KokkosSparse_twostage_gauss_seidel_impl.hpp: symbolic :544-697, numeric :700-772, apply
 * :778-1035; handle sparse/src/KokkosSparse_gauss_seidel_handle.hpp:513-673).  A (n x ncols, ncols >= n; columns >= n address
 * ghost entries of x, read and never written) = L + D + U on its square part.  symbolic builds L and U (and, in the compact
 * form, the complements La / Ua) in A's storage order; numeric takes D = 1 / a_ii -- or given_inverse_diagonal (n entries,
 * the reference's handle->set_diagonal... path, NULL for none) -- and scales L, U by it; apply runs
 *   max(outer sweeps, num_iter) sweeps (symmetric: each a forward then a backward one), per sweep
 *     R = B - A x                          (compact form: R = B - Ua x or La x, + (1/omega - 1) Da.*x)
 *     T = D.*R; R = gamma T;  inner sweeps:  Z = T - omega (L or U) R;  Z = gamma Z + (1 - gamma) R;  R = Z
 *     x += omega Z                         (compact form: x = omega Z)
 * with the library's SpMV for every product (plans of A, L, U, La, Ua kept in this plan) and the KokkosBlas steps in between
 * evaluated expression by expression as the reference does (nrhs > 1: the multivector products, one pass over the matrix for
 * all right-hand sides).  x: ncols x nrhs, b: n x nrhs, column-major with leading
 * dimensions ldx / ldb (LayoutLeft, the reference's default_layout on the GPU); direction 0 = symmetric, 1 = forward,
 * 2 = backward; init_zero_x != 0 zeroes x first (and skips the first residual product).  Options (before symbolic for
 * COMPACT_FORM): KokkosKernelsHandle::set_gs_twostage_compact_form / set_gs_set_num_inner_sweeps / _num_outer_sweeps /
 * _inner_damp_factor (sparse/src/KokkosKernels_Handle.hpp:639-683); defaults 0, 1, 1, 1.0.  TWO_STAGE = 0 (before symbolic) selects
 * the classic form, set_gs_twostage(false, ...): the inner sweeps are replaced by a triangular solve Z = (L + D)^{-1} R with the lower
 * (upper) triangle of A (level sets, b200sp_sptrsv below); omega must be 1 there, as in the reference (apply :886-893).
 * B200SP_ERR_INVALID_ARGUMENT when a row has no diagonal entry,
 * B200SP_ERR_STATE when a phase is called before its predecessor or with another matrix.  symbolic synchronises `stream`. */
#define B200SP_GS2_COMPACT_FORM 1
#define B200SP_GS2_NUM_INNER_SWEEPS 2
#define B200SP_GS2_NUM_OUTER_SWEEPS 3
#define B200SP_GS2_INNER_DAMP_FACTOR 4
#define B200SP_GS2_TWO_STAGE 5
typedef struct b200sp_gs2_plan b200sp_gs2_plan;
int b200sp_gs2_plan_create(b200sp_gs2_plan** plan);
int b200sp_gs2_plan_destroy(b200sp_gs2_plan* plan, void* stream);
int b200sp_gs2_plan_set(b200sp_gs2_plan* plan, int option, double value);
int b200sp_gs2_symbolic_i32(b200sp_gs2_plan* plan, void* stream, int n, int ncols, const int* row_ptr, const int* col_idx);
int b200sp_gs2_numeric_f64_i32(b200sp_gs2_plan* plan, void* stream, int n, int ncols, const int* row_ptr, const int* col_idx,
                               const double* vals, const double* given_inverse_diagonal);
int b200sp_gs2_numeric_f32_i32(b200sp_gs2_plan* plan, void* stream, int n, int ncols, const int* row_ptr, const int* col_idx,
                               const float* vals, const float* given_inverse_diagonal);
int b200sp_gs2_apply_f64_i32(b200sp_gs2_plan* plan, void* stream, int n, int ncols, const int* row_ptr, const int* col_idx,
                             const double* vals, double* x, int64_t ldx, const double* b, int64_t ldb, int nrhs,
                             int init_zero_x, double omega, int num_iter, int direction);
int b200sp_gs2_apply_f32_i32(b200sp_gs2_plan* plan, void* stream, int n, int ncols, const int* row_ptr, const int* col_idx,
                             const float* vals, float* x, int64_t ldx, const float* b, int64_t ldb, int nrhs,
                             int init_zero_x, float omega, int num_iter, int direction);

/* Sparse triangular solve x = T^{-1} b on a lower or upper triangular CrsMatrix with its diagonal stored (any position in the
 * row) -- KokkosSparse::sptrsv_symbolic / sptrsv_solve (sparse/src/KokkosSparse_sptrsv.hpp:40-170, :290-480), which the classic
 * two-stage Gauss-Seidel above calls.  symbolic groups the rows into dependency levels (synchronises `stream`; an entry on the
 * wrong side of the diagonal is B200SP_ERR_INVALID_ARGUMENT); solve runs one launch per level -- or one single-CTA launch for a
 * run of consecutive small levels (environment B200SP_SPTRSV_CHAIN=0 at symbolic time: always one per level), a group of 8 / 16 /
 * 32 lanes per row (B200SP_SPTRSV_GROUP overrides the choice) -- and computes every row as the serial substitution loop does (storage order, unfused multiply / subtract, one division):
 * bit-identical to it.  _levels / _launches: the number of dependency levels and of kernel launches of one solve. */
typedef struct b200sp_sptrsv_plan b200sp_sptrsv_plan;
int b200sp_sptrsv_plan_create(b200sp_sptrsv_plan** plan);
int b200sp_sptrsv_plan_destroy(b200sp_sptrsv_plan* plan, void* stream);
int b200sp_sptrsv_symbolic_i32(b200sp_sptrsv_plan* plan, void* stream, int n, const int* row_ptr, const int* col_idx, int is_lower);
int b200sp_sptrsv_levels(const b200sp_sptrsv_plan* plan);
int b200sp_sptrsv_launches(const b200sp_sptrsv_plan* plan);
int b200sp_sptrsv_solve_f64_i32(b200sp_sptrsv_plan* plan, void* stream, int n, const int* row_ptr, const int* col_idx,
                                const double* vals, const double* b, double* x);
int b200sp_sptrsv_solve_f32_i32(b200sp_sptrsv_plan* plan, void* stream, int n, const int* row_ptr, const int* col_idx,
                                const float* vals, const float* b, float* x);

/* ---- CG driver (SURVEY.md 8f rank 4: callers of spmv in a loop) ---------------------------------------------------
 * KokkosKernels::Experimental::Example::pcgsolve with use_sgs = false (perf_test/sparse/KokkosSparse_pcg.hpp:248-466;
 * the driver perf_test/sparse/KokkosSparse_pcg.cpp:69-122 calls it with tolerance 1e-7): solves A x = b for a symmetric
 * positive definite CrsMatrix, x = initial guess on entry, solution on return.  The recurrence is the reference's,
 * operation for operation; alpha, beta and the residual stay on the device and the host only polls a `done` word every
 * check_every iterations (<= 0: 8), where the reference synchronises three times per iteration.  `plan` is the SpMV
 * plan of A (its analysis is reused by every iteration).  Returns the iteration count and sqrt(r.r) of the recurrence
 * (CGSolveResult::iteration / norm_res).  Synchronous: returns after the solve. */
int b200sp_cg_solve_f64_i32(b200sp_spmv_plan* plan, void* stream, int n, int64_t nnz, const int* row_ptr,
                            const int* col_idx, const double* vals, const double* b, double* x,
                            int maximum_iteration, double tolerance, int check_every, int* iterations,
                            double* norm_res);

/* pcgsolve with use_sgs = true (its default; pcg.hpp:339-358,412-437): the same loop with z = M^-1 r by one symmetric point
 * Gauss-Seidel sweep (zero initial guess, omega = 1) over the colour sets of gs_plan -- b200sp_gs_symbolic / _numeric must have
 * run on this matrix -- alpha = r.z / p.Ap, beta = r.z' / r.z, p = z + beta p; the stopping test stays sqrt(r.r). */
int b200sp_pcg_solve_f64_i32(b200sp_spmv_plan* plan, b200sp_gs_plan* gs_plan, void* stream, int n, int64_t nnz,
                             const int* row_ptr, const int* col_idx, const double* vals, const double* b, double* x,
                             int maximum_iteration, double tolerance, int check_every, int* iterations,
                             double* norm_res);
/* The same with the TWO-STAGE Gauss-Seidel as preconditioner (one symmetric sweep of b200sp_gs2_apply from z = 0, omega = 1): what
 * pcgsolve runs when its kernel handle was given a GS_TWOSTAGE handle -- symmetric_gauss_seidel_apply dispatches on the handle
 * (pcg.hpp:321-335).  b200sp_gs2_symbolic / _numeric must have run on this matrix. */
int b200sp_pcg_solve_gs2_f64_i32(b200sp_spmv_plan* plan, b200sp_gs2_plan* gs2_plan, void* stream, int n, int64_t nnz,
                                 const int* row_ptr, const int* col_idx, const double* vals, const double* b, double* x,
                                 int maximum_iteration, double tolerance, int check_every, int* iterations,
                                 double* norm_res);

/* ---- GMRES (SURVEY.md 8f rank 4) -----------------------------------------------------------------------------------
 * KokkosSparse::Experimental::gmres(handle, A, B, X, precond) (sparse/src/KokkosSparse_gmres.hpp:60-160 ->
 * GmresWrap::gmres, sparse/impl/KokkosSparse_gmres_impl.hpp:58-327) for a CrsMatrix: restarted GMRES(m) with CGS2
 * (ortho = 0) or MGS (ortho = 1), x = initial guess on entry and solution on return.  m, tol, max_restart and the three
 * results are GMRESHandle's (sparse/src/KokkosSparse_gmres_handle.hpp:76-110,175): num_iters, end_rel_res, conv_flag
 * (0 Conv, 1 NoConv, 2 LOA).  The optional right preconditioner is the reference's MatrixPrec -- an spmv with the matrix
 * (row_ptr_M, col_idx_M, vals_M), which needs its own plan; pass row_ptr_M = NULL for none.  B200SP_ERR_STATE with the
 * reference's message where it throws (lucky breakdown without convergence, NaN residual, :211-218);
 * B200SP_ERR_INVALID_ARGUMENT for an unknown ortho (:173).  Synchronous: returns after the solve. */
int b200sp_gmres_f64_i32(b200sp_spmv_plan* plan_A, void* stream, int n, int64_t nnz, const int* row_ptr, const int* col_idx,
                         const double* vals, b200sp_spmv_plan* plan_M, int64_t nnz_M, const int* row_ptr_M,
                         const int* col_idx_M, const double* vals_M, const double* b, double* x, int m, double tol,
                         int max_restart, int ortho, int* num_iters, double* end_rel_res, int* conv_flag);
int b200sp_gmres_f32_i32(b200sp_spmv_plan* plan_A, void* stream, int n, int64_t nnz, const int* row_ptr, const int* col_idx,
                         const float* vals, b200sp_spmv_plan* plan_M, int64_t nnz_M, const int* row_ptr_M,
                         const int* col_idx_M, const float* vals_M, const float* b, float* x, int m, float tol,
                         int max_restart, int ortho, int* num_iters, float* end_rel_res, int* conv_flag);
/* The BsrMatrix overload (sparse/impl/KokkosSparse_gmres_spec.hpp:79-82): A (and the MatrixPrec matrix) are mb x mb blocks of
 * bs x bs; b and x have mb*bs entries; the plans are b200sp_bsr_plan. */
int b200sp_gmres_bsr_f64_i32(b200sp_bsr_plan* plan_A, void* stream, int mb, int64_t nnzb, int bs, const int* row_ptr,
                             const int* col_idx, const double* vals, b200sp_bsr_plan* plan_M, int64_t nnzb_M,
                             const int* row_ptr_M, const int* col_idx_M, const double* vals_M, const double* b, double* x,
                             int m, double tol, int max_restart, int ortho, int* num_iters, double* end_rel_res,
                             int* conv_flag);
int b200sp_gmres_bsr_f32_i32(b200sp_bsr_plan* plan_A, void* stream, int mb, int64_t nnzb, int bs, const int* row_ptr,
                             const int* col_idx, const float* vals, b200sp_bsr_plan* plan_M, int64_t nnzb_M,
                             const int* row_ptr_M, const int* col_idx_M, const float* vals_M, const float* b, float* x, int m,
                             float tol, int max_restart, int ortho, int* num_iters, float* end_rel_res, int* conv_flag);

/* ---- introspection / tuning (bench + tests only) ------------------------- */
/* Counts kernels launched by this library since process start (all plans). */
int64_t b200sp_launch_count(void);
/* Name of the kernel variant the plan's last spmv call used ("tile<...>",
 * "vector<...>", ...); static storage. */
const char* b200sp_spmv_last_kernel(const b200sp_spmv_plan* plan);
/* Override the tiled kernel's configuration for this plan before its first
 * use: cfg = index into the built-in table (see DESIGN.md), grid_mult = CTAs
 * per SM (0 = default).  Returns B200SP_ERR_INVALID_ARGUMENT if out of range. */
/* The analysis a plan caches (tiles, long-row lists, the tiled kernel's 16-bit column stream, rank-2 work items, chunk tables,
 * cached transpose, host-vector piece bounds) is keyed on (row_ptr pointer, m, n, nnz), the column stream and the cached
 * transpose also on the col_idx pointer: a DIFFERENT matrix that reuses the same address with the same shape -- a
 * caching allocator hands the block out again, or row_ptr is edited in place -- would find a stale analysis.  Call this after
 * such a change ("all calls with one handle must use the same matrix", sparse/src/KokkosSparse_spmv_handle.hpp:276-277, is
 * the reference's contract; this is the escape hatch).  Stream-ordered; buffers that depend only on sizes are kept. */
int b200sp_spmv_plan_invalidate(b200sp_spmv_plan* plan, void* stream);

int b200sp_spmv_plan_tune(b200sp_spmv_plan* plan, int cfg, int lanes_per_row, int ctas_per_sm);
#ifdef __cplusplus
}
#endif
#endif /* B200SPARSE_H_ */
