// bspgemm.cu -- numeric phase of the block SpGEMM C = A*B on BsrMatrix data for H100 (sm_90a).
//
// Replaces the reference's Impl::BSPGEMM_NUMERIC (sparse/impl/KokkosSparse_bspgemm_numeric_spec.hpp:113-191: the native
// KokkosBSPGEMM followed by sort_bsr_matrix).  The symbolic phase is the point symbolic on the block graphs
// (b200sp_spgemm_symbolic_i32), as in the reference (sparse/src/KokkosSparse_spgemm.hpp:77-103).
//
// Values are bit-identical to the reference's bspgemm_debug_numeric (sparse/impl/KokkosSparse_bspgemm_impl_seq.hpp:39-130,
// GEMM = SerialGemmInternal<Unblocked>): entry (r, c) of block C(i, j) is one chain from +0.0 over the products of row i in
// ordinal order (A's row in storage order, each B row in storage order) and, within a product, over p = 0..bs-1:
//   acc = acc + a(r, p) * b(p, c)        every multiply and add rounded on its own (no FMA contraction)
//
// Design (DESIGN.md section 5.2): expand / sort / compress with product ids in place of values.  One CTA builds one block
// row of C:
//   expand   product t (its ordinal) -> key (column of its B block << 32 | t), and its A entry and B entry
//   sort     bitonic sort of the keys: runs of equal columns, each run in ordinal order
//   compress run heads -> sorted col_idx_C (a CTA scan gives each run its output position)
//   values   the bs*bs entries of every output block are flat work items of the CTA; each walks its run's products in
//            ordinal order.  A's blocks of the row are staged in shared memory when they fit, B's are gathered through the
//            read-only path.
// Rows of up to 1024 / 4096 products (and A entries) keep everything in shared memory; longer rows run the same code on
// per-CTA global scratch.  No floating-point atomics, deterministic, rows come out sorted.
#include "common.cuh"
#include "scan.cuh"
#include "spgemm_esc.cuh"
#include "bspgemm.cuh"
#include <algorithm>
#include <limits.h>
#include <new>

namespace b200sp {

template <typename S>
__device__ __forceinline__ S add_rn(S a, S b);
template <>
__device__ __forceinline__ double add_rn<double>(double a, double b) { return __dadd_rn(a, b); }
template <>
__device__ __forceinline__ float add_rn<float>(float a, float b) { return __fadd_rn(a, b); }

// block-row bins: products and A entries of a row fit CAP0 / CAP1 (shared memory), else global scratch
static constexpr int kBspCap0 = 1024;
static constexpr int kBspCap1 = 4096;
static constexpr int kBspLongCtas = 32;
static constexpr int kBspAStage = 24 * 1024;  // bytes of A blocks staged per CTA

struct BspState {
  DevArray<int> rows;  // block rows grouped by bin: [<= CAP0 | <= CAP1 | long]
  int off[4] = {0, 0, 0, 0};
  int long_log2 = 1;    // keys per long-row CTA: 2^long_log2 >= the longest row's products and A entries
  DevArray<unsigned char> scratch;
};

void bsp_state_free(BspState* s, cudaStream_t st) {
  if (!s) return;
  s->rows.release(st);
  s->scratch.release(st);
  delete s;
}

// per block row: bin and the key it was binned by, max(products, nnz(A_i) + 1)
__global__ void bsp_count_kernel(int m, const int* __restrict__ flops, const int* __restrict__ rpA, int* __restrict__ counts,
                                 int* __restrict__ maxkey) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < m; r += gridDim.x * blockDim.x) {
    const int key = max(flops[r], rpA[r + 1] - rpA[r] + 1);
    const int b = key <= kBspCap0 ? 0 : (key <= kBspCap1 ? 1 : 2);
    atomicAdd(&counts[b], 1);
    if (b == 2) atomicMax(maxkey, key);
  }
}
__global__ void bsp_scatter_kernel(int m, const int* __restrict__ flops, const int* __restrict__ rpA, int* __restrict__ cursors,
                                   int* __restrict__ rows) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < m; r += gridDim.x * blockDim.x) {
    const int key = max(flops[r], rpA[r + 1] - rpA[r] + 1);
    const int b = key <= kBspCap0 ? 0 : (key <= kBspCap1 ? 1 : 2);
    rows[atomicAdd(&cursors[b], 1)] = r;
  }
}

// Working arrays of one block row (shared memory, or one CTA's slice of global scratch for long rows)
template <typename S>
struct BspRowMem {
  unsigned long long* keys;  // [cap]      (column << 32 | ordinal), sorted in place
  int* sj;                   // [cap]      by ordinal: A entry (0-based within the row)
  int* sjb;                  // [cap]      by ordinal: B entry
  int* rs;                   // [cap + 1]  run starts of the output blocks
  int* pre;                  // [cap + 1]  first ordinal of each A entry's products; pre[nA] = f
  int* bst;                  // [cap]      start of each A entry's B row
  S* sA;                     // A's blocks of the row, when they fit in astage elements
  int astage;
  int* wsum;                 // [40]
};

template <typename S, int T>
__device__ __forceinline__ void bsp_row(const BspRowMem<S>& w, int cap, int i, int bs, const int* __restrict__ rpA,
                                        const int* __restrict__ ciA, const S* __restrict__ vA, const int* __restrict__ rpB,
                                        const int* __restrict__ ciB, const S* __restrict__ vB, const int* __restrict__ rpC,
                                        int* __restrict__ ciC, S* __restrict__ vC) {
  const int tid = threadIdx.x;
  const int a0 = rpA[i], nA = rpA[i + 1] - a0;
  const int cbase = rpC[i], nz = rpC[i + 1] - cbase;
  if (nz == 0) return;  // (uniform over the CTA)
  const int bb = bs * bs;
  // ---- stage: B row starts and the exclusive scan of B row lengths over A's row; A's blocks
  int carry = 0;
  for (int base = 0; base < nA; base += T) {
    const int j = base + tid;
    int len = 0;
    if (j < nA) {
      const int c = ldg(ciA + a0 + j);
      const int b0 = ldg(rpB + c);
      len = ldg(rpB + c + 1) - b0;
      w.bst[j] = b0;
    }
    int total;
    const int excl = esc_block_scan1<T>(len, w.wsum, total);
    if (j < nA) w.pre[j] = carry + excl;
    carry += total;
  }
  const int f = carry;
  if (tid == 0) w.pre[nA] = f;
  const bool staged = (long long)nA * bb <= (long long)w.astage;
  if (staged)
    for (int e = tid; e < nA * bb; e += T) w.sA[e] = ldg(vA + (int64_t)a0 * bb + e);
  int n2 = 2;
  while (n2 < f) n2 <<= 1;
  __syncthreads();
  // ---- expand: key = (column, ordinal); payload by ordinal
  {
    int lo = 0;
    for (int t = tid; t < n2; t += T) {
      if (t < f) {
        int hi = nA;  // largest j with pre[j] <= t; t grows: search from the last answer
        while (hi - lo > 1) {
          const int mid = (lo + hi) >> 1;
          if (w.pre[mid] <= t) lo = mid; else hi = mid;
        }
        const int jb = w.bst[lo] + (t - w.pre[lo]);
        const int c = ldg(ciB + jb);
        w.keys[t] = ((unsigned long long)(unsigned)c << 32) | (unsigned)t;
        w.sj[t] = lo;
        w.sjb[t] = jb;
      } else {
        w.keys[t] = ~0ull;
      }
    }
  }
  __syncthreads();
  // ---- bitonic sort of n2 keys (ascending)
  for (int kk = 2; kk <= n2; kk <<= 1) {
    for (int jj = kk >> 1; jj > 0; jj >>= 1) {
      for (int t = tid; t < (n2 >> 1); t += T) {
        const int x = 2 * jj * (t / jj) + (t % jj);
        const int y = x + jj;
        const unsigned long long kx = w.keys[x], ky = w.keys[y];
        const bool up = (x & kk) == 0;
        if ((kx > ky) == up) {
          w.keys[x] = ky;
          w.keys[y] = kx;
        }
      }
      __syncthreads();
    }
  }
  // ---- compress: run heads -> output positions, sorted col_idx_C
  int runs = 0;
  for (int base = 0; base < f; base += T) {
    const int q = base + tid;
    int head = 0;
    int c = 0;
    if (q < f) {
      c = (int)(w.keys[q] >> 32);
      head = (q == 0) || (c != (int)(w.keys[q - 1] >> 32));
    }
    int total;
    const int excl = esc_block_scan1<T>(head, w.wsum, total);
    if (head) {
      const int o = runs + excl;
      if (o < nz) {  // more distinct columns than the symbolic pattern holds = precondition violated: drop, do not corrupt
        w.rs[o] = q;
        ciC[cbase + o] = c;
      }
    }
    runs += total;
  }
  if (tid == 0) w.rs[min(runs, nz)] = f;
  __syncthreads();
  // ---- values: entry e of the row's output = (block o, row r, column c); its chain runs over the run of block o
  const int nout = min(runs, nz);
  const int64_t vbase = (int64_t)cbase * bb;
  for (int e = tid; e < nout * bb; e += T) {
    const int o = e / bb;
    const int rc = e - o * bb;
    const int r = rc / bs, c = rc - r * bs;
    const int q0 = w.rs[o], q1 = w.rs[o + 1];
    S acc = S(0);
    for (int q = q0; q < q1; ++q) {
      const int t = (int)(unsigned)(w.keys[q] & 0xffffffffull);
      const int j = w.sj[t];
      const S* __restrict__ pb = vB + (int64_t)w.sjb[t] * bb + c;
      if (staged) {
        const S* pa = w.sA + j * bb + r * bs;
        for (int p = 0; p < bs; ++p) acc = add_rn(acc, mul_rn(pa[p], ldg(pb + p * bs)));
      } else {
        const S* __restrict__ pa = vA + (int64_t)(a0 + j) * bb + r * bs;
        for (int p = 0; p < bs; ++p) acc = add_rn(acc, mul_rn(ldg(pa + p), ldg(pb + p * bs)));
      }
    }
    vC[vbase + e] = acc;
  }
  __syncthreads();  // the next row reuses every array
}

// rows of at most CAP products and CAP - 1 entries of A: everything in shared memory; persistent over the bin's rows
template <int CAP>
struct BspSmem {
  static constexpr size_t KEYS = sizeof(unsigned long long) * CAP;
  static constexpr size_t INTS = sizeof(int) * ((size_t)CAP * 5 + 2 + 40);
  static constexpr size_t BYTES = KEYS + ((INTS + 15) & ~(size_t)15) + kBspAStage;
};

// base: keys, then the int arrays (and, in shared memory, A's staging area after them); wsum / sA given: they live
// elsewhere (the long-row kernel keeps them in shared memory while its arrays are global)
template <typename S>
__device__ __forceinline__ BspRowMem<S> bsp_carve(unsigned char* base, int cap, int astage_bytes, int* wsum = nullptr,
                                                  S* sA = nullptr) {
  BspRowMem<S> w;
  w.keys = reinterpret_cast<unsigned long long*>(base);
  int* ip = reinterpret_cast<int*>(base + sizeof(unsigned long long) * (size_t)cap);
  w.sj = ip;
  w.sjb = w.sj + cap;
  w.rs = w.sjb + cap;
  w.pre = w.rs + cap + 1;
  w.bst = w.pre + cap + 1;
  w.wsum = wsum ? wsum : w.bst + cap;
  const size_t ints = sizeof(int) * ((size_t)cap * 5 + 2 + 40);
  w.sA = sA ? sA : reinterpret_cast<S*>(reinterpret_cast<unsigned char*>(ip) + ((ints + 15) & ~(size_t)15));
  w.astage = astage_bytes / (int)sizeof(S);
  return w;
}

template <typename S, int T, int CAP>
__global__ void __launch_bounds__(T) bsp_smem_kernel(int nrows, const int* __restrict__ rows, int bs, const int* __restrict__ rpA,
                                                     const int* __restrict__ ciA, const S* __restrict__ vA, const int* __restrict__ rpB,
                                                     const int* __restrict__ ciB, const S* __restrict__ vB, const int* __restrict__ rpC,
                                                     int* __restrict__ ciC, S* __restrict__ vC) {
  extern __shared__ __align__(16) unsigned char bsp_sm[];
  const BspRowMem<S> w = bsp_carve<S>(bsp_sm, CAP, kBspAStage);
  for (int r = blockIdx.x; r < nrows; r += gridDim.x)
    bsp_row<S, T>(w, CAP, rows[r], bs, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC);
}

// long rows: the same row code on this CTA's slice of global scratch; A's blocks still staged in shared memory if they fit
template <typename S, int T>
__global__ void __launch_bounds__(T) bsp_long_kernel(int nrows, const int* __restrict__ rows, int cap, unsigned char* __restrict__ scratch,
                                                     size_t slice, int bs, const int* __restrict__ rpA, const int* __restrict__ ciA,
                                                     const S* __restrict__ vA, const int* __restrict__ rpB, const int* __restrict__ ciB,
                                                     const S* __restrict__ vB, const int* __restrict__ rpC, int* __restrict__ ciC,
                                                     S* __restrict__ vC) {
  extern __shared__ __align__(16) unsigned char bsp_sm[];
  const BspRowMem<S> w = bsp_carve<S>(scratch + slice * blockIdx.x, cap, kBspAStage, reinterpret_cast<int*>(bsp_sm),
                                      reinterpret_cast<S*>(bsp_sm + 256));
  for (int r = blockIdx.x; r < nrows; r += gridDim.x)
    bsp_row<S, T>(w, cap, rows[r], bs, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC);
}

// grouping of the block rows (first block numeric on a plan; synchronises once, like the point numeric's all-row bins)
static int bsp_state_build(const SpgemmPlanView& v, cudaStream_t st, const int* rpA, BspState** out) {
  BspState* s = new (std::nothrow) BspState();
  if (!s) {
    set_error("bspgemm_numeric: out of host memory");
    return B200SP_ERR_ALLOC;
  }
  const int m = v.m;
  DevTmp tmp(st);
  int* d;  // counts[3] | cursors[3] | maxkey
  cudaError_t e = tmp.alloc(&d, 8);
  if (e == cudaSuccess) e = cudaMemsetAsync(d, 0, sizeof(int) * 8, st);
  if (e == cudaSuccess) e = s->rows.alloc((size_t)std::max(m, 1), st);
  if (e != cudaSuccess) {
    bsp_state_free(s, st);
    set_error("bspgemm_numeric: %s", cudaGetErrorString(e));
    return B200SP_ERR_CUDA;
  }
  const int blocks = std::max(1, std::min((m + 255) / 256, sm_count() * 8));
  bsp_count_kernel<<<blocks, 256, 0, st>>>(m, v.flops, rpA, d, d + 6);
  int h[8] = {0};
  e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpyAsync(h, d, sizeof(int) * 8, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e == cudaSuccess) {
    s->off[0] = 0;
    for (int b = 0; b < 3; ++b) s->off[b + 1] = s->off[b] + h[b];
    e = cudaMemcpyAsync(d + 3, s->off, sizeof(int) * 3, cudaMemcpyHostToDevice, st);
  }
  if (e == cudaSuccess) {
    bsp_scatter_kernel<<<blocks, 256, 0, st>>>(m, v.flops, rpA, d + 3, s->rows);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess && h[2] > 0) {
    int lg = 1;
    while ((1LL << lg) < (long long)h[6]) ++lg;
    s->long_log2 = lg;
    const size_t cap = (size_t)1 << lg;
    const size_t slice = (sizeof(unsigned long long) * cap + sizeof(int) * (cap * 5 + 2 + 40) + 15) & ~(size_t)15;
    e = s->scratch.alloc(slice * (size_t)std::min(h[2], kBspLongCtas), st);
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);  // s->off (pageable) consumed by the copy above
  g_launches.fetch_add(2, std::memory_order_relaxed);
  if (e != cudaSuccess) {
    bsp_state_free(s, st);
    set_error("bspgemm_numeric: %s", cudaGetErrorString(e));
    return B200SP_ERR_CUDA;
  }
  *out = s;
  return B200SP_OK;
}

template <typename S, int T, int CAP>
static int launch_bsp_smem(cudaStream_t st, int nrows, const int* rows, int bs, const int* rpA, const int* ciA, const S* vA,
                           const int* rpB, const int* ciB, const S* vB, const int* rpC, int* ciC, S* vC) {
  if (nrows <= 0) return B200SP_OK;
  auto kern = bsp_smem_kernel<S, T, CAP>;
  static KernelSetup ks;
  int occ = 1;
  if (int rc = kernel_setup(ks, kern, T, BspSmem<CAP>::BYTES, &occ)) return rc;
  const int grid = (int)std::min<int64_t>(nrows, (int64_t)sm_count() * occ);
  kern<<<grid, T, BspSmem<CAP>::BYTES, st>>>(nrows, rows, bs, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC);
  B200SP_LAUNCH_CHECK();
  return B200SP_OK;
}

template <typename S>
static int bspgemm_impl(b200sp_spgemm_plan* plan, cudaStream_t st, int mb, int nb, int kb, int bs, const int* rpA, const int* ciA,
                        const S* vA, const int* rpB, const int* ciB, const S* vB, const int* rpC, int* ciC, S* vC) {
  const SpgemmPlanView v = spgemm_plan_view(plan);
  if (spgemm64_holds_product(*v.s64)) {
    set_error("block_spgemm_numeric: not provided on 64-bit offsets (the symbolic phase on this handle had them)");
    return B200SP_ERR_STATE;
  }
  if (!v.symbolic_done) {
    set_error("KokkosSparse::block_spgemm_numeric: must first call spgemm_symbolic with the same handle.");
    return B200SP_ERR_STATE;
  }
  if (v.m != mb || v.n != nb || v.k != kb) {
    set_error("bspgemm_numeric: block dimensions (%d,%d,%d) differ from symbolic (%d,%d,%d)", mb, nb, kb, v.m, v.n, v.k);
    return B200SP_ERR_STATE;
  }
  if (mb == 0 || v.c_nnz == 0) return B200SP_OK;
  B200SP_REQUIRE(rpA && ciA && vA && rpB && ciB && vB && rpC && ciC && vC, "bspgemm_numeric: null pointer argument");
  // the kernels index one block row's values in 32 bits (the whole matrix in 64)
  B200SP_REQUIRE((int64_t)v.c_max * bs * bs <= INT_MAX, "bspgemm_numeric: a block row of C holds more than 2^31 values");
  if (!*v.bsp) {
    if (int rc = bsp_state_build(v, st, rpA, v.bsp)) return rc;
  }
  const BspState& s = **v.bsp;
  int rc;
  if ((rc = launch_bsp_smem<S, 256, kBspCap0>(st, s.off[1] - s.off[0], s.rows + s.off[0], bs, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC)))
    return rc;
  if ((rc = launch_bsp_smem<S, 512, kBspCap1>(st, s.off[2] - s.off[1], s.rows + s.off[1], bs, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC)))
    return rc;
  const int nlong = s.off[3] - s.off[2];
  if (nlong > 0) {
    const size_t cap = (size_t)1 << s.long_log2;
    const size_t slice = (sizeof(unsigned long long) * cap + sizeof(int) * (cap * 5 + 2 + 40) + 15) & ~(size_t)15;
    const size_t smem = 256 + kBspAStage;
    auto kern = bsp_long_kernel<S, 512>;
    static KernelSetup ks;
    int occ = 1;
    if ((rc = kernel_setup(ks, kern, 512, smem, &occ))) return rc;
    kern<<<std::min(nlong, kBspLongCtas), 512, smem, st>>>(nlong, s.rows + s.off[2], (int)cap, s.scratch, slice, bs,
                                                           rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC);
    B200SP_LAUNCH_CHECK();
  }
  return B200SP_OK;
}

}  // namespace b200sp

using namespace b200sp;

static int bsp_check_args(b200sp_spgemm_plan* plan, int mb, int nb, int kb, int bs) {
  B200SP_REQUIRE(plan != nullptr, "bspgemm_numeric: null plan");
  B200SP_REQUIRE(mb >= 0 && nb >= 0 && kb >= 0, "bspgemm_numeric: negative dimension");
  B200SP_REQUIRE(bs >= 1, "bspgemm_numeric: block size %d < 1", bs);
  B200SP_REQUIRE(bs <= 46340, "bspgemm_numeric: block size %d: bs * bs exceeds int32", bs);
  return B200SP_OK;
}

extern "C" {

int b200sp_bspgemm_numeric_f64_i32(b200sp_spgemm_plan* plan, void* stream, int mb, int nb, int kb, int bs, const int* rpA,
                                   const int* ciA, const double* vA, const int* rpB, const int* ciB, const double* vB,
                                   const int* rpC, int* ciC, double* vC) {
  if (int rc = bsp_check_args(plan, mb, nb, kb, bs)) return rc;
  if (bs == 1)  // the reference's front end: block_dim == 1 is the point product (KokkosSparse_spgemm_numeric.hpp:191)
    return b200sp_spgemm_numeric_f64_i32(plan, stream, mb, nb, kb, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC);
  return bspgemm_impl<double>(plan, (cudaStream_t)stream, mb, nb, kb, bs, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC);
}

int b200sp_bspgemm_numeric_f32_i32(b200sp_spgemm_plan* plan, void* stream, int mb, int nb, int kb, int bs, const int* rpA,
                                   const int* ciA, const float* vA, const int* rpB, const int* ciB, const float* vB,
                                   const int* rpC, int* ciC, float* vC) {
  if (int rc = bsp_check_args(plan, mb, nb, kb, bs)) return rc;
  if (bs == 1)
    return b200sp_spgemm_numeric_f32_i32(plan, stream, mb, nb, kb, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC);
  return bspgemm_impl<float>(plan, (cudaStream_t)stream, mb, nb, kb, bs, rpA, ciA, vA, rpB, ciB, vB, rpC, ciC, vC);
}

}  // extern "C"
