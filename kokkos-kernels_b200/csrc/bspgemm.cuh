// bspgemm.cuh -- what the block SpGEMM numeric phase (bspgemm.cu) and the 64-bit-offset layer (spgemm64.cu) read from the
// SpGEMM plan (spgemm.cu).
//
// Block symbolic is point symbolic on the block graphs, so a block product runs on an ordinary b200sp_spgemm_plan.  The
// plan owns one extra piece of state, the grouping of block rows by product count that the block kernels are launched
// from; it is built by the first block numeric call and freed with the plan (or by a new symbolic).
#pragma once
#include "common.cuh"

namespace b200sp {

struct BspState;
void bsp_state_free(BspState* s, cudaStream_t st);

// windows, child plans and narrowed arrays of a product with 64-bit offsets (spgemm64.cu), freed with the plan
struct Spgemm64State;
bool spgemm64_holds_product(const Spgemm64State* s);  // a 64-bit symbolic completed on the plan
void spgemm64_state_free(Spgemm64State* s, cudaStream_t st);

struct SpgemmPlanView {
  bool symbolic_done;
  int m, n, k;
  int64_t c_nnz;
  int c_max;         // longest row of C
  const int* flops;  // products per row of A*B (device; only when c_nnz > 0)
  BspState** bsp;    // the plan's block-row grouping slot
  Spgemm64State** s64;  // the plan's 64-bit-offset slot
};
SpgemmPlanView spgemm_plan_view(b200sp_spgemm_plan* p);

}  // namespace b200sp
