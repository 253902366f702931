// hbm_read.cu -- the achievable HBM read rate of the card, measured the way the tiled SpMV reads its matrix: one producer
// lane per CTA streams `chunk`-byte pieces of a large buffer into a ring of STAGES shared-memory stages with 1-D bulk
// copies (cp.async.bulk + mbarrier) and discards them, at 2 CTAs per SM.  For comparison, the same bytes read by every
// thread of the grid with 16-byte loads.  Built and run by tools/bench_hbm_read.py; prints one JSON line per case.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

template <int STAGES>
__global__ void __launch_bounds__(32) bulk_read_kernel(const char* __restrict__ src, int64_t bytes, int chunk) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);
  unsigned char* buf = smem + 128;
  if (threadIdx.x != 0) return;
  for (int s = 0; s < STAGES; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&full[s])));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  const int64_t n_chunks = (bytes + chunk - 1) / chunk;
  int it = 0;
  auto wait = [&](int j) {
    uint32_t ok = 0;
    while (!ok)
      asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
                   : "=r"(ok)
                   : "r"(smem_u32(&full[j % STAGES])), "r"((uint32_t)(j / STAGES) & 1u)
                   : "memory");
  };
  for (int64_t c = blockIdx.x; c < n_chunks; c += gridDim.x, ++it) {
    const int stage = it % STAGES;
    if (it >= STAGES) wait(it - STAGES);  // the stage's previous copy has landed: its bytes are discarded
    const uint32_t len = (uint32_t)(bytes - c * chunk < chunk ? bytes - c * chunk : chunk);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&full[stage])), "r"(len) : "memory");
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
            smem_u32(buf + (size_t)stage * chunk)),
        "l"(src + c * chunk), "r"(len), "r"(smem_u32(&full[stage])), "l"(pol)
        : "memory");
  }
  for (int j = it > STAGES ? it - STAGES : 0; j < it; ++j) wait(j);
}

__global__ void __launch_bounds__(512) load_read_kernel(const int4* __restrict__ src, int64_t n, int* __restrict__ sink) {
  int acc = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(src + i));
    acc ^= v.x ^ v.y ^ v.z ^ v.w;
  }
  if (acc == 0x7fffffff) *sink = acc;  // keeps the loads
}

#define CK(x)                                                                 \
  do {                                                                        \
    cudaError_t e_ = (x);                                                     \
    if (e_ != cudaSuccess) {                                                  \
      fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_));                \
      exit(1);                                                                \
    }                                                                         \
  } while (0)

template <class Launch>
static double time_ms(Launch launch, int reps) {
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a));
  CK(cudaEventCreate(&b));
  for (int i = 0; i < 3; ++i) launch();
  CK(cudaEventRecord(a));
  for (int i = 0; i < reps; ++i) launch();
  CK(cudaEventRecord(b));
  CK(cudaEventSynchronize(b));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, a, b));
  CK(cudaGetLastError());
  return ms / reps;
}

template <int STAGES>
static void bulk_case(const char* src, int64_t bytes, int chunk, int ctas_per_sm, int sms, int reps) {
  // at least the SpMV's shared memory per CTA, so that the card holds the same number of CTAs per SM
  const size_t smem_min = (227 * 1024) / ctas_per_sm - 1024 - 128;
  size_t smem = 128 + (size_t)STAGES * chunk;
  if (smem < smem_min) smem = smem_min;
  auto k = bulk_read_kernel<STAGES>;
  CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int grid = sms * ctas_per_sm;
  const double ms = time_ms([&] { k<<<grid, 32, smem>>>(src, bytes, chunk); }, reps);
  printf("{\"kind\": \"bulk\", \"chunk\": %d, \"stages\": %d, \"ctas_per_sm\": %d, \"ms\": %.4f, \"gbs\": %.1f}\n", chunk, STAGES,
         ctas_per_sm, ms, bytes / ms / 1e6);
}

int main(int argc, char** argv) {
  const double gb = argc > 1 ? atof(argv[1]) : 4.3;
  const int reps = argc > 2 ? atoi(argv[2]) : 20;
  const int64_t bytes = ((int64_t)(gb * 1e9)) & ~(int64_t)15;
  int dev = 0, sms = 0;
  CK(cudaGetDevice(&dev));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, dev));
  printf("{\"kind\": \"device\", \"name\": \"%s\", \"sms\": %d, \"bytes\": %lld}\n", prop.name, sms, (long long)bytes);
  char* src = nullptr;
  int* sink = nullptr;
  CK(cudaMalloc(&src, bytes));
  CK(cudaMalloc(&sink, sizeof(int)));
  CK(cudaMemset(src, 1, bytes));
  // the SpMV's value stages: CAP 2048 and 4096 f64 (16 / 32 KB), and the pieces its tiles actually fill (1528 / 3576 values)
  for (int round = 0; round < 2; ++round) {
    bulk_case<4>(src, bytes, 16384, 2, sms, reps);
    bulk_case<4>(src, bytes, 1528 * 8, 2, sms, reps);
    bulk_case<3>(src, bytes, 32768, 2, sms, reps);
    bulk_case<3>(src, bytes, 3576 * 8, 2, sms, reps);
    bulk_case<2>(src, bytes, 32768, 2, sms, reps);
    bulk_case<6>(src, bytes, 16384, 2, sms, reps);
    const int64_t n4 = bytes / 16;
    const double ms = time_ms([&] { load_read_kernel<<<sms * 4, 512>>>(reinterpret_cast<const int4*>(src), n4, sink); }, reps);
    printf("{\"kind\": \"ld128\", \"ms\": %.4f, \"gbs\": %.1f}\n", ms, n4 * 16 / ms / 1e6);
  }
  CK(cudaFree(src));
  CK(cudaFree(sink));
  return 0;
}
