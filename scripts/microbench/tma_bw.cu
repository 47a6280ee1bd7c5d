// tma_bw.cu — microbenchmark: how many bytes per clock per SM can TMA pull from L2 into shared memory
// with the box shape the convolution kernels use (64 channels x R rows, 128-B swizzle), with all SMs
// active — unicast vs 2-CTA-cluster multicast.  Decides whether weight multicast is worth building.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tma_bw tma_bw.cu && ./tma_bw
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>
#include <vector>

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t b, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(b), "r"(c)); }
__device__ __forceinline__ void mbar_expect(uint32_t b, uint32_t n) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(n) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(b) : "memory"); }
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t b, uint32_t cta) {
  asm volatile("{\n\t.reg .b32 r;\n\tmapa.shared::cluster.u32 r, %0, %1;\n\tmbarrier.arrive.shared::cluster.b64 _, [r];\n\t}" ::"r"(b), "r"(cta) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t b, uint32_t par) {
  uint32_t ok = 0; unsigned long long spins = 0;
  while (!ok) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(b), "r"(par) : "memory");
    if (++spins > (1ull << 26)) { printf("timeout blk %d\n", blockIdx.x); __trap(); }
  }
}
__device__ __forceinline__ void tma_2d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(dst), "l"((uint64_t)m), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_2d_mc(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, uint16_t mask) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
               ::"r"(dst), "l"((uint64_t)m), "r"(bar), "r"(c0), "r"(c1), "h"(mask) : "memory");
}

constexpr int kStages = 6;
// mode 0: every CTA loads full boxes (R rows).  mode 1 (cluster of 2): each CTA loads R/2 rows and
// multicasts them to both CTAs, so both receive all R rows while issuing half the requests.
template <int MODE>
__global__ void __launch_bounds__(128, 1) tma_bw_kernel(const __grid_constant__ CUtensorMap map, int rows_box, int kchunks,
                                                          int row_tiles, int iters, long long* cycles) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ __align__(8) uint64_t full[kStages], empty[kStages];
  const uint32_t base = (smem_u32(smem) + 1023u) & ~1023u;
  const uint32_t stage_bytes = rows_box * 128;
  uint32_t rank = 0;
  if (MODE == 1) asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(smem_u32(&full[s]), 1); mbar_init(smem_u32(&empty[s]), MODE == 1 ? 2 : 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (MODE == 1) { asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory"); }
  long long t0 = clock64();
  if (threadIdx.x == 0) {            // producer
    int st = 0; uint32_t ph = 0;
    for (int i = 0; i < iters; ++i) {
      const int c = i % kchunks, rt = (i / kchunks + blockIdx.x / (MODE == 1 ? 2 : 1)) % row_tiles;
      mbar_wait(smem_u32(&empty[st]), ph ^ 1u);
      mbar_expect(smem_u32(&full[st]), stage_bytes);
      if (MODE == 0) tma_2d(base + st * stage_bytes, &map, smem_u32(&full[st]), c * 64, rt * rows_box);
      else tma_2d_mc(base + st * stage_bytes + rank * (stage_bytes / 2), &map, smem_u32(&full[st]), c * 64,
                     rt * rows_box + rank * (rows_box / 2), (uint16_t)3);
      if (++st == kStages) { st = 0; ph ^= 1u; }
    }
  } else if (threadIdx.x == 32) {    // consumer: release immediately
    int st = 0; uint32_t ph = 0;
    for (int i = 0; i < iters; ++i) {
      mbar_wait(smem_u32(&full[st]), ph);
      if (MODE == 0) mbar_arrive(smem_u32(&empty[st]));
      else { mbar_arrive_cluster(smem_u32(&empty[st]), 0); mbar_arrive_cluster(smem_u32(&empty[st]), 1); }
      if (++st == kStages) { st = 0; ph ^= 1u; }
    }
  }
  __syncthreads();
  if (MODE == 1) { asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory"); }
  if (threadIdx.x == 0) cycles[blockIdx.x] = clock64() - t0;
}

typedef CUresult (*EncFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                          const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int main() {
  void* fp = nullptr; cudaDriverEntryPointQueryResult q;
  cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q);
  EncFn enc = (EncFn)fp;
  const int K = 2304, ROWS = 9 * 256;           // dec6 weights: [9*256][2304] fp16 = 10.6 MB (L2 resident)
  void* d; cudaMalloc(&d, (size_t)ROWS * K * 2); cudaMemset(d, 1, (size_t)ROWS * K * 2);
  long long* dc; cudaMalloc(&dc, 148 * 8);
  int nsm = 148;
  for (int rows_box : {256, 128, 64}) {
    for (int mode = 0; mode < 2; ++mode) {
      const int box_rows = mode == 1 ? rows_box / 2 : rows_box;
      CUtensorMap map;
      cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)ROWS}; cuuint64_t strides[1] = {(cuuint64_t)K * 2};
      cuuint32_t box[2] = {64, (cuuint32_t)box_rows}; cuuint32_t es[2] = {1, 1};
      enc(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, d, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
          CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      const int iters = 2000, smem = kStages * rows_box * 128 + 1024;
      cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
      for (int rep = 0; rep < 2; ++rep) {
        cudaEventRecord(e0);
        if (mode == 0) {
          cudaFuncSetAttribute(tma_bw_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
          tma_bw_kernel<0><<<nsm, 128, smem>>>(map, rows_box, K / 64, ROWS / rows_box, iters, dc);
        } else {
          cudaFuncSetAttribute(tma_bw_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
          cudaLaunchConfig_t cfg{}; cfg.gridDim = dim3(nsm); cfg.blockDim = dim3(128); cfg.dynamicSmemBytes = smem;
          cudaLaunchAttribute at[1]; at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim = {2, 1, 1};
          cfg.attrs = at; cfg.numAttrs = 1;
          cudaLaunchKernelEx(&cfg, tma_bw_kernel<1>, map, rows_box, K / 64, ROWS / rows_box, iters, dc);
        }
        cudaEventRecord(e1);
        cudaError_t err = cudaDeviceSynchronize();
        if (err != cudaSuccess) { printf("error: %s\n", cudaGetErrorString(err)); return 1; }
      }
      float ms; cudaEventElapsedTime(&ms, e0, e1);
      std::vector<long long> hc(nsm); cudaMemcpy(hc.data(), dc, nsm * 8, cudaMemcpyDeviceToHost);
      double avg = 0; for (auto c : hc) avg += c; avg /= nsm;
      const double bytes_per_cta = (double)iters * rows_box * 128;
      printf("rows_box %3d %-9s: %.3f ms, %.1f B/clk/SM received, aggregate %.2f TB/s (requests issued per SM: %.1f B/clk)\n", rows_box,
             mode ? "multicast" : "unicast", ms, bytes_per_cta / avg, bytes_per_cta * nsm / (ms * 1e-3) / 1e12,
             bytes_per_cta / avg / (mode ? 2 : 1));
    }
  }
  return 0;
}
