// Microbenchmark: what does a shared-memory atomic cost on sm_90a at full occupancy (32 warps / SM)?
// Variants: no-return add, returning add, plain load+store RMW; address patterns: every lane its own word
// (random rows), a hot word shared by a fraction of the lanes. Prints SM cycles per warp-instruction.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o smem_atomics smem_atomics.cu && ./smem_atomics
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

constexpr int kWords = 36 * 1024;   // 144 KB of cells
constexpr int kIters = 2048;

template <int kMode>
__global__ void __launch_bounds__(1024, 1) k(uint32_t* out, long long* cycles, uint32_t hot_per_32, uint32_t seed) {
  extern __shared__ uint32_t cells[];
  for (int i = threadIdx.x; i < kWords; i += blockDim.x) cells[i] = 0;
  __syncthreads();
  uint32_t x = seed ^ (threadIdx.x * 2654435761u) ^ (blockIdx.x * 40503u);
  uint32_t acc = 0;
  const uint32_t lane = threadIdx.x & 31u;
  const long long t0 = clock64();
#pragma unroll 4
  for (int it = 0; it < kIters; ++it) {
    x = x * 1664525u + 1013904223u;
    uint32_t idx = (x >> 8) % kWords;
    if (lane < hot_per_32) idx = 7;   // these lanes of every warp hit one word
    if (kMode == 0) atomicAdd(&cells[idx], 1u);                       // result unused
    else if (kMode == 1) acc += atomicAdd(&cells[idx], 1u);           // result used
    else if (kMode == 2) { const uint32_t v = cells[idx]; cells[idx] = v + 1u; acc += v; }   // plain RMW (racy; cost only)
    else if (kMode == 3) { acc += atomicAdd(&cells[idx], 1u); acc += atomicAdd(&cells[(idx + 97) % kWords], x); }
    else if (kMode == 4) {                                             // warp-aggregated: one atomic per distinct word
      const uint32_t m = __match_any_sync(0xFFFFFFFFu, idx);
      if (lane == (uint32_t)__ffs((int)m) - 1u) atomicAdd(&cells[idx], (uint32_t)__popc(m));
    }
  }
  const long long t1 = clock64();
  __syncthreads();
  if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc + cells[threadIdx.x];
}

template <int kMode>
void run(const char* name, uint32_t hot) {
  uint32_t* out; long long* cyc;
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);   // one CTA per SM
  cudaMalloc(&out, (size_t)sms * 1024 * 4); cudaMalloc(&cyc, (size_t)sms * 8);
  cudaFuncSetAttribute(k<kMode>, cudaFuncAttributeMaxDynamicSharedMemorySize, kWords * 4);
  k<kMode><<<sms, 1024, kWords * 4>>>(out, cyc, hot, 1);
  k<kMode><<<sms, 1024, kWords * 4>>>(out, cyc, hot, 2);
  cudaDeviceSynchronize();
  long long h[1024]; cudaMemcpy(h, cyc, (size_t)sms * 8, cudaMemcpyDeviceToHost);
  double s = 0; for (int i = 0; i < sms; ++i) s += (double)h[i];
  s /= sms;
  // 32 warps each issue kIters warp-instructions (mode 3: two atomics per iteration)
  printf("%-34s hot lanes/32 = %2u : %7.1f cycles per warp-iteration (all 32 warps), %6.2f per lane-op\n", name, hot,
         s / kIters / 32.0 * 32.0 / 32.0 * 32.0, s / kIters / 1024.0 / (kMode == 3 ? 2.0 : 1.0));
  cudaFree(out); cudaFree(cyc);
}

int main() {
  for (uint32_t hot : {0u, 4u, 12u}) {
    run<0>("atomicAdd, result unused", hot);
    run<1>("atomicAdd, result used", hot);
    run<3>("two atomicAdds, results used", hot);
    run<2>("plain load + store", hot);
    run<4>("match_any + leader atomicAdd", hot);
  }
  return 0;
}
