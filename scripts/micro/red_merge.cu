// How does the L2 price global reductions? Per lane-op, per instruction, or per 32-byte sector request?
// Each "event" adds 1 to a histogram cell and a duration to a latency sum of a random row (rows L2-resident).
//   A  two instructions, two sectors   (hist[row][b] u32 and lat[row] u64 in separate arrays: today's layout)
//   B  two instructions, one sector    (cell and lat partial share a 32-byte sector)
//   C  ONE red.u64 instruction, lane pairs: even lane the cell pair, odd lane the lat partial of the same sector
//   D  one red.u32 only (lower bound)
//   E  like C but four lanes per event all in one sector (cell, lat, err, count)
// nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o red_merge red_merge.cu
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

__device__ __forceinline__ uint32_t mix(uint32_t x) { x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x; }
__device__ __forceinline__ void red32(uint32_t* p, uint32_t v) { asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void red64(uint64_t* p, uint64_t v) { asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }

constexpr uint32_t kRows = 190000;       // like config 2
constexpr uint32_t kSectorsPerRow = 11;  // layout B/C: 11 x {3 x u64 cell pairs, u64 lat partial}

template <int kMode>
__global__ void __launch_bounds__(512) k(uint32_t* hist, uint64_t* lat, uint64_t* sect, uint32_t events_per_thread) {
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31u;
  for (uint32_t i = 0; i < events_per_thread; ++i) {
    if (kMode == 2 || kMode == 4) {
      // one event per lane pair / quad: the lanes of a group compute the same event
      const uint32_t g = kMode == 2 ? 2u : 4u;
      const uint32_t ev = mix((tid / g) * 0x9E3779B1u + i * 0x85EBCA6Bu + 7u);
      const uint32_t row = ev % kRows, b = (ev >> 20) & 63u, dur = (ev >> 8) | 1u;
      uint64_t* s = sect + ((size_t)row * kSectorsPerRow + b / 6u) * 4u;
      const uint32_t sub = lane & (g - 1u);
      if (kMode == 2) red64(sub == 0 ? s + (b % 6u) / 2u : s + 3, sub == 0 ? (1ull << (32u * (b & 1u))) : (uint64_t)dur);
      else red64(s + sub, sub == 3 ? (uint64_t)dur : 1ull);
    } else {
      const uint32_t ev = mix(tid * 0x9E3779B1u + i * 0x85EBCA6Bu + 7u);
      const uint32_t row = ev % kRows, b = (ev >> 20) & 63u, dur = (ev >> 8) | 1u;
      if (kMode == 0) { red32(hist + (size_t)row * 64u + b, 1u); red64(lat + row, dur); }
      if (kMode == 1) {
        uint64_t* s = sect + ((size_t)row * kSectorsPerRow + b / 6u) * 4u;
        red32(reinterpret_cast<uint32_t*>(s) + (b % 6u), 1u);
        red64(s + 3, dur);
      }
      if (kMode == 3) red32(hist + (size_t)row * 64u + b, 1u);
    }
  }
}

template <int kMode>
double run(uint32_t* hist, uint64_t* lat, uint64_t* sect, uint32_t ept, int lanes_per_event, const char* name) {
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  const int blocks = sms * 4;
  k<kMode><<<blocks, 512>>>(hist, lat, sect, ept);   // warm
  cudaEventRecord(a);
  for (int r = 0; r < 5; ++r) k<kMode><<<blocks, 512>>>(hist, lat, sect, ept);
  cudaEventRecord(b);
  cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b);
  const double events = 5.0 * blocks * 512 / lanes_per_event * ept;
  printf("%-44s %8.3f ms / 5 launches  %7.2f G events/s  (%s)\n", name, ms, events / ms / 1e6, cudaGetErrorString(cudaGetLastError()));
  return events / ms / 1e6;
}

int main() {
  uint32_t* hist; uint64_t *lat, *sect;
  cudaMalloc(&hist, (size_t)kRows * 64 * 4); cudaMalloc(&lat, (size_t)kRows * 8);
  cudaMalloc(&sect, (size_t)kRows * kSectorsPerRow * 32);
  cudaMemset(hist, 0, (size_t)kRows * 64 * 4); cudaMemset(lat, 0, (size_t)kRows * 8);
  cudaMemset(sect, 0, (size_t)kRows * kSectorsPerRow * 32);
  const uint32_t ept = 64;
  run<0>(hist, lat, sect, ept, 1, "A red.u32 + red.u64, two sectors");
  run<1>(hist, lat, sect, ept, 1, "B red.u32 + red.u64, one sector");
  run<2>(hist, lat, sect, ept, 2, "C one red.u64, lane pairs share a sector");
  run<3>(hist, lat, sect, ept, 1, "D red.u32 only");
  run<4>(hist, lat, sect, ept, 4, "E one red.u64, four lanes share a sector");
  return 0;
}
