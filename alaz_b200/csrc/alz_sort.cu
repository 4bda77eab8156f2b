// alz_sort.cu — key/value radix sort and prefix scan used once per window flush
// (canonical edge order, cross-rank key merge, CSR build). Off the per-event
// hot path; uses the CUDA toolkit's CUB device primitives.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include "alz_kernels.cuh"

namespace alz {
size_t sort_pairs_temp_bytes(uint32_t n) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                  (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n);
  return bytes;
}
cudaError_t sort_pairs(void* temp, size_t temp_bytes, const uint64_t* keys_in, uint64_t* keys_out,
                       const uint32_t* vals_in, uint32_t* vals_out, uint32_t n, cudaStream_t s, int end_bit) {
  // end_bit: only key bits [0, end_bit) differ between keys (each 8 bits less is one pass over the data less)
  return cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys_in, keys_out, vals_in, vals_out, (int)n, 0, end_bit, s);
}
size_t scan_temp_bytes(uint32_t n) {
  size_t bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n);
  return bytes;
}
cudaError_t exclusive_scan_u32(void* temp, size_t temp_bytes, const uint32_t* in, uint32_t* out, uint32_t n,
                               cudaStream_t s) {
  return cub::DeviceScan::ExclusiveSum(temp, temp_bytes, in, out, (int)n, s);
}
}  // namespace alz
