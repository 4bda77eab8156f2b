// alz_sort.cu — key/value radix sort and prefix scan used once per window flush
// (canonical edge order, cross-rank key merge, CSR build). Off the per-event
// hot path; uses the CUDA toolkit's CUB device primitives.
#include <algorithm>

#include <cooperative_groups.h>
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
size_t sort_keys_temp_bytes(uint32_t n) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)n);
  return bytes;
}
cudaError_t sort_keys(void* temp, size_t temp_bytes, const uint64_t* keys_in, uint64_t* keys_out, uint32_t n,
                      cudaStream_t s, int end_bit) {
  return cub::DeviceRadixSort::SortKeys(temp, temp_bytes, keys_in, keys_out, (int)n, 0, end_bit, s);
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

// ---- the single-rank flush's sort of the live edge keys, sized on the device --------------------------------------
// Edge keys are unique and keep `rev | other_type | pod_id` in the high word (make_edge_key). A counting sort on the
// high word puts each (rev, type, pod) in its own segment, in key order; pod ids from pods - 1 up share the last
// segment of their (rev, type), so every segment is sorted on the whole key below. Small segments are ranked by a
// thread per key, larger ones sorted in shared memory by a block per 4096-key chunk, and the chunks of a segment of
// several (a hub: one pod with many outbound addresses) merged pairwise, runs of 4096 << p keys in pass p, so a
// segment of M keys costs M * log2(M / 4096) binary searches. Every kernel reads the live row count from the edge
// table's allocator, so the host enqueues the sort without knowing it.
namespace alz {
namespace {
constexpr uint32_t kRankSeg = 256;      // segments up to this size: a thread per key counts the smaller keys
constexpr uint32_t kChunk = 4096;       // keys a block sorts in shared memory
constexpr uint32_t kChunkThreads = 1024;

__device__ __forceinline__ uint32_t live_rows(const EdgeTable& t) { return min(*t.n_rows, t.max_rows); }
__device__ __forceinline__ uint32_t key_bucket(uint64_t key, uint32_t pods) {
  const uint32_t hi = (uint32_t)(key >> 32);
  return (hi >> 29) * pods + min(hi & 0x1FFFFFFFu, pods - 1u);
}

// keys per bucket, one atomic per bucket and warp (a hub's keys all land on one word); also empties the list of
// large segments the last sort left
__global__ void __launch_bounds__(256) key_hist_kernel(EdgeTable t, uint32_t pods, uint32_t* __restrict__ cnt,
                                                       uint32_t* __restrict__ n_large) {
  if (blockIdx.x == 0 && threadIdx.x == 0) { n_large[0] = 0u; n_large[1] = 0u; }
  const uint32_t n = live_rows(t), lane = threadIdx.x & 31u;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t base = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < n; base += stride) {
    const uint32_t i = base + lane;
    const uint32_t b = i < n ? key_bucket(t.row_key[i], pods) : ~0u;
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, b);
    if (i < n && lane == (uint32_t)__ffs(peers) - 1u) atomicAdd(&cnt[b], (uint32_t)__popc(peers));
  }
}
// each edge row to a place in its bucket (in no particular order); counts cnt back down to zero for the next sort
__global__ void __launch_bounds__(256) key_scatter_kernel(EdgeTable t, uint32_t pods, uint32_t* __restrict__ cnt,
                                                          const uint32_t* __restrict__ off, uint64_t* __restrict__ keys,
                                                          uint32_t* __restrict__ rows) {
  const uint32_t n = live_rows(t), lane = threadIdx.x & 31u;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t base = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < n; base += stride) {
    const uint32_t i = base + lane;
    const uint64_t k = i < n ? t.row_key[i] : 0ull;
    const uint32_t b = i < n ? key_bucket(k, pods) : ~0u;
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, b);
    const uint32_t leader = (uint32_t)__ffs(peers) - 1u;
    uint32_t top = 0;
    if (i < n && lane == leader) top = atomicSub(&cnt[b], (uint32_t)__popc(peers));
    top = __shfl_sync(0xFFFFFFFFu, top, leader);
    if (i < n) {
      const uint32_t p = off[b] + top - 1u - (uint32_t)__popc(peers & ((1u << lane) - 1u));
      keys[p] = k;
      rows[p] = i;
    }
  }
}
// a key of a small segment straight to its place; the first key of a larger segment lists the segment and raises
// the largest chunk count (n_large[1])
__global__ void __launch_bounds__(256) seg_rank_kernel(EdgeTable t, uint32_t pods, const uint32_t* __restrict__ off,
                                                       const uint64_t* __restrict__ keys, const uint32_t* __restrict__ rows,
                                                       uint64_t* __restrict__ keys_out, uint32_t* __restrict__ rows_out,
                                                       uint32_t* __restrict__ large, uint32_t* __restrict__ n_large) {
  const uint32_t n = live_rows(t);
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
    const uint64_t k = keys[p];
    const uint32_t b = key_bucket(k, pods);
    const uint32_t s = off[b], e = off[b + 1u];
    if (e - s > kRankSeg) {
      if (p == s) {
        large[atomicAdd(&n_large[0], 1u)] = b;
        atomicMax(&n_large[1], (e - s + kChunk - 1u) / kChunk);
      }
      continue;
    }
    uint32_t r = s;
    for (uint32_t q = s; q < e; ++q) r += keys[q] < k ? 1u : 0u;
    keys_out[r] = k;
    rows_out[r] = rows[p];
  }
}
// merge passes a segment of `chunks` chunks needs
__device__ __forceinline__ uint32_t merge_passes(uint32_t chunks) { return chunks <= 1u ? 0u : 32u - __clz(chunks - 1u); }

// chunk c of a large segment sorted in shared memory (bitonic over the next power of two, padded with the largest
// key); a segment of one chunk goes to its place, a longer one's chunks to where seg_merge_kernel's first pass reads
// them: the output when the merge takes an even number of passes, keys / rows otherwise
__global__ void __launch_bounds__(kChunkThreads) seg_chunk_kernel(const uint32_t* __restrict__ off,
                                                                  const uint32_t* __restrict__ large,
                                                                  const uint32_t* __restrict__ n_large,
                                                                  uint64_t* __restrict__ keys, uint32_t* __restrict__ rows,
                                                                  uint64_t* __restrict__ keys_out,
                                                                  uint32_t* __restrict__ rows_out) {
  __shared__ uint64_t sk[kChunk];
  __shared__ uint32_t sr[kChunk];
  const uint32_t nl = n_large[0];
  const bool odd = merge_passes(n_large[1]) & 1u;
  uint32_t w = 0;   // work item: (segment j, chunk c) in list order
  for (uint32_t j = 0; j < nl; ++j) {
    const uint32_t b = large[j];
    const uint32_t s = off[b], e = off[b + 1u];
    const uint32_t chunks = (e - s + kChunk - 1u) / kChunk;
    for (uint32_t c = 0; c < chunks; ++c, ++w) {
      if (w % gridDim.x != blockIdx.x) continue;
      const uint32_t lo = s + c * kChunk, len = min(kChunk, e - lo);
      uint32_t m = 1;
      while (m < len) m <<= 1;
      for (uint32_t i = threadIdx.x; i < m; i += blockDim.x) {
        sk[i] = i < len ? keys[lo + i] : ~0ull;
        sr[i] = i < len ? rows[lo + i] : 0u;
      }
      __syncthreads();
      for (uint32_t size = 2; size <= m; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
          for (uint32_t t = threadIdx.x; t < m / 2u; t += blockDim.x) {
            const uint32_t i = 2u * t - (t & (stride - 1u)), x = i + stride;
            const bool up = (i & size) == 0u;
            const uint64_t a = sk[i], d = sk[x];
            if ((a > d) == up) {
              sk[i] = d; sk[x] = a;
              const uint32_t ra = sr[i]; sr[i] = sr[x]; sr[x] = ra;
            }
          }
          __syncthreads();
        }
      }
      const bool to_out = chunks == 1u || !odd;
      uint64_t* ko = to_out ? keys_out : keys;
      uint32_t* ro = to_out ? rows_out : rows;
      for (uint32_t i = threadIdx.x; i < len; i += blockDim.x) { ko[lo + i] = sk[i]; ro[lo + i] = sr[i]; }
      __syncthreads();
    }
  }
}
// The segments of several chunks, pairwise merged: pass p merges sorted runs of kChunk << p keys into runs twice as
// long, from one buffer into the other, ending in the output. A key's place in the merged run is its index in its
// own run plus its lower bound in the partner run (keys are unique); a run without a partner is copied. One
// cooperative launch, a grid-wide barrier between passes; segments that need fewer passes than the largest are copied
// along.
__global__ void __launch_bounds__(256) seg_merge_kernel(const uint32_t* __restrict__ off, const uint32_t* __restrict__ large,
                                                        const uint32_t* __restrict__ n_large, uint64_t* keys,
                                                        uint32_t* rows, uint64_t* keys_out, uint32_t* rows_out) {
  const uint32_t nl = n_large[0];
  const uint32_t passes = merge_passes(n_large[1]);
  if (passes == 0u) return;   // the same in every block
  cooperative_groups::grid_group grid = cooperative_groups::this_grid();
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t p = 0; p < passes; ++p) {
    // the last pass writes the output
    const bool into_out = ((passes - 1u - p) & 1u) == 0u;
    const uint64_t* ks = into_out ? keys : keys_out;
    const uint32_t* rs = into_out ? rows : rows_out;
    uint64_t* kd = into_out ? keys_out : keys;
    uint32_t* rd = into_out ? rows_out : rows;
    const uint32_t run = kChunk << p;
    for (uint32_t j = 0; j < nl; ++j) {
      const uint32_t b = large[j];
      const uint32_t s = off[b], len = off[b + 1u] - s;
      if (len <= kChunk) continue;
      for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < len; i += stride) {
        const uint32_t r0 = i / run * run;              // own run [r0, r0 + run)
        const uint32_t pair = i / (2u * run) * (2u * run);
        const uint32_t mate = r0 == pair ? pair + run : pair;
        const uint64_t k = ks[s + i];
        uint32_t d = i;
        if (mate < len) {
          const uint32_t rank = lower_bound_u64(ks + s + mate, min(run, len - mate), k);
          d = pair + (i - r0) + rank;
        }
        kd[s + d] = k;
        rd[s + d] = rs[s + i];
      }
    }
    grid.sync();
  }
}
}  // namespace

size_t edge_sort_temp_bytes(uint32_t pods) { return scan_temp_bytes(8u * pods + 1u); }

cudaError_t edge_sort(const EdgeTable& t, const EdgeSortScratch& x, uint64_t* keys_out, uint32_t* rows_out, int sms,
                      cudaStream_t s) {
  const unsigned grid = (unsigned)sms * 4u;
  const uint32_t nb = 8u * x.pods;
  key_hist_kernel<<<grid, 256, 0, s>>>(t, x.pods, x.cnt, x.n_large);
  cudaError_t e = exclusive_scan_u32(x.temp, x.temp_bytes, x.cnt, x.off, nb + 1u, s);
  if (e != cudaSuccess) {   // the counts go back to zero, as the next sort expects them
    cudaMemsetAsync(x.cnt, 0, (size_t)(nb + 1u) * 4, s);
    return e;
  }
  key_scatter_kernel<<<grid, 256, 0, s>>>(t, x.pods, x.cnt, x.off, x.keys, x.rows);
  seg_rank_kernel<<<grid, 256, 0, s>>>(t, x.pods, x.off, x.keys, x.rows, keys_out, rows_out, x.large, x.n_large);
  seg_chunk_kernel<<<(unsigned)sms * 2u, kChunkThreads, 0, s>>>(x.off, x.large, x.n_large, x.keys, x.rows, keys_out,
                                                                rows_out);
  // every block of the merge must be resident at once for its grid barrier
  int per_sm = 0;
  if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, seg_merge_kernel, 256, 0)) != cudaSuccess) return e;
  const uint32_t* off = x.off; const uint32_t* large = x.large; const uint32_t* n_large = x.n_large;
  uint64_t* keys = x.keys; uint32_t* rows = x.rows;
  void* args[] = {&off, &large, &n_large, &keys, &rows, &keys_out, &rows_out};
  e = cudaLaunchCooperativeKernel((const void*)seg_merge_kernel, dim3((unsigned)sms * (unsigned)std::min(per_sm, 8)),
                                  dim3(256), args, 0, s);
  return e != cudaSuccess ? e : cudaGetLastError();
}
}  // namespace alz
