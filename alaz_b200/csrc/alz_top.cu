// alz_top.cu — the top-row selection of docs/SPEC.md §16 and §17, on 32-bit values (GNN scores) and 64-bit values
// (edge metrics). A radix select on the inverted key ik = ~key (ascending ik = rank order), state on the device:
//   hist<P>  digit P (11-bit digits from the top, the last one or two of 10 bits) of every value whose higher digits
//            equal the prefix so far: a shared-memory histogram per CTA, added into one global histogram; pass 0 also
//            counts the eligible values (ik <= ~key(min)) and takes the largest key
//   pick<P>  one CTA: the digit the remaining rank falls into; prefix and remaining rank stay in device memory
//   after the last pass the threshold T is the m-th smallest ik and r of the values with ik == T are taken, lowest
//   index first:
//   count    per tile of 4096 values, those with ik < T and those with ik == T, packed (lt << 32 | eq); an in-place
//            exclusive scan gives each tile the candidates and the ties before it
//   emit     every value with ik < T and the ties of rank < r: m candidates ik - ik_min, in ascending index order
// One wait reads the control block; a stable radix sort of the m candidates over the bits that can differ puts them
// in rank order (equal keys stay in index order), and the gather copies index, value and row of each. Values are
// read 2 + passes times; rows only for the m results.
#include <algorithm>

#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "alz_top.cuh"

namespace alz {
namespace top {
namespace {

// pass P: digit = (ik >> kShift[P]) & (2^kBits[P] - 1), prefix = ik >> (kShift[P] + kBits[P])
template <class U> struct Digits;
template <> struct Digits<uint32_t> {
  static constexpr int kPasses = 3;
  static constexpr uint32_t kShift[3] = {21, 10, 0}, kBits[3] = {11, 11, 10};
};
template <> struct Digits<uint64_t> {
  static constexpr int kPasses = 6;
  static constexpr uint32_t kShift[6] = {53, 42, 31, 20, 10, 0}, kBits[6] = {11, 11, 11, 11, 10, 10};
};

__device__ __forceinline__ uint32_t warp_max(uint32_t x) { return __reduce_max_sync(0xFFFFFFFFu, x); }
__device__ __forceinline__ uint64_t warp_max(uint64_t x) {
  for (int o = 16; o > 0; o >>= 1) x = max(x, (uint64_t)__shfl_xor_sync(0xFFFFFFFFu, (unsigned long long)x, o));
  return x;
}
__device__ __forceinline__ void atomic_max(uint32_t* p, uint32_t x) { atomicMax(p, x); }
__device__ __forceinline__ void atomic_max(uint64_t* p, uint64_t x) {
  atomicMax(reinterpret_cast<unsigned long long*>(p), (unsigned long long)x);
}

template <class U, int P>
__global__ void __launch_bounds__(kThreads) top_hist_kernel(const U* __restrict__ s, uint32_t n, U ik_elig,
                                                            uint32_t* __restrict__ hist, Ctl<U>* __restrict__ ctl) {
  constexpr uint32_t kShift = Digits<U>::kShift[P], kBins = 1u << Digits<U>::kBits[P];
  constexpr uint32_t kHi = P == 0 ? 0u : kShift + Digits<U>::kBits[P];   // the prefix's bits: ik >> kHi (pass 0: none)
  __shared__ uint32_t sh[kBins];
  if (P > 0 && ctl->m == 0) return;
  const U prefix = P > 0 ? ctl->prefix : (U)0;
  for (uint32_t b = threadIdx.x; b < kBins; b += kThreads) sh[b] = 0;
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31u;
  uint32_t above = 0;
  U key_max = 0;
  // i0 is the same in every lane of a warp: the whole warp reaches the __match_any_sync
  for (uint32_t i0 = blockIdx.x * kThreads + (threadIdx.x & ~31u); i0 < n; i0 += gridDim.x * kThreads) {
    const uint32_t i = i0 + lane;
    uint32_t d = 0xFFFFFFFFu;
    if (i < n) {
      const U key = order_key(s[i]), ik = ~key;
      if (P == 0) {
        above += ik <= ik_elig;
        key_max = max(key_max, key);
      }
      if (P == 0 || (ik >> kHi) == prefix) d = (uint32_t)(ik >> kShift) & (kBins - 1);
    }
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, d);   // one shared atomic per distinct digit of the warp
    if (d != 0xFFFFFFFFu && lane == (uint32_t)__ffs(peers) - 1u) atomicAdd(&sh[d], (uint32_t)__popc(peers));
  }
  if (P == 0) {
    above = __reduce_add_sync(0xFFFFFFFFu, above);
    key_max = warp_max(key_max);
    if (lane == 0) {
      if (above) atomicAdd(&ctl->above, above);
      atomic_max(&ctl->key_max, key_max);
    }
  }
  __syncthreads();
  for (uint32_t b = threadIdx.x; b < kBins; b += kThreads)
    if (sh[b]) atomicAdd(&hist[b], sh[b]);
}

// one CTA of 1024 threads, 2 bins each: the digit whose bucket holds the remaining rank; the histogram is cleared for
// the next pass
template <class U, int P>
__global__ void __launch_bounds__(1024) top_pick_kernel(uint32_t k, uint32_t* __restrict__ hist,
                                                        Ctl<U>* __restrict__ ctl) {
  using Scan = cub::BlockScan<uint32_t, 1024>;
  __shared__ typename Scan::TempStorage tmp;
  const uint32_t t = threadIdx.x;
  const uint32_t m = P == 0 ? min(k, ctl->above) : ctl->m;
  const uint32_t rank = P == 0 ? m : ctl->rank;
  const U prefix = P == 0 ? (U)0 : ctl->prefix;
  const uint32_t a = hist[2 * t], b = hist[2 * t + 1];
  hist[2 * t] = hist[2 * t + 1] = 0;
  if (P == 0 && t == 0) ctl->m = m;
  if (m == 0) return;                                  // the same in every thread
  uint32_t ex;
  Scan(tmp).ExclusiveSum(a + b, ex);
  constexpr uint32_t bits = Digits<U>::kBits[P];
  if (ex < rank && rank <= ex + a) {
    ctl->prefix = (U)(prefix << bits) | (U)(2 * t);
    ctl->rank = rank - ex;
  } else if (ex + a < rank && rank <= ex + a + b) {
    ctl->prefix = (U)(prefix << bits) | (U)(2 * t + 1);
    ctl->rank = rank - ex - a;
  }
}

// per tile: (values with ik < T) << 32 | (values with ik == T)
template <class U>
__global__ void __launch_bounds__(kThreads) top_count_kernel(const U* __restrict__ s, uint32_t n,
                                                             const Ctl<U>* __restrict__ ctl,
                                                             uint64_t* __restrict__ cnt) {
  if (ctl->m == 0) return;
  const U T = ctl->prefix;
  __shared__ uint32_t lt_total, eq_total;
  if (threadIdx.x == 0) lt_total = eq_total = 0;
  __syncthreads();
  uint32_t lt = 0, eq = 0;
  for (uint32_t j = 0; j < kRounds; ++j) {
    const uint32_t i = blockIdx.x * kTile + j * kThreads + threadIdx.x;
    if (i < n) {
      const U ik = ~order_key(s[i]);
      lt += ik < T;
      eq += ik == T;
    }
  }
  lt = __reduce_add_sync(0xFFFFFFFFu, lt);
  eq = __reduce_add_sync(0xFFFFFFFFu, eq);
  if ((threadIdx.x & 31u) == 0) {
    if (lt) atomicAdd(&lt_total, lt);
    if (eq) atomicAdd(&eq_total, eq);
  }
  __syncthreads();
  if (threadIdx.x == 0) cnt[blockIdx.x] = ((uint64_t)lt_total << 32) | eq_total;
}

// warp 0: exclusive scan of the kRounds * kWarps = 128 counts in a, 4 per lane
__device__ __forceinline__ void scan128(uint32_t* a, uint32_t lane) {
  uint32_t v[4], sum = 0;
#pragma unroll
  for (int q = 0; q < 4; ++q) { v[q] = a[lane * 4 + q]; sum += v[q]; }
  uint32_t incl = sum;
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t x = __shfl_up_sync(0xFFFFFFFFu, incl, o);
    if ((int)lane >= o) incl += x;
  }
  uint32_t run = incl - sum;
#pragma unroll
  for (int q = 0; q < 4; ++q) { a[lane * 4 + q] = run; run += v[q]; }
}
static_assert(kRounds * kWarps == 128, "scan128 covers one tile's (round, warp) counts");

// per tile, in index order (round j, warp w, lane l holds value tile + 256 j + 32 w + l): the candidates, each at its
// place in ascending index order; base[tile] = the packed exclusive scan of the counts
template <class U>
__global__ void __launch_bounds__(kThreads) top_emit_kernel(const U* __restrict__ s, uint32_t n,
                                                            const Ctl<U>* __restrict__ ctl,
                                                            const uint64_t* __restrict__ base,
                                                            U* __restrict__ cand_key, uint32_t* __restrict__ cand_idx) {
  if (ctl->m == 0) return;
  const U T = ctl->prefix, ik_min = ~ctl->key_max;
  const uint32_t r = ctl->rank;
  __shared__ uint32_t ties[kRounds * kWarps];          // ties per (round, warp), then their exclusive scan
  __shared__ uint32_t kept[kRounds * kWarps];          // candidates per (round, warp), then their exclusive scan
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, lt = (1u << lane) - 1u;
  U ik[kRounds];
  uint32_t mask[kRounds];                              // ties, then candidates
#pragma unroll
  for (uint32_t j = 0; j < kRounds; ++j) {
    const uint32_t i = blockIdx.x * kTile + j * kThreads + threadIdx.x;
    ik[j] = i < n ? (U)~order_key(s[i]) : (U)~(U)0;
    mask[j] = __ballot_sync(0xFFFFFFFFu, i < n && ik[j] == T);
    if (lane == 0) ties[j * kWarps + warp] = __popc(mask[j]);
  }
  __syncthreads();
  if (warp == 0) scan128(ties, lane);
  __syncthreads();
  const uint64_t b = base[blockIdx.x];
  const uint32_t tie_base = (uint32_t)b, out_base = (uint32_t)(b >> 32) + min(r, tie_base);
#pragma unroll
  for (uint32_t j = 0; j < kRounds; ++j) {
    const uint32_t i = blockIdx.x * kTile + j * kThreads + threadIdx.x;
    const uint32_t tie_rank = tie_base + ties[j * kWarps + warp] + __popc(mask[j] & lt);
    const bool keep = i < n && (ik[j] < T || (ik[j] == T && tie_rank < r));
    mask[j] = __ballot_sync(0xFFFFFFFFu, keep);
    if (lane == 0) kept[j * kWarps + warp] = __popc(mask[j]);
  }
  __syncthreads();
  if (warp == 0) scan128(kept, lane);
  __syncthreads();
#pragma unroll
  for (uint32_t j = 0; j < kRounds; ++j) {
    if (mask[j] >> lane & 1u) {
      const uint32_t pos = out_base + kept[j * kWarps + warp] + __popc(mask[j] & lt);
      cand_key[pos] = ik[j] - ik_min;
      cand_idx[pos] = blockIdx.x * kTile + j * kThreads + threadIdx.x;
    }
  }
}

// result j: the index, value and (with rows) row of the j-th candidate in sorted order; a warp per result
template <class U>
__global__ void __launch_bounds__(kThreads) top_gather_kernel(const uint32_t* __restrict__ sorted_idx, uint32_t m,
                                                              const U* __restrict__ s,
                                                              const alz_edge_out* __restrict__ rows,
                                                              uint32_t* __restrict__ out_index, U* __restrict__ out_vals,
                                                              alz_edge_out* __restrict__ out_rows) {
  constexpr uint32_t kWords = sizeof(alz_edge_out) / 8;
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t warps_per_grid = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < m; j += warps_per_grid) {
    const uint32_t i = sorted_idx[j];
    if (lane == 0) { out_index[j] = i; out_vals[j] = s[i]; }
    if (rows) {
      const uint64_t* src = reinterpret_cast<const uint64_t*>(rows + i);
      uint64_t* dst = reinterpret_cast<uint64_t*>(out_rows + j);
      for (uint32_t w = lane; w < kWords; w += 32) dst[w] = src[w];
    }
  }
}
static_assert(sizeof(alz_edge_out) % 8 == 0, "rows are copied in 8-byte words");

template <class U, int P>
void launch_passes(uint32_t grid, cudaStream_t st, const U* vals, uint32_t n, uint32_t k, U ik_elig, uint32_t* hist,
                   Ctl<U>* ctl) {
  top_hist_kernel<U, P><<<grid, kThreads, 0, st>>>(vals, n, ik_elig, hist, ctl);
  top_pick_kernel<U, P><<<1, 1024, 0, st>>>(k, hist, ctl);
  if constexpr (P + 1 < Digits<U>::kPasses) launch_passes<U, P + 1>(grid, st, vals, n, k, ik_elig, hist, ctl);
}

int bits_for(uint64_t x) { int b = 1; while (b < 64 && (x >> b) != 0) ++b; return b; }
}  // namespace

template <class U> size_t tmp_bytes(uint32_t n, uint32_t m_max) {
  size_t a = 0, b = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, a, (const U*)nullptr, (U*)nullptr, (const uint32_t*)nullptr,
                                  (uint32_t*)nullptr, (int)std::max(m_max, 1u));
  cub::DeviceScan::ExclusiveSum(nullptr, b, (uint64_t*)nullptr, (uint64_t*)nullptr, (int)std::max(tiles(n), 1u));
  return std::max(a, b);
}

template <class U> int select_candidates(alz_handle* h, const U* vals, uint32_t n, uint32_t k, U min_bits,
                                         const Scratch& s, Ctl<U>* c) {
  *c = Ctl<U>{};
  if (n == 0) return ALZ_OK;
  cudaStream_t st = h->stream;
  uint32_t* hist = s.words;
  Ctl<U>* ctl = reinterpret_cast<Ctl<U>*>(s.words + kHistWords);
  const uint32_t nt = tiles(n);
  const unsigned grid = std::min<unsigned>(nt, (unsigned)h->sms * 2);
  CK(cudaMemsetAsync(s.words, 0, kWordsBytes, st));
  launch_passes<U, 0>(grid, st, vals, n, k, (U)~order_key(min_bits), hist, ctl);
  top_count_kernel<U><<<nt, kThreads, 0, st>>>(vals, n, ctl, s.tile_cnt);
  size_t tmp_bytes = s.tmp_bytes;
  CK(cub::DeviceScan::ExclusiveSum(s.tmp, tmp_bytes, s.tile_cnt, s.tile_cnt, (int)nt, st));
  top_emit_kernel<U><<<nt, kThreads, 0, st>>>(vals, n, ctl, s.tile_cnt, (U*)s.cand_key, s.cand_idx);
  h->launches += 2 * Digits<U>::kPasses + 2;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(c, ctl, sizeof(Ctl<U>), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return ALZ_OK;
}

template <class U> int select_results(alz_handle* h, const U* vals, uint32_t n, const Ctl<U>& c,
                                      const alz_edge_out* rows, const Scratch& s, uint32_t* out_index, U* out_vals,
                                      alz_edge_out* out_rows) {
  (void)n;
  if (c.m == 0) return ALZ_OK;
  cudaStream_t st = h->stream;
  const U ik_min = ~c.key_max;
  size_t tmp_bytes = s.tmp_bytes;
  CK(cub::DeviceRadixSort::SortPairs(s.tmp, tmp_bytes, (const U*)s.cand_key, (U*)s.sorted_key, s.cand_idx,
                                     s.sorted_idx, (int)c.m, 0, bits_for((uint64_t)(U)(c.prefix - ik_min)), st));
  return gather<U>(h, s.sorted_idx, c.m, vals, rows, out_index, out_vals, out_rows);
}

template <class U> int gather(alz_handle* h, const uint32_t* idx, uint32_t m, const U* vals, const alz_edge_out* rows,
                              uint32_t* out_index, U* out_vals, alz_edge_out* out_rows) {
  if (m == 0) return ALZ_OK;
  top_gather_kernel<U><<<std::min<unsigned>((m + kWarps - 1) / kWarps, (unsigned)h->sms * 4), kThreads, 0,
                         h->stream>>>(idx, m, vals, rows, out_index, out_vals, out_rows);
  h->launches += 1;
  CK(cudaGetLastError());
  return ALZ_OK;
}

#define ALZ_TOP_INSTANTIATE(U)                                                                                      \
  template size_t tmp_bytes<U>(uint32_t, uint32_t);                                                                 \
  template int select_candidates<U>(alz_handle*, const U*, uint32_t, uint32_t, U, const Scratch&, Ctl<U>*);        \
  template int select_results<U>(alz_handle*, const U*, uint32_t, const Ctl<U>&, const alz_edge_out*,              \
                                 const Scratch&, uint32_t*, U*, alz_edge_out*);                                     \
  template int gather<U>(alz_handle*, const uint32_t*, uint32_t, const U*, const alz_edge_out*, uint32_t*, U*,      \
                         alz_edge_out*);
ALZ_TOP_INSTANTIATE(uint32_t)
ALZ_TOP_INSTANTIATE(uint64_t)
#undef ALZ_TOP_INSTANTIATE
}  // namespace top
}  // namespace alz
