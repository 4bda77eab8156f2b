// alz_top.cuh — the device selection of the top rows (docs/SPEC.md §16, §17): the first min(k, above) of n values in
// rank order, over 32-bit values (GNN scores, float32) or 64-bit values (edge metrics, float64). Each value's bits u
// map to the IEEE total-order key u ^ sign (sign bit clear) or ~u (set); rows rank by key descending, then by index
// ascending; a row is eligible when key >= key(min). Callers own the scratch and the result buffers.
#pragma once
#include <cstdint>

#include "alz_handle.h"

namespace alz {
namespace top {
constexpr uint32_t kThreads = 256, kRounds = 16, kTile = kThreads * kRounds, kWarps = kThreads / 32;
constexpr uint32_t kHistWords = 2048;   // the widest digit: 11 bits

// The selection's device-side control block; after select_candidates, its host copy
template <class U> struct Ctl {
  uint32_t above;     // eligible values
  uint32_t m;         // results: min(k, above)
  uint32_t rank;      // remaining rank within the prefix so far; after the last pass, ties at T taken
  U prefix;          // digits picked so far; after the last pass, the threshold T (an inverted key)
  U key_max;          // the largest key of all values
};
// the histogram, then the control block
constexpr size_t kWordsBytes = kHistWords * 4 + sizeof(Ctl<uint64_t>);

inline uint32_t tiles(uint32_t n) { return (n + kTile - 1) / kTile; }

// the IEEE total-order key of a value's bits: ascending keys are ascending values
template <class U> __host__ __device__ __forceinline__ U order_key(U u) {
  constexpr U kSign = (U)1 << (sizeof(U) * 8 - 1);
  return (u & kSign) ? (U)~u : (U)(u ^ kSign);
}

// Device scratch for a selection over n values with at most m_max = min(n, k) results
struct Scratch {
  uint32_t* words;        // kWordsBytes
  uint64_t* tile_cnt;     // tiles(n) words
  void* cand_key;         // m_max keys of the value width
  uint32_t* cand_idx;     // m_max
  void* sorted_key;       // m_max keys of the value width
  uint32_t* sorted_idx;   // m_max
  void* tmp;              // CUB scratch: at least tmp_bytes<U>(n, m_max)
  size_t tmp_bytes;
};
// the CUB scratch a selection over n values of width U with at most m_max results needs
template <class U> size_t tmp_bytes(uint32_t n, uint32_t m_max);

// Radix select and candidate emit on the device, then one wait: *c = the control block (c->m results, c->above
// eligible). min_bits: the bits of the minimum value.
template <class U> int select_candidates(alz_handle* h, const U* vals, uint32_t n, uint32_t k, U min_bits,
                                         const Scratch& s, Ctl<U>* c);
// The c.m results in rank order: out_index[j], out_vals[j] (the value's bits) and, with rows, out_rows[j]
template <class U> int select_results(alz_handle* h, const U* vals, uint32_t n, const Ctl<U>& c,
                                      const alz_edge_out* rows, const Scratch& s, uint32_t* out_index, U* out_vals,
                                      alz_edge_out* out_rows);
// The gather of select_results on its own, on the stream: for j < m, i = idx[j]: out_index[j] = i, out_vals[j] = vals[i]
// and, with rows, out_rows[j] = rows[i]
template <class U> int gather(alz_handle* h, const uint32_t* idx, uint32_t m, const U* vals, const alz_edge_out* rows,
                              uint32_t* out_index, U* out_vals, alz_edge_out* out_rows);
}  // namespace top
}  // namespace alz
