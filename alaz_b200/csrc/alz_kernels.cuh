// alz_kernels.cuh — launcher declarations shared by the kernels and the C-ABI layer.
#pragma once
#include "alz_device.cuh"
#include "../synth/alz_synth.h"

namespace alz {
// time-cut windows (SURVEY §8 row R13, docs/SPEC.md §8): the open window in the records' own (kernel) clock.
// The ingest reads it; a multi-rank merge copies it into the rank's block header (alz_comm.cu).
struct WinClock {
  uint64_t lo;        // first kernel-time ns of the open window
  uint64_t len;       // window length, ns
  uint64_t ready;     // 0: lo not set yet; 1: set (by win_init_kernel from the first record ever submitted, or by a
                      // merge that opened it after the ranks' agreed epoch); 2: the open epoch starts at or past 2^64
                      // in the user clock, so every record is late
  uint64_t off;       // first_user_ns - first_kernel_ns (mod 2^64)
  uint64_t epoch;     // epoch_open
};
void launch_ingest_pairs_v1(const alz_l7_rec* recs, uint64_t n, const PairTable& pairs, Counters* ctr,
                            const EpEntry* ep, uint32_t ep_mask, int sms, cudaStream_t s);
// cursor: the handle's claim cursors (ingest_cursor_bytes(), alz_ingest.cu ChunkSched), zeroed before every launch
void launch_ingest_pairs(const alz_l7_rec* recs, uint64_t n, const PairTable& pairs, Counters* ctr,
                         const HotState* hot, const EpEntry* ep, uint32_t ep_mask, const uint32_t* bloom,
                         uint32_t* cursor, int sms, cudaStream_t s);
void launch_ingest_pairs_rec16(const alz_l7_rec16* recs, uint64_t n, const uint64_t* dur_ovf, const PairTable& pairs,
                               Counters* ctr, const HotState* hot, const EpEntry* ep, uint32_t ep_mask,
                               const uint32_t* bloom, uint32_t* cursor, int sms, cudaStream_t s);
void launch_ingest_pairs_windowed(const alz_l7_rec* recs, uint64_t n, const PairTable& pairs, Counters* ctr,
                                  const HotState* hot, const EpEntry* ep, uint32_t ep_mask, const uint32_t* bloom,
                                  uint64_t* win, alz_l7_rec* defer_buf, uint32_t defer_cap, uint32_t* cursor, int sms,
                                  cudaStream_t s);
void launch_window_advance(uint64_t* win, cudaStream_t s);
void launch_defer_resolve(alz_l7_rec* buf, uint32_t lo, uint32_t hi, const EpEntry* ep, uint32_t ep_mask, Counters* ctr,
                          int sms, cudaStream_t s);
void launch_defer_roll(const alz_l7_rec* src, uint32_t n, const uint64_t* win, alz_l7_rec* dst, uint32_t cap,
                       const EdgeTable& edges, Counters* ctr, int sms, cudaStream_t s);
uint32_t ingest_table_rows();
size_t ingest_cursor_bytes();   // the handle's claim cursors (alz_ingest.cu, ChunkSched)
void launch_hot_select(const PairTable& pairs, HotState* hot, int sms, cudaStream_t s);
void launch_ingest_eager(const alz_l7_rec* recs, uint64_t n, const EpEntry* ep, uint32_t ep_mask,
                         const EdgeTable& edges, Counters* ctr, int sms, cudaStream_t s);
void launch_fold_resolve(const PairTable& pairs, const EpEntry* ep, uint32_t ep_mask, const EdgeTable& edges,
                         HotState* hot, int sms, cudaStream_t s);
void launch_fold_add(const PairTable& pairs, const EdgeTable& edges, Counters* ctr, HotState* hot, int sms,
                     cudaStream_t s);
void launch_ep_patch(EpEntry* tab, const void* patch, uint32_t n, int sms, cudaStream_t s);
void launch_iota(uint32_t* out, uint32_t n, int sms, cudaStream_t s);
// the distinct keys of sorted[0, n) into out, in order: out has pos[n - 1] + flags[n - 1] entries (alz_kernels.cu)
cudaError_t launch_unique_sorted(const uint64_t* sorted, uint32_t n, uint32_t* flags, uint32_t* pos, uint64_t* out,
                                 void* temp, size_t temp_bytes, int sms, cudaStream_t s);   // the scan's status
void launch_gather_edges(const EdgeTable& edges, const uint64_t* keys, const uint32_t* rows, uint32_t n_live,
                         alz_edge_out* out, int sms, cudaStream_t s);
// single-rank flush scratch: pair rows bucketed by edge row (alz_kernels.cu, emit_edges_kernel)
struct FlushBuckets {
  uint32_t* cnt;       // [max_edges + 1] pair rows per edge row; all zero between flushes
  uint32_t* off;       // [max_edges + 1] exclusive scan of cnt: bucket of edge row e = rows[off[e], off[e + 1])
  uint32_t* rows;      // [cap] bucketed pair rows from the front, rows that reach no edge row from the back
  uint32_t cap;        // max_pairs + kPairKinds
  uint32_t* n_stray;   // rows at the back of `rows`
};
void launch_bucket_count(const PairTable& pairs, uint32_t max_edges, const FlushBuckets& b, int sms, cudaStream_t s);
void launch_bucket_fill(const PairTable& pairs, uint32_t max_edges, const FlushBuckets& b, int sms, cudaStream_t s);
// b == nullptr: no pair rows to take. Emits the edge table's live rows, as many as its allocator counts.
void launch_emit_edges(const PairTable& pairs, const EdgeTable& edges, Counters* ctr, HotState* hot, const uint64_t* keys,
                       const uint32_t* rows, const FlushBuckets* b, bool with_edges, alz_edge_out* out, int sms,
                       cudaStream_t s);
// the pair dictionaries emptied from their claimed-slot log; reset_rows: the row allocator back to zero too
void launch_pair_dict_clear(const PairTable& pairs, bool reset_rows, int sms, cudaStream_t s);
void launch_compact_raw(const uint8_t* raw, uint64_t n, alz_l7_rec* out, int sms, cudaStream_t s);
void launch_synth(const alz_synth_view& v, uint64_t first, uint64_t n, alz_l7_rec* out, int sms, cudaStream_t s);
void launch_synth_owned(const alz_synth_view& v, uint64_t first, uint64_t n, uint32_t nranks, uint32_t rank,
                        alz_l7_rec* out, uint64_t cap, unsigned long long* n_written, int sms, cudaStream_t s);
// radix sort of (edge key, row) pairs by key (alz_sort.cu)
size_t sort_pairs_temp_bytes(uint32_t n);
// both return CUB's status: cudaErrorInvalidValue, with nothing enqueued, when temp_bytes is too small
cudaError_t sort_pairs(void* temp, size_t temp_bytes, const uint64_t* keys_in, uint64_t* keys_out,
                       const uint32_t* vals_in, uint32_t* vals_out, uint32_t n, cudaStream_t s, int end_bit = 64);
// radix sort of 64-bit keys alone, on bits [0, end_bit) (alz_sort.cu)
size_t sort_keys_temp_bytes(uint32_t n);
cudaError_t sort_keys(void* temp, size_t temp_bytes, const uint64_t* keys_in, uint64_t* keys_out, uint32_t n,
                      cudaStream_t s, int end_bit);
size_t scan_temp_bytes(uint32_t n);
cudaError_t exclusive_scan_u32(void* temp, size_t temp_bytes, const uint32_t* in, uint32_t* out, uint32_t n,
                               cudaStream_t s);
// single-rank flush: the live edge rows of a table sorted by key, sized on the device (alz_sort.cu). pods bounds the
// pod ids that get a segment of their own (any larger id still sorts right, in one shared segment).
struct EdgeSortScratch {
  uint32_t pods;
  uint32_t* cnt;       // [8 * pods + 1] all zero between sorts
  uint32_t* off;       // [8 * pods + 1]
  uint64_t* keys;      // [max_edges] keys bucketed by their high word
  uint32_t* rows;      // [max_edges]
  uint32_t* large;     // [max_edges / 257 + 1] buckets of segments too large for a thread per key
  uint32_t* n_large;   // [2] large segments listed, most 4096-key chunks in one of them
  void* temp;          // the scan's
  size_t temp_bytes;
};
size_t edge_sort_temp_bytes(uint32_t pods);
// kEdgeSortKernels launches of its own and a CUB scan; the scan's status, or the launches'
constexpr int kEdgeSortKernels = 5;
cudaError_t edge_sort(const EdgeTable& t, const EdgeSortScratch& x, uint64_t* keys_out, uint32_t* rows_out, int sms,
                      cudaStream_t s);
}  // namespace alz
