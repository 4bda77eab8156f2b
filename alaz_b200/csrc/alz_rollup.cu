// alz_rollup.cu — rolling windows (docs/SPEC.md §12): the rows of the last flushed windows kept on the device, and
// the sum of the last k of them as one edge list.
//
// Every accumulator of an output row is an integer sum (docs/SPEC.md §3), so the sum of k windows' rows per edge
// is what one window holding those windows' events would have returned. The flush is left as it is: a flush that
// consumed its window copies its rows into the arena (one device-to-device copy, no kernel, no synchronisation).
// A rollup has the shape of the single-rank flush (DESIGN.md §5.3) applied to output rows instead of pair rows:
// packed key of every retained row -> radix sort of (key, arena row) -> the distinct keys -> eight lanes per output
// row add up the key's run of source rows in registers and store the row once.
#include <algorithm>
#include <deque>
#include <new>
#include <vector>

#include "alz_handle.h"

using namespace alz;

namespace {
struct Entry {            // one retained window; host-side record of rows [first_row, first_row + n) of the arena
  uint64_t first_row, n;
  uint64_t window;        // alz_stats.windows after its flush
  uint32_t slot;          // its clock in d_clk
  bool clocked;           // a window clock was set when it was flushed
};
}  // namespace

struct alz_rollup_state {
  uint32_t depth = 0;
  uint64_t arena_rows = 0;
  alz_edge_out* d_arena = nullptr;
  WinClock* d_clk = nullptr;          // [depth] the clock of the epoch each entry's flush closed
  std::vector<WinClock> h_clk;
  std::deque<Entry> entries;          // oldest first: a contiguous run of the most recent consumed windows
  uint64_t appended = 0;              // entries ever appended: the next one's clock slot is appended % depth
  // rollup scratch, sized by the number of source rows (which max_edges does not bound), grown on demand
  uint32_t cap_rows = 0;
  uint64_t* d_keys[2] = {nullptr, nullptr};   // [cap_rows] packed keys of the source rows, unsorted / sorted
  uint32_t* d_src[2] = {nullptr, nullptr};    // [cap_rows] their arena rows
  uint64_t* d_ukeys = nullptr;                // [cap_rows] the distinct keys in order
  void* d_tmp = nullptr;                      // CUB scratch of the sort, then of the scan
  size_t tmp_bytes = 0;
  alz_edge_out* d_sum = nullptr;              // the last rollup's rows
  size_t sum_rows = 0;
};

// keys[i], src[i] = packed edge key and arena row of source row first_row + i (16 of the row's 296 bytes are read)
__global__ void __launch_bounds__(256) rollup_keys_kernel(const alz_edge_out* __restrict__ arena, uint32_t first_row,
                                                          uint32_t n, uint64_t* __restrict__ keys,
                                                          uint32_t* __restrict__ src) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    keys[i] = row_key_of(arena + first_row + i);
    src[i] = first_row + i;
  }
}

// Output row u = the sum of the source rows src[b, e), the run of ukeys[u] in sorted[0, n). Eight lanes per output
// row, a lane owning 8 histogram cells and lane 0 the three u64 sums as everywhere else (edge_row_load): lanes 0 and 1
// find the two ends of the run, every source row is read once and the output row is written once with plain
// stores. All sums wrap (u64 sums mod 2^64, cells mod 2^32, docs/SPEC.md §3).
__global__ void __launch_bounds__(256) rollup_emit_kernel(const alz_edge_out* __restrict__ arena,
                                                          const uint64_t* __restrict__ sorted,
                                                          const uint32_t* __restrict__ src, uint32_t n,
                                                          const uint64_t* __restrict__ ukeys, uint32_t n_out,
                                                          alz_edge_out* __restrict__ out) {
  const uint32_t lane = threadIdx.x & 31u, sl = lane & 7u;
  const uint32_t gmask = 0xFFu << (lane & ~7u);
  const uint32_t groups_per_grid = (gridDim.x * blockDim.x) >> 3;
  for (uint32_t u = (blockIdx.x * blockDim.x + threadIdx.x) >> 3; u < n_out; u += groups_per_grid) {
    const uint64_t key = ukeys[u];
    uint32_t end_of = 0;
    if (sl == 0) end_of = lower_bound_u64(sorted, n, key);
    if (sl == 1) end_of = u + 1u < n_out ? lower_bound_u64(sorted, n, ukeys[u + 1u]) : n;
    const uint32_t b = __shfl_sync(gmask, end_of, lane & ~7u), e = __shfl_sync(gmask, end_of, (lane & ~7u) + 1u);
    uint32_t c[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
    uint64_t count = 0, lat = 0, e5 = 0;
    for (uint32_t j = b; j < e; ++j) {
      uint32_t rc[8];
      uint64_t r_count, r_lat, r_e5;
      load_edge_out(arena + src[j], sl, rc, r_count, r_lat, r_e5);
#pragma unroll
      for (int q = 0; q < 8; ++q) c[q] += rc[q];
      count += r_count; lat += r_lat; e5 += r_e5;
    }
    store_edge_out(&out[u], sl, key, c, count, e5, lat);
  }
}

static void free_scratch(alz_rollup_state* st) {
  cudaFree(st->d_keys[0]); cudaFree(st->d_tmp);
  st->d_keys[0] = st->d_keys[1] = st->d_ukeys = nullptr;
  st->d_src[0] = st->d_src[1] = nullptr;
  st->d_tmp = nullptr;
  st->cap_rows = 0; st->tmp_bytes = 0;
}

void alz_internal_free_rollup(alz_handle* h) {
  alz_rollup_state* st = h->roll;
  if (!st) return;
  free_scratch(st);
  cudaFree(st->d_arena); cudaFree(st->d_clk); cudaFree(st->d_sum);
  delete st;
  h->roll = nullptr;
}

extern "C" int alz_window_history(alz_handle* h, uint32_t depth, uint64_t arena_rows) {
  if (!h || arena_rows >= (1ull << 31) || (depth != 0 && arena_rows == 0)) return ALZ_E_INVAL;   // rows are indexed by u32, counted by int
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  if (h->roll && h->roll->depth == depth && h->roll->arena_rows == arena_rows) return ALZ_OK;
  CK(cudaStreamSynchronize(h->stream));   // copies into the arena and a rollup's kernels may still be running
  alz_internal_free_rollup(h);
  if (depth == 0) return ALZ_OK;
  alz_rollup_state* st = new (std::nothrow) alz_rollup_state();
  if (!st) return ALZ_E_NOMEM;
  h->roll = st;
  st->depth = depth;
  st->arena_rows = arena_rows;
  st->h_clk.resize(depth);
  if (cudaMalloc(&st->d_arena, (size_t)arena_rows * sizeof(alz_edge_out)) != cudaSuccess ||
      cudaMalloc(&st->d_clk, (size_t)depth * sizeof(WinClock)) != cudaSuccess) {
    h->last_err = std::string("alz_window_history: ") + cudaGetErrorString(cudaGetLastError());
    alz_internal_free_rollup(h);
    return ALZ_E_NOMEM;
  }
  return ALZ_OK;
}

int alz_internal_history_append(alz_handle* h, const uint64_t* d_clk) {
  alz_rollup_state* st = h->roll;
  if (!st) return ALZ_OK;
  const uint64_t n = h->last_n_edges;
  if (n > st->arena_rows) { st->entries.clear(); return ALZ_OK; }   // not retained, and the run would have a gap
  // The arena is a ring in rows: the entry goes behind the newest one, or to row 0 when it would pass the end (the
  // rows skipped there are free again once the entries before them have gone). The oldest entries are evicted
  // until at most depth - 1 remain and the place overlaps none of the rest.
  uint64_t at = 0;
  for (;;) {
    while (st->entries.size() >= st->depth) st->entries.pop_front();
    at = st->entries.empty() ? 0 : st->entries.back().first_row + st->entries.back().n;
    if (at + n > st->arena_rows) at = 0;
    bool overlaps = false;
    for (const Entry& e : st->entries) overlaps |= at < e.first_row + e.n && e.first_row < at + n;
    if (!overlaps) break;
    st->entries.pop_front();
  }
  const uint32_t slot = (uint32_t)(st->appended++ % st->depth);
  if (n) CK(cudaMemcpyAsync(st->d_arena + at, h->d_out, (size_t)n * sizeof(alz_edge_out), cudaMemcpyDeviceToDevice, h->stream));
  if (d_clk) CK(cudaMemcpyAsync(st->d_clk + slot, d_clk, sizeof(WinClock), cudaMemcpyDeviceToDevice, h->stream));
  st->entries.push_back(Entry{at, n, h->windows, slot, d_clk != nullptr});
  return ALZ_OK;
}

// scratch for n source rows
static int ensure_scratch(alz_handle* h, alz_rollup_state* st, uint32_t n) {
  if (n <= st->cap_rows) return ALZ_OK;
  CK(cudaStreamSynchronize(h->stream));
  free_scratch(st);
  const uint32_t cap = (uint32_t)std::min<uint64_t>(st->arena_rows + 63u, ((uint64_t)n + n / 2u + 63u)) & ~63u;   // regions stay 256-byte aligned
  const size_t tmp = std::max(sort_pairs_temp_bytes(cap), scan_temp_bytes(cap));
  char* base = nullptr;
  if (cudaMalloc(&base, (size_t)cap * 32u) != cudaSuccess || cudaMalloc(&st->d_tmp, tmp) != cudaSuccess) {
    h->last_err = std::string("alz_window_rollup scratch: ") + cudaGetErrorString(cudaGetLastError());
    cudaFree(base);
    st->d_tmp = nullptr;
    return ALZ_E_NOMEM;
  }
  st->d_keys[0] = (uint64_t*)base;
  st->d_keys[1] = st->d_keys[0] + cap;
  st->d_ukeys = st->d_keys[1] + cap;
  st->d_src[0] = (uint32_t*)(st->d_ukeys + cap);
  st->d_src[1] = st->d_src[0] + cap;
  st->cap_rows = cap;
  st->tmp_bytes = tmp;
  return ALZ_OK;
}

// The sum of the last k entries into st->d_sum; *n_out rows. Caller holds h->mu and has set the device.
static int rollup_locked(alz_handle* h, uint32_t k, size_t* n_out, alz_rollup_info* info) {
  alz_rollup_state* st = h->roll;
  if (!st) return ALZ_E_STATE;
  if (k == 0) return ALZ_E_INVAL;
  cudaStream_t s = h->stream;
  const size_t m = std::min<size_t>(k, st->entries.size());
  const size_t first = st->entries.size() - m;
  uint64_t n_src = 0;
  for (size_t i = first; i < st->entries.size(); ++i) n_src += st->entries[i].n;
  const uint32_t n = (uint32_t)n_src;   // at most arena_rows: the entries do not overlap
  uint32_t n_sum = 0;
  CK(cudaMemcpyAsync(st->h_clk.data(), st->d_clk, (size_t)st->depth * sizeof(WinClock), cudaMemcpyDeviceToHost, s));
  if (n) {
    int rc = ensure_scratch(h, st, n);
    if (rc != ALZ_OK) return rc;
    // entries that follow one another in the arena (all of them, or all but one jump back to row 0) take one launch
    const unsigned grid = (unsigned)h->sms * 4u;
    uint32_t done = 0;
    for (size_t i = first; i < st->entries.size();) {
      const uint64_t run_first = st->entries[i].first_row;
      uint64_t run_n = 0;
      for (; i < st->entries.size() && st->entries[i].first_row == run_first + run_n; ++i) run_n += st->entries[i].n;
      if (run_n == 0) continue;
      rollup_keys_kernel<<<grid, 256, 0, s>>>(st->d_arena, (uint32_t)run_first, (uint32_t)run_n, st->d_keys[0] + done,
                                              st->d_src[0] + done);
      h->launches += 1;
      done += (uint32_t)run_n;
    }
    sort_pairs(st->d_tmp, st->tmp_bytes, st->d_keys[0], st->d_keys[1], st->d_src[0], st->d_src[1], n, s);
    // the unsorted keys are done with: their buffer takes the head flags and their scan. No row of a flush has the
    // key that equals the free marker (alz_device.cuh, EdgeTable), which launch_unique_sorted never takes as a head.
    uint32_t* flags = reinterpret_cast<uint32_t*>(st->d_keys[0]);
    uint32_t* pos = flags + st->cap_rows;
    launch_unique_sorted(st->d_keys[1], n, flags, pos, st->d_ukeys, st->d_tmp, st->tmp_bytes, h->sms, s);
    h->launches += 2;
    CK(cudaGetLastError());
    uint32_t last[2];
    CK(cudaMemcpyAsync(&last[0], pos + (n - 1), 4, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(&last[1], flags + (n - 1), 4, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));   // the one count the host needs, as a flush needs its edge count
    n_sum = last[0] + last[1];
    if (n_sum > st->sum_rows) {
      cudaFree(st->d_sum);
      st->d_sum = nullptr;
      st->sum_rows = 0;
      const size_t want = std::min<size_t>(st->arena_rows, (size_t)n_sum + n_sum / 2u);
      if (cudaMalloc(&st->d_sum, want * sizeof(alz_edge_out)) != cudaSuccess) {
        h->last_err = std::string("alz_window_rollup rows: ") + cudaGetErrorString(cudaGetLastError());
        return ALZ_E_NOMEM;
      }
      st->sum_rows = want;
    }
    rollup_emit_kernel<<<(unsigned)h->sms * 8u, 256, 0, s>>>(st->d_arena, st->d_keys[1], st->d_src[1], n, st->d_ukeys,
                                                             n_sum, st->d_sum);
    h->launches += 1;
    CK(cudaGetLastError());
  } else {
    CK(cudaStreamSynchronize(s));
  }
  *n_out = n_sum;
  if (info) {
    *info = alz_rollup_info{};
    info->windows = (uint32_t)m;
    info->rows_in = n_src;
    if (m) {
      const Entry& a = st->entries[first];
      const Entry& b = st->entries.back();
      info->window_first = a.window;
      info->window_last = b.window;
      bool clocked = true;
      for (size_t i = first; i < st->entries.size(); ++i)
        clocked &= st->entries[i].clocked && st->h_clk[st->entries[i].slot].ready != 0ull;
      if (clocked) {
        info->clocked = 1u;
        info->epoch_first = st->h_clk[a.slot].epoch;
        info->epoch_last = st->h_clk[b.slot].epoch;
      }
    }
  }
  return ALZ_OK;
}

extern "C" int alz_window_rollup_device(alz_handle* h, uint32_t k, const alz_edge_out** dev_rows, size_t* n_out,
                                        alz_rollup_info* info) {
  if (!h || !n_out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  const int rc = rollup_locked(h, k, n_out, info);
  if (rc == ALZ_OK && dev_rows) *dev_rows = h->roll->d_sum;
  return rc;
}

extern "C" int alz_window_rollup(alz_handle* h, uint32_t k, alz_edge_out* out, size_t cap, size_t* n_out,
                                 alz_rollup_info* info) {
  if (!h || !n_out || (!out && cap)) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  const int rc = rollup_locked(h, k, n_out, info);
  if (rc != ALZ_OK) return rc;
  if (*n_out > cap) return ALZ_E_CAPACITY;
  if (*n_out) CK(cudaMemcpyAsync(out, h->roll->d_sum, *n_out * sizeof(alz_edge_out), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return ALZ_OK;
}
