// alz_rollup.cu — rolling windows (docs/SPEC.md §12): the rows of the last flushed windows kept on the device, and
// the sum of the last k of them as one edge list; tiered history (docs/SPEC.md §13): every consumed window merged
// into coarser blocks on the device, each closed block retained as an entry of its tier; and span rollups
// (docs/SPEC.md §14): the last m windows summed from pieces of all of these.
//
// Every accumulator of an output row is an integer sum (docs/SPEC.md §3), so the sum of k windows' rows per edge
// is what one window holding those windows' events would have returned. The flush is left as it is: a flush that
// consumed its window copies its rows into the arena (one device-to-device copy, no kernel, no synchronisation).
//
// The window history and each tier keep their retained entries in a Ring: an arena of rows, a clock per entry and
// the host's list of entries. Every rollup is one sum over pieces (sum_pieces), a piece being a run of rows of one
// buffer: a ring entry or a tier's open block. A window or tier rollup takes the last k entries of one ring; a span
// takes the pieces the host plans. The sum has the shape of the single-rank flush (DESIGN.md §5.3) applied to output
// rows instead of pair rows: packed key of every source row -> radix sort of (key, source row) -> the distinct keys
// -> eight lanes per output row add up the key's run of source rows in registers and store the row once.
//
// A tier's open block is a sorted row list. Both it and its input (a flushed window, or a closed block of the tier
// below) are strictly ascending by packed key, so feeding it is a 2-way merge that adds matching keys (DESIGN.md
// §5.6): tier_match_kernel, an exclusive scan of the unmatched input rows, tier_merge_kernel. The block's row count
// and overflow flag stay on the device; only a block that closes (once per `factor` inputs) is waited for.
#include <algorithm>
#include <deque>
#include <new>
#include <type_traits>
#include <unordered_map>
#include <vector>

#include "alz_handle.h"

using namespace alz;

namespace {
struct Entry {            // one retained entry; host-side record of rows [first_row, first_row + n) of an arena
  uint64_t first_row, n;
  uint64_t window_first;  // alz_stats.windows after the flush of the oldest / newest window it covers
  uint64_t window_last;
  uint32_t windows;       // flushed windows it covers (1 in the window history)
  uint32_t slot;          // its clock(s) in the arena's clock array
  bool clocked;           // a window clock was set at every covered window's flush
};

// The ring rule of docs/SPEC.md §12: where an entry of n rows goes in an arena of arena_rows rows that keeps at most
// depth entries; evicts the oldest entries until it fits. The caller has checked n <= arena_rows.
uint64_t ring_place(std::deque<Entry>& entries, uint32_t depth, uint64_t arena_rows, uint64_t n) {
  // The entry goes behind the newest one, or to row 0 when it would pass the end (the rows skipped there are free
  // again once the entries before them have gone). The oldest entries are evicted until at most depth - 1 remain
  // and the place overlaps none of the rest.
  for (;;) {
    while (entries.size() >= depth) entries.pop_front();
    uint64_t at = entries.empty() ? 0 : entries.back().first_row + entries.back().n;
    if (at + n > arena_rows) at = 0;
    bool overlaps = false;
    for (const Entry& e : entries) overlaps |= at < e.first_row + e.n && e.first_row < at + n;
    if (!overlaps) return at;
    entries.pop_front();
  }
}

// sort-based rollup scratch, sized by the number of source rows (which max_edges does not bound), grown on demand
struct RollupScratch {
  uint32_t cap_rows = 0;
  uint64_t* d_keys[2] = {nullptr, nullptr};   // [cap_rows] packed keys of the source rows, unsorted / sorted
  uint32_t* d_src[2] = {nullptr, nullptr};    // [cap_rows] their virtual rows
  uint64_t* d_ukeys = nullptr;                // [cap_rows] the distinct keys in order
  void* d_tmp = nullptr;                      // CUB scratch of the sort, then of the scan
  size_t tmp_bytes = 0;
  alz_edge_out* d_sum = nullptr;              // the last rollup's rows
  size_t sum_rows = 0;
  // the last call of this kind returned ALZ_OK with held_rows rows in d_sum: what alz_gnn_score_rollup scores;
  // held_info is what that call reported (kept whether or not the caller asked for it)
  bool held = false;
  size_t held_rows = 0;
  alz_rollup_info held_info{};
};

// the clock of a tier's open block and of each of its entries: the oldest and newest covered window's clocks
struct TierClk {
  WinClock first, last;
  uint64_t unready;   // some covered window's clock was not ready (no open epoch)
};
// device state of a tier's open block
struct TierOpen {
  TierClk clk;
  uint32_t count[2];  // rows in block buffer 0 / 1
  uint32_t overflow;  // the open block would have passed block_rows: it is dropped when it closes
  uint32_t _pad;
};

// The clock rule: a clock gives epochs when every covered window's clock was ready. *first / *last: the epochs of
// the oldest and newest covered window.
bool clock_epochs(const WinClock& c, uint64_t* first, uint64_t* last) {
  *first = *last = c.epoch;
  return c.ready != 0ull;
}
bool clock_epochs(const TierClk& c, uint64_t* first, uint64_t* last) {
  *first = c.first.epoch;
  *last = c.last.epoch;
  return c.unready == 0ull;
}

// one piece of a rollup: a retained entry or a tier's open block
struct Piece {
  const alz_edge_out* buf;              // the buffer that holds its rows
  const uint64_t* keys;                 // the buffer's packed keys (an open block's key array), or null: read the rows
  uint64_t first_row, n;                // its rows in buf
  uint64_t window_first, window_last;   // the consumed windows it covers, alz_stats.windows numbering
  uint32_t windows;
  uint32_t level;                       // 0: the window history, t: tier t
  bool open;                            // tier `level`'s open block
  bool clocked;                         // the clock rule holds: epoch_first / epoch_last are its epochs
  uint64_t epoch_first, epoch_last;
};

// Retained entries (docs/SPEC.md §12): an arena of arena_rows rows holding at most depth entries, each with a clock
// in slot appended % depth of the clock array. The window history's clock is the WinClock its flush closed, a tier
// entry's the TierClk of its block.
template <class Clk>
struct Ring {
  using value_type = Clk;
  uint32_t depth = 0;
  uint64_t arena_rows = 0;
  alz_edge_out* d_arena = nullptr;    // [arena_rows]
  Clk* d_clk = nullptr;               // [depth]
  std::vector<Clk> h_clk;             // host copy of d_clk, read by rollups
  std::deque<Entry> entries;          // oldest first: a contiguous run of the most recent inputs
  uint64_t appended = 0;              // entries ever appended: the next one's clock slot is appended % depth

  bool alloc(uint32_t d, uint64_t rows) {
    depth = d;
    arena_rows = rows;
    h_clk.resize(d);
    return cudaMalloc(&d_arena, (size_t)rows * sizeof(alz_edge_out)) == cudaSuccess &&
           cudaMalloc(&d_clk, (size_t)d * sizeof(Clk)) == cudaSuccess;
  }
  void free() { cudaFree(d_arena); cudaFree(d_clk); }

  // The newest entry: n rows copied from rows and its clock from d_c (null: not clocked), in stream order. An entry
  // larger than the arena is not retained and clears the ring: the run would have a gap.
  int append(alz_handle* h, const alz_edge_out* rows, uint64_t n, const Clk* d_c, uint64_t window_first,
             uint64_t window_last, uint32_t windows) {
    if (n > arena_rows) { entries.clear(); return ALZ_OK; }
    const uint64_t at = ring_place(entries, depth, arena_rows, n);
    const uint32_t slot = (uint32_t)(appended++ % depth);
    if (n) CK(cudaMemcpyAsync(d_arena + at, rows, (size_t)n * sizeof(alz_edge_out), cudaMemcpyDeviceToDevice, h->stream));
    if (d_c) CK(cudaMemcpyAsync(d_clk + slot, d_c, sizeof(Clk), cudaMemcpyDeviceToDevice, h->stream));
    entries.push_back(Entry{at, n, window_first, window_last, windows, slot, d_c != nullptr});
    return ALZ_OK;
  }

  Piece piece(const Entry& e, uint32_t level) const {   // its clock is left to clocked()
    return Piece{d_arena, nullptr, e.first_row, e.n, e.window_first, e.window_last, e.windows, level, false, false, 0, 0};
  }
  // whether entry e is clocked, and the epochs of its oldest and newest window; from h_clk, which the caller has
  // copied from the device
  bool clocked(const Entry& e, uint64_t* first, uint64_t* last) const {
    return e.clocked && clock_epochs(h_clk[e.slot], first, last);
  }
};
}  // namespace

struct alz_rollup_state {
  Ring<WinClock> ring;
  RollupScratch sc;                   // window rollups' rows
};

namespace {
struct Tier {
  alz_history_tier cfg{};
  Ring<TierClk> ring;
  alz_edge_out* d_block[2] = {nullptr, nullptr};   // [block_rows] the open block, ping-pong
  uint64_t* d_bkeys[2] = {nullptr, nullptr};       // [block_rows] its packed keys
  int cur = 0;                        // the buffer that holds the open block
  uint32_t inputs = 0;                // inputs merged into the open block
  uint64_t window_first = 0;          // alz_stats.windows of the open block's oldest window
  uint64_t window_last = 0;           // and of its newest: that of the flush that fed its last input
  bool clocked = true;                // every input so far was clocked
  bool poisoned = false;              // the open block would contain a dropped block of a tier below
  uint64_t dropped = 0;
  uint32_t windows_per_input = 1;     // flushed windows one input covers
};
}  // namespace

struct alz_tier_set {
  std::vector<Tier> tiers;            // tiers 1..n
  TierOpen* d_open = nullptr;         // [n]
  // merge scratch, for an input of up to max_in rows
  uint32_t max_in = 0;
  uint64_t* d_ikeys = nullptr;        // [max_in] packed keys of the input rows
  uint32_t* d_pos = nullptr;          // [max_in] insertion point of each input row in the block
  uint32_t* d_unm = nullptr;          // [max_in + 1] 1: the input row's key is not in the block
  uint32_t* d_scan = nullptr;         // [max_in + 1] exclusive scan of d_unm
  void* d_tmp = nullptr;
  size_t tmp_bytes = 0;
  TierOpen h_open{};                  // host copy of the closing tier's TierOpen
  RollupScratch sc;                   // tier rollups' rows
};

struct alz_span_state {
  RollupScratch sc;                   // span rollups' rows
  std::vector<TierOpen> h_open;       // host copy of every tier's TierOpen
};

// Output row u = the sum of the source rows row_of(src[b, e)), the run of ukeys[u] in sorted[0, n). Eight lanes per
// output row, a lane owning 8 histogram cells and lane 0 the three u64 sums as everywhere else (edge_row_load): lanes
// 0 and 1 find the two ends of the run, every source row is read once and the output row is written once with plain
// stores. All sums wrap (u64 sums mod 2^64, cells mod 2^32, docs/SPEC.md §3).
template <class RowOf>
__device__ __forceinline__ void emit_sums(RowOf row_of, const uint64_t* __restrict__ sorted,
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
      load_edge_out(row_of(src[j]), sl, rc, r_count, r_lat, r_e5);
#pragma unroll
      for (int q = 0; q < 8; ++q) c[q] += rc[q];
      count += r_count; lat += r_lat; e5 += r_e5;
    }
    store_edge_out(&out[u], sl, key, c, count, e5, lat);
  }
}

// The source buffers of one rollup: the window-history arena, each tier's arena and each tier's open block (the
// buffer that holds it). Their rows are numbered in one virtual space, buffer b taking [vbase[b], vbase[b + 1]);
// the keys pass writes virtual rows and the emit maps them back to a buffer and a row.
constexpr int kSpanSources = 1 + 2 * ALZ_MAX_TIERS;
struct SpanSources {
  const alz_edge_out* buf[kSpanSources];
  uint32_t vbase[kSpanSources + 1];
  uint32_t n;
};

// keys[i], vrow[i] = packed key and virtual row of row i of a contiguous run (rows, virtual rows v0 + i); 16 of a
// row's 296 bytes are read, and the keys of an open block are read from its key array (bkeys) instead
__global__ void __launch_bounds__(256) span_keys_kernel(const alz_edge_out* __restrict__ rows,
                                                        const uint64_t* __restrict__ bkeys, uint32_t n, uint32_t v0,
                                                        uint64_t* __restrict__ keys, uint32_t* __restrict__ vrow) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    keys[i] = bkeys ? bkeys[i] : row_key_of(rows + i);
    vrow[i] = v0 + i;
  }
}

struct SpanRowOf {
  const alz_edge_out* const* buf;
  const uint32_t* vbase;
  uint32_t n;
  __device__ __forceinline__ const alz_edge_out* operator()(uint32_t v) const {
    uint32_t lo = 0, hi = n;   // the last buffer b with vbase[b] <= v
    while (hi - lo > 1u) {
      const uint32_t mid = (lo + hi) >> 1;
      if (vbase[mid] <= v) lo = mid; else hi = mid;
    }
    return buf[lo] + (v - vbase[lo]);
  }
};

// the sum of the pieces: src[] holds virtual rows. With one buffer (kOneBuffer) a virtual row is a row of it;
// otherwise each is mapped to its buffer by a binary search over vbase, which the block keeps in shared memory.
template <bool kOneBuffer>
__global__ void __launch_bounds__(256) span_emit_kernel(const __grid_constant__ SpanSources sources,
                                                        const uint64_t* __restrict__ sorted,
                                                        const uint32_t* __restrict__ src, uint32_t n,
                                                        const uint64_t* __restrict__ ukeys, uint32_t n_out,
                                                        alz_edge_out* __restrict__ out) {
  if constexpr (kOneBuffer) {
    const alz_edge_out* buf = sources.buf[0];
    emit_sums([buf](uint32_t v) { return buf + v; }, sorted, src, n, ukeys, n_out, out);
  } else {
    __shared__ const alz_edge_out* s_buf[kSpanSources];
    __shared__ uint32_t s_vbase[kSpanSources + 1];
    if (threadIdx.x < kSpanSources) s_buf[threadIdx.x] = sources.buf[threadIdx.x];
    if (threadIdx.x <= kSpanSources) s_vbase[threadIdx.x] = sources.vbase[threadIdx.x];
    __syncthreads();
    emit_sums(SpanRowOf{s_buf, s_vbase, sources.n}, sorted, src, n, ukeys, n_out, out);
  }
}

// Step 1 of merging n input rows into a tier's open block (bkeys, open->count[cur] rows): for every input row j its
// packed key, its insertion point in the block and whether the block lacks its key (unm[n] = 0 closes the scan).
// Thread 0 also carries the input's clocks into the open block's: clk_first / clk_last are the input's oldest and
// newest window clock, clk_unready its unready flag (null: the input is one window, unready when its clock is not).
__global__ void __launch_bounds__(256) tier_match_kernel(const alz_edge_out* __restrict__ in,
                                                         const uint64_t* __restrict__ in_keys, uint32_t n,
                                                         const uint64_t* __restrict__ bkeys, TierOpen* open, int cur,
                                                         uint64_t* __restrict__ ikeys, uint32_t* __restrict__ pos,
                                                         uint32_t* __restrict__ unm, const WinClock* clk_first,
                                                         const WinClock* clk_last, const uint64_t* clk_unready,
                                                         bool first_input) {
  const uint32_t n_b = open->count[cur];
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x;
  for (uint32_t j = t0; j < n; j += stride) {
    const uint64_t key = in_keys ? in_keys[j] : row_key_of(in + j);
    const uint32_t p = lower_bound_u64(bkeys, n_b, key);
    ikeys[j] = key;
    pos[j] = p;
    unm[j] = (p < n_b && bkeys[p] == key) ? 0u : 1u;
  }
  if (t0 == 0) {
    unm[n] = 0u;
    if (clk_first) {
      const uint64_t u = clk_unready ? *clk_unready : (uint64_t)(clk_last->ready == 0ull);
      if (first_input) { open->clk.first = *clk_first; open->clk.unready = 0ull; }
      open->clk.last = *clk_last;
      open->clk.unready |= u;
    }
  }
}

// Step 2: the merged block into the other buffer, each output row written once by eight lanes. scan = exclusive scan
// of unm, so scan[n] input rows are new. Block row i goes to i + (new input rows before its key), and adds the input
// row with its key if there is one; new input row j goes to pos[j] + scan[j]. A block that would pass block_rows is
// flagged and left empty: it is dropped when it closes. Bounds come from the device; the grid from the host's bound.
__global__ void __launch_bounds__(256) tier_merge_kernel(const alz_edge_out* __restrict__ blk,
                                                         const uint64_t* __restrict__ bkeys, TierOpen* open, int cur,
                                                         const alz_edge_out* __restrict__ in,
                                                         const uint64_t* __restrict__ ikeys,
                                                         const uint32_t* __restrict__ pos,
                                                         const uint32_t* __restrict__ unm,
                                                         const uint32_t* __restrict__ scan, uint32_t n,
                                                         uint32_t block_rows, alz_edge_out* __restrict__ out,
                                                         uint64_t* __restrict__ okeys) {
  const uint32_t n_b = open->count[cur];
  const uint32_t total = n_b + scan[n];
  const bool over = open->overflow != 0u || total > block_rows;
  const uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x;
  if (over) {
    if (t0 == 0) { open->overflow = 1u; open->count[cur ^ 1] = 0u; }
    return;
  }
  if (t0 == 0) open->count[cur ^ 1] = total;
  const uint32_t sl = threadIdx.x & 7u;
  const uint32_t groups_per_grid = (gridDim.x * blockDim.x) >> 3;
  for (uint32_t g = t0 >> 3; g < n_b + n; g += groups_per_grid) {
    uint32_t c[8];
    uint64_t count, lat, e5, key;
    uint32_t o;
    if (g < n_b) {
      key = bkeys[g];
      const uint32_t p = lower_bound_u64(ikeys, n, key);
      o = g + scan[p];
      load_edge_out(blk + g, sl, c, count, lat, e5);
      if (p < n && ikeys[p] == key) {
        uint32_t rc[8];
        uint64_t r_count, r_lat, r_e5;
        load_edge_out(in + p, sl, rc, r_count, r_lat, r_e5);
#pragma unroll
        for (int q = 0; q < 8; ++q) c[q] += rc[q];
        count += r_count; lat += r_lat; e5 += r_e5;
      }
    } else {
      const uint32_t j = g - n_b;
      if (!unm[j]) continue;
      key = ikeys[j];
      o = pos[j] + scan[j];
      load_edge_out(in + j, sl, c, count, lat, e5);
    }
    store_edge_out(&out[o], sl, key, c, count, e5, lat);
    if (sl == 0) okeys[o] = key;
  }
}

static void free_scratch(RollupScratch& sc) {
  cudaFree(sc.d_keys[0]); cudaFree(sc.d_tmp); cudaFree(sc.d_sum);
  sc = RollupScratch{};
}

void alz_internal_free_rollup(alz_handle* h) {
  alz_rollup_state* st = h->roll;
  if (!st) return;
  free_scratch(st->sc);
  st->ring.free();
  delete st;
  h->roll = nullptr;
}

extern "C" int alz_window_history(alz_handle* h, uint32_t depth, uint64_t arena_rows) {
  if (!h || arena_rows >= (1ull << 31) || (depth != 0 && arena_rows == 0)) return ALZ_E_INVAL;   // rows are indexed by u32, counted by int
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  if (h->roll && h->roll->ring.depth == depth && h->roll->ring.arena_rows == arena_rows) return ALZ_OK;
  CK(cudaStreamSynchronize(h->stream));   // copies into the arena and a rollup's kernels may still be running
  alz_internal_free_rollup(h);
  if (depth == 0) return ALZ_OK;
  alz_rollup_state* st = new (std::nothrow) alz_rollup_state();
  if (!st) return ALZ_E_NOMEM;
  h->roll = st;
  if (!st->ring.alloc(depth, arena_rows)) {
    h->last_err = std::string("alz_window_history: ") + cudaGetErrorString(cudaGetLastError());
    alz_internal_free_rollup(h);
    return ALZ_E_NOMEM;
  }
  return ALZ_OK;
}

static int tiers_input_window(alz_handle* h, const uint64_t* d_clk);

// The window a flush has just consumed becomes the newest entry of the window history (docs/SPEC.md §12). The
// window history and the tiers each take the window whatever happens to the other.
int alz_internal_history_append(alz_handle* h, const uint64_t* d_clk) {
  const int rc0 = h->roll ? h->roll->ring.append(h, h->d_out, h->last_n_edges, reinterpret_cast<const WinClock*>(d_clk),
                                                 h->windows, h->windows, 1u)
                          : ALZ_OK;
  const int rc1 = h->tiers ? tiers_input_window(h, d_clk) : ALZ_OK;
  return rc0 != ALZ_OK ? rc0 : rc1;
}

// scratch for n source rows of at most row_bound
static int ensure_scratch(alz_handle* h, RollupScratch& sc, uint64_t row_bound, uint32_t n) {
  if (n <= sc.cap_rows) return ALZ_OK;
  CK(cudaStreamSynchronize(h->stream));
  cudaFree(sc.d_keys[0]); cudaFree(sc.d_tmp);
  sc.d_keys[0] = sc.d_keys[1] = sc.d_ukeys = nullptr;
  sc.d_src[0] = sc.d_src[1] = nullptr;
  sc.d_tmp = nullptr;
  sc.cap_rows = 0; sc.tmp_bytes = 0;
  const uint32_t cap = (uint32_t)std::min<uint64_t>(row_bound + 63u, ((uint64_t)n + n / 2u + 63u)) & ~63u;   // regions stay 256-byte aligned
  const size_t tmp = std::max(sort_pairs_temp_bytes(cap), scan_temp_bytes(cap));
  char* base = nullptr;
  if (cudaMalloc(&base, (size_t)cap * 32u) != cudaSuccess || cudaMalloc(&sc.d_tmp, tmp) != cudaSuccess) {
    h->last_err = std::string("alz_window_rollup scratch: ") + cudaGetErrorString(cudaGetLastError());
    cudaFree(base);
    sc.d_tmp = nullptr;
    return ALZ_E_NOMEM;
  }
  sc.d_keys[0] = (uint64_t*)base;
  sc.d_keys[1] = sc.d_keys[0] + cap;
  sc.d_ukeys = sc.d_keys[1] + cap;
  sc.d_src[0] = (uint32_t*)(sc.d_ukeys + cap);
  sc.d_src[1] = sc.d_src[0] + cap;
  sc.cap_rows = cap;
  sc.tmp_bytes = tmp;
  return ALZ_OK;
}

// The n >= 1 (key, source) pairs in sc.d_keys[0] / sc.d_src[0] sorted into sc.d_keys[1] / sc.d_src[1], their
// distinct keys into sc.d_ukeys, *n_sum of them: the one count the host waits for. sc.d_sum is grown to hold them
// (at most out_bound rows).
static int sort_distinct(alz_handle* h, RollupScratch& sc, uint32_t n, uint64_t out_bound, uint32_t* n_sum) {
  cudaStream_t s = h->stream;
  sort_pairs(sc.d_tmp, sc.tmp_bytes, sc.d_keys[0], sc.d_keys[1], sc.d_src[0], sc.d_src[1], n, s);
  // the unsorted keys are done with: their buffer takes the head flags and their scan. No row of a flush has the
  // key that equals the free marker (alz_device.cuh, EdgeTable), which launch_unique_sorted never takes as a head.
  uint32_t* flags = reinterpret_cast<uint32_t*>(sc.d_keys[0]);
  uint32_t* pos = flags + sc.cap_rows;
  launch_unique_sorted(sc.d_keys[1], n, flags, pos, sc.d_ukeys, sc.d_tmp, sc.tmp_bytes, h->sms, s);
  h->launches += 2;
  CK(cudaGetLastError());
  uint32_t last[2];
  CK(cudaMemcpyAsync(&last[0], pos + (n - 1), 4, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(&last[1], flags + (n - 1), 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));   // the one count the host needs, as a flush needs its edge count
  *n_sum = last[0] + last[1];
  if (*n_sum > sc.sum_rows) {
    cudaFree(sc.d_sum);
    sc.d_sum = nullptr;
    sc.sum_rows = 0;
    const size_t want = std::min<size_t>(out_bound, (size_t)*n_sum + *n_sum / 2u);
    if (cudaMalloc(&sc.d_sum, want * sizeof(alz_edge_out)) != cudaSuccess) {
      h->last_err = std::string("alz_window_rollup rows: ") + cudaGetErrorString(cudaGetLastError());
      return ALZ_E_NOMEM;
    }
    sc.sum_rows = want;
  }
  return ALZ_OK;
}

// The sum of the pieces' rows into sc.d_sum, *n_out rows; row_bound bounds the source rows of any call with this
// scratch. Whatever the caller has enqueued before is complete when this returns. Caller holds h->mu and has set the
// device.
static int sum_pieces(alz_handle* h, RollupScratch& sc, std::vector<Piece> pieces, uint64_t row_bound,
                      size_t* n_out) {
  // by buffer (the window history, then tier by tier its arena and its open block), then by row
  std::sort(pieces.begin(), pieces.end(), [](const Piece& a, const Piece& b) {
    if (a.level != b.level) return a.level < b.level;
    return a.open != b.open ? b.open : a.first_row < b.first_row;
  });
  // the buffers the pieces read, numbered in one virtual row space up to the end of their last used row
  std::vector<uint32_t> vbase(pieces.size());   // of each piece's buffer
  SpanSources srcs{};
  uint64_t n_src = 0, vtop = 0;
  for (size_t i = 0; i < pieces.size();) {
    const alz_edge_out* buf = pieces[i].buf;
    uint64_t used = 0;
    for (; i < pieces.size() && pieces[i].buf == buf; ++i) {
      used = std::max(used, pieces[i].first_row + pieces[i].n);
      n_src += pieces[i].n;
      vbase[i] = (uint32_t)vtop;
    }
    if (!used) continue;
    srcs.buf[srcs.n] = buf;
    srcs.vbase[srcs.n++] = (uint32_t)vtop;
    vtop += used;
  }
  if (n_src > 0x7FFFFFFFull) return ALZ_E_CAPACITY;   // rows are indexed by u32, counted by int
  // the used buffers hold fewer than 2^32 rows on any device below 1.2 TB; a bound, never reached
  if (vtop >= (1ull << 32)) return ALZ_E_CAPACITY;
  srcs.vbase[srcs.n] = (uint32_t)vtop;

  cudaStream_t s = h->stream;
  uint32_t n_sum = 0;
  if (n_src) {
    int rc = ensure_scratch(h, sc, row_bound, (uint32_t)n_src);
    if (rc != ALZ_OK) return rc;
    // keys pass: pieces that follow one another in a buffer take one launch
    const unsigned grid = (unsigned)h->sms * 4u;
    uint32_t done = 0;
    for (size_t i = 0; i < pieces.size();) {
      const Piece& p = pieces[i];
      const uint32_t v0 = vbase[i] + (uint32_t)p.first_row;
      uint64_t run_n = 0;
      for (; i < pieces.size() && pieces[i].buf == p.buf && pieces[i].first_row == p.first_row + run_n; ++i)
        run_n += pieces[i].n;
      if (run_n == 0) continue;
      span_keys_kernel<<<grid, 256, 0, s>>>(p.buf + p.first_row, p.keys ? p.keys + p.first_row : nullptr,
                                            (uint32_t)run_n, v0, sc.d_keys[0] + done, sc.d_src[0] + done);
      h->launches += 1;
      done += (uint32_t)run_n;
    }
    rc = sort_distinct(h, sc, (uint32_t)n_src, row_bound, &n_sum);
    if (rc != ALZ_OK) return rc;
    if (srcs.n == 1)
      span_emit_kernel<true><<<(unsigned)h->sms * 8u, 256, 0, s>>>(srcs, sc.d_keys[1], sc.d_src[1], (uint32_t)n_src,
                                                                   sc.d_ukeys, n_sum, sc.d_sum);
    else
      span_emit_kernel<false><<<(unsigned)h->sms * 8u, 256, 0, s>>>(srcs, sc.d_keys[1], sc.d_src[1], (uint32_t)n_src,
                                                                    sc.d_ukeys, n_sum, sc.d_sum);
    h->launches += 1;
    CK(cudaGetLastError());
  } else {
    CK(cudaStreamSynchronize(s));
  }
  *n_out = n_sum;
  return ALZ_OK;
}

// What the pieces (oldest first, covering a contiguous run of windows) cover; epochs when every one is clocked.
static void fill_info(const std::vector<Piece>& pieces, alz_rollup_info* info) {
  *info = alz_rollup_info{};
  if (pieces.empty()) return;
  bool clocked = true;
  for (const Piece& p : pieces) {
    info->windows += p.windows;
    info->rows_in += p.n;
    clocked &= p.clocked;
  }
  info->window_first = pieces.front().window_first;
  info->window_last = pieces.back().window_last;
  if (clocked) {
    info->clocked = 1u;
    info->epoch_first = pieces.front().epoch_first;
    info->epoch_last = pieces.back().epoch_last;
  }
}

// The sum of the last k entries of a ring into sc.d_sum; *n_out rows. The ring's clocks are copied to the host in
// stream order, so they are read when the sum returns.
template <class Clk>
static int ring_rollup(alz_handle* h, Ring<Clk>& r, uint32_t level, uint32_t k, RollupScratch& sc, size_t* n_out,
                       alz_rollup_info* info) {
  CK(cudaMemcpyAsync(r.h_clk.data(), r.d_clk, (size_t)r.depth * sizeof(Clk), cudaMemcpyDeviceToHost, h->stream));
  size_t first = r.entries.size() - std::min<size_t>(k, r.entries.size());
  std::vector<Piece> pieces;
  for (size_t i = first; i < r.entries.size(); ++i) pieces.push_back(r.piece(r.entries[i], level));
  const int rc = sum_pieces(h, sc, pieces, r.arena_rows, n_out);
  if (rc != ALZ_OK) return rc;
  if (info) {
    for (Piece& p : pieces) p.clocked = r.clocked(r.entries[first++], &p.epoch_first, &p.epoch_last);
    fill_info(pieces, info);
  }
  return ALZ_OK;
}

// The sum of the last k entries of the window history (level 0) or of tier `level` into the scratch of that kind of
// rollup, so that each one's rows stay valid until the next of its kind; *rows, *n_out, *info and, with ALZ_OK,
// *caller_info (when not null) = *info. Caller holds h->mu and has set the device.
static int rollup_locked(alz_handle* h, uint32_t level, uint32_t k, size_t* n_out, alz_rollup_info* info,
                         alz_rollup_info* caller_info, const alz_edge_out** rows) {
  RollupScratch* sc = nullptr;
  int rc;
  if (level == 0) {
    if (!h->roll) return ALZ_E_STATE;
    if (k == 0) return ALZ_E_INVAL;
    sc = &h->roll->sc;
    rc = ring_rollup(h, h->roll->ring, 0, k, *sc, n_out, info);
  } else {
    alz_tier_set* ts = h->tiers;
    if (!ts) return ALZ_E_STATE;
    if (k == 0 || level > ts->tiers.size()) return ALZ_E_INVAL;
    sc = &ts->sc;
    rc = ring_rollup(h, ts->tiers[level - 1].ring, level, k, *sc, n_out, info);
  }
  *rows = sc->d_sum;
  if (rc == ALZ_OK && caller_info) *caller_info = *info;
  return rc;
}

// The scratch of a kind of rollup (ALZ_ROLLUP_*), or null when it has none
static RollupScratch* scratch_of(alz_handle* h, uint32_t kind) {
  switch (kind) {
    case ALZ_ROLLUP_WINDOWS: return h->roll ? &h->roll->sc : nullptr;
    case ALZ_ROLLUP_TIER: return h->tiers ? &h->tiers->sc : nullptr;
    case ALZ_ROLLUP_SPAN: return h->span ? &h->span->sc : nullptr;
    default: return nullptr;
  }
}

static uint32_t kind_of_tier(uint32_t tier) { return tier == 0 ? ALZ_ROLLUP_WINDOWS : ALZ_ROLLUP_TIER; }

int alz_internal_rollup_rows(alz_handle* h, uint32_t kind, const alz_edge_out** rows, size_t* n,
                             alz_rollup_info* info) {
  if (kind > ALZ_ROLLUP_SPAN) return ALZ_E_INVAL;
  const RollupScratch* sc = scratch_of(h, kind);
  if (!sc || !sc->held) return ALZ_E_STATE;
  *rows = sc->d_sum;
  *n = sc->held_rows;
  if (info) *info = sc->held_info;
  return ALZ_OK;
}

int alz_internal_window_info(alz_handle* h, alz_rollup_info* info) {
  *info = alz_rollup_info{};
  info->windows = 1;
  info->window_first = info->window_last = h->windows;
  info->rows_in = h->last_n_edges;
  const alz_rollup_state* st = h->roll;
  if (!st || st->ring.entries.empty() || st->ring.entries.back().window_last != h->windows) return ALZ_OK;
  // the window history's newest entry is this window: its clock, as a k = 1 window rollup reads it
  const Entry& e = st->ring.entries.back();
  if (!e.clocked) return ALZ_OK;
  WinClock c;
  CK(cudaMemcpyAsync(&c, st->ring.d_clk + e.slot, sizeof(WinClock), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  uint64_t first, last;
  if (clock_epochs(c, &first, &last)) {
    info->clocked = 1u;
    info->epoch_first = first;
    info->epoch_last = last;
  }
  return ALZ_OK;
}

// the ring of tier `tier` (0: the window history) as f(ring, level), or the status when there is none
template <class F>
static int with_ring(alz_handle* h, uint32_t tier, F f) {
  if (tier == 0) {
    if (!h->roll) return ALZ_E_STATE;
    f(h->roll->ring);
    return ALZ_OK;
  }
  if (!h->tiers) return ALZ_E_STATE;
  if (tier > h->tiers->tiers.size()) return ALZ_E_INVAL;
  f(h->tiers->tiers[tier - 1].ring);
  return ALZ_OK;
}

int alz_internal_ring_view(alz_handle* h, uint32_t tier, uint32_t k, alz_ring_view* v) {
  int rc = ALZ_OK;
  const int st = with_ring(h, tier, [&](auto& r) {
    using Clk = typename std::remove_reference_t<decltype(r)>::value_type;
    const cudaError_t e = cudaMemcpyAsync(r.h_clk.data(), r.d_clk, (size_t)r.depth * sizeof(Clk),
                                          cudaMemcpyDeviceToHost, h->stream);
    if (e != cudaSuccess) { h->last_err = std::string("alz_internal_ring_view: ") + cudaGetErrorString(e); rc = ALZ_E_CUDA; }
    v->arena = r.d_arena;
    v->first_row.clear();
    v->n.clear();
    for (size_t i = r.entries.size() - std::min<size_t>(k, r.entries.size()); i < r.entries.size(); ++i) {
      v->first_row.push_back(r.entries[i].first_row);
      v->n.push_back(r.entries[i].n);
    }
  });
  return st != ALZ_OK ? st : rc;
}

void alz_internal_ring_points(alz_handle* h, uint32_t tier, uint32_t k, alz_rollup_info* points) {
  with_ring(h, tier, [&](auto& r) {
    size_t j = 0;
    for (size_t i = r.entries.size() - std::min<size_t>(k, r.entries.size()); i < r.entries.size(); ++i, ++j) {
      std::vector<Piece> one{r.piece(r.entries[i], tier)};
      one[0].clocked = r.clocked(r.entries[i], &one[0].epoch_first, &one[0].epoch_last);
      fill_info(one, &points[j]);
    }
  });
}

uint64_t alz_internal_ring_last(alz_handle* h, uint32_t tier) {
  uint64_t last = 0;
  with_ring(h, tier, [&](auto& r) {
    if (!r.entries.empty()) last = r.entries.back().window_last;
  });
  return last;
}

// A rollup entry point of a kind (ALZ_ROLLUP_*): lock, set the device and run the rollup (run(&rows, &info), which
// sets *n_out and, with ALZ_OK, info). Into out (to_host): ALZ_E_CAPACITY when the rows do not fit, and nothing is
// written; else *dev_rows (when not null) = the device rows. The kind's scratch holds rows to score, and their info,
// only after a call that returns ALZ_OK.
template <class Run>
static int rollup_call(alz_handle* h, uint32_t kind, bool to_host, alz_edge_out* out, size_t cap,
                       const alz_edge_out** dev_rows, size_t* n_out, Run run) {
  if (!h) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  if (RollupScratch* sc = scratch_of(h, kind)) sc->held = false;
  if (!n_out || (!out && cap)) return ALZ_E_INVAL;
  CK(cudaSetDevice(h->device));
  const alz_edge_out* rows = nullptr;
  alz_rollup_info info{};
  const int rc = run(&rows, &info);
  if (rc != ALZ_OK) return rc;
  if (to_host) {
    if (*n_out > cap) return ALZ_E_CAPACITY;
    if (*n_out) CK(cudaMemcpyAsync(out, rows, *n_out * sizeof(alz_edge_out), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  } else if (dev_rows) {
    *dev_rows = rows;
  }
  RollupScratch* sc = scratch_of(h, kind);
  sc->held = true;
  sc->held_rows = *n_out;
  sc->held_info = info;
  return ALZ_OK;
}

extern "C" int alz_window_rollup_device(alz_handle* h, uint32_t k, const alz_edge_out** dev_rows, size_t* n_out,
                                        alz_rollup_info* info) {
  return alz_window_rollup_tier_device(h, 0, k, dev_rows, n_out, info);
}

extern "C" int alz_window_rollup(alz_handle* h, uint32_t k, alz_edge_out* out, size_t cap, size_t* n_out,
                                 alz_rollup_info* info) {
  return alz_window_rollup_tier(h, 0, k, out, cap, n_out, info);
}

extern "C" int alz_window_rollup_tier_device(alz_handle* h, uint32_t tier, uint32_t k, const alz_edge_out** dev_rows,
                                             size_t* n_out, alz_rollup_info* info) {
  return rollup_call(h, kind_of_tier(tier), false, nullptr, 0, dev_rows, n_out,
                     [&](const alz_edge_out** rows, alz_rollup_info* ri) {
                       return rollup_locked(h, tier, k, n_out, ri, info, rows);
                     });
}

extern "C" int alz_window_rollup_tier(alz_handle* h, uint32_t tier, uint32_t k, alz_edge_out* out, size_t cap,
                                      size_t* n_out, alz_rollup_info* info) {
  return rollup_call(h, kind_of_tier(tier), true, out, cap, nullptr, n_out,
                     [&](const alz_edge_out** rows, alz_rollup_info* ri) {
                       return rollup_locked(h, tier, k, n_out, ri, info, rows);
                     });
}

// ---- tiered history (docs/SPEC.md §13) ------------------------------------------------------------------------------

void alz_internal_free_tiers(alz_handle* h) {
  alz_tier_set* ts = h->tiers;
  if (!ts) return;
  for (Tier& t : ts->tiers) {
    t.ring.free();
    cudaFree(t.d_block[0]); cudaFree(t.d_block[1]); cudaFree(t.d_bkeys[0]); cudaFree(t.d_bkeys[1]);
  }
  cudaFree(ts->d_open); cudaFree(ts->d_ikeys); cudaFree(ts->d_tmp);
  free_scratch(ts->sc);
  delete ts;
  h->tiers = nullptr;
}

static bool same_tiers(const alz_tier_set* ts, const alz_history_tier* tiers, uint32_t n) {
  if (!ts) return n == 0;
  if (ts->tiers.size() != n) return false;
  for (uint32_t i = 0; i < n; ++i) {
    const alz_history_tier& a = ts->tiers[i].cfg;
    if (a.factor != tiers[i].factor || a.depth != tiers[i].depth || a.arena_rows != tiers[i].arena_rows ||
        a.block_rows != tiers[i].block_rows)
      return false;
  }
  return true;
}

extern "C" int alz_window_history_tiers(alz_handle* h, const alz_history_tier* tiers, uint32_t n) {
  if (!h || n > ALZ_MAX_TIERS || (n && !tiers)) return ALZ_E_INVAL;
  uint64_t span = 1;                   // flushed windows one entry of tier i covers
  for (uint32_t i = 0; i < n; ++i) {   // rows are indexed by u32, counted by int
    const alz_history_tier& t = tiers[i];
    if (t.factor < 2 || t.depth == 0 || t.arena_rows == 0 || t.arena_rows >= (1ull << 31) || t.block_rows == 0 ||
        t.block_rows >= (1ull << 31))
      return ALZ_E_INVAL;
    // windows are counted in u32 (alz_rollup_info.windows, alz_tier_state.open_windows): the windows of all
    // retained entries of a tier must stay below 2^32 (both factors are below 2^32, so the products fit in u64)
    span *= t.factor;
    if (span >= (1ull << 32) || span * t.depth >= (1ull << 32)) return ALZ_E_INVAL;
  }
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  if (same_tiers(h->tiers, tiers, n)) return ALZ_OK;
  CK(cudaStreamSynchronize(h->stream));   // merges, copies into the arenas and a rollup may still be running
  alz_internal_free_tiers(h);
  if (n == 0) return ALZ_OK;
  alz_tier_set* ts = new (std::nothrow) alz_tier_set();
  if (!ts) return ALZ_E_NOMEM;
  h->tiers = ts;
  ts->tiers.resize(n);
  // an input of tier 1 is a flushed window (at most max_edges rows); of tier t + 1, a block of tier t
  uint64_t max_in = h->cfg.max_edges;
  uint32_t wpi = 1;
  for (uint32_t i = 0; i < n; ++i) {
    ts->tiers[i].cfg = tiers[i];
    ts->tiers[i].windows_per_input = wpi;
    wpi *= tiers[i].factor;
    if (i + 1 < n) max_in = std::max<uint64_t>(max_in, tiers[i].block_rows);
  }
  ts->max_in = (uint32_t)max_in;
  ts->tmp_bytes = scan_temp_bytes(ts->max_in + 1);
  bool ok = cudaMalloc(&ts->d_open, n * sizeof(TierOpen)) == cudaSuccess &&
            cudaMalloc(&ts->d_ikeys, (size_t)(max_in + 1) * 8u + 3u * (size_t)(max_in + 1) * 4u) == cudaSuccess &&
            cudaMalloc(&ts->d_tmp, ts->tmp_bytes) == cudaSuccess;
  for (Tier& t : ts->tiers) {
    if (!ok) break;
    ok = t.ring.alloc(t.cfg.depth, t.cfg.arena_rows);
    for (int b = 0; b < 2 && ok; ++b)
      ok = cudaMalloc(&t.d_block[b], (size_t)t.cfg.block_rows * sizeof(alz_edge_out)) == cudaSuccess &&
           cudaMalloc(&t.d_bkeys[b], (size_t)t.cfg.block_rows * 8u) == cudaSuccess;
  }
  if (!ok) {
    h->last_err = std::string("alz_window_history_tiers: ") + cudaGetErrorString(cudaGetLastError());
    alz_internal_free_tiers(h);
    return ALZ_E_NOMEM;
  }
  ts->d_pos = reinterpret_cast<uint32_t*>(ts->d_ikeys + max_in + 1);
  ts->d_unm = ts->d_pos + max_in + 1;
  ts->d_scan = ts->d_unm + max_in + 1;
  CK(cudaMemsetAsync(ts->d_open, 0, n * sizeof(TierOpen), h->stream));
  return ALZ_OK;
}

// Merge n rows (in, with their keys in_keys or null) into tier ti's open block. clocks: see tier_match_kernel.
static int tier_merge(alz_handle* h, uint32_t ti, const alz_edge_out* in, const uint64_t* in_keys, uint32_t n,
                      const WinClock* clk_first, const WinClock* clk_last, const uint64_t* clk_unready) {
  alz_tier_set* ts = h->tiers;
  Tier& t = ts->tiers[ti];
  TierOpen* open = ts->d_open + ti;
  cudaStream_t s = h->stream;
  const int c = t.cur;
  const unsigned match_grid = (unsigned)std::min<uint64_t>((uint64_t)h->sms * 4u, (n + 255u) / 256u + 1u);
  tier_match_kernel<<<match_grid, 256, 0, s>>>(in, in_keys, n, t.d_bkeys[c], open, c, ts->d_ikeys, ts->d_pos,
                                               ts->d_unm, clk_first, clk_last, clk_unready, t.inputs == 0);
  exclusive_scan_u32(ts->d_tmp, ts->tmp_bytes, ts->d_unm, ts->d_scan, n + 1, s);
  const uint64_t groups = (uint64_t)t.cfg.block_rows + n;   // the block has at most block_rows rows
  const unsigned merge_grid = (unsigned)std::min<uint64_t>((uint64_t)h->sms * 8u, (groups * 8u + 255u) / 256u);
  tier_merge_kernel<<<merge_grid, 256, 0, s>>>(t.d_block[c], t.d_bkeys[c], open, c, in, ts->d_ikeys, ts->d_pos,
                                               ts->d_unm, ts->d_scan, n, (uint32_t)t.cfg.block_rows,
                                               t.d_block[c ^ 1], t.d_bkeys[c ^ 1]);
  h->launches += 3;
  CK(cudaGetLastError());
  t.cur = c ^ 1;
  return ALZ_OK;
}

static int tier_input(alz_handle* h, uint32_t ti, const alz_edge_out* in, const uint64_t* in_keys, uint32_t n,
                      const WinClock* clk_first, const WinClock* clk_last, const uint64_t* clk_unready,
                      uint64_t window_first, bool clocked, bool poisoned);

// Tier ti's open block has its factor-th input: retain it as the tier's newest entry, or drop it, and feed it to the
// tier above. One wait, for the block's count and overflow flag.
static int tier_close(alz_handle* h, uint32_t ti) {
  alz_tier_set* ts = h->tiers;
  Tier& t = ts->tiers[ti];
  TierOpen* open = ts->d_open + ti;
  cudaStream_t s = h->stream;
  CK(cudaMemcpyAsync(&ts->h_open, open, sizeof(TierOpen), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  const uint32_t n = ts->h_open.count[t.cur];
  const bool drop = t.poisoned || ts->h_open.overflow != 0u || n > t.cfg.arena_rows;
  const uint64_t window_first = t.window_first, window_last = h->windows;
  const bool clocked = t.clocked;
  if (drop) {
    t.ring.entries.clear();   // not retained, and the run would have a gap
    t.dropped += 1;
  } else {
    const int rc = t.ring.append(h, t.d_block[t.cur], n, clocked ? &open->clk : nullptr, window_first, window_last,
                                 t.inputs * t.windows_per_input);
    if (rc != ALZ_OK) return rc;
  }
  // the next input of the tier above reads this block before it is emptied (stream order)
  int rc = ALZ_OK;
  if (ti + 1 < ts->tiers.size())
    rc = tier_input(h, ti + 1, t.d_block[t.cur], t.d_bkeys[t.cur], drop ? 0u : n, &open->clk.first, &open->clk.last,
                    &open->clk.unready, window_first, clocked, drop);
  t.inputs = 0;
  t.poisoned = false;
  t.clocked = true;
  if (rc == ALZ_OK) {
    CK(cudaMemsetAsync(&open->count[t.cur], 0, sizeof(uint32_t), s));
    CK(cudaMemsetAsync(&open->overflow, 0, sizeof(uint32_t), s));
  }
  return rc;
}

static int tier_input(alz_handle* h, uint32_t ti, const alz_edge_out* in, const uint64_t* in_keys, uint32_t n,
                      const WinClock* clk_first, const WinClock* clk_last, const uint64_t* clk_unready,
                      uint64_t window_first, bool clocked, bool poisoned) {
  Tier& t = h->tiers->tiers[ti];
  if (t.inputs == 0) t.window_first = window_first;
  t.window_last = h->windows;   // an input is the flushed window, or a block closed by this flush
  t.clocked &= clocked;
  t.poisoned |= poisoned;
  if (!t.poisoned) {   // a poisoned block is dropped when it closes: what it holds does not matter
    const int rc = tier_merge(h, ti, in, in_keys, n, clocked ? clk_first : nullptr, clk_last, clk_unready);
    if (rc != ALZ_OK) return rc;
  }
  t.inputs += 1;
  return t.inputs == t.cfg.factor ? tier_close(h, ti) : ALZ_OK;
}

// the window a flush has just consumed (h->last_n_edges rows in h->d_out) is the next input of tier 1
static int tiers_input_window(alz_handle* h, const uint64_t* d_clk) {
  const WinClock* clk = reinterpret_cast<const WinClock*>(d_clk);
  return tier_input(h, 0, h->d_out, nullptr, h->last_n_edges, clk, clk, nullptr, h->windows, d_clk != nullptr, false);
}

extern "C" int alz_window_tier_state(alz_handle* h, uint32_t tier, alz_tier_state* out) {
  if (!h || !out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  const alz_tier_set* ts = h->tiers;
  if (!ts) return ALZ_E_STATE;
  if (tier == 0 || tier > ts->tiers.size()) return ALZ_E_INVAL;
  const Tier& t = ts->tiers[tier - 1];
  *out = alz_tier_state{};
  out->entries = (uint32_t)t.ring.entries.size();
  out->open_windows = t.inputs * t.windows_per_input;
  out->dropped = t.dropped;
  return ALZ_OK;
}

// ---- span rollups (docs/SPEC.md §14) --------------------------------------------------------------------------------

void alz_internal_free_span(alz_handle* h) {
  if (!h->span) return;
  free_scratch(h->span->sc);
  delete h->span;
  h->span = nullptr;
}

namespace {
// the best decomposition of the windows (p, W] found so far: its cost and its oldest unit, behind which comes the
// best decomposition of (units[unit].window_last, W]
struct SpanBest {
  uint64_t rows, units;
  int unit;
};

// a before b under the rule of docs/SPEC.md §14: fewer source rows, then fewer units; two decompositions of one
// span with equal counts have their oldest units start at the same window, so the coarser oldest unit decides
bool span_better(const SpanBest& a, const SpanBest& b, const std::vector<Piece>& units) {
  if (a.rows != b.rows) return a.rows < b.rows;
  if (a.units != b.units) return a.units < b.units;
  return units[a.unit].level > units[b.unit].level;
}
}  // namespace

// Every retained piece, with what the host must read from the device for it: every tier's TierOpen and the clocks
// of every arena, in one wait.
static int span_units(alz_handle* h, alz_span_state* sp, std::vector<Piece>& units) {
  cudaStream_t s = h->stream;
  alz_rollup_state* st = h->roll;
  alz_tier_set* ts = h->tiers;
  if (st) CK(cudaMemcpyAsync(st->ring.h_clk.data(), st->ring.d_clk, (size_t)st->ring.depth * sizeof(WinClock),
                             cudaMemcpyDeviceToHost, s));
  if (ts) {
    sp->h_open.resize(ts->tiers.size());
    CK(cudaMemcpyAsync(sp->h_open.data(), ts->d_open, ts->tiers.size() * sizeof(TierOpen), cudaMemcpyDeviceToHost, s));
    for (Tier& t : ts->tiers)
      CK(cudaMemcpyAsync(t.ring.h_clk.data(), t.ring.d_clk, (size_t)t.ring.depth * sizeof(TierClk),
                         cudaMemcpyDeviceToHost, s));
  }
  CK(cudaStreamSynchronize(s));
  units.clear();
  auto add_ring = [&units](const auto& r, uint32_t level) {
    for (const Entry& e : r.entries) {
      units.push_back(r.piece(e, level));
      units.back().clocked = r.clocked(e, &units.back().epoch_first, &units.back().epoch_last);
    }
  };
  if (st) add_ring(st->ring, 0u);
  if (ts)
    for (uint32_t i = 0; i < ts->tiers.size(); ++i) {
      const Tier& t = ts->tiers[i];
      add_ring(t.ring, i + 1u);
      const TierOpen& o = sp->h_open[i];
      if (t.inputs == 0 || t.poisoned || o.overflow != 0u) continue;   // nothing in it, or not what it covers
      Piece p{t.d_block[t.cur], t.d_bkeys[t.cur], 0, o.count[t.cur], t.window_first, t.window_last,
              t.inputs * t.windows_per_input, i + 1u, true, false, 0, 0};
      p.clocked = t.clocked && clock_epochs(o.clk, &p.epoch_first, &p.epoch_last);
      units.push_back(p);
    }
  return ALZ_OK;
}

// The plan: the span m the mode picks among the coverable ones, and the units that cover (W - m, W] (oldest first).
static uint64_t span_plan(const std::vector<Piece>& units, uint64_t W, uint64_t N, uint32_t mode,
                          std::vector<int>& plan) {
  // best[p]: the best decomposition of (p, W]. A unit [a, b] extends best[b] to best[a - 1]; taking units by
  // descending b, best[b] is final when its units come (every unit that ends at b' > b came before).
  std::vector<int> order(units.size());
  for (size_t i = 0; i < units.size(); ++i) order[i] = (int)i;
  std::sort(order.begin(), order.end(), [&](int a, int b) { return units[a].window_last > units[b].window_last; });
  std::unordered_map<uint64_t, SpanBest> best;
  best[W] = SpanBest{0, 0, -1};
  for (int i : order) {
    const Piece& u = units[i];
    const auto it = best.find(u.window_last);
    if (it == best.end()) continue;
    const SpanBest c{it->second.rows + u.n, it->second.units + 1u, i};
    const auto at = best.find(u.window_first - 1u);
    if (at == best.end()) best.emplace(u.window_first - 1u, c);
    else if (span_better(c, at->second, units)) at->second = c;
  }
  // windows are counted in 32 bits (alz_rollup_info.windows): larger spans are not offered
  uint64_t lo = 0, hi = 0;   // the largest coverable m <= N; the smallest >= N (0: none)
  uint64_t top = 0;          // the largest coverable m
  for (const auto& kv : best) {
    const uint64_t m = W - kv.first;
    if (m >= (1ull << 32)) continue;
    top = std::max(top, m);
    if (m <= N) lo = std::max(lo, m);
    if (m >= N && (hi == 0 || m < hi)) hi = m;
  }
  const uint64_t m = mode == ALZ_SPAN_AT_MOST ? lo : (hi ? hi : top);
  plan.clear();
  for (uint64_t p = W - m; p != W;) {
    const int i = best[p].unit;
    plan.push_back(i);
    p = units[i].window_last;
  }
  return m;
}

// Sums the units of the plan into sp->sc.d_sum; *rows, *n_out. Caller holds h->mu and has set the device.
static int span_locked(alz_handle* h, uint64_t N, uint32_t mode, size_t* n_out, alz_span_info* info,
                       const alz_edge_out** rows) {
  *n_out = 0;
  if (!h->roll && !h->tiers) return ALZ_E_STATE;
  if (N == 0 || (mode != ALZ_SPAN_AT_MOST && mode != ALZ_SPAN_AT_LEAST)) return ALZ_E_INVAL;
  if (!h->span) {
    h->span = new (std::nothrow) alz_span_state();
    if (!h->span) return ALZ_E_NOMEM;
  }
  alz_span_state* sp = h->span;
  std::vector<Piece> units;
  int rc = span_units(h, sp, units);
  if (rc != ALZ_OK) return rc;
  std::vector<int> plan;
  span_plan(units, h->windows, N, mode, plan);
  std::vector<Piece> pieces;
  for (int i : plan) pieces.push_back(units[i]);
  uint64_t n_src = 0;
  for (const Piece& p : pieces) n_src += p.n;
  rc = sum_pieces(h, sp->sc, pieces, n_src, n_out);
  if (rc != ALZ_OK) return rc;
  *rows = sp->sc.d_sum;
  if (info) {
    *info = alz_span_info{};
    fill_info(pieces, &info->r);
    for (const Piece& p : pieces) {
      if (p.open) info->open_blocks |= 1u << p.level;
      else info->entries[p.level] += 1u;
    }
  }
  return ALZ_OK;
}

extern "C" int alz_window_rollup_span_device(alz_handle* h, uint64_t windows, uint32_t mode,
                                             const alz_edge_out** dev_rows, size_t* n_out, alz_span_info* info) {
  return rollup_call(h, ALZ_ROLLUP_SPAN, false, nullptr, 0, dev_rows, n_out,
                     [&](const alz_edge_out** rows, alz_rollup_info* ri) {
                       alz_span_info si;
                       const int rc = span_locked(h, windows, mode, n_out, &si, rows);
                       if (rc == ALZ_OK) { *ri = si.r; if (info) *info = si; }
                       return rc;
                     });
}

extern "C" int alz_window_rollup_span(alz_handle* h, uint64_t windows, uint32_t mode, alz_edge_out* out, size_t cap,
                                      size_t* n_out, alz_span_info* info) {
  return rollup_call(h, ALZ_ROLLUP_SPAN, true, out, cap, nullptr, n_out,
                     [&](const alz_edge_out** rows, alz_rollup_info* ri) {
                       alz_span_info si;
                       const int rc = span_locked(h, windows, mode, n_out, &si, rows);
                       if (rc == ALZ_OK) { *ri = si.r; if (info) *info = si; }
                       return rc;
                     });
}
