// alz_metrics.cuh — what alz_metrics.cu shares with the changes (alz_changes.cu), the edge series (alz_series.cu),
// the edge, node and group trends (alz_trends.cu), the node calls (alz_nodes.cu), the node series
// (alz_node_series.cu), the groups (alz_groups.cu), the group series (alz_group_series.cu), the reach calls
// (alz_reach.cu) and the cycles calls (alz_cycles.cu): the §17 metric values of a row list, of node rows or of series
// slots, a source's rows, the rows' packed keys, the grow-on-demand device buffers and launch grids, the node
// group-by, a source's edge, node or group series into given buffers, the 64-bit top selection with its own scratch,
// the §24 group-by into given buffers, the map lookup and the graph of a row list.
#pragma once
#include <algorithm>
#include <cstdint>
#include <initializer_list>
#include <utility>

#include "alz_handle.h"

namespace alz {
namespace metrics {

// the CUB item counts are ints and the selection's tile counts pack two 32-bit counts: at most 2^30 - 1 rows
constexpr uint32_t kMaxRows = (1u << 30) - 1u;

// a node key a flush can produce (§22's key rule): a type up to ALZ_NODE_OUTBOUND_HOST, a pod or service value below
// 2^29
inline bool valid_node_key(uint32_t type, uint32_t value) {
  if (type > ALZ_NODE_OUTBOUND_HOST) return false;
  return (type != ALZ_NODE_POD && type != ALZ_NODE_SVC) || value < (1u << 29);
}
// a node key of §26: one valid_node_key accepts, or a group below 2^29
inline bool valid_group_node_key(uint32_t type, uint32_t value) {
  return type == ALZ_NODE_GROUP ? value < (1u << 29) : valid_node_key(type, value);
}

struct MetricSet {
  uint32_t nm;
  uint32_t kind[ALZ_MAX_METRICS];
  double q[ALZ_MAX_METRICS];
};
// m[0, nm) is a valid metric list (docs/SPEC.md §17); *ms its kernel form
bool valid_metrics(const alz_metric* m, uint32_t nm, MetricSet* ms);

struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
};
void free_bufs(std::initializer_list<DevBuf*> bufs);

// Every buffer in `need` holds at least its bytes. The last calls may still read them: one wait before the first
// buffer is replaced. A failed allocation leaves that buffer empty and returns ALZ_E_NOMEM.
int reserve(alz_handle* h, std::initializer_list<std::pair<DevBuf*, size_t>> need);

// The blocks of a 256-thread grid-stride launch over `threads` items: one per 256, at least 1, at most per_sm per SM
inline unsigned grid_for(alz_handle* h, uint64_t threads, unsigned per_sm) {
  return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((threads + 255) / 256, (uint64_t)h->sms * per_sm));
}

// The metrics of n rows into out[n * ms.nm], on the stream; no wait
int run_metrics(alz_handle* h, const alz_edge_out* rows, uint32_t n, const MetricSet& ms, double* out);

// The packed keys of n rows into keys[n], on the stream (16 of a row's 296 bytes read)
void launch_row_keys(alz_handle* h, const alz_edge_out* rows, uint32_t n, uint64_t* keys);

// The rows of an edge series (alz_series.cu): output row i = (series row i / P, point i % P) reads the arena row in
// slot[u * P + point], u = map[series row] (map null: u = the series row), or nothing when that slot is kSlotAbsent;
// present[i] says which.
constexpr uint32_t kSlotAbsent = 0xFFFFFFFFu;
struct SeriesRows {
  static constexpr bool kMayBeAbsent = true;
  const alz_edge_out* arena;
  const uint32_t* slot;
  const uint32_t* map;
  uint32_t points;
  uint8_t* present;
#ifdef __CUDACC__
  __device__ __forceinline__ const alz_edge_out* operator()(uint32_t i) const {
    const uint32_t e = i / points, j = i - e * points;
    const uint32_t s = slot[(map ? map[e] : e) * points + j];
    return s == kSlotAbsent ? nullptr : arena + s;
  }
  __device__ __forceinline__ void mark(uint32_t i, bool p) const { present[i] = p ? 1u : 0u; }
#endif
};
// The metrics of the n = rows x P series slots into out[n * ms.nm] and present[n], on the stream; no wait
int run_metrics_series(alz_handle* h, const SeriesRows& rows, uint32_t n, const MetricSet& ms, double* out);

// The rows of a node metric (alz_nodes.cu): output row i reads side `side` of node row i in place. A side's sums are
// laid out as alz_edge_out from count on, so the row it reads starts sizeof(alz_node_sums) x side bytes into the node
// row (alz_nodes.cu asserts the offsets this relies on).
struct NodeRows {
  static constexpr bool kMayBeAbsent = false;
  const alz_node_out* nodes;
  uint32_t side;
#ifdef __CUDACC__
  __device__ __forceinline__ const alz_edge_out* operator()(uint32_t i) const {
    return reinterpret_cast<const alz_edge_out*>(reinterpret_cast<const char*>(nodes + i) +
                                                 (size_t)side * sizeof(alz_node_sums));
  }
#endif
};
// The metrics of n node rows' one side into out[n * ms.nm], on the stream; no wait
int run_metrics_nodes(alz_handle* h, const NodeRows& rows, uint32_t n, const MetricSet& ms, double* out);

// The rows of a node series (alz_node_series.cu): output row i = (series row i / P, point i % P) reads side `side` of
// the node row slot[u * P + point], u = map[series row] (map null: u = the series row), or nothing when that slot is
// kSlotAbsent; present[i] says which.
struct NodeSeriesRows {
  static constexpr bool kMayBeAbsent = true;
  const alz_node_out* nodes;
  const uint32_t* slot;
  const uint32_t* map;
  uint32_t points, side;
  uint8_t* present;
#ifdef __CUDACC__
  __device__ __forceinline__ const alz_edge_out* operator()(uint32_t i) const {
    const uint32_t e = i / points, j = i - e * points;
    const uint32_t s = slot[(map ? map[e] : e) * points + j];
    return s == kSlotAbsent ? nullptr : NodeRows{nodes, side}(s);
  }
  __device__ __forceinline__ void mark(uint32_t i, bool p) const { present[i] = p ? 1u : 0u; }
#endif
};
// The metrics of the n = rows x P node series slots into out[n * ms.nm] and present[n], on the stream; no wait
int run_metrics_node_series(alz_handle* h, const NodeSeriesRows& rows, uint32_t n, const MetricSet& ms, double* out);

// The node group-by of alz_nodes.cu over (key, 2 x row + side) pairs, in buffers its caller owns, so the node calls
// and the node series each keep their own
struct NodeGroup {
  DevBuf keys_in, keys_out, vals_in, vals_out, heads, idx, tmp;
  uint32_t* h_words = nullptr;   // pinned: [0] the runs of the last node_group_runs, [1] free for the caller
  void free();
};
// node calls read sources of at most this many rows: their 2n pairs stay within the selection's 2^30 - 1
constexpr uint32_t kMaxNodeSourceRows = (1u << 29) - 1u;
// the node key's bits: a uint8 type above a 32-bit value
constexpr int kNodeKeyBits = 40;
// Room for n2 pairs in g.keys_in / g.vals_in and the scratch of node_group_runs. ALZ_E_NOMEM when one cannot grow.
int node_group_reserve(alz_handle* h, NodeGroup& g, uint32_t n2);
// The 2n pairs of n rows into g.keys_in / g.vals_in, on the stream: pair 2i + side is row i's end on `side` (§21)
void node_group_keys(alz_handle* h, NodeGroup& g, const alz_edge_out* rows, uint32_t n);
// g's n2 pairs sorted on the keys' low key_bits bits (g.keys_out / g.vals_out), the run heads (g.heads) and run
// numbers (g.idx, an exclusive scan of the heads), then one wait; g.h_words[0] = the runs after it
int node_group_runs(alz_handle* h, NodeGroup& g, uint32_t n2, int key_bits);
// One node row per run of the first n2 sorted pairs into out[g.idx[run head]], on the stream; a pair's row is
// rows + (val >> 1) and its side val & 1. A row's head word is its run's key as (key >> 32, key).
int node_group_reduce(alz_handle* h, const NodeGroup& g, const alz_edge_out* rows, uint32_t n2, alz_node_out* out);
// out[j] = nodes[idx[j]] for j < m, on the stream
int node_gather(alz_handle* h, const uint32_t* idx, uint32_t m, const alz_node_out* nodes, alz_node_out* out);
// The rows of `source`, checked against kMaxNodeSourceRows (ALZ_E_CAPACITY). Caller holds h->mu.
int node_source(alz_handle* h, uint32_t source, const alz_edge_out** rows, size_t* n);
// The §21 node rows of n rows into `out`, grown to hold them, with g as the group-by's scratch: node_group_keys,
// node_group_runs (one wait), then node_group_reduce on the stream. *n_nodes = the nodes; more than cap:
// ALZ_E_CAPACITY before the reduce is enqueued. Caller holds h->mu and has set the device; n <= kMaxNodeSourceRows.
int node_rows_of(alz_handle* h, NodeGroup& g, DevBuf& out, const alz_edge_out* rows, size_t n, size_t cap,
                 size_t* n_nodes);

// The rows of a source and its windows (ALZ_SOURCE_WINDOW: the last flushed window, 1), or of the last rollup of a
// kind with what it reported (alz_changes.cu). Caller holds h->mu.
int source_rows(alz_handle* h, uint32_t source, const alz_edge_out** rows, size_t* n, alz_rollup_info* info);

// The buffers one edge series fills (alz_series.cu), grown on demand: the series calls own one set, the trend calls
// (alz_trends.cu) another, so neither clobbers the other's device results
struct SeriesBufs {
  DevBuf keys, map, runs, slot;   // the distinct query keys, caller row -> distinct key, the entries' runs, the slots
  DevBuf values, present;         // the results
  alz_ring_view view;
  void free();
};
// The series of the n source rows `rows` over the last min(k, retained) entries of tier `tier` into b.values /
// b.present, on the stream, with no wait of its own. *n_out = n, *n_points = P, *rows_in = the entries' rows.
// ALZ_E_CAPACITY for more than 2^30 - 1 slots or n > cap. Caller holds h->mu and has set the device.
int run_series_rows(alz_handle* h, SeriesBufs& b, const alz_edge_out* rows, size_t n, uint32_t tier, uint32_t k,
                    const MetricSet& ms, size_t cap, size_t* n_out, uint32_t* n_points, uint64_t* rows_in);

// The buffers one node series fills (alz_node_series.cu), grown on demand: the node series calls own one set, the
// node trend calls (alz_trends.cu) another
struct NodeSeriesBufs {
  NodeGroup g;                           // the group-by of the source's nodes, then of the entries' (node, point) slots
  DevBuf keys, map, runs, slot, miss;    // the distinct node keys, caller row -> distinct key, the entries' runs,
                                         // the slots' node rows, the entry rows that name no queried node
  DevBuf slot_rows, src_rows;            // one node row per present slot; the source's node rows (with_rows)
  DevBuf values, present;                // the results
  alz_ring_view view;
  void free();
};
// The node series of side `side` of the nodes of the n source rows `rows` over the last min(k, retained) entries of
// tier `tier` into b.values / b.present, on the stream: *n_out = the source's nodes (their keys in b.keys), *n_points =
// P, *rows_in = the entries' rows. with_rows: the source's node rows too, in b.src_rows. Waits once for the node count
// and the ring's clocks (when the source has rows) and once for the present slots (when the entries have rows).
// ALZ_E_CAPACITY for more than 2^30 - 1 slots or nodes > cap. Caller holds h->mu and has set the device;
// n <= kMaxNodeSourceRows.
int run_node_series_rows(alz_handle* h, NodeSeriesBufs& b, const alz_edge_out* rows, size_t n, uint32_t side,
                         uint32_t tier, uint32_t k, const MetricSet& ms, bool with_rows, size_t cap, size_t* n_out,
                         uint32_t* n_points, uint64_t* rows_in);

// The group map (alz_groups.cu): n node keys ascending and each one's group
struct GroupMap {
  const uint64_t* keys = nullptr;
  const uint32_t* groups = nullptr;
  uint32_t n = 0;
};
GroupMap group_map(const alz_handle* h);
#ifdef __CUDACC__
// the group node of a node key when the map holds it, the key itself otherwise; *hit += 1 when it held it
__device__ __forceinline__ uint64_t map_end(uint64_t key, const uint64_t* __restrict__ mk,
                                            const uint32_t* __restrict__ mg, uint32_t m, uint32_t* hit) {
  uint32_t lo = 0, hi = m;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (mk[mid] < key) lo = mid + 1; else hi = mid;
  }
  if (lo < m && mk[lo] == key) {
    *hit += 1u;
    return ((uint64_t)ALZ_NODE_GROUP << 32) | mg[lo];
  }
  return key;
}
// map_end for callers that do not count the keys the map held
__device__ __forceinline__ uint64_t map_end(uint64_t key, const uint64_t* __restrict__ mk,
                                            const uint32_t* __restrict__ mg, uint32_t m) {
  uint32_t held = 0;   // dropped: the compiler removes the count
  return map_end(key, mk, mg, m, &held);
}
#endif

// A node series whose entry rows' ends pass through the group map `map` before the lookup (group node series,
// alz_group_series.cu): of the nodes of the n rows `rows` (by_source, as run_node_series_rows; the group-edge rows of a
// source give its group nodes), or of the caller's n_keys keys (each already checked). *waited as run_node_series_rows'
// waits happened after the ring's clocks were enqueued.
int run_mapped_node_series(alz_handle* h, NodeSeriesBufs& b, bool by_source, const alz_edge_out* rows, size_t n,
                           const alz_node_ends* keys, size_t n_keys, const GroupMap& map, uint32_t side,
                           uint32_t tier, uint32_t k, const MetricSet& ms, bool with_rows, size_t cap, size_t* n_out,
                           uint32_t* n_points, uint64_t* rows_in, bool* waited);
// The entries of a ring view as one virtual row space: runs = first[P] then vbase[P + 1]; returns the entries' rows
uint64_t entry_runs(const alz_ring_view& v, std::vector<uint32_t>* runs);
// The slot group-by of a node series once its R pairs (slot key, 2 x arena row + side) are in b.g.keys_in /
// b.g.vals_in, slot keys below n_slots and n_slots for a row that names no queried key, those counted in b.miss: one
// node row per present slot into b.slot_rows and b.slot[slot key] = its row (the caller set b.slot to kSlotAbsent).
// One wait. Caller holds h->mu and has set the device.
int node_series_slots(alz_handle* h, NodeSeriesBufs& b, const alz_edge_out* arena, uint32_t R, uint64_t n_slots);

// The buffers one group series fills (alz_group_series.cu): the source's group-edge rows and the series over them.
// The group series calls own one set, the group trend calls (alz_trends.cu) another.
struct GroupSeriesBufs {
  NodeSeriesBufs s;   // the series (for group edges, keys holds 16-byte (from key, to key) pairs)
  DevBuf edges;       // the source's §24 group-edge rows
  void free();
};
// The group series of the n source rows `rows` into b (s.values / s.present), on the stream: nodes false, every group
// edge of the rows (series rows in b.edges, *n_out of them); nodes true, every group node on side `side` (keys in
// b.s.keys; with_rows: their node rows in b.s.src_rows). *n_points = P, *rows_in = the entries' rows. ALZ_E_CAPACITY
// for more than 2^30 - 1 slots or series rows > cap. Caller holds h->mu and has set the device; n <=
// kMaxNodeSourceRows.
int run_group_series_rows(alz_handle* h, GroupSeriesBufs& b, const alz_edge_out* rows, size_t n, bool nodes,
                          uint32_t side, uint32_t tier, uint32_t k, const MetricSet& ms, bool with_rows, size_t cap,
                          size_t* n_out, uint32_t* n_points, uint64_t* rows_in);

// The scratch and the results of one top selection over 64-bit values, grown on demand
struct Selection {
  DevBuf words, tile_cnt, cand_key, cand_idx, sorted_key, sorted_idx, tmp;   // the selection's scratch
  DevBuf top_rows, top_values, top_index;                                      // its results
  void free();
};
// The selection of the top k of n float64 values (their bits, in device memory); rows: the rows to gather from, or
// null. *m_out results in s.top_index / s.top_values (/ s.top_rows), *above eligible values.
int select_top(alz_handle* h, Selection& s, const uint64_t* vals, uint32_t n, uint32_t k, double min_value,
               const alz_edge_out* rows, size_t* m_out, uint64_t* above);

// The §24 group-edge rows of n rows under the handle's map into `out`, grown to hold them, with the group calls'
// scratch (alz_groups.cu): two waits, then the reduce on the stream. *n_out = the rows; more than cap: ALZ_E_CAPACITY
// before the reduce is enqueued. Caller holds h->mu and has set the device; n <= kMaxNodeSourceRows.
int group_edges_into(alz_handle* h, DevBuf& out, const alz_edge_out* rows, size_t n, size_t cap, size_t* n_out,
                     alz_group_info* info);
// The §21 node rows of n group-edge rows into `out` with the group calls' scratch, as node_rows_of
int group_nodes_into(alz_handle* h, DevBuf& out, const alz_edge_out* edges, size_t n, size_t* n_nodes);
// The map's generation: every alz_group_set that succeeds moves it on (0 before the first)
uint64_t group_map_generation(const alz_handle* h);

// The graph of a traversed row list (alz_reach.cu), which the reach and cycles calls (alz_cycles.cu) search: each row
// end's node index (§21 node list order), each node's key, which rows are traversable, and CSRs by tail
struct Graph {
  NodeGroup g;                  // the §21 group-by of the rows' ends
  DevBuf end_node, node_keys;   // end_node[2r] row r's to end's index, [2r + 1] its from end's; node_keys[index]
  DevBuf values, trav;          // the filter's metric values, each row traversable (1) or not (0)
  DevBuf tmp;                   // CUB scratch: a scan of max(nodes, rows) + 1 words
  uint32_t nodes = 0;
  void free();
};
// A CSR by tail: off[nodes + 1], and adj[off[u] ..] = (head << 32) | row for each orientation of a traversable row
// with tail u that the direction follows (ALZ_REACH_DOWN: from -> to; UP: to -> from; ANY: both)
struct Csr {
  DevBuf off, cursor, adj;
  void free();
};
// gr over n rows: the §21 sort of the ends (one wait, for the node count), the index scatter, with ms the metric
// filter (a row is traversable when key(value) >= key(min_value)), then one CSR per (direction, csr) pair, on the
// stream. Caller holds h->mu and has set the device; 0 < n <= kMaxNodeSourceRows.
int graph_build(alz_handle* h, Graph& gr, const alz_edge_out* rows, uint32_t n, const MetricSet* ms, double min_value,
                std::initializer_list<std::pair<uint32_t, Csr*>> csrs);

// Buffers of one family of scored calls (below), each grown on demand and never shrunk; freed in alz_destroy. The edge
// trend calls own one (h->trends), the node trend calls another (h->node_trends), the group trend calls a third
// (h->group_trends), and the edge, node and group correlation calls (alz_corr.cu) three more, each using its own
// series buffers.
}  // namespace metrics
}  // namespace alz
struct alz_trend_state {
  alz::metrics::SeriesBufs ser;        // edges: the series of the source's rows, one metric
  alz::metrics::NodeSeriesBufs nser;   // nodes: the series of the source's nodes, one metric, and their node rows
  alz::metrics::GroupSeriesBufs gser;  // groups: the source's group-edge rows and their or their group nodes' series
  alz::metrics::DevBuf rec, sel_val, valid_cnt;   // the records, the selection values, the valid count
  alz::metrics::DevBuf top_rec, top_values, top_present, top_nodes;   // the top call's records, series and node rows
  alz::metrics::Selection sel;         // the top call's selection (and, for edges, its gathered source rows)
  uint32_t* h_valid = nullptr;         // pinned: the valid count, read after the call's wait
  alz::metrics::DevBuf target;         // correlations: the target's values, then its presence bytes
  void* h_target = nullptr;            // correlations: pinned staging of the same
  size_t h_target_bytes = 0;
};
namespace alz {
namespace metrics {

// One call of a family that scores each series row of a source (alz_trends.cu: the trends; alz_corr.cu: the
// correlations): the series of one metric, one 48-byte record per row, and for a top call the selection and a gather of
// the top records with their series. The family's state is an alz_trend_state.
struct ScoredCall {
  bool top = false, node = false, group = false;
  uint32_t source = 0, side = 0, tier = 0, k = 0, n_top = 0;
  double min_value = 0.0;
  MetricSet ms{};
  // given: score these N x P device series (values[i * P + j], present[i * P + j]) instead of a source's; no rows,
  // no ring
  bool given = false;
  const double* given_values = nullptr;
  const uint8_t* given_present = nullptr;
  size_t given_n = 0;
  uint32_t given_points = 0;
};
// What the per-row pass reads: N series rows of P points, and what the records' heads come from (rows: the edge rows,
// keys: the node keys; both null for given series)
struct ScoredInput {
  size_t n = 0;
  uint32_t points = 0;
  const double* values = nullptr;
  const uint8_t* present = nullptr;
  const alz_edge_out* rows = nullptr;
  const uint64_t* keys = nullptr;
};
// The family's per-row pass: rec[i] (48 bytes) for every row and, with sel, the row's selection value (its score's
// bits when valid, all ones otherwise); *valid_cnt += the valid rows. Enqueued on the stream, no wait.
struct ScorePass {
  virtual int launch(alz_handle* h, alz_trend_state& s, const ScoredInput& in, void* rec, uint64_t* sel,
                     uint32_t* valid_cnt) = 0;
};
// A call's results, on the device: m records (and, for a top call, m source rows or node rows, their selection indices
// and m x P series points)
struct ScoredResult {
  const void* rec = nullptr;
  const void* rows = nullptr;
  const uint32_t* index = nullptr;
  const double* values = nullptr;
  const uint8_t* present = nullptr;
  size_t m = 0;
};
// The skeleton of one call into the state sp (created on first use; `what` names the family in errors): the source's
// series, pass.launch, the selection and the gather, then the waits, after which *res, *n_points, points and *info
// (points = P, edges = the series rows) are final. cap: a host full-list call's room (checked before the entries are
// read); copy_out: where that call's records go, copied before its last wait. Caller holds h->mu.
int scored_series_locked(alz_handle* h, alz_trend_state*& sp, const char* what, const ScoredCall& c, size_t cap,
                         void* copy_out, ScorePass& pass, ScoredResult* res, uint32_t* n_points,
                         alz_rollup_info* points, alz_trend_info* info);
void free_scored_state(alz_trend_state*& s);

#ifdef __CUDACC__
// The first 16 bytes of an edge record: the source row's ends, with `valid` at byte 2
struct EdgeHead {
  const alz_edge_out* rows;
  __device__ __forceinline__ uint4 operator()(uint32_t i, bool ok) const {
    const uint2* row = reinterpret_cast<const uint2*>(rows + i);
    const uint2 ty = row[0], ft = row[1];   // from_type, to_type, pad | from, to
    return make_uint4((ty.x & 0xFFFFu) | ((ok ? 1u : 0u) << 16), 0u, ft.x, ft.y);
  }
};

// The first 16 bytes of a node record: the node's type and value from its key (type << 32) | value
struct NodeHead {
  const uint64_t* keys;
  __device__ __forceinline__ uint4 operator()(uint32_t i, bool ok) const {
    const uint64_t k = keys[i];
    return make_uint4((uint32_t)(k >> 32) | ((ok ? 1u : 0u) << 16), 0u, (uint32_t)k, 0u);
  }
};
#endif

}  // namespace metrics
}  // namespace alz
