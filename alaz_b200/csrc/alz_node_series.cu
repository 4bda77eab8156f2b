// alz_node_series.cu — node series (docs/SPEC.md §22): the §17 metric values of one side of a source's nodes, or of
// nodes the caller names, in each of the last P closed entries of one ring (the window history or a tier), oldest
// first. Point j of a node sums every row of entry j on that side of it, so unlike an edge series it is a group-by of
// the entry's rows, and it reuses the §21 one (alz_nodes.cu, DESIGN.md §5.14):
//   keys    a source's nodes: the §21 group-by's sort, heads and scan over its rows' 2n ends, one wait for the node
//           count, then the run heads' keys (and, for a top trend call, the §21 reduce into the source's node rows).
//           Caller keys are checked first, then packed (type << 32) | value, sorted and made distinct on the host,
//           with a map from each caller row to its distinct key.
//   pairs   one thread per row of the P entries, numbered in one virtual row space (entry j takes [vbase[j],
//           vbase[j + 1])): the node key of its end on the side, a lower bound into the N query keys, and the pair
//           (slot key u x P + j, 2 x arena row + side). A row that names no queried node gets the key N x P, which
//           sorts after every slot, and is counted.
//   group   the same sort (on the bits of N x P), heads, scan and one wait for the runs; the present slots are the
//           runs less the misses' run. The §21 split and reduce over the hit pairs, with the arena as the rows, give
//           one node row per present slot, summed on the side (a hub's runs cross tiles and take the red.add path).
//   slots   slot[u x P + j] = that node row, or kSlotAbsent
//   values  the §17 metric kernels of alz_metrics.cu over the slots (NodeSeriesRows)
// Waits: the device call waits for the node count (with the ring's clocks) and for the runs; the host call once more,
// for its results. Growing a buffer adds one.
#include <algorithm>
#include <mutex>
#include <string>
#include <vector>

#include "alz_metrics.cuh"

using namespace alz;
using namespace alz::metrics;

static_assert(sizeof(alz_node_ends) == 8, "alz_node_ends is the head of alz_node_out");
static_assert(offsetof(alz_node_ends, value) == offsetof(alz_node_out, value), "alz_node_ends is alz_node_out's head");

namespace {

// Thread t: row t of the entries' virtual row space (entry j holds arena rows [first[j], first[j] + vbase[j + 1] -
// vbase[j]), n_rows = vbase[points]): its pair, and a warp-reduced count of the rows that name no queried node.
// kMapped: the row's end passes through the group map (mk, mg, m) first (group node series, alz_group_series.cu); the
// map's arguments come last, so the unmapped kernel reads its arguments where it always did.
template <bool kMapped>
__global__ void __launch_bounds__(256) node_series_pairs_kernel(const alz_edge_out* __restrict__ arena,
                                                                const uint32_t* __restrict__ first,
                                                                const uint32_t* __restrict__ vbase, uint32_t points,
                                                                uint32_t n_rows, uint32_t side,
                                                                const uint64_t* __restrict__ keys, uint32_t n_keys,
                                                                uint64_t* __restrict__ pair_keys,
                                                                uint32_t* __restrict__ pair_vals,
                                                                uint32_t* __restrict__ misses,
                                                                const uint64_t* __restrict__ mk,
                                                                const uint32_t* __restrict__ mg, uint32_t m) {
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint64_t miss_key = (uint64_t)n_keys * points;
  uint32_t n_miss = 0;
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n_rows; t += stride) {
    uint32_t lo = 0, hi = points;   // the last entry j with vbase[j] <= t (an empty entry is passed over)
    while (hi - lo > 1u) {
      const uint32_t mid = (lo + hi) >> 1;
      if (vbase[mid] <= t) lo = mid; else hi = mid;
    }
    const uint32_t row = first[lo] + (t - vbase[lo]);
    const uint2* r = reinterpret_cast<const uint2*>(arena + row);   // rows are 296 bytes apart: 8-byte aligned
    const uint2 ty = r[0], ft = r[1];                               // from_type, to_type, pad | from, to
    uint64_t key = side == ALZ_SIDE_IN ? node_key((ty.x >> 8) & 0xFFu, ft.y) : node_key(ty.x & 0xFFu, ft.x);
    if (kMapped) key = map_end(key, mk, mg, m);
    const uint32_t u = lower_bound_u64(keys, n_keys, key);
    const bool hit = u < n_keys && keys[u] == key;
    pair_keys[t] = hit ? (uint64_t)u * points + lo : miss_key;
    pair_vals[t] = 2u * row + side;   // arena rows are below 2^31
    n_miss += hit ? 0u : 1u;
  }
  n_miss = __reduce_add_sync(0xFFFFFFFFu, n_miss);   // every lane of the warp leaves the loop to get here
  if ((threadIdx.x & 31u) == 0 && n_miss) atomicAdd(misses, n_miss);
}

// keys[idx[j]] = the key of the run that starts at sorted pair j: the source's distinct node keys, ascending
__global__ void __launch_bounds__(256) node_run_keys_kernel(const uint64_t* __restrict__ sorted,
                                                            const uint32_t* __restrict__ heads,
                                                            const uint32_t* __restrict__ idx, uint32_t n2,
                                                            uint64_t* __restrict__ keys) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n2; j += stride)
    if (heads[j]) keys[idx[j]] = sorted[j];
}

// slot[key] = idx[j] for the run that starts at sorted hit pair j: the slot's node row
__global__ void __launch_bounds__(256) node_slot_kernel(const uint64_t* __restrict__ sorted,
                                                        const uint32_t* __restrict__ heads,
                                                        const uint32_t* __restrict__ idx, uint32_t n_hits,
                                                        uint32_t* __restrict__ slot) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n_hits; j += stride)
    if (heads[j]) slot[sorted[j]] = idx[j];
}

int key_bits_of(uint64_t max_key) { return 64 - __builtin_clzll(max_key); }

}  // namespace

// Buffers of the node series calls, each grown on demand and never shrunk; freed in alz_destroy
struct alz_node_series_state {
  NodeSeriesBufs b;
};

void alz::metrics::NodeSeriesBufs::free() {
  g.free();
  free_bufs({&keys, &map, &runs, &slot, &miss, &slot_rows, &src_rows, &values, &present});
}

void alz_internal_free_node_series(alz_handle* h) {
  alz_node_series_state* s = h->node_series;
  if (!s) return;
  s->b.free();
  delete s;
  h->node_series = nullptr;
}

namespace {

// The nodes of a series: a source's rows (rows, n_rows) or the caller's keys, packed, as distinct sorted keys and a map
struct Nodes {
  bool by_source = false;
  const alz_edge_out* rows = nullptr;    // source rows
  size_t n_rows = 0;
  const alz_node_ends* ends = nullptr;   // caller keys
  size_t n = 0;                          // series rows
  std::vector<uint64_t> keys;            // caller keys: the distinct packed keys
  std::vector<uint32_t> map;             // caller row -> index into keys
};

// whether a caller's key names a node a flush can produce: a type up to ALZ_NODE_OUTBOUND_HOST, a pod or service
// value below 2^29
bool valid_node(const alz_node_ends& e) { return valid_node_key(e.type, e.value); }

// q->keys and q->map from the caller's keys, every one valid_node
void caller_nodes(Nodes* q) {
  std::vector<uint64_t> packed(q->n);
  for (size_t i = 0; i < q->n; ++i) packed[i] = ((uint64_t)q->ends[i].type << 32) | q->ends[i].value;
  q->keys = packed;
  std::sort(q->keys.begin(), q->keys.end());
  q->keys.erase(std::unique(q->keys.begin(), q->keys.end()), q->keys.end());
  q->map.resize(q->n);
  for (size_t i = 0; i < q->n; ++i)
    q->map[i] = (uint32_t)(std::lower_bound(q->keys.begin(), q->keys.end(), packed[i]) - q->keys.begin());
}

// The series of `q` over the last min(k, retained) entries of tier `tier` into b, on the stream: *n_out series rows,
// *n_points = P, *rows_in entry rows read, *waited when the call has waited since the ring's clocks were enqueued.
// map: the entry rows' ends pass through it before the lookup (null: they do not). n_out > cap: ALZ_E_CAPACITY before
// the entries are read. Caller holds h->mu and has set the device.
int node_series_enqueue(alz_handle* h, NodeSeriesBufs& b, Nodes& q, uint32_t side, uint32_t tier, uint32_t k,
                        const MetricSet& ms, bool with_rows, size_t cap, const GroupMap* map, size_t* n_out,
                        uint32_t* n_points, uint64_t* rows_in_out, bool* waited) {
  *waited = false;
  int rc = alz_internal_ring_view(h, tier, k, &b.view);
  if (rc != ALZ_OK) return rc;
  const alz_ring_view& v = b.view;
  const uint32_t P = (uint32_t)v.n.size();
  *n_points = P;
  cudaStream_t st = h->stream;
  NodeGroup& g = b.g;
  if (q.by_source && q.n_rows) {   // the source's nodes: the first wait, which also brings the ring's clocks
    const uint32_t n2 = 2u * (uint32_t)q.n_rows;
    rc = node_group_reserve(h, g, n2);
    if (rc != ALZ_OK) return rc;
    node_group_keys(h, g, q.rows, (uint32_t)q.n_rows);
    rc = node_group_runs(h, g, n2, kNodeKeyBits);
    if (rc != ALZ_OK) return rc;
    *waited = true;
    q.n = g.h_words[0];
  }
  const size_t n = q.n;
  *n_out = n;
  if ((uint64_t)n * P > kMaxRows) return ALZ_E_CAPACITY;
  if (n > cap) return ALZ_E_CAPACITY;
  if (!q.by_source) caller_nodes(&q);   // sorted once the sizes are known to fit
  const size_t n_keys = q.by_source ? n : q.keys.size();
  const size_t slots = n * P;
  std::vector<uint32_t> runs;
  const uint64_t rows_in = entry_runs(v, &runs);
  *rows_in_out = rows_in;
  rc = reserve(h, {{&b.keys, std::max<size_t>(n_keys, 1) * 8},
                   {&b.map, q.by_source ? 0 : std::max<size_t>(n, 1) * 4},
                   {&b.runs, runs.size() * 4},
                   {&b.slot, std::max<size_t>(n_keys * P, 1) * 4},
                   {&b.miss, 4},
                   {&b.src_rows, with_rows ? std::max<size_t>(n, 1) * sizeof(alz_node_out) : 0},
                   {&b.values, std::max<size_t>(slots * ms.nm, 1) * 8},
                   {&b.present, std::max<size_t>(slots, 1)}});
  if (rc != ALZ_OK) return rc;
  uint64_t* d_keys = static_cast<uint64_t*>(b.keys.p);
  if (q.by_source && n) {   // g still holds the source's sorted ends
    const uint32_t n2 = 2u * (uint32_t)q.n_rows;
    node_run_keys_kernel<<<grid_for(h, n2, 8), 256, 0, st>>>(static_cast<const uint64_t*>(g.keys_out.p),
                                                             static_cast<const uint32_t*>(g.heads.p),
                                                             static_cast<const uint32_t*>(g.idx.p), n2, d_keys);
    h->launches += 1;
    CK(cudaGetLastError());
    if (with_rows) {
      rc = node_group_reduce(h, g, q.rows, n2, static_cast<alz_node_out*>(b.src_rows.p));
      if (rc != ALZ_OK) return rc;
    }
  }
  if (!slots) return ALZ_OK;
  if (!q.by_source) {
    CK(cudaMemcpyAsync(d_keys, q.keys.data(), n_keys * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(b.map.p, q.map.data(), n * 4, cudaMemcpyHostToDevice, st));
  }
  uint32_t* d_runs = static_cast<uint32_t*>(b.runs.p);
  uint32_t* d_slot = static_cast<uint32_t*>(b.slot.p);
  CK(cudaMemcpyAsync(d_runs, runs.data(), runs.size() * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(d_slot, 0xFF, n_keys * P * 4, st));
  if (rows_in) {   // the entries' (slot, row) pairs, grouped by slot: the second wait
    const uint32_t R = (uint32_t)rows_in;
    rc = node_group_reserve(h, g, R);
    if (rc != ALZ_OK) return rc;
    uint32_t* d_miss = static_cast<uint32_t*>(b.miss.p);
    CK(cudaMemsetAsync(d_miss, 0, 4, st));
    uint64_t* pk = static_cast<uint64_t*>(g.keys_in.p);
    uint32_t* pv = static_cast<uint32_t*>(g.vals_in.p);
    if (map)
      node_series_pairs_kernel<true><<<grid_for(h, R, 8), 256, 0, st>>>(
          v.arena, d_runs, d_runs + P, P, R, side, d_keys, (uint32_t)n_keys, pk, pv, d_miss, map->keys, map->groups,
          map->n);
    else
      node_series_pairs_kernel<false><<<grid_for(h, R, 8), 256, 0, st>>>(
          v.arena, d_runs, d_runs + P, P, R, side, d_keys, (uint32_t)n_keys, pk, pv, d_miss, nullptr, nullptr, 0);
    h->launches += 1;
    rc = node_series_slots(h, b, v.arena, R, (uint64_t)n_keys * P);
    if (rc != ALZ_OK) return rc;
    *waited = true;
  }
  const NodeSeriesRows sr{static_cast<const alz_node_out*>(b.slot_rows.p), d_slot,
                          q.by_source ? nullptr : static_cast<const uint32_t*>(b.map.p), P, side,
                          static_cast<uint8_t*>(b.present.p)};
  return run_metrics_node_series(h, sr, (uint32_t)slots, ms, static_cast<double*>(b.values.p));
}

// The four entry points. by_source: the nodes of `source`; else the caller's keys. Device call: *dev_values /
// *dev_present; host call: cap series rows into values / present (either may be null when nothing is copied).
int series_entry(alz_handle* h, bool by_source, uint32_t source, const alz_node_ends* keys, size_t n_keys,
                 uint32_t side, uint32_t tier, uint32_t k, const alz_metric* m, uint32_t nm, bool device,
                 double* values, uint8_t* present, size_t cap, const double** dev_values, const uint8_t** dev_present,
                 size_t* n_out, uint32_t* n_points, alz_rollup_info* points, alz_series_info* info) {
  if (!h || !n_out || !n_points) {
    if (n_out) *n_out = 0;
    if (n_points) *n_points = 0;
    return ALZ_E_INVAL;
  }
  *n_out = 0;
  *n_points = 0;
  MetricSet ms;
  if (k == 0 || side > ALZ_SIDE_OUT || !valid_metrics(m, nm, &ms)) return ALZ_E_INVAL;
  if (device ? !dev_values : (!values && cap)) return ALZ_E_INVAL;
  Nodes q;
  if (by_source) {
    if (source != ALZ_SOURCE_WINDOW && source > ALZ_ROLLUP_SPAN) return ALZ_E_INVAL;
    q.by_source = true;
  } else {
    if (!keys && n_keys) return ALZ_E_INVAL;
    for (size_t i = 0; i < n_keys; ++i)   // a malformed key is refused whatever the sizes
      if (!valid_node(keys[i])) return ALZ_E_INVAL;
    q.ends = keys;
    q.n = n_keys;
  }
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  if (by_source) {
    const int rc = node_source(h, source, &q.rows, &q.n_rows);
    if (rc != ALZ_OK) return rc;
  }
  if (!h->node_series) h->node_series = new alz_node_series_state();
  NodeSeriesBufs& b = h->node_series->b;
  uint64_t rows_in = 0;
  bool waited = false;
  const int rc = node_series_enqueue(h, b, q, side, tier, k, ms, false, device ? SIZE_MAX : cap, nullptr, n_out,
                                     n_points, &rows_in, &waited);
  if (rc != ALZ_OK) return rc;
  const size_t slots = *n_out * *n_points;
  if (info) {
    *info = alz_series_info{};
    info->edges = *n_out;
    info->rows_in = rows_in;
    info->points = *n_points;
    info->tier = tier;
  }
  cudaStream_t st = h->stream;
  if (device) {
    if (points) {
      if (!waited) CK(cudaStreamSynchronize(st));   // the ring's clocks
      alz_internal_ring_points(h, tier, k, points);
    }
    *dev_values = static_cast<const double*>(b.values.p);
    if (dev_present) *dev_present = static_cast<const uint8_t*>(b.present.p);
    return ALZ_OK;
  }
  if (slots && values) CK(cudaMemcpyAsync(values, b.values.p, slots * ms.nm * 8, cudaMemcpyDeviceToHost, st));
  if (slots && present) CK(cudaMemcpyAsync(present, b.present.p, slots, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));   // the host call's last wait: its results
  if (points) alz_internal_ring_points(h, tier, k, points);
  return ALZ_OK;
}

}  // namespace

uint64_t alz::metrics::entry_runs(const alz_ring_view& v, std::vector<uint32_t>* runs) {
  const uint32_t P = (uint32_t)v.n.size();
  runs->assign(2 * (size_t)P + 1, 0u);   // first[P], vbase[P + 1]
  uint64_t rows_in = 0;
  for (uint32_t j = 0; j < P; ++j) {
    (*runs)[j] = (uint32_t)v.first_row[j];   // arena rows are below 2^31
    (*runs)[P + j] = (uint32_t)rows_in;      // entries do not overlap: their rows add up to at most the arena's
    rows_in += v.n[j];
  }
  (*runs)[2 * (size_t)P] = (uint32_t)rows_in;
  return rows_in;
}

int alz::metrics::node_series_slots(alz_handle* h, NodeSeriesBufs& b, const alz_edge_out* arena, uint32_t R,
                                    uint64_t n_slots) {
  NodeGroup& g = b.g;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(g.h_words + 1, b.miss.p, 4, cudaMemcpyDeviceToHost, h->stream));   // read after the runs' wait
  int rc = node_group_runs(h, g, R, key_bits_of(n_slots));
  if (rc != ALZ_OK) return rc;
  const uint32_t misses = g.h_words[1];
  const uint32_t present = g.h_words[0] - (misses ? 1u : 0u), hits = R - misses;
  rc = reserve(h, {{&b.slot_rows, (size_t)present * sizeof(alz_node_out)}});
  if (rc != ALZ_OK) return rc;
  if (!hits) return ALZ_OK;
  rc = node_group_reduce(h, g, arena, hits, static_cast<alz_node_out*>(b.slot_rows.p));
  if (rc != ALZ_OK) return rc;
  node_slot_kernel<<<grid_for(h, hits, 8), 256, 0, h->stream>>>(static_cast<const uint64_t*>(g.keys_out.p),
                                                                static_cast<const uint32_t*>(g.heads.p),
                                                                static_cast<const uint32_t*>(g.idx.p), hits,
                                                                static_cast<uint32_t*>(b.slot.p));
  h->launches += 1;
  CK(cudaGetLastError());
  return ALZ_OK;
}

int alz::metrics::run_mapped_node_series(alz_handle* h, NodeSeriesBufs& b, bool by_source, const alz_edge_out* rows,
                                         size_t n, const alz_node_ends* keys, size_t n_keys, const GroupMap& map,
                                         uint32_t side, uint32_t tier, uint32_t k, const MetricSet& ms,
                                         bool with_rows, size_t cap, size_t* n_out, uint32_t* n_points,
                                         uint64_t* rows_in, bool* waited) {
  Nodes q;
  q.by_source = by_source;
  q.rows = rows;
  q.n_rows = n;
  q.ends = keys;
  q.n = by_source ? 0 : n_keys;
  return node_series_enqueue(h, b, q, side, tier, k, ms, with_rows, cap, &map, n_out, n_points, rows_in, waited);
}

int alz::metrics::run_node_series_rows(alz_handle* h, NodeSeriesBufs& b, const alz_edge_out* rows, size_t n,
                                       uint32_t side, uint32_t tier, uint32_t k, const MetricSet& ms, bool with_rows,
                                       size_t cap, size_t* n_out, uint32_t* n_points, uint64_t* rows_in) {
  Nodes q;
  q.by_source = true;
  q.rows = rows;
  q.n_rows = n;
  bool waited = false;
  return node_series_enqueue(h, b, q, side, tier, k, ms, with_rows, cap, nullptr, n_out, n_points, rows_in, &waited);
}

extern "C" int alz_node_series(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                               const alz_metric* m, uint32_t nm, double* values, uint8_t* present, size_t cap,
                               size_t* n_out, uint32_t* n_points, alz_rollup_info* points, alz_series_info* info) {
  return series_entry(h, true, source, nullptr, 0, side, tier, k, m, nm, false, values, present, cap, nullptr, nullptr,
                      n_out, n_points, points, info);
}

extern "C" int alz_node_series_device(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                      const alz_metric* m, uint32_t nm, const double** dev_values,
                                      const uint8_t** dev_present, size_t* n_out, uint32_t* n_points,
                                      alz_rollup_info* points, alz_series_info* info) {
  return series_entry(h, true, source, nullptr, 0, side, tier, k, m, nm, true, nullptr, nullptr, 0, dev_values,
                      dev_present, n_out, n_points, points, info);
}

extern "C" int alz_node_series_keys(alz_handle* h, const alz_node_ends* keys, size_t n_keys, uint32_t side,
                                    uint32_t tier, uint32_t k, const alz_metric* m, uint32_t nm, double* values,
                                    uint8_t* present, size_t cap, size_t* n_out, uint32_t* n_points,
                                    alz_rollup_info* points, alz_series_info* info) {
  return series_entry(h, false, 0, keys, n_keys, side, tier, k, m, nm, false, values, present, cap, nullptr, nullptr,
                      n_out, n_points, points, info);
}

extern "C" int alz_node_series_keys_device(alz_handle* h, const alz_node_ends* keys, size_t n_keys, uint32_t side,
                                           uint32_t tier, uint32_t k, const alz_metric* m, uint32_t nm,
                                           const double** dev_values, const uint8_t** dev_present, size_t* n_out,
                                           uint32_t* n_points, alz_rollup_info* points, alz_series_info* info) {
  return series_entry(h, false, 0, keys, n_keys, side, tier, k, m, nm, true, nullptr, nullptr, 0, dev_values,
                      dev_present, n_out, n_points, points, info);
}
