// alz_group_series.cu — group series (docs/SPEC.md §26): the §17 metric values of a source's group edges or of one side
// of its group nodes (§24, under the map in force at the call), or of group edges or nodes the caller names, in each
// of the last P closed entries of one ring, oldest first. Point j of a group sums every row of entry j that maps onto
// it, so, as a node series (§22), it is a group-by of the entries' rows keyed by (series row, point) (DESIGN.md §5.18):
//   keys    by source: the §24 group-by of the source's rows into this state's group-edge rows (alz_groups.cu, two
//           waits); group edges are keyed by their 16-byte (from key, to key), already ascending, group nodes by the
//           node keys of those rows' ends (the §22 source path over them). Caller keys are checked first, then packed,
//           sorted and made distinct on the host, with a map from each caller row to its distinct key.
//   pairs   group nodes: §22's pairs kernel with the row's end passed through the map first. Group edges: one thread
//           per entry row maps both ends, looks the (from key, to key) pair up among the query keys and writes the
//           pair (u x P + j, 2 x arena row + IN), a miss keyed N x P, as §22 does.
//   group   §22's slot group-by (node_series_slots: sort, one wait, reduce, slots). A group edge's sums land on the IN
//           side of its slot row, laid out as alz_edge_out from count on, so the §17 kernels read them as a row.
//   values  the §17 metric kernels over the slots (NodeSeriesRows)
// Reads the source rows, the ring and the map only: every buffer written is this state's or the group calls' scratch.
#include <algorithm>
#include <mutex>
#include <string>
#include <vector>

#include "alz_metrics.cuh"

using namespace alz;
using namespace alz::metrics;

namespace {

// A group edge's key: the node keys of its from and to ends, compared in that order (§25)
struct EndsKey {
  uint64_t from, to;
};
bool operator<(const EndsKey& x, const EndsKey& y) { return x.from < y.from || (x.from == y.from && x.to < y.to); }
bool operator==(const EndsKey& x, const EndsKey& y) { return x.from == y.from && x.to == y.to; }

// keys[i] = group-edge row i's (from key, to key)
__global__ void __launch_bounds__(256) group_edge_ends_kernel(const alz_edge_out* __restrict__ rows, uint32_t n,
                                                              ulonglong2* __restrict__ keys) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint2 ty = reinterpret_cast<const uint2*>(rows + i)[0], ft = reinterpret_cast<const uint2*>(rows + i)[1];
    keys[i] = make_ulonglong2(node_key(ty.x & 0xFFu, ft.x), node_key((ty.x >> 8) & 0xFFu, ft.y));
  }
}

// Thread t: row t of the entries' virtual row space (as node_series_pairs_kernel): both ends mapped, the lower bound of
// (from key, to key) among the n_keys ascending query keys, and the pair (u x P + j, 2 x row + IN), or N x P on a
// miss; a warp-reduced count of the misses
__global__ void __launch_bounds__(256) group_edge_pairs_kernel(const alz_edge_out* __restrict__ arena,
                                                               const uint32_t* __restrict__ first,
                                                               const uint32_t* __restrict__ vbase, uint32_t points,
                                                               uint32_t n_rows, const ulonglong2* __restrict__ keys,
                                                               uint32_t n_keys, const uint64_t* __restrict__ mk,
                                                               const uint32_t* __restrict__ mg, uint32_t m,
                                                               uint64_t* __restrict__ pair_keys,
                                                               uint32_t* __restrict__ pair_vals,
                                                               uint32_t* __restrict__ misses) {
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
    const uint64_t kf = map_end(node_key(ty.x & 0xFFu, ft.x), mk, mg, m);
    const uint64_t kt = map_end(node_key((ty.x >> 8) & 0xFFu, ft.y), mk, mg, m);
    uint32_t a = 0, b = n_keys;
    while (a < b) {
      const uint32_t mid = (a + b) >> 1;
      const ulonglong2 q = keys[mid];
      if (q.x < kf || (q.x == kf && q.y < kt)) a = mid + 1; else b = mid;
    }
    bool hit = false;
    if (a < n_keys) {
      const ulonglong2 q = keys[a];
      hit = q.x == kf && q.y == kt;
    }
    pair_keys[t] = hit ? (uint64_t)a * points + lo : miss_key;
    pair_vals[t] = 2u * row + ALZ_SIDE_IN;   // arena rows are below 2^31
    n_miss += hit ? 0u : 1u;
  }
  n_miss = __reduce_add_sync(0xFFFFFFFFu, n_miss);   // every lane of the warp leaves the loop to get here
  if ((threadIdx.x & 31u) == 0 && n_miss) atomicAdd(misses, n_miss);
}

}  // namespace

void alz::metrics::GroupSeriesBufs::free() {
  s.free();
  free_bufs({&edges});
}

// Buffers of the group series calls, each grown on demand and never shrunk; freed in alz_destroy
struct alz_group_series_state {
  GroupSeriesBufs b;
};

void alz_internal_free_group_series(alz_handle* h) {
  alz_group_series_state* s = h->group_series;
  if (!s) return;
  s->b.free();
  delete s;
  h->group_series = nullptr;
}

namespace {

// a node key of §26: one §22 accepts, or a group below 2^29
bool valid_group_node(uint32_t type, uint32_t value) { return valid_group_node_key(type, value); }

// a group-edge key of §26: §19's rules when neither end is a group, else two valid node keys
bool valid_group_edge(const alz_edge_ends& e) {
  if (e.from_type != ALZ_NODE_GROUP && e.to_type != ALZ_NODE_GROUP) {
    uint64_t key;
    return pack_edge_ends(e, &key);
  }
  return valid_group_node(e.from_type, e.from) && valid_group_node(e.to_type, e.to);
}

// The group edge series of the n_edges rows in b.edges (by_source) or of the caller's n keys over the last min(k,
// retained) entries of tier `tier` into b.s, on the stream: *n_out series rows, *n_points = P, *rows_in entry rows
// read, *waited when it waited after the ring's clocks were enqueued. Series rows > cap: ALZ_E_CAPACITY before the
// entries are read. Caller holds h->mu and has set the device.
int group_edge_series(alz_handle* h, GroupSeriesBufs& gb, bool by_source, size_t n_edges, const alz_edge_ends* ends,
                      size_t n_ends, uint32_t tier, uint32_t k, const MetricSet& ms, size_t cap, size_t* n_out,
                      uint32_t* n_points, uint64_t* rows_in_out, bool* waited) {
  *waited = false;
  NodeSeriesBufs& b = gb.s;
  int rc = alz_internal_ring_view(h, tier, k, &b.view);
  if (rc != ALZ_OK) return rc;
  const alz_ring_view& v = b.view;
  const uint32_t P = (uint32_t)v.n.size();
  *n_points = P;
  const size_t n = by_source ? n_edges : n_ends;
  *n_out = n;
  if ((uint64_t)n * P > kMaxRows) return ALZ_E_CAPACITY;
  if (n > cap) return ALZ_E_CAPACITY;
  std::vector<EndsKey> keys;   // caller keys: distinct and ascending, and each caller row's index among them
  std::vector<uint32_t> map;
  if (!by_source) {
    std::vector<EndsKey> packed(n);
    for (size_t i = 0; i < n; ++i)
      packed[i] = EndsKey{((uint64_t)ends[i].from_type << 32) | ends[i].from, ((uint64_t)ends[i].to_type << 32) | ends[i].to};
    keys = packed;
    std::sort(keys.begin(), keys.end());
    keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
    map.resize(n);
    for (size_t i = 0; i < n; ++i)
      map[i] = (uint32_t)(std::lower_bound(keys.begin(), keys.end(), packed[i]) - keys.begin());
  }
  const size_t n_keys = by_source ? n : keys.size();
  const size_t slots = n * P;
  std::vector<uint32_t> runs;
  const uint64_t rows_in = entry_runs(v, &runs);
  *rows_in_out = rows_in;
  rc = reserve(h, {{&b.keys, std::max<size_t>(n_keys, 1) * sizeof(ulonglong2)},
                   {&b.map, by_source ? 0 : std::max<size_t>(n, 1) * 4},
                   {&b.runs, runs.size() * 4},
                   {&b.slot, std::max<size_t>(n_keys * P, 1) * 4},
                   {&b.miss, 4},
                   {&b.values, std::max<size_t>(slots * ms.nm, 1) * 8},
                   {&b.present, std::max<size_t>(slots, 1)}});
  if (rc != ALZ_OK) return rc;
  cudaStream_t st = h->stream;
  ulonglong2* d_keys = static_cast<ulonglong2*>(b.keys.p);
  if (!slots) return ALZ_OK;
  if (by_source) {
    group_edge_ends_kernel<<<grid_for(h, n, 8), 256, 0, st>>>(static_cast<const alz_edge_out*>(gb.edges.p),
                                                              (uint32_t)n, d_keys);
    h->launches += 1;
    CK(cudaGetLastError());
  } else {
    static_assert(sizeof(EndsKey) == sizeof(ulonglong2), "a key is copied as (from key, to key)");
    CK(cudaMemcpyAsync(d_keys, keys.data(), n_keys * sizeof(EndsKey), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(b.map.p, map.data(), n * 4, cudaMemcpyHostToDevice, st));
  }
  uint32_t* d_runs = static_cast<uint32_t*>(b.runs.p);
  uint32_t* d_slot = static_cast<uint32_t*>(b.slot.p);
  CK(cudaMemcpyAsync(d_runs, runs.data(), runs.size() * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(d_slot, 0xFF, n_keys * P * 4, st));
  if (rows_in) {   // the entries' (slot, row) pairs, grouped by slot: one wait
    const uint32_t R = (uint32_t)rows_in;
    rc = node_group_reserve(h, b.g, R);
    if (rc != ALZ_OK) return rc;
    CK(cudaMemsetAsync(b.miss.p, 0, 4, st));
    const GroupMap gm = group_map(h);
    group_edge_pairs_kernel<<<grid_for(h, R, 8), 256, 0, st>>>(
        v.arena, d_runs, d_runs + P, P, R, d_keys, (uint32_t)n_keys, gm.keys, gm.groups, gm.n,
        static_cast<uint64_t*>(b.g.keys_in.p), static_cast<uint32_t*>(b.g.vals_in.p),
        static_cast<uint32_t*>(b.miss.p));
    h->launches += 1;
    rc = node_series_slots(h, b, v.arena, R, (uint64_t)n_keys * P);
    if (rc != ALZ_OK) return rc;
    *waited = true;
  }
  const NodeSeriesRows sr{static_cast<const alz_node_out*>(b.slot_rows.p), d_slot,
                          by_source ? nullptr : static_cast<const uint32_t*>(b.map.p), P, ALZ_SIDE_IN,
                          static_cast<uint8_t*>(b.present.p)};
  return run_metrics_node_series(h, sr, (uint32_t)slots, ms, static_cast<double*>(b.values.p));
}

// The series of a source's group edges or group nodes into b, as run_group_series_rows, with *waited
int source_series(alz_handle* h, GroupSeriesBufs& b, const alz_edge_out* rows, size_t n, bool nodes, uint32_t side,
                  uint32_t tier, uint32_t k, const MetricSet& ms, bool with_rows, size_t cap, size_t* n_out,
                  uint32_t* n_points, uint64_t* rows_in, bool* waited) {
  *waited = false;
  *n_out = 0;
  *n_points = 0;
  // A tier the ring view refuses is refused before the source is grouped. The series below takes its own view after
  // the grouping's waits: a view enqueues the copy of the ring's clocks, which the series' own waits then bring.
  int rc = alz_internal_ring_view(h, tier, k, &b.s.view);
  if (rc != ALZ_OK) return rc;
  size_t n_edges = 0;
  alz_group_info gi;
  rc = group_edges_into(h, b.edges, rows, n, SIZE_MAX, &n_edges, &gi);
  if (rc != ALZ_OK) return rc;
  if (!nodes)
    return group_edge_series(h, b, true, n_edges, nullptr, 0, tier, k, ms, cap, n_out, n_points, rows_in, waited);
  return run_mapped_node_series(h, b.s, true, static_cast<const alz_edge_out*>(b.edges.p), n_edges, nullptr, 0,
                                group_map(h), side, tier, k, ms, with_rows, cap, n_out, n_points, rows_in, waited);
}

// The eight entry points. nodes: group nodes on `side`, else group edges; by_source: those of `source`, else the
// caller's edge_keys / node_keys. Device call: *dev_values / *dev_present; host call: cap series rows into values /
// present (either may be null when nothing is copied).
int series_entry(alz_handle* h, bool nodes, bool by_source, uint32_t source, const alz_edge_ends* edge_keys,
                 const alz_node_ends* node_keys, size_t n_keys, uint32_t side, uint32_t tier, uint32_t k,
                 const alz_metric* m, uint32_t nm, bool device, double* values, uint8_t* present, size_t cap,
                 const double** dev_values, const uint8_t** dev_present, size_t* n_out, uint32_t* n_points,
                 alz_rollup_info* points, alz_series_info* info) {
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
  if (by_source) {
    if (source != ALZ_SOURCE_WINDOW && source > ALZ_ROLLUP_SPAN) return ALZ_E_INVAL;
  } else {
    if (nodes ? (!node_keys && n_keys) : (!edge_keys && n_keys)) return ALZ_E_INVAL;
    for (size_t i = 0; i < n_keys; ++i)   // a malformed key is refused whatever the sizes
      if (nodes ? !valid_group_node(node_keys[i].type, node_keys[i].value) : !valid_group_edge(edge_keys[i]))
        return ALZ_E_INVAL;
  }
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  const alz_edge_out* rows = nullptr;
  size_t n_rows = 0;
  if (by_source) {
    const int rc = node_source(h, source, &rows, &n_rows);   // more than 2^29 - 1 rows: ALZ_E_CAPACITY
    if (rc != ALZ_OK) return rc;
  }
  if (!h->group_series) h->group_series = new alz_group_series_state();
  GroupSeriesBufs& b = h->group_series->b;
  const size_t room = device ? SIZE_MAX : cap;
  uint64_t rows_in = 0;
  bool waited = false;
  int rc;
  if (by_source)
    rc = source_series(h, b, rows, n_rows, nodes, side, tier, k, ms, false, room, n_out, n_points, &rows_in, &waited);
  else if (nodes)
    rc = run_mapped_node_series(h, b.s, false, nullptr, 0, node_keys, n_keys, group_map(h), side, tier, k, ms, false,
                                room, n_out, n_points, &rows_in, &waited);
  else
    rc = group_edge_series(h, b, false, 0, edge_keys, n_keys, tier, k, ms, room, n_out, n_points, &rows_in, &waited);
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
    *dev_values = static_cast<const double*>(b.s.values.p);
    if (dev_present) *dev_present = static_cast<const uint8_t*>(b.s.present.p);
    return ALZ_OK;
  }
  if (slots && values) CK(cudaMemcpyAsync(values, b.s.values.p, slots * ms.nm * 8, cudaMemcpyDeviceToHost, st));
  if (slots && present) CK(cudaMemcpyAsync(present, b.s.present.p, slots, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));   // the host call's last wait: its results
  if (points) alz_internal_ring_points(h, tier, k, points);
  return ALZ_OK;
}

}  // namespace

int alz::metrics::run_group_series_rows(alz_handle* h, GroupSeriesBufs& b, const alz_edge_out* rows, size_t n,
                                        bool nodes, uint32_t side, uint32_t tier, uint32_t k, const MetricSet& ms,
                                        bool with_rows, size_t cap, size_t* n_out, uint32_t* n_points,
                                        uint64_t* rows_in) {
  bool waited = false;
  return source_series(h, b, rows, n, nodes, side, tier, k, ms, with_rows, cap, n_out, n_points, rows_in, &waited);
}

extern "C" int alz_group_edge_series(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                                     uint32_t nm, double* values, uint8_t* present, size_t cap, size_t* n_out,
                                     uint32_t* n_points, alz_rollup_info* points, alz_series_info* info) {
  return series_entry(h, false, true, source, nullptr, nullptr, 0, ALZ_SIDE_IN, tier, k, m, nm, false, values, present,
                      cap, nullptr, nullptr, n_out, n_points, points, info);
}

extern "C" int alz_group_edge_series_device(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k,
                                            const alz_metric* m, uint32_t nm, const double** dev_values,
                                            const uint8_t** dev_present, size_t* n_out, uint32_t* n_points,
                                            alz_rollup_info* points, alz_series_info* info) {
  return series_entry(h, false, true, source, nullptr, nullptr, 0, ALZ_SIDE_IN, tier, k, m, nm, true, nullptr, nullptr,
                      0, dev_values, dev_present, n_out, n_points, points, info);
}

extern "C" int alz_group_edge_series_keys(alz_handle* h, const alz_edge_ends* keys, size_t n_keys, uint32_t tier,
                                          uint32_t k, const alz_metric* m, uint32_t nm, double* values,
                                          uint8_t* present, size_t cap, size_t* n_out, uint32_t* n_points,
                                          alz_rollup_info* points, alz_series_info* info) {
  return series_entry(h, false, false, 0, keys, nullptr, n_keys, ALZ_SIDE_IN, tier, k, m, nm, false, values, present,
                      cap, nullptr, nullptr, n_out, n_points, points, info);
}

extern "C" int alz_group_edge_series_keys_device(alz_handle* h, const alz_edge_ends* keys, size_t n_keys,
                                                 uint32_t tier, uint32_t k, const alz_metric* m, uint32_t nm,
                                                 const double** dev_values, const uint8_t** dev_present,
                                                 size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                                                 alz_series_info* info) {
  return series_entry(h, false, false, 0, keys, nullptr, n_keys, ALZ_SIDE_IN, tier, k, m, nm, true, nullptr, nullptr,
                      0, dev_values, dev_present, n_out, n_points, points, info);
}

extern "C" int alz_group_node_series(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                     const alz_metric* m, uint32_t nm, double* values, uint8_t* present, size_t cap,
                                     size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                                     alz_series_info* info) {
  return series_entry(h, true, true, source, nullptr, nullptr, 0, side, tier, k, m, nm, false, values, present, cap,
                      nullptr, nullptr, n_out, n_points, points, info);
}

extern "C" int alz_group_node_series_device(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                            const alz_metric* m, uint32_t nm, const double** dev_values,
                                            const uint8_t** dev_present, size_t* n_out, uint32_t* n_points,
                                            alz_rollup_info* points, alz_series_info* info) {
  return series_entry(h, true, true, source, nullptr, nullptr, 0, side, tier, k, m, nm, true, nullptr, nullptr, 0,
                      dev_values, dev_present, n_out, n_points, points, info);
}

extern "C" int alz_group_node_series_keys(alz_handle* h, const alz_node_ends* keys, size_t n_keys, uint32_t side,
                                          uint32_t tier, uint32_t k, const alz_metric* m, uint32_t nm, double* values,
                                          uint8_t* present, size_t cap, size_t* n_out, uint32_t* n_points,
                                          alz_rollup_info* points, alz_series_info* info) {
  return series_entry(h, true, false, 0, nullptr, keys, n_keys, side, tier, k, m, nm, false, values, present, cap,
                      nullptr, nullptr, n_out, n_points, points, info);
}

extern "C" int alz_group_node_series_keys_device(alz_handle* h, const alz_node_ends* keys, size_t n_keys,
                                                 uint32_t side, uint32_t tier, uint32_t k, const alz_metric* m,
                                                 uint32_t nm, const double** dev_values, const uint8_t** dev_present,
                                                 size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                                                 alz_series_info* info) {
  return series_entry(h, true, false, 0, nullptr, keys, n_keys, side, tier, k, m, nm, true, nullptr, nullptr, 0,
                      dev_values, dev_present, n_out, n_points, points, info);
}
