// alz_series.cu — edge series (docs/SPEC.md §19): the §17 metric values of a source's rows, or of edges the caller
// names, in each of the last P closed entries of one ring (the window history or a tier), oldest first.
//
// Every entry is a run of rows of the ring's arena in ascending packed-key order, and the query keys are sorted and
// distinct, so the series needs no sort (DESIGN.md §5.11):
//   keys    a source's rows' packed keys (16 of 296 bytes read per row); caller keys are packed, sorted and made
//           distinct on the host, with a map from each caller row to its distinct key
//   match   one thread per row of the P entries, numbered in one virtual row space (entry j takes [vbase[j],
//           vbase[j + 1])): its packed key, a lower bound into the query keys, and on a hit its arena row into
//           slot[u * P + j]. slot starts as kSlotAbsent everywhere. O(rows read), no atomics.
//   values  the §17 metric kernels of alz_metrics.cu over the slots (SeriesRows): an absent slot gives +0.0 and
//           present 0, a present one exactly the values alz_edge_metrics* gives for its row
// The device call waits once, for the ring's clocks, before it launches anything; the host call once, for its results.
#include <algorithm>
#include <mutex>
#include <string>
#include <vector>

#include "alz_metrics.cuh"

using namespace alz;
using namespace alz::metrics;

namespace {

// Thread t: row t of the entries' virtual row space, entry j holding arena rows [first[j], first[j] + vbase[j + 1] -
// vbase[j]); n_rows = vbase[points]
__global__ void __launch_bounds__(256) series_match_kernel(const alz_edge_out* __restrict__ arena,
                                                           const uint32_t* __restrict__ first,
                                                           const uint32_t* __restrict__ vbase, uint32_t points,
                                                           uint32_t n_rows, const uint64_t* __restrict__ keys,
                                                           uint32_t n_keys, uint32_t* __restrict__ slot) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n_rows; t += stride) {
    uint32_t lo = 0, hi = points;   // the last entry j with vbase[j] <= t (an empty entry is passed over)
    while (hi - lo > 1u) {
      const uint32_t mid = (lo + hi) >> 1;
      if (vbase[mid] <= t) lo = mid; else hi = mid;
    }
    const uint32_t row = first[lo] + (t - vbase[lo]);
    const uint64_t key = row_key_of(arena + row);
    const uint32_t u = lower_bound_u64(keys, n_keys, key);
    if (u < n_keys && keys[u] == key) slot[u * points + lo] = row;
  }
}

}  // namespace

// Buffers of the series calls, each grown on demand and never shrunk; freed in alz_destroy
struct alz_series_state {
  SeriesBufs b;
};

void alz::metrics::SeriesBufs::free() { free_bufs({&keys, &map, &runs, &slot, &values, &present}); }

void alz_internal_free_series(alz_handle* h) {
  alz_series_state* s = h->series;
  if (!s) return;
  s->b.free();
  delete s;
  h->series = nullptr;
}

namespace {

// The edges of a series: a source's rows (rows, n) or the caller's keys, packed, as distinct sorted keys and a map
struct Edges {
  bool by_source = false;
  const alz_edge_out* rows = nullptr;    // source rows
  const alz_edge_ends* ends = nullptr;   // caller keys
  size_t n = 0;                          // series rows
  std::vector<uint64_t> keys;            // caller keys: the distinct packed keys
  std::vector<uint32_t> map;             // caller row -> index into keys
};

// e->keys and e->map from the caller's keys; false for a malformed key
bool caller_edges(Edges* e) {
  std::vector<uint64_t> packed(e->n);
  for (size_t i = 0; i < e->n; ++i)
    if (!pack_edge_ends(e->ends[i], &packed[i])) return false;
  e->keys = packed;
  std::sort(e->keys.begin(), e->keys.end());
  e->keys.erase(std::unique(e->keys.begin(), e->keys.end()), e->keys.end());
  e->map.resize(e->n);
  for (size_t i = 0; i < e->n; ++i)
    e->map[i] = (uint32_t)(std::lower_bound(e->keys.begin(), e->keys.end(), packed[i]) - e->keys.begin());
  return true;
}

// The series of `edges` over the last min(k, retained) entries of tier `tier` into b, on the stream: *n_out series
// rows, *n_points = P, *rows_in entry rows read. n_out > cap: ALZ_E_CAPACITY before anything is enqueued. wait_first:
// one wait once the buffers are in place, before the first launch (the series device call's wait for the ring's
// clocks); otherwise no wait of its own. Caller holds h->mu and has set the device.
int series_enqueue(alz_handle* h, SeriesBufs& b, Edges& edges, uint32_t tier, uint32_t k, const MetricSet& ms,
                   size_t cap, bool wait_first, size_t* n_out, uint32_t* n_points, uint64_t* rows_in_out) {
  int rc = alz_internal_ring_view(h, tier, k, &b.view);
  if (rc != ALZ_OK) return rc;
  const alz_ring_view& v = b.view;
  const uint32_t P = (uint32_t)v.n.size();
  const size_t n = edges.n;
  *n_out = n;
  *n_points = P;
  if ((uint64_t)n * P > kMaxRows) return ALZ_E_CAPACITY;
  if (n > cap) return ALZ_E_CAPACITY;
  const bool by_source = edges.by_source;
  if (!by_source && !caller_edges(&edges)) return ALZ_E_INVAL;   // packed once the sizes are known to fit
  const size_t n_keys = by_source ? n : edges.keys.size();
  const size_t slots = (size_t)n * P;
  uint64_t rows_in = 0;
  std::vector<uint32_t> runs(2 * (size_t)P + 1);   // first[P], vbase[P + 1]
  for (uint32_t j = 0; j < P; ++j) {
    runs[j] = (uint32_t)v.first_row[j];   // arena rows are below 2^31
    runs[P + j] = (uint32_t)rows_in;      // entries do not overlap: their rows add up to at most the arena's
    rows_in += v.n[j];
  }
  runs[2 * (size_t)P] = (uint32_t)rows_in;
  *rows_in_out = rows_in;
  rc = reserve(h, {{&b.keys, std::max<size_t>(n_keys, 1) * 8},
                   {&b.map, by_source ? 0 : std::max<size_t>(n, 1) * 4},
                   {&b.runs, runs.size() * 4},
                   {&b.slot, std::max<size_t>(n_keys * P, 1) * 4},
                   {&b.values, std::max<size_t>(slots * ms.nm, 1) * 8},
                   {&b.present, std::max<size_t>(slots, 1)}});
  if (rc != ALZ_OK) return rc;
  cudaStream_t st = h->stream;
  if (wait_first) CK(cudaStreamSynchronize(st));   // the one wait: the ring's clocks
  uint64_t* d_keys = static_cast<uint64_t*>(b.keys.p);
  uint32_t* d_runs = static_cast<uint32_t*>(b.runs.p);
  uint32_t* d_slot = static_cast<uint32_t*>(b.slot.p);
  if (!slots) return ALZ_OK;
  if (by_source) {
    launch_row_keys(h, edges.rows, (uint32_t)n, d_keys);
  } else {
    CK(cudaMemcpyAsync(d_keys, edges.keys.data(), n_keys * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(b.map.p, edges.map.data(), n * 4, cudaMemcpyHostToDevice, st));
  }
  CK(cudaMemcpyAsync(d_runs, runs.data(), runs.size() * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(d_slot, 0xFF, n_keys * P * 4, st));
  if (rows_in) {
    const unsigned grid = (unsigned)std::min<uint64_t>((rows_in + 255) / 256, (uint64_t)h->sms * 8);
    series_match_kernel<<<grid, 256, 0, st>>>(v.arena, d_runs, d_runs + P, P, (uint32_t)rows_in, d_keys,
                                              (uint32_t)n_keys, d_slot);
    h->launches += 1;
  }
  const SeriesRows sr{v.arena, d_slot, by_source ? nullptr : static_cast<const uint32_t*>(b.map.p), P,
                      static_cast<uint8_t*>(b.present.p)};
  return run_metrics_series(h, sr, (uint32_t)slots, ms, static_cast<double*>(b.values.p));
}

// The series of `edges` over the last min(k, retained) entries of tier `tier`. Device call: *dev_values /
// *dev_present; host call: cap series rows into values / present (either may be null when nothing is copied).
// Caller holds h->mu.
int series_locked(alz_handle* h, Edges& edges, uint32_t tier, uint32_t k, const MetricSet& ms, bool device,
                  double* values, uint8_t* present, size_t cap, const double** dev_values,
                  const uint8_t** dev_present, size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                  alz_series_info* info) {
  CK(cudaSetDevice(h->device));
  if (!h->series) h->series = new alz_series_state();
  SeriesBufs& b = h->series->b;
  uint64_t rows_in = 0;
  const int rc = series_enqueue(h, b, edges, tier, k, ms, device ? SIZE_MAX : cap, device, n_out, n_points, &rows_in);
  if (rc != ALZ_OK) return rc;
  const size_t slots = *n_out * *n_points;
  if (info) {
    *info = alz_series_info{};
    info->edges = *n_out;
    info->rows_in = rows_in;
    info->points = *n_points;
    info->tier = tier;
  }
  if (device) {
    if (points) alz_internal_ring_points(h, tier, k, points);   // the clocks arrived before the first launch
    *dev_values = static_cast<const double*>(b.values.p);
    if (dev_present) *dev_present = static_cast<const uint8_t*>(b.present.p);
    return ALZ_OK;
  }
  cudaStream_t st = h->stream;
  if (slots && values) CK(cudaMemcpyAsync(values, b.values.p, slots * ms.nm * 8, cudaMemcpyDeviceToHost, st));
  if (slots && present) CK(cudaMemcpyAsync(present, b.present.p, slots, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));   // the one wait of a host call: the results and the ring's clocks
  if (points) alz_internal_ring_points(h, tier, k, points);
  return ALZ_OK;
}

// The four entry points. by_source: the rows of `source`; else the caller's keys.
int series_entry(alz_handle* h, bool by_source, uint32_t source, const alz_edge_ends* keys, size_t n_keys,
                 uint32_t tier, uint32_t k, const alz_metric* m, uint32_t nm, bool device, double* values,
                 uint8_t* present, size_t cap, const double** dev_values, const uint8_t** dev_present, size_t* n_out,
                 uint32_t* n_points, alz_rollup_info* points, alz_series_info* info) {
  if (!h || !n_out || !n_points) {
    if (n_out) *n_out = 0;
    if (n_points) *n_points = 0;
    return ALZ_E_INVAL;
  }
  *n_out = 0;
  *n_points = 0;
  MetricSet ms;
  if (k == 0 || !valid_metrics(m, nm, &ms)) return ALZ_E_INVAL;
  if (device ? !dev_values : (!values && cap)) return ALZ_E_INVAL;
  Edges edges;
  if (by_source) {
    if (source != ALZ_SOURCE_WINDOW && source > ALZ_ROLLUP_SPAN) return ALZ_E_INVAL;
  } else {
    if (!keys && n_keys) return ALZ_E_INVAL;
    edges.ends = keys;
    edges.n = n_keys;
  }
  std::lock_guard<std::mutex> g(h->mu);
  if (by_source) {
    edges.by_source = true;
    if (source == ALZ_SOURCE_WINDOW) {
      edges.rows = h->d_out;
      edges.n = h->last_n_edges;
    } else {
      const int rc = alz_internal_rollup_rows(h, source, &edges.rows, &edges.n);
      if (rc != ALZ_OK) return rc;
    }
    if (edges.n > kMaxRows) return ALZ_E_CAPACITY;
  }
  return series_locked(h, edges, tier, k, ms, device, values, present, cap, dev_values, dev_present, n_out, n_points,
                       points, info);
}

}  // namespace

int alz::metrics::run_series_rows(alz_handle* h, SeriesBufs& b, const alz_edge_out* rows, size_t n, uint32_t tier,
                                  uint32_t k, const MetricSet& ms, size_t cap, size_t* n_out, uint32_t* n_points,
                                  uint64_t* rows_in) {
  Edges edges;
  edges.by_source = true;
  edges.rows = rows;
  edges.n = n;
  return series_enqueue(h, b, edges, tier, k, ms, cap, false, n_out, n_points, rows_in);
}

extern "C" int alz_edge_series(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                               uint32_t nm, double* values, uint8_t* present, size_t cap, size_t* n_out,
                               uint32_t* n_points, alz_rollup_info* points, alz_series_info* info) {
  return series_entry(h, true, source, nullptr, 0, tier, k, m, nm, false, values, present, cap, nullptr, nullptr,
                      n_out, n_points, points, info);
}

extern "C" int alz_edge_series_device(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                                      uint32_t nm, const double** dev_values, const uint8_t** dev_present,
                                      size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                                      alz_series_info* info) {
  return series_entry(h, true, source, nullptr, 0, tier, k, m, nm, true, nullptr, nullptr, 0, dev_values, dev_present,
                      n_out, n_points, points, info);
}

extern "C" int alz_edge_series_keys(alz_handle* h, const alz_edge_ends* keys, size_t n_keys, uint32_t tier, uint32_t k,
                                    const alz_metric* m, uint32_t nm, double* values, uint8_t* present, size_t cap,
                                    size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                                    alz_series_info* info) {
  return series_entry(h, false, 0, keys, n_keys, tier, k, m, nm, false, values, present, cap, nullptr, nullptr, n_out,
                      n_points, points, info);
}

extern "C" int alz_edge_series_keys_device(alz_handle* h, const alz_edge_ends* keys, size_t n_keys, uint32_t tier,
                                           uint32_t k, const alz_metric* m, uint32_t nm, const double** dev_values,
                                           const uint8_t** dev_present, size_t* n_out, uint32_t* n_points,
                                           alz_rollup_info* points, alz_series_info* info) {
  return series_entry(h, false, 0, keys, n_keys, tier, k, m, nm, true, nullptr, nullptr, 0, dev_values, dev_present,
                      n_out, n_points, points, info);
}
