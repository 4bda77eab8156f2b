// alz_changes.cu — edge changes against a pinned baseline (docs/SPEC.md §18): a copy of a window's or rollup's rows
// kept on the handle, and the change list of a source against it: one sorted join of two row lists, each side's §17
// metric values and one record per row of the filtered union, or only its top rows by change.
//
// Both sides are strictly ascending by packed key (§3, §12), so the join needs no sort (DESIGN.md §5.10):
//   keys    the source rows' packed keys (the baseline's were stored when it was pinned)
//   match   every row of either side: lower_bound into the other side's keys, whether the key is there, and whether
//           the row is kept by the presence filter (a source row: BOTH or NEW; a baseline row: GONE when unmatched,
//           else it is listed through its source row)
//   scan    two exclusive scans of the keep flags. A kept source row i goes to scanA[i] + scanG[lb_B(key_i)], a
//           kept gone baseline row j to scanA[lb_A(key_j)] + scanG[j]: the tier merge's arithmetic (alz_rollup.cu)
//   values  the §17 metric kernel over each side's rows
//   emit    one 48-byte record per listed row, and for the top call its change into an 8-byte array, which the §17
//           selection ranks; the selected records are gathered by position
// One host wait per call reads the union's counts; the top call's selection adds its own (alz_top.cu). The node
// changes (alz_node_changes.cu) read the baseline through pinned_baseline and share change_of, the gather and the
// list-or-top tail; the group changes (alz_group_changes.cu) run this join on (from node key, to node key) keys, the
// 16-byte instantiation of the keys and match kernels, into buffers of their own.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <mutex>
#include <string>
#include <tuple>

#include "alz_metrics.cuh"

using namespace alz;
using namespace alz::metrics;

static_assert(sizeof(alz_edge_change) == 48, "alz_edge_change is three 16-byte stores");

namespace {

constexpr uint32_t kAbsent = 0xFFFFFFFFu;
constexpr uint32_t kMatched = 0x80000000u;   // in a lower bound: the other side holds the key (bounds are < 2^30)

// A group-edge row's join key (docs/SPEC.md §25): the node keys of its from and to ends, compared in that order. A
// pair of ends needs 70 bits (a 3-bit type and any 32-bit value each), so it does not pack into one word.
struct __align__(16) EndsKey {
  uint64_t from, to;
};
__device__ __forceinline__ bool operator==(const EndsKey& x, const EndsKey& y) { return x.from == y.from && x.to == y.to; }
__device__ __forceinline__ bool operator<(const EndsKey& x, const EndsKey& y) {
  return x.from < y.from || (x.from == y.from && x.to < y.to);
}

// a row's key: its packed key (§3), or its ends (from the 16-byte head: types, pad | from, to)
template <class Key> __device__ __forceinline__ Key key_of(const alz_edge_out* r);
template <> __device__ __forceinline__ uint64_t key_of<uint64_t>(const alz_edge_out* r) { return row_key_of(r); }
template <> __device__ __forceinline__ EndsKey key_of<EndsKey>(const alz_edge_out* r) {
  const uint2 ty = reinterpret_cast<const uint2*>(r)[0], ft = reinterpret_cast<const uint2*>(r)[1];
  return EndsKey{node_key(ty.x & 0xFFu, ft.x), node_key((ty.x >> 8) & 0xFFu, ft.y)};
}

__device__ __forceinline__ uint32_t lower_bound_key(const uint64_t* __restrict__ a, uint32_t n, uint64_t k) {
  return lower_bound_u64(a, n, k);
}
__device__ __forceinline__ uint32_t lower_bound_key(const EndsKey* __restrict__ a, uint32_t n, EndsKey k) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (a[mid] < k) lo = mid + 1; else hi = mid; }
  return lo;
}

// the rows' keys
template <class Key>
__global__ void __launch_bounds__(256) change_keys_kernel(const alz_edge_out* __restrict__ rows, uint32_t n,
                                                          Key* __restrict__ keys) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) keys[i] = key_of<Key>(rows + i);
}

// Thread t < n_a: source row t; t >= n_a: baseline row t - n_a. lb_*: the lower bound into the other side's keys, with
// kMatched when that side holds the key; keep_*: the row is listed by its own thread (keep_*[n] = 0 closes each
// scan); *both: the matched source rows.
template <class Key>
__global__ void __launch_bounds__(256) change_match_kernel(const Key* __restrict__ ka, uint32_t n_a,
                                                           const Key* __restrict__ kb, uint32_t n_b,
                                                           uint32_t presence, uint32_t* __restrict__ lb_a,
                                                           uint32_t* __restrict__ lb_b, uint32_t* __restrict__ keep_a,
                                                           uint32_t* __restrict__ keep_b, uint32_t* __restrict__ both) {
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t matched = 0;
  for (uint32_t t = t0; t < n_a + n_b; t += stride) {
    if (t < n_a) {
      const Key key = ka[t];
      const uint32_t p = lower_bound_key(kb, n_b, key);
      const bool m = p < n_b && kb[p] == key;
      lb_a[t] = p | (m ? kMatched : 0u);
      keep_a[t] = (presence & (m ? ALZ_PRESENT_BOTH : ALZ_PRESENT_NEW)) ? 1u : 0u;
      matched += m;
    } else {
      const uint32_t j = t - n_a;
      const Key key = kb[j];
      const uint32_t p = lower_bound_key(ka, n_a, key);
      const bool m = p < n_a && ka[p] == key;
      lb_b[j] = p | (m ? kMatched : 0u);
      keep_b[j] = (!m && (presence & ALZ_PRESENT_GONE)) ? 1u : 0u;
    }
  }
  matched = __reduce_add_sync(0xFFFFFFFFu, matched);   // every lane of the warp leaves the loop to get here
  if ((threadIdx.x & 31u) == 0 && matched) atomicAdd(both, matched);
  if (t0 == 0) { keep_a[n_a] = 0u; keep_b[n_b] = 0u; }
}

struct EmitArgs {
  const alz_edge_out* rows_a;
  const alz_edge_out* rows_b;
  uint32_t n_a, n_b;
  const uint32_t *lb_a, *lb_b, *keep_a, *keep_b, *scan_a, *scan_b;
  const double *val_a, *val_b;
  double win_a, win_b;
  bool divide;
  uint32_t mode;
};

// one record per listed row, written by the thread of its source row (BOTH, NEW) or of its baseline row (GONE); with
// chg, its change too
__global__ void __launch_bounds__(256) change_emit_kernel(const __grid_constant__ EmitArgs a,
                                                          alz_edge_change* __restrict__ out,
                                                          uint64_t* __restrict__ chg) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < a.n_a + a.n_b; t += stride) {
    const bool src = t < a.n_a;
    const uint32_t i = src ? t : t - a.n_a;
    if (!(src ? a.keep_a[i] : a.keep_b[i])) continue;
    const uint32_t lb = src ? a.lb_a[i] : a.lb_b[i];
    const uint32_t p = lb & ~kMatched;
    const uint32_t pos = src ? a.scan_a[i] + a.scan_b[p] : a.scan_a[p] + a.scan_b[i];
    const uint2* row = reinterpret_cast<const uint2*>(src ? a.rows_a + i : a.rows_b + i);
    const uint2 ty = row[0], ft = row[1];   // from_type, to_type, pad | from, to
    uint32_t presence, index, base_index;
    double value, base;
    if (src) {
      const bool m = (lb & kMatched) != 0u;
      presence = m ? ALZ_PRESENT_BOTH : ALZ_PRESENT_NEW;
      index = i;
      base_index = m ? p : kAbsent;
      value = per_window(a.val_a[i], a.divide, a.win_a);
      base = m ? per_window(a.val_b[p], a.divide, a.win_b) : 0.0;
    } else {
      presence = ALZ_PRESENT_GONE;
      index = kAbsent;
      base_index = i;
      value = 0.0;
      base = per_window(a.val_b[i], a.divide, a.win_b);
    }
    const double c = change_of(a.mode, value, base);
    uint4* o = reinterpret_cast<uint4*>(out + pos);
    o[0] = make_uint4((ty.x & 0xFFFFu) | (presence << 16), 0u, ft.x, ft.y);
    o[1] = make_uint4(index, base_index, (uint32_t)__double_as_longlong(value),
                      (uint32_t)((uint64_t)__double_as_longlong(value) >> 32));
    const uint64_t bb = (uint64_t)__double_as_longlong(base), cb = (uint64_t)__double_as_longlong(c);
    o[2] = make_uint4((uint32_t)bb, (uint32_t)(bb >> 32), (uint32_t)cb, (uint32_t)(cb >> 32));
    if (chg) chg[pos] = cb;
  }
}

// result j = the record at the j-th selected position (Record: alz_edge_change, or alz_node_change of
// alz_node_changes.cu)
template <class Record>
__global__ void __launch_bounds__(256) change_gather_kernel(const uint32_t* __restrict__ idx, uint32_t m,
                                                            const Record* __restrict__ list,
                                                            Record* __restrict__ out) {
  static_assert(sizeof(Record) == 48, "three 16-byte words");
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < 3u * m; t += stride) {   // three 16-byte words each
    const uint32_t j = t / 3u, w = t % 3u;
    reinterpret_cast<uint4*>(out + j)[w] = reinterpret_cast<const uint4*>(list + idx[j])[w];
  }
}

}  // namespace

// The pinned baseline and the buffers of the change calls, each grown on demand and never shrunk; freed in alz_destroy
struct alz_changes_state {
  DevBuf base_rows, base_keys;   // the baseline: its rows and their packed keys
  size_t base_n = 0;
  bool pinned = false;
  uint64_t generation = 0;       // pins so far: tells the node and group changes' cached baseline from a later pin's
  alz_rollup_info base_info{};
  ChangeBufs j;                  // the join's scratch and results
};

void alz::metrics::ChangeBufs::free() {
  free_bufs({&keys_a, &keys_b, &member_a, &member_b, &lb_a, &lb_b, &keep_a, &keep_b, &scan_a, &scan_b, &val_a, &val_b,
             &counts, &tmp, &list, &chg, &top_list});
  sel.free();
}

void alz_internal_free_changes(alz_handle* h) {
  alz_changes_state* s = h->changes;
  if (!s) return;
  free_bufs({&s->base_rows, &s->base_keys});
  s->j.free();
  delete s;
  h->changes = nullptr;
}

namespace {

// allocated on first use; its buffers start empty
alz_changes_state* changes_state(alz_handle* h) {
  if (!h->changes) h->changes = new alz_changes_state();
  return h->changes;
}

}  // namespace

int alz::metrics::source_rows(alz_handle* h, uint32_t source, const alz_edge_out** rows, size_t* n,
                              alz_rollup_info* info) {
  if (source == ALZ_SOURCE_WINDOW) {
    *rows = h->d_out;
    *n = h->last_n_edges;
    *info = alz_rollup_info{};
    info->windows = 1;
    return ALZ_OK;
  }
  return alz_internal_rollup_rows(h, source, rows, n, info);
}

void alz::metrics::launch_row_keys(alz_handle* h, const alz_edge_out* rows, uint32_t n, uint64_t* keys) {
  if (n == 0) return;
  change_keys_kernel<uint64_t><<<std::min<unsigned>((n + 255) / 256, (unsigned)h->sms * 8), 256, 0, h->stream>>>(rows, n,
                                                                                                        keys);
  h->launches += 1;
}

int alz::metrics::pinned_baseline(alz_handle* h, const alz_edge_out** rows, size_t* n, alz_rollup_info* info,
                                  uint64_t* generation) {
  const alz_changes_state* s = h->changes;
  if (!s || !s->pinned) return ALZ_E_STATE;
  *rows = static_cast<const alz_edge_out*>(s->base_rows.p);
  *n = s->base_n;
  *info = s->base_info;
  *generation = s->generation;
  return ALZ_OK;
}

template <class Record>
int alz::metrics::gather_changes(alz_handle* h, const uint32_t* idx, uint32_t m, const Record* list, Record* out) {
  if (m == 0) return ALZ_OK;
  change_gather_kernel<<<std::min<unsigned>((3u * m + 255) / 256, (unsigned)h->sms * 4), 256, 0, h->stream>>>(
      idx, m, list, out);
  h->launches += 1;
  CK(cudaGetLastError());
  return ALZ_OK;
}
template int alz::metrics::gather_changes(alz_handle*, const uint32_t*, uint32_t, const alz_edge_change*,
                                          alz_edge_change*);
template int alz::metrics::gather_changes(alz_handle*, const uint32_t*, uint32_t, const alz_node_change*,
                                          alz_node_change*);

int alz::metrics::edge_change_join(alz_handle* h, ChangeBufs& cb, EdgeChangeSide a, EdgeChangeSide b, bool ends,
                                   const MetricSet& ms, uint32_t mode, uint32_t presence, bool top, uint64_t* listed,
                                   alz_change_info* ci) {
  cudaStream_t st = h->stream;
  const size_t na = a.n, nb = b.n;
  const size_t key_bytes = ends ? sizeof(EndsKey) : 8;
  int rc = reserve(h, {{&cb.keys_a, a.keys ? 0 : std::max<size_t>(na, 1) * key_bytes},
                       {&cb.keys_b, b.keys ? 0 : std::max<size_t>(nb, 1) * key_bytes},
                       {&cb.lb_a, std::max<size_t>(na, 1) * 4},
                       {&cb.lb_b, std::max<size_t>(nb, 1) * 4},
                       {&cb.keep_a, (na + 1) * 4},
                       {&cb.keep_b, (nb + 1) * 4},
                       {&cb.scan_a, (na + 1) * 4},
                       {&cb.scan_b, (nb + 1) * 4},
                       {&cb.val_a, std::max<size_t>(na, 1) * 8},
                       {&cb.val_b, std::max<size_t>(nb, 1) * 8},
                       {&cb.counts, 4},
                       {&cb.tmp, scan_temp_bytes((uint32_t)std::max(na, nb) + 1)}});
  if (rc != ALZ_OK) return rc;
  uint32_t* lb_a = static_cast<uint32_t*>(cb.lb_a.p);
  uint32_t* lb_b = static_cast<uint32_t*>(cb.lb_b.p);
  uint32_t* keep_a = static_cast<uint32_t*>(cb.keep_a.p);
  uint32_t* keep_b = static_cast<uint32_t*>(cb.keep_b.p);
  uint32_t* scan_a = static_cast<uint32_t*>(cb.scan_a.p);
  uint32_t* scan_b = static_cast<uint32_t*>(cb.scan_b.p);
  uint32_t* both = static_cast<uint32_t*>(cb.counts.p);
  CK(cudaMemsetAsync(both, 0, 4, st));
  const uint32_t n_ab = a.n + b.n;   // each side is below 2^30
  const unsigned grid = std::max<unsigned>(1u, std::min<unsigned>((n_ab + 255) / 256, (unsigned)h->sms * 8));
  if (ends) {
    EndsKey* ka = static_cast<EndsKey*>(cb.keys_a.p);
    EndsKey* kb = static_cast<EndsKey*>(cb.keys_b.p);
    for (auto [rows, n, keys] : {std::make_tuple(a.rows, a.n, ka), std::make_tuple(b.rows, b.n, kb)}) {
      if (n == 0) continue;
      change_keys_kernel<EndsKey><<<std::min<unsigned>((n + 255) / 256, (unsigned)h->sms * 8), 256, 0, st>>>(rows, n,
                                                                                                             keys);
      h->launches += 1;
    }
    change_match_kernel<EndsKey><<<grid, 256, 0, st>>>(ka, a.n, kb, b.n, presence, lb_a, lb_b, keep_a, keep_b, both);
  } else {
    if (!a.keys) { launch_row_keys(h, a.rows, a.n, static_cast<uint64_t*>(cb.keys_a.p)); a.keys = static_cast<uint64_t*>(cb.keys_a.p); }
    if (!b.keys) { launch_row_keys(h, b.rows, b.n, static_cast<uint64_t*>(cb.keys_b.p)); b.keys = static_cast<uint64_t*>(cb.keys_b.p); }
    change_match_kernel<uint64_t><<<grid, 256, 0, st>>>(a.keys, a.n, b.keys, b.n, presence, lb_a, lb_b, keep_a,
                                                        keep_b, both);
  }
  h->launches += 1;
  CK(exclusive_scan_u32(cb.tmp.p, cb.tmp.bytes, keep_a, scan_a, a.n + 1, st));
  CK(exclusive_scan_u32(cb.tmp.p, cb.tmp.bytes, keep_b, scan_b, b.n + 1, st));
  rc = run_metrics(h, a.rows, a.n, ms, static_cast<double*>(cb.val_a.p));
  if (rc != ALZ_OK) return rc;
  rc = run_metrics(h, b.rows, b.n, ms, static_cast<double*>(cb.val_b.p));
  if (rc != ALZ_OK) return rc;
  CK(cudaGetLastError());
  uint32_t cnt[3];   // listed source rows, listed gone rows, matched source rows
  CK(cudaMemcpyAsync(&cnt[0], scan_a + a.n, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(&cnt[1], scan_b + b.n, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(&cnt[2], both, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));   // the one wait: the union's counts
  const uint64_t n_both = cnt[2];
  *ci = alz_change_info{};
  ci->source_rows = na;
  ci->base_rows = nb;
  ci->both = n_both;
  ci->added = na - n_both;
  ci->gone = nb - n_both;
  ci->listed = (uint64_t)cnt[0] + cnt[1];
  ci->source_windows = a.windows;
  ci->base_windows = b.windows;
  *listed = ci->listed;
  if (na + nb - n_both > kMaxRows) return ALZ_E_CAPACITY;
  rc = reserve(h, {{&cb.list, std::max<size_t>(*listed, 1) * sizeof(alz_edge_change)},
                   {&cb.chg, top ? std::max<size_t>(*listed, 1) * 8 : 0}});
  if (rc != ALZ_OK) return rc;
  if (*listed) {
    const bool divide = ms.kind[0] == ALZ_METRIC_COUNT || ms.kind[0] == ALZ_METRIC_ERR5XX;
    const EmitArgs ea{a.rows, b.rows, a.n, b.n, lb_a, lb_b, keep_a, keep_b, scan_a, scan_b,
                      static_cast<const double*>(cb.val_a.p), static_cast<const double*>(cb.val_b.p),
                      (double)a.windows, (double)b.windows, divide, mode};
    change_emit_kernel<<<grid, 256, 0, st>>>(ea, static_cast<alz_edge_change*>(cb.list.p),
                                             top ? static_cast<uint64_t*>(cb.chg.p) : nullptr);
    h->launches += 1;
    CK(cudaGetLastError());
  }
  return ALZ_OK;
}

template <class Record>
int alz::metrics::change_results(alz_handle* h, ChangeBufs& cb, bool top, uint64_t listed, uint32_t k,
                                 double min_change, const Record** res, size_t* n, alz_change_info* ci) {
  if (!top) {
    *res = static_cast<const Record*>(cb.list.p);
    *n = listed;
    return ALZ_OK;
  }
  size_t m = 0;
  uint64_t above = 0;
  int rc = select_top(h, cb.sel, static_cast<const uint64_t*>(cb.chg.p), (uint32_t)listed, k, min_change, nullptr,
                      &m, &above);
  if (rc != ALZ_OK) return rc;
  ci->above = above;
  rc = reserve(h, {{&cb.top_list, std::max<size_t>(m, 1) * sizeof(Record)}});
  if (rc != ALZ_OK) return rc;
  rc = gather_changes(h, static_cast<const uint32_t*>(cb.sel.top_index.p), (uint32_t)m,
                      static_cast<const Record*>(cb.list.p), static_cast<Record*>(cb.top_list.p));
  if (rc != ALZ_OK) return rc;
  *res = static_cast<const Record*>(cb.top_list.p);
  *n = m;
  return ALZ_OK;
}
template int alz::metrics::change_results(alz_handle*, ChangeBufs&, bool, uint64_t, uint32_t, double,
                                          const alz_edge_change**, size_t*, alz_change_info*);
template int alz::metrics::change_results(alz_handle*, ChangeBufs&, bool, uint64_t, uint32_t, double,
                                          const alz_node_change**, size_t*, alz_change_info*);

namespace {

// The change list of `source` against the baseline (top: its first min(k, above) records by change) into s->j.list or
// s->j.top_list; *n = records. Caller holds h->mu.
int changes_locked(alz_handle* h, uint32_t source, const MetricSet& ms, uint32_t mode, uint32_t presence, bool top,
                   uint32_t k, double min_change, const alz_edge_change** res, size_t* n, alz_change_info* ci) {
  CK(cudaSetDevice(h->device));
  const alz_edge_out* rows = nullptr;
  size_t n_src = 0;
  alz_rollup_info ri;
  int rc = source_rows(h, source, &rows, &n_src, &ri);
  if (rc != ALZ_OK) return rc;
  alz_changes_state* s = h->changes;
  if (!s || !s->pinned) return ALZ_E_STATE;
  if (n_src > kMaxRows || s->base_n > kMaxRows) return ALZ_E_CAPACITY;
  uint64_t listed = 0;
  rc = edge_change_join(h, s->j, EdgeChangeSide{rows, nullptr, (uint32_t)n_src, ri.windows},
                        EdgeChangeSide{static_cast<const alz_edge_out*>(s->base_rows.p),
                                       static_cast<const uint64_t*>(s->base_keys.p), (uint32_t)s->base_n,
                                       s->base_info.windows},
                        false, ms, mode, presence, top, &listed, ci);
  if (rc != ALZ_OK) return rc;
  return change_results(h, s->j, top, listed, k, min_change, res, n, ci);
}

bool valid_change(const alz_metric* m, uint32_t mode, uint32_t presence, MetricSet* ms) {
  return valid_metrics(m, 1, ms) && mode <= ALZ_CHANGE_RATIO && presence != 0 && presence <= 7u;
}

// The four entry points: device (dev_out set) or host (cap records in out, one more wait for the copy)
int changes_entry(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode, uint32_t presence, bool top,
                  uint32_t k, double min_change, alz_edge_change* out, size_t cap, const alz_edge_change** dev_out,
                  size_t* n_out, alz_change_info* info) {
  if (!h || !n_out) return ALZ_E_INVAL;
  *n_out = 0;
  if (info) *info = alz_change_info{};
  MetricSet ms;
  if (!valid_change(m, mode, presence, &ms) || (!dev_out && !out && cap)) return ALZ_E_INVAL;
  if (source != ALZ_SOURCE_WINDOW && source > ALZ_ROLLUP_SPAN) return ALZ_E_INVAL;
  if (top && (k == 0 || std::isnan(min_change))) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  changes_state(h);
  const alz_edge_change* res = nullptr;
  size_t n = 0;
  alz_change_info ci{};
  const int rc = changes_locked(h, source, ms, mode, presence, top, k, min_change, &res, &n, &ci);
  if (info) *info = ci;
  if (rc != ALZ_OK) return rc;
  *n_out = n;
  if (dev_out) {
    *dev_out = res;
    return ALZ_OK;
  }
  if (n > cap) return ALZ_E_CAPACITY;
  if (n) CK(cudaMemcpyAsync(out, res, n * sizeof(alz_edge_change), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return ALZ_OK;
}

}  // namespace

extern "C" int alz_baseline_pin(alz_handle* h, uint32_t source, alz_rollup_info* info) {
  if (!h) return ALZ_E_INVAL;
  if (source != ALZ_SOURCE_WINDOW && source > ALZ_ROLLUP_SPAN) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  const alz_edge_out* rows = nullptr;
  size_t n = 0;
  alz_rollup_info ri;
  int rc = source_rows(h, source, &rows, &n, &ri);
  if (rc == ALZ_OK && source == ALZ_SOURCE_WINDOW) rc = alz_internal_window_info(h, &ri);
  if (rc != ALZ_OK) return rc;   // the baseline, if any, stays as it was
  alz_changes_state* s = changes_state(h);
  s->pinned = false;   // a failure below leaves no baseline
  s->base_n = 0;
  s->generation += 1;
  if (n > kMaxRows) return ALZ_E_CAPACITY;
  rc = reserve(h, {{&s->base_rows, std::max<size_t>(n, 1) * sizeof(alz_edge_out)},
                   {&s->base_keys, std::max<size_t>(n, 1) * 8}});
  if (rc != ALZ_OK) return rc;
  if (n) {
    CK(cudaMemcpyAsync(s->base_rows.p, rows, n * sizeof(alz_edge_out), cudaMemcpyDeviceToDevice, h->stream));
    launch_row_keys(h, static_cast<const alz_edge_out*>(s->base_rows.p), (uint32_t)n, static_cast<uint64_t*>(s->base_keys.p));
    CK(cudaGetLastError());
  }
  s->base_n = n;
  s->base_info = ri;
  s->pinned = true;
  if (info) *info = ri;
  return ALZ_OK;
}

extern "C" int alz_baseline_clear(alz_handle* h) {
  if (!h) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  if (h->changes) {
    h->changes->pinned = false;
    h->changes->base_n = 0;
  }
  return ALZ_OK;
}

extern "C" int alz_edge_changes(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode, uint32_t presence,
                                alz_edge_change* out, size_t cap, size_t* n_out, alz_change_info* info) {
  return changes_entry(h, source, m, mode, presence, false, 0, 0.0, out, cap, nullptr, n_out, info);
}

extern "C" int alz_edge_changes_device(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode,
                                       uint32_t presence, const alz_edge_change** dev_out, size_t* n_out,
                                       alz_change_info* info) {
  if (!dev_out) return n_out ? (*n_out = 0, ALZ_E_INVAL) : ALZ_E_INVAL;
  return changes_entry(h, source, m, mode, presence, false, 0, 0.0, nullptr, 0, dev_out, n_out, info);
}

extern "C" int alz_edge_changes_top(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode,
                                    uint32_t presence, uint32_t k, double min_change, alz_edge_change* out, size_t cap,
                                    size_t* n_out, alz_change_info* info) {
  return changes_entry(h, source, m, mode, presence, true, k, min_change, out, cap, nullptr, n_out, info);
}

extern "C" int alz_edge_changes_top_device(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode,
                                           uint32_t presence, uint32_t k, double min_change,
                                           const alz_edge_change** dev_out, size_t* n_out, alz_change_info* info) {
  if (!dev_out) return n_out ? (*n_out = 0, ALZ_E_INVAL) : ALZ_E_INVAL;
  return changes_entry(h, source, m, mode, presence, true, k, min_change, nullptr, 0, dev_out, n_out, info);
}

extern "C" int alz_debug_edge_changes_rows(alz_handle* h, const alz_edge_out* dev_src, size_t n_src,
                                           uint32_t src_windows, const alz_edge_out* dev_base, size_t n_base,
                                           uint32_t base_windows, const alz_metric* m, uint32_t mode,
                                           uint32_t presence, alz_edge_change* out, size_t cap, size_t* n_out,
                                           alz_change_info* info) {
  if (!h || !n_out) return ALZ_E_INVAL;
  *n_out = 0;
  if (info) *info = alz_change_info{};
  MetricSet ms;
  if (!valid_change(m, mode, presence, &ms) || (!out && cap) || (!dev_src && n_src) || (!dev_base && n_base) ||
      src_windows == 0 || base_windows == 0)
    return ALZ_E_INVAL;
  if (n_src > kMaxRows || n_base > kMaxRows) return ALZ_E_CAPACITY;
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  alz_changes_state* s = changes_state(h);
  uint64_t listed = 0;
  alz_change_info ci{};
  const int rc = edge_change_join(h, s->j, EdgeChangeSide{dev_src, nullptr, (uint32_t)n_src, src_windows},
                                  EdgeChangeSide{dev_base, nullptr, (uint32_t)n_base, base_windows}, false, ms, mode,
                                  presence, false, &listed, &ci);
  if (info) *info = ci;
  if (rc != ALZ_OK) return rc;
  *n_out = listed;
  if (listed > cap) return ALZ_E_CAPACITY;
  if (listed) CK(cudaMemcpyAsync(out, s->j.list.p, listed * sizeof(alz_edge_change), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return ALZ_OK;
}
