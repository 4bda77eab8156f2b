// alz_node_changes.cu — node changes against the pinned baseline (docs/SPEC.md §23): the §21 node lists of a source
// and of the baseline, joined by node key as §18 joins edge rows, with each side's §17 values of one side (IN or OUT)
// of each node, and one record per node of the filtered union or only its top nodes by change (DESIGN.md §5.15).
//   group   the §21 group-by (alz_nodes.cu) of the source's rows into this state's node rows, one wait for the node
//           count. The baseline's rows are grouped the same way on the first call after a pin and kept: the pin's
//           generation (alz_changes.cu) says when they are stale, so alz_baseline_pin enqueues nothing more.
//   keys    each node row's head word as its key (type << 32) | value, and whether it has a row on the side (member)
//   match   every node of either list: lower_bound into the other list's keys; a key matches only a member there.
//           A member source node is kept as BOTH or NEW, a member baseline node as GONE when unmatched; a non-member
//           is never kept. Both lists stay sorted, so §18's positions hold: a kept source node i goes to scanA[i] +
//           scanG[lb_B(key_i)], a kept gone baseline node j to scanA[lb_A(key_j)] + scanG[j]
//   scan    two exclusive scans of the keep flags, then one wait for the union's counts
//   values  the §17 metric kernels over each list's node side (NodeRows)
//   emit    one 48-byte record per listed node in three 16-byte stores, and for the top call its change into an
//           8-byte array, which the §17 selection ranks; the selected records are gathered by position
// Waits: the source's node count, the baseline's (first call after a pin only), the union's counts, and on a top call
// the selection's; a host call adds one for its copy. Growing a buffer adds one.
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <mutex>
#include <string>

#include "alz_metrics.cuh"

using namespace alz;
using namespace alz::metrics;

static_assert(sizeof(alz_node_change) == 48, "alz_node_change is three 16-byte stores");
static_assert(offsetof(alz_node_change, presence) == offsetof(alz_edge_change, presence) &&
                  offsetof(alz_node_change, index) == offsetof(alz_edge_change, index) &&
                  offsetof(alz_node_change, base_index) == offsetof(alz_edge_change, base_index) &&
                  offsetof(alz_node_change, value) == offsetof(alz_edge_change, value) &&
                  offsetof(alz_node_change, base_value) == offsetof(alz_edge_change, base_value) &&
                  offsetof(alz_node_change, change) == offsetof(alz_edge_change, change),
              "alz_node_change shares alz_edge_change's offsets from presence on");
static_assert(offsetof(alz_node_out, value) == 4 && offsetof(alz_node_out, in_edges) == 8 &&
                  offsetof(alz_node_out, out_edges) == 12,
              "a node row's first 16 bytes are type, value, in_edges, out_edges");

namespace {

constexpr uint32_t kAbsent = 0xFFFFFFFFu;
constexpr uint32_t kMatched = 0x80000000u;   // in a lower bound: the other list holds the key as a member

// Node i's key from its head word, and whether it has a row on `side`; *members += the nodes that do
__global__ void __launch_bounds__(256) node_change_keys_kernel(const alz_node_out* __restrict__ nodes, uint32_t n,
                                                               uint32_t side, uint64_t* __restrict__ keys,
                                                               uint8_t* __restrict__ member,
                                                               uint32_t* __restrict__ members) {
  const uint32_t stride = gridDim.x * blockDim.x;
  uint32_t count = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint4 w = reinterpret_cast<const uint4*>(nodes + i)[0];   // type, value, in_edges, out_edges
    keys[i] = ((uint64_t)w.x << 32) | w.y;
    const bool m = (side == ALZ_SIDE_IN ? w.z : w.w) != 0u;
    member[i] = m ? 1u : 0u;
    count += m;
  }
  count = __reduce_add_sync(0xFFFFFFFFu, count);   // every lane of the warp leaves the loop to get here
  if ((threadIdx.x & 31u) == 0 && count) atomicAdd(members, count);
}

// Thread t < n_a: source node t; t >= n_a: baseline node t - n_a. lb_*: the lower bound into the other list's keys,
// with kMatched when that list holds the key as a member (0 for a non-member, which is never kept); keep_*: the node
// is listed by its own thread (keep_*[n] = 0 closes each scan); *both: the matched source nodes.
__global__ void __launch_bounds__(256) node_change_match_kernel(const uint64_t* __restrict__ ka,
                                                                const uint8_t* __restrict__ ma, uint32_t n_a,
                                                                const uint64_t* __restrict__ kb,
                                                                const uint8_t* __restrict__ mb, uint32_t n_b,
                                                                uint32_t presence, uint32_t* __restrict__ lb_a,
                                                                uint32_t* __restrict__ lb_b,
                                                                uint32_t* __restrict__ keep_a,
                                                                uint32_t* __restrict__ keep_b,
                                                                uint32_t* __restrict__ both) {
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t matched = 0;
  for (uint32_t t = t0; t < n_a + n_b; t += stride) {
    const bool src = t < n_a;
    const uint32_t i = src ? t : t - n_a;
    const uint64_t* other = src ? kb : ka;
    const uint8_t* other_member = src ? mb : ma;
    const uint32_t n_other = src ? n_b : n_a;
    const bool in = (src ? ma[i] : mb[i]) != 0u;
    uint32_t p = 0;
    bool m = false;
    if (in) {
      const uint64_t key = src ? ka[i] : kb[i];
      p = lower_bound_u64(other, n_other, key);
      m = p < n_other && other[p] == key && other_member[p] != 0u;
    }
    const uint32_t lb = p | (m ? kMatched : 0u);
    if (src) {
      lb_a[i] = lb;
      keep_a[i] = (in && (presence & (m ? ALZ_PRESENT_BOTH : ALZ_PRESENT_NEW))) ? 1u : 0u;
      matched += m;
    } else {
      lb_b[i] = lb;
      keep_b[i] = (in && !m && (presence & ALZ_PRESENT_GONE)) ? 1u : 0u;
    }
  }
  matched = __reduce_add_sync(0xFFFFFFFFu, matched);
  if ((threadIdx.x & 31u) == 0 && matched) atomicAdd(both, matched);
  if (t0 == 0) { keep_a[n_a] = 0u; keep_b[n_b] = 0u; }
}

struct EmitArgs {
  const alz_node_out* nodes_a;
  const alz_node_out* nodes_b;
  uint32_t n_a, n_b;
  const uint32_t *lb_a, *lb_b, *keep_a, *keep_b, *scan_a, *scan_b;
  const double *val_a, *val_b;
  double win_a, win_b;
  bool divide;
  uint32_t mode;
};

// one record per listed node, written by the thread of its source node (BOTH, NEW) or of its baseline node (GONE);
// with chg, its change too
__global__ void __launch_bounds__(256) node_change_emit_kernel(const __grid_constant__ EmitArgs a,
                                                               alz_node_change* __restrict__ out,
                                                               uint64_t* __restrict__ chg) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < a.n_a + a.n_b; t += stride) {
    const bool src = t < a.n_a;
    const uint32_t i = src ? t : t - a.n_a;
    if (!(src ? a.keep_a[i] : a.keep_b[i])) continue;
    const uint32_t lb = src ? a.lb_a[i] : a.lb_b[i];
    const uint32_t p = lb & ~kMatched;
    const uint32_t pos = src ? a.scan_a[i] + a.scan_b[p] : a.scan_a[p] + a.scan_b[i];
    const uint2 tv = reinterpret_cast<const uint2*>(src ? a.nodes_a + i : a.nodes_b + i)[0];   // type | value
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
    const uint64_t vb = (uint64_t)__double_as_longlong(value);
    o[0] = make_uint4((tv.x & 0xFFu) | (presence << 16), 0u, tv.y, 0u);
    o[1] = make_uint4(index, base_index, (uint32_t)vb, (uint32_t)(vb >> 32));
    const uint64_t bb = (uint64_t)__double_as_longlong(base), cb = (uint64_t)__double_as_longlong(c);
    o[2] = make_uint4((uint32_t)bb, (uint32_t)(bb >> 32), (uint32_t)cb, (uint32_t)(cb >> 32));
    if (chg) chg[pos] = cb;
  }
}

unsigned grid_for(alz_handle* h, uint64_t threads, unsigned per_sm) {
  return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((threads + 255) / 256, (uint64_t)h->sms * per_sm));
}

}  // namespace

// Buffers of the node change calls, each grown on demand and never shrunk; freed in alz_destroy
struct alz_node_changes_state {
  NodeGroup g;                     // the group-by's scratch
  DevBuf src_nodes, base_nodes;    // the source's node rows; the baseline's (or the hook's second list's)
  size_t base_n = 0;               // base_nodes' rows
  bool base_cached = false;        // base_nodes hold the baseline of pin base_gen
  uint64_t base_gen = 0;
  ChangeBufs j;                    // the join's scratch and results
};

void alz_internal_free_node_changes(alz_handle* h) {
  alz_node_changes_state* s = h->node_changes;
  if (!s) return;
  s->g.free();
  free_bufs({&s->src_nodes, &s->base_nodes});
  s->j.free();
  delete s;
  h->node_changes = nullptr;
}

int alz::metrics::node_change_join(alz_handle* h, ChangeBufs& cb, NodeChangeSide a, NodeChangeSide b, uint32_t side,
                                   const MetricSet& ms, uint32_t mode, uint32_t presence, bool top, uint64_t* listed,
                                   alz_change_info* ci) {
  cudaStream_t st = h->stream;
  const size_t na = a.n, nb = b.n;
  int rc = reserve(h, {{&cb.keys_a, std::max<size_t>(na, 1) * 8},
                       {&cb.keys_b, std::max<size_t>(nb, 1) * 8},
                       {&cb.member_a, std::max<size_t>(na, 1)},
                       {&cb.member_b, std::max<size_t>(nb, 1)},
                       {&cb.lb_a, std::max<size_t>(na, 1) * 4},
                       {&cb.lb_b, std::max<size_t>(nb, 1) * 4},
                       {&cb.keep_a, (na + 1) * 4},
                       {&cb.keep_b, (nb + 1) * 4},
                       {&cb.scan_a, (na + 1) * 4},
                       {&cb.scan_b, (nb + 1) * 4},
                       {&cb.val_a, std::max<size_t>(na, 1) * 8},
                       {&cb.val_b, std::max<size_t>(nb, 1) * 8},
                       {&cb.counts, 3 * 4},
                       {&cb.tmp, scan_temp_bytes((uint32_t)std::max(na, nb) + 1)}});
  if (rc != ALZ_OK) return rc;
  uint64_t* keys_a = static_cast<uint64_t*>(cb.keys_a.p);
  uint64_t* keys_b = static_cast<uint64_t*>(cb.keys_b.p);
  uint8_t* member_a = static_cast<uint8_t*>(cb.member_a.p);
  uint8_t* member_b = static_cast<uint8_t*>(cb.member_b.p);
  uint32_t* lb_a = static_cast<uint32_t*>(cb.lb_a.p);
  uint32_t* lb_b = static_cast<uint32_t*>(cb.lb_b.p);
  uint32_t* keep_a = static_cast<uint32_t*>(cb.keep_a.p);
  uint32_t* keep_b = static_cast<uint32_t*>(cb.keep_b.p);
  uint32_t* scan_a = static_cast<uint32_t*>(cb.scan_a.p);
  uint32_t* scan_b = static_cast<uint32_t*>(cb.scan_b.p);
  uint32_t* counts = static_cast<uint32_t*>(cb.counts.p);   // members of a, members of b, matched members
  CK(cudaMemsetAsync(counts, 0, 3 * 4, st));
  if (na) {
    node_change_keys_kernel<<<grid_for(h, na, 8), 256, 0, st>>>(a.nodes, a.n, side, keys_a, member_a, counts);
    h->launches += 1;
  }
  if (nb) {
    node_change_keys_kernel<<<grid_for(h, nb, 8), 256, 0, st>>>(b.nodes, b.n, side, keys_b, member_b, counts + 1);
    h->launches += 1;
  }
  const uint32_t n_ab = a.n + b.n;   // each list is below 2^30
  const unsigned grid = grid_for(h, n_ab, 8);
  node_change_match_kernel<<<grid, 256, 0, st>>>(keys_a, member_a, a.n, keys_b, member_b, b.n, presence, lb_a, lb_b,
                                                 keep_a, keep_b, counts + 2);
  h->launches += 1;
  CK(exclusive_scan_u32(cb.tmp.p, cb.tmp.bytes, keep_a, scan_a, a.n + 1, st));
  CK(exclusive_scan_u32(cb.tmp.p, cb.tmp.bytes, keep_b, scan_b, b.n + 1, st));
  rc = run_metrics_nodes(h, NodeRows{a.nodes, side}, a.n, ms, static_cast<double*>(cb.val_a.p));
  if (rc != ALZ_OK) return rc;
  rc = run_metrics_nodes(h, NodeRows{b.nodes, side}, b.n, ms, static_cast<double*>(cb.val_b.p));
  if (rc != ALZ_OK) return rc;
  CK(cudaGetLastError());
  uint32_t cnt[5];   // listed source nodes, listed gone nodes, members of a, members of b, matched members
  CK(cudaMemcpyAsync(&cnt[0], scan_a + a.n, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(&cnt[1], scan_b + b.n, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(&cnt[2], counts, 3 * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));   // the one wait: the union's counts
  const uint64_t mem_a = cnt[2], mem_b = cnt[3], n_both = cnt[4];
  *ci = alz_change_info{};
  ci->source_rows = mem_a;
  ci->base_rows = mem_b;
  ci->both = n_both;
  ci->added = mem_a - n_both;
  ci->gone = mem_b - n_both;
  ci->listed = (uint64_t)cnt[0] + cnt[1];
  ci->source_windows = a.windows;
  ci->base_windows = b.windows;
  *listed = ci->listed;
  if (mem_a + mem_b - n_both > kMaxRows) return ALZ_E_CAPACITY;
  rc = reserve(h, {{&cb.list, std::max<size_t>(*listed, 1) * sizeof(alz_node_change)},
                   {&cb.chg, top ? std::max<size_t>(*listed, 1) * 8 : 0}});
  if (rc != ALZ_OK) return rc;
  if (*listed) {
    const bool divide = ms.kind[0] == ALZ_METRIC_COUNT || ms.kind[0] == ALZ_METRIC_ERR5XX;
    const EmitArgs ea{a.nodes, b.nodes, a.n, b.n, lb_a, lb_b, keep_a, keep_b, scan_a, scan_b,
                      static_cast<const double*>(cb.val_a.p), static_cast<const double*>(cb.val_b.p),
                      (double)a.windows, (double)b.windows, divide, mode};
    node_change_emit_kernel<<<grid, 256, 0, st>>>(ea, static_cast<alz_node_change*>(cb.list.p),
                                                  top ? static_cast<uint64_t*>(cb.chg.p) : nullptr);
    h->launches += 1;
    CK(cudaGetLastError());
  }
  return ALZ_OK;
}

namespace {

// The §21 node rows of n rows into *out, on the stream after one wait for the node count (none for n = 0); *nodes =
// that count. Caller holds h->mu and has set the device; n <= kMaxNodeSourceRows.
int group(alz_handle* h, NodeGroup& g, DevBuf* out, const alz_edge_out* rows, size_t n, size_t* nodes) {
  *nodes = 0;
  if (n == 0) return ALZ_OK;
  const uint32_t n2 = 2u * (uint32_t)n;
  int rc = node_group_reserve(h, g, n2);
  if (rc != ALZ_OK) return rc;
  node_group_keys(h, g, rows, (uint32_t)n);
  rc = node_group_runs(h, g, n2, kNodeKeyBits);
  if (rc != ALZ_OK) return rc;
  *nodes = g.h_words[0];
  rc = reserve(h, {{out, *nodes * sizeof(alz_node_out)}});
  if (rc != ALZ_OK) return rc;
  return node_group_reduce(h, g, rows, n2, static_cast<alz_node_out*>(out->p));
}

// The node change list of `source` against the baseline (top: its first min(k, above) records by change) into
// s->j.list or s->j.top_list; *n = records. Caller holds h->mu.
int node_changes_locked(alz_handle* h, uint32_t source, uint32_t side, const MetricSet& ms, uint32_t mode,
                        uint32_t presence, bool top, uint32_t k, double min_change, const alz_node_change** res,
                        size_t* n, alz_change_info* ci) {
  CK(cudaSetDevice(h->device));
  const alz_edge_out* rows = nullptr;
  size_t n_src = 0;
  alz_rollup_info ri;
  int rc = source_rows(h, source, &rows, &n_src, &ri);
  if (rc != ALZ_OK) return rc;
  const alz_edge_out* base_rows = nullptr;
  size_t n_base = 0;
  alz_rollup_info bi;
  uint64_t gen = 0;
  rc = pinned_baseline(h, &base_rows, &n_base, &bi, &gen);
  if (rc != ALZ_OK) return rc;
  if (n_src > kMaxNodeSourceRows || n_base > kMaxNodeSourceRows) return ALZ_E_CAPACITY;
  alz_node_changes_state* s = h->node_changes;
  size_t nodes_a = 0;
  rc = group(h, s->g, &s->src_nodes, rows, n_src, &nodes_a);
  if (rc != ALZ_OK) return rc;
  if (!s->base_cached || s->base_gen != gen) {
    s->base_cached = false;   // a failure below leaves no cached baseline nodes
    rc = group(h, s->g, &s->base_nodes, base_rows, n_base, &s->base_n);
    if (rc != ALZ_OK) return rc;
    s->base_cached = true;
    s->base_gen = gen;
  }
  uint64_t listed = 0;
  rc = node_change_join(h, s->j, NodeChangeSide{static_cast<const alz_node_out*>(s->src_nodes.p), (uint32_t)nodes_a,
                                                 ri.windows},
                        NodeChangeSide{static_cast<const alz_node_out*>(s->base_nodes.p), (uint32_t)s->base_n,
                                       bi.windows},
                        side, ms, mode, presence, top, &listed, ci);
  if (rc != ALZ_OK) return rc;
  return change_results(h, s->j, top, listed, k, min_change, res, n, ci);
}

bool valid_node_change(uint32_t side, const alz_metric* m, uint32_t mode, uint32_t presence, MetricSet* ms) {
  return side <= ALZ_SIDE_OUT && valid_metrics(m, 1, ms) && mode <= ALZ_CHANGE_RATIO && presence != 0 &&
         presence <= 7u;
}

alz_node_changes_state* node_changes_state(alz_handle* h) {
  if (!h->node_changes) h->node_changes = new alz_node_changes_state();
  return h->node_changes;
}

// The four entry points: device (dev_out set) or host (cap records in out, one more wait for the copy)
int node_changes_entry(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t mode,
                       uint32_t presence, bool top, uint32_t k, double min_change, alz_node_change* out, size_t cap,
                       const alz_node_change** dev_out, size_t* n_out, alz_change_info* info) {
  if (!h || !n_out) return ALZ_E_INVAL;
  *n_out = 0;
  if (info) *info = alz_change_info{};
  MetricSet ms;
  if (!valid_node_change(side, m, mode, presence, &ms) || (!dev_out && !out && cap)) return ALZ_E_INVAL;
  if (source != ALZ_SOURCE_WINDOW && source > ALZ_ROLLUP_SPAN) return ALZ_E_INVAL;
  if (top && (k == 0 || std::isnan(min_change))) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  node_changes_state(h);
  const alz_node_change* res = nullptr;
  size_t n = 0;
  alz_change_info ci{};
  const int rc = node_changes_locked(h, source, side, ms, mode, presence, top, k, min_change, &res, &n, &ci);
  if (info) *info = ci;
  if (rc != ALZ_OK) return rc;
  *n_out = n;
  if (dev_out) {
    *dev_out = res;
    return ALZ_OK;
  }
  if (n > cap) return ALZ_E_CAPACITY;
  if (n) CK(cudaMemcpyAsync(out, res, n * sizeof(alz_node_change), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return ALZ_OK;
}

}  // namespace

extern "C" int alz_node_changes(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t mode,
                                uint32_t presence, alz_node_change* out, size_t cap, size_t* n_out,
                                alz_change_info* info) {
  return node_changes_entry(h, source, side, m, mode, presence, false, 0, 0.0, out, cap, nullptr, n_out, info);
}

extern "C" int alz_node_changes_device(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m,
                                       uint32_t mode, uint32_t presence, const alz_node_change** dev_out,
                                       size_t* n_out, alz_change_info* info) {
  if (!dev_out) return n_out ? (*n_out = 0, ALZ_E_INVAL) : ALZ_E_INVAL;
  return node_changes_entry(h, source, side, m, mode, presence, false, 0, 0.0, nullptr, 0, dev_out, n_out, info);
}

extern "C" int alz_node_changes_top(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t mode,
                                    uint32_t presence, uint32_t k, double min_change, alz_node_change* out,
                                    size_t cap, size_t* n_out, alz_change_info* info) {
  return node_changes_entry(h, source, side, m, mode, presence, true, k, min_change, out, cap, nullptr, n_out, info);
}

extern "C" int alz_node_changes_top_device(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m,
                                           uint32_t mode, uint32_t presence, uint32_t k, double min_change,
                                           const alz_node_change** dev_out, size_t* n_out, alz_change_info* info) {
  if (!dev_out) return n_out ? (*n_out = 0, ALZ_E_INVAL) : ALZ_E_INVAL;
  return node_changes_entry(h, source, side, m, mode, presence, true, k, min_change, nullptr, 0, dev_out, n_out,
                            info);
}

extern "C" int alz_debug_node_changes_rows(alz_handle* h, const alz_edge_out* dev_src, size_t n_src,
                                           uint32_t src_windows, const alz_edge_out* dev_base, size_t n_base,
                                           uint32_t base_windows, uint32_t side, const alz_metric* m, uint32_t mode,
                                           uint32_t presence, alz_node_change* out, size_t cap, size_t* n_out,
                                           alz_change_info* info) {
  if (!h || !n_out) return ALZ_E_INVAL;
  *n_out = 0;
  if (info) *info = alz_change_info{};
  MetricSet ms;
  if (!valid_node_change(side, m, mode, presence, &ms) || (!out && cap) || (!dev_src && n_src) ||
      (!dev_base && n_base) || src_windows == 0 || base_windows == 0)
    return ALZ_E_INVAL;
  if (n_src > kMaxNodeSourceRows || n_base > kMaxNodeSourceRows) return ALZ_E_CAPACITY;
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  alz_node_changes_state* s = node_changes_state(h);
  s->base_cached = false;   // base_nodes take the hook's second list
  size_t nodes_a = 0;
  int rc = group(h, s->g, &s->src_nodes, dev_src, n_src, &nodes_a);
  if (rc != ALZ_OK) return rc;
  rc = group(h, s->g, &s->base_nodes, dev_base, n_base, &s->base_n);
  if (rc != ALZ_OK) return rc;
  uint64_t listed = 0;
  alz_change_info ci{};
  rc = node_change_join(h, s->j,
                        NodeChangeSide{static_cast<const alz_node_out*>(s->src_nodes.p), (uint32_t)nodes_a,
                                       src_windows},
                        NodeChangeSide{static_cast<const alz_node_out*>(s->base_nodes.p), (uint32_t)s->base_n,
                                       base_windows},
                        side, ms, mode, presence, false, &listed, &ci);
  if (info) *info = ci;
  if (rc != ALZ_OK) return rc;
  *n_out = listed;
  if (listed > cap) return ALZ_E_CAPACITY;
  if (listed) CK(cudaMemcpyAsync(out, s->j.list.p, listed * sizeof(alz_node_change), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return ALZ_OK;
}
