// alz_group_changes.cu — group changes against the pinned baseline (docs/SPEC.md §25): the source and the baseline
// each grouped by the map in force (§24), then the §18 join of their group-edge lists or the §23 join of their group
// node lists, and one record per entry of the filtered union or only its top entries by change (DESIGN.md §5.17).
//   group   the §24 group-by of the source's rows into this state's group-edge rows (alz_groups.cu, two waits), and
//           for a node call the §21 group-by of those rows (one wait). The baseline's are grouped the same way on the
//           first call that needs them and kept: the pin's generation (alz_changes.cu) and the map's (alz_groups.cu)
//           say when they are stale, so neither alz_baseline_pin nor alz_group_set enqueues anything for them.
//   join    edge calls: §18's keys, match, scans, values and emit on the 16-byte key (node key of from, node key of
//           to), the §24 order both lists come out in (alz_changes.cu); node calls: §23's (alz_node_changes.cu)
//   top     §18's selection and gather
// Every buffer written is this state's or scratch of the group calls, so no other family's results move.
#include <algorithm>
#include <cmath>
#include <mutex>
#include <string>

#include "alz_metrics.cuh"

using namespace alz;
using namespace alz::metrics;

// The buffers of the group change calls and the baseline's groups, each grown on demand and never shrunk; freed in
// alz_destroy
struct alz_group_changes_state {
  DevBuf src_edges, src_nodes;     // the source's group-edge rows and group nodes
  DevBuf base_edges, base_nodes;   // the baseline's, kept across calls
  DevBuf hook_edges;               // the hook's second list's group-edge rows
  size_t base_edges_n = 0, base_nodes_n = 0;
  bool edges_cached = false;       // base_edges hold the baseline of pin pin_gen grouped by map map_gen
  bool nodes_cached = false;       // base_nodes hold the group nodes of base_edges
  uint64_t pin_gen = 0, map_gen = 0;
  ChangeBufs j;                    // the join's scratch and results
};

void alz_internal_free_group_changes(alz_handle* h) {
  alz_group_changes_state* s = h->group_changes;
  if (!s) return;
  free_bufs({&s->src_edges, &s->src_nodes, &s->base_edges, &s->base_nodes, &s->hook_edges});
  s->j.free();
  delete s;
  h->group_changes = nullptr;
}

namespace {

alz_group_changes_state* state(alz_handle* h) {
  if (!h->group_changes) h->group_changes = new alz_group_changes_state();
  return h->group_changes;
}

// The baseline's group edges and, with nodes, its group nodes, regrouped when the pin or the map moved on
int base_groups(alz_handle* h, alz_group_changes_state* s, const alz_edge_out* rows, size_t n, uint64_t pin_gen,
                bool nodes) {
  const uint64_t map_gen = group_map_generation(h);
  if (!s->edges_cached || s->pin_gen != pin_gen || s->map_gen != map_gen) {
    s->edges_cached = s->nodes_cached = false;   // a failure below leaves nothing cached
    alz_group_info gi;
    const int rc = group_edges_into(h, s->base_edges, rows, n, SIZE_MAX, &s->base_edges_n, &gi);
    if (rc != ALZ_OK) return rc;
    s->edges_cached = true;
    s->pin_gen = pin_gen;
    s->map_gen = map_gen;
  }
  if (nodes && !s->nodes_cached) {
    const int rc = group_nodes_into(h, s->base_nodes, static_cast<const alz_edge_out*>(s->base_edges.p),
                                    s->base_edges_n, &s->base_nodes_n);
    if (rc != ALZ_OK) return rc;
    s->nodes_cached = true;
  }
  return ALZ_OK;
}

// The group edge (nodes false) or group node change list of `source` against the baseline, or its first min(k, above)
// records by change (top), in s->j; *n = records. Caller holds h->mu.
template <class Record>
int changes_locked(alz_handle* h, uint32_t source, bool nodes, uint32_t side, const MetricSet& ms, uint32_t mode,
                   uint32_t presence, bool top, uint32_t k, double min_change, const Record** res, size_t* n,
                   alz_change_info* ci) {
  CK(cudaSetDevice(h->device));
  const alz_edge_out* rows = nullptr;
  size_t n_src = 0;
  alz_rollup_info ri;
  int rc = source_rows(h, source, &rows, &n_src, &ri);
  if (rc != ALZ_OK) return rc;
  const alz_edge_out* base_rows = nullptr;
  size_t n_base = 0;
  alz_rollup_info bi;
  uint64_t pin_gen = 0;
  rc = pinned_baseline(h, &base_rows, &n_base, &bi, &pin_gen);
  if (rc != ALZ_OK) return rc;
  if (n_src > kMaxNodeSourceRows || n_base > kMaxNodeSourceRows) return ALZ_E_CAPACITY;
  alz_group_changes_state* s = h->group_changes;
  size_t edges_a = 0;
  alz_group_info gi;
  rc = group_edges_into(h, s->src_edges, rows, n_src, SIZE_MAX, &edges_a, &gi);
  if (rc != ALZ_OK) return rc;
  rc = base_groups(h, s, base_rows, n_base, pin_gen, nodes);
  if (rc != ALZ_OK) return rc;
  uint64_t listed = 0;
  if (nodes) {
    size_t nodes_a = 0;
    rc = group_nodes_into(h, s->src_nodes, static_cast<const alz_edge_out*>(s->src_edges.p), edges_a, &nodes_a);
    if (rc != ALZ_OK) return rc;
    rc = node_change_join(h, s->j,
                          NodeChangeSide{static_cast<const alz_node_out*>(s->src_nodes.p), (uint32_t)nodes_a,
                                         ri.windows},
                          NodeChangeSide{static_cast<const alz_node_out*>(s->base_nodes.p), (uint32_t)s->base_nodes_n,
                                         bi.windows},
                          side, ms, mode, presence, top, &listed, ci);
  } else {
    rc = edge_change_join(h, s->j,
                          EdgeChangeSide{static_cast<const alz_edge_out*>(s->src_edges.p), nullptr, (uint32_t)edges_a,
                                         ri.windows},
                          EdgeChangeSide{static_cast<const alz_edge_out*>(s->base_edges.p), nullptr,
                                         (uint32_t)s->base_edges_n, bi.windows},
                          true, ms, mode, presence, top, &listed, ci);
  }
  if (rc != ALZ_OK) return rc;
  return change_results(h, s->j, top, listed, k, min_change, res, n, ci);
}

bool valid_change(uint32_t side, const alz_metric* m, uint32_t mode, uint32_t presence, MetricSet* ms) {
  return side <= ALZ_SIDE_OUT && valid_metrics(m, 1, ms) && mode <= ALZ_CHANGE_RATIO && presence != 0 &&
         presence <= 7u;
}

// The eight entry points: device (dev_out set) or host (cap records in out, one more wait for the copy)
template <class Record>
int changes_entry(alz_handle* h, uint32_t source, bool nodes, uint32_t side, const alz_metric* m, uint32_t mode,
                  uint32_t presence, bool top, uint32_t k, double min_change, Record* out, size_t cap,
                  const Record** dev_out, size_t* n_out, alz_change_info* info) {
  if (!h || !n_out) return ALZ_E_INVAL;
  *n_out = 0;
  if (info) *info = alz_change_info{};
  MetricSet ms;
  if (!valid_change(side, m, mode, presence, &ms) || (!dev_out && !out && cap)) return ALZ_E_INVAL;
  if (source != ALZ_SOURCE_WINDOW && source > ALZ_ROLLUP_SPAN) return ALZ_E_INVAL;
  if (top && (k == 0 || std::isnan(min_change))) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  state(h);
  const Record* res = nullptr;
  size_t n = 0;
  alz_change_info ci{};
  const int rc = changes_locked(h, source, nodes, side, ms, mode, presence, top, k, min_change, &res, &n, &ci);
  if (info) *info = ci;
  if (rc != ALZ_OK) return rc;
  *n_out = n;
  if (dev_out) {
    *dev_out = res;
    return ALZ_OK;
  }
  if (n > cap) return ALZ_E_CAPACITY;
  if (n) CK(cudaMemcpyAsync(out, res, n * sizeof(Record), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return ALZ_OK;
}

}  // namespace

extern "C" int alz_group_edge_changes(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode,
                                      uint32_t presence, alz_edge_change* out, size_t cap, size_t* n_out,
                                      alz_change_info* info) {
  return changes_entry<alz_edge_change>(h, source, false, ALZ_SIDE_IN, m, mode, presence, false, 0, 0.0, out, cap,
                                        nullptr, n_out, info);
}

extern "C" int alz_group_edge_changes_device(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode,
                                             uint32_t presence, const alz_edge_change** dev_out, size_t* n_out,
                                             alz_change_info* info) {
  if (!dev_out) return n_out ? (*n_out = 0, ALZ_E_INVAL) : ALZ_E_INVAL;
  return changes_entry<alz_edge_change>(h, source, false, ALZ_SIDE_IN, m, mode, presence, false, 0, 0.0, nullptr, 0,
                                        dev_out, n_out, info);
}

extern "C" int alz_group_edge_changes_top(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode,
                                          uint32_t presence, uint32_t k, double min_change, alz_edge_change* out,
                                          size_t cap, size_t* n_out, alz_change_info* info) {
  return changes_entry<alz_edge_change>(h, source, false, ALZ_SIDE_IN, m, mode, presence, true, k, min_change, out,
                                        cap, nullptr, n_out, info);
}

extern "C" int alz_group_edge_changes_top_device(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode,
                                                 uint32_t presence, uint32_t k, double min_change,
                                                 const alz_edge_change** dev_out, size_t* n_out,
                                                 alz_change_info* info) {
  if (!dev_out) return n_out ? (*n_out = 0, ALZ_E_INVAL) : ALZ_E_INVAL;
  return changes_entry<alz_edge_change>(h, source, false, ALZ_SIDE_IN, m, mode, presence, true, k, min_change,
                                        nullptr, 0, dev_out, n_out, info);
}

extern "C" int alz_group_node_changes(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m,
                                      uint32_t mode, uint32_t presence, alz_node_change* out, size_t cap,
                                      size_t* n_out, alz_change_info* info) {
  return changes_entry<alz_node_change>(h, source, true, side, m, mode, presence, false, 0, 0.0, out, cap, nullptr,
                                        n_out, info);
}

extern "C" int alz_group_node_changes_device(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m,
                                             uint32_t mode, uint32_t presence, const alz_node_change** dev_out,
                                             size_t* n_out, alz_change_info* info) {
  if (!dev_out) return n_out ? (*n_out = 0, ALZ_E_INVAL) : ALZ_E_INVAL;
  return changes_entry<alz_node_change>(h, source, true, side, m, mode, presence, false, 0, 0.0, nullptr, 0, dev_out,
                                        n_out, info);
}

extern "C" int alz_group_node_changes_top(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m,
                                          uint32_t mode, uint32_t presence, uint32_t k, double min_change,
                                          alz_node_change* out, size_t cap, size_t* n_out, alz_change_info* info) {
  return changes_entry<alz_node_change>(h, source, true, side, m, mode, presence, true, k, min_change, out, cap,
                                        nullptr, n_out, info);
}

extern "C" int alz_group_node_changes_top_device(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m,
                                                 uint32_t mode, uint32_t presence, uint32_t k, double min_change,
                                                 const alz_node_change** dev_out, size_t* n_out,
                                                 alz_change_info* info) {
  if (!dev_out) return n_out ? (*n_out = 0, ALZ_E_INVAL) : ALZ_E_INVAL;
  return changes_entry<alz_node_change>(h, source, true, side, m, mode, presence, true, k, min_change, nullptr, 0,
                                        dev_out, n_out, info);
}

extern "C" int alz_debug_group_edge_changes_rows(alz_handle* h, const alz_edge_out* dev_src, size_t n_src,
                                                 uint32_t src_windows, const alz_edge_out* dev_base, size_t n_base,
                                                 uint32_t base_windows, const alz_metric* m, uint32_t mode,
                                                 uint32_t presence, alz_edge_change* out, size_t cap, size_t* n_out,
                                                 alz_change_info* info) {
  if (!h || !n_out) return ALZ_E_INVAL;
  *n_out = 0;
  if (info) *info = alz_change_info{};
  MetricSet ms;
  if (!valid_change(ALZ_SIDE_IN, m, mode, presence, &ms) || (!out && cap) || (!dev_src && n_src) ||
      (!dev_base && n_base) || src_windows == 0 || base_windows == 0)
    return ALZ_E_INVAL;
  if (n_src > kMaxNodeSourceRows || n_base > kMaxNodeSourceRows) return ALZ_E_CAPACITY;
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  alz_group_changes_state* s = state(h);
  size_t edges_a = 0, edges_b = 0;
  alz_group_info gi;
  int rc = group_edges_into(h, s->src_edges, dev_src, n_src, SIZE_MAX, &edges_a, &gi);
  if (rc != ALZ_OK) return rc;
  rc = group_edges_into(h, s->hook_edges, dev_base, n_base, SIZE_MAX, &edges_b, &gi);
  if (rc != ALZ_OK) return rc;
  uint64_t listed = 0;
  alz_change_info ci{};
  rc = edge_change_join(h, s->j,
                        EdgeChangeSide{static_cast<const alz_edge_out*>(s->src_edges.p), nullptr, (uint32_t)edges_a,
                                       src_windows},
                        EdgeChangeSide{static_cast<const alz_edge_out*>(s->hook_edges.p), nullptr, (uint32_t)edges_b,
                                       base_windows},
                        true, ms, mode, presence, false, &listed, &ci);
  if (info) *info = ci;
  if (rc != ALZ_OK) return rc;
  *n_out = listed;
  if (listed > cap) return ALZ_E_CAPACITY;
  if (listed) CK(cudaMemcpyAsync(out, s->j.list.p, listed * sizeof(alz_edge_change), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return ALZ_OK;
}
