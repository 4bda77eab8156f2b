// alz_changes.cu — changes against a pinned baseline: a copy of a window's or rollup's rows kept on the handle, and the
// change list of a source against it on one of four levels: its edge rows (docs/SPEC.md §18), its §21 nodes on one
// side (§23), or its §24 group edges and group nodes under the map in force (§25). Each is one sorted join of two
// lists, each side's §17 metric values and one record per entry of the filtered union, or only its top entries by
// change.
//
// Both lists are strictly ascending by key, so the join needs no sort (DESIGN.md §5.10, §5.15, §5.17):
//   sides   edge calls: the source's rows and the baseline's. Node calls: the §21 group-by (alz_nodes.cu) of each, one
//           wait for each node count. Group calls: the §24 group-by (alz_groups.cu) of each, two waits, and for group
//           nodes the §21 group-by of those rows, one wait. The baseline's are derived on the first call that needs
//           them and kept: the pin's generation and the map's say when they are stale, so neither alz_baseline_pin
//           nor alz_group_set enqueues anything for them.
//   keys    an edge row's packed key (§3; the baseline's were stored when it was pinned), a group-edge row's (node key
//           of from, node key of to), a node row's head word (type << 32) | value and whether it has a row on the
//           side (member)
//   match   every entry of either list: lower_bound into the other list's keys, whether the key is there (for nodes:
//           as a member), and whether the entry is kept by the presence filter (a source entry: BOTH or NEW; a
//           baseline entry: GONE when unmatched, else it is listed through its source entry; a non-member: never)
//   scan    two exclusive scans of the keep flags. A kept source entry i goes to scanA[i] + scanG[lb_B(key_i)], a kept
//           gone baseline entry j to scanA[lb_A(key_j)] + scanG[j]: the tier merge's arithmetic (alz_rollup.cu)
//   values  the §17 metric kernels over each list's rows (for nodes, one side of each node: NodeRows)
//   emit    one 48-byte record per listed entry in three 16-byte stores, and for the top call its change into an
//           8-byte array, which the §17 selection ranks; the selected records are gathered by position
// Waits: the sides' above, one for the union's counts, and on a top call the selection's (alz_top.cu); a host call
// adds one for its copy. Growing a buffer adds one. The edge calls, the node calls and the group calls each own their
// join buffers, so none moves another's device results.
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <mutex>
#include <string>
#include <type_traits>

#include "alz_metrics.cuh"

using namespace alz;
using namespace alz::metrics;

static_assert(sizeof(alz_edge_change) == 48 && sizeof(alz_node_change) == 48,
              "a change record is three 16-byte stores");
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
// in a lower bound: the other list holds the key (for nodes: as a member); bounds are < 2^30
constexpr uint32_t kMatched = 0x80000000u;

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
// is listed by its own thread (keep_*[n] = 0 closes each scan); *both: the matched source nodes. A separate kernel
// from change_match_kernel: a non-member skips the search (DESIGN.md §5.15).
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

// A §18 side's value: COUNT and ERR5XX per window (one rounding), the others as they are
__device__ __forceinline__ double per_window(double v, bool divide, double windows) {
  return divide ? __ddiv_rn(v, windows) : v;
}
// The §18 change of mode from a source value and a baseline value, one rounding
__device__ __forceinline__ double change_of(uint32_t mode, double cur, double base) {
  if (mode == ALZ_CHANGE_DELTA) return __dsub_rn(cur, base);
  if (mode == ALZ_CHANGE_DROP) return __dsub_rn(base, cur);
  if (base > 0.0) return __ddiv_rn(cur, base);   // ALZ_CHANGE_RATIO
  return cur > 0.0 ? __longlong_as_double(0x7FF0000000000000ll) : 1.0;
}

// A record's first 16 bytes from its row's, without the presence: an edge row's types (its pad cleared), from and to
// (types, pad | from, to); a node row's type and value (type | value)
__device__ __forceinline__ uint4 head_of(const alz_edge_out* r) {
  const uint2 ty = reinterpret_cast<const uint2*>(r)[0], ft = reinterpret_cast<const uint2*>(r)[1];
  return make_uint4(ty.x & 0xFFFFu, 0u, ft.x, ft.y);
}
__device__ __forceinline__ uint4 head_of(const alz_node_out* r) {
  const uint2 tv = reinterpret_cast<const uint2*>(r)[0];
  return make_uint4(tv.x & 0xFFu, 0u, tv.y, 0u);
}

// the record of a join of edge rows (edge and group edge calls) or of node rows (node and group node calls)
template <class Row>
using RecordOf = std::conditional_t<std::is_same_v<Row, alz_node_out>, alz_node_change, alz_edge_change>;
template <class Record>
using RowOf = std::conditional_t<std::is_same_v<Record, alz_node_change>, alz_node_out, alz_edge_out>;

template <class Row>
struct EmitArgs {
  const Row* rows_a;
  const Row* rows_b;
  uint32_t n_a, n_b;
  const uint32_t *lb_a, *lb_b, *keep_a, *keep_b, *scan_a, *scan_b;
  const double *val_a, *val_b;
  double win_a, win_b;
  bool divide;
  uint32_t mode;
};

// one record per listed entry, written by the thread of its source entry (BOTH, NEW) or of its baseline entry (GONE);
// with chg, its change too
template <class Row>
__global__ void __launch_bounds__(256) change_emit_kernel(const __grid_constant__ EmitArgs<Row> a,
                                                          RecordOf<Row>* __restrict__ out,
                                                          uint64_t* __restrict__ chg) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < a.n_a + a.n_b; t += stride) {
    const bool src = t < a.n_a;
    const uint32_t i = src ? t : t - a.n_a;
    if (!(src ? a.keep_a[i] : a.keep_b[i])) continue;
    const uint32_t lb = src ? a.lb_a[i] : a.lb_b[i];
    const uint32_t p = lb & ~kMatched;
    const uint32_t pos = src ? a.scan_a[i] + a.scan_b[p] : a.scan_a[p] + a.scan_b[i];
    const uint4 head = head_of(src ? a.rows_a + i : a.rows_b + i);
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
    o[0] = make_uint4(head.x | (presence << 16), head.y, head.z, head.w);
    o[1] = make_uint4(index, base_index, (uint32_t)vb, (uint32_t)(vb >> 32));
    const uint64_t bb = (uint64_t)__double_as_longlong(base), cb = (uint64_t)__double_as_longlong(c);
    o[2] = make_uint4((uint32_t)bb, (uint32_t)(bb >> 32), (uint32_t)cb, (uint32_t)(cb >> 32));
    if (chg) chg[pos] = cb;
  }
}

// result j = the record at the j-th selected position
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

template <class T>
T* as(const DevBuf& b) {
  return static_cast<T*>(b.p);
}

// The keys of n rows into keys[n], on the stream
template <class Key>
void launch_keys(alz_handle* h, const alz_edge_out* rows, uint32_t n, Key* keys) {
  if (n == 0) return;
  change_keys_kernel<Key><<<grid_for(h, n, 8), 256, 0, h->stream>>>(rows, n, keys);
  h->launches += 1;
}

// The scratch and the results of one level's joins, grown on demand
struct ChangeBufs {
  DevBuf keys_a, keys_b, member_a, member_b;   // the sides' keys when derived; the node sides' membership
  DevBuf lb_a, lb_b, keep_a, keep_b, scan_a, scan_b, val_a, val_b, counts, tmp;   // the join's scratch
  DevBuf list, chg, top_list;                  // the results: the filtered union, its changes, the top records
  Selection sel;                               // the top call's selection
  void free() {
    free_bufs({&keys_a, &keys_b, &member_a, &member_b, &lb_a, &lb_b, &keep_a, &keep_b, &scan_a, &scan_b, &val_a,
               &val_b, &counts, &tmp, &list, &chg, &top_list});
    sel.free();
  }
};

}  // namespace

// The pinned baseline, what each level derives from it, and the buffers of the change calls, each grown on demand and
// never shrunk; freed in alz_destroy
struct alz_changes_state {
  DevBuf base_rows, base_keys;   // the baseline: its rows and their packed keys
  size_t base_n = 0;
  bool pinned = false;
  uint64_t generation = 0;       // pins so far: tells the cached baseline nodes and groups from a later pin's
  alz_rollup_info base_info{};
  // node calls: the group-by's scratch, the source's node rows and the baseline's (or the node hook's second list's)
  NodeGroup g;
  DevBuf src_nodes, base_nodes;
  size_t base_nodes_n = 0;
  bool nodes_cached = false;     // base_nodes hold the baseline of pin nodes_pin
  uint64_t nodes_pin = 0;
  // group calls: the source's group edges and group nodes, the baseline's, the group hook's second list's group edges
  DevBuf src_gedges, src_gnodes, base_gedges, base_gnodes, hook_gedges;
  size_t base_gedges_n = 0, base_gnodes_n = 0;
  bool gedges_cached = false;    // base_gedges hold the baseline of pin groups_pin grouped by map groups_map
  bool gnodes_cached = false;    // base_gnodes hold the group nodes of base_gedges
  uint64_t groups_pin = 0, groups_map = 0;
  ChangeBufs edges, nodes, groups;   // the joins of the edge calls, of the node calls and of both group calls
};

void alz_internal_free_changes(alz_handle* h) {
  alz_changes_state* s = h->changes;
  if (!s) return;
  s->g.free();
  free_bufs({&s->base_rows, &s->base_keys, &s->src_nodes, &s->base_nodes, &s->src_gedges, &s->src_gnodes,
             &s->base_gedges, &s->base_gnodes, &s->hook_gedges});
  s->edges.free();
  s->nodes.free();
  s->groups.free();
  delete s;
  h->changes = nullptr;
}

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
  launch_keys(h, rows, n, keys);
}

namespace {

enum Level : uint32_t { kEdges, kNodes, kGroupEdges, kGroupNodes };

// One change call: its level, the node side (node levels), the source, the metric, the mode and the presence filter,
// and for a top call k and min_change. device: the results stay on the device.
struct ChangeCall {
  Level level = kEdges;
  bool device = false, top = false;
  uint32_t side = ALZ_SIDE_IN, source = ALZ_SOURCE_WINDOW, mode = 0, presence = 0, k = 0;
  double min_change = 0.0;
  MetricSet ms{};
};

// allocated on first use; its buffers start empty
alz_changes_state* changes_state(alz_handle* h) {
  if (!h->changes) h->changes = new alz_changes_state();
  return h->changes;
}

// One list of a join: n edge rows or node rows strictly ascending in the join's key, the packed keys of edge rows when
// stored (null: derived), and the windows its values are divided by
template <class Row>
struct Side {
  const Row* rows;
  const uint64_t* keys;
  uint32_t n;
  uint32_t windows;
};

// An edge list's keys: its stored packed keys, or Key's derived into buf on the stream
template <class Key>
const Key* keys_of(alz_handle* h, const Side<alz_edge_out>& s, DevBuf& buf) {
  if constexpr (std::is_same_v<Key, uint64_t>) {
    if (s.keys) return s.keys;
  }
  launch_keys(h, s.rows, s.n, as<Key>(buf));
  return as<const Key>(buf);
}

// The keys and the match of edge lists, by packed key or (group edges) by ends: the matched source rows into counts[0]
template <class Key>
void match_rows(alz_handle* h, ChangeBufs& cb, const Side<alz_edge_out>& a, const Side<alz_edge_out>& b,
                uint32_t presence, unsigned grid) {
  const Key* ka = keys_of<Key>(h, a, cb.keys_a);
  const Key* kb = keys_of<Key>(h, b, cb.keys_b);
  change_match_kernel<Key><<<grid, 256, 0, h->stream>>>(ka, a.n, kb, b.n, presence, as<uint32_t>(cb.lb_a),
                                                        as<uint32_t>(cb.lb_b), as<uint32_t>(cb.keep_a),
                                                        as<uint32_t>(cb.keep_b), as<uint32_t>(cb.counts));
}
void match(alz_handle* h, ChangeBufs& cb, const ChangeCall& c, const Side<alz_edge_out>& a,
           const Side<alz_edge_out>& b, unsigned grid) {
  if (c.level == kGroupEdges)
    match_rows<EndsKey>(h, cb, a, b, c.presence, grid);
  else
    match_rows<uint64_t>(h, cb, a, b, c.presence, grid);
}
// The keys and the match of node lists: the members of a and of b into counts[0] and counts[1], the matched members
// into counts[2]
void match(alz_handle* h, ChangeBufs& cb, const ChangeCall& c, const Side<alz_node_out>& a,
           const Side<alz_node_out>& b, unsigned grid) {
  cudaStream_t st = h->stream;
  uint64_t* ka = as<uint64_t>(cb.keys_a);
  uint64_t* kb = as<uint64_t>(cb.keys_b);
  uint8_t* ma = as<uint8_t>(cb.member_a);
  uint8_t* mb = as<uint8_t>(cb.member_b);
  uint32_t* counts = as<uint32_t>(cb.counts);
  if (a.n) {
    node_change_keys_kernel<<<grid_for(h, a.n, 8), 256, 0, st>>>(a.rows, a.n, c.side, ka, ma, counts);
    h->launches += 1;
  }
  if (b.n) {
    node_change_keys_kernel<<<grid_for(h, b.n, 8), 256, 0, st>>>(b.rows, b.n, c.side, kb, mb, counts + 1);
    h->launches += 1;
  }
  node_change_match_kernel<<<grid, 256, 0, st>>>(ka, ma, a.n, kb, mb, b.n, c.presence, as<uint32_t>(cb.lb_a),
                                                 as<uint32_t>(cb.lb_b), as<uint32_t>(cb.keep_a),
                                                 as<uint32_t>(cb.keep_b), counts + 2);
}

// a list's §17 values: of its rows, or of one side of its nodes
int values_of(alz_handle* h, const ChangeCall& c, const Side<alz_edge_out>& s, DevBuf& out) {
  return run_metrics(h, s.rows, s.n, c.ms, as<double>(out));
}
int values_of(alz_handle* h, const ChangeCall& c, const Side<alz_node_out>& s, DevBuf& out) {
  return run_metrics_nodes(h, NodeRows{s.rows, c.side}, s.n, c.ms, as<double>(out));
}

// The join of a and b on c's level into cb.list, *listed records, and with c.top their changes into cb.chg. One wait.
// ci: the counts (above left 0). Caller holds h->mu and has set the device.
template <class Row>
int change_join(alz_handle* h, ChangeBufs& cb, const ChangeCall& c, const Side<Row>& a, const Side<Row>& b,
                uint64_t* listed, alz_change_info* ci) {
  constexpr bool nodes = std::is_same_v<Row, alz_node_out>;
  constexpr size_t count_bytes = nodes ? 3 * 4 : 4;   // see match
  cudaStream_t st = h->stream;
  const size_t na = a.n, nb = b.n;
  const size_t key_bytes = c.level == kGroupEdges ? sizeof(EndsKey) : 8;
  int rc = reserve(h, {{&cb.keys_a, a.keys ? 0 : std::max<size_t>(na, 1) * key_bytes},
                       {&cb.keys_b, b.keys ? 0 : std::max<size_t>(nb, 1) * key_bytes},
                       {&cb.member_a, nodes ? std::max<size_t>(na, 1) : 0},
                       {&cb.member_b, nodes ? std::max<size_t>(nb, 1) : 0},
                       {&cb.lb_a, std::max<size_t>(na, 1) * 4},
                       {&cb.lb_b, std::max<size_t>(nb, 1) * 4},
                       {&cb.keep_a, (na + 1) * 4},
                       {&cb.keep_b, (nb + 1) * 4},
                       {&cb.scan_a, (na + 1) * 4},
                       {&cb.scan_b, (nb + 1) * 4},
                       {&cb.val_a, std::max<size_t>(na, 1) * 8},
                       {&cb.val_b, std::max<size_t>(nb, 1) * 8},
                       {&cb.counts, count_bytes},
                       {&cb.tmp, scan_temp_bytes((uint32_t)std::max(na, nb) + 1)}});
  if (rc != ALZ_OK) return rc;
  const uint32_t* scan_a = as<uint32_t>(cb.scan_a);
  const uint32_t* scan_b = as<uint32_t>(cb.scan_b);
  CK(cudaMemsetAsync(cb.counts.p, 0, count_bytes, st));
  const unsigned grid = grid_for(h, na + nb, 8);   // each list is below 2^30
  match(h, cb, c, a, b, grid);
  h->launches += 1;
  CK(exclusive_scan_u32(cb.tmp.p, cb.tmp.bytes, as<uint32_t>(cb.keep_a), as<uint32_t>(cb.scan_a), a.n + 1, st));
  CK(exclusive_scan_u32(cb.tmp.p, cb.tmp.bytes, as<uint32_t>(cb.keep_b), as<uint32_t>(cb.scan_b), b.n + 1, st));
  rc = values_of(h, c, a, cb.val_a);
  if (rc != ALZ_OK) return rc;
  rc = values_of(h, c, b, cb.val_b);
  if (rc != ALZ_OK) return rc;
  CK(cudaGetLastError());
  // listed source entries, listed gone entries, members of a, members of b (every row of an edge list), matched members
  uint32_t cnt[5] = {0, 0, a.n, b.n, 0};
  CK(cudaMemcpyAsync(&cnt[0], scan_a + a.n, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(&cnt[1], scan_b + b.n, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(nodes ? &cnt[2] : &cnt[4], cb.counts.p, count_bytes, cudaMemcpyDeviceToHost, st));
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
  rc = reserve(h, {{&cb.list, std::max<size_t>(*listed, 1) * sizeof(RecordOf<Row>)},
                   {&cb.chg, c.top ? std::max<size_t>(*listed, 1) * 8 : 0}});
  if (rc != ALZ_OK) return rc;
  if (*listed) {
    const bool divide = c.ms.kind[0] == ALZ_METRIC_COUNT || c.ms.kind[0] == ALZ_METRIC_ERR5XX;
    const EmitArgs<Row> ea{a.rows, b.rows, a.n, b.n, as<uint32_t>(cb.lb_a), as<uint32_t>(cb.lb_b),
                           as<uint32_t>(cb.keep_a), as<uint32_t>(cb.keep_b), scan_a, scan_b,
                           as<double>(cb.val_a), as<double>(cb.val_b), (double)a.windows, (double)b.windows,
                           divide, c.mode};
    change_emit_kernel<Row><<<grid, 256, 0, st>>>(ea, as<RecordOf<Row>>(cb.list),
                                                  c.top ? as<uint64_t>(cb.chg) : nullptr);
    h->launches += 1;
    CK(cudaGetLastError());
  }
  return ALZ_OK;
}

// After a join into cb: the listed records in cb.list (a list call), or the first min(k, above) of them by change
// gathered into cb.top_list (a top call, ci->above set). *res, *n = the records. Caller holds h->mu.
template <class Record>
int change_results(alz_handle* h, ChangeBufs& cb, const ChangeCall& c, uint64_t listed, const Record** res, size_t* n,
                   alz_change_info* ci) {
  if (!c.top) {
    *res = as<const Record>(cb.list);
    *n = listed;
    return ALZ_OK;
  }
  size_t m = 0;
  uint64_t above = 0;
  int rc = select_top(h, cb.sel, as<const uint64_t>(cb.chg), (uint32_t)listed, c.k, c.min_change, nullptr, &m, &above);
  if (rc != ALZ_OK) return rc;
  ci->above = above;
  rc = reserve(h, {{&cb.top_list, std::max<size_t>(m, 1) * sizeof(Record)}});
  if (rc != ALZ_OK) return rc;
  if (m) {
    change_gather_kernel<<<grid_for(h, 3ull * m, 4), 256, 0, h->stream>>>(
        as<const uint32_t>(cb.sel.top_index), (uint32_t)m, as<const Record>(cb.list), as<Record>(cb.top_list));
    h->launches += 1;
    CK(cudaGetLastError());
  }
  *res = as<const Record>(cb.top_list);
  *n = m;
  return ALZ_OK;
}

// The rows a node call (level kNodes: §21 node rows) or a group call (kGroupEdges: §24 group-edge rows) derives from n
// edge rows, into out; *n_out of them. Caller holds h->mu and has set the device; n <= kMaxNodeSourceRows.
int derive(alz_handle* h, alz_changes_state* s, Level level, const alz_edge_out* rows, size_t n, DevBuf& out,
           size_t* n_out) {
  if (level == kNodes) return node_rows_of(h, s->g, out, rows, n, SIZE_MAX, n_out);
  alz_group_info gi;
  return group_edges_into(h, out, rows, n, SIZE_MAX, n_out, &gi);
}

// What `level` derives from the pinned baseline, derived again only when the pin or (group levels) the map moved on:
// its node rows, or its group edges and for group nodes their group nodes
int cached_base(alz_handle* h, alz_changes_state* s, Level level) {
  const alz_edge_out* rows = as<const alz_edge_out>(s->base_rows);
  if (level == kNodes) {
    if (s->nodes_cached && s->nodes_pin == s->generation) return ALZ_OK;
    s->nodes_cached = false;   // a failure below leaves no cached baseline nodes
    const int rc = derive(h, s, kNodes, rows, s->base_n, s->base_nodes, &s->base_nodes_n);
    if (rc != ALZ_OK) return rc;
    s->nodes_cached = true;
    s->nodes_pin = s->generation;
    return ALZ_OK;
  }
  const uint64_t map_gen = group_map_generation(h);
  if (!s->gedges_cached || s->groups_pin != s->generation || s->groups_map != map_gen) {
    s->gedges_cached = s->gnodes_cached = false;   // a failure below leaves nothing cached
    const int rc = derive(h, s, kGroupEdges, rows, s->base_n, s->base_gedges, &s->base_gedges_n);
    if (rc != ALZ_OK) return rc;
    s->gedges_cached = true;
    s->groups_pin = s->generation;
    s->groups_map = map_gen;
  }
  if (level == kGroupNodes && !s->gnodes_cached) {
    const int rc = group_nodes_into(h, s->base_gnodes, as<const alz_edge_out>(s->base_gedges), s->base_gedges_n,
                                    &s->base_gnodes_n);
    if (rc != ALZ_OK) return rc;
    s->gnodes_cached = true;
  }
  return ALZ_OK;
}

// The lists an edge or group edge call joins: the source's rows and the baseline's with its stored keys, or the
// group edges of each
int sides_of(alz_handle* h, alz_changes_state* s, const ChangeCall& c, const Side<alz_edge_out>& src,
             Side<alz_edge_out>* a, Side<alz_edge_out>* b) {
  const uint32_t base_windows = s->base_info.windows;
  if (c.level == kEdges) {
    *a = src;
    *b = {as<const alz_edge_out>(s->base_rows), as<const uint64_t>(s->base_keys), (uint32_t)s->base_n, base_windows};
    return ALZ_OK;
  }
  size_t n = 0;
  int rc = derive(h, s, kGroupEdges, src.rows, src.n, s->src_gedges, &n);
  if (rc != ALZ_OK) return rc;
  rc = cached_base(h, s, kGroupEdges);
  if (rc != ALZ_OK) return rc;
  *a = {as<const alz_edge_out>(s->src_gedges), nullptr, (uint32_t)n, src.windows};
  *b = {as<const alz_edge_out>(s->base_gedges), nullptr, (uint32_t)s->base_gedges_n, base_windows};
  return ALZ_OK;
}
// The lists a node or group node call joins: the node rows of the source's rows and of the baseline's, or of the
// group edges of each
int sides_of(alz_handle* h, alz_changes_state* s, const ChangeCall& c, const Side<alz_edge_out>& src,
             Side<alz_node_out>* a, Side<alz_node_out>* b) {
  const uint32_t base_windows = s->base_info.windows;
  size_t n = 0;
  if (c.level == kNodes) {
    int rc = derive(h, s, kNodes, src.rows, src.n, s->src_nodes, &n);
    if (rc != ALZ_OK) return rc;
    rc = cached_base(h, s, kNodes);
    if (rc != ALZ_OK) return rc;
    *a = {as<const alz_node_out>(s->src_nodes), nullptr, (uint32_t)n, src.windows};
    *b = {as<const alz_node_out>(s->base_nodes), nullptr, (uint32_t)s->base_nodes_n, base_windows};
    return ALZ_OK;
  }
  size_t edges = 0;
  int rc = derive(h, s, kGroupEdges, src.rows, src.n, s->src_gedges, &edges);
  if (rc != ALZ_OK) return rc;
  rc = cached_base(h, s, kGroupNodes);
  if (rc != ALZ_OK) return rc;
  rc = group_nodes_into(h, s->src_gnodes, as<const alz_edge_out>(s->src_gedges), edges, &n);
  if (rc != ALZ_OK) return rc;
  *a = {as<const alz_node_out>(s->src_gnodes), nullptr, (uint32_t)n, src.windows};
  *b = {as<const alz_node_out>(s->base_gnodes), nullptr, (uint32_t)s->base_gnodes_n, base_windows};
  return ALZ_OK;
}

ChangeBufs& bufs_of(alz_changes_state* s, Level level) {
  return level == kEdges ? s->edges : level == kNodes ? s->nodes : s->groups;
}

// edge and group edge calls read sources of at most kMaxRows rows, node and group node calls kMaxNodeSourceRows
size_t row_limit(Level level) { return level == kEdges ? kMaxRows : kMaxNodeSourceRows; }

// The change list of c.source against the baseline on c's level (top: its first min(k, above) records by change) in
// that level's buffers; *n = records. Caller holds h->mu.
template <class Record>
int changes_locked(alz_handle* h, const ChangeCall& c, const Record** res, size_t* n, alz_change_info* ci) {
  CK(cudaSetDevice(h->device));
  const alz_edge_out* rows = nullptr;
  size_t n_src = 0;
  alz_rollup_info ri;
  int rc = source_rows(h, c.source, &rows, &n_src, &ri);
  if (rc != ALZ_OK) return rc;
  alz_changes_state* s = h->changes;
  if (!s->pinned) return ALZ_E_STATE;
  if (n_src > row_limit(c.level) || s->base_n > row_limit(c.level)) return ALZ_E_CAPACITY;
  Side<RowOf<Record>> a, b;
  rc = sides_of(h, s, c, Side<alz_edge_out>{rows, nullptr, (uint32_t)n_src, ri.windows}, &a, &b);
  if (rc != ALZ_OK) return rc;
  ChangeBufs& cb = bufs_of(s, c.level);
  uint64_t listed = 0;
  rc = change_join(h, cb, c, a, b, &listed, ci);
  if (rc != ALZ_OK) return rc;
  return change_results(h, cb, c, listed, res, n, ci);
}

// c's arguments are valid (the side only on the node levels); *c.ms the metric's kernel form
bool valid_change(ChangeCall* c, const alz_metric* m) {
  const bool node_level = c->level == kNodes || c->level == kGroupNodes;
  return (!node_level || c->side <= ALZ_SIDE_OUT) && valid_metrics(m, 1, &c->ms) && c->mode <= ALZ_CHANGE_RATIO &&
         c->presence != 0 && c->presence <= 7u;
}

// The 16 entry points: device (c.device, *dev_out required) or host (cap records in out, one more wait for the copy)
template <class Record>
int changes_entry(alz_handle* h, ChangeCall c, const alz_metric* m, Record* out, size_t cap, const Record** dev_out,
                  size_t* n_out, alz_change_info* info) {
  if (c.device && !dev_out) return n_out ? (*n_out = 0, ALZ_E_INVAL) : ALZ_E_INVAL;
  if (!h || !n_out) return ALZ_E_INVAL;
  *n_out = 0;
  if (info) *info = alz_change_info{};
  if (!valid_change(&c, m) || (!dev_out && !out && cap)) return ALZ_E_INVAL;
  if (c.source != ALZ_SOURCE_WINDOW && c.source > ALZ_ROLLUP_SPAN) return ALZ_E_INVAL;
  if (c.top && (c.k == 0 || std::isnan(c.min_change))) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  changes_state(h);
  const Record* res = nullptr;
  size_t n = 0;
  alz_change_info ci{};
  const int rc = changes_locked(h, c, &res, &n, &ci);
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

ChangeCall call_of(Level level, bool device, bool top, uint32_t source, uint32_t side, uint32_t mode,
                   uint32_t presence, uint32_t k = 0, double min_change = 0.0) {
  return ChangeCall{level, device, top, side, source, mode, presence, k, min_change};
}

// The three hooks: the join of two caller row lists on c's level, the list copied to the host. The node hook groups
// both into the node calls' buffers (the cached baseline nodes go stale), the group hook into the source's group
// edges and a buffer of its own, so the cached baseline groups stay.
template <class Record>
int debug_rows(alz_handle* h, ChangeCall c, const alz_edge_out* dev_src, size_t n_src, uint32_t src_windows,
               const alz_edge_out* dev_base, size_t n_base, uint32_t base_windows, const alz_metric* m, Record* out,
               size_t cap, size_t* n_out, alz_change_info* info) {
  if (!h || !n_out) return ALZ_E_INVAL;
  *n_out = 0;
  if (info) *info = alz_change_info{};
  if (!valid_change(&c, m) || (!out && cap) || (!dev_src && n_src) || (!dev_base && n_base) || src_windows == 0 ||
      base_windows == 0)
    return ALZ_E_INVAL;
  if (n_src > row_limit(c.level) || n_base > row_limit(c.level)) return ALZ_E_CAPACITY;
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  alz_changes_state* s = changes_state(h);
  using Row = RowOf<Record>;
  Side<Row> a{nullptr, nullptr, (uint32_t)n_src, src_windows}, b{nullptr, nullptr, (uint32_t)n_base, base_windows};
  if constexpr (std::is_same_v<Row, alz_edge_out>) {
    a.rows = dev_src;
    b.rows = dev_base;
  }
  if (c.level != kEdges) {
    if (c.level == kNodes) s->nodes_cached = false;   // base_nodes take the hook's second list
    DevBuf& out_a = c.level == kNodes ? s->src_nodes : s->src_gedges;
    DevBuf& out_b = c.level == kNodes ? s->base_nodes : s->hook_gedges;
    size_t na = 0, nb = 0;
    int rc = derive(h, s, c.level, dev_src, n_src, out_a, &na);
    if (rc != ALZ_OK) return rc;
    rc = derive(h, s, c.level, dev_base, n_base, out_b, &nb);
    if (rc != ALZ_OK) return rc;
    a = {as<const Row>(out_a), nullptr, (uint32_t)na, src_windows};
    b = {as<const Row>(out_b), nullptr, (uint32_t)nb, base_windows};
  }
  ChangeBufs& cb = bufs_of(s, c.level);
  uint64_t listed = 0;
  alz_change_info ci{};
  const int rc = change_join(h, cb, c, a, b, &listed, &ci);
  if (info) *info = ci;
  if (rc != ALZ_OK) return rc;
  *n_out = listed;
  if (listed > cap) return ALZ_E_CAPACITY;
  if (listed) CK(cudaMemcpyAsync(out, cb.list.p, listed * sizeof(Record), cudaMemcpyDeviceToHost, h->stream));
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
    launch_row_keys(h, as<const alz_edge_out>(s->base_rows), (uint32_t)n, as<uint64_t>(s->base_keys));
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
  return changes_entry<alz_edge_change>(h, call_of(kEdges, false, false, source, ALZ_SIDE_IN, mode, presence), m, out,
                                        cap, nullptr, n_out, info);
}

extern "C" int alz_edge_changes_device(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode,
                                       uint32_t presence, const alz_edge_change** dev_out, size_t* n_out,
                                       alz_change_info* info) {
  return changes_entry<alz_edge_change>(h, call_of(kEdges, true, false, source, ALZ_SIDE_IN, mode, presence), m,
                                        nullptr, 0, dev_out, n_out, info);
}

extern "C" int alz_edge_changes_top(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode,
                                    uint32_t presence, uint32_t k, double min_change, alz_edge_change* out, size_t cap,
                                    size_t* n_out, alz_change_info* info) {
  return changes_entry<alz_edge_change>(
      h, call_of(kEdges, false, true, source, ALZ_SIDE_IN, mode, presence, k, min_change), m, out, cap, nullptr,
      n_out, info);
}

extern "C" int alz_edge_changes_top_device(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode,
                                           uint32_t presence, uint32_t k, double min_change,
                                           const alz_edge_change** dev_out, size_t* n_out, alz_change_info* info) {
  return changes_entry<alz_edge_change>(
      h, call_of(kEdges, true, true, source, ALZ_SIDE_IN, mode, presence, k, min_change), m, nullptr, 0, dev_out,
      n_out, info);
}

extern "C" int alz_node_changes(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t mode,
                                uint32_t presence, alz_node_change* out, size_t cap, size_t* n_out,
                                alz_change_info* info) {
  return changes_entry<alz_node_change>(h, call_of(kNodes, false, false, source, side, mode, presence), m, out, cap,
                                        nullptr, n_out, info);
}

extern "C" int alz_node_changes_device(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m,
                                       uint32_t mode, uint32_t presence, const alz_node_change** dev_out,
                                       size_t* n_out, alz_change_info* info) {
  return changes_entry<alz_node_change>(h, call_of(kNodes, true, false, source, side, mode, presence), m, nullptr, 0,
                                        dev_out, n_out, info);
}

extern "C" int alz_node_changes_top(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t mode,
                                    uint32_t presence, uint32_t k, double min_change, alz_node_change* out,
                                    size_t cap, size_t* n_out, alz_change_info* info) {
  return changes_entry<alz_node_change>(h, call_of(kNodes, false, true, source, side, mode, presence, k, min_change),
                                        m, out, cap, nullptr, n_out, info);
}

extern "C" int alz_node_changes_top_device(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m,
                                           uint32_t mode, uint32_t presence, uint32_t k, double min_change,
                                           const alz_node_change** dev_out, size_t* n_out, alz_change_info* info) {
  return changes_entry<alz_node_change>(h, call_of(kNodes, true, true, source, side, mode, presence, k, min_change),
                                        m, nullptr, 0, dev_out, n_out, info);
}

extern "C" int alz_group_edge_changes(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode,
                                      uint32_t presence, alz_edge_change* out, size_t cap, size_t* n_out,
                                      alz_change_info* info) {
  return changes_entry<alz_edge_change>(h, call_of(kGroupEdges, false, false, source, ALZ_SIDE_IN, mode, presence),
                                        m, out, cap, nullptr, n_out, info);
}

extern "C" int alz_group_edge_changes_device(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode,
                                             uint32_t presence, const alz_edge_change** dev_out, size_t* n_out,
                                             alz_change_info* info) {
  return changes_entry<alz_edge_change>(h, call_of(kGroupEdges, true, false, source, ALZ_SIDE_IN, mode, presence),
                                        m, nullptr, 0, dev_out, n_out, info);
}

extern "C" int alz_group_edge_changes_top(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode,
                                          uint32_t presence, uint32_t k, double min_change, alz_edge_change* out,
                                          size_t cap, size_t* n_out, alz_change_info* info) {
  return changes_entry<alz_edge_change>(
      h, call_of(kGroupEdges, false, true, source, ALZ_SIDE_IN, mode, presence, k, min_change), m, out, cap, nullptr,
      n_out, info);
}

extern "C" int alz_group_edge_changes_top_device(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode,
                                                 uint32_t presence, uint32_t k, double min_change,
                                                 const alz_edge_change** dev_out, size_t* n_out,
                                                 alz_change_info* info) {
  return changes_entry<alz_edge_change>(
      h, call_of(kGroupEdges, true, true, source, ALZ_SIDE_IN, mode, presence, k, min_change), m, nullptr, 0, dev_out,
      n_out, info);
}

extern "C" int alz_group_node_changes(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m,
                                      uint32_t mode, uint32_t presence, alz_node_change* out, size_t cap,
                                      size_t* n_out, alz_change_info* info) {
  return changes_entry<alz_node_change>(h, call_of(kGroupNodes, false, false, source, side, mode, presence), m, out,
                                        cap, nullptr, n_out, info);
}

extern "C" int alz_group_node_changes_device(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m,
                                             uint32_t mode, uint32_t presence, const alz_node_change** dev_out,
                                             size_t* n_out, alz_change_info* info) {
  return changes_entry<alz_node_change>(h, call_of(kGroupNodes, true, false, source, side, mode, presence), m,
                                        nullptr, 0, dev_out, n_out, info);
}

extern "C" int alz_group_node_changes_top(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m,
                                          uint32_t mode, uint32_t presence, uint32_t k, double min_change,
                                          alz_node_change* out, size_t cap, size_t* n_out, alz_change_info* info) {
  return changes_entry<alz_node_change>(
      h, call_of(kGroupNodes, false, true, source, side, mode, presence, k, min_change), m, out, cap, nullptr, n_out,
      info);
}

extern "C" int alz_group_node_changes_top_device(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m,
                                                 uint32_t mode, uint32_t presence, uint32_t k, double min_change,
                                                 const alz_node_change** dev_out, size_t* n_out,
                                                 alz_change_info* info) {
  return changes_entry<alz_node_change>(
      h, call_of(kGroupNodes, true, true, source, side, mode, presence, k, min_change), m, nullptr, 0, dev_out, n_out,
      info);
}

extern "C" int alz_debug_edge_changes_rows(alz_handle* h, const alz_edge_out* dev_src, size_t n_src,
                                           uint32_t src_windows, const alz_edge_out* dev_base, size_t n_base,
                                           uint32_t base_windows, const alz_metric* m, uint32_t mode,
                                           uint32_t presence, alz_edge_change* out, size_t cap, size_t* n_out,
                                           alz_change_info* info) {
  return debug_rows(h, call_of(kEdges, false, false, ALZ_SOURCE_WINDOW, ALZ_SIDE_IN, mode, presence), dev_src, n_src,
                    src_windows, dev_base, n_base, base_windows, m, out, cap, n_out, info);
}

extern "C" int alz_debug_node_changes_rows(alz_handle* h, const alz_edge_out* dev_src, size_t n_src,
                                           uint32_t src_windows, const alz_edge_out* dev_base, size_t n_base,
                                           uint32_t base_windows, uint32_t side, const alz_metric* m, uint32_t mode,
                                           uint32_t presence, alz_node_change* out, size_t cap, size_t* n_out,
                                           alz_change_info* info) {
  return debug_rows(h, call_of(kNodes, false, false, ALZ_SOURCE_WINDOW, side, mode, presence), dev_src, n_src,
                    src_windows, dev_base, n_base, base_windows, m, out, cap, n_out, info);
}

extern "C" int alz_debug_group_edge_changes_rows(alz_handle* h, const alz_edge_out* dev_src, size_t n_src,
                                                 uint32_t src_windows, const alz_edge_out* dev_base, size_t n_base,
                                                 uint32_t base_windows, const alz_metric* m, uint32_t mode,
                                                 uint32_t presence, alz_edge_change* out, size_t cap, size_t* n_out,
                                                 alz_change_info* info) {
  return debug_rows(h, call_of(kGroupEdges, false, false, ALZ_SOURCE_WINDOW, ALZ_SIDE_IN, mode, presence), dev_src,
                    n_src, src_windows, dev_base, n_base, base_windows, m, out, cap, n_out, info);
}
