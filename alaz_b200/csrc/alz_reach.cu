// alz_reach.cu — reach (docs/SPEC.md §27): a hop-bounded breadth-first search over a source's rows (node form) or its
// §24 group-edge rows (group form) from chosen seed nodes, with the nodes, their hops, one shortest-path parent and row
// each, and the rows the search crossed. Reads the source rows only; every buffer written is this state's, or scratch
// of the group calls (group_edges_into), so no other family's results move.
//
//   group    group form: group_edges_into (two waits) into this state's rows first. Then node_group_keys /
//            node_group_runs over the traversed rows (the §21 sort of the 2n ends, heads and scan, one wait); the
//            index kernel scatters each sorted end's node index back to its row end through vals_out (pair 2i: row
//            i's to end, 2i + 1: its from end) and writes each node's key at its index
//   seeds    uploaded as packed keys; each is binary-searched among the node keys and marks hops = 0 where found
//   filter   with a metric, run_metrics over the traversed rows, then a row is traversable when the order key of its
//            value is at least the order key of min_value (§17's eligibility rule)
//   adjacency a CSR by tail over the traversable rows: count per node (atomicAdd), exclusive scan, fill (atomicAdd
//            cursors: the order inside a list is arbitrary and does not reach the result). ANY lists a row under both
//            ends. An entry is (head node << 32) | row.
//   levels   frontier l is a run of the result list, in node order. Its degrees are scanned, and the expand runs one
//            thread per adjacency entry, found by a binary search in that scan, so a hub's list is spread over the
//            grid. Each entry u -> v with v unreached does atomicMin(best[v], (u << 32) | row): the smallest parent
//            index, then the smallest row from it. The discover kernel sets hops = l + 1 where best was set, and a
//            flag, scan and scatter appends frontier l + 1 in node order. One read per level (the next frontier's size and
//            adjacency entries, which size its expand) ends the loop at the first empty frontier or at max_hops.
//   rows     one pass flags the listed rows (traversable, tail hops < max_hops) and counts the cut; a scan and scatter
//            lists their positions, and the top calls' gather copies the rows
//   emit     one kernel writes the node records; parent maps best >> 32 through the node -> result position scatter
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "alz_metrics.cuh"
#include "alz_top.cuh"

using namespace alz;
using namespace alz::metrics;

static_assert(sizeof(alz_reach_node) == 24 && offsetof(alz_reach_node, value) == 4 &&
                  offsetof(alz_reach_node, hops) == 8 && offsetof(alz_reach_node, index) == 12 &&
                  offsetof(alz_reach_node, parent) == 16 && offsetof(alz_reach_node, row) == 20,
              "alz_reach_node is six u32 words, the first two an alz_node_ends");
static_assert(sizeof(alz_reach_info) == 48, "alz_reach_info is six u64");
static_assert(sizeof(alz_node_ends) == 8 && offsetof(alz_node_ends, value) == 4, "a seed is (type, value)");

namespace {

constexpr uint32_t kUnreached = 0xFFFFFFFFu;
constexpr uint64_t kNoBest = ~0ull;
constexpr uint32_t kMaxSeeds = (1u << 30) - 1u;

// j over the n2 sorted ends: end_node[vals[j]] = the node index of j's run; node_keys[index] = its key at a run head
__global__ void __launch_bounds__(256) reach_index_kernel(const uint64_t* __restrict__ keys,
                                                          const uint32_t* __restrict__ vals,
                                                          const uint32_t* __restrict__ heads,
                                                          const uint32_t* __restrict__ idx, uint32_t n2,
                                                          uint32_t* __restrict__ end_node,
                                                          uint64_t* __restrict__ node_keys) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n2; j += stride) {
    const uint32_t head = heads[j], node = idx[j] + head - 1u;   // idx is the exclusive scan of the heads
    end_node[vals[j]] = node;
    if (head) node_keys[node] = keys[j];
  }
}

// hops[node] = 0 for each seed that is a node
__global__ void __launch_bounds__(256) reach_seed_kernel(const uint64_t* __restrict__ seeds, uint32_t ns,
                                                         const uint64_t* __restrict__ node_keys, uint32_t nodes,
                                                         uint32_t* __restrict__ hops) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < ns; i += stride) {
    const uint64_t key = seeds[i];
    uint32_t lo = 0, hi = nodes;
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if (node_keys[mid] < key) lo = mid + 1; else hi = mid;
    }
    if (lo < nodes && node_keys[lo] == key) hops[lo] = 0u;
  }
}

// the node indices of row r's ends: .x its to end's, .y its from end's
__device__ __forceinline__ uint2 row_ends(const uint32_t* __restrict__ end_node, uint32_t r) {
  return reinterpret_cast<const uint2*>(end_node)[r];
}

// trav[r]: row r is traversable (no metric: every row; else key(value) >= min_key); cnt[tail] += 1 per orientation
// the direction follows
__global__ void __launch_bounds__(256) reach_count_kernel(const uint32_t* __restrict__ end_node, uint32_t n,
                                                          uint32_t dir, const uint64_t* __restrict__ vals,
                                                          uint64_t min_key, uint8_t* __restrict__ trav,
                                                          uint32_t* __restrict__ cnt) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) {
    const bool t = !vals || top::order_key(vals[r]) >= min_key;
    trav[r] = t ? 1u : 0u;
    if (!t) continue;
    const uint2 e = row_ends(end_node, r);
    if (dir != ALZ_REACH_UP) atomicAdd(cnt + e.y, 1u);     // from -> to
    if (dir != ALZ_REACH_DOWN) atomicAdd(cnt + e.x, 1u);   // to -> from
  }
}

// adj[cursor[tail]++] = (head << 32) | r for each orientation of each traversable row
__global__ void __launch_bounds__(256) reach_fill_kernel(const uint32_t* __restrict__ end_node, uint32_t n,
                                                         uint32_t dir, const uint8_t* __restrict__ trav,
                                                         uint32_t* __restrict__ cursor,
                                                         uint64_t* __restrict__ adj) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) {
    if (!trav[r]) continue;
    const uint2 e = row_ends(end_node, r);
    if (dir != ALZ_REACH_UP) adj[atomicAdd(cursor + e.y, 1u)] = ((uint64_t)e.x << 32) | r;
    if (dir != ALZ_REACH_DOWN) adj[atomicAdd(cursor + e.x, 1u)] = ((uint64_t)e.y << 32) | r;
  }
}

// flag[v] = 1 for the nodes of level `level`: level 0 the seeds found; else the unreached nodes an expand reached,
// which get hops = level. *entries += the adjacency entries of the flagged nodes, which size the next expand's grid.
// flag[nodes] = 0 closes the scan.
__global__ void __launch_bounds__(256) reach_discover_kernel(const uint64_t* __restrict__ best, uint32_t nodes,
                                                             uint32_t level, const uint32_t* __restrict__ adj_off,
                                                             uint32_t* __restrict__ hops,
                                                             uint32_t* __restrict__ flag,
                                                             uint32_t* __restrict__ entries) {
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31u;
  for (uint32_t base = t0 - lane; base < nodes; base += stride) {   // whole warps: the entries are summed per warp
    const uint32_t v = base + lane;
    uint32_t d = 0;
    if (v < nodes) {
      bool f;
      if (level == 0) {
        f = hops[v] == 0u;
      } else {
        f = hops[v] == kUnreached && best[v] != kNoBest;
        if (f) hops[v] = level;
      }
      flag[v] = f ? 1u : 0u;
      if (f) d = adj_off[v + 1] - adj_off[v];
    }
    d = __reduce_add_sync(0xFFFFFFFFu, d);
    if (lane == 0 && d) atomicAdd(entries, d);
  }
  if (t0 == 0) flag[nodes] = 0u;
}

// order[base + scan[v]] = v and pos[v] = base + scan[v] for the flagged v
__global__ void __launch_bounds__(256) reach_scatter_kernel(const uint32_t* __restrict__ flag,
                                                            const uint32_t* __restrict__ scan, uint32_t n,
                                                            uint32_t base, uint32_t* __restrict__ order,
                                                            uint32_t* __restrict__ pos) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += stride) {
    if (!flag[v]) continue;
    const uint32_t p = base + scan[v];
    order[p] = v;
    if (pos) pos[v] = p;
  }
}

// deg[i] = the adjacency list length of frontier node i; deg[s] = 0 closes the scan
__global__ void __launch_bounds__(256) reach_degree_kernel(const uint32_t* __restrict__ frontier, uint32_t s,
                                                           const uint32_t* __restrict__ adj_off,
                                                           uint32_t* __restrict__ deg) {
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x;
  for (uint32_t i = t0; i < s; i += stride) {
    const uint32_t u = frontier[i];
    deg[i] = adj_off[u + 1] - adj_off[u];
  }
  if (t0 == 0) deg[s] = 0u;
}

// One thread per adjacency entry of the frontier (dscan[s] of them): entry t belongs to the frontier node i with
// dscan[i] <= t < dscan[i + 1]. An unreached head takes the smallest (tail index << 32) | row.
__global__ void __launch_bounds__(256) reach_expand_kernel(const uint32_t* __restrict__ frontier, uint32_t s,
                                                           const uint32_t* __restrict__ dscan,
                                                           const uint32_t* __restrict__ adj_off,
                                                           const uint64_t* __restrict__ adj,
                                                           const uint32_t* __restrict__ hops,
                                                           unsigned long long* __restrict__ best) {
  const uint32_t total = dscan[s];
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
    uint32_t lo = 0, hi = s;   // the last i with dscan[i] <= t
    while (hi - lo > 1u) {
      const uint32_t mid = (lo + hi) >> 1;
      if (dscan[mid] <= t) lo = mid; else hi = mid;
    }
    const uint32_t u = frontier[lo];
    const uint64_t e = adj[adj_off[u] + (t - dscan[lo])];
    const uint32_t v = (uint32_t)(e >> 32);
    if (hops[v] != kUnreached) continue;
    const unsigned long long cand = ((unsigned long long)u << 32) | (uint32_t)e;
    if (cand < best[v]) atomicMin(best + v, cand);
  }
}

// flag[r] = 1 for the listed rows (traversable, tail hops < max_hops); *cut += the traversable rows from a node at
// max_hops to an unreached one. flag[n] = 0 closes the scan.
__global__ void __launch_bounds__(256) reach_rows_kernel(const uint32_t* __restrict__ end_node, uint32_t n,
                                                         uint32_t dir, const uint8_t* __restrict__ trav,
                                                         const uint32_t* __restrict__ hops, uint32_t max_hops,
                                                         uint32_t* __restrict__ flag,
                                                         unsigned long long* __restrict__ cut) {
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31u;
  for (uint32_t base = t0 - lane; base < n; base += stride) {   // whole warps: the cut is summed by ballot
    const uint32_t r = base + lane;
    bool listed = false, c = false;
    if (r < n && trav[r]) {
      const uint2 e = row_ends(end_node, r);
      const uint32_t hf = hops[e.y], ht = hops[e.x];
      const bool down = dir != ALZ_REACH_UP, up = dir != ALZ_REACH_DOWN;
      listed = (down && hf < max_hops) || (up && ht < max_hops);
      c = (down && hf == max_hops && ht == kUnreached) || (up && ht == max_hops && hf == kUnreached);
    }
    if (r < n) flag[r] = listed ? 1u : 0u;
    const uint32_t b = __ballot_sync(0xFFFFFFFFu, c);
    if (lane == 0 && b) atomicAdd(cut, (unsigned long long)__popc(b));
  }
  if (t0 == 0) flag[n] = 0u;
}

// record j of the result: node order[j]
__global__ void __launch_bounds__(256) reach_emit_kernel(const uint32_t* __restrict__ order, uint32_t m,
                                                         const uint64_t* __restrict__ node_keys,
                                                         const uint32_t* __restrict__ hops,
                                                         const uint64_t* __restrict__ best,
                                                         const uint32_t* __restrict__ pos,
                                                         alz_reach_node* __restrict__ out) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += stride) {
    const uint32_t v = order[j];
    const uint64_t key = node_keys[v], b = best[v];
    const bool seed = b == kNoBest;
    uint2* o = reinterpret_cast<uint2*>(out + j);
    o[0] = make_uint2((uint32_t)(key >> 32), (uint32_t)key);
    o[1] = make_uint2(hops[v], v);
    o[2] = make_uint2(seed ? 0xFFFFFFFFu : pos[(uint32_t)(b >> 32)], (uint32_t)b);
  }
}

}  // namespace

namespace alz {
namespace metrics {

void Graph::free() {
  g.free();
  free_bufs({&end_node, &node_keys, &values, &trav, &tmp});
}

void Csr::free() { free_bufs({&off, &cursor, &adj}); }

int graph_build(alz_handle* h, Graph& gr, const alz_edge_out* rows, uint32_t n, const MetricSet* ms, double min_value,
                std::initializer_list<std::pair<uint32_t, Csr*>> csrs) {
  cudaStream_t st = h->stream;
  const uint32_t n2 = 2u * n;
  NodeGroup& g = gr.g;
  int rc = node_group_reserve(h, g, n2);
  if (rc != ALZ_OK) return rc;
  node_group_keys(h, g, rows, n);
  rc = node_group_runs(h, g, n2, kNodeKeyBits);   // the wait for the node count
  if (rc != ALZ_OK) return rc;
  const uint32_t N = g.h_words[0];
  gr.nodes = N;
  rc = reserve(h, {{&gr.end_node, (size_t)n2 * 4},
                   {&gr.node_keys, (size_t)N * 8},
                   {&gr.values, ms ? (size_t)n * 8 : 0},
                   {&gr.trav, n},
                   {&gr.tmp, scan_temp_bytes(std::max(N, n) + 1u)}});
  if (rc != ALZ_OK) return rc;
  for (const auto& c : csrs) {
    const uint32_t entries_max = c.first == ALZ_REACH_ANY ? n2 : n;
    rc = reserve(h, {{&c.second->off, ((size_t)N + 1) * 4},
                     {&c.second->cursor, ((size_t)N + 1) * 4},
                     {&c.second->adj, (size_t)entries_max * 8}});
    if (rc != ALZ_OK) return rc;
  }
  uint32_t* end_node = static_cast<uint32_t*>(gr.end_node.p);
  uint8_t* trav = static_cast<uint8_t*>(gr.trav.p);
  reach_index_kernel<<<grid_for(h, n2, 8), 256, 0, st>>>(static_cast<const uint64_t*>(g.keys_out.p),
                                                         static_cast<const uint32_t*>(g.vals_out.p),
                                                         static_cast<const uint32_t*>(g.heads.p),
                                                         static_cast<const uint32_t*>(g.idx.p), n2, end_node,
                                                         static_cast<uint64_t*>(gr.node_keys.p));
  h->launches += 1;
  const uint64_t* vals = nullptr;
  uint64_t min_key = 0;
  if (ms) {
    rc = run_metrics(h, rows, n, *ms, static_cast<double*>(gr.values.p));
    if (rc != ALZ_OK) return rc;
    vals = static_cast<const uint64_t*>(gr.values.p);
    uint64_t bits;
    memcpy(&bits, &min_value, 8);
    min_key = top::order_key(bits);
  }
  for (const auto& c : csrs) {
    uint32_t* adj_off = static_cast<uint32_t*>(c.second->off.p);
    uint32_t* cursor = static_cast<uint32_t*>(c.second->cursor.p);
    CK(cudaMemsetAsync(cursor, 0, ((size_t)N + 1) * 4, st));
    reach_count_kernel<<<grid_for(h, n, 8), 256, 0, st>>>(end_node, n, c.first, vals, min_key, trav, cursor);
    CK(cudaGetLastError());
    CK(exclusive_scan_u32(gr.tmp.p, gr.tmp.bytes, cursor, adj_off, N + 1, st));
    CK(cudaMemcpyAsync(cursor, adj_off, (size_t)N * 4, cudaMemcpyDeviceToDevice, st));
    reach_fill_kernel<<<grid_for(h, n, 8), 256, 0, st>>>(end_node, n, c.first, trav, cursor,
                                                         static_cast<uint64_t*>(c.second->adj.p));
    h->launches += 2;
  }
  return ALZ_OK;
}

}  // namespace metrics
}  // namespace alz

// Buffers of the reach calls, each grown on demand and never shrunk; freed in alz_destroy
struct alz_reach_state {
  Graph gr;                            // the traversed rows' nodes, traversable rows and scan scratch
  Csr csr;                             // by tail, in the call's direction
  DevBuf edges;                        // group form: the source's group-edge rows
  DevBuf seeds;                        // the packed seeds
  DevBuf hops, best, flag, scan;       // per node (flag and scan also per row)
  DevBuf pos, deg, dscan, ctr;         // node -> result position, the frontier's degrees, the cut
  DevBuf row_pos, row_vals;            // the listed rows' positions, the gather's value scratch
  DevBuf order, row_index, rows;       // the results: nodes in result order (then the records), rows
  DevBuf rec;
  uint64_t* h_words = nullptr;         // pinned: [0] a scan total, [1] the cut, [2] all entries, [3] a frontier's
};

void alz_internal_free_reach(alz_handle* h) {
  alz_reach_state* s = h->reach;
  if (!s) return;
  s->gr.free();
  s->csr.free();
  free_bufs({&s->edges, &s->seeds, &s->hops, &s->best, &s->flag, &s->scan, &s->pos, &s->deg, &s->dscan, &s->ctr,
             &s->row_pos, &s->row_vals, &s->order, &s->row_index, &s->rows, &s->rec});
  if (s->h_words) cudaFreeHost(s->h_words);
  delete s;
  h->reach = nullptr;
}

namespace {

bool valid_source(uint32_t source) { return source == ALZ_SOURCE_WINDOW || source <= ALZ_ROLLUP_SPAN; }

// a seed of the node form (§22's key rule), or of the group form (§26's)
bool valid_seed(const alz_node_ends& e, bool group) {
  return group ? valid_group_node_key(e.type, e.value) : valid_node_key(e.type, e.value);
}

struct Query {
  const alz_node_ends* seeds;
  size_t n_seeds;
  uint32_t dir, max_hops;
  bool filter;
  MetricSet ms;
  double min_value;
};

struct Result {
  const alz_edge_out* traversed = nullptr;   // the rows the search ran over
  size_t nodes = 0, rows = 0;                // listed
  alz_reach_info info{};
};

// copy a device word to h_words[slot] on the stream
#define REACH_READ(slot, src, bytes) CK(cudaMemcpyAsync(s->h_words + (slot), (src), (bytes), cudaMemcpyDeviceToHost, st))

// The search over n traversed rows: the records in s->rec, the row positions in s->row_index and the rows in s->rows.
// Caller holds h->mu and has set the device; n <= kMaxNodeSourceRows.
int run_reach(alz_handle* h, alz_reach_state* s, const alz_edge_out* rows, size_t n_rows, const Query& q, Result* res) {
  res->traversed = rows;
  res->info.rows = n_rows;
  if (n_rows == 0) return ALZ_OK;
  cudaStream_t st = h->stream;
  const uint32_t n = (uint32_t)n_rows;
  int rc = graph_build(h, s->gr, rows, n, q.filter ? &q.ms : nullptr, q.min_value, {{q.dir, &s->csr}});
  if (rc != ALZ_OK) return rc;
  const uint32_t N = s->gr.nodes;
  const uint32_t flags = std::max(N, n) + 1u;
  rc = reserve(h, {{&s->seeds, q.n_seeds * 8},
                   {&s->hops, (size_t)N * 4},
                   {&s->best, (size_t)N * 8},
                   {&s->flag, (size_t)flags * 4},
                   {&s->scan, (size_t)flags * 4},
                   {&s->pos, (size_t)N * 4},
                   {&s->deg, ((size_t)N + 1) * 4},
                   {&s->dscan, ((size_t)N + 1) * 4},
                   {&s->ctr, 16},
                   {&s->order, (size_t)N * 4},
                   {&s->row_pos, (size_t)n * 4}});
  if (rc != ALZ_OK) return rc;
  if (!s->h_words) {
    void* p = nullptr;
    if (cudaMallocHost(&p, 4 * sizeof(uint64_t)) != cudaSuccess) {
      h->last_err = std::string("reach: ") + cudaGetErrorString(cudaGetLastError());
      return ALZ_E_NOMEM;
    }
    s->h_words = static_cast<uint64_t*>(p);
  }
  const uint32_t* end_node = static_cast<const uint32_t*>(s->gr.end_node.p);
  const uint64_t* node_keys = static_cast<const uint64_t*>(s->gr.node_keys.p);
  const uint32_t* adj_off = static_cast<const uint32_t*>(s->csr.off.p);
  const uint64_t* adj = static_cast<const uint64_t*>(s->csr.adj.p);
  const uint8_t* trav = static_cast<const uint8_t*>(s->gr.trav.p);
  void* tmp = s->gr.tmp.p;
  const size_t tmp_bytes = s->gr.tmp.bytes;
  uint32_t* hops = static_cast<uint32_t*>(s->hops.p);
  uint64_t* best = static_cast<uint64_t*>(s->best.p);
  uint32_t* flag = static_cast<uint32_t*>(s->flag.p);
  uint32_t* scan = static_cast<uint32_t*>(s->scan.p);
  uint32_t* pos = static_cast<uint32_t*>(s->pos.p);
  uint32_t* order = static_cast<uint32_t*>(s->order.p);
  unsigned long long* cut = static_cast<unsigned long long*>(s->ctr.p);
  uint32_t* entries = reinterpret_cast<uint32_t*>(cut + 1);   // the next frontier's adjacency entries
  // seeds
  std::vector<uint64_t> packed(q.n_seeds);
  for (size_t i = 0; i < q.n_seeds; ++i) packed[i] = ((uint64_t)q.seeds[i].type << 32) | q.seeds[i].value;
  CK(cudaMemcpyAsync(s->seeds.p, packed.data(), q.n_seeds * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(hops, 0xFF, (size_t)N * 4, st));
  CK(cudaMemsetAsync(best, 0xFF, (size_t)N * 8, st));
  reach_seed_kernel<<<grid_for(h, q.n_seeds, 8), 256, 0, st>>>(static_cast<const uint64_t*>(s->seeds.p),
                                                                (uint32_t)q.n_seeds, node_keys, N, hops);
  h->launches += 1;
  // level 0: the seeds found
  uint32_t off = 0, size = 0;
  CK(cudaMemsetAsync(entries, 0, 4, st));
  reach_discover_kernel<<<grid_for(h, N, 8), 256, 0, st>>>(best, N, 0, adj_off, hops, flag, entries);
  CK(cudaGetLastError());
  CK(exclusive_scan_u32(tmp, tmp_bytes, flag, scan, N + 1, st));
  reach_scatter_kernel<<<grid_for(h, N, 8), 256, 0, st>>>(flag, scan, N, 0, order, pos);
  h->launches += 2;
  REACH_READ(0, scan + N, 4);
  REACH_READ(2, adj_off + N, 4);
  REACH_READ(3, entries, 4);
  CK(cudaStreamSynchronize(st));   // the wait for the seeds found
  size = (uint32_t)s->h_words[0];
  res->info.seeds_found = size;
  res->info.traversable = q.dir == ALZ_REACH_ANY ? (uint32_t)s->h_words[2] / 2u : (uint32_t)s->h_words[2];
  uint32_t level = 0;
  while (size && level < q.max_hops) {
    const uint32_t* frontier = order + off;
    uint32_t* deg = static_cast<uint32_t*>(s->deg.p);
    uint32_t* dscan = static_cast<uint32_t*>(s->dscan.p);
    reach_degree_kernel<<<grid_for(h, size, 8), 256, 0, st>>>(frontier, size, adj_off, deg);
    CK(cudaGetLastError());
    CK(exclusive_scan_u32(tmp, tmp_bytes, deg, dscan, size + 1, st));
    const uint32_t frontier_entries = (uint32_t)s->h_words[3];   // read with the frontier's size
    reach_expand_kernel<<<grid_for(h, frontier_entries, 8), 256, 0, st>>>(frontier, size, dscan, adj_off, adj, hops,
                                                                          reinterpret_cast<unsigned long long*>(best));
    CK(cudaMemsetAsync(entries, 0, 4, st));
    reach_discover_kernel<<<grid_for(h, N, 8), 256, 0, st>>>(best, N, level + 1, adj_off, hops, flag, entries);
    CK(cudaGetLastError());
    CK(exclusive_scan_u32(tmp, tmp_bytes, flag, scan, N + 1, st));
    reach_scatter_kernel<<<grid_for(h, N, 8), 256, 0, st>>>(flag, scan, N, off + size, order, pos);
    h->launches += 4;
    REACH_READ(0, scan + N, 4);
    REACH_READ(3, entries, 4);
    CK(cudaStreamSynchronize(st));   // the wait of this level: the next frontier's size and entries
    off += size;
    size = (uint32_t)s->h_words[0];
    if (size) level += 1;
  }
  const uint32_t listed_nodes = off + size;
  res->nodes = listed_nodes;
  res->info.nodes = listed_nodes;
  res->info.levels = level;
  // rows and cut
  CK(cudaMemsetAsync(cut, 0, 8, st));
  reach_rows_kernel<<<grid_for(h, n, 8), 256, 0, st>>>(end_node, n, q.dir, trav, hops, q.max_hops, flag, cut);
  CK(cudaGetLastError());
  CK(exclusive_scan_u32(tmp, tmp_bytes, flag, scan, n + 1, st));
  reach_scatter_kernel<<<grid_for(h, n, 8), 256, 0, st>>>(flag, scan, n, 0, static_cast<uint32_t*>(s->row_pos.p),
                                                          nullptr);
  h->launches += 2;
  REACH_READ(0, scan + n, 4);
  REACH_READ(1, cut, 8);
  CK(cudaStreamSynchronize(st));   // the wait for the listed rows
  const uint32_t m = (uint32_t)s->h_words[0];
  res->rows = m;
  res->info.cut = s->h_words[1];
  rc = reserve(h, {{&s->rec, std::max<size_t>(listed_nodes, 1) * sizeof(alz_reach_node)},
                   {&s->row_index, std::max<size_t>(m, 1) * 4},
                   {&s->row_vals, std::max<size_t>(m, 1) * 4},
                   {&s->rows, std::max<size_t>(m, 1) * sizeof(alz_edge_out)}});
  if (rc != ALZ_OK) return rc;
  if (listed_nodes) {
    reach_emit_kernel<<<grid_for(h, listed_nodes, 8), 256, 0, st>>>(order, listed_nodes, node_keys, hops, best, pos,
                                                                    static_cast<alz_reach_node*>(s->rec.p));
    h->launches += 1;
    CK(cudaGetLastError());
  }
  // The gather of the top calls copies each listed row and its position; it also copies one value per result, which
  // reach has no use for: the rows' flags go to row_vals, scratch that nothing reads, so the shared kernel stays as it
  // is
  return top::gather<uint32_t>(h, static_cast<const uint32_t*>(s->row_pos.p), m, flag, rows,
                               static_cast<uint32_t*>(s->row_index.p), static_cast<uint32_t*>(s->row_vals.p),
                               static_cast<alz_edge_out*>(s->rows.p));
}
#undef REACH_READ

// The five entry points: the node form over a source or the hook's caller rows, or the group form over a source's
// group-edge rows. Device call (device true): the dev_* pointers that are not null; host call: the arrays that are not
// null, within their caps, and one more wait for the copies.
int reach_entry(alz_handle* h, bool group, bool hook, uint32_t source, const alz_edge_out* dev_rows, size_t n_in,
                const alz_node_ends* seeds, size_t n_seeds, uint32_t dir, uint32_t max_hops, const alz_metric* m,
                double min_value, bool device, alz_reach_node* nodes, size_t node_cap, uint32_t* row_index,
                alz_edge_out* rows_out, size_t row_cap, const alz_reach_node** dev_nodes,
                const uint32_t** dev_row_index, const alz_edge_out** dev_rows_out, size_t* n_nodes, size_t* n_rows,
                alz_reach_info* info) {
  if (n_nodes) *n_nodes = 0;
  if (n_rows) *n_rows = 0;
  if (info) *info = alz_reach_info{};
  if (!h || !n_nodes || !n_rows || !seeds || n_seeds == 0) return ALZ_E_INVAL;
  if (hook ? (!dev_rows && n_in) : !valid_source(source)) return ALZ_E_INVAL;
  if (dir > ALZ_REACH_ANY || max_hops == 0 || max_hops > ALZ_REACH_MAX_HOPS) return ALZ_E_INVAL;
  Query q{seeds, n_seeds, dir, max_hops, m != nullptr, MetricSet{}, min_value};
  if (m && (!valid_metrics(m, 1, &q.ms) || std::isnan(min_value))) return ALZ_E_INVAL;
  for (size_t i = 0; i < n_seeds; ++i)   // a malformed seed is refused whatever the sizes
    if (!valid_seed(seeds[i], group)) return ALZ_E_INVAL;
  if (n_seeds > kMaxSeeds) return ALZ_E_CAPACITY;
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  const alz_edge_out* src = dev_rows;
  size_t n = n_in;
  int rc = hook ? (n > kMaxNodeSourceRows ? ALZ_E_CAPACITY : ALZ_OK) : node_source(h, source, &src, &n);
  if (rc != ALZ_OK) return rc;
  if (!h->reach) h->reach = new alz_reach_state();
  alz_reach_state* s = h->reach;
  if (group) {
    size_t edges = 0;
    alz_group_info gi;
    rc = group_edges_into(h, s->edges, src, n, SIZE_MAX, &edges, &gi);   // §24's two waits
    if (rc != ALZ_OK) return rc;
    src = static_cast<const alz_edge_out*>(s->edges.p);
    n = edges;
  }
  Result res;
  rc = run_reach(h, s, src, n, q, &res);
  if (rc != ALZ_OK) return rc;
  *n_nodes = res.nodes;
  *n_rows = res.rows;
  if (info) *info = res.info;
  const alz_reach_node* rec = static_cast<const alz_reach_node*>(s->rec.p);
  const uint32_t* ri = static_cast<const uint32_t*>(s->row_index.p);
  const alz_edge_out* rr = static_cast<const alz_edge_out*>(s->rows.p);
  if (device) {
    if (dev_nodes) *dev_nodes = rec;
    if (dev_row_index) *dev_row_index = ri;
    if (dev_rows_out) *dev_rows_out = rr;
    return ALZ_OK;
  }
  if ((nodes && res.nodes > node_cap) || ((row_index || rows_out) && res.rows > row_cap)) return ALZ_E_CAPACITY;
  cudaStream_t st = h->stream;
  if (nodes && res.nodes) CK(cudaMemcpyAsync(nodes, rec, res.nodes * sizeof(alz_reach_node), cudaMemcpyDeviceToHost, st));
  if (row_index && res.rows) CK(cudaMemcpyAsync(row_index, ri, res.rows * 4, cudaMemcpyDeviceToHost, st));
  if (rows_out && res.rows) CK(cudaMemcpyAsync(rows_out, rr, res.rows * sizeof(alz_edge_out), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return ALZ_OK;
}

}  // namespace

extern "C" int alz_reach(alz_handle* h, uint32_t source, const alz_node_ends* seeds, size_t n_seeds, uint32_t dir,
                         uint32_t max_hops, const alz_metric* m, double min_value, alz_reach_node* nodes,
                         size_t node_cap, size_t* n_nodes, uint32_t* row_index, alz_edge_out* rows, size_t row_cap,
                         size_t* n_rows, alz_reach_info* info) {
  return reach_entry(h, false, false, source, nullptr, 0, seeds, n_seeds, dir, max_hops, m, min_value, false, nodes,
                     node_cap, row_index, rows, row_cap, nullptr, nullptr, nullptr, n_nodes, n_rows, info);
}

extern "C" int alz_reach_device(alz_handle* h, uint32_t source, const alz_node_ends* seeds, size_t n_seeds,
                                uint32_t dir, uint32_t max_hops, const alz_metric* m, double min_value,
                                const alz_reach_node** dev_nodes, size_t* n_nodes, const uint32_t** dev_row_index,
                                const alz_edge_out** dev_rows, size_t* n_rows, alz_reach_info* info) {
  return reach_entry(h, false, false, source, nullptr, 0, seeds, n_seeds, dir, max_hops, m, min_value, true, nullptr,
                     0, nullptr, nullptr, 0, dev_nodes, dev_row_index, dev_rows, n_nodes, n_rows, info);
}

extern "C" int alz_group_reach(alz_handle* h, uint32_t source, const alz_node_ends* seeds, size_t n_seeds,
                               uint32_t dir, uint32_t max_hops, const alz_metric* m, double min_value,
                               alz_reach_node* nodes, size_t node_cap, size_t* n_nodes, uint32_t* row_index,
                               alz_edge_out* rows, size_t row_cap, size_t* n_rows, alz_reach_info* info) {
  return reach_entry(h, true, false, source, nullptr, 0, seeds, n_seeds, dir, max_hops, m, min_value, false, nodes,
                     node_cap, row_index, rows, row_cap, nullptr, nullptr, nullptr, n_nodes, n_rows, info);
}

extern "C" int alz_group_reach_device(alz_handle* h, uint32_t source, const alz_node_ends* seeds, size_t n_seeds,
                                      uint32_t dir, uint32_t max_hops, const alz_metric* m, double min_value,
                                      const alz_reach_node** dev_nodes, size_t* n_nodes,
                                      const uint32_t** dev_row_index, const alz_edge_out** dev_rows, size_t* n_rows,
                                      alz_reach_info* info) {
  return reach_entry(h, true, false, source, nullptr, 0, seeds, n_seeds, dir, max_hops, m, min_value, true, nullptr,
                     0, nullptr, nullptr, 0, dev_nodes, dev_row_index, dev_rows, n_nodes, n_rows, info);
}

extern "C" int alz_debug_reach_rows(alz_handle* h, const alz_edge_out* dev_rows, size_t n, const alz_node_ends* seeds,
                                    size_t n_seeds, uint32_t dir, uint32_t max_hops, const alz_metric* m,
                                    double min_value, alz_reach_node* nodes, size_t node_cap, size_t* n_nodes,
                                    uint32_t* row_index, alz_edge_out* rows, size_t row_cap, size_t* n_rows,
                                    alz_reach_info* info) {
  return reach_entry(h, false, true, 0, dev_rows, n, seeds, n_seeds, dir, max_hops, m, min_value, false, nodes,
                     node_cap, row_index, rows, row_cap, nullptr, nullptr, nullptr, n_nodes, n_rows, info);
}
