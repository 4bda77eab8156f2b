// alz_cycles.cu — cycles (docs/SPEC.md §28): the strongly connected components of a source's rows (node form) or of its
// §24 group-edge rows (group form), each component's number, size, depth and height, and the rows inside the listed
// cyclic components. Reads the source rows only; every buffer written is this state's, or scratch of the group calls
// (group_edges_into), so no other family's results move.
//
//   graph    group form: group_edges_into (two waits) into this state's rows first. graph_build (alz_reach.cu) over the
//            traversed rows: node indices (one wait), the filter, and the CSRs by from end (out) and by to end (in)
//   degrees  per node, the traversable rows into and out of it that are not self rows; the traversable and self rows
//   scc      one cooperative launch. Trim: a node without remaining in-rows or out-rows is a component of its own;
//            removing it lowers its neighbours' counters, and one that reaches 0 joins the next frontier. Then, until
//            no node is left: max-label colouring over the remaining nodes (a frontier of the nodes whose colour rose),
//            roots (colour = own index), a sweep the other way from each root over nodes of its colour, which is the
//            root's component, and a compaction of the nodes still left; even iterations colour along out-rows, odd
//            ones along in-rows. comp[v] = the component's
//            representative (a trimmed node itself, else its root, the largest index in it). Frontiers are queues
//            sized by counters in device memory, so the rounds cost no host wait; a round's work is its frontier's
//            adjacency, or the nodes still left
//   number   per representative, the smallest index (atomicMin) and the size; a node heads its component when it is
//            that smallest index; a scan of the heads numbers the components in ascending order of it
//   order    the records' keys (component << 32) | index sorted; each component's first position in them
//   kahn     condensation rows counted per component both ways, then two cooperative launches of Kahn's algorithm
//            level by level (out CSR: depth; in CSR: height): a component's level is the round its counter reaches 0
//   rows     the listed rows' keys (component << 32) | row sorted, unlisted rows after them
//   totals   the one wait that sizes the results; then the records are emitted and the top calls' gather copies the
//            rows
#include <cooperative_groups.h>

#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstring>
#include <mutex>
#include <string>

#include "alz_metrics.cuh"
#include "alz_top.cuh"

using namespace alz;
using namespace alz::metrics;
namespace cg = cooperative_groups;

static_assert(sizeof(alz_cycle_node) == 28 && offsetof(alz_cycle_node, value) == 4 &&
                  offsetof(alz_cycle_node, index) == 8 && offsetof(alz_cycle_node, component) == 12 &&
                  offsetof(alz_cycle_node, size) == 16 && offsetof(alz_cycle_node, depth) == 20 &&
                  offsetof(alz_cycle_node, height) == 24,
              "alz_cycle_node is seven u32 words, the first two an alz_node_ends");
static_assert(sizeof(alz_cycle_info) == 80, "alz_cycle_info is ten u64");

namespace {

constexpr uint32_t kNone = 0xFFFFFFFFu;

// the device totals, read in the one wait that sizes the results
enum Total {
  kTraversable, kSelf, kComponents, kCyclic, kCyclicNodes, kLargest, kCycleRows, kDepth, kListedNodes, kListedRows,
  kTotals
};
// the queue counters of the cooperative launches: three frontier sizes in rotation, two more in alternation
constexpr uint32_t kCtlWords = 8;

__device__ __forceinline__ uint32_t ld(const uint32_t* p) { return __ldcg(p); }

// q[atomicAdd(cnt, 1)] = v, one atomic per coalesced group of the calling threads
__device__ __forceinline__ void push(uint32_t* q, uint32_t* cnt, uint32_t v) {
  cg::coalesced_group g = cg::coalesced_threads();
  uint32_t base = 0;
  if (g.thread_rank() == 0) base = atomicAdd(cnt, g.size());
  base = g.shfl(base, 0);
  q[base + g.thread_rank()] = v;
}

// the node indices of row r's ends: .x its to end's, .y its from end's
__device__ __forceinline__ uint2 row_ends(const uint32_t* __restrict__ end_node, uint32_t r) {
  return reinterpret_cast<const uint2*>(end_node)[r];
}

// in_deg[to] and out_deg[from] += 1 per traversable row that is not a self row; the traversable and self rows counted
__global__ void __launch_bounds__(256) cycle_degree_kernel(const uint32_t* __restrict__ end_node, uint32_t n,
                                                           const uint8_t* __restrict__ trav,
                                                           uint32_t* __restrict__ in_deg,
                                                           uint32_t* __restrict__ out_deg,
                                                           unsigned long long* __restrict__ totals) {
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t lane = threadIdx.x & 31u;
  for (uint32_t base = blockIdx.x * blockDim.x + threadIdx.x - lane; base < n; base += stride) {
    const uint32_t r = base + lane;
    bool t = false, self = false;
    if (r < n && trav[r]) {
      t = true;
      const uint2 e = row_ends(end_node, r);
      self = e.x == e.y;
      if (!self) {
        atomicAdd(in_deg + e.x, 1u);
        atomicAdd(out_deg + e.y, 1u);
      }
    }
    const uint32_t bt = __ballot_sync(0xFFFFFFFFu, t), bs = __ballot_sync(0xFFFFFFFFu, self);
    if (lane == 0 && bt) atomicAdd(totals + kTraversable, (unsigned long long)__popc(bt));
    if (lane == 0 && bs) atomicAdd(totals + kSelf, (unsigned long long)__popc(bs));
  }
}

struct SccArgs {
  const uint32_t* out_off;
  const uint64_t* out_adj;
  const uint32_t* in_off;
  const uint64_t* in_adj;
  uint32_t nodes;
  uint32_t* in_deg;    // the trim's counters: rows into / out of each node from nodes not yet removed
  uint32_t* out_deg;
  uint32_t* comp;      // each node's representative, kNone until assigned
  uint32_t* color;
  uint32_t* stamp;     // the round a node was last queued in (kNone before the first)
  uint32_t* qa;        // frontier queues, nodes words each
  uint32_t* qb;
  uint32_t* la;        // the nodes still left, nodes words each
  uint32_t* lb;
  uint32_t* ctl;       // kCtlWords, zero
};

// The rounds of one frontier phase from round *r on: the frontier of round r is queue (r & 1) with ctl[r % 3] nodes,
// and a round queues the next in the other queue, counting into ctl[(r + 1) % 3], while ctl[(r + 2) % 3], read in the
// round before, is zeroed for the round after. One warp per frontier node; visit(u, lane, next, count, r) runs on
// each lane. Returns after the first empty frontier, with every block past its read of the count.
template <class Visit>
__device__ __forceinline__ void rounds(cg::grid_group& grid, uint32_t* qa, uint32_t* qb, uint32_t* ctl, uint32_t& r, Visit visit) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, warps = (gridDim.x * blockDim.x) >> 5;
  for (;;) {
    const uint32_t size = ld(ctl + r % 3u);
    if (size == 0) break;
    const uint32_t* cur = (r & 1u) ? qb : qa;
    uint32_t* next = (r & 1u) ? qa : qb;
    if (blockIdx.x == 0 && threadIdx.x == 0) ctl[(r + 2u) % 3u] = 0u;
    for (uint32_t i = warp; i < size; i += warps) visit(cur[i], lane, next, ctl + (r + 1u) % 3u, r);
    grid.sync();
    ++r;
  }
  grid.sync();
}

// The components: comp[v] for every node (a trimmed node is its own representative; any other node's is the root of
// its colour, the largest index in its component). Four blocks per SM, as coop_grid launches it: without the minimum
// ptxas holds the kernel to 32 registers and spills.
__global__ void __launch_bounds__(256, 4) cycle_scc_kernel(SccArgs a) {
  cg::grid_group grid = cg::this_grid();
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t N = a.nodes;
  uint32_t r = 0;
  // trim: the first frontier is every node without an in-row or an out-row
  for (uint32_t v = t0; v < N; v += stride) {
    const bool f = a.in_deg[v] == 0u || a.out_deg[v] == 0u;
    a.comp[v] = f ? v : kNone;
    if (f) push(a.qa, a.ctl, v);
  }
  grid.sync();
  rounds(grid, a.qa, a.qb, a.ctl, r, [=](uint32_t u, uint32_t lane, uint32_t* next, uint32_t* cnt, uint32_t round) {
    for (uint32_t j = a.out_off[u] + lane; j < a.out_off[u + 1]; j += 32u) {
      const uint32_t w = (uint32_t)(a.out_adj[j] >> 32);
      if (w != u && atomicSub(a.in_deg + w, 1u) == 1u && atomicCAS(a.comp + w, kNone, w) == kNone) push(next, cnt, w);
    }
    for (uint32_t j = a.in_off[u] + lane; j < a.in_off[u + 1]; j += 32u) {
      const uint32_t w = (uint32_t)(a.in_adj[j] >> 32);
      if (w != u && atomicSub(a.out_deg + w, 1u) == 1u && atomicCAS(a.comp + w, kNone, w) == kNone) push(next, cnt, w);
    }
  });
  // the nodes left
  uint32_t* left = a.la;
  uint32_t* spare = a.lb;
  uint32_t* n_left = a.ctl + 3;
  uint32_t* n_spare = a.ctl + 4;
  for (uint32_t v = t0; v < N; v += stride)
    if (ld(a.comp + v) == kNone) push(left, n_left, v);
  grid.sync();
  // Iterations alternate direction: odd ones colour along in-rows and sweep along out-rows, which finds the same
  // components of the reversed graph. A chain of loops whose indices fall (or rise) downstream settles one loop per
  // iteration in one direction and all of them in the other.
  bool flip = false;
  for (uint32_t L = ld(n_left); L; L = ld(n_left), flip = !flip) {
    const uint32_t* f_off = flip ? a.in_off : a.out_off;
    const uint64_t* f_adj = flip ? a.in_adj : a.out_adj;
    const uint32_t* b_off = flip ? a.out_off : a.in_off;
    const uint64_t* b_adj = flip ? a.out_adj : a.in_adj;
    // colouring: color[w] = the largest index that reaches w among the nodes left
    uint32_t* first = (r & 1u) ? a.qb : a.qa;
    for (uint32_t i = t0; i < L; i += stride) {
      const uint32_t v = left[i];
      a.color[v] = v;
      first[i] = v;
    }
    if (t0 == 0) a.ctl[r % 3u] = L;
    grid.sync();
    rounds(grid, a.qa, a.qb, a.ctl, r, [=](uint32_t u, uint32_t lane, uint32_t* next, uint32_t* cnt, uint32_t round) {
      const uint32_t c = ld(a.color + u);
      for (uint32_t j = f_off[u] + lane; j < f_off[u + 1]; j += 32u) {
        const uint32_t w = (uint32_t)(f_adj[j] >> 32);
        if (w == u || ld(a.comp + w) != kNone || ld(a.color + w) >= c) continue;
        if (atomicMax(a.color + w, c) < c && atomicExch(a.stamp + w, round) != round) push(next, cnt, w);
      }
    });
    // roots, then the backward sweep over each root's colour
    first = (r & 1u) ? a.qb : a.qa;
    for (uint32_t i = t0; i < L; i += stride) {
      const uint32_t v = left[i];
      if (ld(a.color + v) == v) {
        a.comp[v] = v;
        push(first, a.ctl + r % 3u, v);
      }
    }
    grid.sync();
    rounds(grid, a.qa, a.qb, a.ctl, r, [=](uint32_t u, uint32_t lane, uint32_t* next, uint32_t* cnt, uint32_t round) {
      const uint32_t c = ld(a.color + u);
      for (uint32_t j = b_off[u] + lane; j < b_off[u + 1]; j += 32u) {
        const uint32_t w = (uint32_t)(b_adj[j] >> 32);
        if (w != u && ld(a.color + w) == c && atomicCAS(a.comp + w, kNone, c) == kNone) push(next, cnt, w);
      }
    });
    // compaction: the nodes still left
    for (uint32_t i = t0; i < L; i += stride) {
      const uint32_t v = left[i];
      if (ld(a.comp + v) == kNone) push(spare, n_spare, v);
    }
    grid.sync();
    if (t0 == 0) {
      *n_left = ld(n_spare);
      *n_spare = 0u;
    }
    uint32_t* t = left;
    left = spare;
    spare = t;
    grid.sync();
  }
}

// per representative: the smallest index of its component and its size
__global__ void __launch_bounds__(256) cycle_min_kernel(const uint32_t* __restrict__ comp, uint32_t N,
                                                        uint32_t* __restrict__ min_idx, uint32_t* __restrict__ size) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < N; v += stride) {
    const uint32_t c = comp[v];
    atomicMin(min_idx + c, v);
    atomicAdd(size + c, 1u);
  }
}

// flag[v] = 1 when v is its component's smallest index; flag[N] = 0 closes the scan
__global__ void __launch_bounds__(256) cycle_head_kernel(const uint32_t* __restrict__ comp, uint32_t N,
                                                         const uint32_t* __restrict__ min_idx,
                                                         uint32_t* __restrict__ flag) {
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x;
  for (uint32_t v = t0; v < N; v += stride) flag[v] = min_idx[comp[v]] == v ? 1u : 0u;
  if (t0 == 0) flag[N] = 0u;
}

// cid[v] = the component number, key[v] = (cid << 32) | v; the head writes the component's size
__global__ void __launch_bounds__(256) cycle_number_kernel(const uint32_t* __restrict__ comp, uint32_t N,
                                                           const uint32_t* __restrict__ min_idx,
                                                           const uint32_t* __restrict__ rep_size,
                                                           const uint32_t* __restrict__ scan,
                                                           uint32_t* __restrict__ cid, uint64_t* __restrict__ key,
                                                           uint32_t* __restrict__ size) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < N; v += stride) {
    const uint32_t rep = comp[v], m = min_idx[rep], c = scan[m];
    cid[v] = c;
    key[v] = ((uint64_t)c << 32) | v;
    if (m == v) size[c] = rep_size[rep];
  }
}

// start[c] = the first sorted position of component c; start[C] = N
__global__ void __launch_bounds__(256) cycle_start_kernel(const uint64_t* __restrict__ sorted, uint32_t N,
                                                          uint32_t* __restrict__ start) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < N; j += stride) {
    const uint32_t c = (uint32_t)(sorted[j] >> 32);
    if (j == 0 || (uint32_t)(sorted[j - 1] >> 32) != c) start[c] = j;
    if (j == N - 1) start[c + 1] = N;
  }
}

// Per traversable row u -> v: in another component, a condensation row (cnt_in[cid v] and cnt_out[cid u] += 1); in the
// same one and not a self row, a cycle row, listed when its component has at least min_size nodes. key[r] =
// (cid << 32) | r for a listed row, (N << 32) | r otherwise, so the listed rows sort first.
__global__ void __launch_bounds__(256) cycle_rows_kernel(const uint32_t* __restrict__ end_node, uint32_t n,
                                                         const uint8_t* __restrict__ trav,
                                                         const uint32_t* __restrict__ cid,
                                                         const uint32_t* __restrict__ size, uint32_t N,
                                                         uint32_t min_size, uint32_t* __restrict__ cnt_in,
                                                         uint32_t* __restrict__ cnt_out, uint64_t* __restrict__ key,
                                                         unsigned long long* __restrict__ totals) {
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t lane = threadIdx.x & 31u;
  for (uint32_t base = blockIdx.x * blockDim.x + threadIdx.x - lane; base < n; base += stride) {
    const uint32_t r = base + lane;
    bool cyc = false, listed = false;
    if (r < n) {
      uint32_t k = N;
      if (trav[r]) {
        const uint2 e = row_ends(end_node, r);
        const uint32_t cu = cid[e.y], cv = cid[e.x];
        if (cu != cv) {
          atomicAdd(cnt_in + cv, 1u);
          atomicAdd(cnt_out + cu, 1u);
        } else if (e.x != e.y) {
          cyc = true;
          listed = size[cu] >= min_size;
          if (listed) k = cu;
        }
      }
      key[r] = ((uint64_t)k << 32) | r;
    }
    const uint32_t bc = __ballot_sync(0xFFFFFFFFu, cyc), bl = __ballot_sync(0xFFFFFFFFu, listed);
    if (lane == 0 && bc) atomicAdd(totals + kCycleRows, (unsigned long long)__popc(bc));
    if (lane == 0 && bl) atomicAdd(totals + kListedRows, (unsigned long long)__popc(bl));
  }
}

struct KahnArgs {
  const uint32_t* off;      // the out CSR (depth) or the in CSR (height)
  const uint64_t* adj;
  const uint32_t* cid;
  const uint64_t* sorted;   // the records' keys, sorted: each component's nodes are a run
  const uint32_t* start;
  const uint32_t* n_comp;   // C, on the device
  uint32_t* cnt;            // condensation rows into each component along the direction; consumed
  uint32_t* level;          // the result
  uint32_t* qa;             // component queues, C words each
  uint32_t* qb;
  uint32_t* nodes;          // the current components' nodes
  uint32_t* ctl;            // kCtlWords, zero
};

// Kahn's algorithm level by level: round d takes the components whose counters are 0 (level d), queues their nodes,
// and each of their rows into another component lowers its counter; one that reaches 0 has level d + 1
__global__ void __launch_bounds__(256) cycle_kahn_kernel(KahnArgs a) {
  cg::grid_group grid = cg::this_grid();
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t warp = t0 >> 5, warps = stride >> 5;
  const uint32_t C = *a.n_comp;
  for (uint32_t c = t0; c < C; c += stride)
    if (a.cnt[c] == 0u) {
      a.level[c] = 0u;
      push(a.qa, a.ctl, c);
    }
  grid.sync();
  for (uint32_t r = 0;; ++r) {
    const uint32_t size = ld(a.ctl + r % 3u);
    if (size == 0) break;
    const uint32_t* cur = (r & 1u) ? a.qb : a.qa;
    uint32_t* next = (r & 1u) ? a.qa : a.qb;
    uint32_t* n_nodes = a.ctl + 3u + (r & 1u);
    if (t0 == 0) {
      a.ctl[(r + 2u) % 3u] = 0u;
      a.ctl[3u + ((r + 1u) & 1u)] = 0u;
    }
    for (uint32_t i = warp; i < size; i += warps) {   // one warp per component: its nodes
      const uint32_t c = cur[i], lo = a.start[c], hi = a.start[c + 1];
      for (uint32_t j = lo + lane; j < hi; j += 32u) push(a.nodes, n_nodes, (uint32_t)a.sorted[j]);
    }
    grid.sync();
    const uint32_t m = ld(n_nodes);
    for (uint32_t i = warp; i < m; i += warps) {   // one warp per node: its rows
      const uint32_t u = a.nodes[i], cu = a.cid[u];
      for (uint32_t j = a.off[u] + lane; j < a.off[u + 1]; j += 32u) {
        const uint32_t cw = a.cid[(uint32_t)(a.adj[j] >> 32)];
        if (cw != cu && atomicSub(a.cnt + cw, 1u) == 1u) {
          a.level[cw] = r + 1u;
          push(next, a.ctl + (r + 1u) % 3u, cw);
        }
      }
    }
    grid.sync();
  }
}

// Per component c < C: the totals (the cyclic ones, their nodes, the largest, the largest depth, the listed nodes)
__global__ void __launch_bounds__(256) cycle_totals_kernel(const uint32_t* __restrict__ size,
                                                           const uint32_t* __restrict__ depth,
                                                           const uint32_t* __restrict__ n_comp, uint32_t min_size,
                                                           unsigned long long* __restrict__ totals) {
  const uint32_t C = *n_comp;
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x;
  if (t0 == 0) totals[kComponents] = C;
  for (uint32_t c = t0; c < C; c += stride) {
    const uint32_t s = size[c];
    if (s >= 2u) {
      atomicAdd(totals + kCyclic, 1ull);
      atomicAdd(totals + kCyclicNodes, (unsigned long long)s);
    }
    if (s >= min_size) atomicAdd(totals + kListedNodes, (unsigned long long)s);
    atomicMax(totals + kLargest, (unsigned long long)s);
    atomicMax(totals + kDepth, (unsigned long long)depth[c]);
  }
}

// flag[j] = 1 when sorted record j is listed (its component has at least min_size nodes); flag[N] = 0
__global__ void __launch_bounds__(256) cycle_list_kernel(const uint64_t* __restrict__ sorted, uint32_t N,
                                                         const uint32_t* __restrict__ size, uint32_t min_size,
                                                         uint32_t* __restrict__ flag) {
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x;
  for (uint32_t j = t0; j < N; j += stride) flag[j] = size[(uint32_t)(sorted[j] >> 32)] >= min_size ? 1u : 0u;
  if (t0 == 0) flag[N] = 0u;
}

// record scan[j] of the result: sorted record j, when flagged
__global__ void __launch_bounds__(256) cycle_emit_kernel(const uint64_t* __restrict__ sorted, uint32_t N,
                                                         const uint32_t* __restrict__ flag,
                                                         const uint32_t* __restrict__ scan,
                                                         const uint64_t* __restrict__ node_keys,
                                                         const uint32_t* __restrict__ size,
                                                         const uint32_t* __restrict__ depth,
                                                         const uint32_t* __restrict__ height,
                                                         alz_cycle_node* __restrict__ out) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < N; j += stride) {
    if (!flag[j]) continue;
    const uint64_t k = sorted[j];
    const uint32_t c = (uint32_t)(k >> 32), v = (uint32_t)k;
    const uint64_t key = node_keys[v];
    uint32_t* o = reinterpret_cast<uint32_t*>(out + scan[j]);
    o[0] = (uint32_t)(key >> 32);
    o[1] = (uint32_t)key;
    o[2] = v;
    o[3] = c;
    o[4] = size[c];
    o[5] = depth[c];
    o[6] = height[c];
  }
}

// pos[j] = the row of sorted row key j
__global__ void __launch_bounds__(256) cycle_row_pos_kernel(const uint64_t* __restrict__ sorted, uint32_t m,
                                                            uint32_t* __restrict__ pos) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += stride) pos[j] = (uint32_t)sorted[j];
}

// the blocks of a cooperative launch of `kernel`: every block resident at once for its grid barriers
template <class K> cudaError_t coop_grid(alz_handle* h, K kernel, unsigned* blocks) {
  int per_sm = 0;
  const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, 256, 0);
  if (e != cudaSuccess) return e;
  *blocks = (unsigned)h->sms * (unsigned)std::max(1, std::min(per_sm, 4));
  return cudaSuccess;
}

// the bits of the largest component number or sentinel key word a sort sees: up to N
int key_bits(uint32_t N) { return 32 + std::max(1, 32 - __builtin_clz(N)); }

}  // namespace

// Buffers of the cycles calls, each grown on demand and never shrunk; freed in alz_destroy
struct alz_cycle_state {
  Graph gr;                                  // the traversed rows' nodes, traversable rows and scan scratch
  Csr out, in;                               // by from end, by to end
  DevBuf edges;                              // group form: the source's group-edge rows
  DevBuf in_deg, out_deg, comp, color;       // per node
  DevBuf stamp, qa, qb, la, lb, ctl;         // the cooperative launches' queues and counters
  DevBuf min_idx, rep_size, cid;             // per representative, per representative, per node
  DevBuf flag, scan, keys, sorted, sort_tmp;   // heads, listings and sorts
  DevBuf size, depth, height, cnt, start;    // per component
  DevBuf row_keys, row_sorted, row_pos, row_vals;   // the rows: keys, sorted keys, positions, the gather's scratch
  DevBuf totals;
  DevBuf rec, row_index, rows;               // the results
  uint64_t* h_totals = nullptr;              // pinned: the totals
};

void alz_internal_free_cycles(alz_handle* h) {
  alz_cycle_state* s = h->cycles;
  if (!s) return;
  s->gr.free();
  s->out.free();
  s->in.free();
  free_bufs({&s->edges, &s->in_deg, &s->out_deg, &s->comp, &s->color, &s->stamp, &s->qa, &s->qb, &s->la, &s->lb,
             &s->ctl, &s->min_idx, &s->rep_size, &s->cid, &s->flag, &s->scan, &s->keys, &s->sorted, &s->sort_tmp, &s->size, &s->depth, &s->height, &s->cnt, &s->start, &s->row_keys,
             &s->row_sorted, &s->row_pos, &s->row_vals, &s->totals, &s->rec, &s->row_index, &s->rows});
  if (s->h_totals) cudaFreeHost(s->h_totals);
  delete s;
  h->cycles = nullptr;
}

namespace {

bool valid_source(uint32_t source) { return source == ALZ_SOURCE_WINDOW || source <= ALZ_ROLLUP_SPAN; }

struct Query {
  bool filter;
  MetricSet ms;
  double min_value;
  uint32_t min_size;
};

struct Result {
  size_t nodes = 0, rows = 0;   // listed
  alz_cycle_info info{};
};

// The components of n traversed rows: the records in s->rec, the row positions in s->row_index and the rows in
// s->rows. Caller holds h->mu and has set the device; n <= kMaxNodeSourceRows.
int run_cycles(alz_handle* h, alz_cycle_state* s, const alz_edge_out* rows, size_t n_rows, const Query& q,
               Result* res) {
  res->info.rows = n_rows;
  if (n_rows == 0) return ALZ_OK;
  cudaStream_t st = h->stream;
  const uint32_t n = (uint32_t)n_rows;
  int rc = graph_build(h, s->gr, rows, n, q.filter ? &q.ms : nullptr, q.min_value,
                       {{ALZ_REACH_DOWN, &s->out}, {ALZ_REACH_UP, &s->in}});   // the wait for the node count
  if (rc != ALZ_OK) return rc;
  const uint32_t N = s->gr.nodes;
  const uint32_t most = std::max(N, n);
  const size_t sort_tmp = std::max(sort_keys_temp_bytes(most), scan_temp_bytes(most + 1u));
  rc = reserve(h, {{&s->in_deg, (size_t)N * 4},
                   {&s->out_deg, (size_t)N * 4},
                   {&s->comp, (size_t)N * 4},
                   {&s->color, (size_t)N * 4},
                   {&s->stamp, (size_t)N * 4},
                   {&s->qa, (size_t)N * 4},
                   {&s->qb, (size_t)N * 4},
                   {&s->la, (size_t)N * 4},
                   {&s->lb, (size_t)N * 4},
                   {&s->ctl, kCtlWords * 4},
                   {&s->min_idx, (size_t)N * 4},
                   {&s->rep_size, (size_t)N * 4},
                   {&s->cid, (size_t)N * 4},
                   {&s->flag, ((size_t)most + 1) * 4},   // also the gather's values, read at row positions
                   {&s->scan, ((size_t)N + 1) * 4},
                   {&s->keys, (size_t)N * 8},
                   {&s->sorted, (size_t)N * 8},
                   {&s->sort_tmp, sort_tmp},
                   {&s->size, (size_t)N * 4},
                   {&s->depth, (size_t)N * 4},
                   {&s->height, (size_t)N * 4},
                   {&s->cnt, (size_t)N * 8},
                   {&s->start, ((size_t)N + 1) * 4},
                   {&s->row_keys, (size_t)n * 8},
                   {&s->row_sorted, (size_t)n * 8},
                   {&s->totals, kTotals * 8}});
  if (rc != ALZ_OK) return rc;
  if (!s->h_totals) {
    void* p = nullptr;
    if (cudaMallocHost(&p, kTotals * sizeof(uint64_t)) != cudaSuccess) {
      h->last_err = std::string("cycles: ") + cudaGetErrorString(cudaGetLastError());
      return ALZ_E_NOMEM;
    }
    s->h_totals = static_cast<uint64_t*>(p);
  }
  auto u32 = [](DevBuf& b) { return static_cast<uint32_t*>(b.p); };
  const uint32_t* end_node = static_cast<const uint32_t*>(s->gr.end_node.p);
  const uint8_t* trav = static_cast<const uint8_t*>(s->gr.trav.p);
  uint64_t* keys = static_cast<uint64_t*>(s->keys.p);
  uint64_t* sorted = static_cast<uint64_t*>(s->sorted.p);
  unsigned long long* totals = static_cast<unsigned long long*>(s->totals.p);
  uint32_t* cnt_in = u32(s->cnt);
  uint32_t* cnt_out = cnt_in + N;
  const uint32_t* n_comp = u32(s->scan) + N;   // the scan of the heads' total
  const unsigned g_n = grid_for(h, n, 8), g_N = grid_for(h, N, 8);
  // degrees
  CK(cudaMemsetAsync(s->in_deg.p, 0, (size_t)N * 4, st));
  CK(cudaMemsetAsync(s->out_deg.p, 0, (size_t)N * 4, st));
  CK(cudaMemsetAsync(totals, 0, kTotals * 8, st));
  cycle_degree_kernel<<<g_n, 256, 0, st>>>(end_node, n, trav, u32(s->in_deg), u32(s->out_deg), totals);
  CK(cudaGetLastError());
  // components
  CK(cudaMemsetAsync(s->stamp.p, 0xFF, (size_t)N * 4, st));
  CK(cudaMemsetAsync(s->ctl.p, 0, kCtlWords * 4, st));
  SccArgs sa{u32(s->out.off), static_cast<const uint64_t*>(s->out.adj.p), u32(s->in.off),
             static_cast<const uint64_t*>(s->in.adj.p), N, u32(s->in_deg), u32(s->out_deg), u32(s->comp),
             u32(s->color), u32(s->stamp), u32(s->qa), u32(s->qb), u32(s->la), u32(s->lb), u32(s->ctl)};
  unsigned blocks = 0;
  CK(coop_grid(h, cycle_scc_kernel, &blocks));
  void* scc_args[] = {&sa};
  CK(cudaLaunchCooperativeKernel((const void*)cycle_scc_kernel, dim3(blocks), dim3(256), scc_args, 0, st));
  // numbering
  CK(cudaMemsetAsync(s->min_idx.p, 0xFF, (size_t)N * 4, st));
  CK(cudaMemsetAsync(s->rep_size.p, 0, (size_t)N * 4, st));
  cycle_min_kernel<<<g_N, 256, 0, st>>>(u32(s->comp), N, u32(s->min_idx), u32(s->rep_size));
  cycle_head_kernel<<<g_N, 256, 0, st>>>(u32(s->comp), N, u32(s->min_idx), u32(s->flag));
  CK(cudaGetLastError());
  CK(exclusive_scan_u32(s->sort_tmp.p, s->sort_tmp.bytes, u32(s->flag), u32(s->scan), N + 1, st));
  cycle_number_kernel<<<g_N, 256, 0, st>>>(u32(s->comp), N, u32(s->min_idx), u32(s->rep_size), u32(s->scan),
                                           u32(s->cid), keys, u32(s->size));
  CK(cudaGetLastError());
  const int bits = key_bits(N);
  CK(sort_keys(s->sort_tmp.p, s->sort_tmp.bytes, keys, sorted, N, st, bits));
  cycle_start_kernel<<<g_N, 256, 0, st>>>(sorted, N, u32(s->start));
  // rows, and the condensation's counters
  CK(cudaMemsetAsync(cnt_in, 0, (size_t)N * 8, st));
  cycle_rows_kernel<<<g_n, 256, 0, st>>>(end_node, n, trav, u32(s->cid), u32(s->size), N, q.min_size, cnt_in, cnt_out,
                                         static_cast<uint64_t*>(s->row_keys.p), totals);
  CK(cudaGetLastError());
  CK(sort_keys(s->sort_tmp.p, s->sort_tmp.bytes, static_cast<const uint64_t*>(s->row_keys.p),
               static_cast<uint64_t*>(s->row_sorted.p), n, st, bits));
  // depth over the out CSR, height over the in CSR
  CK(coop_grid(h, cycle_kahn_kernel, &blocks));
  for (int dir = 0; dir < 2; ++dir) {
    Csr& c = dir == 0 ? s->out : s->in;
    CK(cudaMemsetAsync(s->ctl.p, 0, kCtlWords * 4, st));
    KahnArgs ka{u32(c.off), static_cast<const uint64_t*>(c.adj.p), u32(s->cid), sorted,
                u32(s->start), n_comp, dir == 0 ? cnt_in : cnt_out, u32(dir == 0 ? s->depth : s->height), u32(s->qa),
                u32(s->qb), u32(s->la), u32(s->ctl)};
    void* kahn_args[] = {&ka};
    CK(cudaLaunchCooperativeKernel((const void*)cycle_kahn_kernel, dim3(blocks), dim3(256), kahn_args, 0, st));
  }
  // totals and the listed records
  cycle_totals_kernel<<<g_N, 256, 0, st>>>(u32(s->size), u32(s->depth), n_comp, q.min_size, totals);
  cycle_list_kernel<<<g_N, 256, 0, st>>>(sorted, N, u32(s->size), q.min_size, u32(s->flag));
  CK(cudaGetLastError());
  CK(exclusive_scan_u32(s->sort_tmp.p, s->sort_tmp.bytes, u32(s->flag), u32(s->scan), N + 1, st));
  h->launches += 14;
  CK(cudaMemcpyAsync(s->h_totals, totals, kTotals * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));   // the wait for the totals
  const uint64_t* t = s->h_totals;
  alz_cycle_info& info = res->info;
  info.traversable = t[kTraversable];
  info.self_rows = t[kSelf];
  info.nodes = N;
  info.components = t[kComponents];
  info.cyclic = t[kCyclic];
  info.cyclic_nodes = t[kCyclicNodes];
  info.largest = t[kLargest];
  info.cycle_rows = t[kCycleRows];
  info.depth = t[kDepth];
  res->nodes = t[kListedNodes];
  res->rows = t[kListedRows];
  const uint32_t m = (uint32_t)res->rows;
  rc = reserve(h, {{&s->rec, std::max<size_t>(res->nodes, 1) * sizeof(alz_cycle_node)},
                   {&s->row_pos, std::max<size_t>(m, 1) * 4},
                   {&s->row_index, std::max<size_t>(m, 1) * 4},
                   {&s->row_vals, std::max<size_t>(m, 1) * 4},
                   {&s->rows, std::max<size_t>(m, 1) * sizeof(alz_edge_out)}});
  if (rc != ALZ_OK) return rc;
  if (res->nodes) {
    cycle_emit_kernel<<<g_N, 256, 0, st>>>(sorted, N, u32(s->flag), u32(s->scan),
                                           static_cast<const uint64_t*>(s->gr.node_keys.p), u32(s->size),
                                           u32(s->depth), u32(s->height), static_cast<alz_cycle_node*>(s->rec.p));
    h->launches += 1;
    CK(cudaGetLastError());
  }
  if (m) {
    cycle_row_pos_kernel<<<grid_for(h, m, 8), 256, 0, st>>>(static_cast<const uint64_t*>(s->row_sorted.p), m,
                                                            u32(s->row_pos));
    h->launches += 1;
    CK(cudaGetLastError());
  }
  // the gather also copies one value per result, which cycles has no use for: the flags go to row_vals, scratch that
  // nothing reads, as in reach
  return top::gather<uint32_t>(h, u32(s->row_pos), m, u32(s->flag), rows, u32(s->row_index), u32(s->row_vals),
                               static_cast<alz_edge_out*>(s->rows.p));
}

// The five entry points: the node form over a source or the hook's caller rows, or the group form over a source's
// group-edge rows. Device call (device true): the dev_* pointers that are not null; host call: the arrays that are not
// null, within their caps, and one more wait for the copies.
int cycles_entry(alz_handle* h, bool group, bool hook, uint32_t source, const alz_edge_out* dev_rows, size_t n_in,
                 const alz_metric* m, double min_value, uint32_t min_size, bool device, alz_cycle_node* nodes,
                 size_t node_cap, uint32_t* row_index, alz_edge_out* rows_out, size_t row_cap,
                 const alz_cycle_node** dev_nodes, const uint32_t** dev_row_index, const alz_edge_out** dev_rows_out,
                 size_t* n_nodes, size_t* n_rows, alz_cycle_info* info) {
  if (n_nodes) *n_nodes = 0;
  if (n_rows) *n_rows = 0;
  if (info) *info = alz_cycle_info{};
  if (!h || !n_nodes || !n_rows) return ALZ_E_INVAL;
  if (hook ? (!dev_rows && n_in) : !valid_source(source)) return ALZ_E_INVAL;
  Query q{m != nullptr, MetricSet{}, min_value, min_size};
  if (m && (!valid_metrics(m, 1, &q.ms) || std::isnan(min_value))) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  const alz_edge_out* src = dev_rows;
  size_t n = n_in;
  int rc = hook ? (n > kMaxNodeSourceRows ? ALZ_E_CAPACITY : ALZ_OK) : node_source(h, source, &src, &n);
  if (rc != ALZ_OK) return rc;
  if (!h->cycles) h->cycles = new alz_cycle_state();
  alz_cycle_state* s = h->cycles;
  if (group) {
    size_t edges = 0;
    alz_group_info gi;
    rc = group_edges_into(h, s->edges, src, n, SIZE_MAX, &edges, &gi);   // §24's two waits
    if (rc != ALZ_OK) return rc;
    src = static_cast<const alz_edge_out*>(s->edges.p);
    n = edges;
  }
  Result res;
  rc = run_cycles(h, s, src, n, q, &res);
  if (rc != ALZ_OK) return rc;
  *n_nodes = res.nodes;
  *n_rows = res.rows;
  if (info) *info = res.info;
  const alz_cycle_node* rec = static_cast<const alz_cycle_node*>(s->rec.p);
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
  if (nodes && res.nodes) CK(cudaMemcpyAsync(nodes, rec, res.nodes * sizeof(alz_cycle_node), cudaMemcpyDeviceToHost, st));
  if (row_index && res.rows) CK(cudaMemcpyAsync(row_index, ri, res.rows * 4, cudaMemcpyDeviceToHost, st));
  if (rows_out && res.rows) CK(cudaMemcpyAsync(rows_out, rr, res.rows * sizeof(alz_edge_out), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return ALZ_OK;
}

}  // namespace

extern "C" int alz_cycles(alz_handle* h, uint32_t source, const alz_metric* m, double min_value, uint32_t min_size,
                          alz_cycle_node* nodes, size_t node_cap, size_t* n_nodes, uint32_t* row_index,
                          alz_edge_out* rows, size_t row_cap, size_t* n_rows, alz_cycle_info* info) {
  return cycles_entry(h, false, false, source, nullptr, 0, m, min_value, min_size, false, nodes, node_cap, row_index,
                      rows, row_cap, nullptr, nullptr, nullptr, n_nodes, n_rows, info);
}

extern "C" int alz_cycles_device(alz_handle* h, uint32_t source, const alz_metric* m, double min_value,
                                 uint32_t min_size, const alz_cycle_node** dev_nodes, size_t* n_nodes,
                                 const uint32_t** dev_row_index, const alz_edge_out** dev_rows, size_t* n_rows,
                                 alz_cycle_info* info) {
  return cycles_entry(h, false, false, source, nullptr, 0, m, min_value, min_size, true, nullptr, 0, nullptr, nullptr,
                      0, dev_nodes, dev_row_index, dev_rows, n_nodes, n_rows, info);
}

extern "C" int alz_group_cycles(alz_handle* h, uint32_t source, const alz_metric* m, double min_value,
                                uint32_t min_size, alz_cycle_node* nodes, size_t node_cap, size_t* n_nodes,
                                uint32_t* row_index, alz_edge_out* rows, size_t row_cap, size_t* n_rows,
                                alz_cycle_info* info) {
  return cycles_entry(h, true, false, source, nullptr, 0, m, min_value, min_size, false, nodes, node_cap, row_index,
                      rows, row_cap, nullptr, nullptr, nullptr, n_nodes, n_rows, info);
}

extern "C" int alz_group_cycles_device(alz_handle* h, uint32_t source, const alz_metric* m, double min_value,
                                       uint32_t min_size, const alz_cycle_node** dev_nodes, size_t* n_nodes,
                                       const uint32_t** dev_row_index, const alz_edge_out** dev_rows, size_t* n_rows,
                                       alz_cycle_info* info) {
  return cycles_entry(h, true, false, source, nullptr, 0, m, min_value, min_size, true, nullptr, 0, nullptr, nullptr,
                      0, dev_nodes, dev_row_index, dev_rows, n_nodes, n_rows, info);
}

extern "C" int alz_debug_cycles_rows(alz_handle* h, const alz_edge_out* dev_rows, size_t n, const alz_metric* m,
                                     double min_value, uint32_t min_size, alz_cycle_node* nodes, size_t node_cap,
                                     size_t* n_nodes, uint32_t* row_index, alz_edge_out* rows, size_t row_cap,
                                     size_t* n_rows, alz_cycle_info* info) {
  return cycles_entry(h, false, true, 0, dev_rows, n, m, min_value, min_size, false, nodes, node_cap, row_index, rows,
                      row_cap, nullptr, nullptr, nullptr, n_nodes, n_rows, info);
}
