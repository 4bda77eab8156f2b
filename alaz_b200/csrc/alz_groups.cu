// alz_groups.cu — groups (docs/SPEC.md §24): a source's rows with their ends mapped into caller-defined groups and
// summed into group-edge rows, the §17 metrics and top of those rows, and the §21 nodes, metrics and top over them.
// Reads the source rows only; touches no GNN, metric, change, series, trend or node state.
//
//   map     alz_group_set: the (node key, group) pairs sorted on the device on the 40-bit node key, one kernel that
//           flags adjacent duplicates, one wait; the sorted keys and groups replace the previous map only on success
//   ends    2n (mapped node key, 2 x row + side) pairs, laid out as node_group_keys' (pair 2i: row i's to end, 2i + 1:
//           its from end); each end is looked up by binary search in the map's sorted keys, and the row ends found and
//           the rows whose two mapped ends are equal are counted
//   nodes   node_group_runs over the pairs (sort, heads, scan, one wait): every mapped end gets its index in the group
//           graph's node list, which ascends with the node key; the index kernel writes each end's index at its pair
//           position and each node's key at its index
//   keys    per row, (index(from') << b) | index(to') on 2b bits, b = ceil(log2 nodes): ascending in this key is the
//           §24 order. node_group_runs again (sort with the row index, heads, scan, one wait) gives the group-edge
//           count
//   reduce  the sorted rows in chunks of kWarpRows per warp, kBlockRows per block. A warp walks its chunk once, a lane
//           owning two histogram cells (lanes 0..2 one of the three sums), and stores each run that starts and ends in
//           the chunk plainly with its head. A run that crosses a chunk boundary leaves its part in shared memory; the
//           parts of one run are added there, and the sum is stored plainly when the run lies inside the block, or
//           added with one red.add per word per block when it crosses the block's boundary (its row was zeroed and
//           headed by the split kernel). The arithmetic is integer, mod 2^64 and mod 2^32, so every order of the adds
//           gives the same bytes.
//   metrics §17 over the group-edge rows (run_metrics, select_top); nodes: §21 over them (node_rows_of,
//           run_metrics_nodes, select_top, node_gather)
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <mutex>
#include <string>
#include <vector>

#include "alz_metrics.cuh"

using namespace alz;
using namespace alz::metrics;

namespace {

constexpr uint32_t kWarps = 8;                         // warps per block of the reduce
constexpr uint32_t kWarpRows = 64;                     // sorted rows per warp
constexpr uint32_t kBlockRows = kWarps * kWarpRows;    // sorted rows per block
constexpr uint32_t kSlotWords = 3 + ALZ_NB / 2;        // a run's partial sums: the three u64 sums, 32 cell pairs
constexpr uint32_t kMaxMap = (1u << 30) - 1u;          // map entries: the CUB item counts are ints

static_assert(sizeof(alz_group_info) == 32, "alz_group_info is four u64");
static_assert(offsetof(alz_edge_out, count) == 16 && offsetof(alz_edge_out, hist) == 40 && sizeof(alz_edge_out) == 296,
              "the reduce stores a row as 37 8-byte words: head (2), sums (3), cell pairs (32)");

// flag[0] = 1 when two adjacent sorted keys are equal
__global__ void __launch_bounds__(256) map_dup_kernel(const uint64_t* __restrict__ keys, uint32_t n,
                                                      uint32_t* __restrict__ flag) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x + 1; j < n; j += stride)
    if (keys[j] == keys[j - 1]) *flag = 1u;
}

// Pair 2i + side: row i's mapped to end (IN) or from end (OUT) and its own position; ctr[0] += ends the map held,
// ctr[1] += rows whose two mapped ends are one node
__global__ void __launch_bounds__(256) group_ends_kernel(const alz_edge_out* __restrict__ rows, uint32_t n,
                                                         const uint64_t* __restrict__ mk,
                                                         const uint32_t* __restrict__ mg, uint32_t m,
                                                         uint64_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                                         unsigned long long* __restrict__ ctr) {
  static_assert(ALZ_SIDE_IN == 0u && ALZ_SIDE_OUT == 1u, "pair 2i + side");
  const uint32_t stride = gridDim.x * blockDim.x;
  uint32_t hit = 0, internal = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint2 ty = reinterpret_cast<const uint2*>(rows + i)[0];   // from_type, to_type, pad (rows are 8-aligned)
    const uint2 ft = reinterpret_cast<const uint2*>(rows + i)[1];   // from, to
    const uint64_t kf = map_end(node_key(ty.x & 0xFFu, ft.x), mk, mg, m, &hit);
    const uint64_t kt = map_end(node_key((ty.x >> 8) & 0xFFu, ft.y), mk, mg, m, &hit);
    internal += kf == kt ? 1u : 0u;
    reinterpret_cast<ulonglong2*>(keys)[i] = make_ulonglong2(kt, kf);
    reinterpret_cast<uint2*>(vals)[i] = make_uint2(2u * i, 2u * i + 1u);
  }
  hit = __reduce_add_sync(0xFFFFFFFFu, hit);
  internal = __reduce_add_sync(0xFFFFFFFFu, internal);
  if ((threadIdx.x & 31u) == 0) {
    if (hit) atomicAdd(ctr, (unsigned long long)hit);
    if (internal) atomicAdd(ctr + 1, (unsigned long long)internal);
  }
}

// For sorted pair j: end[val[j]] = its node index; a run head also writes its node key at that index
__global__ void __launch_bounds__(256) group_index_kernel(const uint64_t* __restrict__ keys,
                                                          const uint32_t* __restrict__ vals,
                                                          const uint32_t* __restrict__ heads,
                                                          const uint32_t* __restrict__ idx, uint32_t n2,
                                                          uint32_t* __restrict__ end, uint64_t* __restrict__ nkeys) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n2; j += stride) {
    const uint32_t hd = heads[j], u = idx[j];
    end[vals[j]] = u + hd - 1u;
    if (hd) nkeys[u] = keys[j];
  }
}

// Row i's group-edge key: (index of its from end << bits) | index of its to end, and its position
__global__ void __launch_bounds__(256) group_edge_keys_kernel(const uint32_t* __restrict__ end, uint32_t n,
                                                              uint32_t bits, uint64_t* __restrict__ keys,
                                                              uint32_t* __restrict__ vals) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint2 e = reinterpret_cast<const uint2*>(end)[i];   // .x: the to end (pair 2i), .y: the from end
    keys[i] = ((uint64_t)e.y << bits) | e.x;
    vals[i] = i;
  }
}

// The two head words of the group-edge row of an edge key: types, zero padding, from, to
__device__ __forceinline__ ulonglong2 edge_head(uint64_t key, uint32_t bits, const uint64_t* __restrict__ nkeys) {
  const uint64_t kf = nkeys[key >> bits], kt = nkeys[key & ((1ull << bits) - 1ull)];
  return make_ulonglong2((kf >> 32) | ((kt >> 32) << 8), (kf & 0xFFFFFFFFull) | (kt << 32));
}

// Warp w: block boundary b = (w + 1) x kBlockRows. When one run crosses b, its row is zeroed with its head set, for the
// reduce's red.add. A run over several boundaries is written once per boundary, with the same bytes.
__global__ void __launch_bounds__(256) group_split_kernel(const uint64_t* __restrict__ keys,
                                                          const uint32_t* __restrict__ idx, uint32_t n, uint32_t bits,
                                                          const uint64_t* __restrict__ nkeys,
                                                          alz_edge_out* __restrict__ out) {
  constexpr uint32_t kRowWords = sizeof(alz_edge_out) / 8;
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t bounds = (n - 1u) / kBlockRows;   // boundaries strictly inside [0, n)
  for (uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < bounds; w += warps) {
    const uint32_t b = (w + 1u) * kBlockRows;
    const uint64_t key = keys[b];
    if (keys[b - 1] != key) continue;   // a run starts at b: none crosses it
    uint64_t* o = reinterpret_cast<uint64_t*>(out + (idx[b] - 1u));
    const ulonglong2 hd = edge_head(key, bits, nkeys);
    for (uint32_t q = lane; q < kRowWords; q += 32u) o[q] = q == 0 ? hd.x : q == 1 ? hd.y : 0ull;
  }
}

// Lane l's part of a run: cells 2l, 2l + 1 and, for l < 3, the sum at count + 8l
struct Part {
  uint32_t c0, c1;
  uint64_t s;
  __device__ __forceinline__ void zero() { c0 = c1 = 0u; s = 0ull; }
};

// Lane l's part of row r
__device__ __forceinline__ void load_part(const alz_edge_out* r, uint32_t lane, uint2* c, uint64_t* s) {
  const char* p = reinterpret_cast<const char*>(r);
  *c = *reinterpret_cast<const uint2*>(p + offsetof(alz_edge_out, hist) + 8u * lane);
  *s = lane < 3u ? *reinterpret_cast<const uint64_t*>(p + offsetof(alz_edge_out, count) + 8u * lane) : 0ull;
}

// The whole row of a run, plainly: head, sums, cells
__device__ __forceinline__ void store_row(alz_edge_out* o, uint32_t lane, const Part& d, uint64_t key, uint32_t bits,
                                          const uint64_t* __restrict__ nkeys) {
  char* p = reinterpret_cast<char*>(o);
  *reinterpret_cast<uint2*>(p + offsetof(alz_edge_out, hist) + 8u * lane) = make_uint2(d.c0, d.c1);
  if (lane < 3u) *reinterpret_cast<uint64_t*>(p + offsetof(alz_edge_out, count) + 8u * lane) = d.s;
  if (lane == 3u) {
    const ulonglong2 hd = edge_head(key, bits, nkeys);
    reinterpret_cast<uint64_t*>(p)[0] = hd.x;
    reinterpret_cast<uint64_t*>(p)[1] = hd.y;
  }
}

// A run's part in a row the split kernel zeroed and headed: one red.add per non-zero word
__device__ __forceinline__ void add_row(alz_edge_out* o, uint32_t lane, const Part& d) {
  char* p = reinterpret_cast<char*>(o);
  uint32_t* cells = reinterpret_cast<uint32_t*>(p + offsetof(alz_edge_out, hist)) + 2u * lane;
  if (d.c0) atomicAdd(cells, d.c0);
  if (d.c1) atomicAdd(cells + 1, d.c1);
  if (lane < 3u && d.s)
    atomicAdd(reinterpret_cast<unsigned long long*>(p + offsetof(alz_edge_out, count) + 8u * lane),
              (unsigned long long)d.s);
}

// Block b: sorted rows [b x kBlockRows, ...), warp w the kWarpRows from b x kBlockRows + w x kWarpRows, by the rule at
// the top of the file. A warp's part of a run open at its chunk's start goes to slot 0, of one open at its end to slot
// 1 (a run open at both: slot 0); s_open says which ends are open (bit 0 start, bit 1 end; 0: the slot is empty).
__global__ void __launch_bounds__(kWarps * 32) group_reduce_kernel(const alz_edge_out* __restrict__ rows,
                                                                   const uint64_t* __restrict__ keys,
                                                                   const uint32_t* __restrict__ vals,
                                                                   const uint32_t* __restrict__ heads,
                                                                   const uint32_t* __restrict__ idx, uint32_t n,
                                                                   uint32_t bits, const uint64_t* __restrict__ nkeys,
                                                                   alz_edge_out* __restrict__ out) {
  __shared__ uint64_t s_part[kWarps][2][kSlotWords];
  __shared__ uint64_t s_key[kWarps][2];
  __shared__ uint32_t s_out[kWarps][2];
  __shared__ uint32_t s_open[kWarps][2];
  const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
  const uint32_t lo = blockIdx.x * kBlockRows + w * kWarpRows;
  if (lane == 0) s_open[w][0] = s_open[w][1] = 0u;
  if (lo < n) {
    const uint32_t hi = min(lo + kWarpRows, n);
    const bool open_lo = lo > 0 && keys[lo - 1] == keys[lo];
    const bool open_hi = hi < n && keys[hi] == keys[hi - 1];
    uint32_t o = idx[lo] + heads[lo] - 1u;   // the current run's group-edge row
    uint64_t cur = keys[lo];
    bool first = true;                       // the current run is the chunk's first
    Part d;
    d.zero();
    // one run of the chunk ends: stored plainly when it is closed on both sides, else left in its slot
    auto finish = [&](bool at_hi) {
      const bool ol = first && open_lo, oh = at_hi && open_hi;
      if (!ol && !oh) {
        store_row(out + o, lane, d, cur, bits, nkeys);
        return;
      }
      const uint32_t slot = ol ? 0u : 1u;
      s_part[w][slot][3 + lane] = ((uint64_t)d.c1 << 32) | d.c0;
      if (lane < 3u) s_part[w][slot][lane] = d.s;
      if (lane == 0) {
        s_key[w][slot] = cur;
        s_out[w][slot] = o;
        s_open[w][slot] = (ol ? 1u : 0u) | (oh ? 2u : 0u);
      }
    };
    for (uint32_t base = lo; base < hi; base += 32u) {
      const uint32_t len = min(32u, hi - base);
      const uint64_t my_key = lane < len ? keys[base + lane] : 0ull;
      const uint32_t my_val = lane < len ? vals[base + lane] : 0u;
      for (uint32_t j0 = 0; j0 < len; j0 += 4u) {
        uint2 c[4];
        uint64_t s[4], k[4];
#pragma unroll
        for (uint32_t q = 0; q < 4; ++q) {   // four rows' loads in flight; past len, the batch's last row again
          const uint32_t j = min(j0 + q, len - 1u);
          k[q] = __shfl_sync(0xFFFFFFFFu, my_key, j);
          load_part(rows + __shfl_sync(0xFFFFFFFFu, my_val, j), lane, &c[q], &s[q]);
        }
#pragma unroll
        for (uint32_t q = 0; q < 4; ++q) {
          if (j0 + q >= len) break;
          if (k[q] != cur) {
            finish(false);
            first = false;
            cur = k[q];
            o += 1u;
            d.zero();
          }
          d.c0 += c[q].x;
          d.c1 += c[q].y;
          d.s += s[q];
        }
      }
    }
    finish(true);
  }
  __syncthreads();
  // Slot (w, 0) or (w, 1) starts a run's chain unless it continues one from warp w - 1 (open at its start, w > 0).
  // The chain follows the next warps' slot 0 while the run stays open at a chunk's end.
#pragma unroll
  for (uint32_t slot = 0; slot < 2; ++slot) {
    const uint32_t op = s_open[w][slot];
    if (op == 0u || ((op & 1u) && w > 0)) continue;
    Part t;
    t.c0 = (uint32_t)s_part[w][slot][3 + lane];
    t.c1 = (uint32_t)(s_part[w][slot][3 + lane] >> 32);
    t.s = lane < 3u ? s_part[w][slot][lane] : 0ull;
    uint32_t last = op, v = w;
    while ((last & 2u) && v + 1 < kWarps) {
      ++v;
      last = s_open[v][0];
      const uint64_t q = s_part[v][0][3 + lane];
      t.c0 += (uint32_t)q;
      t.c1 += (uint32_t)(q >> 32);
      if (lane < 3u) t.s += s_part[v][0][lane];
    }
    alz_edge_out* o = out + s_out[w][slot];
    if ((op & 1u) || (last & 2u)) add_row(o, lane, t);   // the run crosses the block's start or end
    else store_row(o, lane, t, s_key[w][slot], bits, nkeys);
  }
}

}  // namespace

// The group map and the buffers of the group calls, each grown on demand and never shrunk; freed in alz_destroy
struct alz_group_state {
  DevBuf map_keys, map_groups;   // the map: node keys ascending, each one's group
  uint32_t map_n = 0;
  uint64_t map_gen = 0;          // successful alz_group_set calls: tells the group changes' cached baseline groups stale
  NodeGroup ends, edge_keys;     // the group-by of the mapped ends, then of the group-edge keys; ends also serves the
                                 // group nodes' group-by once the group edges are enqueued
  DevBuf end_idx, nkeys, ctr;    // each end's node index, each node's key, the ends kernel's two counters
  DevBuf edges, node_rows, values, top_rows;   // the results
  Selection sel;
  uint64_t* h_ctr = nullptr;     // pinned: the two counters
};

void alz_internal_free_groups(alz_handle* h) {
  alz_group_state* s = h->groups;
  if (!s) return;
  s->ends.free();
  s->edge_keys.free();
  free_bufs({&s->map_keys, &s->map_groups, &s->end_idx, &s->nkeys, &s->ctr, &s->edges, &s->node_rows, &s->values,
             &s->top_rows});
  s->sel.free();
  if (s->h_ctr) cudaFreeHost(s->h_ctr);
  delete s;
  h->groups = nullptr;
}

namespace {

alz_group_state* state(alz_handle* h) {
  if (!h->groups) h->groups = new alz_group_state();
  return h->groups;
}

bool valid_source(uint32_t source) { return source == ALZ_SOURCE_WINDOW || source <= ALZ_ROLLUP_SPAN; }

// a node a flush can produce: a type up to ALZ_NODE_OUTBOUND_HOST, a pod or service value below 2^29
bool valid_member(const alz_node_ends& e) { return valid_node_key(e.type, e.value); }

// ceil(log2(u)), at least 1
uint32_t index_bits(uint64_t u) {
  uint32_t b = 1;
  while ((1ull << b) < u) ++b;
  return b;
}

}  // namespace

// The group-edge rows of n rows into `out`, on the stream after two waits: *n_out = their count, *info what §24
// reports. More than cap: ALZ_E_CAPACITY before the reduce is enqueued. Caller holds h->mu and has set the device;
// n <= kMaxNodeSourceRows.
int alz::metrics::group_edges_into(alz_handle* h, DevBuf& out_buf, const alz_edge_out* rows, size_t n, size_t cap,
                                   size_t* n_out, alz_group_info* info) {
  *n_out = 0;
  *info = alz_group_info{};
  info->source_rows = n;
  alz_group_state* s = state(h);
  if (n == 0) return reserve(h, {{&out_buf, sizeof(alz_edge_out)}});
  if (!s->h_ctr) {
    void* p = nullptr;
    if (cudaMallocHost(&p, 2 * sizeof(uint64_t)) != cudaSuccess) {
      h->last_err = std::string("groups: ") + cudaGetErrorString(cudaGetLastError());
      return ALZ_E_NOMEM;
    }
    s->h_ctr = static_cast<uint64_t*>(p);
  }
  const uint32_t n1 = (uint32_t)n, n2 = 2u * n1;
  int rc = node_group_reserve(h, s->ends, n2);
  if (rc == ALZ_OK) rc = node_group_reserve(h, s->edge_keys, n1);
  if (rc == ALZ_OK) rc = reserve(h, {{&s->end_idx, (size_t)n2 * 4}, {&s->nkeys, (size_t)n2 * 8}, {&s->ctr, 16}});
  if (rc != ALZ_OK) return rc;
  cudaStream_t st = h->stream;
  unsigned long long* ctr = static_cast<unsigned long long*>(s->ctr.p);
  CK(cudaMemsetAsync(ctr, 0, 16, st));
  group_ends_kernel<<<grid_for(h, n1, 8), 256, 0, st>>>(
      rows, n1, static_cast<const uint64_t*>(s->map_keys.p), static_cast<const uint32_t*>(s->map_groups.p), s->map_n,
      static_cast<uint64_t*>(s->ends.keys_in.p), static_cast<uint32_t*>(s->ends.vals_in.p), ctr);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(s->h_ctr, ctr, 16, cudaMemcpyDeviceToHost, st));
  h->launches += 1;
  rc = node_group_runs(h, s->ends, n2, kNodeKeyBits);   // waits: the node count, the counters
  if (rc != ALZ_OK) return rc;
  info->mapped_ends = s->h_ctr[0];
  info->internal = s->h_ctr[1];
  const uint32_t bits = index_bits(s->ends.h_words[0]);
  uint32_t* end_idx = static_cast<uint32_t*>(s->end_idx.p);
  const uint64_t* nkeys = static_cast<const uint64_t*>(s->nkeys.p);
  group_index_kernel<<<grid_for(h, n2, 8), 256, 0, st>>>(
      static_cast<const uint64_t*>(s->ends.keys_out.p), static_cast<const uint32_t*>(s->ends.vals_out.p),
      static_cast<const uint32_t*>(s->ends.heads.p), static_cast<const uint32_t*>(s->ends.idx.p), n2, end_idx,
      static_cast<uint64_t*>(s->nkeys.p));
  group_edge_keys_kernel<<<grid_for(h, n1, 8), 256, 0, st>>>(end_idx, n1, bits,
                                                             static_cast<uint64_t*>(s->edge_keys.keys_in.p),
                                                             static_cast<uint32_t*>(s->edge_keys.vals_in.p));
  h->launches += 2;
  rc = node_group_runs(h, s->edge_keys, n1, (int)(2 * bits));   // waits: the group-edge count
  if (rc != ALZ_OK) return rc;
  const size_t edges = s->edge_keys.h_words[0];
  info->edges = edges;
  *n_out = edges;
  if (edges > cap) return ALZ_E_CAPACITY;
  rc = reserve(h, {{&out_buf, edges * sizeof(alz_edge_out)}});
  if (rc != ALZ_OK) return rc;
  alz_edge_out* out = static_cast<alz_edge_out*>(out_buf.p);
  const uint64_t* keys = static_cast<const uint64_t*>(s->edge_keys.keys_out.p);
  const uint32_t* idx = static_cast<const uint32_t*>(s->edge_keys.idx.p);
  if (n1 > kBlockRows) {
    group_split_kernel<<<grid_for(h, (uint64_t)((n1 - 1) / kBlockRows) * 32, 8), 256, 0, st>>>(keys, idx, n1, bits,
                                                                                               nkeys, out);
    h->launches += 1;
  }
  group_reduce_kernel<<<(n1 + kBlockRows - 1) / kBlockRows, kWarps * 32, 0, st>>>(
      rows, keys, static_cast<const uint32_t*>(s->edge_keys.vals_out.p),
      static_cast<const uint32_t*>(s->edge_keys.heads.p), idx, n1, bits, nkeys, out);
  h->launches += 1;
  CK(cudaGetLastError());
  return ALZ_OK;
}

int alz::metrics::group_nodes_into(alz_handle* h, DevBuf& out, const alz_edge_out* edges, size_t n, size_t* n_nodes) {
  return node_rows_of(h, state(h)->ends, out, edges, n, SIZE_MAX, n_nodes);
}

uint64_t alz::metrics::group_map_generation(const alz_handle* h) { return h->groups ? h->groups->map_gen : 0; }

GroupMap alz::metrics::group_map(const alz_handle* h) {
  GroupMap m;
  if (!h->groups) return m;
  m.keys = static_cast<const uint64_t*>(h->groups->map_keys.p);
  m.groups = static_cast<const uint32_t*>(h->groups->map_groups.p);
  m.n = h->groups->map_n;
  return m;
}

namespace {

// The group-edge rows of n rows into s->edges (group_edges_into)
int group_edges(alz_handle* h, const alz_edge_out* rows, size_t n, size_t cap, size_t* n_out, alz_group_info* info) {
  return group_edges_into(h, state(h)->edges, rows, n, cap, n_out, info);
}

// The rows of a source (node_source's rules) or of the hook's caller rows
int input_rows(alz_handle* h, bool hook, uint32_t source, const alz_edge_out** rows, size_t* n) {
  if (hook) return *n > kMaxNodeSourceRows ? ALZ_E_CAPACITY : ALZ_OK;
  return node_source(h, source, rows, n);
}

// alz_group_edges* and alz_debug_group_edges. Device variant: *dev set; host variant: cap rows in out, one more wait.
int edges_entry(alz_handle* h, bool hook, uint32_t source, const alz_edge_out* dev_rows, size_t n_rows,
                alz_edge_out* out, size_t cap, const alz_edge_out** dev, size_t* n_out, alz_group_info* info) {
  if (!n_out) return ALZ_E_INVAL;
  *n_out = 0;
  if (info) *info = alz_group_info{};
  if (!h || (!dev && !out && cap) || (hook ? (!dev_rows && n_rows) : !valid_source(source))) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  const alz_edge_out* rows = dev_rows;
  size_t n = n_rows;
  int rc = input_rows(h, hook, source, &rows, &n);
  if (rc != ALZ_OK) return rc;
  alz_group_info gi;
  rc = group_edges(h, rows, n, dev ? SIZE_MAX : cap, n_out, &gi);
  if (info) *info = gi;
  if (rc != ALZ_OK) return rc;
  const alz_edge_out* res = static_cast<const alz_edge_out*>(h->groups->edges.p);
  if (dev) {
    *dev = res;
    return ALZ_OK;
  }
  if (*n_out) CK(cudaMemcpyAsync(out, res, *n_out * sizeof(alz_edge_out), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return ALZ_OK;
}

// The group-edge rows of a source, then, with nodes, their §21 node rows: *n = the rows or nodes. More than cap:
// ALZ_E_CAPACITY. Caller holds h->mu and has set the device.
int source_groups(alz_handle* h, uint32_t source, bool nodes, size_t cap, size_t* n) {
  const alz_edge_out* rows = nullptr;
  size_t n_rows = 0, edges = 0;
  int rc = node_source(h, source, &rows, &n_rows);
  if (rc != ALZ_OK) return rc;
  alz_group_info gi;
  rc = group_edges(h, rows, n_rows, nodes ? SIZE_MAX : cap, &edges, &gi);
  *n = edges;
  if (rc != ALZ_OK || !nodes) return rc;
  alz_group_state* s = h->groups;
  return node_rows_of(h, s->ends, s->node_rows, static_cast<const alz_edge_out*>(s->edges.p), edges, cap, n);
}

// alz_group_nodes*: the group nodes. Device variant: *dev set; host: cap nodes.
int nodes_entry(alz_handle* h, uint32_t source, alz_node_out* out, size_t cap, const alz_node_out** dev,
                size_t* n_out) {
  if (!n_out) return ALZ_E_INVAL;
  *n_out = 0;
  if (!h || (!dev && !out && cap) || !valid_source(source)) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  const int rc = source_groups(h, source, true, dev ? SIZE_MAX : cap, n_out);
  if (rc != ALZ_OK) return rc;
  const alz_node_out* res = static_cast<const alz_node_out*>(h->groups->node_rows.p);
  if (dev) {
    *dev = res;
    return ALZ_OK;
  }
  if (*n_out) CK(cudaMemcpyAsync(out, res, *n_out * sizeof(alz_node_out), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return ALZ_OK;
}

// alz_group_edge_metrics* (nodes false) and alz_group_node_metrics* (nodes true, one side). Device variant: *dev set;
// host: cap rows or nodes.
int metrics_entry(alz_handle* h, uint32_t source, bool nodes, uint32_t side, const alz_metric* m, uint32_t nm,
                  double* values, size_t cap, const double** dev, size_t* n_out) {
  if (!n_out) return ALZ_E_INVAL;
  *n_out = 0;
  MetricSet ms;
  if (!h || !valid_source(source) || side > ALZ_SIDE_OUT || !valid_metrics(m, nm, &ms) || (!dev && !values && cap))
    return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  int rc = source_groups(h, source, nodes, dev ? SIZE_MAX : cap, n_out);
  if (rc != ALZ_OK) return rc;
  alz_group_state* s = h->groups;
  const size_t n = *n_out;
  rc = reserve(h, {{&s->values, std::max<size_t>(n * nm, 1) * 8}});
  if (rc != ALZ_OK) return rc;
  double* vals = static_cast<double*>(s->values.p);
  rc = nodes ? run_metrics_nodes(h, NodeRows{static_cast<const alz_node_out*>(s->node_rows.p), side}, (uint32_t)n, ms,
                                 vals)
             : run_metrics(h, static_cast<const alz_edge_out*>(s->edges.p), (uint32_t)n, ms, vals);
  if (rc != ALZ_OK) return rc;
  if (dev) {
    *dev = vals;
    return ALZ_OK;
  }
  if (n) CK(cudaMemcpyAsync(values, vals, n * nm * 8, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return ALZ_OK;
}

// alz_group_edge_top* (nodes false: group-edge rows into rows_out) and alz_group_node_top* (nodes true: node rows into
// nodes_out): one metric, the selection and the gather of the selected rows
int top_entry(alz_handle* h, uint32_t source, bool nodes, uint32_t side, const alz_metric* m, uint32_t k,
              double min_value, alz_edge_out* rows_out, alz_node_out* nodes_out, double* values, uint32_t* index,
              size_t cap, bool device, const void** dev_rows, const double** dev_values, const uint32_t** dev_index,
              size_t* n_out, alz_top_info* info) {
  if (!n_out) return ALZ_E_INVAL;
  *n_out = 0;
  if (info) *info = alz_top_info{};
  MetricSet ms;
  if (!h || !valid_source(source) || side > ALZ_SIDE_OUT || k == 0 || std::isnan(min_value) ||
      !valid_metrics(m, 1, &ms))
    return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  size_t n = 0;
  int rc = source_groups(h, source, nodes, SIZE_MAX, &n);
  if (rc != ALZ_OK) return rc;
  alz_group_state* s = h->groups;
  rc = reserve(h, {{&s->values, std::max<size_t>(n, 1) * 8}});
  if (rc != ALZ_OK) return rc;
  const alz_edge_out* edges = static_cast<const alz_edge_out*>(s->edges.p);
  const alz_node_out* node_rows = static_cast<const alz_node_out*>(s->node_rows.p);
  rc = nodes ? run_metrics_nodes(h, NodeRows{node_rows, side}, (uint32_t)n, ms, static_cast<double*>(s->values.p))
             : run_metrics(h, edges, (uint32_t)n, ms, static_cast<double*>(s->values.p));
  if (rc != ALZ_OK) return rc;
  size_t mm = 0;
  uint64_t above = 0;
  rc = select_top(h, s->sel, static_cast<const uint64_t*>(s->values.p), (uint32_t)n, k, min_value,
                  nodes ? nullptr : edges, &mm, &above);
  if (rc != ALZ_OK) return rc;
  const void* top_rows = s->sel.top_rows.p;
  size_t row_bytes = sizeof(alz_edge_out);
  if (nodes) {
    rc = reserve(h, {{&s->top_rows, std::max<size_t>(mm, 1) * sizeof(alz_node_out)}});
    if (rc != ALZ_OK) return rc;
    rc = node_gather(h, static_cast<const uint32_t*>(s->sel.top_index.p), (uint32_t)mm, node_rows,
                     static_cast<alz_node_out*>(s->top_rows.p));
    if (rc != ALZ_OK) return rc;
    top_rows = s->top_rows.p;
    row_bytes = sizeof(alz_node_out);
  }
  *n_out = mm;
  if (info) { info->scored = n; info->above = above; }
  if (device) {
    if (dev_rows) *dev_rows = top_rows;
    if (dev_values) *dev_values = static_cast<const double*>(s->sel.top_values.p);
    if (dev_index) *dev_index = static_cast<const uint32_t*>(s->sel.top_index.p);
    return ALZ_OK;
  }
  if (mm > cap) return ALZ_E_CAPACITY;
  cudaStream_t st = h->stream;
  void* host_rows = nodes ? static_cast<void*>(nodes_out) : static_cast<void*>(rows_out);
  if (mm && host_rows) CK(cudaMemcpyAsync(host_rows, top_rows, mm * row_bytes, cudaMemcpyDeviceToHost, st));
  if (mm && values) CK(cudaMemcpyAsync(values, s->sel.top_values.p, mm * 8, cudaMemcpyDeviceToHost, st));
  if (mm && index) CK(cudaMemcpyAsync(index, s->sel.top_index.p, mm * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return ALZ_OK;
}

// The new map in buffers of its own: the pairs sorted on the device, then checked for a repeated node (one wait).
// The handle's map is replaced only when every step succeeded.
int set_map(alz_handle* h, const alz_node_ends* nodes, const uint32_t* groups, size_t n) {
  alz_group_state* s = state(h);
  if (n == 0) {
    free_bufs({&s->map_keys, &s->map_groups});
    s->map_n = 0;
    s->map_gen += 1;
    return ALZ_OK;
  }
  std::vector<uint64_t> keys(n);
  for (size_t i = 0; i < n; ++i) keys[i] = ((uint64_t)nodes[i].type << 32) | nodes[i].value;
  DevBuf k_in, k_out, g_in, g_out, tmp, flag;
  auto fail = [&](int rc) {
    cudaStreamSynchronize(h->stream);
    free_bufs({&k_in, &k_out, &g_in, &g_out, &tmp, &flag});
    return rc;
  };
  const uint32_t m = (uint32_t)n;
  const std::initializer_list<std::pair<DevBuf*, size_t>> need = {
      {&k_in, n * 8}, {&k_out, n * 8}, {&g_in, n * 4}, {&g_out, n * 4},
      {&tmp, std::max<size_t>(sort_pairs_temp_bytes(m), 1)}, {&flag, 4}};
  for (auto [b, bytes] : need) {
    if (cudaMalloc(&b->p, bytes) != cudaSuccess) {
      b->p = nullptr;
      h->last_err = std::string("group map: ") + cudaGetErrorString(cudaGetLastError());
      return fail(ALZ_E_NOMEM);
    }
    b->bytes = bytes;
  }
  cudaStream_t st = h->stream;
  uint32_t dup = 0;
  cudaError_t e = cudaMemcpyAsync(k_in.p, keys.data(), n * 8, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(g_in.p, groups, n * 4, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(flag.p, 0, 4, st);
  if (e == cudaSuccess)
    e = sort_pairs(tmp.p, tmp.bytes, static_cast<const uint64_t*>(k_in.p), static_cast<uint64_t*>(k_out.p),
                   static_cast<const uint32_t*>(g_in.p), static_cast<uint32_t*>(g_out.p), m, st, kNodeKeyBits);
  if (e == cudaSuccess) {
    map_dup_kernel<<<grid_for(h, m, 8), 256, 0, st>>>(static_cast<const uint64_t*>(k_out.p), m,
                                                       static_cast<uint32_t*>(flag.p));
    h->launches += 2;
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(&dup, flag.p, 4, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) {
    h->last_err = std::string("group map: ") + cudaGetErrorString(e);
    return fail(ALZ_E_CUDA);
  }
  if (dup) return fail(ALZ_E_INVAL);
  free_bufs({&s->map_keys, &s->map_groups, &k_in, &g_in, &tmp, &flag});
  s->map_keys = k_out;
  s->map_groups = g_out;
  s->map_n = m;
  s->map_gen += 1;
  return ALZ_OK;
}

}  // namespace

extern "C" int alz_group_set(alz_handle* h, const alz_node_ends* nodes, const uint32_t* groups, size_t n) {
  if (!h || (n && (!nodes || !groups))) return ALZ_E_INVAL;
  if (n > kMaxMap) return ALZ_E_CAPACITY;
  for (size_t i = 0; i < n; ++i)
    if (!valid_member(nodes[i]) || groups[i] >= (1u << 29)) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  return set_map(h, nodes, groups, n);
}

extern "C" int alz_group_edges(alz_handle* h, uint32_t source, alz_edge_out* out, size_t cap, size_t* n_out,
                               alz_group_info* info) {
  return edges_entry(h, false, source, nullptr, 0, out, cap, nullptr, n_out, info);
}

extern "C" int alz_group_edges_device(alz_handle* h, uint32_t source, const alz_edge_out** dev_out, size_t* n_out,
                                      alz_group_info* info) {
  if (!dev_out) return n_out ? (*n_out = 0, ALZ_E_INVAL) : ALZ_E_INVAL;
  return edges_entry(h, false, source, nullptr, 0, nullptr, 0, dev_out, n_out, info);
}

extern "C" int alz_group_edge_metrics(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t nm, double* values,
                                      size_t cap, size_t* n_out) {
  return metrics_entry(h, source, false, ALZ_SIDE_IN, m, nm, values, cap, nullptr, n_out);
}

extern "C" int alz_group_edge_metrics_device(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t nm,
                                             const double** dev_values, size_t* n_out) {
  if (!dev_values) return n_out ? (*n_out = 0, ALZ_E_INVAL) : ALZ_E_INVAL;
  return metrics_entry(h, source, false, ALZ_SIDE_IN, m, nm, nullptr, 0, dev_values, n_out);
}

extern "C" int alz_group_edge_top(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t k, double min_value,
                                  alz_edge_out* rows, double* values, uint32_t* index, size_t cap, size_t* n_out,
                                  alz_top_info* info) {
  return top_entry(h, source, false, ALZ_SIDE_IN, m, k, min_value, rows, nullptr, values, index, cap, false, nullptr,
                   nullptr, nullptr, n_out, info);
}

extern "C" int alz_group_edge_top_device(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t k,
                                         double min_value, const alz_edge_out** dev_rows, const double** dev_values,
                                         const uint32_t** dev_index, size_t* n_out, alz_top_info* info) {
  return top_entry(h, source, false, ALZ_SIDE_IN, m, k, min_value, nullptr, nullptr, nullptr, nullptr, 0, true,
                   reinterpret_cast<const void**>(dev_rows), dev_values, dev_index, n_out, info);
}

extern "C" int alz_group_nodes(alz_handle* h, uint32_t source, alz_node_out* out, size_t cap, size_t* n_out) {
  return nodes_entry(h, source, out, cap, nullptr, n_out);
}

extern "C" int alz_group_nodes_device(alz_handle* h, uint32_t source, const alz_node_out** dev_out, size_t* n_out) {
  if (!dev_out) return n_out ? (*n_out = 0, ALZ_E_INVAL) : ALZ_E_INVAL;
  return nodes_entry(h, source, nullptr, 0, dev_out, n_out);
}

extern "C" int alz_group_node_metrics(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t nm,
                                      double* values, size_t cap, size_t* n_out) {
  return metrics_entry(h, source, true, side, m, nm, values, cap, nullptr, n_out);
}

extern "C" int alz_group_node_metrics_device(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m,
                                             uint32_t nm, const double** dev_values, size_t* n_out) {
  if (!dev_values) return n_out ? (*n_out = 0, ALZ_E_INVAL) : ALZ_E_INVAL;
  return metrics_entry(h, source, true, side, m, nm, nullptr, 0, dev_values, n_out);
}

extern "C" int alz_group_node_top(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t k,
                                  double min_value, alz_node_out* nodes, double* values, uint32_t* index, size_t cap,
                                  size_t* n_out, alz_top_info* info) {
  return top_entry(h, source, true, side, m, k, min_value, nullptr, nodes, values, index, cap, false, nullptr, nullptr,
                   nullptr, n_out, info);
}

extern "C" int alz_group_node_top_device(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m,
                                         uint32_t k, double min_value, const alz_node_out** dev_nodes,
                                         const double** dev_values, const uint32_t** dev_index, size_t* n_out,
                                         alz_top_info* info) {
  return top_entry(h, source, true, side, m, k, min_value, nullptr, nullptr, nullptr, nullptr, 0, true,
                   reinterpret_cast<const void**>(dev_nodes), dev_values, dev_index, n_out, info);
}

extern "C" int alz_debug_group_edges(alz_handle* h, const alz_edge_out* dev_rows, size_t n, alz_edge_out* out,
                                     size_t cap, size_t* n_out, alz_group_info* info) {
  return edges_entry(h, true, 0, dev_rows, n, out, cap, nullptr, n_out, info);
}
