// alz_nodes.cu — node metrics (docs/SPEC.md §21): a source's rows grouped by node, each node with the sums of the rows
// into it (side IN) and out of it (side OUT), the §17 metrics of one side, and the top nodes by one of them. Reads the
// source rows only; touches no GNN, metric, change, series or trend state.
//
//   keys    2n (node key, 2 x row + side) pairs: the to end of each row (IN) and its from end (OUT)
//   sort    CUB's radix sort of the pairs on the key's 40 bits (a uint8 type above a 32-bit value): five 8-bit passes,
//           as many as the 34 bits of the four node types need
//   group   run heads of the sorted keys, one exclusive scan into node indices, one wait that reads the node count
//   reduce  the sorted pairs in tiles of kTile, one 8-lane group per tile (lane l owns cells 8l..8l+7 of both sides,
//           lanes 0..2 one of the three sums): each node's pairs in the tile are summed in registers. A run inside one
//           tile is stored plainly, with the node's type, value and edge counts. A run that crosses a tile boundary
//           (a hub) was zeroed and headed by the split kernel, and each of its tiles adds its part with red.add. The
//           arithmetic is integer, mod 2^64 and mod 2^32, so every order of the adds gives the same bytes.
//   The sort, heads and scan (node_group_runs) and the split and reduce (node_group_reduce) work on a NodeGroup their
//   caller owns: the node series (alz_node_series.cu) run them a second time over (node, point) pairs.
//   metrics the §17 kernels through NodeRows, which reads one side of a node row in place as an alz_edge_out
//   top     the §17 selection over those values, then one gather of the selected node rows
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <mutex>
#include <string>

#include "alz_metrics.cuh"

using namespace alz;
using namespace alz::metrics;

static_assert(sizeof(alz_node_sums) == 280, "alz_node_sums is the tail of alz_edge_out from count on");
static_assert(sizeof(alz_node_out) == 576 && sizeof(alz_node_out) % 16 == 0, "alz_node_out is 36 16-byte words");
static_assert(offsetof(alz_node_out, in) + offsetof(alz_node_sums, count) == offsetof(alz_edge_out, count),
              "NodeRows reads side IN of a node row in place as an alz_edge_out");
static_assert(offsetof(alz_node_out, out) == offsetof(alz_node_out, in) + sizeof(alz_node_sums),
              "NodeRows reads side OUT one alz_node_sums further on");
static_assert(offsetof(alz_node_sums, err5xx) - offsetof(alz_node_sums, count) ==
                      offsetof(alz_edge_out, err5xx) - offsetof(alz_edge_out, count) &&
                  offsetof(alz_node_sums, lat_sum_ns) - offsetof(alz_node_sums, count) ==
                      offsetof(alz_edge_out, lat_sum_ns) - offsetof(alz_edge_out, count) &&
                  offsetof(alz_node_sums, hist) - offsetof(alz_node_sums, count) ==
                      offsetof(alz_edge_out, hist) - offsetof(alz_edge_out, count),
              "a side's sums are laid out as alz_edge_out's");

namespace {

constexpr uint32_t kTile = 32;                         // pairs per lane group; a longer run is split across groups
constexpr uint32_t kGroups = 256 / 8;                  // lane groups per block
constexpr uint32_t kRowWords = sizeof(alz_node_out) / 8;

// the row's fields at byte offset 8 x w (8-byte aligned: rows are 296 bytes apart)
__device__ __forceinline__ uint2 ld2(const alz_edge_out* r, uint32_t byte_off) {
  return *reinterpret_cast<const uint2*>(reinterpret_cast<const char*>(r) + byte_off);
}

// Pair 2i + side: the node key of row i's to end (ALZ_SIDE_IN) or from end (ALZ_SIDE_OUT), and its own position
__global__ void __launch_bounds__(256) node_keys_kernel(const alz_edge_out* __restrict__ rows, uint32_t n,
                                                        uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  static_assert(ALZ_SIDE_IN == 0u && ALZ_SIDE_OUT == 1u, "pair 2i + side");
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint2 ty = ld2(rows + i, 0), ft = ld2(rows + i, 8);   // from_type, to_type, pad | from, to
    reinterpret_cast<ulonglong2*>(keys)[i] = make_ulonglong2(node_key((ty.x >> 8) & 0xFFu, ft.y), node_key(ty.x & 0xFFu, ft.x));
    reinterpret_cast<uint2*>(vals)[i] = make_uint2(2u * i, 2u * i + 1u);
  }
}

// heads[j] = 1 where a run of equal keys starts; heads[n2] = 0 closes the scan
__global__ void __launch_bounds__(256) node_heads_kernel(const uint64_t* __restrict__ keys, uint32_t n2,
                                                         uint32_t* __restrict__ heads) {
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x;
  for (uint32_t j = t0; j < n2; j += stride) heads[j] = (j == 0 || keys[j] != keys[j - 1]) ? 1u : 0u;
  if (t0 == 0) heads[n2] = 0u;
}

// the node row's first word: type, zero padding, value
__device__ __forceinline__ uint64_t head_word(uint64_t key) { return (key >> 32) | (key << 32); }

// Warp w: tile boundary b = (w + 1) x kTile. When one run crosses b, its node row is zeroed with its type and value
// set, for the reduce's red.add. A run over several boundaries is written once per boundary, with the same bytes.
__global__ void __launch_bounds__(256) node_split_kernel(const uint64_t* __restrict__ keys,
                                                         const uint32_t* __restrict__ idx, uint32_t n2,
                                                         alz_node_out* __restrict__ out) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t bounds = (n2 - 1u) / kTile;   // boundaries strictly inside [0, n2)
  for (uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < bounds; w += warps) {
    const uint32_t b = (w + 1u) * kTile;
    const uint64_t key = keys[b];
    if (keys[b - 1] != key) continue;   // a run starts at b: none crosses it
    uint64_t* o = reinterpret_cast<uint64_t*>(out + (idx[b] - 1u));
    for (uint32_t q = lane; q < kRowWords; q += 32u) o[q] = q == 0 ? head_word(key) : 0ull;
  }
}

// The per-lane sums of one side: lane l's cells 8l..8l+7, and for l < 3 the sum at count + 8l
struct Side {
  uint32_t c[8];
  uint64_t s;
  uint32_t rows;
  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int q = 0; q < 8; ++q) c[q] = 0u;
    s = 0ull;
    rows = 0u;
  }
  __device__ __forceinline__ void add(const uint2 (&h)[4], uint64_t v) {
#pragma unroll
    for (int q = 0; q < 4; ++q) { c[2 * q] += h[q].x; c[2 * q + 1] += h[q].y; }
    s += v;
    rows += 1u;
  }
};

// Lane l's part of one side's sums at byte offset `at` of node row o: plain stores or red.add
__device__ __forceinline__ void store_side(alz_node_out* o, uint32_t at, uint32_t lane, const Side& d, bool plain) {
  char* base = reinterpret_cast<char*>(o) + at;
  uint32_t* cells = reinterpret_cast<uint32_t*>(base + 24) + 8u * lane;
  uint64_t* sum = reinterpret_cast<uint64_t*>(base) + lane;
  if (plain) {
#pragma unroll
    for (int q = 0; q < 4; ++q) reinterpret_cast<uint2*>(cells)[q] = make_uint2(d.c[2 * q], d.c[2 * q + 1]);
    if (lane < 3u) *sum = d.s;
  } else {
#pragma unroll
    for (int q = 0; q < 8; ++q)
      if (d.c[q]) atomicAdd(cells + q, d.c[q]);
    if (lane < 3u && d.s) atomicAdd(reinterpret_cast<unsigned long long*>(sum), (unsigned long long)d.s);
  }
}

// Group g (8 lanes) of the grid: tile t = pairs [t x kTile, min((t + 1) x kTile, n2)). Each node's pairs in the tile
// are one segment, summed in registers and stored by the rule at the top of the file.
__global__ void __launch_bounds__(256) node_reduce_kernel(const alz_edge_out* __restrict__ rows,
                                                          const uint64_t* __restrict__ keys,
                                                          const uint32_t* __restrict__ vals,
                                                          const uint32_t* __restrict__ idx, uint32_t n2,
                                                          alz_node_out* __restrict__ out) {
  __shared__ uint64_t s_key[kGroups][kTile + 1];   // [kTile]: the key after the tile (or ~0 past the end)
  __shared__ uint32_t s_val[kGroups][kTile];
  const uint32_t lane = threadIdx.x & 7u, g = threadIdx.x >> 3;
  const unsigned gmask = 0xFFu << (threadIdx.x & 24u);
  const uint32_t tiles = (n2 + kTile - 1u) / kTile;
  const uint32_t groups = (gridDim.x * blockDim.x) >> 3;
  for (uint32_t t = (blockIdx.x * blockDim.x + threadIdx.x) >> 3; t < tiles; t += groups) {
    const uint32_t lo = t * kTile, len = min(kTile, n2 - lo);
    for (uint32_t q = lane; q <= kTile; q += 8u) {
      if (q < len) { s_key[g][q] = keys[lo + q]; s_val[g][q] = vals[lo + q]; }
      else if (q == kTile) s_key[g][q] = lo + kTile < n2 ? keys[lo + kTile] : ~0ull;
    }
    const uint64_t before = lo ? keys[lo - 1] : ~0ull;   // node keys are below 2^40: ~0 matches none
    __syncwarp(gmask);
    uint32_t j = 0;
    while (j < len) {
      const uint64_t key = s_key[g][j];
      const bool head = j ? true : before != key;   // j > 0 starts a segment only where the key changed
      Side in, outs;
      in.zero();
      outs.zero();
      uint32_t e = j;
      for (; e < len && s_key[g][e] == key; ++e) {
        const uint32_t p = s_val[g][e];
        const alz_edge_out* r = rows + (p >> 1);
        uint2 hc[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) hc[q] = ld2(r, (uint32_t)offsetof(alz_edge_out, hist) + 32u * lane + 8u * q);
        uint64_t v = 0;
        if (lane < 3u) {
          const uint2 w = ld2(r, (uint32_t)offsetof(alz_edge_out, count) + 8u * lane);
          v = ((uint64_t)w.y << 32) | w.x;
        }
        if (p & 1u) outs.add(hc, v); else in.add(hc, v);
      }
      // whole: the run starts in this tile and ends in it
      const bool whole = head && (e < len || s_key[g][kTile] != key);
      alz_node_out* o = out + (idx[lo + j] - (head ? 0u : 1u));
      store_side(o, (uint32_t)offsetof(alz_node_out, in), lane, in, whole);
      store_side(o, (uint32_t)offsetof(alz_node_out, out), lane, outs, whole);
      if (lane == 3u) {
        if (whole) {
          reinterpret_cast<uint4*>(o)[0] = make_uint4((uint32_t)(key >> 32), (uint32_t)key, in.rows, outs.rows);
        } else {
          if (in.rows) atomicAdd(&o->in_edges, in.rows);
          if (outs.rows) atomicAdd(&o->out_edges, outs.rows);
        }
      }
      j = e;
    }
    __syncwarp(gmask);   // the group's next tile overwrites its shared rows
  }
}

// result j = node row idx[j], 36 16-byte words each
__global__ void __launch_bounds__(256) node_gather_kernel(const uint32_t* __restrict__ idx, uint32_t m,
                                                          const alz_node_out* __restrict__ nodes,
                                                          alz_node_out* __restrict__ out) {
  constexpr uint32_t kWords = sizeof(alz_node_out) / 16;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < m * kWords; t += stride) {
    const uint32_t j = t / kWords, w = t - j * kWords;
    reinterpret_cast<uint4*>(out + j)[w] = reinterpret_cast<const uint4*>(nodes + idx[j])[w];
  }
}

}  // namespace

// Buffers of the node calls, each grown on demand and never shrunk; freed in alz_destroy
struct alz_node_state {
  NodeGroup g;                      // the group-by's scratch
  DevBuf rows, values, top_rows;    // the results: node rows, metric values, top rows
  Selection sel;                    // the top call's selection
};

void alz::metrics::NodeGroup::free() {
  free_bufs({&keys_in, &keys_out, &vals_in, &vals_out, &heads, &idx, &tmp});
  if (h_words) cudaFreeHost(h_words);
  h_words = nullptr;
}

void alz_internal_free_nodes(alz_handle* h) {
  alz_node_state* s = h->nodes;
  if (!s) return;
  s->g.free();
  free_bufs({&s->rows, &s->values, &s->top_rows});
  s->sel.free();
  delete s;
  h->nodes = nullptr;
}

namespace alz {
namespace metrics {

int node_group_reserve(alz_handle* h, NodeGroup& g, uint32_t n2) {
  if (!g.h_words) {
    void* p = nullptr;
    if (cudaMallocHost(&p, 2 * sizeof(uint32_t)) != cudaSuccess) {
      h->last_err = std::string("node metrics: ") + cudaGetErrorString(cudaGetLastError());
      return ALZ_E_NOMEM;
    }
    g.h_words = static_cast<uint32_t*>(p);
  }
  return reserve(h, {{&g.keys_in, (size_t)n2 * 8},
                     {&g.keys_out, (size_t)n2 * 8},
                     {&g.vals_in, (size_t)n2 * 4},
                     {&g.vals_out, (size_t)n2 * 4},
                     {&g.heads, ((size_t)n2 + 1) * 4},
                     {&g.idx, ((size_t)n2 + 1) * 4},
                     {&g.tmp, std::max(sort_pairs_temp_bytes(n2), scan_temp_bytes(n2 + 1))}});
}

void node_group_keys(alz_handle* h, NodeGroup& g, const alz_edge_out* rows, uint32_t n) {
  node_keys_kernel<<<grid_for(h, n, 8), 256, 0, h->stream>>>(rows, n, static_cast<uint64_t*>(g.keys_in.p),
                                                             static_cast<uint32_t*>(g.vals_in.p));
  h->launches += 1;
}

int node_group_runs(alz_handle* h, NodeGroup& g, uint32_t n2, int key_bits) {
  cudaStream_t st = h->stream;
  uint64_t* keys = static_cast<uint64_t*>(g.keys_out.p);
  uint32_t* heads = static_cast<uint32_t*>(g.heads.p);
  uint32_t* idx = static_cast<uint32_t*>(g.idx.p);
  CK(cudaGetLastError());
  CK(sort_pairs(g.tmp.p, g.tmp.bytes, static_cast<const uint64_t*>(g.keys_in.p), keys,
                static_cast<const uint32_t*>(g.vals_in.p), static_cast<uint32_t*>(g.vals_out.p), n2, st, key_bits));
  node_heads_kernel<<<grid_for(h, n2, 8), 256, 0, st>>>(keys, n2, heads);
  CK(cudaGetLastError());
  CK(exclusive_scan_u32(g.tmp.p, g.tmp.bytes, heads, idx, n2 + 1, st));
  CK(cudaMemcpyAsync(g.h_words, idx + n2, 4, cudaMemcpyDeviceToHost, st));
  h->launches += 3;
  CK(cudaStreamSynchronize(st));   // the one wait: the run count
  return ALZ_OK;
}

int node_group_reduce(alz_handle* h, const NodeGroup& g, const alz_edge_out* rows, uint32_t n2, alz_node_out* out) {
  if (n2 == 0) return ALZ_OK;
  cudaStream_t st = h->stream;
  const uint64_t* keys = static_cast<const uint64_t*>(g.keys_out.p);
  const uint32_t* idx = static_cast<const uint32_t*>(g.idx.p);
  if (n2 > kTile) {
    node_split_kernel<<<grid_for(h, (uint64_t)((n2 - 1) / kTile) * 32, 8), 256, 0, st>>>(keys, idx, n2, out);
    h->launches += 1;
  }
  const uint64_t tiles = (n2 + kTile - 1) / kTile;
  node_reduce_kernel<<<grid_for(h, tiles * 8, 8), 256, 0, st>>>(rows, keys, static_cast<const uint32_t*>(g.vals_out.p),
                                                                idx, n2, out);
  h->launches += 1;
  CK(cudaGetLastError());
  return ALZ_OK;
}

int node_gather(alz_handle* h, const uint32_t* idx, uint32_t m, const alz_node_out* nodes, alz_node_out* out) {
  if (m == 0) return ALZ_OK;
  node_gather_kernel<<<grid_for(h, (uint64_t)m * (sizeof(alz_node_out) / 16), 4), 256, 0, h->stream>>>(idx, m, nodes,
                                                                                                      out);
  h->launches += 1;
  CK(cudaGetLastError());
  return ALZ_OK;
}

int node_source(alz_handle* h, uint32_t source, const alz_edge_out** rows, size_t* n) {
  alz_rollup_info ri;
  const int rc = source_rows(h, source, rows, n, &ri);
  if (rc != ALZ_OK) return rc;
  return *n > kMaxNodeSourceRows ? ALZ_E_CAPACITY : ALZ_OK;
}

int node_rows_of(alz_handle* h, NodeGroup& g, DevBuf& out, const alz_edge_out* rows, size_t n, size_t cap,
                 size_t* n_nodes) {
  *n_nodes = 0;
  const uint32_t n2 = 2u * (uint32_t)n;
  if (n == 0) return reserve(h, {{&out, sizeof(alz_node_out)}});
  int rc = node_group_reserve(h, g, n2);
  if (rc != ALZ_OK) return rc;
  node_group_keys(h, g, rows, (uint32_t)n);
  rc = node_group_runs(h, g, n2, kNodeKeyBits);
  if (rc != ALZ_OK) return rc;
  const size_t nodes = g.h_words[0];
  *n_nodes = nodes;
  if (nodes > cap) return ALZ_E_CAPACITY;
  rc = reserve(h, {{&out, nodes * sizeof(alz_node_out)}});
  if (rc != ALZ_OK) return rc;
  return node_group_reduce(h, g, rows, n2, static_cast<alz_node_out*>(out.p));
}

}  // namespace metrics
}  // namespace alz

namespace {

// The node rows of n rows into s->rows, on the stream after one wait for the node count; *n_nodes = that count. More
// nodes than cap: ALZ_E_CAPACITY before the reduce is enqueued. Caller holds h->mu and has set the device;
// n <= kMaxNodeSourceRows.
int group_nodes(alz_handle* h, const alz_edge_out* rows, size_t n, size_t cap, size_t* n_nodes) {
  if (!h->nodes) h->nodes = new alz_node_state();
  return node_rows_of(h, h->nodes->g, h->nodes->rows, rows, n, cap, n_nodes);
}

bool valid_source(uint32_t source) { return source == ALZ_SOURCE_WINDOW || source <= ALZ_ROLLUP_SPAN; }

// alz_node_rows* and alz_debug_node_rows: the node rows of a source, or of caller rows (hook). Device variant: *dev
// set; host variant: cap nodes in out, one more wait for the copy.
int rows_entry(alz_handle* h, bool hook, uint32_t source, const alz_edge_out* dev_rows, size_t n_rows,
               alz_node_out* out, size_t cap, const alz_node_out** dev, size_t* n_out) {
  if (!n_out) return ALZ_E_INVAL;
  *n_out = 0;
  if (!h || (!dev && !out && cap) || (hook ? (!dev_rows && n_rows) : !valid_source(source))) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  const alz_edge_out* rows = dev_rows;
  size_t n = n_rows;
  int rc = hook ? (n > kMaxNodeSourceRows ? ALZ_E_CAPACITY : ALZ_OK) : node_source(h, source, &rows, &n);
  if (rc != ALZ_OK) return rc;
  rc = group_nodes(h, rows, n, dev ? SIZE_MAX : cap, n_out);
  if (rc != ALZ_OK) return rc;
  const alz_node_out* res = static_cast<const alz_node_out*>(h->nodes->rows.p);
  if (dev) {
    *dev = res;
    return ALZ_OK;
  }
  if (*n_out) CK(cudaMemcpyAsync(out, res, *n_out * sizeof(alz_node_out), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return ALZ_OK;
}

// alz_node_metrics*: the node rows, then the metrics of one side. Device variant: *dev set; host: cap nodes.
int metrics_entry(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t nm, double* values,
                  size_t cap, const double** dev, size_t* n_out) {
  if (!n_out) return ALZ_E_INVAL;
  *n_out = 0;
  MetricSet ms;
  if (!h || !valid_source(source) || side > ALZ_SIDE_OUT || !valid_metrics(m, nm, &ms) || (!dev && !values && cap))
    return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  const alz_edge_out* rows = nullptr;
  size_t n = 0;
  int rc = node_source(h, source, &rows, &n);
  if (rc != ALZ_OK) return rc;
  rc = group_nodes(h, rows, n, dev ? SIZE_MAX : cap, n_out);
  if (rc != ALZ_OK) return rc;
  alz_node_state* s = h->nodes;
  const size_t nodes = *n_out;
  rc = reserve(h, {{&s->values, std::max<size_t>(nodes * nm, 1) * 8}});
  if (rc != ALZ_OK) return rc;
  double* vals = static_cast<double*>(s->values.p);
  rc = run_metrics_nodes(h, NodeRows{static_cast<const alz_node_out*>(s->rows.p), side}, (uint32_t)nodes, ms, vals);
  if (rc != ALZ_OK) return rc;
  if (dev) {
    *dev = vals;
    return ALZ_OK;
  }
  if (nodes) CK(cudaMemcpyAsync(values, vals, nodes * nm * 8, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return ALZ_OK;
}

// alz_node_top*: the node rows, one metric of one side, the selection and the gather of the selected rows
int top_entry(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t k, double min_value,
              alz_node_out* nodes_out, double* values, uint32_t* index, size_t cap, bool device,
              const alz_node_out** dev_nodes, const double** dev_values, const uint32_t** dev_index, size_t* n_out,
              alz_top_info* info) {
  if (!n_out) return ALZ_E_INVAL;
  *n_out = 0;
  if (info) *info = alz_top_info{};
  MetricSet ms;
  if (!h || !valid_source(source) || side > ALZ_SIDE_OUT || k == 0 || std::isnan(min_value) ||
      !valid_metrics(m, 1, &ms))
    return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  const alz_edge_out* rows = nullptr;
  size_t n = 0, nodes = 0;
  int rc = node_source(h, source, &rows, &n);
  if (rc != ALZ_OK) return rc;
  rc = group_nodes(h, rows, n, SIZE_MAX, &nodes);
  if (rc != ALZ_OK) return rc;
  alz_node_state* s = h->nodes;
  rc = reserve(h, {{&s->values, std::max<size_t>(nodes, 1) * 8}});
  if (rc != ALZ_OK) return rc;
  const alz_node_out* node_rows = static_cast<const alz_node_out*>(s->rows.p);
  rc = run_metrics_nodes(h, NodeRows{node_rows, side}, (uint32_t)nodes, ms, static_cast<double*>(s->values.p));
  if (rc != ALZ_OK) return rc;
  size_t mm = 0;
  uint64_t above = 0;
  rc = select_top(h, s->sel, static_cast<const uint64_t*>(s->values.p), (uint32_t)nodes, k, min_value, nullptr, &mm,
                  &above);
  if (rc != ALZ_OK) return rc;
  rc = reserve(h, {{&s->top_rows, std::max<size_t>(mm, 1) * sizeof(alz_node_out)}});
  if (rc != ALZ_OK) return rc;
  cudaStream_t st = h->stream;
  rc = node_gather(h, static_cast<const uint32_t*>(s->sel.top_index.p), (uint32_t)mm, node_rows,
                   static_cast<alz_node_out*>(s->top_rows.p));
  if (rc != ALZ_OK) return rc;
  *n_out = mm;
  if (info) { info->scored = nodes; info->above = above; }
  const alz_node_out* top_rows = static_cast<const alz_node_out*>(s->top_rows.p);
  if (device) {
    if (dev_nodes) *dev_nodes = top_rows;
    if (dev_values) *dev_values = static_cast<const double*>(s->sel.top_values.p);
    if (dev_index) *dev_index = static_cast<const uint32_t*>(s->sel.top_index.p);
    return ALZ_OK;
  }
  if (mm > cap) return ALZ_E_CAPACITY;
  if (mm && nodes_out) CK(cudaMemcpyAsync(nodes_out, top_rows, mm * sizeof(alz_node_out), cudaMemcpyDeviceToHost, st));
  if (mm && values) CK(cudaMemcpyAsync(values, s->sel.top_values.p, mm * 8, cudaMemcpyDeviceToHost, st));
  if (mm && index) CK(cudaMemcpyAsync(index, s->sel.top_index.p, mm * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return ALZ_OK;
}

}  // namespace

extern "C" int alz_node_rows(alz_handle* h, uint32_t source, alz_node_out* out, size_t cap, size_t* n_out) {
  return rows_entry(h, false, source, nullptr, 0, out, cap, nullptr, n_out);
}

extern "C" int alz_node_rows_device(alz_handle* h, uint32_t source, const alz_node_out** dev_out, size_t* n_out) {
  if (!dev_out) return n_out ? (*n_out = 0, ALZ_E_INVAL) : ALZ_E_INVAL;
  return rows_entry(h, false, source, nullptr, 0, nullptr, 0, dev_out, n_out);
}

extern "C" int alz_node_metrics(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t nm,
                                double* values, size_t cap, size_t* n_out) {
  return metrics_entry(h, source, side, m, nm, values, cap, nullptr, n_out);
}

extern "C" int alz_node_metrics_device(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t nm,
                                       const double** dev_values, size_t* n_out) {
  if (!dev_values) return n_out ? (*n_out = 0, ALZ_E_INVAL) : ALZ_E_INVAL;
  return metrics_entry(h, source, side, m, nm, nullptr, 0, dev_values, n_out);
}

extern "C" int alz_node_top(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t k,
                            double min_value, alz_node_out* nodes, double* values, uint32_t* index, size_t cap,
                            size_t* n_out, alz_top_info* info) {
  return top_entry(h, source, side, m, k, min_value, nodes, values, index, cap, false, nullptr, nullptr, nullptr,
                   n_out, info);
}

extern "C" int alz_node_top_device(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t k,
                                   double min_value, const alz_node_out** dev_nodes, const double** dev_values,
                                   const uint32_t** dev_index, size_t* n_out, alz_top_info* info) {
  return top_entry(h, source, side, m, k, min_value, nullptr, nullptr, nullptr, 0, true, dev_nodes, dev_values,
                   dev_index, n_out, info);
}

extern "C" int alz_debug_node_rows(alz_handle* h, const alz_edge_out* dev_rows, size_t n, alz_node_out* out,
                                   size_t cap, size_t* n_out) {
  return rows_entry(h, true, 0, dev_rows, n, out, cap, nullptr, n_out);
}
