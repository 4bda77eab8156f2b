// alz_kernels.cu — sm_90a kernels of the aggregation hot path.
//
// Plan (DESIGN.md §3): the reference resolves every event through the IP->UID
// tables and then emits one row (aggregator/data.go:827-870, :1244). Grouping
// commutes with that join, so the default plan here reduces the stream per
// socket pair (saddr,daddr,direction) first — one dictionary probe and two
// reductions per event — and joins only the DISTINCT pairs against the tables
// (fold_resolve_kernel). ALZ_CFG_EAGER_JOIN keeps the textbook plan (join every
// event, then reduce) for comparison; both give bit-identical edges.
//
// Control flow in the per-event loops is kept warp-convergent on purpose: every
// lane walks the same statements under predicates and meets at __syncwarp()
// between the divergent dictionary probes and the reductions. The first
// version let lanes leave the probe loops on their own paths and the
// reductions then issued with ~2 active lanes per instruction.
#include <algorithm>

#include "alz_kernels.cuh"

namespace alz {

// per-event fields every plan needs
struct Ev {
  uint64_t key;   // make_pair_key(saddr, daddr)
  uint64_t dur;
  uint32_t bucket;
  bool act;       // the reference would hand a row to PersistRequest (before resolve)
  bool rev;       // ReverseDirection applies
  bool err;       // counts as 5xx
  bool hostkey;   // daddr is a Host-header id (ALZ_PROTO_F_HOSTKEY)
};
__device__ __forceinline__ Ev decode(const Rec& r, bool live) {
  Ev e;
  const uint32_t proto = rec_protocol(r), mf = rec_mflags(r);
  e.act = live && emits_request_row(proto, mf);
  e.rev = is_reversed(proto, mf);
  e.hostkey = rec_hostkey(r);
  e.key = make_pair_key(rec_saddr(r), rec_daddr(r));
  e.dur = rec_duration(r);
  e.bucket = latency_bucket(e.dur);
  e.err = is_5xx(proto, rec_status(r));
  return e;
}

// one event into a pair row (sectored layout, alz_device.cuh); v1 plan: one lane per event, three instructions
__device__ __forceinline__ void pair_accumulate(const PairTable& t, uint32_t row, uint32_t bucket, uint64_t dur, bool err) {
  uint64_t* sc = pair_sect(t, row, bucket);
  atomicAdd(reinterpret_cast<uint32_t*>(sc) + (bucket & 3u), 1u);
  atomicAdd((unsigned long long*)(sc + 2), (unsigned long long)dur);
  if (err) atomicAdd((unsigned long long*)(sc + 3), 1ull);
}

__device__ __forceinline__ void flush_thread_counters(Counters* ctr, uint32_t not_request, uint32_t unresolved,
                                                      uint32_t lost) {
  for (int o = 16; o > 0; o >>= 1) {
    not_request += __shfl_xor_sync(0xFFFFFFFFu, not_request, o);
    unresolved += __shfl_xor_sync(0xFFFFFFFFu, unresolved, o);
    lost += __shfl_xor_sync(0xFFFFFFFFu, lost, o);
  }
  if ((threadIdx.x & 31) == 0) {
    if (not_request) atomicAdd(&ctr->not_request, (unsigned long long)not_request);
    if (unresolved) atomicAdd(&ctr->src_unresolved, (unsigned long long)unresolved);
    if (lost) atomicAdd(&ctr->capacity_events, (unsigned long long)lost);
  }
}

// ---------------------------------------------------------------------------
// ingest v1 (ALZ_CFG_NO_SMEM_CACHE): global reductions only
// ---------------------------------------------------------------------------
template <int UNROLL>
__global__ void __launch_bounds__(256) ingest_pairs_kernel(const alz_l7_rec* __restrict__ recs, uint64_t n,
                                                           PairTable pairs, Counters* ctr, const EpEntry* __restrict__ ep,
                                                           uint32_t ep_mask) {
  uint32_t not_request = 0, lost = 0, unresolved = 0;
  const uint32_t lane = threadIdx.x & 31u;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < n; base += stride * UNROLL) {
    Rec r[UNROLL];
    bool live[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const uint64_t j = base + (uint64_t)u * stride + lane;
      live[u] = j < n;
      if (live[u]) r[u] = load_rec(recs + j);
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const Ev e = decode(r[u], live[u]);
      not_request += (live[u] && !e.act) ? 1u : 0u;
      uint32_t row = kLostRow;
      if (e.act) row = find_or_insert_pair(pairs, e.key, e.hostkey ? kPairHost : e.rev ? kPairRev : kPairFwd, ep, ep_mask);
      __syncwarp();
      if (e.act) {
        if (row == kDropRow) ++unresolved;
        else if (row >= kLostRow) ++lost;
        else pair_accumulate(pairs, row, e.bucket, e.dur, e.err);
      }
    }
  }
  flush_thread_counters(ctr, not_request, unresolved, lost);
}

// ---------------------------------------------------------------------------
// ingest, eager plan: join every event, then reduce per edge
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ingest_eager_kernel(const alz_l7_rec* __restrict__ recs, uint64_t n,
                                                           const EpEntry* __restrict__ ep, uint32_t ep_mask,
                                                           EdgeTable edges, Counters* ctr) {
  uint32_t not_request = 0, unresolved = 0, lost = 0;
  const uint32_t lane = threadIdx.x & 31u;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < n; base += stride) {
    const uint64_t j = base + lane;
    const bool live = j < n;
    Rec r = {};
    if (live) r = load_rec(recs + j);
    const Ev e = decode(r, live);
    not_request += (live && !e.act) ? 1u : 0u;
    uint64_t ekey = 0;
    bool ok = false;
    if (e.act) ok = resolve_pair(ep, ep_mask, e.key, e.hostkey ? kPairHost : e.rev ? kPairRev : kPairFwd, &ekey);
    __syncwarp();
    unresolved += (e.act && !ok) ? 1u : 0u;
    uint32_t row = kLostRow;
    if (ok) row = find_or_insert(edges, ekey);
    __syncwarp();
    if (ok) {
      if (row >= kLostRow) ++lost;
      else edge_add(edges, row, e.bucket, e.dur, e.err);
    }
  }
  flush_thread_counters(ctr, not_request, unresolved, lost);
}

// ---------------------------------------------------------------------------
// fold: the hash join proper, on distinct socket pairs. One warp per pair row:
// resolve (saddr,daddr) -> edge, add the row into the edge accumulators and
// zero it. The caller clears the pair dictionary afterwards.
// ---------------------------------------------------------------------------
// pass 1, a thread per pair row: resolve and find the edge row. All the dependent
// table/dictionary probes of a pair sit in one thread, 32 pairs per warp in flight
// (the one-warp-per-row version spent its time in lane 0's probe chain).
__global__ void __launch_bounds__(256) fold_resolve_kernel(PairTable pairs, const EpEntry* __restrict__ ep,
                                                           uint32_t ep_mask, EdgeTable edges, HotState* hot) {
  // the hot-list bookkeeping of this fold starts from zero (fold_pairs_kernel or emit_edges_kernel fills the bins, hot_emit
  // the list; both run after this kernel, the ingest launches that read the list ran before it)
  if (blockIdx.x == 0) {
    if (threadIdx.x < 128) hot->bins[threadIdx.x] = 0u;
    if (threadIdx.x == 0) { hot->n_a = 0u; hot->n_b = 0u; hot->n_s = 0u; }
  }
  const uint32_t n_rows = min(*pairs.n_rows, pairs.max_rows);
  const uint32_t stride = gridDim.x * blockDim.x;
  // rows [0, n_rows) plus the sentinel rows (index n_rows + kind stands for row max_rows + kind)
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_rows + kPairKinds; i += stride) {
    const bool sentinel = i >= n_rows;
    const uint32_t row = sentinel ? pairs.max_rows + (i - n_rows) : i;
    const uint64_t key = sentinel ? kEmptyKey : pairs.row_key[row];
    const uint32_t kind = sentinel ? (i - n_rows) : pairs.row_kind[row];
    if (sentinel) {                                            // the sentinel rows exist even when unused
      uint64_t any = 0;
      for (uint32_t g = 0; g < kSectPerRow; ++g) { const uint64_t* sc = pairs.sect + ((size_t)row * kSectPerRow + g) * 4u; any |= sc[0] | sc[1]; }
      if (any == 0ull) { pairs.row_aux[row] = kDropRow; continue; }
    }
    uint64_t ekey = 0;
    uint32_t erow = kDropRow;                                  // source is not a pod: data.go:829-832
    if (resolve_pair(ep, ep_mask, key, kind, &ekey)) erow = find_or_insert(edges, ekey);
    pairs.row_aux[row] = erow;
  }
}

// One pair row taken by an 8-lane group (mask gmask): lane sl holds sectors 2sl and 2sl+1, that is 64 contiguous
// bytes = cells 8sl..8sl+3 | lat, 5xx partials | cells 8sl+4..8sl+7 | partials. Leaves the next ingest its feedback
// (row_base, row_cnt and the count bin of a forward row), zeroes what was not zero and returns the row's event count,
// the same in all eight lanes. Every lane of the group calls it; `valid` is uniform over the group.
struct PairSlice { uint4 a, pa, b, pb; };
// The count bins of the hot list are summed per block in shared memory and added to hot_bins once per block: the
// counts of a window's rows fall into a few dozen bins, and one global atomic per row piles up on those few words.
// take_pair_row adds to the block's bins in between; every thread of the block calls both.
__device__ __forceinline__ void block_bins_begin(uint32_t* s_bins) {
  for (uint32_t b = threadIdx.x; b < 128u; b += blockDim.x) s_bins[b] = 0u;
  __syncthreads();
}
__device__ __forceinline__ void block_bins_end(const uint32_t* s_bins, uint32_t* hot_bins) {
  __syncthreads();
  for (uint32_t b = threadIdx.x; b < 128u; b += blockDim.x) if (s_bins[b]) atomicAdd(&hot_bins[b], s_bins[b]);
}
__device__ __forceinline__ uint64_t take_pair_row(const PairTable& pairs, uint32_t row, bool valid, uint32_t gmask,
                                                  uint32_t* __restrict__ hot_bins, PairSlice& s) {
  const uint32_t lane = threadIdx.x & 31u, sl = lane & 7u;
  uint4* cells = reinterpret_cast<uint4*>(pairs.sect + ((size_t)row * kSectPerRow + sl * 2u) * 4u);
  s.a = make_uint4(0u, 0u, 0u, 0u); s.b = s.a; s.pa = s.a; s.pb = s.a;
  if (valid) { s.a = cells[0]; s.pa = cells[1]; s.b = cells[2]; s.pb = cells[3]; }
  const uint4 a = s.a, b = s.b;
  uint64_t cnt = (uint64_t)a.x + a.y + a.z + a.w + b.x + b.y + b.z + b.w;
  cnt += __shfl_xor_sync(gmask, cnt, 1);
  cnt += __shfl_xor_sync(gmask, cnt, 2);
  cnt += __shfl_xor_sync(gmask, cnt, 4);
  // the 16-bucket window (aligned to 4 buckets) that holds most of the row's events: group sums of 4 cells,
  // two candidates per lane, arg-max over the row's eight lanes
  const uint64_t g0 = (uint64_t)a.x + a.y + a.z + a.w, g1 = (uint64_t)b.x + b.y + b.z + b.w;   // groups 2sl, 2sl+1
  const uint32_t seg = lane & ~7u;
  const uint64_t n0 = __shfl_sync(gmask, g0, seg | ((sl + 1u) & 7u)), n1 = __shfl_sync(gmask, g1, seg | ((sl + 1u) & 7u));
  const uint64_t m0 = __shfl_sync(gmask, g0, seg | ((sl + 2u) & 7u));
  // candidate j covers groups j..j+3 (j <= 12); lanes past the end contribute nothing
  uint64_t c0 = sl <= 6u ? g0 + g1 + n0 + n1 : 0ull;                    // j = 2 sl       (sl = 6 -> j = 12)
  uint64_t c1 = sl <= 5u ? g1 + n0 + n1 + m0 : 0ull;                    // j = 2 sl + 1   (sl = 5 -> j = 11)
  uint64_t best = c0 >= c1 ? (c0 << 4) | (2u * sl) : (c1 << 4) | (2u * sl + 1u);   // counts < 2^37: room for 4 index bits
  for (int o = 1; o < 8; o <<= 1) { const uint64_t x = __shfl_xor_sync(gmask, best, o); best = x > best ? x : best; }
  if (sl == 0 && valid && row < pairs.max_rows) pairs.row_base[row] = (uint8_t)(best & 15u);
  if (!valid || cnt == 0) return cnt;  // unused sentinel row (allocated rows always hold >= 1 event)
  if (sl == 0 && row < pairs.max_rows) {    // feedback for the next ingest
    const uint32_t c32 = cnt > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)cnt;
    pairs.row_cnt[row] = c32;
    if (pairs.row_kind[row] != kPairHost) atomicAdd(&hot_bins[count_bin(c32)], 1u);
  }
  // zero what was not zero: a pair's latencies fall into a few of its 16 sectors, the rest was never written
  const uint4 pa = s.pa, pb = s.pb;
  if (a.x | a.y | a.z | a.w | pa.x | pa.y | pa.z | pa.w) { cells[0] = make_uint4(0u, 0u, 0u, 0u); cells[1] = make_uint4(0u, 0u, 0u, 0u); }
  if (b.x | b.y | b.z | b.w | pb.x | pb.y | pb.z | pb.w) { cells[2] = make_uint4(0u, 0u, 0u, 0u); cells[3] = make_uint4(0u, 0u, 0u, 0u); }
  return cnt;
}
__device__ __forceinline__ uint64_t lat_partial(const PairSlice& s) {
  return (((uint64_t)s.pa.y << 32) | s.pa.x) + (((uint64_t)s.pb.y << 32) | s.pb.x);
}
__device__ __forceinline__ uint64_t err_partial(const PairSlice& s) {
  return (((uint64_t)s.pa.w << 32) | s.pa.z) + (((uint64_t)s.pb.w << 32) | s.pb.z);
}
// events of a pair row that reaches no output row: its source is not a pod (kDropRow), or the edge table was full
__device__ __forceinline__ void count_stray_events(Counters* ctr, uint32_t erow, uint64_t cnt) {
  if (erow == kDropRow) atomicAdd(&ctr->src_unresolved, (unsigned long long)cnt);
  else if (erow >= kLostRow) atomicAdd(&ctr->fold_lost_events, (unsigned long long)cnt);
  // else: the edge row of the free-marker key, which no flush emits
}

// pass 2 of a fold in the middle of a window (a table commit, 2^31 pending events) or before a multi-rank merge,
// eight lanes per pair row (four rows per warp in flight): add the row into its edge row and zero it. Each lane
// owns 8 histogram cells = two 16-byte loads; the one-warp-per-row version was bound by its chain of dependent L2
// round trips.
__global__ void __launch_bounds__(256) fold_pairs_kernel(PairTable pairs, EdgeTable edges, Counters* ctr,
                                                         uint32_t* __restrict__ hot_bins) {
  const uint32_t lane = threadIdx.x & 31u, sl = lane & 7u;
  const uint32_t gmask = 0xFFu << (lane & ~7u);
  const uint32_t groups_per_grid = (gridDim.x * blockDim.x) >> 3;
  const uint32_t n_rows = min(*pairs.n_rows, pairs.max_rows);
  __shared__ uint32_t s_bins[128];
  block_bins_begin(s_bins);
  uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 3;
  // rows [0, n_rows) plus the sentinel rows (index n_rows + kind stands for row max_rows + kind)
  for (; i < n_rows + kPairKinds; i += groups_per_grid) {
    const uint32_t row = i >= n_rows ? pairs.max_rows + (i - n_rows) : i;
    PairSlice s;
    const uint64_t cnt = take_pair_row(pairs, row, true, gmask, s_bins, s);
    if (cnt == 0) continue;
    uint64_t lat = lat_partial(s), e5 = err_partial(s);
    for (int o = 1; o < 8; o <<= 1) {
      lat += __shfl_xor_sync(gmask, lat, o);
      e5 += __shfl_xor_sync(gmask, e5, o);
    }
    const uint32_t erow = pairs.row_aux[row];
    if (erow < kDropRow) {
      const uint4 a = s.a, b = s.b;
      uint32_t* dst = edges.hist + (size_t)erow * ALZ_NB + sl * 8u;
      if (a.x) atomicAdd(dst + 0, a.x);
      if (a.y) atomicAdd(dst + 1, a.y);
      if (a.z) atomicAdd(dst + 2, a.z);
      if (a.w) atomicAdd(dst + 3, a.w);
      if (b.x) atomicAdd(dst + 4, b.x);
      if (b.y) atomicAdd(dst + 5, b.y);
      if (b.z) atomicAdd(dst + 6, b.z);
      if (b.w) atomicAdd(dst + 7, b.w);
      if (sl == 0) {
        atomicAdd((unsigned long long*)&edges.count[erow], (unsigned long long)cnt);
        atomicAdd((unsigned long long*)&edges.lat_sum[erow], (unsigned long long)lat);
        if (e5) atomicAdd((unsigned long long*)&edges.err5xx[erow], (unsigned long long)e5);
      }
    } else if (sl == 0) {
      count_stray_events(ctr, erow, cnt);
    }
  }
  block_bins_end(s_bins, hot_bins);
}

// ---------------------------------------------------------------------------
// flush: rows [0, n) of the edge table are the live edges. iota -> sort by key
// (alz_sort.cu) -> output rows in key order.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) iota_kernel(uint32_t* out, uint32_t n) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = i;
}

// unique of a sorted key array (the merge's canonical keys, the GNN's node set): flag the run heads, exclusive-scan
// the flags, scatter the heads. kEmptyKey is never a head: the merge pads its gathered key lists with it, and no GNN
// node key equals it (node_key, alz_gnn.cu, puts a node type, below 4, in the high word).
__global__ void flag_heads_kernel(const uint64_t* __restrict__ sorted, uint32_t n, uint32_t* __restrict__ flags) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint64_t k = sorted[i];
    flags[i] = (k != kEmptyKey && (i == 0 || sorted[i - 1] != k)) ? 1u : 0u;
  }
}
__global__ void scatter_heads_kernel(const uint64_t* __restrict__ sorted, const uint32_t* __restrict__ flags,
                                     const uint32_t* __restrict__ pos, uint32_t n, uint64_t* __restrict__ out) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    if (flags[i]) out[pos[i]] = sorted[i];
}

// multi-rank flush: the live edge rows, as they are, into the send buffer (the window stays in the table until
// every rank has taken part in the merge, alz_comm.cu)
__global__ void __launch_bounds__(256) gather_edges_kernel(EdgeTable edges, const uint64_t* __restrict__ keys,
                                                           const uint32_t* __restrict__ rows, uint32_t n_live,
                                                           alz_edge_out* __restrict__ out) {
  // eight lanes per edge, four edges per warp in flight; a lane moves 8 histogram cells (2 x 16 bytes)
  const uint32_t sl = threadIdx.x & 7u;
  const uint32_t groups_per_grid = (gridDim.x * blockDim.x) >> 3;
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 3; i < n_live; i += groups_per_grid) {
    uint32_t c[8];
    uint64_t count, lat, e5;
    edge_row_load(edges, rows[i], sl, c, count, lat, e5);
    store_edge_out(&out[i], sl, keys[i], c, count, e5, lat);
  }
}

// ---------------------------------------------------------------------------
// single-rank flush: the pair rows go straight into the output rows. fold_resolve_kernel gave every pair row its
// edge row (row_aux); the rows are bucketed by edge row (count, exclusive scan, fill) and emit_edges_kernel sums
// each bucket in registers into the output row of its edge. Every sum is an integer sum, so the order of the rows
// in a bucket does not change the result.
// ---------------------------------------------------------------------------
// pair rows per edge row into cnt[]; a row that reaches no edge row (unresolved source, full edge table, the
// free-marker edge key) goes to the back of row_list, *n_stray of them
__global__ void __launch_bounds__(256) bucket_count_kernel(PairTable pairs, uint32_t max_edges, uint32_t* __restrict__ cnt,
                                                           uint32_t* __restrict__ row_list, uint32_t list_cap,
                                                           uint32_t* __restrict__ n_stray) {
  const uint32_t n_rows = min(*pairs.n_rows, pairs.max_rows);
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_rows + kPairKinds; i += stride) {
    const uint32_t row = i >= n_rows ? pairs.max_rows + (i - n_rows) : i;
    const uint32_t erow = pairs.row_aux[row];
    if (erow < max_edges) atomicAdd(&cnt[erow], 1u);
    else row_list[list_cap - 1u - atomicAdd(n_stray, 1u)] = row;
  }
}
// each row to its place in its edge's bucket; counts cnt[] back down to zero for the next flush
__global__ void __launch_bounds__(256) bucket_fill_kernel(PairTable pairs, uint32_t max_edges, uint32_t* __restrict__ cnt,
                                                          const uint32_t* __restrict__ off, uint32_t* __restrict__ row_list) {
  const uint32_t n_rows = min(*pairs.n_rows, pairs.max_rows);
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_rows + kPairKinds; i += stride) {
    const uint32_t row = i >= n_rows ? pairs.max_rows + (i - n_rows) : i;
    const uint32_t erow = pairs.row_aux[row];
    if (erow < max_edges) row_list[off[erow] + atomicSub(&cnt[erow], 1u) - 1u] = row;
  }
}

// Output row i (edge row rows[i]) = the sum of the pair rows of its bucket, row_list[off[erow], off[erow + 1]),
// plus, when a fold already ran in this window (with_edges), what the edge accumulators hold, which it zeroes.
// Eight lanes per output row as in fold_pairs_kernel, plain stores only. The n_stray pair rows at the back of
// row_list follow as groups n_live.. : they leave their feedback and their events in the counters. off == nullptr:
// no pair rows to take (nothing was ingested since the last fold, or ALZ_CFG_EAGER_JOIN).
__global__ void __launch_bounds__(256) emit_edges_kernel(PairTable pairs, EdgeTable edges, Counters* ctr,
                                                         uint32_t* __restrict__ hot_bins, const uint64_t* __restrict__ keys,
                                                         const uint32_t* __restrict__ rows,
                                                         const uint32_t* __restrict__ off,
                                                         const uint32_t* __restrict__ row_list, uint32_t list_cap,
                                                         const uint32_t* __restrict__ n_stray, bool with_edges,
                                                         alz_edge_out* __restrict__ out) {
  const uint32_t lane = threadIdx.x & 31u, sl = lane & 7u;
  const uint32_t gmask = 0xFFu << (lane & ~7u);
  const uint32_t groups_per_grid = (gridDim.x * blockDim.x) >> 3;
  const uint32_t n_live = min(*edges.n_rows, edges.max_rows);
  const uint32_t n_groups = n_live + (off != nullptr ? *n_stray : 0u);
  __shared__ uint32_t s_bins[128];
  block_bins_begin(s_bins);
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 3; i < n_groups; i += groups_per_grid) {
    if (i >= n_live) {
      const uint32_t row = row_list[list_cap - 1u - (i - n_live)];
      PairSlice s;
      const uint64_t cnt = take_pair_row(pairs, row, true, gmask, s_bins, s);
      if (sl == 0 && cnt != 0) count_stray_events(ctr, pairs.row_aux[row], cnt);
      continue;
    }
    const uint32_t erow = rows[i];
    uint32_t c[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
    uint64_t count = 0, lat = 0, e5 = 0;   // lane partials of the latency and 5xx sums; count in lane 0
    if (with_edges) {
      edge_row_load(edges, erow, sl, c, count, lat, e5);
      edge_row_zero(edges, erow, sl);
    }
    if (off != nullptr) {
      const uint32_t end = off[erow + 1u];
      for (uint32_t j = off[erow]; j < end; ++j) {
        PairSlice s;
        count += take_pair_row(pairs, row_list[j], true, gmask, s_bins, s);
        c[0] += s.a.x; c[1] += s.a.y; c[2] += s.a.z; c[3] += s.a.w;
        c[4] += s.b.x; c[5] += s.b.y; c[6] += s.b.z; c[7] += s.b.w;
        lat += lat_partial(s);
        e5 += err_partial(s);
      }
    }
    for (int o = 1; o < 8; o <<= 1) {
      lat += __shfl_xor_sync(gmask, lat, o);
      e5 += __shfl_xor_sync(gmask, e5, o);
    }
    store_edge_out(&out[i], sl, keys[i], c, count, e5, lat);
  }
  block_bins_end(s_bins, hot_bins);
}

// ---------------------------------------------------------------------------
// raw perf samples (1096-B struct l7_event, ebpf/l7_req/l7.go:345-369) -> 32-B
// records. One thread per sample; the 72 useful bytes sit in the first 36 and
// the last 36 bytes of each sample.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) compact_raw_kernel(const uint8_t* __restrict__ raw, uint64_t n,
                                                          alz_l7_rec* __restrict__ out) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint8_t* p = raw + i * ALZ_BPF_L7_EVENT_SIZE;  // 1096 = 8 * 137: 8-byte aligned
    const uint64_t write_time = *reinterpret_cast<const uint64_t*>(p + 8);
    const uint32_t status = *reinterpret_cast<const uint32_t*>(p + 20);
    const uint64_t duration = *reinterpret_cast<const uint64_t*>(p + 24);
    const uint32_t pm = *reinterpret_cast<const uint32_t*>(p + 32);      // protocol, method, pad
    const uint32_t fl = *reinterpret_cast<const uint32_t*>(p + 1064);    // read_complete, failed, is_tls
    const uint32_t saddr = *reinterpret_cast<const uint32_t*>(p + 1076);
    const uint32_t sport = *reinterpret_cast<const uint16_t*>(p + 1080);
    const uint32_t daddr = *reinterpret_cast<const uint32_t*>(p + 1084);
    const uint32_t dport = *reinterpret_cast<const uint16_t*>(p + 1088);
    uint32_t protocol = pm & 0xFFu;
    const uint32_t method = (pm >> 8) & 0xFFu;
    const uint32_t is_tls = (fl >> 16) & 0xFFu;
    // the eBPF byte has no flag bits: one that would read as ALZ_PROTO_F_HOSTKEY (or anything else >= 0x40) is an
    // undefined protocol and must stay one (alz_pack_l7 does the same)
    if (protocol >= 0x40u) protocol = 0x3Fu;
    uint4 lo, hi;
    lo.x = saddr; lo.y = daddr; lo.z = sport | (dport << 16);
    lo.w = (status > 65535u ? 65535u : status) | (protocol << 16) |
           (((method & ALZ_MF_METHOD_MASK) | (is_tls ? ALZ_MF_TLS : 0u)) << 24);
    hi.x = (uint32_t)duration; hi.y = (uint32_t)(duration >> 32);
    hi.z = (uint32_t)write_time; hi.w = (uint32_t)(write_time >> 32);
    uint4* o = reinterpret_cast<uint4*>(out + i);
    o[0] = lo; o[1] = hi;
  }
}

// synthetic stream on the device (bench/test support; alaz_b200/synth/alz_synth.h)
__global__ void __launch_bounds__(256) synth_kernel(alz_synth_view v, uint64_t first, uint64_t n,
                                                    alz_l7_rec* __restrict__ out) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    alz_l7_rec r;
    alz_synth_event(&v, first + i, &r);
    out[i] = r;
  }
}

// events first..first+n of the global stream, keeping only those owned by `rank`
// (alz_owner_rank: hash of saddr). Appends in arbitrary order; stops writing at cap.
__global__ void __launch_bounds__(256) synth_owned_kernel(alz_synth_view v, uint64_t first, uint64_t n, uint32_t nranks,
                                                          uint32_t rank, alz_l7_rec* __restrict__ out, uint64_t cap,
                                                          unsigned long long* n_written) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < n; base += stride) {
    const uint64_t i = base + lane;
    alz_l7_rec r;
    bool mine = false;
    if (i < n) {
      alz_synth_event(&v, first + i, &r);
      mine = owner_rank(r.saddr, nranks) == rank;
    }
    const uint32_t m = __ballot_sync(0xFFFFFFFFu, mine);
    if (m == 0u) continue;
    unsigned long long pos = 0;
    if (lane == 0) pos = atomicAdd(n_written, (unsigned long long)__popc(m));
    pos = __shfl_sync(0xFFFFFFFFu, pos, 0) + __popc(m & ((1u << lane) - 1u));
    if (mine && pos < cap) out[pos] = r;
  }
}

// Empties a table's dictionaries (a, then b; b_mask + 1 slots of b, or none) from its claimed-slot log: the logged
// slots go back to kEmptyKey, or every slot of both when the log overflowed. The last block to finish resets the log
// and, when n_rows is given, the row allocator; every block has read the log count before any block finishes.
__global__ void __launch_bounds__(256) dict_clear_kernel(DictEnt* __restrict__ a, uint32_t a_mask, DictEnt* __restrict__ b,
                                                         uint32_t b_slots, SlotLog log, uint32_t* __restrict__ n_rows) {
  const uint32_t n = *reinterpret_cast<volatile uint32_t*>(log.n);
  const uint4 empty = make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu);
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t first = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n <= log.cap) {
    for (size_t i = first; i < n; i += stride) {
      const uint32_t v = log.slot[i];
      DictEnt* e = v <= a_mask ? &a[v] : &b[v - a_mask - 1u];
      *reinterpret_cast<uint4*>(e) = empty;
    }
  } else {
    const size_t total = (size_t)a_mask + 1u + b_slots;
    for (size_t i = first; i < total; i += stride)
      *reinterpret_cast<uint4*>(i <= a_mask ? &a[i] : &b[i - a_mask - 1u]) = empty;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(&log.n[1], 1u) == gridDim.x - 1u) {
      log.n[0] = 0u;
      log.n[1] = 0u;
      if (n_rows) *n_rows = 0u;
    }
  }
}

// ---------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------
static inline unsigned grid_for(int sms, int per_sm) { return (unsigned)(sms * per_sm); }

void launch_ingest_pairs_v1(const alz_l7_rec* recs, uint64_t n, const PairTable& pairs, Counters* ctr,
                            const EpEntry* ep, uint32_t ep_mask, int sms, cudaStream_t s) {
  if (n == 0) return;   // global reductions only (ALZ_CFG_NO_SMEM_CACHE; kept for the ncu comparison)
  ingest_pairs_kernel<4><<<grid_for(sms, 8), 256, 0, s>>>(recs, n, pairs, ctr, ep, ep_mask);
}
void launch_ingest_eager(const alz_l7_rec* recs, uint64_t n, const EpEntry* ep, uint32_t ep_mask,
                         const EdgeTable& edges, Counters* ctr, int sms, cudaStream_t s) {
  if (n == 0) return;
  ingest_eager_kernel<<<grid_for(sms, 8), 256, 0, s>>>(recs, n, ep, ep_mask, edges, ctr);
}
void launch_fold_resolve(const PairTable& pairs, const EpEntry* ep, uint32_t ep_mask, const EdgeTable& edges,
                         HotState* hot, int sms, cudaStream_t s) {
  fold_resolve_kernel<<<grid_for(sms, 4), 256, 0, s>>>(pairs, ep, ep_mask, edges, hot);
}
void launch_fold_add(const PairTable& pairs, const EdgeTable& edges, Counters* ctr, HotState* hot, int sms,
                     cudaStream_t s) {
  fold_pairs_kernel<<<grid_for(sms, 8), 256, 0, s>>>(pairs, edges, ctr, hot->bins);
}
// changed slots of the endpoint table (alz_table_commit): patch[i] = {slot, pad x3, entry}
__global__ void __launch_bounds__(256) ep_patch_kernel(EpEntry* __restrict__ tab, const uint4* __restrict__ patch, uint32_t n) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint4 hd = patch[2 * i], e = patch[2 * i + 1];
    *reinterpret_cast<uint4*>(&tab[hd.x]) = e;
  }
}
void launch_ep_patch(EpEntry* tab, const void* patch, uint32_t n, int sms, cudaStream_t s) {
  if (n == 0) return;
  const unsigned grid = (unsigned)std::min<uint32_t>((n + 255u) / 256u, (uint32_t)sms * 4u);
  ep_patch_kernel<<<grid, 256, 0, s>>>(tab, (const uint4*)patch, n);
}
void launch_iota(uint32_t* out, uint32_t n, int sms, cudaStream_t s) {
  if (n == 0) return;
  iota_kernel<<<grid_for(sms, 4), 256, 0, s>>>(out, n);
}
cudaError_t launch_unique_sorted(const uint64_t* sorted, uint32_t n, uint32_t* flags, uint32_t* pos, uint64_t* out,
                                 void* temp, size_t temp_bytes, int sms, cudaStream_t s) {
  flag_heads_kernel<<<grid_for(sms, 4), 256, 0, s>>>(sorted, n, flags);
  const cudaError_t e = exclusive_scan_u32(temp, temp_bytes, flags, pos, n, s);
  if (e != cudaSuccess) return e;
  scatter_heads_kernel<<<grid_for(sms, 4), 256, 0, s>>>(sorted, flags, pos, n, out);
  return cudaSuccess;
}
void launch_gather_edges(const EdgeTable& edges, const uint64_t* keys, const uint32_t* rows, uint32_t n_live,
                         alz_edge_out* out, int sms, cudaStream_t s) {
  if (n_live == 0) return;
  gather_edges_kernel<<<grid_for(sms, 8), 256, 0, s>>>(edges, keys, rows, n_live, out);
}
void launch_bucket_count(const PairTable& pairs, uint32_t max_edges, const FlushBuckets& b, int sms, cudaStream_t s) {
  bucket_count_kernel<<<grid_for(sms, 4), 256, 0, s>>>(pairs, max_edges, b.cnt, b.rows, b.cap, b.n_stray);
}
void launch_bucket_fill(const PairTable& pairs, uint32_t max_edges, const FlushBuckets& b, int sms, cudaStream_t s) {
  bucket_fill_kernel<<<grid_for(sms, 4), 256, 0, s>>>(pairs, max_edges, b.cnt, b.off, b.rows);
}
void launch_emit_edges(const PairTable& pairs, const EdgeTable& edges, Counters* ctr, HotState* hot, const uint64_t* keys,
                       const uint32_t* rows, const FlushBuckets* b, bool with_edges, alz_edge_out* out, int sms,
                       cudaStream_t s) {
  emit_edges_kernel<<<grid_for(sms, 8), 256, 0, s>>>(pairs, edges, ctr, hot->bins, keys, rows,
                                                     b ? b->off : nullptr, b ? b->rows : nullptr, b ? b->cap : 0u,
                                                     b ? b->n_stray : nullptr, with_edges, out);
}
void launch_pair_dict_clear(const PairTable& pairs, bool reset_rows, int sms, cudaStream_t s) {
  dict_clear_kernel<<<grid_for(sms, 4), 256, 0, s>>>(pairs.dict, pairs.dict_mask, pairs.dict_host, pairs.dict_host_mask + 1u,
                                                     pairs.log, reset_rows ? pairs.n_rows : nullptr);
}
cudaError_t edge_table_clear(const EdgeTable& t, int sms, cudaStream_t s) {
  dict_clear_kernel<<<grid_for(sms, 4), 256, 0, s>>>(t.dict, t.dict_mask, nullptr, 0u, t.log, t.n_rows);
  return cudaGetLastError();
}
void launch_compact_raw(const uint8_t* raw, uint64_t n, alz_l7_rec* out, int sms, cudaStream_t s) {
  if (n == 0) return;
  compact_raw_kernel<<<grid_for(sms, 8), 256, 0, s>>>(raw, n, out);
}
void launch_synth(const alz_synth_view& v, uint64_t first, uint64_t n, alz_l7_rec* out, int sms, cudaStream_t s) {
  if (n == 0) return;
  synth_kernel<<<grid_for(sms, 8), 256, 0, s>>>(v, first, n, out);
}
void launch_synth_owned(const alz_synth_view& v, uint64_t first, uint64_t n, uint32_t nranks, uint32_t rank,
                        alz_l7_rec* out, uint64_t cap, unsigned long long* n_written, int sms, cudaStream_t s) {
  if (n == 0) return;
  synth_owned_kernel<<<grid_for(sms, 8), 256, 0, s>>>(v, first, n, nranks, rank, out, cap, n_written);
}

}  // namespace alz
