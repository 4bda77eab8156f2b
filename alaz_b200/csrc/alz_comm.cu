// alz_comm.cu — multi-GPU window merge (SURVEY.md §8e): one rank per GPU, events
// pre-partitioned by alz_owner_rank(saddr), tables replicated. Every event of an edge
// reaches one rank, so the ranks' edge sets are disjoint and a rank's accumulators are
// already final: what the flush has to do is hand every rank every other rank's rows.
//
// Default path — ONE collective, no host round trip before it:
//   1. each rank writes its sorted live rows behind a one-row header {count, status} in a
//      send buffer; the per-rank block size of the collective comes from the previous
//      window's counts (+25 %), so no count exchange is needed
//   2. ncclAllGather of the blocks                      <- the single exchange step
//   3. every rank merges the R sorted, disjoint lists: a row's place in the canonical
//      (ascending packed key) order is its index in its own list plus its lower bounds
//      in the other lists. The same kernel notices a key present on two ranks, a rank
//      whose rows did not fit its block, a rank that reported a local error, or a rank
//      that lost events in its own tables — all ranks see the same headers, so all ranks
//      take the same decision and return the same status.
//   4. one device->host read of {total, flags}: the only synchronisation, and the one the
//      API needs anyway to return the edge count.
// A block that was too small (traffic grew by more than 25 % in one window) is sent
// again, larger; the local rows are only reset after a successful merge.
// A merged graph larger than max_edges is cut in canonical order: every rank keeps the
// first max_edges rows, consumes its window and counts the events of its own rows past
// the cut as lost, so the ranks' rows_emitted still add up to the rows returned.
//
// General path (a key present on several ranks: the caller did not partition by
// alz_owner_rank): canonical dictionary by all-gather + sort + unique, local rows
// scattered into a zeroed canonical array, ONE ncclAllReduce(sum) on the accumulators.
// Integer sums either way, so bit-exact for any rank count. When the gathered keys or
// their union do not fit max_edges, every rank drops its window and counts its events lost.
//
// NCCL is loaded lazily with dlopen so that single-GPU users (and the Go agent
// on a box without NCCL) never need libnccl.so.2.
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <cstddef>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>

#include "alz_handle.h"

using namespace alz;

namespace {

struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
NcclApi g_nccl;

bool load_nccl_once() {
  void* lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!lib) return false;
#define SYM(field, name)                                             \
  g_nccl.field = reinterpret_cast<decltype(g_nccl.field)>(dlsym(lib, name)); \
  if (!g_nccl.field) return false;
  SYM(GetUniqueId, "ncclGetUniqueId");
  SYM(CommInitRank, "ncclCommInitRank");
  SYM(CommDestroy, "ncclCommDestroy");
  SYM(AllGather, "ncclAllGather");
  SYM(AllReduce, "ncclAllReduce");
  SYM(GetErrorString, "ncclGetErrorString");
#undef SYM
  g_nccl.lib = lib;
  return true;
}
// several rank threads of one process may get here together (tests/test_gpu_multi.py)
bool load_nccl() {
  static std::once_flag once;
  static bool ok = false;
  std::call_once(once, [] { ok = load_nccl_once(); });
  return ok;
}

constexpr int kCanWords = 3 + ALZ_NB;      // u64 words per canonical edge row of the general path: count, err5xx,
                                           // lat_sum and one word per histogram cell (a cell is u32 modulo 2^32: the
                                           // low halves of the sums are taken, nothing can carry between cells)
constexpr uint32_t kRowBytes = sizeof(alz_edge_out);   // 296 = 37 x 8
constexpr uint32_t kRowWords64 = kRowBytes / 8;
constexpr uint32_t kHdrMagic = 0xA1A2C0DEu;
struct BlockHeader {      // first row of a rank's block
  uint32_t magic, count;
  int32_t status;
  uint32_t lost;          // 1: this rank's pair or edge table lost events in this window
  uint32_t clk_on, pad;   // 1: the rank has a window clock, copied into clk on the device; 0: clk is all zero
  WinClock clk;
};
// What a merge does to this rank's window (docs/SPEC.md §8 "Several ranks"): E is the smallest open epoch of the
// ranks, the past state after every epoch. Clockless ranks are always at E.
enum : uint32_t {
  kAtE = 0,        // the rank's rows are E's: merged, consumed, and the clock advances
  kKeep = 1,       // the rank is ahead of E, or no rank has an epoch: nothing sent, nothing changes
  kOpenNext = 2,   // the rank has no epoch: it opens E + 1 (info->clk is E's clock, advanced by the roll)
};
struct MergeInfo {        // written by the merge kernel, read by the host
  uint32_t total, dup, overflow, max_count;
  int32_t peer_status;
  uint32_t lost;          // some rank at E has lost = 1
  uint32_t roll;          // kAtE, kKeep or kOpenNext for this rank
  uint32_t pad;
  unsigned long long lost_events;   // counts of this rank's rows that fell at or past max_edges in the merged order
  WinClock clk;           // the clock of the first rank at E
};

// the order of open epochs across ranks: the past state (ready 2) after every epoch, and all past states equal
__device__ __forceinline__ bool clk_before(const WinClock& a, const WinClock& b) {
  const bool pa = a.ready > 1ull, pb = b.ready > 1ull;
  return pa != pb ? pb : (!pa && a.epoch < b.epoch);
}
__device__ __forceinline__ bool clk_same(const WinClock& a, const WinClock& b) {
  return !clk_before(a, b) && !clk_before(b, a);
}

// out[i] = keys[i] for i < n, kEmptyKey padding up to n_pad
__global__ void pad_keys_kernel(const uint64_t* __restrict__ keys, uint32_t n, uint64_t* __restrict__ out,
                                uint32_t n_pad) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_pad; i += stride)
    out[i] = i < n ? keys[i] : kEmptyKey;
}

// union of R sorted, pairwise disjoint key lists (segment r = gathered[r * pad .. + counts[r])):
// out[sum of lower bounds] = key. *dup is set if a key occurs in two lists.
__global__ void __launch_bounds__(256) merge_disjoint_kernel(const uint64_t* __restrict__ gathered, uint32_t pad,
                                                             uint32_t R, const uint32_t* __restrict__ counts,
                                                             uint64_t* __restrict__ out, uint32_t* __restrict__ dup) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < pad * R; t += stride) {
    const uint32_t r = t / pad, i = t - r * pad;
    if (i >= counts[r]) continue;
    const uint64_t k = gathered[t];
    uint32_t pos = i;
    for (uint32_t q = 0; q < R; ++q) {
      if (q == r) continue;
      const uint64_t* seg = gathered + (size_t)q * pad;
      const uint32_t lb = lower_bound_u64(seg, counts[q], k);
      if (lb < counts[q] && seg[lb] == k) *dup = 1u;
      pos += lb;
    }
    out[pos] = k;
  }
}

// local live rows -> canonical array (zeroed beforehand); eight lanes per local edge; rows are zeroed
__global__ void __launch_bounds__(256) scatter_canonical_kernel(EdgeTable edges, const uint64_t* __restrict__ keys,
                                                                const uint32_t* __restrict__ rows, uint32_t n_local,
                                                                const uint64_t* __restrict__ can_keys, uint32_t n_can,
                                                                uint64_t* __restrict__ can) {
  const uint32_t sl = threadIdx.x & 7u;
  const uint32_t groups = (gridDim.x * blockDim.x) >> 3;
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 3; i < n_local; i += groups) {
    const uint32_t row = rows[i];
    uint32_t c[8];
    uint64_t count, lat, e5;
    edge_row_load(edges, row, sl, c, count, lat, e5);
    edge_row_zero(edges, row, sl);
    uint64_t* dst = can + (size_t)lower_bound_u64(can_keys, n_can, keys[i]) * kCanWords;   // always present
    for (int k = 0; k < 8; ++k) dst[3 + sl * 8u + k] = c[k];
    if (sl == 0) { dst[0] = count; dst[1] = e5; dst[2] = lat; }
  }
}

__global__ void __launch_bounds__(256) unpack_canonical_kernel(const uint64_t* __restrict__ can_keys,
                                                               const uint64_t* __restrict__ can, uint32_t n_can,
                                                               alz_edge_out* __restrict__ out) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t warps_per_grid = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n_can; i += warps_per_grid) {
    const uint64_t* src = can + (size_t)i * kCanWords;
    alz_edge_out* o = &out[i];
    o->hist[lane] = (uint32_t)src[3 + lane];
    o->hist[32 + lane] = (uint32_t)src[3 + 32 + lane];
    if (lane == 0) {
      uint8_t ft, tt; uint32_t f, t;
      unpack_edge_key(can_keys[i], &ft, &f, &tt, &t);
      o->from_type = ft; o->to_type = tt;
      for (int k = 0; k < 6; ++k) o->_pad[k] = 0;
      o->from = f; o->to = t;
      o->count = src[0]; o->err5xx = src[1]; o->lat_sum_ns = src[2];
    }
  }
}

__device__ __forceinline__ uint32_t lower_bound_rows(const alz_edge_out* rows, uint32_t n, uint64_t k, bool* equal) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (row_key_of(rows + mid) < k) lo = mid + 1; else hi = mid; }
  *equal = lo < n && row_key_of(rows + lo) == k;
  return lo;
}

// Merge of the gathered blocks: block q = header row + cap rows, of which header.count are live and sorted.
// Eight lanes per row: the lanes split the other ranks' binary searches among them, then copy the row. Rows whose
// place is at or past out_cap are not written; those of rank `me` add their counts to info->lost_events.
// Under a window clock only the ranks at the merged epoch E take part: another rank counts as 0 rows.
__global__ void __launch_bounds__(256) merge_blocks_kernel(const alz_edge_out* __restrict__ recv, uint32_t cap, uint32_t R,
                                                           uint32_t me, alz_edge_out* __restrict__ out,
                                                           uint32_t out_cap, MergeInfo* __restrict__ info) {
  __shared__ uint32_t s_cnt[64];
  __shared__ uint32_t s_bad;
  __shared__ uint32_t s_clk, s_open;
  __shared__ WinClock s_e;
  const size_t stride_rows = (size_t)cap + 1;
  auto header = [&](uint32_t q) { return reinterpret_cast<const BlockHeader*>(recv + q * stride_rows); };
  if (threadIdx.x == 0) {
    s_bad = 0u;
    // the clock must be the same on every rank (length and offset); E = the smallest open epoch
    const BlockHeader* h0 = header(0);
    uint32_t open = 0u, mismatch = 0u;
    WinClock e{};
    for (uint32_t q = 0; q < R; ++q) {
      const BlockHeader* hq = header(q);
      mismatch |= (hq->clk_on != h0->clk_on || hq->clk.len != h0->clk.len || hq->clk.off != h0->clk.off) ? 1u : 0u;
      if (hq->clk.ready != 0ull && (!open || clk_before(hq->clk, e))) { e = hq->clk; open = 1u; }
    }
    s_clk = h0->clk_on;
    s_open = open;
    s_e = e;
    if (mismatch) {
      s_bad = 1u;
      if (blockIdx.x == 0) info->peer_status = (int32_t)ALZ_E_STATE;
    }
    if (blockIdx.x == 0) {
      const WinClock& mine = header(me)->clk;
      info->roll = !s_clk ? kAtE : !open ? kKeep : mine.ready == 0ull ? kOpenNext : clk_same(mine, e) ? kAtE : kKeep;
      info->clk = e;
    }
  }
  __syncthreads();
  if (threadIdx.x < R) {
    const BlockHeader* hd = header(threadIdx.x);
    uint32_t cnt = hd->count;
    if (hd->magic != kHdrMagic || hd->status != ALZ_OK) {
      atomicOr(&s_bad, 1u);
      if (blockIdx.x == 0) info->peer_status = hd->magic != kHdrMagic ? (int32_t)ALZ_E_STATE : hd->status;
      cnt = 0;
    }
    if (blockIdx.x == 0) atomicMax(&info->max_count, cnt);   // block sizing: every rank's rows, at E or not
    const bool at_e = !s_clk || (s_open && hd->clk.ready != 0ull && clk_same(hd->clk, s_e));
    if (!at_e) cnt = 0;
    if (cnt > cap) { atomicOr(&s_bad, 2u); if (blockIdx.x == 0) info->overflow = 1u; }
    if (blockIdx.x == 0 && hd->lost != 0u && at_e) info->lost = 1u;   // an ahead rank's loss waits for its window
    s_cnt[threadIdx.x] = cnt;
  }
  __syncthreads();
  uint32_t total = 0;
  for (uint32_t q = 0; q < R; ++q) total += s_cnt[q];
  if (blockIdx.x == 0 && threadIdx.x == 0) info->total = total;
  if (s_bad != 0u) return;
  const uint32_t sl = threadIdx.x & 7u;
  const uint32_t groups = (gridDim.x * blockDim.x) >> 3;
  const uint32_t n_iter = (total + groups - 1) / groups;
  uint32_t g = (blockIdx.x * blockDim.x + threadIdx.x) >> 3;
  for (uint32_t it = 0; it < n_iter; ++it, g += groups) {
    const bool valid = g < total;
    // (q, i) of flat index g
    uint32_t q = 0, i = valid ? g : 0u;
    while (valid && i >= s_cnt[q]) { i -= s_cnt[q]; ++q; }
    const alz_edge_out* src = recv + q * stride_rows + 1 + i;
    const uint64_t key = valid ? row_key_of(src) : 0ull;
    uint32_t part = 0;
    bool dup = false;
    for (uint32_t p = sl; p < R; p += 8u) {
      if (!valid || p == q) continue;
      bool eq;
      part += lower_bound_rows(recv + p * stride_rows + 1, s_cnt[p], key, &eq);
      dup |= eq;
    }
    part += __shfl_xor_sync(0xFFFFFFFFu, part, 1);
    part += __shfl_xor_sync(0xFFFFFFFFu, part, 2);
    part += __shfl_xor_sync(0xFFFFFFFFu, part, 4);
    if (dup) info->dup = 1u;
    if (!valid) continue;
    if (i + part >= out_cap) {   // past the cut: the owner counts the row's events as lost
      if (q == me && sl == 0u) atomicAdd(&info->lost_events, (unsigned long long)src->count);
      continue;
    }
    const uint64_t* s64 = reinterpret_cast<const uint64_t*>(src);
    uint64_t* d64 = reinterpret_cast<uint64_t*>(out + (i + part));
    for (uint32_t w = sl; w < kRowWords64; w += 8u) d64[w] = s64[w];
  }
}

// a successful merge consumes the window: zero the local edge rows that were sent, empty the edge dictionary, reset
// the row allocator. Decided on the device from the merge kernel's verdict, so the host reads that verdict once, at
// the end, instead of synchronising in the middle of the flush to decide whether to launch this.
__global__ void __launch_bounds__(256) consume_window_kernel(const MergeInfo* __restrict__ info, EdgeTable edges,
                                                             const uint32_t* __restrict__ rows, uint32_t n) {
  if (info->peer_status != ALZ_OK || info->overflow != 0u || info->dup != 0u || info->roll != kAtE) return;
  const uint32_t sl = threadIdx.x & 7u;
  const uint32_t groups = (gridDim.x * blockDim.x) >> 3;
  const size_t dict_words = ((size_t)edges.dict_mask + 1u) * (sizeof(DictEnt) / 16u);
  uint4* dict = reinterpret_cast<uint4*>(edges.dict);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < dict_words; i += (size_t)gridDim.x * blockDim.x)
    dict[i] = make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu);
  if (blockIdx.x == 0 && threadIdx.x == 0) { *edges.n_rows = 0u; edges.log.n[0] = 0u; }
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 3; i < n; i += groups) edge_row_zero(edges, rows[i], sl);
}

// info->lost_events += the counts of n rows (the general path's dropped window)
__global__ void __launch_bounds__(256) sum_counts_kernel(const alz_edge_out* __restrict__ rows, uint32_t n,
                                                         MergeInfo* __restrict__ info) {
  unsigned long long s = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) s += rows[i].count;
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, o);
  if ((threadIdx.x & 31u) == 0u && s) atomicAdd(&info->lost_events, s);
}

}  // namespace

struct alz_comm_state {
  ncclComm_t comm = nullptr;
  uint32_t* d_counts = nullptr;   // [nranks]
  uint32_t* h_counts = nullptr;   // pinned
  uint64_t* d_gather = nullptr;   // [nranks * pad] gathered keys, then sorted copy behind it
  uint64_t* d_sorted = nullptr;
  uint32_t* d_flags = nullptr;
  uint32_t* d_pos = nullptr;
  uint64_t* d_can_keys = nullptr; // [max_edges]
  uint64_t* d_can = nullptr;      // [max_edges * kCanWords]
  uint32_t* d_iota = nullptr;
  uint32_t* d_vals = nullptr;
  void* d_tmp = nullptr;
  size_t tmp_bytes = 0;
  size_t gather_cap = 0;          // keys
  // default path
  alz_edge_out* d_send = nullptr; // [1 + block_rows_for(max_edges)]: header row + local sorted rows (+ head room)
  alz_edge_out* d_recv = nullptr; // [R * (1 + cap_r)]
  size_t recv_rows = 0;           // allocated rows of d_recv
  uint32_t cap_r = 0;             // rows per rank block of the next collective (0 = not known yet)
  BlockHeader* h_hdr = nullptr;   // pinned
  MergeInfo* d_info = nullptr;
  MergeInfo* h_info = nullptr;    // pinned
};

#define NK(expr)                                                                       \
  do {                                                                                 \
    ncclResult_t _r = (expr);                                                          \
    if (_r != ncclSuccess) {                                                           \
      h->last_err = std::string(#expr) + ": " + g_nccl.GetErrorString(_r);             \
      return ALZ_E_NCCL;                                                               \
    }                                                                                  \
  } while (0)

extern "C" int alz_comm_unique_id(void* out_id) {
  if (!out_id) return ALZ_E_INVAL;
  if (!load_nccl()) return ALZ_E_NCCL;
  static_assert(sizeof(ncclUniqueId) <= ALZ_COMM_ID_BYTES, "ncclUniqueId larger than ALZ_COMM_ID_BYTES");
  ncclUniqueId id;
  if (g_nccl.GetUniqueId(&id) != ncclSuccess) return ALZ_E_NCCL;
  memset(out_id, 0, ALZ_COMM_ID_BYTES);
  memcpy(out_id, &id, sizeof(id));
  return ALZ_OK;
}

static uint32_t block_rows_for(uint64_t max_count) {   // +25 % head room, in steps of 1024 rows
  const uint64_t want = max_count + max_count / 4 + 1024;
  return (uint32_t)((want + 1023) / 1024 * 1024);
}

extern "C" int alz_comm_init(alz_handle* h, int nranks, int rank, const void* id_bytes) {
  if (!h || !id_bytes || nranks < 1 || rank < 0 || rank >= nranks) return ALZ_E_INVAL;
  if (nranks > 64) return ALZ_E_UNSUPPORTED;   // the merge kernel keeps one block count per rank in 64 shared words
  std::lock_guard<std::mutex> g(h->mu);
  if (h->comm) return ALZ_E_STATE;
  if (!load_nccl()) { h->last_err = "dlopen(libnccl.so.2) failed"; return ALZ_E_NCCL; }
  CK(cudaSetDevice(h->device));
  alz_comm_state* c = new alz_comm_state();
  ncclUniqueId id;
  memcpy(&id, id_bytes, sizeof(id));
  ncclResult_t r = g_nccl.CommInitRank(&c->comm, nranks, id, rank);
  if (r != ncclSuccess) { h->last_err = g_nccl.GetErrorString(r); delete c; return ALZ_E_NCCL; }
  h->comm = c;
  h->comm_nranks = nranks;
  h->comm_rank = rank;
  const size_t me = h->cfg.max_edges;
  c->gather_cap = me;  // every rank holds the merged graph, so max_edges bounds the gathered keys too
  CK(cudaMalloc(&c->d_counts, sizeof(uint32_t) * nranks));
  CK(cudaMallocHost(&c->h_counts, sizeof(uint32_t) * nranks));
  CK(cudaMalloc(&c->d_gather, me * 8 * 2));
  c->d_sorted = c->d_gather + me;
  CK(cudaMalloc(&c->d_flags, me * 4));
  CK(cudaMalloc(&c->d_pos, me * 4));
  CK(cudaMalloc(&c->d_can_keys, me * 8));
  CK(cudaMalloc(&c->d_can, me * kCanWords * 8));
  CK(cudaMalloc(&c->d_iota, me * 4));
  CK(cudaMalloc(&c->d_vals, me * 4));
  c->tmp_bytes = std::max(sort_pairs_temp_bytes((uint32_t)me), scan_temp_bytes((uint32_t)me));
  CK(cudaMalloc(&c->d_tmp, c->tmp_bytes));
  // a block is sized from the largest rank's count plus head room: up to block_rows_for(max_edges) rows are SENT
  // from here even when this rank has fewer (max_edges must be the same on every rank)
  const size_t send_rows = (size_t)block_rows_for(me) + 1;
  CK(cudaMalloc(&c->d_send, send_rows * sizeof(alz_edge_out)));
  CK(cudaMemset(c->d_send, 0, send_rows * sizeof(alz_edge_out)));
  CK(cudaMallocHost(&c->h_hdr, sizeof(alz_edge_out)));
  CK(cudaMalloc(&c->d_info, sizeof(MergeInfo)));
  CK(cudaMallocHost(&c->h_info, sizeof(MergeInfo)));
  return ALZ_OK;
}

void alz_internal_free_comm(alz_handle* h) {
  alz_comm_state* c = h->comm;
  if (!c) return;
  if (c->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(c->comm);
  cudaFree(c->d_counts); if (c->h_counts) cudaFreeHost(c->h_counts);
  cudaFree(c->d_gather); cudaFree(c->d_flags); cudaFree(c->d_pos); cudaFree(c->d_can_keys);
  cudaFree(c->d_can); cudaFree(c->d_iota); cudaFree(c->d_vals); cudaFree(c->d_tmp);
  cudaFree(c->d_send); cudaFree(c->d_recv); cudaFree(c->d_info);
  if (c->h_hdr) cudaFreeHost(c->h_hdr);
  if (c->h_info) cudaFreeHost(c->h_info);
  delete c;
  h->comm = nullptr;
}

// The general path's keys do not fit max_edges: this rank's window is consumed without a merge, its events are
// counted lost and the flush returns no rows. Every rank decides this from the same gathered counts or keys.
// The local rows are in d_send (gathered before the block exchange). A rank that is not at the merged epoch
// (at_e false) keeps its window.
static int drop_window(alz_handle* h, bool* lost, bool at_e) {
  alz_comm_state* c = h->comm;
  cudaStream_t s = h->stream;
  const unsigned grid = (unsigned)h->sms * 4;
  CK(cudaMemsetAsync(c->d_info, 0, offsetof(MergeInfo, clk), s));   // E's clock stays (alz_internal_merged_clock)
  if (at_e && h->n_live) {
    sum_counts_kernel<<<grid, 256, 0, s>>>(c->d_send + 1, h->n_live, c->d_info);
    consume_window_kernel<<<grid, 256, 0, s>>>(c->d_info, h->edges, h->d_rows[1], h->n_live);
    h->launches += 2;
  } else if (at_e) {
    CK(edge_table_clear(h->edges, h->sms, s));
    h->launches += 1;
  }
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(c->h_info, c->d_info, sizeof(MergeInfo), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  h->merge_lost_events += c->h_info->lost_events;
  *lost = true;
  h->last_n_edges = 0;
  h->windows++;
  return ALZ_OK;
}

// General path: keys may live on several ranks. Local live edges are sorted in d_keys[1] / d_rows[1]. A rank that
// is not at the merged epoch (at_e false) contributes no rows and keeps its window.
static int merge_allreduce(alz_handle* h, bool* lost, bool at_e) {
  alz_comm_state* c = h->comm;
  const int R = h->comm_nranks;
  cudaStream_t s = h->stream;
  const unsigned grid = (unsigned)h->sms * 4;
  const uint32_t n_local = at_e ? h->n_live : 0u;

  // 1. counts
  CK(cudaMemcpyAsync(c->d_counts + h->comm_rank, &n_local, 4, cudaMemcpyHostToDevice, s));
  NK(g_nccl.AllGather(c->d_counts + h->comm_rank, c->d_counts, 1, ncclUint32, c->comm, s));
  CK(cudaMemcpyAsync(c->h_counts, c->d_counts, 4 * R, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  uint32_t pad = 0;
  uint64_t total = 0;
  for (int r = 0; r < R; ++r) { pad = std::max(pad, c->h_counts[r]); total += c->h_counts[r]; }
  if (total == 0) {
    h->last_n_edges = 0;
    h->windows++;
    if (at_e) { CK(edge_table_clear(h->edges, h->sms, s)); h->launches += 1; }
    return ALZ_OK;
  }
  if ((uint64_t)pad * R > c->gather_cap) return drop_window(h, lost, at_e);
  const uint32_t n_g = pad * (uint32_t)R;

  // 2. keys: pad, all-gather, merge. Each rank's list is sorted and, when the caller partitioned by
  //    alz_owner_rank, the lists are disjoint: a key's place in the union is then the sum of its lower
  //    bounds in the R lists - no sort. A key found on two ranks (caller routed one source to two ranks)
  //    raises a flag and the general path (sort + unique) runs instead; the sums are right either way.
  pad_keys_kernel<<<grid, 256, 0, s>>>(h->d_keys[1], n_local, c->d_sorted, pad);
  NK(g_nccl.AllGather(c->d_sorted, c->d_gather, pad, ncclUint64, c->comm, s));
  CK(cudaMemsetAsync(c->d_flags, 0, 4, s));
  merge_disjoint_kernel<<<grid, 256, 0, s>>>(c->d_gather, pad, (uint32_t)R, c->d_counts, c->d_can_keys, c->d_flags);
  uint32_t dup = 0;
  CK(cudaMemcpyAsync(&dup, c->d_flags, 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  uint32_t n_can = (uint32_t)total;
  if (dup) {
    launch_iota(c->d_iota, n_g, h->sms, s);
    sort_pairs(c->d_tmp, c->tmp_bytes, c->d_gather, c->d_sorted, c->d_iota, c->d_vals, n_g, s);
    launch_unique_sorted(c->d_sorted, n_g, c->d_flags, c->d_pos, c->d_can_keys, c->d_tmp, c->tmp_bytes, h->sms, s);
    uint32_t last[2];
    CK(cudaMemcpyAsync(&last[0], c->d_pos + (n_g - 1), 4, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(&last[1], c->d_flags + (n_g - 1), 4, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    n_can = last[0] + last[1];
  }
  if (n_can > h->cfg.max_edges) return drop_window(h, lost, at_e);

  // 3. scatter local rows into the zeroed canonical array
  const size_t can_bytes = (size_t)n_can * kCanWords * 8;
  CK(cudaMemsetAsync(c->d_can, 0, can_bytes, s));
  if (n_local)
    scatter_canonical_kernel<<<grid * 2, 256, 0, s>>>(h->edges, h->d_keys[1], h->d_rows[1], n_local,
                                                      c->d_can_keys, n_can, c->d_can);
  // 4. the single exchange step
  NK(g_nccl.AllReduce(c->d_can, c->d_can, (size_t)n_can * kCanWords, ncclUint64, ncclSum, c->comm, s));
  h->collective_bytes_last += can_bytes;
  h->launches += 5;
  // 5. unpack; local edge table back to empty
  unpack_canonical_kernel<<<grid * 2, 256, 0, s>>>(c->d_can_keys, c->d_can, n_can, h->d_out);
  CK(cudaGetLastError());
  if (at_e) { CK(edge_table_clear(h->edges, h->sms, s)); h->launches += 1; }
  h->last_n_edges = n_can;
  h->windows++;
  return ALZ_OK;
}

// Called by the flush after prepare_flush(): local live edges are sorted in d_keys[1] (keys) / d_rows[1]
// (rows), h->n_live of them; local_rc is this rank's status so far, *lost whether it lost events. Every rank
// enters the collective whatever its own status, so nobody is left waiting in NCCL, and all ranks return the
// same status. Under a window clock the header carries the rank's clock, and *roll says whether the flush closes
// this rank's window (see kAtE / kKeep / kOpenNext).
const uint64_t* alz_internal_merged_clock(alz_handle* h) { return reinterpret_cast<const uint64_t*>(&h->comm->d_info->clk); }

int alz_internal_merge_ranks(alz_handle* h, int local_rc, bool* lost, bool* roll) {
  alz_comm_state* c = h->comm;
  const int R = h->comm_nranks;
  if (!c || R <= 1 || R > 64) return ALZ_E_STATE;   // alz_comm_init admits 2..64 ranks here
  cudaStream_t s = h->stream;
  const unsigned grid = (unsigned)h->sms * 4;
  const uint32_t n_local = local_rc == ALZ_OK ? h->n_live : 0u;
  const bool lost_here = *lost;
  h->collective_bytes_last = 0;
  *roll = true;

  if (c->cap_r == 0) {   // first window: nothing to size the blocks from, exchange the counts once
    CK(cudaMemcpyAsync(c->d_counts + h->comm_rank, &n_local, 4, cudaMemcpyHostToDevice, s));
    NK(g_nccl.AllGather(c->d_counts + h->comm_rank, c->d_counts, 1, ncclUint32, c->comm, s));
    CK(cudaMemcpyAsync(c->h_counts, c->d_counts, 4 * R, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    uint32_t mx = 0;
    for (int r = 0; r < R; ++r) mx = std::max(mx, c->h_counts[r]);
    c->cap_r = block_rows_for(mx);
  }
  // local rows behind the header, in canonical order; the window is NOT reset yet
  if (n_local) {
    launch_gather_edges(h->edges, h->d_keys[1], h->d_rows[1], n_local, c->d_send + 1, h->sms, s);
    h->launches += 1;
  }
  for (int attempt = 0; attempt < 4; ++attempt) {
    memset(c->h_hdr, 0, sizeof(alz_edge_out));
    c->h_hdr->magic = kHdrMagic; c->h_hdr->count = n_local; c->h_hdr->status = local_rc;
    c->h_hdr->lost = lost_here ? 1u : 0u;
    c->h_hdr->clk_on = h->win_on ? 1u : 0u;
    CK(cudaMemcpyAsync(c->d_send, c->h_hdr, sizeof(alz_edge_out), cudaMemcpyHostToDevice, s));
    if (h->win_on)   // the clock as the device has it: win_init_kernel may have opened it in this window
      CK(cudaMemcpyAsync(&reinterpret_cast<BlockHeader*>(c->d_send)->clk, h->d_win, sizeof(WinClock),
                         cudaMemcpyDeviceToDevice, s));
    const size_t block_rows = (size_t)c->cap_r + 1;
    if (block_rows * R > c->recv_rows) {
      CK(cudaStreamSynchronize(s));
      cudaFree(c->d_recv);
      c->d_recv = nullptr;
      c->recv_rows = block_rows * R;
      CK(cudaMalloc(&c->d_recv, c->recv_rows * sizeof(alz_edge_out)));
    }
    CK(cudaMemsetAsync(c->d_info, 0, sizeof(MergeInfo), s));
    // the single exchange step: every rank's header + its first cap_r rows
    NK(g_nccl.AllGather(c->d_send, c->d_recv, block_rows * kRowWords64, ncclUint64, c->comm, s));
    h->collective_bytes_last += (uint64_t)block_rows * R * kRowBytes;
    merge_blocks_kernel<<<grid, 256, 0, s>>>(c->d_recv, c->cap_r, (uint32_t)R, (uint32_t)h->comm_rank, h->d_out,
                                             h->cfg.max_edges, c->d_info);
    consume_window_kernel<<<grid, 256, 0, s>>>(c->d_info, h->edges, h->d_rows[1], n_local);
    h->launches += 2;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(c->h_info, c->d_info, sizeof(MergeInfo), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));   // the flush's one synchronisation: the caller needs the edge count
    const MergeInfo inf = *c->h_info;
    if (inf.peer_status != ALZ_OK) return local_rc != ALZ_OK ? local_rc : inf.peer_status;   // the window stays intact
    if (inf.overflow != 0u) { c->cap_r = block_rows_for(inf.max_count); continue; }   // every rank sees the same headers
    c->cap_r = block_rows_for(inf.max_count);                                         // next window's block size
    *lost = inf.lost != 0u;                                                           // some rank at E lost events
    *roll = inf.roll != kKeep;
    if (inf.roll == kKeep && lost_here) h->lost_reported = ~0ull;   // the window is kept: report its loss with it
    if (inf.roll == kOpenNext)   // E's clock; the flush's roll advances it to E + 1
      CK(cudaMemcpyAsync(h->d_win, &c->d_info->clk, sizeof(WinClock), cudaMemcpyDeviceToDevice, s));
    if (inf.dup) return merge_allreduce(h, lost, inf.roll == kAtE);                   // not partitioned by owner: general path
    // success: consume_window_kernel has consumed the window; rows past max_edges were left out
    if (inf.total > h->cfg.max_edges) { *lost = true; h->merge_lost_events += inf.lost_events; }
    h->last_n_edges = std::min<uint32_t>(inf.total, h->cfg.max_edges);
    h->windows++;
    return ALZ_OK;
  }
  return ALZ_E_CAPACITY;
}
