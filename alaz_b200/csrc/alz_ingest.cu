// alz_ingest.cu — the dominant kernel: l7 events -> per-socket-pair accumulators
// (DESIGN.md §3 step 1, §5). One persistent CTA per SM.
//
// Data movement: every warp owns a two-stage ring in shared memory and streams its chunks of the
// record array into it with TMA bulk copies (cp.async.bulk + mbarrier complete_tx, issued by one
// elected lane, L2 evict-first). Lanes copy their records from the ring into registers, the stage
// goes back to the TMA as soon as those loads have returned, and the next two chunks are in flight
// while the warp works: no per-lane address arithmetic, no scoreboard stall on the first use of a
// streamed record (plain loads, even prefetched into L2 by the TMA engine, stall on it), no
// cross-warp barrier anywhere in the main loop.
//
// Work per event, three tiers:
//   hot   the event's socket pair is in the CTA's shared-memory table. A row holds a 16-bucket
//         WINDOW of the latency histogram in 16-bit cells (52 bytes instead of 292: the window is
//         where the pair's latencies fall, chosen from its own histogram at the previous fold), so
//         ~1250 pairs fit and ~77 % of the events of a Zipf(1.1) stream end here: one 8-byte load of a
//         2-way bucket of the index (fingerprint | window | row per entry), one key load, two shared
//         reductions. 16-bit cells stay exact: the lane that sees a cell at 0x7FFF spills 0x8000
//         counts into the global table (bit 15 is head room for the increments racing with it).
//   cold  everything else (a pair without a row, a latency outside its row's window, a host-keyed
//         row) is NOT handled inline: the lane pushes the event onto its warp's
//         queue (ballot-compacted, no atomics) and the warp runs the cold path for 32 queued
//         events at a time with all lanes busy — global dictionary probe of the home slot, then
//         the reduction into the pair's row in L2: ONE red.u64 per event, a lane pair adding the
//         histogram cell and the duration into the 32-byte sector of the row that holds both
//         (global_add_paired; the SM pays per sector an instruction touches, not per lane). The
//         probes are cp.async copies into shared memory and are consumed when the next batch is
//         requested, one to three iterations later, so their L2/DRAM round trip is off the warp's
//         critical path. A source address
//         that cannot be a pod (a 128-Kbit filter of the pod addresses, built by the host at table
//         commit) is dropped right there, as setFromToV2 would (aggregator/data.go:829-832).
//   slow  a cold event whose home slot does not hold its pair (new pair, collision) is queued once
//         more and 32 of them at a time walk find_or_insert_pair.

#include <algorithm>

#include "alz_kernels.cuh"
#include "alz_mbar.cuh"

namespace alz {

// Cycle accounting per section of the main loop, summed over warps (profiling build only: -DALZ_INGEST_PROF,
// alaz_b200/build.py --prof -> libalazgpu_prof.so; read with alz_debug_ingest_prof). Tells where a warp's time
// goes in a REAL run — ncu's kernel replay flushes the caches between passes unless told otherwise.
#ifdef ALZ_INGEST_PROF
__device__ unsigned long long g_ingest_prof[8];
__device__ unsigned long long g_ingest_phase[4];   // per CTA, summed: prologue, main loop until the slowest warp, drain; CTAs
#define PROF_PHASE(i, v) do { if (threadIdx.x == 0) atomicAdd(&g_ingest_phase[i], (unsigned long long)(v)); } while (0)
#define PROF_DECL unsigned long long pt[8] = {0, 0, 0, 0, 0, 0, 0, 0}; long long pc0 = 0, pc1 = 0; (void)pc0; (void)pc1
#define PROF_NOW() clock64()
#define PROF_ADD(i, v) pt[i] += (unsigned long long)(v)
#define PROF_FLUSH() do { if ((threadIdx.x & 31u) == 0) for (int i_ = 0; i_ < 8; ++i_) atomicAdd(&g_ingest_prof[i_], pt[i_]); } while (0)
// Per-CTA timeline of the last kTlLaunches launches (read with alz_debug_ingest_timeline): for every CTA, %globaltimer
// at entry, at the end of the main loop (after its __syncthreads) and at the end of the drain, %smid, clock64 at entry
// and at the end (their ratio to the timer is the SM clock), and the chunks its warps took. Launches are numbered in
// stream order: the last CTA of a launch to finish moves the number on, before the next launch can start.
constexpr uint32_t kTlLaunches = 64, kTlCtas = 256, kTlWords = 8;
__device__ unsigned long long g_ingest_tl[kTlLaunches][kTlCtas][kTlWords];
__device__ unsigned int g_ingest_tl_launch, g_ingest_tl_done;
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ unsigned int sm_id() {
  unsigned int r;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(r));
  return r;
}
#define TL_DECL unsigned long long tl_t0 = 0, tl_c0 = 0, tl_t1 = 0; unsigned int tl_launch = 0; (void)tl_t1; (void)tl_launch
#define TL_ENTRY() do { if (threadIdx.x == 0) { tl_launch = *(volatile unsigned int*)&g_ingest_tl_launch; tl_c0 = clock64(); tl_t0 = global_ns(); } } while (0)
#define TL_LOOP_END() do { if (threadIdx.x == 0) tl_t1 = global_ns(); } while (0)
#define TL_CHUNKS(v) do { if ((threadIdx.x & 31u) == 0 && blockIdx.x < kTlCtas) \
    atomicAdd(&g_ingest_tl[*(volatile unsigned int*)&g_ingest_tl_launch % kTlLaunches][blockIdx.x][6], (unsigned long long)(v)); } while (0)
#define TL_EXIT() do { if (threadIdx.x == 0) {                                                              \
    const unsigned long long t2_ = global_ns(), c2_ = clock64();                                            \
    if (blockIdx.x < kTlCtas) {                                                                             \
      unsigned long long* e_ = g_ingest_tl[tl_launch % kTlLaunches][blockIdx.x];                           \
      e_[0] = tl_t0; e_[1] = tl_t1; e_[2] = t2_; e_[3] = sm_id(); e_[4] = tl_c0; e_[5] = c2_;             \
    }                                                                                                       \
    __threadfence();                                                                                        \
    if (atomicAdd(&g_ingest_tl_done, 1u) == gridDim.x - 1u) { g_ingest_tl_done = 0u; atomicAdd(&g_ingest_tl_launch, 1u); } \
  } } while (0)
#else
#define PROF_DECL long long pc0 = 0, pc1 = 0; (void)pc0; (void)pc1
#define PROF_NOW() 0ll
#define PROF_ADD(i, v)
#define PROF_FLUSH()
#define PROF_PHASE(i, v)
#define TL_DECL
#define TL_ENTRY()
#define TL_LOOP_END()
#define TL_CHUNKS(v)
#define TL_EXIT()
#endif

namespace {

constexpr uint32_t kRowWords = 13;         // 8 words = 16 x u16 histogram cells, err5xx u32, 2 x (lat_lo, lat_hi); odd stride
constexpr uint32_t kCellSpill = 0x7FFFu;   // a 16-bit cell seen at this value is spilled (bit 15 = head room)
constexpr uint32_t kTab = 4096;            // index entries: fingerprint 16 | window base 4 | row 12, in buckets of two
constexpr uint32_t kTabShift = 20;
constexpr uint32_t kRowMask = 0xFFFu;
constexpr uint32_t kBusy = kRowMask;       // entry whose row field is no row: claimed, not (or never) published
constexpr uint32_t kColdQ = 128;           // cold queue entries per warp (ring): up to 31 left over + 32 + 64 new ones
constexpr uint32_t kSlowQ = 64;            // slow queue entries per warp (ring)
constexpr uint32_t kQBytes = 16;           // queue entry {key u64, dur_lo u32, meta u32}
constexpr uint32_t kSmemMax = 232448;      // 227 KB per CTA on sm_90
constexpr int kDefaultWarps = 16;
constexpr int kMaxWarps = kDefaultWarps;   // cursors per handle (ChunkSched)
constexpr int kU = 2;                      // events per lane per iteration
constexpr uint32_t kChunk = 32u * kU;      // events per warp per iteration = one TMA copy
constexpr uint32_t kDynEighths = 3;        // the last 3/8 of a launch's rounds of chunks are claimed, not assigned
constexpr uint32_t kClaim = 2;             // chunks per claim from a cursor
constexpr uint32_t kCursorStride = 64;     // u32 words between two cursors: one 256-byte line each

template <int kWarps, int kRecWords>
struct Layout {
  static constexpr uint32_t kChunkBytes = kChunk * kRecWords * 4u;
  static constexpr uint32_t kRing = (uint32_t)kWarps * 2u * kChunkBytes;
  static constexpr uint32_t kBars = kRing;                              // kWarps * 2 mbarriers
  static constexpr uint32_t kTabOff = kBars + (uint32_t)kWarps * 16u;
  static constexpr uint32_t kBloomOff = kTabOff + kTab * 4u;            // pod-address filter, ALZ_BLOOM_WORDS words
  static constexpr uint32_t kColdOff = kBloomOff + ALZ_BLOOM_WORDS * 4u;
  static constexpr uint32_t kSlowOff = kColdOff + (uint32_t)kWarps * kColdQ * kQBytes;
  static constexpr uint32_t kProbeOff = kSlowOff + (uint32_t)kWarps * kSlowQ * kQBytes;   // per warp: 32 x 16-B DictEnt
  static constexpr uint32_t kMisc = kProbeOff + (uint32_t)kWarps * 512u;                  // row allocator
  static constexpr uint32_t kScratchOff = kMisc + 16u;                                    // per warp: one word per lane
  static constexpr uint32_t kRowKeys = kScratchOff + (uint32_t)kWarps * 128u;
  static constexpr uint32_t kPerRow = 8u + kRowWords * 4u + 1u;         // key, cells, window base
  static constexpr uint32_t kRowsRaw = (kSmemMax - kRowKeys - 64u) / kPerRow - 1u;
  static constexpr uint32_t kRows = (kRowsRaw < 4064u ? kRowsRaw : 4064u) / 32u * 32u;
  static constexpr uint32_t kRowsOff = kRowKeys + (kRows + 1u) * 8u;    // row kRows: scratch target of clamped indices
  static constexpr uint32_t kBaseOff = kRowsOff + (kRows + 1u) * kRowWords * 4u;
  static constexpr uint32_t kBytes = kBaseOff + ((kRows + 1u + 15u) / 16u) * 16u;
  static constexpr uint32_t kPreload = kRows - kRows / 8u;              // rows the hot list may take
  static_assert(kBytes <= kSmemMax, "shared memory layout too large");
  static_assert(kRows < kBusy, "row field is 12 bits");
  static_assert(kRows * 3u <= kTab * 2u, "index too small for the rows");
};

// ---- PTX helpers ----------------------------------------------------------------------------
// global reductions are written as PTX red so that no fence elsewhere in the kernel can turn them into
// returning atomics (r1 found nvcc emitting ATOMG for every atomicAdd once a __threadfence_block() was present)
__device__ __forceinline__ void red_add_u32(uint32_t* p, uint32_t v) {
  asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void red_add_u64(uint64_t* p, uint64_t v) {
  asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// the same with an L2 eviction-priority hint: the pair dictionary and the pair rows are the kernel's random-access
// working set (~100 MB at config 2, against 50 MB of L2 on an H100, with 3.2 GB of records streaming through): marked
// evict-last, as much of it as fits stays resident instead of being pushed out by the stream
__device__ __forceinline__ void red_add_u32_keep(uint32_t* p, uint32_t v, uint64_t pol) {
  asm volatile("red.relaxed.gpu.global.add.L2::cache_hint.u32 [%0], %1, %2;" ::"l"(p), "r"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void red_add_u64_keep(uint64_t* p, uint64_t v, uint64_t pol) {
  asm volatile("red.relaxed.gpu.global.add.L2::cache_hint.u64 [%0], %1, %2;" ::"l"(p), "l"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ bool elect_one() {   // one lane of the (converged) warp
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xFFFFFFFF;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0u;
}
__device__ __forceinline__ uint32_t shr_clamp(uint32_t v, uint32_t by) {   // PTX shr: amounts > 31 give 0
  uint32_t r;
  asm("shr.b32 %0, %1, %2;" : "=r"(r) : "r"(v), "r"(by));
  return r;
}
// ---- TMA / cp.async (PTX; the mbarrier helpers are in alz_mbar.cuh) ----------------------------
// global -> shared bulk copy, completion counted on the mbarrier; L2 evict-first so that the stream does not
// push the accumulator rows out of L2
__device__ __forceinline__ void tma_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, uint64_t policy) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar), "l"(policy) : "memory");
}
// 16-byte global -> shared copy that no register waits on (LDGSTS); L2 only (the dictionary is written by other CTAs)
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint64_t pol) {
  asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "l"(pol) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// docs/SPEC.md §4 through the float exponent: round-toward-zero keeps floor(log2 d) and the next mantissa bit
// exact for every u64, so bits >> 22 = 2 * (127 + o) + bit(o-1); one conversion instead of a 64-bit clz chain
__device__ __forceinline__ uint32_t latency_bucket_rz(uint64_t d) {
  const int b = (int)(__float_as_uint(__ull2float_rz(d)) >> 22) - 2 * (127 + 8);
  return (uint32_t)min(max(b, 0), ALZ_NB - 1);
}

// processL7's switch (aggregator/data.go:1364-1383) as a 3-bit class per protocol value, packed in one word:
// bit 0 a request row is built (HTTP 1, AMQP 2, POSTGRES 3, REDIS 5, MYSQL 7, MONGO 8), bit 1 the row is dropped
// when the payload parser rejected it (POSTGRES, MYSQL, MONGO), bit 2 method 2 reverses the row (AMQP DELIVER,
// REDIS PUSHED_EVENT). Protocol values > 8 shift everything out: class 0 = no row.
constexpr uint32_t proto_class(uint32_t p) {
  return ((0x1AEu >> p) & 1u) | (((0x188u >> p) & 1u) << 1) | (((0x024u >> p) & 1u) << 2);
}
constexpr uint32_t kProtoLut = proto_class(0) | proto_class(1) << 3 | proto_class(2) << 6 | proto_class(3) << 9 |
                               proto_class(4) << 12 | proto_class(5) << 15 | proto_class(6) << 18 |
                               proto_class(7) << 21 | proto_class(8) << 24;

// hash of the per-CTA table only: two multiply-adds; index 1 from its top bits, index 2 from the top bits of
// one more multiply, the fingerprint from its low bits. Weak low bits only cost a wasted key load (the row's key
// decides). The dictionary hash (pair_hash) is computed for cold events only.
__device__ __forceinline__ uint32_t table_hash(uint64_t key) {
  return (uint32_t)key * 0x9E3779B1u + (uint32_t)(key >> 32) * 0x85EBCA6Bu;
}
// Forward and reversed rows of one socket pair are separate rows of the table (the per-CTA table holds no host-keyed
// rows). A reversed pair hashes to table_hash(key) ^ kRevSalt: another index bucket, and a fingerprint that differs
// from the forward one of the same key in bit 17 (kRevSalt bit 1), so an entry whose row holds the event's key is
// always of the event's kind.
constexpr uint32_t kRevSalt = 0x5BD1E996u;
static_assert((kRevSalt & 2u) != 0u, "the two kinds of one key must differ in a fingerprint bit");
__device__ __forceinline__ uint32_t table_hash_kind(uint64_t key, uint32_t kind) {
  return table_hash(key) ^ (kind == kPairRev ? kRevSalt : 0u);
}
// the key's two index slots are the two halves of one 8-byte bucket: one LDS.64 fetches both (two independent
// 4-byte probes cost two instructions and, with 32 random addresses each, about twice the shared-memory passes)
__device__ __forceinline__ uint32_t tab_idx1(uint32_t h) { return (h >> kTabShift) & ~1u; }
__device__ __forceinline__ uint32_t tab_idx2(uint32_t h) { return (h >> kTabShift) | 1u; }
// the filter of pod addresses (alz_api.cu keeps it in step with the table): false = certainly not a pod
__device__ __forceinline__ bool maybe_pod(const uint32_t* bloom, uint32_t ip) {
  const uint32_t h = hash32(ip);
  const uint32_t b1 = h & (ALZ_BLOOM_WORDS * 32u - 1u), b2 = (h >> 15) & (ALZ_BLOOM_WORDS * 32u - 1u);
  return ((bloom[b1 >> 5] >> (b1 & 31u)) & (bloom[b2 >> 5] >> (b2 & 31u)) & 1u) != 0u;
}
__device__ __forceinline__ uint32_t tab_fp(uint32_t h) { return (h << 16) | 0x10000u; }   // never 0 in bits 31..16
__device__ __forceinline__ uint32_t tab_entry(uint32_t h, uint32_t base4, uint32_t row) { return tab_fp(h) | (base4 << 12) | row; }

struct Shared {
  uint32_t* tab;      // [kTab]
  uint32_t* bloom;    // [ALZ_BLOOM_WORDS]
  uint64_t* rowkey;   // [kRows + 1], entry kRows = kEmptyKey (never a hit)
  uint32_t* rows;     // [(kRows + 1) * kRowWords]
  uint8_t* rowbase;   // [kRows + 1] first bucket / 4 of the row's window (also in its index entry) | pair kind << 4
  uint32_t* n_rows;   // rows handed out
};

// claim one of the key's two index slots and give it a row; false if both are taken or the rows are used up.
// h = table_hash_kind(key, kind). `publish_fenced`: other warps are probing concurrently, so the row's key must be
// visible before the entry
__device__ __forceinline__ bool smem_admit(const Shared& s, uint64_t key, uint32_t kind, uint32_t h, uint32_t base4,
                                           uint32_t limit, bool publish_fenced) {
  uint32_t idx = tab_idx1(h);
  if (atomicCAS(&s.tab[idx], 0u, kBusy) != 0u) {
    idx = tab_idx2(h);
    if (atomicCAS(&s.tab[idx], 0u, kBusy) != 0u) return false;
  }
  const uint32_t row = atomicAdd(s.n_rows, 1u);
  if (row >= limit) return false;                       // slot stays kBusy: reads as a miss for everyone
  s.rowkey[row] = key;
  s.rowbase[row] = (uint8_t)(base4 | (kind << 4));
  if (publish_fenced) __threadfence_block();
  *reinterpret_cast<volatile uint32_t*>(&s.tab[idx]) = tab_entry(h, base4, row);
  return true;
}
// window for a pair admitted without history: centred on the bucket of the event that brought it in
__device__ __forceinline__ uint32_t base4_around(uint32_t bucket) { return (uint32_t)min(max((int)bucket - 6, 0), 48) >> 2; }

// one warp's queue of deferred events in shared memory: a ring of 16-byte entries {key u64, dur_lo u32, meta u32}
// filled by ballot compaction. meta: bits 0..5 latency bucket, 6..7 pair kind, bit 8 counts as 5xx, bits 9..31
// the duration's high word (events whose duration does not fit, >= 2^55 ns, are handled on the spot)
template <uint32_t kCap>
struct Queue {
  uint8_t* base;
  uint32_t head, count;
  __device__ __forceinline__ void bind(uint8_t* b) { base = b; head = 0; count = 0; }
  __device__ __forceinline__ uint4* at(uint32_t i) const {
    return reinterpret_cast<uint4*>(base + ((head + i) & (kCap - 1u)) * kQBytes);
  }
  __device__ __forceinline__ uint32_t push(bool want, uint64_t k, uint32_t dlo, uint32_t m, uint32_t lane_lt) {
    const uint32_t mask = __ballot_sync(0xFFFFFFFFu, want);
    if (want) *at(count + __popc(mask & lane_lt)) = make_uint4((uint32_t)k, (uint32_t)(k >> 32), dlo, m);
    const uint32_t added = __popc(mask);
    count += added;
    return added;
  }
  __device__ __forceinline__ void pop(uint32_t n) { head = (head + n) & (kCap - 1u); count -= n; }
};
using SlowQueue = Queue<kSlowQ>;
using ColdQueue = Queue<kColdQ>;

// Which chunks a warp takes, in order. The first rounds keep a static map: in round r, warp w of the grid takes
// chunk r * stride + w. The chunks after them, the last kDynEighths / 8 of the rounds, are claimed, so a warp whose
// SM runs fast takes more of them and every SM finishes the launch at about the same time (the static share alone
// left the latest CTA ~0.45 ms after the median one at config 2, DESIGN.md §5.2). Claimed chunk dyn0 + j belongs to
// warp slot j mod kWarps of whichever CTA claims it: slot p's chunks are handed out kClaim at a time from cursor p,
// which is zero at the start of every launch. One cursor for all warps took ~0.3 G claims/s at config 2, enough to
// queue the claims at that line's L2 slice for longer than two loop iterations; kWarps cursors on their own lines
// see 1/kWarps of them each. Warps of one CTA run at about the same speed, so the split by slot costs no balance.
// Lane 0 makes the claims; the result is broadcast only when its first chunk is needed, kClaim chunks later (two loop
// iterations), so the issue of the copy does not wait on the atomic. The sequence is strictly increasing: static
// chunks lie below `dyn0`, and one thread's claims on one address come back in increasing order. So once it reaches
// n_chunks, the warp has taken every chunk it was handed, and every chunk below n_chunks is taken by exactly one warp
// (tests/test_ingest_sched_model.py runs the protocol on the host). All lanes call next() together and hold the same
// state, so any lane can be the one that issues the copy.
template <int kWarps>
struct ChunkSched {
  uint32_t* cursor;                    // this warp slot's cursor
  uint32_t st_next, st_left, stride;   // next static chunk, static chunks left, chunks per round
  uint32_t dyn0;                       // first claimed chunk of this warp slot
  uint32_t blk, blk_left;              // the claimed chunks being handed out: blk, blk + kWarps, ...
  uint32_t claim;                      // lane 0: the cursor value of the claim made ahead
  __device__ __forceinline__ void claim_ahead(uint32_t lane) { if (lane == 0u) claim = atomicAdd(cursor, kClaim); }
  __device__ __forceinline__ void init(uint32_t* cursors, uint32_t n_chunks, uint32_t warp, uint32_t c_stride,
                                       uint32_t lane) {
    cursor = cursors + warp * kCursorStride;
    stride = c_stride;
    const uint32_t first = blockIdx.x * kWarps + warp;
    const uint32_t rounds = (uint32_t)(((uint64_t)n_chunks + c_stride - 1u) / c_stride);
    st_left = rounds - (uint32_t)((uint64_t)rounds * kDynEighths / 8u);
    st_next = first;
    dyn0 = st_left * c_stride + warp;
    blk = 0u; blk_left = 0u; claim = 0u;
    if (st_left <= kClaim) claim_ahead(lane);
  }
  __device__ __forceinline__ uint32_t next(uint32_t lane) {
    if (st_left != 0u) {
      const uint32_t c = st_next;
      st_next += stride;
      if (--st_left == kClaim) claim_ahead(lane);
      return c;
    }
    if (blk_left == 0u) {
      blk = dyn0 + __shfl_sync(0xFFFFFFFFu, claim, 0) * kWarps;
      blk_left = kClaim;
      claim_ahead(lane);
    }
    --blk_left;
    const uint32_t c = blk;
    blk += kWarps;
    return c;
  }
};

// the global path for one event whose pair row is known
__device__ __forceinline__ uint64_t keep_policy() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void global_add(const PairTable& t, uint32_t row, uint32_t bucket, uint64_t dur, bool err) {
  const uint64_t pol = keep_policy();
  uint64_t* sc = pair_sect(t, row, bucket);
  red_add_u32_keep(reinterpret_cast<uint32_t*>(sc) + (bucket & 3u), 1u, pol);
  red_add_u64_keep(sc + 2, dur, pol);
  if (err) red_add_u64_keep(sc + 3, 1ull, pol);
}
// The same for up to 32 events held one per lane (`on`, row, meta = bucket | ... | err << 8 | dur_hi << 9, dur_lo), as
// ONE red.u64 instruction per 16 events: lane pair (2j, 2j+1) takes one event, the even lane adds to the cell pair,
// the odd lane the duration, both in the event's sector, which the LSU serves in one pass (alz_device.cuh, PairTable).
// Round r takes the events of lanes 16r..16r+15. All lanes must call this.
__device__ __forceinline__ void global_add_paired(const PairTable& t, bool on, uint32_t row, uint32_t meta, uint32_t dlo) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t have = __ballot_sync(0xFFFFFFFFu, on);
  if (have == 0u) return;
  const uint64_t pol = keep_policy();
  const uint32_t odd = lane & 1u;
#pragma unroll
  for (uint32_t r = 0; r < 2u; ++r) {
    if ((have & (r ? 0xFFFF0000u : 0x0000FFFFu)) == 0u) continue;   // warp-uniform
    const uint32_t src = r * 16u + (lane >> 1);
    const uint32_t row_s = __shfl_sync(0xFFFFFFFFu, row, src);
    const uint32_t meta_s = __shfl_sync(0xFFFFFFFFu, meta, src);
    const uint32_t dlo_s = __shfl_sync(0xFFFFFFFFu, dlo, src);
    if ((have >> src) & 1u) {
      uint64_t* sc = pair_sect(t, row_s, meta_s & 0x3Fu);
      const uint64_t dur = ((uint64_t)(meta_s >> 9) << 32) | dlo_s;
      red_add_u64_keep(odd ? sc + 2 : sc + ((meta_s & 3u) >> 1), odd ? dur : 1ull << (32u * (meta_s & 1u)), pol);
      if (odd && (meta_s & 0x100u)) red_add_u64_keep(sc + 3, 1ull, pol);   // 5xx: rare
    }
  }
}

// slow tier for one event (walks the dictionary): the pair is new to it, or its home slot is taken by another
// pair, or its source is no pod (dropped like the reference does, aggregator/data.go:829-832)
template <uint32_t kRows>
__device__ __forceinline__ void slow_one(uint64_t key, uint64_t dur, uint32_t bucket, uint32_t kind, bool err,
                                         const PairTable& t, const Shared& s, const EpEntry* __restrict__ ep,
                                         uint32_t ep_mask, uint32_t* lost, uint32_t* unresolved) {
  const uint32_t row = find_or_insert_pair(t, key, kind, ep, ep_mask);
  if (row >= kDropRow) { if (row == kDropRow) *unresolved += 1u; else *lost += 1u; return; }
  global_add(t, row, bucket, dur, err);
  // a pair the per-CTA table does not hold: give it a private row while some are left (first-come)
  if (kind != kPairHost && key != kEmptyKey && *reinterpret_cast<volatile uint32_t*>(s.n_rows) < kRows)
    smem_admit(s, key, kind, table_hash_kind(key, kind), base4_around(bucket), kRows, true);
}
template <uint32_t kRows>
__device__ __forceinline__ void slow_batch(SlowQueue& q, uint32_t count, const PairTable& t, const Shared& s,
                                           const EpEntry* __restrict__ ep, uint32_t ep_mask, uint32_t* lost,
                                           uint32_t* unresolved) {
  const uint32_t lane = threadIdx.x & 31u;
  if (lane < count) {
    const uint4 e = *q.at(lane);
    const uint64_t key = ((uint64_t)e.y << 32) | e.x;
    const uint64_t dur = ((uint64_t)(e.w >> 9) << 32) | e.z;
    slow_one<kRows>(key, dur, e.w & 0x3Fu, (e.w >> 6) & 3u, (e.w & 0x100u) != 0u, t, s, ep, ep_mask, lost, unresolved);
  }
  __syncwarp();
  q.pop(count);
}

// cold tier, step 1: request the dictionary home slots of the first `count` queued events — unless the event's
// source address cannot be a pod, in which case no row would be emitted (aggregator/data.go:829-832): its probe
// slot is marked instead. The 16-byte entries are copied straight into the warp's probe buffer in shared memory
// (cp.async): nothing waits on them until the batch is consumed, which happens when the NEXT batch is ready to be
// requested. (Holding the probes in registers did not work: handing them from one loop trip to the next needs a
// move, and the move waits for the load.)
__device__ __forceinline__ void cold_issue(const ColdQueue& q, uint32_t count, const PairTable& t, const Shared& s,
                                           uint4* probe, uint32_t probe_a) {
  const uint32_t lane = threadIdx.x & 31u;
  if (lane < count) {
    const uint4 e = *q.at(lane);
    const uint32_t kind = (e.w >> 6) & 3u;
    if (!maybe_pod(s.bloom, e.x)) probe[lane] = make_uint4(0u, 0u, kDropRow, 1u);      // e.x = the key's low word = saddr
    else {
      const uint64_t key = ((uint64_t)e.y << 32) | e.x;
      cp_async16(probe_a + lane * 16u, &t.dict_of(kind)[pair_hash(key) & t.mask_of(kind)], keep_policy());
    }
  }
  cp_async_commit();
}
// cold tier, step 2: the probes have landed. A home-slot hit is reduced into its row at once, a filtered source is
// counted, anything else joins the slow queue.
template <uint32_t kRows>
__device__ __forceinline__ void cold_consume(ColdQueue& q, uint32_t count, const uint4* probe, SlowQueue& slow,
                                             const PairTable& t, const Shared& s, const EpEntry* __restrict__ ep,
                                             uint32_t ep_mask, uint32_t lane_lt, uint32_t* lost, uint32_t* unresolved,
                                             unsigned long long* t_wait, unsigned long long* t_slow) {
  const uint32_t lane = threadIdx.x & 31u;
  const long long w0 = PROF_NOW();
  cp_async_wait_all();
  *t_wait += (unsigned long long)(PROF_NOW() - w0);
  const bool valid = lane < count;
  uint4 e = make_uint4(0u, 0u, 0u, 0u), ent = make_uint4(0u, 0u, kNoRow, 0u);
  if (valid) { e = *q.at(lane); ent = probe[lane]; }
  const bool filtered = valid && ent.z == kDropRow && ent.w == 1u;
  // the row word of the event's kind; a slot that has the pair but no row of this kind yet goes to the slow queue
  const uint32_t row = ((e.w >> 6) & 3u) == kPairRev ? ent.w : ent.z;
  const bool home = valid && !filtered && ent.x == e.x && ent.y == e.y && row < kClaimRow && (e.x & e.y) != 0xFFFFFFFFu;
  global_add_paired(t, home, row, e.w, e.z);
  if (filtered) *unresolved += 1u;
  slow.push(valid && !home && !filtered, ((uint64_t)e.y << 32) | e.x, e.z, e.w, lane_lt);
  __syncwarp();
  q.pop(count);
  if (slow.count >= 32u) {
    const long long s0 = PROF_NOW();
    slow_batch<kRows>(slow, 32u, t, s, ep, ep_mask, lost, unresolved);
    *t_slow += (unsigned long long)(PROF_NOW() - s0);
  }
}

// End of a launch, all warps (after a __syncthreads): drain the private rows into the global table and publish
// the launch's counters.
template <int kWarps, uint32_t kRows, bool kWin>
__device__ __forceinline__ void drain_rows_and_count(const Shared& s, const PairTable& pairs, Counters* ctr,
                                                     const EpEntry* __restrict__ ep, uint32_t ep_mask, uint32_t lost,
                                                     uint32_t unresolved, uint32_t n_hit, uint32_t n_live,
                                                     uint32_t n_cold, uint32_t n_late) {
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  // drain the private rows into the global table. Phase 1, a thread per row: find (or create) the pair's global
  // row — the dependent dictionary probes of up to 32 rows per warp overlap; the row number replaces the key's
  // low word. Phase 2, a half-warp per row: add the window's cells, 5xx count and latency sums.
  const uint32_t used = min(*s.n_rows, kRows);
  for (uint32_t r = threadIdx.x; r < used; r += kWarps * 32) {
    const uint64_t key = s.rowkey[r];
    const uint32_t* row = s.rows + r * kRowWords;
    uint32_t any = 0;
#pragma unroll
    for (int k = 0; k < (int)kRowWords; ++k) any |= row[k];
    uint32_t grow = kNoRow;                       // never hit in this launch: no global row needed
    if (key != kEmptyKey && any != 0u) grow = find_or_insert_pair(pairs, key, s.rowbase[r] >> 4, ep, ep_mask);
    reinterpret_cast<uint32_t*>(&s.rowkey[r])[0] = grow;
  }
  __syncthreads();
  const uint32_t hl = lane & 15u, half = lane >> 4;
  const uint32_t n_pass = (used + kWarps * 2u - 1u) / (kWarps * 2u);     // same trip count for both halves of a warp
  for (uint32_t ps = 0; ps < n_pass; ++ps) {
    const uint32_t r = ps * kWarps * 2u + warp * 2u + half;
    const bool valid = r < used;
    const uint32_t grow = valid ? reinterpret_cast<const uint32_t*>(&s.rowkey[r])[0] : kNoRow;
    const uint32_t* row = s.rows + (valid ? r : kRows) * kRowWords;
    const uint32_t cnt = (row[hl >> 1] >> ((hl & 1u) * 16u)) & 0xFFFFu;
    uint32_t tot = cnt;
    for (int o = 8; o > 0; o >>= 1) tot += __shfl_xor_sync(0xFFFFFFFFu, tot, o);
    if (grow == kNoRow) continue;
    if (grow >= kDropRow) {   // source is not a pod any more (dropped like the reference does) or capacity
      if (hl == 0) { if (grow == kDropRow) unresolved += tot; else lost += tot; }
      continue;
    }
    // the window's 16 cells = 4 sectors of the global row, 4 lanes each; the row's latency and 5xx totals go to the
    // partials of the window's first sector (any sector of the row would do: the fold sums them)
    const uint32_t base = ((uint32_t)s.rowbase[r] & 15u) * 4u;
    if (cnt) red_add_u32(pair_cell(pairs, grow, base + hl), cnt);
    if (hl == 0) {
      const uint64_t lat = (((uint64_t)row[10] << 32) + row[9]) + (((uint64_t)row[12] << 32) + row[11]);
      uint64_t* sc = pair_sect(pairs, grow, base);
      if (lat) red_add_u64(sc + 2, lat);
      if (row[8]) red_add_u64(sc + 3, (uint64_t)row[8]);
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    n_hit += __shfl_xor_sync(0xFFFFFFFFu, n_hit, o);
    n_cold += __shfl_xor_sync(0xFFFFFFFFu, n_cold, o);
    lost += __shfl_xor_sync(0xFFFFFFFFu, lost, o);
    unresolved += __shfl_xor_sync(0xFFFFFFFFu, unresolved, o);
  }
  // events that built no request row = events seen - hot hits - cold events (the last two are counted anyway);
  // n_live is the same in every lane
  const uint32_t not_request = n_live - n_cold - n_hit;
  if (kWin) for (int o = 16; o > 0; o >>= 1) n_late += __shfl_xor_sync(0xFFFFFFFFu, n_late, o);
  if (lane == 0) {
    if (not_request) atomicAdd(&ctr->not_request, (unsigned long long)not_request);
    if (lost) atomicAdd(&ctr->capacity_events, (unsigned long long)lost);
    if (unresolved) atomicAdd(&ctr->src_unresolved, (unsigned long long)unresolved);
    if (kWin && n_late) atomicAdd(&ctr->late_events, (unsigned long long)n_late);
  }
}

// Start of a launch, all threads: build the per-CTA table from the hot list of the previous fold. Tier S pairs get
// kHotRep rows each in rows [0, kHotS * kHotRep) (the index entry names the first, a lane adds lane % kHotRep), then
// tier A, then tier B while rows are left below `limit`. Returns the number of replicated rows (0 or kHotS * kHotRep).
template <int kThreads>
__device__ __forceinline__ uint32_t preload_hot(const Shared& s, const HotState* __restrict__ hot, uint32_t limit) {
  if (hot == nullptr) return 0u;
  const uint32_t ns = min(hot->n_s, (uint32_t)kHotS);
  const uint32_t rep_rows = ns ? (uint32_t)(kHotS * kHotRep) : 0u;
  // a hot-list base byte is the window's first bucket / 4 | pair kind << 4
  if (threadIdx.x < ns * kHotRep) {
    const uint32_t b = hot->sbase[threadIdx.x / kHotRep];
    s.rowkey[threadIdx.x] = hot->skeys[threadIdx.x / kHotRep];
    s.rowbase[threadIdx.x] = (uint8_t)(min(b & 15u, 12u) | (b & 0x10u));
  }
  if (threadIdx.x < ns) {
    const uint64_t k = hot->skeys[threadIdx.x];
    const uint32_t b = hot->sbase[threadIdx.x];
    const uint32_t h = table_hash_kind(k, b >> 4);
    uint32_t idx = tab_idx1(h);
    bool got = atomicCAS(&s.tab[idx], 0u, kBusy) == 0u;
    if (!got) { idx = tab_idx2(h); got = atomicCAS(&s.tab[idx], 0u, kBusy) == 0u; }
    if (got && k != kEmptyKey) s.tab[idx] = tab_entry(h, min(b & 15u, 12u), threadIdx.x * kHotRep);
  }
  if (threadIdx.x == 0) *s.n_rows = rep_rows;
  __syncthreads();
  const uint32_t na = min(hot->n_a, (uint32_t)kHotA);
  const uint32_t room = limit - min(limit, rep_rows + na);
  const uint32_t nb = min(min(hot->n_b, (uint32_t)(kHotMax - kHotA)), room);
  for (uint32_t i = threadIdx.x; i < na; i += kThreads) {   // tier A before B: the hotter pairs cannot lose their slots
    const uint64_t k = hot->keys[i];
    const uint32_t b = hot->base[i];
    if (k != kEmptyKey) smem_admit(s, k, b >> 4, table_hash_kind(k, b >> 4), min(b & 15u, 12u), limit, false);
  }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < nb; i += kThreads) {
    const uint64_t k = hot->keys[kHotA + i];
    const uint32_t b = hot->base[kHotA + i];
    if (k != kEmptyKey) smem_admit(s, k, b >> 4, table_hash_kind(k, b >> 4), min(b & 15u, 12u), limit, false);
  }
  __syncthreads();
  if (threadIdx.x == 0 && *s.n_rows > limit) *s.n_rows = limit;   // failed claims past the limit
  __syncthreads();
  return rep_rows;
}

// SPEC §8 orders epochs by user time, unsigned: a record is late iff its user time lies below the open window's
// start (lo + off), and in the open window iff wt - lo < len. No division.
__device__ __forceinline__ bool win_late(uint64_t wt, uint64_t lo, uint64_t off, bool past) {
  return past || wt + off < lo + off;
}

// kRecWords = 8: alz_l7_rec (32 B). kRecWords = 4: alz_l7_rec16 (16 B; durations >= 2^32 ns sit in dur_ovf).
// kWin (32-B records only): an event whose write_time lies beyond the open window is not reduced but appended
// to `defer_buf` (it is submitted again when its window opens); one that lies before it is late: reduced into
// the open window and counted.
template <int kWarps, int kRecWords, bool kWin>
__global__ void __launch_bounds__(kWarps * 32, 1)
ingest_pairs_v8_kernel(const uint32_t* __restrict__ recs, uint64_t n, PairTable pairs, Counters* ctr,
                       const HotState* __restrict__ hot, const EpEntry* __restrict__ ep, uint32_t ep_mask,
                       const uint32_t* __restrict__ bloom_g, const uint64_t* __restrict__ dur_ovf,
                       const WinClock* __restrict__ win, uint4* __restrict__ defer_buf, uint32_t defer_cap,
                       uint32_t* __restrict__ cursor) {
  using L = Layout<kWarps, kRecWords>;
  constexpr uint32_t kRows = L::kRows;
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const long long k_entry = PROF_NOW();
  (void)k_entry;
  TL_DECL;
  TL_ENTRY();
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t lane_lt = (1u << lane) - 1u;
  Shared s;
  s.tab = reinterpret_cast<uint32_t*>(smem_raw + L::kTabOff);
  s.bloom = reinterpret_cast<uint32_t*>(smem_raw + L::kBloomOff);
  s.n_rows = reinterpret_cast<uint32_t*>(smem_raw + L::kMisc);
  s.rowkey = reinterpret_cast<uint64_t*>(smem_raw + L::kRowKeys);
  s.rows = reinterpret_cast<uint32_t*>(smem_raw + L::kRowsOff);
  s.rowbase = smem_raw + L::kBaseOff;
  ColdQueue cold;
  SlowQueue slow;
  cold.bind(smem_raw + L::kColdOff + (size_t)warp * kColdQ * kQBytes);
  slow.bind(smem_raw + L::kSlowOff + (size_t)warp * kSlowQ * kQBytes);
  uint4* probe = reinterpret_cast<uint4*>(smem_raw + L::kProbeOff + (size_t)warp * 512u);
  const uint32_t probe_a = smem_u32(probe);
  // where the reductions of a lane whose event is not a hit go (they add 0): the hot tier's reductions are issued
  // by all lanes with selected operands instead of sitting in divergent regions
  uint32_t* const idle = reinterpret_cast<uint32_t*>(smem_raw + L::kScratchOff + (size_t)warp * 128u) + lane;
  const uint8_t* ring = smem_raw + (size_t)warp * 2u * L::kChunkBytes;
  const uint32_t ring_a = smem_u32(ring);
  const uint32_t bar_a = smem_u32(smem_raw + L::kBars + warp * 16u);

  // a chunk = 64 consecutive records; all but possibly the last chunk of the array are full. 32-bit chunk numbers:
  // n < 2^37 events per launch (the ABI layer splits above).
  const uint32_t n_chunks = (uint32_t)((n + kChunk - 1u) / kChunk);
  const uint32_t tail = (uint32_t)(n - (uint64_t)(n_chunks - 1u) * kChunk);   // events in the last chunk, 1..kChunk
  uint64_t policy;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(policy));
  ChunkSched<kWarps> sched;
  sched.init(cursor, n_chunks, warp, gridDim.x * kWarps, lane);
  // `dep` is always 0 but computed from the words just loaded out of the stage (see the main loop): the copy cannot
  // be issued before those loads have returned
  auto issue = [&](uint32_t stage, uint32_t c_req, uint32_t dep) {   // one lane; requests chunk c_req if there is one
    if (c_req < n_chunks) {
      const uint32_t bytes = (c_req == n_chunks - 1u ? tail : kChunk) * (uint32_t)kRecWords * 4u + dep;
      mbar_expect_tx(bar_a + stage * 8u, bytes);
      tma_load(ring_a + stage * L::kChunkBytes, recs + (uint64_t)c_req * (kChunk * kRecWords), bytes,
               bar_a + stage * 8u, policy);
    }
  };
  // the first two chunks are requested before the table is even built
  const uint32_t c_first = sched.next(lane);
  uint32_t c_ahead = sched.next(lane);          // chunk of the next iteration (requested)
  if (lane == 0) {
    mbar_init(bar_a, 1u);
    mbar_init(bar_a + 8u, 1u);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    issue(0u, c_first, 0u);
    issue(1u, c_ahead, 0u);
  }

  for (uint32_t i = threadIdx.x; i < kTab; i += kWarps * 32) s.tab[i] = 0u;
  for (uint32_t i = threadIdx.x; i < ALZ_BLOOM_WORDS; i += kWarps * 32) s.bloom[i] = bloom_g ? bloom_g[i] : 0xFFFFFFFFu;
  for (uint32_t i = threadIdx.x; i <= kRows; i += kWarps * 32) { s.rowkey[i] = kEmptyKey; s.rowbase[i] = 0; }
  for (uint32_t i = threadIdx.x; i < (kRows + 1u) * kRowWords; i += kWarps * 32) s.rows[i] = 0u;
  if (threadIdx.x == 0) *s.n_rows = 0u;
  __syncthreads();
  const uint32_t rep_rows = preload_hot<kWarps * 32>(s, hot, L::kPreload);
  __syncthreads();

  const uint32_t zero = (uint32_t)(n >> 63);   // n < 2^37
  uint32_t lost = 0, unresolved = 0, n_hit = 0, n_live = 0, n_cold = 0, n_late = 0;
  uint32_t probing = 0;                        // events at the head of the cold queue whose probes are in flight
  uint64_t win_lo = 0, win_len = ~0ull, win_off = 0;
  bool win_past = false;
  if (kWin) { win_lo = win->lo; win_len = win->len; win_off = win->off; win_past = win->ready > 1ull; }
  PROF_DECL;
  unsigned long long t_wait = 0, t_slow = 0;
  const long long p_begin = PROF_NOW();
  (void)p_begin;
  uint32_t it = 0;
  uint32_t c_req = 0;                           // chunk two iterations ahead, requested in this iteration
  for (uint32_t c = c_first; c < n_chunks; c = c_ahead, c_ahead = c_req, ++it) {
    const uint32_t stage = it & 1u;
    pc0 = PROF_NOW();
    mbar_wait(bar_a + stage * 8u, (it >> 1) & 1u);
    pc1 = PROF_NOW();
    PROF_ADD(1, pc1 - pc0);
    PROF_ADD(6, 1);
    // records of this chunk into registers (lane l takes records l and l + 32)
    uint32_t w[kU][8];
    const uint8_t* st = ring + stage * L::kChunkBytes;
    uint32_t seen = 0;
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const uint4* p = reinterpret_cast<const uint4*>(st + ((size_t)u * 32u + lane) * (kRecWords * 4u));
      const uint4 a = p[0];
      w[u][0] = a.x; w[u][1] = a.y; w[u][2] = a.z; w[u][3] = a.w;
      seen ^= a.x;
      w[u][4] = w[u][5] = w[u][6] = w[u][7] = 0u;
      if (kRecWords == 8) {
        if (kWin) { const uint4 b = p[1]; w[u][4] = b.x; w[u][5] = b.y; w[u][6] = b.z; w[u][7] = b.w; seen ^= b.x; }
        else { const uint2 b = *reinterpret_cast<const uint2*>(p + 1); w[u][4] = b.x; w[u][5] = b.y; seen ^= b.x; }
      }
    }
    // The stage goes back to the TMA only when the loads above have RETURNED: the byte count of the copy is made
    // to depend on the loaded words (`zero` is a run-time 0 the compiler cannot see through), so the copy's issue
    // waits on their scoreboard. A __syncwarp() alone orders the instructions, not the completion of the
    // shared-memory loads, and under load the TMA write of the next chunk overtook the duration loads of this one
    // (right keys with the wrong latencies).
    __syncwarp();
    c_req = sched.next(lane);
    if (elect_one()) issue(stage, c_req, seen & zero);
    uint32_t n_here = (c == n_chunks - 1u) ? tail : kChunk;

    bool live[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      live[u] = (uint32_t)u * 32u + lane < n_here;
      if constexpr (kWin && kRecWords == 8) {
        const uint64_t wt = ((uint64_t)w[u][7] << 32) | w[u][6];
        const bool late = live[u] && win_late(wt, win_lo, win_off, win_past);      // before the open window
        const bool future = live[u] && !late && wt - win_lo >= win_len;
        n_late += late ? 1u : 0u;
        const uint32_t fm = __ballot_sync(0xFFFFFFFFu, future);
        if (fm != 0u) {   // warp-uniform and rare: only around a window boundary
          uint32_t at = 0;
          if (lane == (uint32_t)__ffs((int)fm) - 1u) at = atomicAdd(&ctr->defer_count, (uint32_t)__popc(fm));
          at = __shfl_sync(0xFFFFFFFFu, at, __ffs((int)fm) - 1) + __popc(fm & lane_lt);
          if (future) {
            if (at < defer_cap) {
              defer_buf[2u * at] = make_uint4(w[u][0], w[u][1], w[u][2], w[u][3]);
              defer_buf[2u * at + 1u] = make_uint4(w[u][4], w[u][5], w[u][6], w[u][7]);
            } else ++lost;
            live[u] = false;          // not this window's event
          }
          n_live -= (uint32_t)__popc(fm);   // handed on: not this launch's events (see not_request below)
        }
      }
    }
    n_live += n_here;

    // hot tier for both events of the lane, then one pass over the cold queue. The two events go through the tier
    // phase by phase (decode + index bucket, row key, reductions) rather than one after the other: a phase's loads
    // of both events are in flight together, and the divergent regions (the reductions) come last
    uint64_t key[kU], dur[kU];
    uint32_t dlo[kU], meta[kU], cell[kU], rowi[kU];
    bool coldf[kU], act[kU], cand[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const uint32_t mw = (kRecWords == 8) ? w[u][3] : w[u][2];   // status | protocol << 16 | method_flags << 24
      uint32_t p = __byte_perm(mw, 0u, 0x4442u);                  // protocol byte, flag bits still on
      if (kRecWords == 8) dur[u] = ((uint64_t)w[u][5] << 32) | w[u][4];
      else {
        dur[u] = w[u][3];
        if (p & ALZ_REC16_DUR_OVERFLOW) dur[u] = live[u] ? __ldg(&dur_ovf[w[u][3]]) : 0ull;
      }
      const bool hk = (p & ALZ_PROTO_F_HOSTKEY) != 0u;             // daddr is a Host-header id: own key space, cold tier
      // bit 7 is ALZ_REC16_DUR_OVERFLOW on packed records; on 32-B records it is no flag, and a byte with it set is
      // no protocol (class 0 below, as for any value > 8)
      p &= (kRecWords == 8) ? 0xBFu : 0x3Fu;
      const uint32_t cls = shr_clamp(kProtoLut, 3u * p);
      // a row is built unless the class says "payload parser decides" and the parser said no (bit 30 of mw)
      act[u] = live[u] && (cls & 1u) && !((cls & 2u) && (mw & ((uint32_t)ALZ_MF_PAYLOAD_REJECT << 24)));
      const bool rv = (cls & 4u) && (mw & ((uint32_t)ALZ_MF_METHOD_MASK << 24)) == (2u << 24);   // DELIVER / PUSHED_EVENT
      const bool err = p == ALZ_PROTO_HTTP && ((mw & 0xFFFFu) - 500u) < 100u;
      key[u] = ((uint64_t)w[u][1] << 32) | w[u][0];               // make_pair_key: the record's first two words as they lie
      const uint32_t bucket = latency_bucket_rz(dur[u]);
      const uint32_t kind = hk ? kPairHost : rv ? kPairRev : kPairFwd;
      dlo[u] = (uint32_t)dur[u];
      meta[u] = bucket | (kind << 6) | (err ? 0x100u : 0u) | ((uint32_t)(dur[u] >> 32) << 9);

      // per-CTA table: the key's bucket of two index entries, the matching one names the row and its histogram window
      const uint32_t h = table_hash(key[u]) ^ (rv ? kRevSalt : 0u);   // table_hash_kind; host-keyed: never a candidate
      const uint32_t fp = tab_fp(h);
      const uint2 t2 = *reinterpret_cast<const uint2*>(&s.tab[tab_idx1(h)]);
      const uint32_t x1 = t2.x ^ fp, x2 = t2.y ^ fp;
      const uint32_t x = x1 < 0x10000u ? x1 : x2;                    // upper 16 bits 0: the fingerprint matched
      rowi[u] = min(x & kRowMask, kRows);
      rowi[u] += rowi[u] < rep_rows ? (lane & (uint32_t)(kHotRep - 1)) : 0u;   // tier S: this lane's row of the group
      cell[u] = bucket - ((x >> 12) & 15u) * 4u;                     // cell of this latency in the row's window
      cand[u] = act[u] && !hk && x < 0x10000u && (x & kRowMask) < kRows && cell[u] < 16u;
    }
    bool hit[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) hit[u] = cand[u] && s.rowkey[rowi[u]] == key[u];   // row kRows holds no key
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const bool ht = hit[u];
      uint32_t* row = s.rows + rowi[u] * kRowWords;
      const uint32_t d = cell[u];
      const uint32_t dhi = (uint32_t)(dur[u] >> 32);
      const uint32_t sh = (d & 1u) * 16u;
      uint32_t* cellp = ht ? row + (d >> 1) : idle;
      const uint32_t old = atomicAdd(cellp, ht ? (1u << sh) : 0u);
      const bool spill = ht && ((old >> sh) & 0xFFFFu) == kCellSpill;
      if (__any_sync(0xFFFFFFFFu, spill)) {
        if (spill) {
          // this lane took the cell to 0x8000: move 0x8000 counts into the global table (rare: a pair with more
          // than 32767 events in one bucket within one launch of one CTA)
          const uint32_t grow = find_or_insert_pair(pairs, key[u], (meta[u] >> 6) & 3u, ep, ep_mask);
          if (grow < kDropRow) red_add_u32(pair_cell(pairs, grow, meta[u] & 0x3Fu), 0x8000u);
          else if (grow == kDropRow) unresolved += 0x8000u; else lost += 0x8000u;
          atomicSub(cellp, 0x8000u << sh);
        }
        __syncwarp();
      }
      uint32_t* latp = ht ? row + 9u + 2u * (lane & 1u) : idle;
      const uint32_t oldl = atomicAdd(latp, ht ? dlo[u] : 0u);
      const bool carry = ht && oldl > ~dlo[u];                           // out of the low word
      const bool more = ht && (carry || dhi != 0u);
      if (__any_sync(0xFFFFFFFFu, more)) {
        if (more) atomicAdd(latp + 1, dhi + (carry ? 1u : 0u));
      }
      if (ht && (meta[u] & 0x100u)) atomicAdd(&row[8], 1u);
      n_hit += ht ? 1u : 0u;
      coldf[u] = act[u] && !hit[u];
      // a duration that does not fit the queue entry (>= 2^55 ns) is handled on the spot: rare beyond words
      if (coldf[u] && dhi >= (1u << 23)) {
        ++n_cold;                    // per-lane here, folded into the warp total below
        slow_one<kRows>(key[u], dur[u], meta[u] & 0x3Fu, (meta[u] >> 6) & 3u, (meta[u] & 0x100u) != 0u, pairs, s, ep, ep_mask,
                        &lost, &unresolved);
        coldf[u] = false;
      }
    }
    uint32_t pushed = 0;
#pragma unroll
    for (int u = 0; u < kU; ++u) pushed += cold.push(coldf[u], key[u], dlo[u], meta[u], lane_lt);
    __syncwarp();
    pc0 = PROF_NOW();
    PROF_ADD(5, pc0 - pc1);
    // a batch is consumed when the next one is ready to be requested
    while (cold.count - probing >= 32u) {
      if (probing) {
        cold_consume<kRows>(cold, probing, probe, slow, pairs, s, ep, ep_mask, lane_lt, &lost, &unresolved, &t_wait, &t_slow);
        probing = 0;
        PROF_ADD(7, 1);
      }
      cold_issue(cold, 32u, pairs, s, probe, probe_a);
      probing = 32u;
    }
    PROF_ADD(3, PROF_NOW() - pc0);
    // cold pushes are warp totals: keep them in lane 0's counter only
    if (lane == 0) n_cold += pushed;
  }
  if (probing) cold_consume<kRows>(cold, probing, probe, slow, pairs, s, ep, ep_mask, lane_lt, &lost, &unresolved, &t_wait, &t_slow);
  if (cold.count) {
    const uint32_t rest = cold.count;
    cold_issue(cold, rest, pairs, s, probe, probe_a);
    cold_consume<kRows>(cold, rest, probe, slow, pairs, s, ep, ep_mask, lane_lt, &lost, &unresolved, &t_wait, &t_slow);
  }
  while (slow.count) slow_batch<kRows>(slow, min(slow.count, 32u), pairs, s, ep, ep_mask, &lost, &unresolved);
  PROF_ADD(0, PROF_NOW() - p_begin);
  PROF_ADD(2, t_wait);
  PROF_ADD(4, t_slow);
  PROF_FLUSH();
  TL_CHUNKS(it);
  __syncthreads();
  const long long k_loop_end = PROF_NOW();
  (void)k_loop_end;
  TL_LOOP_END();

  drain_rows_and_count<kWarps, kRows, kWin>(s, pairs, ctr, ep, ep_mask, lost, unresolved, n_hit, n_live, n_cold, n_late);
  PROF_PHASE(0, p_begin - k_entry);
  PROF_PHASE(1, k_loop_end - p_begin);
  PROF_PHASE(2, PROF_NOW() - k_loop_end);
  PROF_PHASE(3, 1);
  TL_EXIT();
}

// open the first window on the first record ever submitted: epoch = (write_time + off) / len, docs/SPEC.md §8
// (off = FirstUserspaceTime - FirstKernelTime, aggregator/data.go:1740-1743)
__global__ void win_init_kernel(const uint32_t* __restrict__ recs, uint64_t n, WinClock* win) {
  if (threadIdx.x != 0 || blockIdx.x != 0 || n == 0 || win->ready) return;
  const uint64_t wt = ((uint64_t)recs[7] << 32) | recs[6];
  const uint64_t e = (wt + win->off) / win->len;
  win->lo = e * win->len - win->off;
  win->epoch = e;
  win->ready = 1ull;
}
__global__ void win_advance_kernel(WinClock* win) {
  if (threadIdx.x != 0 || blockIdx.x != 0 || !win->ready) return;
  const uint64_t start = win->lo + win->off;                  // user time where the closed epoch began
  if (start + win->len < start) win->ready = 2ull;            // the next one would begin at 2^64 or later
  win->lo += win->len;
  win->epoch += 1ull;
}

// At a table commit: the set-aside records [lo, hi) are resolved under the tables they arrived under, before the
// patch. A record that makes a row gets its edge key in place of saddr | daddr (kEmptyKey: its source is not a pod,
// which no real edge key equals: the type-3 end is never reversed). A record that makes no row keeps its words.
__global__ void __launch_bounds__(256) defer_resolve_kernel(alz_l7_rec* buf, uint32_t lo, uint32_t hi, const EpEntry* __restrict__ ep,
                                                            uint32_t ep_mask, Counters* ctr) {
  if (blockIdx.x == 0 && threadIdx.x == 0) ctr->defer_resolved = hi;   // nothing reads it while this kernel runs
  for (uint32_t i = lo + blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += gridDim.x * blockDim.x) {
    Rec r;
    for (int k = 0; k < 8; ++k) r.w[k] = reinterpret_cast<const uint32_t*>(buf + i)[k];
    const uint32_t proto = rec_protocol(r), mf = rec_mflags(r);
    if (!emits_request_row(proto, mf)) continue;
    uint64_t ekey = kEmptyKey;
    const uint32_t kind = rec_hostkey(r) ? kPairHost : is_reversed(proto, mf) ? kPairRev : kPairFwd;
    if (!resolve_pair(ep, ep_mask, make_pair_key(rec_saddr(r), rec_daddr(r)), kind, &ekey)) ekey = kEmptyKey;
    buf[i].saddr = (uint32_t)ekey;
    buf[i].daddr = (uint32_t)(ekey >> 32);
  }
}

// At a flush, after the clock has advanced: the resolved set-aside records src[0, n) (defer_resolve_kernel). Those
// of the window now open are reduced straight into the edge accumulators, as the eager plan does; those of a later
// window are set aside again into dst, resolution kept, ahead of any raw record (the caller ingests those after).
__global__ void __launch_bounds__(256) defer_roll_kernel(const alz_l7_rec* __restrict__ src, uint32_t n,
                                                         const WinClock* __restrict__ win, alz_l7_rec* __restrict__ dst,
                                                         uint32_t cap, EdgeTable edges, Counters* ctr) {
  const uint64_t lo = win->lo, len = win->len, off = win->off;
  const bool past = win->ready > 1ull;
  uint32_t not_request = 0, unresolved = 0, lost = 0, late = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const Rec r = load_rec(src + i);
    const uint64_t wt = ((uint64_t)r.w[7] << 32) | r.w[6];
    const bool is_late = win_late(wt, lo, off, past);
    if (!is_late && wt - lo >= len) {
      const uint32_t at = atomicAdd(&ctr->defer_count, 1u);
      atomicAdd(&ctr->defer_resolved, 1u);
      if (at < cap) {
        uint4* d = reinterpret_cast<uint4*>(dst + at);
        d[0] = make_uint4(r.w[0], r.w[1], r.w[2], r.w[3]);
        d[1] = make_uint4(r.w[4], r.w[5], r.w[6], r.w[7]);
      } else {
        ++lost;
      }
      continue;
    }
    late += is_late ? 1u : 0u;
    const uint32_t proto = rec_protocol(r);
    if (!emits_request_row(proto, rec_mflags(r))) { ++not_request; continue; }
    const uint64_t ekey = ((uint64_t)r.w[1] << 32) | r.w[0];
    if (ekey == kEmptyKey) { ++unresolved; continue; }
    const uint32_t row = find_or_insert(edges, ekey);
    if (row >= kLostRow) { ++lost; continue; }
    const uint64_t dur = rec_duration(r);
    edge_add(edges, row, latency_bucket(dur), dur, is_5xx(proto, rec_status(r)));
  }
  if (not_request) atomicAdd(&ctr->not_request, (unsigned long long)not_request);
  if (unresolved) atomicAdd(&ctr->src_unresolved, (unsigned long long)unresolved);
  if (lost) atomicAdd(&ctr->capacity_events, (unsigned long long)lost);
  if (late) atomicAdd(&ctr->late_events, (unsigned long long)late);
}

// ---- hot-pair feedback: after a fold, pick the pairs that took the most events -----
// the fold (fold_pairs_kernel, or emit_edges_kernel at a single-rank flush) left row_cnt[row], row_base[row] and a 128-bin (quarter-octave) histogram of the counts of
// the forward rows; thresholds = the lowest bins that keep tier A <= kHotA and A+B <= target. Every block derives
// the same two thresholds from the bins itself (128 adds) instead of a separate launch.
__global__ void __launch_bounds__(256) hot_emit_kernel(PairTable pairs, HotState* hot, uint32_t target_total) {
  __shared__ uint32_t s_thr[3];
  if (threadIdx.x == 0) {
    uint32_t cum = 0, thr_s = 128, thr_a = 128, thr_b = 128;
    for (int b = 127; b >= 0; --b) {
      cum += hot->bins[b];
      if (cum <= (uint32_t)kHotS) thr_s = (uint32_t)b;
      if (cum <= (uint32_t)kHotA) thr_a = (uint32_t)b;
      if (cum <= target_total) thr_b = (uint32_t)b;
    }
    s_thr[0] = thr_a; s_thr[1] = thr_b; s_thr[2] = thr_s;
    if (blockIdx.x == 0) { hot->thr_a = thr_a; hot->thr_b = thr_b; hot->thr_s = thr_s; }
  }
  __syncthreads();
  const uint32_t thr_a = s_thr[0], thr_b = s_thr[1], thr_s = s_thr[2];
  const uint32_t n_rows = min(*pairs.n_rows, pairs.max_rows);
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t row = blockIdx.x * blockDim.x + threadIdx.x; row < n_rows; row += stride) {
    const uint32_t c = pairs.row_cnt[row];
    const uint32_t kind = pairs.row_kind[row];
    if (c == 0u || kind == kPairHost) continue;   // host-keyed pairs do not enter the per-CTA table
    const uint32_t b = count_bin(c);
    const uint8_t base = (uint8_t)(pairs.row_base[row] | (kind << 4));   // window base | kind, see preload_hot
    if (b >= thr_s) {
      const uint32_t p = atomicAdd(&hot->n_s, 1u);
      if (p < (uint32_t)kHotS) { hot->skeys[p] = pairs.row_key[row]; hot->sbase[p] = base; }
    } else if (b >= thr_a) {
      const uint32_t p = atomicAdd(&hot->n_a, 1u);
      if (p < (uint32_t)kHotA) { hot->keys[p] = pairs.row_key[row]; hot->base[p] = base; }
    } else if (b >= thr_b) {
      const uint32_t p = atomicAdd(&hot->n_b, 1u);
      if (p < (uint32_t)(kHotMax - kHotA)) { hot->keys[kHotA + p] = pairs.row_key[row]; hot->base[kHotA + p] = base; }
    }
  }
}

template <int kWarps, int kRecWords, bool kWin = false>
void launch_variant(const void* recs, uint64_t n, const PairTable& pairs, Counters* ctr, const HotState* hot,
                    const EpEntry* ep, uint32_t ep_mask, const uint32_t* bloom, const uint64_t* dur_ovf, int sms,
                    uint32_t* cursor, cudaStream_t s, const WinClock* win = nullptr, void* defer_buf = nullptr,
                    uint32_t defer_cap = 0) {
  using L = Layout<kWarps, kRecWords>;
  static_assert(kWarps <= kMaxWarps, "one cursor per warp slot");
  cudaMemsetAsync(cursor, 0, kWarps * kCursorStride * sizeof(uint32_t), s);   // every launch's claims start over
  // per device (a process may drive several GPUs), so not cached in a static
  cudaFuncSetAttribute(ingest_pairs_v8_kernel<kWarps, kRecWords, kWin>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                       (int)L::kBytes);
  ingest_pairs_v8_kernel<kWarps, kRecWords, kWin><<<(unsigned)sms, kWarps * 32, L::kBytes, s>>>(
      (const uint32_t*)recs, n, pairs, ctr, hot, ep, ep_mask, bloom, dur_ovf, win, (uint4*)defer_buf, defer_cap, cursor);
}

}  // namespace

uint32_t ingest_table_rows() { return Layout<kDefaultWarps, 8>::kRows; }
size_t ingest_cursor_bytes() { return (size_t)kMaxWarps * kCursorStride * sizeof(uint32_t); }

void launch_ingest_pairs(const alz_l7_rec* recs, uint64_t n, const PairTable& pairs, Counters* ctr,
                         const HotState* hot, const EpEntry* ep, uint32_t ep_mask, const uint32_t* bloom,
                         uint32_t* cursor, int sms, cudaStream_t s) {
  if (n == 0) return;
  launch_variant<kDefaultWarps, 8>(recs, n, pairs, ctr, hot, ep, ep_mask, bloom, nullptr, sms, cursor, s);
}

void launch_ingest_pairs_rec16(const alz_l7_rec16* recs, uint64_t n, const uint64_t* dur_ovf, const PairTable& pairs,
                               Counters* ctr, const HotState* hot, const EpEntry* ep, uint32_t ep_mask,
                               const uint32_t* bloom, uint32_t* cursor, int sms, cudaStream_t s) {
  if (n == 0) return;
  launch_variant<kDefaultWarps, 4>(recs, n, pairs, ctr, hot, ep, ep_mask, bloom, dur_ovf, sms, cursor, s);
}

// time-cut windows: `win` = device WinClock {lo, len, ready}; records beyond the open window land in defer_buf
void launch_ingest_pairs_windowed(const alz_l7_rec* recs, uint64_t n, const PairTable& pairs, Counters* ctr,
                                  const HotState* hot, const EpEntry* ep, uint32_t ep_mask, const uint32_t* bloom,
                                  uint64_t* win, alz_l7_rec* defer_buf, uint32_t defer_cap, uint32_t* cursor, int sms,
                                  cudaStream_t s) {
  if (n == 0) return;
  win_init_kernel<<<1, 32, 0, s>>>((const uint32_t*)recs, n, (WinClock*)win);
  launch_variant<kDefaultWarps, 8, true>(recs, n, pairs, ctr, hot, ep, ep_mask, bloom, nullptr, sms, cursor, s,
                                         (const WinClock*)win, defer_buf, defer_cap);
}
void launch_window_advance(uint64_t* win, cudaStream_t s) { win_advance_kernel<<<1, 32, 0, s>>>((WinClock*)win); }
void launch_defer_resolve(alz_l7_rec* buf, uint32_t lo, uint32_t hi, const EpEntry* ep, uint32_t ep_mask, Counters* ctr,
                          int sms, cudaStream_t s) {
  const uint32_t grid = std::min<uint32_t>((uint32_t)sms * 4u, std::max<uint32_t>(1u, (hi - lo + 255u) / 256u));
  defer_resolve_kernel<<<grid, 256, 0, s>>>(buf, lo, hi, ep, ep_mask, ctr);
}
void launch_defer_roll(const alz_l7_rec* src, uint32_t n, const uint64_t* win, alz_l7_rec* dst, uint32_t cap,
                       const EdgeTable& edges, Counters* ctr, int sms, cudaStream_t s) {
  const uint32_t grid = std::min<uint32_t>((uint32_t)sms * 4u, std::max<uint32_t>(1u, (n + 255u) / 256u));
  defer_roll_kernel<<<grid, 256, 0, s>>>(src, n, (const WinClock*)win, dst, cap, edges, ctr);
}

// after fold_pairs_kernel / emit_edges_kernel filled hot->bins: choose next window's hot list
void launch_hot_select(const PairTable& pairs, HotState* hot, int sms, cudaStream_t s) {
  hot_emit_kernel<<<(unsigned)sms * 2, 256, 0, s>>>(pairs, hot, Layout<kDefaultWarps, 8>::kPreload);
}

}  // namespace alz

// profiling build only: cycles per section of the ingest main loop since the last call (see g_ingest_prof)
// profiling build only: the per-CTA timeline (see g_ingest_tl) into out[kTlLaunches][kTlCtas][kTlWords], and the
// number of launches recorded since the last call (only the last kTlLaunches are kept); then starts over
extern "C" int alz_debug_ingest_timeline(unsigned long long* out, unsigned int* n_launches, unsigned int* dims) {
#ifdef ALZ_INGEST_PROF
  dims[0] = alz::kTlLaunches; dims[1] = alz::kTlCtas; dims[2] = alz::kTlWords;
  if (out == nullptr) return ALZ_OK;   // sizes only
  if (cudaDeviceSynchronize() != cudaSuccess) return ALZ_E_CUDA;
  if (cudaMemcpyFromSymbol(out, alz::g_ingest_tl, sizeof(alz::g_ingest_tl)) != cudaSuccess) return ALZ_E_CUDA;
  if (cudaMemcpyFromSymbol(n_launches, alz::g_ingest_tl_launch, sizeof(unsigned int)) != cudaSuccess) return ALZ_E_CUDA;
  void* z = nullptr;
  if (cudaGetSymbolAddress(&z, alz::g_ingest_tl) != cudaSuccess || cudaMemset(z, 0, sizeof(alz::g_ingest_tl)) != cudaSuccess)
    return ALZ_E_CUDA;
  const unsigned int zero = 0;
  if (cudaMemcpyToSymbol(alz::g_ingest_tl_launch, &zero, sizeof(zero)) != cudaSuccess) return ALZ_E_CUDA;
  return cudaDeviceSynchronize() == cudaSuccess ? ALZ_OK : ALZ_E_CUDA;
#else
  (void)out; (void)n_launches; (void)dims;
  return ALZ_E_UNSUPPORTED;
#endif
}

extern "C" int alz_debug_ingest_prof(unsigned long long* out12) {   // 8 section counters + 4 phase counters
#ifdef ALZ_INGEST_PROF
  unsigned long long z[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (cudaDeviceSynchronize() != cudaSuccess) return ALZ_E_CUDA;
  if (cudaMemcpyFromSymbol(out12, alz::g_ingest_prof, sizeof(z)) != cudaSuccess) return ALZ_E_CUDA;
  if (cudaMemcpyToSymbol(alz::g_ingest_prof, z, sizeof(z)) != cudaSuccess) return ALZ_E_CUDA;
  if (cudaMemcpyFromSymbol(out12 + 8, alz::g_ingest_phase, 4 * sizeof(unsigned long long)) != cudaSuccess) return ALZ_E_CUDA;
  if (cudaMemcpyToSymbol(alz::g_ingest_phase, z, 4 * sizeof(unsigned long long)) != cudaSuccess) return ALZ_E_CUDA;
  return ALZ_OK;
#else
  (void)out12;
  return ALZ_E_UNSUPPORTED;
#endif
}
