// alz_device.cuh — device-side building blocks of libalazgpu (sm_90a).
//
// Semantics restated from the reference (file:line = getanteon/alaz @ 828b997f):
//   row-emit rule      aggregator/data.go:1364-1383 (processL7 switch), :1252-1255,
//                      :1288-1292, :1328-1332 (payload parse failure => no row)
//   direction reversal aggregator/data.go:1110-1112 (AMQP DELIVER), :1151-1153
//                      (REDIS PUSHED_EVENT); datastore/dto.go:246-251
//   resolve            aggregator/data.go:827-870 (setFromToV2)
// Everything else (edge key, buckets, accumulators) is docs/SPEC.md.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "../../include/alazgpu.h"

namespace alz {

constexpr uint64_t kEmptyKey = ~0ull;   // open-addressing empty marker (u64 tables)
constexpr uint32_t kMaxProbe = 4096;    // linear-probe bound before "capacity"

// ---- endpoint table: the join's build side, one entry per IPv4 ---------------
// (ClusterInfo.PodIPToPodUid + ServiceIPToServiceUid, aggregator/cluster.go:15-16,
// merged: one probe answers "is it a pod" and "is it a service")
struct __align__(16) EpEntry {
  uint32_t ip;
  uint32_t state;  // bit0 occupied, bit1 has pod id, bit2 has service id
  uint32_t pod;
  uint32_t svc;
};
constexpr uint32_t kEpOcc = 1u, kEpPod = 2u, kEpSvc = 4u;

// Filter of the pod addresses (two bits per address out of hash32): the ingest kernel keeps a copy in shared memory
// and drops an event whose source cannot be a pod without touching the dictionary (alz_ingest.cu). The host keeps
// counters per bit so that deletes are exact (alz_api.cu). A cluster far larger than the filter just saturates it.
#define ALZ_BLOOM_WORDS 4096u   /* 128 Kbit */

__host__ __device__ __forceinline__ uint32_t hash32(uint32_t x) {
  x ^= x >> 16; x *= 0x85EBCA6Bu; x ^= x >> 13; x *= 0xC2B2AE35u; x ^= x >> 16;
  return x;
}
__host__ __device__ __forceinline__ uint64_t hash64(uint64_t x) {
  x ^= x >> 33; x *= 0xFF51AFD7ED558CCDull; x ^= x >> 33; x *= 0xC4CEB9FE1A85EC53ull; x ^= x >> 33;
  return x;
}

// rank that owns an event (alz_owner_rank): a function of the source address only
__host__ __device__ __forceinline__ uint32_t owner_rank(uint32_t saddr, uint32_t nranks) {
  if (nranks <= 1u) return 0u;
  return (uint32_t)(((uint64_t)hash32(saddr ^ 0xA1A2B200u) * nranks) >> 32);
}

// Socket-pair key of the pair dictionaries: daddr in the high word, saddr in the low word — the order the two
// words have in a record, so a record's first 8 bytes ARE its key (no shuffling in the per-event path).
__host__ __device__ __forceinline__ uint64_t make_pair_key(uint32_t saddr, uint32_t daddr) { return ((uint64_t)daddr << 32) | saddr; }
__host__ __device__ __forceinline__ uint32_t pair_saddr(uint64_t key) { return (uint32_t)key; }
__host__ __device__ __forceinline__ uint32_t pair_daddr(uint64_t key) { return (uint32_t)(key >> 32); }

// cheap 32-bit hash of a socket pair for the pair dictionaries and the per-CTA table (the per-event
// path pays for this once; hash64 costs two 64-bit multiplies)
__host__ __device__ __forceinline__ uint32_t pair_hash(uint64_t key) {
  uint32_t h = (uint32_t)(key >> 32) * 0x9E3779B1u ^ (uint32_t)key * 0x85EBCA6Bu;
  h ^= h >> 15; h *= 0x2C1B3C6Du; h ^= h >> 13;
  return h;
}

// ---- packed edge key (docs/SPEC.md §3) -----------------------------------------
// One end of every edge is the pod that setFromToV2 resolved from saddr.
//   bit 63      rev: 0 = pod is From, 1 = pod is To (row was reversed)
//   bits 62..61 type of the other end (ALZ_NODE_*)
//   bits 60..32 pod id (< 2^29)
//   bits 31..0  other end: pod/service id, or raw IPv4 for outbound
// Canonical form: a reversed pod<->pod row is stored with rev = 0 and the ends
// swapped, so equal (From,To) always give equal keys.
__host__ __device__ __forceinline__ uint64_t make_edge_key(uint32_t pod_id, uint32_t other_type,
                                                           uint32_t other, bool rev) {
  if (rev && other_type == ALZ_NODE_POD) { uint32_t t = pod_id; pod_id = other; other = t; rev = false; }
  return ((uint64_t)(rev ? 1u : 0u) << 63) | ((uint64_t)other_type << 61) |
         ((uint64_t)(pod_id & 0x1FFFFFFFu) << 32) | (uint64_t)other;
}
__host__ __device__ __forceinline__ void unpack_edge_key(uint64_t k, uint8_t* from_type, uint32_t* from,
                                                         uint8_t* to_type, uint32_t* to) {
  const bool rev = (k >> 63) != 0;
  const uint8_t ot = (uint8_t)((k >> 61) & 3u);
  const uint32_t pod = (uint32_t)((k >> 32) & 0x1FFFFFFFu);
  const uint32_t other = (uint32_t)k;
  if (!rev) { *from_type = ALZ_NODE_POD; *from = pod; *to_type = ot; *to = other; }
  else      { *from_type = ot; *from = other; *to_type = ALZ_NODE_POD; *to = pod; }
}

// node key of an edge end (type, value), docs/SPEC.md §21: the GNN pass's node set (alz_gnn.cu) and the node calls'
// group-by (alz_nodes.cu) both order nodes by it
__device__ __forceinline__ uint64_t node_key(uint32_t kind, uint32_t value) { return ((uint64_t)kind << 32) | value; }

// packed edge key of an output row (inverse of unpack_edge_key)
__device__ __forceinline__ uint64_t row_key_of(const alz_edge_out* r) {
  // rows are 296 bytes apart: 8-byte aligned only
  const uint2 ty = reinterpret_cast<const uint2*>(r)[0];   // from_type, to_type, pad | pad
  const uint2 ft_ = reinterpret_cast<const uint2*>(r)[1];  // from | to
  const uint32_t ft = ty.x & 0xFFu, tt = (ty.x >> 8) & 0xFFu;
  if (ft == ALZ_NODE_POD) return ((uint64_t)tt << 61) | ((uint64_t)(ft_.x & 0x1FFFFFFFu) << 32) | ft_.y;
  return (1ull << 63) | ((uint64_t)ft << 61) | ((uint64_t)(ft_.y & 0x1FFFFFFFu) << 32) | ft_.x;
}
// packed edge key of a caller's edge (the inverse of unpack_edge_key, what row_key_of gives for the row a flush
// emitted with these ends); false for ends no flush emits: a type above ALZ_NODE_OUTBOUND_HOST, no pod end, or a pod
// or service id >= 2^29. A pod <-> pod edge is keyed with its from end as the pod.
inline bool pack_edge_ends(const alz_edge_ends& e, uint64_t* key) {
  const uint32_t ft = e.from_type, tt = e.to_type;
  if (ft > ALZ_NODE_OUTBOUND_HOST || tt > ALZ_NODE_OUTBOUND_HOST) return false;
  auto id_ok = [](uint32_t type, uint32_t v) { return (type != ALZ_NODE_POD && type != ALZ_NODE_SVC) || v < (1u << 29); };
  if (!id_ok(ft, e.from) || !id_ok(tt, e.to)) return false;
  if (ft == ALZ_NODE_POD) { *key = ((uint64_t)tt << 61) | ((uint64_t)e.from << 32) | e.to; return true; }
  if (tt == ALZ_NODE_POD) { *key = (1ull << 63) | ((uint64_t)ft << 61) | ((uint64_t)e.to << 32) | e.from; return true; }
  return false;
}
// the fixed part of an output row and the lane's 8 histogram cells (hist sits at byte 40 of a 296-byte row:
// 8-byte aligned only)
__device__ __forceinline__ void store_edge_out(alz_edge_out* o, uint32_t sl, uint64_t key, const uint32_t (&c)[8],
                                               uint64_t count, uint64_t err5xx, uint64_t lat_sum) {
  uint2* d2 = reinterpret_cast<uint2*>(&o->hist[sl * 8u]);
  d2[0] = make_uint2(c[0], c[1]); d2[1] = make_uint2(c[2], c[3]);
  d2[2] = make_uint2(c[4], c[5]); d2[3] = make_uint2(c[6], c[7]);
  if (sl == 0) {
    uint8_t ft, tt; uint32_t f, t;
    unpack_edge_key(key, &ft, &f, &tt, &t);
    o->from_type = ft; o->to_type = tt;
    for (int k = 0; k < 6; ++k) o->_pad[k] = 0;
    o->from = f; o->to = t;
    o->count = count;
    o->err5xx = err5xx;
    o->lat_sum_ns = lat_sum;
  }
}

// the lane's part of an output row, the layout edge_row_load gives an edge-table row: 8 histogram cells, and in lane 0
// the row's count, latency and 5xx sums (0 in the other lanes)
__device__ __forceinline__ void load_edge_out(const alz_edge_out* r, uint32_t sl, uint32_t (&c)[8], uint64_t& count,
                                              uint64_t& lat, uint64_t& e5) {
  const uint2* s2 = reinterpret_cast<const uint2*>(&r->hist[sl * 8u]);
  const uint2 a = s2[0], b = s2[1], d = s2[2], e = s2[3];
  c[0] = a.x; c[1] = a.y; c[2] = b.x; c[3] = b.y; c[4] = d.x; c[5] = d.y; c[6] = e.x; c[7] = e.y;
  count = 0; lat = 0; e5 = 0;
  if (sl == 0) { count = r->count; lat = r->lat_sum_ns; e5 = r->err5xx; }
}

// ---- per-record rules ------------------------------------------------------------
// Does processL7 hand a row to PersistRequest for this record (before resolve)?
__host__ __device__ __forceinline__ bool emits_request_row(uint32_t protocol, uint32_t method_flags) {
  switch (protocol) {
    case ALZ_PROTO_HTTP: case ALZ_PROTO_AMQP: case ALZ_PROTO_REDIS:
      return true;
    case ALZ_PROTO_POSTGRES: case ALZ_PROTO_MYSQL: case ALZ_PROTO_MONGO:
      return (method_flags & ALZ_MF_PAYLOAD_REJECT) == 0;
    default:  // HTTP2 (frame pairing), KAFKA (PersistKafkaEvent), UNKNOWN
      return false;
  }
}
__host__ __device__ __forceinline__ bool is_reversed(uint32_t protocol, uint32_t method_flags) {
  const uint32_t m = method_flags & ALZ_MF_METHOD_MASK;
  return (protocol == ALZ_PROTO_AMQP && m == ALZ_AMQP_DELIVER) ||
         (protocol == ALZ_PROTO_REDIS && m == ALZ_REDIS_PUSHED_EVENT);
}
// Protocol is "HTTP" or "HTTPS" (HTTPS = HTTP && tls, data.go:1240-1242)
__host__ __device__ __forceinline__ bool is_5xx(uint32_t protocol, uint32_t status) {
  return protocol == ALZ_PROTO_HTTP && status >= 500u && status < 600u;
}
// docs/SPEC.md §4: two sub-buckets per octave over [2^8, 2^40), clamped
__device__ __forceinline__ uint32_t latency_bucket(uint64_t d) {
  if (d < 256ull) return 0u;
  const uint32_t o = 63u - (uint32_t)__clzll((long long)d);
  if (o >= 40u) return ALZ_NB - 1u;
  return 2u * (o - 8u) + (uint32_t)((d >> (o - 1u)) & 1ull);
}

// ---- open-addressed u64 dictionary -> dense accumulator rows ---------------------------
// The dictionary only maps a key to a row number; rows are handed out densely
// by an atomic counter, so the accumulators of the live keys stay contiguous
// however large the dictionary was sized. v1 indexed the accumulators by
// dictionary slot and nearly every reduction missed L2.
// In the pair table one slot serves both directions of a socket pair: row[kPairFwd] is the row of its forward
// events, row[kPairRev] the row of its reversed ones (AMQP DELIVER, REDIS PUSHED_EVENT), each allocated on first use.
// The edge table and the host-keyed dictionary use row[0] only.
struct __align__(16) DictEnt {
  uint64_t key;     // kEmptyKey = free
  uint32_t row[2];  // kNoRow = none yet, kClaimRow = being allocated, then the row (or kLostRow)
};
constexpr uint32_t kNoRow = 0xFFFFFFFFu;
constexpr uint32_t kLostRow = 0xFFFFFFFEu;  // dictionary or row pool exhausted
constexpr uint32_t kClaimRow = 0xFFFFFFFCu; // pair table: a thread is allocating this row word's row; every row
                                            // word from kClaimRow up names no row

constexpr uint32_t kPairFwd = 0u, kPairRev = 1u, kPairHost = 2u, kPairKinds = 3u;

// Claimed-slot log of a table's dictionaries: every CAS that takes a slot from kEmptyKey appends the slot, so a clear
// resets the slots a window used instead of the whole capacity (dict_clear_kernel, alz_kernels.cu). A table with two
// dictionaries logs the second one's slots after the first one's (index dict_mask + 1 + slot). A log that overflowed
// (n[0] > cap) makes the clear take the whole capacity. n[1] counts the clear's finished blocks.
struct SlotLog {
  uint32_t* slot;   // [cap]
  uint32_t* n;      // [2]: slots claimed since the last clear (counted past cap), blocks done
  uint32_t cap;
};
__device__ __forceinline__ void log_claim(const SlotLog& l, uint32_t idx) {
  const uint32_t i = atomicAdd(l.n, 1u);
  if (i < l.cap) l.slot[i] = idx;
}

// The pair table: socket pairs -> rows of the sectored layout below. One dictionary slot serves both directions of
// a pair (kPairFwd, kPairRev); the host-keyed outbound events (kind kPairHost: the key's high word is a Host-header
// id, not a daddr; ALZ_PROTO_F_HOSTKEY) have a dictionary of their own, a key space of its own. Both dictionaries
// hand out rows of the same pool; row_kind[row] says which kind a row is.
struct PairTable {
  DictEnt* dict;      // [dict_mask + 1] socket pairs, forward and reversed rows in one slot
  uint32_t dict_mask;
  DictEnt* dict_host; // [dict_host_mask + 1] host-keyed outbound pairs
  uint32_t dict_host_mask;
  __device__ __forceinline__ DictEnt* dict_of(uint32_t kind) const { return kind == kPairHost ? dict_host : dict; }
  __device__ __forceinline__ uint32_t mask_of(uint32_t kind) const { return kind == kPairHost ? dict_host_mask : dict_mask; }
  uint32_t max_rows;  // rows [0, max_rows) are allocatable; rows max_rows + kind are the sentinel rows of the key that
                      // equals the free marker (one per kind); every per-row array has max_rows + kPairKinds entries
  uint32_t* n_rows;   // device counter of allocated rows
  uint64_t* row_key;  // [max_rows + 3]
  uint8_t* row_kind;  // [max_rows + 3] kPairFwd / kPairRev / kPairHost
  uint32_t* row_cnt;  // [max_rows + 3] events of the row at the last fold, saturated
  uint8_t* row_base;  // [max_rows + 3] first bucket / 4 of the 16-bucket window that held most of the row's events at
                      // the last fold (the per-CTA table keeps only such a window per pair)
  uint32_t* row_aux;  // [max_rows + 3] edge row found by fold_resolve_kernel
  // Rows are kept in 32-byte SECTORS, 16 per row (512 B): sector g = { cells 4g, 4g+1 | cells 4g+2, 4g+3 |
  // latency partial u64 | 5xx partial u64 }. A global reduction costs the SM one LSU pass per distinct sector an
  // instruction touches, not per lane (scripts/micro/red_merge.cu: a histogram increment and a latency add as
  // two instructions = 93 G events/s chip-wide whether or not they share a sector; as ONE red.u64 instruction with two
  // lanes on the same sector = 172 G/s, the price of a single reduction, 188 G/s). So an event's cell and latency live
  // in one sector and are added by a lane pair of one instruction; a row's latency / 5xx totals are the sums of its 16
  // partials (take_pair_row, alz_kernels.cu). A cell pair is added to as a u64: cells are u32 and a fold runs before any cell
  // could reach 2^31 (alz_api.cu), so nothing carries from the low cell into the high one.
  uint64_t* sect;     // [(max_rows + 3) * kSectPerRow * 4]
  SlotLog log;        // slots of dict, then of dict_host
};
constexpr uint32_t kSectPerRow = 16;
__device__ __forceinline__ uint64_t* pair_sect(const PairTable& t, uint32_t row, uint32_t bucket) {
  return t.sect + ((size_t)row * kSectPerRow + (bucket >> 2)) * 4u;
}
__device__ __forceinline__ uint32_t* pair_cell(const PairTable& t, uint32_t row, uint32_t bucket) {
  return reinterpret_cast<uint32_t*>(pair_sect(t, row, bucket)) + (bucket & 3u);
}

// The edge table: packed edge keys -> dense rows of a window's sums (docs/SPEC.md §3), one dictionary (row[0] only).
struct EdgeTable {
  DictEnt* dict;      // [dict_mask + 1]
  uint32_t dict_mask;
  uint32_t max_rows;  // rows [0, max_rows) are allocatable; row max_rows is the sentinel row of the key that equals
                      // the free marker, which no flush emits; every per-row array has max_rows + 1 entries
  uint32_t* n_rows;   // device counter of allocated rows
  uint64_t* row_key;  // [max_rows + 1]
  uint64_t* count;    // [max_rows + 1]
  uint64_t* lat_sum;  // [max_rows + 1]
  uint64_t* err5xx;   // [max_rows + 1]
  uint32_t* hist;     // [(max_rows + 1) * ALZ_NB]
  SlotLog log;
};

// one event into an edge row
__device__ __forceinline__ void edge_add(const EdgeTable& t, uint32_t row, uint32_t bucket, uint64_t dur, bool err) {
  atomicAdd(&t.hist[(size_t)row * ALZ_NB + bucket], 1u);
  atomicAdd((unsigned long long*)&t.lat_sum[row], (unsigned long long)dur);
  if (err) atomicAdd((unsigned long long*)&t.err5xx[row], 1ull);
  atomicAdd((unsigned long long*)&t.count[row], 1ull);
}
// An edge row taken by an 8-lane group: lane sl (0..7) holds histogram cells 8sl..8sl+7 (two 16-byte accesses),
// lane 0 also the row's count, latency and 5xx sums (0 in the other lanes).
__device__ __forceinline__ void edge_row_load(const EdgeTable& t, uint32_t row, uint32_t sl, uint32_t (&c)[8],
                                              uint64_t& count, uint64_t& lat, uint64_t& e5) {
  const uint4* cells = reinterpret_cast<const uint4*>(t.hist + (size_t)row * ALZ_NB + sl * 8u);
  const uint4 a = cells[0], b = cells[1];
  c[0] = a.x; c[1] = a.y; c[2] = a.z; c[3] = a.w; c[4] = b.x; c[5] = b.y; c[6] = b.z; c[7] = b.w;
  count = 0; lat = 0; e5 = 0;
  if (sl == 0) { count = t.count[row]; lat = t.lat_sum[row]; e5 = t.err5xx[row]; }
}
__device__ __forceinline__ void edge_row_zero(const EdgeTable& t, uint32_t row, uint32_t sl) {
  uint4* cells = reinterpret_cast<uint4*>(t.hist + (size_t)row * ALZ_NB + sl * 8u);
  cells[0] = make_uint4(0u, 0u, 0u, 0u);
  cells[1] = make_uint4(0u, 0u, 0u, 0u);
  if (sl == 0) { t.count[row] = 0ull; t.lat_sum[row] = 0ull; t.err5xx[row] = 0ull; }
}
// all keys out of the dictionary and the row allocator back to zero, in stream order (whoever took the rows zeroed
// them); one dict_clear_kernel launch (alz_kernels.cu)
cudaError_t edge_table_clear(const EdgeTable& t, int sms, cudaStream_t s);

// row of `key`, inserting it if absent; >= kLostRow when capacity is exhausted
__device__ __forceinline__ uint32_t find_or_insert(const EdgeTable& t, uint64_t key) {
  if (key == kEmptyKey) return t.max_rows;  // the one key that collides with the free marker
  uint32_t slot = (uint32_t)hash64(key) & t.dict_mask;
#pragma unroll 1
  for (uint32_t p = 0; p < kMaxProbe; ++p) {
    const uint4 e = __ldcg(reinterpret_cast<const uint4*>(&t.dict[slot]));
    uint64_t k = ((uint64_t)e.y << 32) | e.x;
    uint32_t row = e.z;
    if (k == kEmptyKey) {
      const uint64_t old = atomicCAS((unsigned long long*)&t.dict[slot].key, (unsigned long long)kEmptyKey,
                                     (unsigned long long)key);
      if (old == kEmptyKey) {
        log_claim(t.log, slot);
        row = atomicAdd(t.n_rows, 1u);
        if (row >= t.max_rows) row = kLostRow; else t.row_key[row] = key;
        *reinterpret_cast<volatile uint32_t*>(&t.dict[slot].row[0]) = row;
        return row;
      }
      k = old;
      row = kNoRow;
    }
    if (k == key) {
      while (row == kNoRow) row = *reinterpret_cast<volatile uint32_t*>(&t.dict[slot].row[0]);
      return row;
    }
    slot = (slot + 1u) & t.dict_mask;
  }
  return kLostRow;
}

// probe the endpoint table; returns state bits (0 = absent) and ids
__device__ __forceinline__ uint32_t ep_lookup(const EpEntry* __restrict__ tab, uint32_t mask, uint32_t ip,
                                              uint32_t* pod, uint32_t* svc) {
  uint32_t slot = hash32(ip) & mask;
  for (;;) {
    const uint4 e = __ldg(reinterpret_cast<const uint4*>(&tab[slot]));
    if ((e.y & kEpOcc) == 0u) return 0u;
    if (e.x == ip) { *pod = e.z; *svc = e.w; return e.y; }
    slot = (slot + 1u) & mask;
  }
}

// Pair-dictionary insert with the drop rule applied at admission: a NEW socket pair is only
// inserted if its source address is a pod right now (setFromToV2's first test, data.go:829-832).
// Unresolvable traffic is often high-cardinality (every event a new pair); letting it into the
// dictionary cost a CAS, a row and two DRAM-missing reductions per event.
// Existing rows are found without touching the endpoint table. Returns kDropRow for a rejected pair.
// A forward and a reversed event of one socket pair share the slot; each kind's row is allocated the first time an
// event of that kind comes, by the thread whose CAS takes that row word from kNoRow to kClaimRow.
constexpr uint32_t kDropRow = 0xFFFFFFFDu;
__device__ __forceinline__ uint32_t find_or_insert_pair(const PairTable& t, uint64_t key, uint32_t kind,
                                                        const EpEntry* __restrict__ ep, uint32_t ep_mask) {
  // the one key that collides with the free marker has a fixed row per kind
  if (key == kEmptyKey) return t.max_rows + kind;
  DictEnt* const dict = t.dict_of(kind);
  const uint32_t mask = t.mask_of(kind);
  const uint32_t w = kind == kPairRev ? 1u : 0u;   // the slot's row word of this kind
  uint32_t slot = pair_hash(key) & mask;
  bool checked = false;
  auto is_pod = [&]() {
    if (!checked) {
      uint32_t pod, svc;
      if ((ep_lookup(ep, ep_mask, pair_saddr(key), &pod, &svc) & kEpPod) == 0u) return false;
      checked = true;
    }
    return true;
  };
#pragma unroll 1
  for (uint32_t p = 0; p < kMaxProbe; ++p) {
    const uint4 e = __ldcg(reinterpret_cast<const uint4*>(&dict[slot]));
    uint64_t k = ((uint64_t)e.y << 32) | e.x;
    uint32_t row = w ? e.w : e.z;
    if (k == kEmptyKey) {
      if (!is_pod()) return kDropRow;
      k = atomicCAS((unsigned long long*)&dict[slot].key, (unsigned long long)kEmptyKey, (unsigned long long)key);
      if (k == kEmptyKey) { log_claim(t.log, kind == kPairHost ? t.dict_mask + 1u + slot : slot); k = key; }
      row = *reinterpret_cast<volatile uint32_t*>(&dict[slot].row[w]);
    }
    if (k == key) {
      uint32_t* const rw = &dict[slot].row[w];
#pragma unroll 1
      while (row == kNoRow || row == kClaimRow) {
        if (row == kNoRow) {
          if (!is_pod()) return kDropRow;
          row = atomicCAS(rw, kNoRow, kClaimRow);
          if (row == kNoRow) {
            row = atomicAdd(t.n_rows, 1u);
            if (row >= t.max_rows) row = kLostRow; else { t.row_key[row] = key; t.row_kind[row] = (uint8_t)kind; }
            *reinterpret_cast<volatile uint32_t*>(rw) = row;
            return row;
          }
        } else {
          row = *reinterpret_cast<volatile uint32_t*>(rw);
        }
      }
      return row;
    }
    slot = (slot + 1u) & mask;
  }
  return kLostRow;
}

// setFromToV2 on integers for a socket pair of kind kPairFwd / kPairRev / kPairHost: false = "error finding pod with
// sockets saddr" (drop). A host-keyed pair (ALZ_PROTO_F_HOSTKEY) has its Host-header id where daddr would be: the
// caller has already established that the destination is neither service nor pod, and HTTP rows are never
// reversed; only the drop rule is left (data.go:851-854).
__device__ __forceinline__ bool resolve_pair(const EpEntry* __restrict__ tab, uint32_t mask, uint64_t key, uint32_t kind,
                                             uint64_t* edge_key) {
  uint32_t pod, svc;
  const uint32_t s = ep_lookup(tab, mask, pair_saddr(key), &pod, &svc);
  if ((s & kEpPod) == 0u) return false;                 // data.go:829-832
  const uint32_t from_pod = pod;
  uint32_t ot = ALZ_NODE_OUTBOUND_HOST, ov = pair_daddr(key);
  if (kind != kPairHost) {
    const uint32_t d = ep_lookup(tab, mask, ov, &pod, &svc);
    if (d & kEpSvc) { ot = ALZ_NODE_SVC; ov = svc; }       // :840-843 service first
    else if (d & kEpPod) { ot = ALZ_NODE_POD; ov = pod; }  // :845-849
    else ot = ALZ_NODE_OUTBOUND;                           // :862 raw daddr
  }
  *edge_key = make_edge_key(from_pod, ot, ov, kind == kPairRev);
  return true;
}

// first index of a sorted array whose element is not below k
__device__ __forceinline__ uint32_t lower_bound_u64(const uint64_t* __restrict__ a, uint32_t n, uint64_t k) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (a[mid] < k) lo = mid + 1; else hi = mid; }
  return lo;
}

// 32-byte record, two 128-bit loads (the widest global load on sm_90a), streaming: bypass L1
struct Rec { uint32_t w[8]; };
__device__ __forceinline__ Rec load_rec(const alz_l7_rec* p) {
  Rec r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.w[0]), "=r"(r.w[1]), "=r"(r.w[2]), "=r"(r.w[3]) : "l"(p));
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4+16];"
               : "=r"(r.w[4]), "=r"(r.w[5]), "=r"(r.w[6]), "=r"(r.w[7]) : "l"(p));
  return r;
}
// field accessors of the packed words (layout of alz_l7_rec)
__device__ __forceinline__ uint32_t rec_saddr(const Rec& r) { return r.w[0]; }
__device__ __forceinline__ uint32_t rec_daddr(const Rec& r) { return r.w[1]; }
__device__ __forceinline__ uint32_t rec_status(const Rec& r) { return r.w[3] & 0xFFFFu; }
// without ALZ_PROTO_F_HOSTKEY; bit 7 is no flag of a 32-B record, so a byte with it set stays an undefined protocol
__device__ __forceinline__ uint32_t rec_protocol(const Rec& r) { return (r.w[3] >> 16) & 0xBFu; }
__device__ __forceinline__ bool rec_hostkey(const Rec& r) { return (r.w[3] & ((uint32_t)ALZ_PROTO_F_HOSTKEY << 16)) != 0u; }
__device__ __forceinline__ uint32_t rec_mflags(const Rec& r) { return r.w[3] >> 24; }
__device__ __forceinline__ uint64_t rec_duration(const Rec& r) { return ((uint64_t)r.w[5] << 32) | r.w[4]; }

// ---- hot-pair feedback (alz_ingest.cu): which socket pairs took the most events last fold ----
constexpr int kHotMax = 4096;   // capacity of the list; the ingest kernel preloads as many as its table takes
struct HotState {
  uint32_t bins[128];          // quarter-octave histogram of per-pair event counts (forward pairs)
  uint32_t thr_a, thr_b;       // lowest bin of tier A (hottest, listed first) / of tier B
  uint32_t n_a, n_b;           // tier A occupies keys[0, n_a), tier B keys[kHotA, kHotA + n_b)
  uint64_t keys[kHotMax];
  uint8_t base[kHotMax];       // the pair's histogram window (first bucket / 4), see PairTable::row_base
  // tier S: the (at most) kHotS hottest pairs of all. The per-CTA table gives each of them kHotRep rows and a lane
  // uses row (lane % kHotRep) of the group: when one pair is most of a GPU's traffic — the rank that owns the
  // hottest pair of a sharded stream sees it in every second event — its reductions would otherwise pile up on
  // one shared-memory word and serialise (8 GPUs, config 2: that rank's ingest 2.2 ms against 1.13 ms elsewhere)
  uint32_t thr_s, n_s;
  uint64_t skeys[8];
  uint8_t sbase[8];
};
constexpr int kHotA = 64;
constexpr int kHotS = 8, kHotRep = 8;
// monotone bin of a count >= 1: 4 bins per octave
__device__ __forceinline__ uint32_t count_bin(uint32_t c) {
  const uint32_t o = 31u - (uint32_t)__clz((int)c);
  const uint32_t sub = o >= 2u ? (c >> (o - 2u)) & 3u : (c << (2u - o)) & 3u;
  return o * 4u + sub;
}

// device-side counters (per handle)
struct Counters {
  unsigned long long not_request;
  unsigned long long src_unresolved;
  unsigned long long capacity_events;   // events lost at ingest to an exhausted pair dictionary / row pool
  unsigned long long fold_lost_events;  // events lost at fold to an exhausted edge dictionary / row pool
  uint32_t pair_rows, edge_rows;            // row allocators of the two tables
  // time-cut windows (alz_ingest.cu): records set aside for a later window, counted past the buffer's capacity too;
  // the first defer_resolved of them were resolved by a table commit (defer_resolve_kernel)
  uint32_t defer_count, defer_resolved;
  unsigned long long late_events;           // time-cut windows: records older than the open window (reduced into it)
  unsigned long long pad2;
};

}  // namespace alz
