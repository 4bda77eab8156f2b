"""Constructed l7 streams for the ingest kernel's tiers (alaz_b200/csrc/alz_ingest.cu). TEST INFRASTRUCTURE ONLY.

Plain numpy plus the oracle:
  - restatements of the kernel's hashes (`table_hash`, `tab_idx1/2`, `tab_fp` of the per-CTA table, `pair_hash` of the
    pair dictionaries) and of `latency_bucket` (docs/SPEC.md §4), so that a test can build keys that collide where it
    wants them to;
  - the dictionary sizes `alloc_table` (alz_api.cu) derives from `max_pairs`;
  - the kernel's split of the records over CTAs, warps, lanes and tier-S replicas, so that a test can state how many
    events each CTA row and each replica takes;
  - `scaled_oracle`: the oracle's edges of a stream that repeats one period many times, computed from one period, so
    that streams of 10^8..4·10^9 events are checked exactly without running the oracle on them.
"""
import numpy as np

import oracle_lib as ol
from alaz_b200 import abi
from gnn_graphs import HOST, HOST_DADDR

M32, M64 = (1 << 32) - 1, (1 << 64) - 1
WARPS, CHUNK = 16, 64            # warps per CTA, records per chunk (one TMA copy of a warp)
HOT_S, HOT_REP = 8, 8            # tier S: the hottest pairs, kHotRep rows each
CELL_SPILL = 0x8000              # a 16-bit cell moves this many counts to the global row when it reaches it
TAB_SHIFT = 20
_A, _B = 0x9E3779B1, 0x85EBCA6B
_B_INV = pow(_B, -1, 1 << 32)    # B is odd


def pair_key(saddr, daddr):
    """make_pair_key: daddr in the high word, saddr in the low word."""
    return (np.asarray(daddr, np.uint64) << np.uint64(32)) | np.asarray(saddr, np.uint64)


def _lo_hi(key):
    key = np.asarray(key, np.uint64)
    return key & np.uint64(M32), key >> np.uint64(32)


def table_hash(key):
    """The per-CTA table's hash: lo * 0x9E3779B1 + hi * 0x85EBCA6B mod 2^32 (linear in both words)."""
    lo, hi = _lo_hi(key)
    return ((lo * np.uint64(_A) + hi * np.uint64(_B)) & np.uint64(M32)).astype(np.uint32)


def tab_idx1(h):
    return (np.asarray(h, np.uint32) >> np.uint32(TAB_SHIFT)) & np.uint32(0xFFFFFFFE)


def tab_idx2(h):
    return (np.asarray(h, np.uint32) >> np.uint32(TAB_SHIFT)) | np.uint32(1)


def tab_fp(h):
    """Fingerprint of an index entry: the hash's low 16 bits, in bits 31..16, never 0."""
    return ((np.asarray(h, np.uint64) << np.uint64(16)) | np.uint64(0x10000)).astype(np.uint32)


def pair_hash(key):
    """The pair dictionaries' hash (alz_device.cuh)."""
    lo, hi = _lo_hi(key)
    h = ((hi * np.uint64(_A)) & np.uint64(M32)) ^ ((lo * np.uint64(_B)) & np.uint64(M32))
    h ^= h >> np.uint64(15)
    h = (h * np.uint64(0x2C1B3C6D)) & np.uint64(M32)
    h ^= h >> np.uint64(13)
    return h.astype(np.uint32)


def latency_bucket(d):
    """docs/SPEC.md §4: two sub-buckets per octave over [2^8, 2^40), clamped to 0..63."""
    d = int(d)
    if d < 256:
        return 0
    o = d.bit_length() - 1
    if o >= 40:
        return abi.NB - 1
    return 2 * (o - 8) + ((d >> (o - 1)) & 1)


def bucket_lo(b):
    """Smallest duration of bucket b (b >= 1)."""
    return (1 << (8 + b // 2)) * (3 if b % 2 else 2) // 2


def next_pow2(x):
    p = 1
    while p < x:
        p <<= 1
    return min(p, 1 << 31)


def dict_masks(max_pairs):
    """(forward, reversed, host-keyed) dictionary masks of a handle with `max_pairs` (alloc_table)."""
    cap = next_pow2(2 * max_pairs)
    return cap - 1, max(1024, cap >> 2) - 1, max(1024, cap >> 3) - 1


def daddr_for_table_hash(saddr, h):
    """The daddr that gives the key (saddr, daddr) the per-CTA table hash h."""
    return (((int(h) - int(saddr) * _A) * _B_INV) & M32)


def collide_table(pod_saddr, d1, s2):
    """The daddr that gives a key from source s2 the same table_hash as (pod_saddr, d1): same bucket, same
    fingerprint, so only the row's key tells the two apart."""
    return daddr_for_table_hash(s2, int(table_hash(pair_key(pod_saddr, d1))))


def collide_home(mask, pods, n, daddr_base=abi.ip("203.0.0.0"), span=1 << 22):
    """n keys (saddr, daddr) from the given pod addresses that share one home slot `pair_hash & mask` of a
    dictionary, found by search over the outbound addresses daddr_base + [0, span)."""
    d = np.arange(span, dtype=np.uint64) + np.uint64(daddr_base)
    target, out = None, []
    for s in pods:
        slots = pair_hash(pair_key(np.full(span, s, np.uint64), d)) & np.uint32(mask)
        if target is None:
            target = int(slots[0])
        hit = d[slots == target]
        out += [(int(s), int(x)) for x in hit[: n - len(out)]]
        if len(out) == n:
            return out, target
    raise ValueError("not enough colliding keys in the span")


# ---- which CTA, lane and replica takes a record ----------------------------------------------------------------

def round_size(sms):
    """Records in one round of chunks: every warp of every CTA one chunk."""
    return sms * WARPS * CHUNK


def cta_of_record(i, sms):
    """Chunk c = i // 64 goes to warp c mod (sms * 16) of the grid, i.e. CTA (c mod (sms * 16)) // 16."""
    c = np.asarray(i, np.int64) // CHUNK
    return (c % (sms * WARPS)) // WARPS


def replica_of_record(i):
    """Record p of a chunk is taken by lane p mod 32; a tier-S pair's row group is indexed by lane mod 8."""
    return (np.asarray(i, np.int64) % CHUNK) % 32 % HOT_REP


def per_cta_counts(n, sms, mask=None):
    """Events of the first n records (or of those where mask) that each CTA takes."""
    i = np.arange(n, dtype=np.int64)
    cta = cta_of_record(i, sms)
    return np.bincount(cta if mask is None else cta[np.asarray(mask)[:n]], minlength=sms)


# ---- expected edges ----------------------------------------------------------------------------------------------

def records(saddr, daddr, dur, protocol=abi.PROTO_HTTP, method=1, status=200, write_time=0):
    """alz_l7_rec per element (scalars broadcast)."""
    saddr, daddr, dur = np.broadcast_arrays(*(np.atleast_1d(np.asarray(x, np.uint64)) for x in (saddr, daddr, dur)))
    n = len(saddr)
    r = np.zeros(n, dtype=abi.L7_REC)
    r["saddr"], r["daddr"], r["duration_ns"] = saddr, daddr, dur
    r["sport"] = 40000 + np.arange(n) % 20000
    r["dport"] = 80
    r["status"], r["protocol"], r["method_flags"] = status, protocol, method
    r["write_time_ns"] = write_time
    return r


STAT_KEYS = ("events_in", "rows_emitted", "not_request", "src_unresolved")


def oracle_run(tables, recs):
    """(edges, stats) of the oracle on `recs` under `tables` = [(table, ips, ids), ...]. Host-keyed rows
    (ALZ_PROTO_F_HOSTKEY, daddr = the host id) reach it as they reach the reference: daddr a placeholder address
    that is in no table, the header text in the names."""
    recs = np.ascontiguousarray(recs, dtype=abi.L7_REC)
    hk = (recs["protocol"] & abi.PROTO_F_HOSTKEY) != 0
    host_ids = np.unique(recs["daddr"][hk]).astype(np.uint64)
    orc = recs.copy()
    orc["protocol"] &= np.uint8(~abi.PROTO_F_HOSTKEY & 0xFF)
    host_idx = np.zeros(len(recs), np.uint32)
    host_idx[hk] = 1 + np.searchsorted(host_ids, recs["daddr"][hk])
    orc["daddr"][hk] = HOST_DADDR
    o = ol.Oracle()
    for tab, ips, ids in tables:
        for ip, i in zip(np.asarray(ips).tolist(), np.asarray(ids).tolist()):
            o.upsert(tab, ip, i)
    o.process_hosts(orc, host_idx, ["h%d.example" % int(x) for x in host_ids])
    e, st = o.edges(), o.stats()
    o.close()
    m = e["to_type"] == HOST
    e["to"][m] = host_ids[e["to"][m]]
    return e, {k: st[k] for k in STAT_KEYS}


def _key(e):
    return int(e["from_type"]), int(e["from"]), int(e["to_type"]), int(e["to"])


def scaled_oracle(tables, pattern, reps, prefix=None):
    """(edges, stats) of prefix + tile(pattern, reps), from the oracle on one period: count, err5xx and lat_sum_ns
    times reps mod 2^64, hist cells times reps mod 2^32, plus the prefix's (same rules)."""
    e, st = oracle_run(tables, pattern)
    e = e.copy()
    for f in ("count", "err5xx", "lat_sum_ns"):
        e[f] = [int(v) * reps & M64 for v in e[f]]
    e["hist"] = (e["hist"].astype(object) * reps & M32).astype(np.uint32)
    stats = {k: v * reps for k, v in st.items()}
    if prefix is None or len(prefix) == 0:
        return e, stats
    e0, st0 = oracle_run(tables, prefix)
    at = {_key(x): i for i, x in enumerate(e)}
    new = []
    for x in e0:
        i = at.get(_key(x))
        if i is None:
            new.append(x)
            continue
        for f in ("count", "err5xx", "lat_sum_ns"):
            e[f][i] = (int(e[f][i]) + int(x[f])) & M64
        e["hist"][i] = ((e["hist"][i].astype(np.uint64) + x["hist"]) & np.uint64(M32)).astype(np.uint32)
    if new:
        e = np.concatenate([e, np.array(new, dtype=abi.EDGE_OUT)])
    return e, {k: stats[k] + st0[k] for k in stats}
