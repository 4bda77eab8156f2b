"""GPU: the ingest kernel's tiers (alaz_b200/csrc/alz_ingest.cu) on constructed streams.

ingest_pairs_v8_kernel has three tiers: per-CTA rows in shared memory with 16-bit cells (replicated 8x for the tier-S
pairs of the hot list), a cold path through per-warp queues, and a slow path that walks the pair dictionary. Synthetic
Zipf streams reach some of their branches only by luck. Each test here builds a stream that reaches a named branch,
and its docstring gives the arithmetic. Every case is compared per edge, bit for bit, with the oracle (or with
`scaled_oracle` for streams that repeat one period), and the stats counters with the oracle's. The tier tests run on
the three instantiations of the kernel: 32-B records, 32-B records with a window clock under which every record lies in
the open window, and 16-B packed records. Big streams go through device memory in ONE submit, so that one launch sees
them (the per-CTA rows are drained at the end of every launch)."""
import numpy as np
import pytest

import ingest_streams as ist
import oracle_lib as ol
from alaz_b200 import abi, capi
from helpers import edges_equal, explain_diff

pytestmark = pytest.mark.gpu

VARIANTS = ["rec32", "rec32_clock", "rec16"]
WIN_NS = 1 << 40                                     # rec32_clock: window w holds write times [w, w + 1) * 2^40
POD = [abi.ip("10.0.0.%d" % i) for i in range(1, 40)]
SVC = abi.ip("172.16.0.1")
TABLES = [(abi.TABLE_POD, POD, list(range(1, len(POD) + 1))), (abi.TABLE_SVC, [SVC], [7])]
OUT = abi.ip("203.0.113.9")


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def handle(variant, tables=TABLES, max_pairs=1 << 16, flags=0):
    h = capi.Handle(max_endpoints=256, max_pairs=max_pairs, flags=flags)
    if variant == "rec32_clock":
        h.window_clock(0, 0, WIN_NS)
    for tab, ips, ids in tables:
        h.upsert_batch(tab, np.asarray(ips, np.uint32), np.asarray(ids, np.uint32))
    h.commit()
    return h


def stamp(recs, window):
    """Write times inside window `window` of the rec32_clock variant (the other variants ignore them)."""
    recs = recs.copy()
    recs["write_time_ns"] = window * WIN_NS + np.arange(len(recs)) % 1000
    return recs


def submit_tiled(h, variant, tile, reps=1):
    """tile repeated reps times, in device memory, as ONE submit (32-B or packed records)."""
    tile = np.ascontiguousarray(tile, dtype=abi.L7_REC)
    recs, ovf = capi.pack_l7(tile) if variant == "rec16" else (tile, np.zeros(0, np.uint64))
    m, b = len(recs), recs.dtype.itemsize
    group = max(1, min(reps, (1 << 22) // m))
    block = np.tile(recs, group)
    p = h.dev_alloc(m * reps * b)
    po = h.dev_alloc(ovf.nbytes) if len(ovf) else None
    try:
        for r in range(0, reps, group):
            h.h2d(p + r * m * b, block[: min(group, reps - r) * m])
        if po:
            h.h2d(po, ovf)
        if variant == "rec16":
            h.submit_packed_device(p, m * reps, po)
        else:
            h.submit_device(p, m * reps)
        h.sync()
    finally:
        h.dev_free(p)
        if po:
            h.dev_free(po)


def check(h, exp, est, before=None):
    """Flush and compare edges (bit for bit) and the stats counters of this window with the oracle's."""
    before = before or {k: 0 for k in ist.STAT_KEYS + ("capacity_events",)}
    got = h.flush()
    assert edges_equal(got, exp), explain_diff(got, exp)
    st = h.stats()
    for k in ist.STAT_KEYS:
        assert st[k] - before[k] == est[k], (k, st[k] - before[k], est[k])
    assert st["capacity_events"] == before["capacity_events"]
    return st


def window(h, variant, pattern, reps, w, tables=TABLES, before=None):
    """One window: pattern x reps in one launch, flushed and checked against scaled_oracle."""
    pattern = stamp(pattern, w)
    submit_tiled(h, variant, pattern, reps)
    exp, est = ist.scaled_oracle(tables, pattern, reps)
    return check(h, exp, est, before)


def two_cell_pattern(src=POD[0], dst=SVC):
    """64 records of one pair: positions 0..39 in bucket 46 [2^31, 1.5 * 2^31), 40..63 in bucket 47
    [1.5 * 2^31, 2^32) (durations up to 2^32 - 1, so the low latency word carries), four of them 5xx. Both buckets
    lie in the window a private row gets (base4_around: buckets 40..55) and in the same 32-bit word of the row
    (cells 6 and 7). A chunk is one period; tier-S replica r takes positions r + 8j, 5 of them in bucket 46 and 3 in
    47. The two cells get unequal counts, so a spill into the wrong cell shows."""
    p = np.arange(64)
    d = np.where(p < 40, (1 << 31) + 12345 + 1000 * p, (1 << 32) - 1 - 1000 * p)
    assert [ist.latency_bucket(x) for x in d] == [46] * 40 + [47] * 24
    return ist.records(src, dst, d.astype(np.uint64), status=np.where(np.isin(p, [3, 11, 43, 60]), 503, 200))


# ---- the 16-bit cell spill ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("variant", VARIANTS)
def test_spill_private_row(variant):
    """First window, one pair (no hot list yet: the pair gets a private row in every CTA through slow_one).
    200 rounds of chunks: each CTA takes 200 x 16 chunks = 128,000 events in bucket 46 and 76,800 in 47, i.e. 3 and
    2 spills of 0x8000 per CTA (less what arrives before the row is admitted), into both halves of one word, and
    remainders of ~29,696 and ~11,264 for the drain."""
    sms = sm_count()
    pat = two_cell_pattern()
    rounds = 200
    assert rounds * ist.WARPS * 24 >= 2 * ist.CELL_SPILL
    h = handle(variant)
    window(h, variant, pat, rounds * ist.round_size(sms) // len(pat), 0)
    h.close()


REP_ROUNDS = 1400   # per tier-S replica of a CTA: 1400 x 16 chunks x (5 | 3) = 112,000 | 67,200 events per cell


@pytest.mark.parametrize("variant", VARIANTS)
def test_spill_replicated_row(variant):
    """The same pair after a flush: the hot list makes it tier S, so each CTA gives it 8 rows and lane l adds to row
    l mod 8. 1400 rounds: each replica of each CTA takes 112,000 events in bucket 46 and 67,200 in 47: 3 and 2
    spills per replica, and remainders of 13,696 and 1,664 that the drain adds from the 8 replicas."""
    sms = sm_count()
    pat = two_cell_pattern()
    h = handle(variant)
    st = window(h, variant, pat, ist.round_size(sms) // len(pat), 0)
    assert REP_ROUNDS * ist.WARPS * 3 >= 2 * ist.CELL_SPILL
    window(h, variant, pat, REP_ROUNDS * ist.round_size(sms) // len(pat), 1, before=st)
    h.close()


@pytest.mark.parametrize("variant", VARIANTS)
def test_unresolved_hot_row(variant):
    """A tier-S pair whose source is erased from the pod table (and committed) after the hot list was chosen: its
    events still hit the replicated rows, and both the spills (3 and 2 per replica, as in test_spill_replicated_row)
    and the drain (the remainders) must count them as src_unresolved, not emit them."""
    sms = sm_count()
    pat = two_cell_pattern()
    h = handle(variant)
    st = window(h, variant, pat, ist.round_size(sms) // len(pat), 0)
    h.erase(abi.TABLE_POD, POD[0])
    h.commit()
    tables = [(abi.TABLE_POD, POD[1:], list(range(2, len(POD) + 1))), (abi.TABLE_SVC, [SVC], [7])]
    window(h, variant, pat, REP_ROUNDS * ist.round_size(sms) // len(pat), 1, tables=tables, before=st)
    h.close()


# ---- hot-tier latency high words, cold queue packing --------------------------------------------------------------

@pytest.mark.parametrize("variant", VARIANTS)
def test_hot_high_words(variant):
    """A pair whose durations are 2^32 .. 2^64 - 1 (buckets 48..63, most in 63). In window 0 a CTA's row gets the
    window of the event that brought the pair in (base 12 for buckets >= 54); the fold then picks base 12, the
    window 48..63 that holds every event, so in window 1 every event is a hit. Every hit adds a high word
    (dhi != 0), low words near 2^32 carry, and the latency sum wraps mod 2^64."""
    sms = sm_count()
    d = np.array([(1 << 63) + 5, 1 << 32, (1 << 32) + 1, 3 << 31, (1 << 40) - 1, 1 << 40, (1 << 47) - 1,
                  (1 << 55) - 1, 1 << 55, (1 << 64) - 1, (1 << 63) + (1 << 62), 0xFFFFFFFF + (1 << 36)], np.uint64)
    assert min(ist.latency_bucket(x) for x in d) == 48
    pat = ist.records(POD[0], SVC, d, status=np.where(np.arange(len(d)) % 5 == 0, 500, 200))
    h = handle(variant)
    st = None
    for w, rounds in enumerate((1, 4)):
        st = window(h, variant, pat, rounds * ist.round_size(sms) // len(pat) + 3, w, before=st)
    h.close()


@pytest.mark.parametrize("variant", VARIANTS)
def test_queue_packing(variant):
    """Reversed (AMQP DELIVER) and Host-keyed rows never have a per-CTA row: they always go cold. The queue entry
    holds 23 bits of the duration's high word, so 2^55 - 1 is queued and 2^55, 2^56 and 2^64 - 1 are reduced on the
    spot; a forward pair with the same durations mixes hot hits in."""
    sms = sm_count()
    d = np.array([(1 << 55) - 1, 1 << 55, 1 << 56, (1 << 64) - 1, (1 << 55) + 1, 12345], np.uint64)
    rev = ist.records(POD[2], POD[3], d, protocol=abi.PROTO_AMQP, method=abi.AMQP_DELIVER)
    host = ist.records(POD[4], 77, d, protocol=abi.PROTO_HTTP | abi.PROTO_F_HOSTKEY)
    fwd = ist.records(POD[5], OUT, d, status=503)
    pat = np.concatenate([rev, host, fwd])
    h = handle(variant)
    st = None
    for w in range(2):
        st = window(h, variant, pat, 2 * ist.round_size(sms) // len(pat) + 7, w, before=st)
    h.close()


# ---- hot list tiers -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("k", [8, 9])
def test_tier_s_boundary(variant, k):
    """k equally hot pairs, three windows. hot_emit_kernel takes the pairs of the top count bins while their number
    is <= 8 (kHotS): 8 equal pairs are all tier S (8 rows each), 9 are all tier A."""
    sms = sm_count()
    pat = ist.records(POD[:k], SVC, 1_000_000 + 100_000 * np.arange(k), status=np.where(np.arange(k) == 2, 500, 200))
    h = handle(variant)
    st = None
    for w in range(3):
        st = window(h, variant, pat, 2 * ist.round_size(sms) // k + w, w, before=st)
    h.close()


@pytest.mark.parametrize("variant", VARIANTS)
def test_window_miss(variant):
    """A hot pair whose 16-bucket window no longer fits its latencies. Window 0 puts it at buckets 0..3 (base 0);
    window 1 is bimodal over buckets 0, 5, 15 (in the row's window) and 16, 40, 63 (cold), most events at the top,
    so window 2 gets base 12 and sees buckets 0 and 63 again: every pair row gets hot and cold contributions."""
    sms = sm_count()
    low = ist.records(POD[0], SVC, np.array([0, 100, 255, 300, 600, 1000], np.uint64))
    d = [0, 200, ist.bucket_lo(5), ist.bucket_lo(15) + 7, ist.bucket_lo(16), ist.bucket_lo(40)] + [1 << 40] * 5 + \
        [(1 << 41) + 3, ist.bucket_lo(60), ist.bucket_lo(62) + 1]
    bim = ist.records(POD[0], SVC, np.array(d, np.uint64))
    assert sorted({ist.latency_bucket(x) for x in d}) == [0, 5, 15, 16, 40, 60, 62, 63]
    h = handle(variant)
    st = None
    for w, pat in enumerate((low, bim, bim)):
        st = window(h, variant, pat, 2 * ist.round_size(sms) // len(pat) + 1, w, before=st)
    h.close()


# ---- collisions ---------------------------------------------------------------------------------------------------

def colliding_keys():
    """Three keys with one table_hash (one bucket, one fingerprint: the first admitted owns the entry the lookup
    finds, the second has a row no lookup reaches, the third no slot) and three keys in one 2-way bucket with
    different fingerprints (two entries, the third no slot). Destinations are outbound addresses."""
    a = [(POD[6], OUT)] + [(s, ist.collide_table(POD[6], OUT, s)) for s in (POD[7], POD[8])]
    h0 = int(ist.table_hash(ist.pair_key(POD[9], OUT)))
    b = [(POD[9], OUT)] + [(s, ist.daddr_for_table_hash(s, h0 ^ x)) for s, x in ((POD[10], 2), (POD[11], 4))]
    for keys in (a, b):
        hs = ist.table_hash(ist.pair_key([s for s, _ in keys], [d for _, d in keys]))
        assert len(set(ist.tab_idx1(hs).tolist())) == 1
    assert len(set(ist.table_hash(ist.pair_key([s for s, _ in a], [d for _, d in a])).tolist())) == 1
    assert len(set(ist.tab_fp(ist.table_hash(ist.pair_key([s for s, _ in b], [d for _, d in b]))).tolist())) == 3
    table_ips = set(POD) | {SVC}
    assert not any(d in table_ips for _, d in a + b)
    return a + b


@pytest.mark.parametrize("variant", VARIANTS)
def test_per_cta_collisions(variant):
    """Six colliding keys (colliding_keys), each with its own edge, and eight hotter pairs that take tier S, so that
    after the first flush the colliding keys come back through the hot list as tier A. Window 0 admits them as
    private rows in whatever order the warps meet them. A key served by another key's entry must go cold and leave
    that key's row alone."""
    sms = sm_count()
    keys = colliding_keys()
    s = np.array([k[0] for k in keys] + POD[12:20] * 4, np.uint64)
    d = np.array([k[1] for k in keys] + [SVC] * 32, np.uint64)
    pat = ist.records(s, d, 1_500_000 + 7919 * np.arange(len(s)), status=np.where(np.arange(len(s)) % 7 == 1, 500, 200))
    h = handle(variant)
    st = None
    for w in range(3):
        st = window(h, variant, pat, 2 * ist.round_size(sms) // len(pat) + w, w, before=st)
    h.close()


@pytest.mark.parametrize("variant", VARIANTS)
def test_dictionary_home_slot_collisions(variant):
    """Eight keys per dictionary (forward, reversed, Host-keyed) that share one home slot `pair_hash & mask`: every
    cold probe of all but the first misses its home slot and goes down the slow path, which walks the probe chain."""
    sms = sm_count()
    fm, rm, hm = ist.dict_masks(1 << 12)
    parts = []
    for mask, proto, method in ((fm, abi.PROTO_HTTP, 1), (rm, abi.PROTO_AMQP, abi.AMQP_DELIVER),
                                (hm, abi.PROTO_HTTP | abi.PROTO_F_HOSTKEY, 1)):
        keys, _ = ist.collide_home(mask, POD[20:24], 8)
        parts.append(ist.records([k[0] for k in keys], [k[1] for k in keys], 2_000_000 + np.arange(8) * 333_333,
                                 protocol=proto, method=method))
    pat = np.concatenate(parts)
    h = handle(variant, max_pairs=1 << 12)
    st = None
    for w in range(2):
        st = window(h, variant, pat, ist.round_size(sms) // len(pat) + 5, w, before=st)
    h.close()


@pytest.mark.parametrize("variant", VARIANTS)
def test_sentinel_key(variant):
    """255.255.255.255 -> 255.255.255.255 from a pod: the key equals the dictionaries' free marker, so it has a
    fixed row per kind, is never given a per-CTA row and never taken as a home-slot hit. A flood of it, forward,
    reversed and Host-keyed (host id 2^32 - 1), next to an ordinary pair."""
    sms = sm_count()
    ff = 0xFFFFFFFF
    tables = [(abi.TABLE_POD, POD + [ff], list(range(1, len(POD) + 1)) + [99]), (abi.TABLE_SVC, [SVC], [7])]
    d = np.array([300, 2_000_000, 1 << 33, 5_000_000], np.uint64)
    pat = np.concatenate([ist.records(ff, ff, d, status=500), ist.records(ff, ff, d, status=500)[:2],
                          ist.records(ff, ff, d, protocol=abi.PROTO_AMQP, method=abi.AMQP_DELIVER),
                          ist.records(ff, ff, d, protocol=abi.PROTO_HTTP | abi.PROTO_F_HOSTKEY),
                          ist.records(POD[0], SVC, d)])
    h = handle(variant, tables=tables)
    st = None
    for w in range(2):
        st = window(h, variant, pat, 2 * ist.round_size(sms) // len(pat) + 1, w, tables=tables, before=st)
    h.close()


# ---- launch shapes --------------------------------------------------------------------------------------------------

def mixed_stream(n, seed):
    """n records over a few pairs: forward to a service, a pod and an outbound address, reversed, Host-keyed, from
    an unknown source, and not-a-request protocols; durations over the whole bucket range."""
    rng = np.random.default_rng(seed)
    src = np.array(POD[:5] + [abi.ip("9.9.9.9")], np.uint64)[rng.integers(0, 6, n)]
    dst = np.array([SVC, POD[30], OUT, 77], np.uint64)[rng.integers(0, 4, n)]
    r = ist.records(src, dst, rng.integers(0, 1 << 45, n, dtype=np.uint64),
                    status=rng.choice([200, 404, 500, 503], n))
    kind = rng.integers(0, 10, n)
    r["protocol"] = np.select([kind == 0, kind == 1, dst == 77], [abi.PROTO_KAFKA, abi.PROTO_AMQP,
                                                                   abi.PROTO_HTTP | abi.PROTO_F_HOSTKEY], abi.PROTO_HTTP)
    r["method_flags"] = np.where(kind == 1, abi.AMQP_DELIVER, 1)
    return r


RAGGED = ["1", "63", "64", "65", "round-1", "round+1"]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("size", RAGGED)
def test_ragged_launches(variant, size):
    """Launches smaller than one round of chunks (CTAs without a chunk), one chunk +- 1 (a tail chunk), and one round
    +- 1 record."""
    r = ist.round_size(sm_count())
    n = {"1": 1, "63": 63, "64": 64, "65": 65, "round-1": r - 1, "round+1": r + 1}[size]
    recs = stamp(mixed_stream(n, n), 0)
    h = handle(variant)
    submit_tiled(h, variant, recs)
    exp, est = ist.oracle_run(TABLES, recs)
    check(h, exp, est)
    h.close()


@pytest.mark.parametrize("variant", VARIANTS)
def test_high_cardinality(variant):
    """Every event a new pair (a pod to a fresh outbound address), one round + 37 records: every event takes the
    slow path, slow queues fill, and warps of every CTA insert into the dictionary at once."""
    n = ist.round_size(sm_count()) + 37
    recs = stamp(ist.records(np.array(POD[:4], np.uint64)[np.arange(n) % 4], abi.ip("198.18.0.0") + np.arange(n),
                             1000 + np.arange(n) * 977), 0)
    h = handle(variant, max_pairs=1 << 18)
    submit_tiled(h, variant, recs)
    exp, est = ist.oracle_run(TABLES, recs)
    assert len(exp) == n
    check(h, exp, est)
    h.close()


# ---- protocol bytes ----------------------------------------------------------------------------------------------

def protocol_records(values):
    """For every protocol byte: forward and reversing methods, the payload-reject flag, TLS, 200 and 5xx."""
    v = np.repeat(np.asarray(values, np.uint8), 8)
    k = np.tile(np.arange(8), len(values))
    r = ist.records(np.where(k % 4 == 3, POD[1], POD[0]), np.where(k % 2 == 0, SVC, POD[1]),
                    1000 + 37 * np.arange(len(v), dtype=np.uint64) ** 3, status=np.where(k < 4, 503, 200))
    r["protocol"] = v
    r["method_flags"] = np.array([1, 2, 2 | abi.MF_PAYLOAD_REJECT, 3, 1 | abi.MF_TLS, 2 | abi.MF_TLS, 1 | abi.MF_PAYLOAD_REJECT,
                                  0], np.uint8)[k]
    return r


NO_BIT6 = [p for p in range(256) if not p & abi.PROTO_F_HOSTKEY]


@pytest.mark.parametrize("flags", [0, abi.CFG_EAGER_JOIN, abi.CFG_NO_SMEM_CACHE])
def test_protocol_bytes_on_32b_records(flags):
    """Every protocol byte without the Host-key flag, on each plan: the bytes the ABI does not define (9..63 and
    anything with bit 7) produce no row, as in the oracle."""
    recs = protocol_records(NO_BIT6)
    h = handle("rec32", flags=flags)
    h.submit(recs)
    exp, est = ist.oracle_run(TABLES, recs)
    check(h, exp, est)
    h.close()


def to_raw(recs):
    """32-B records -> 1096-B eBPF samples (struct l7_event) carrying the same fields."""
    n = len(recs)
    raw = np.zeros((n, abi.BPF_L7_EVENT_SIZE), np.uint8)

    def put(off, a, dt):
        b = np.ascontiguousarray(np.asarray(a).astype(dt)).view(np.uint8).reshape(n, -1)
        raw[:, off:off + b.shape[1]] = b
    put(8, recs["write_time_ns"], "<u8")
    put(20, recs["status"], "<u4")
    put(24, recs["duration_ns"], "<u8")
    raw[:, 32] = recs["protocol"]
    raw[:, 33] = recs["method_flags"] & abi.MF_METHOD_MASK
    raw[:, 1066] = (recs["method_flags"] & abi.MF_TLS) != 0
    put(1076, recs["saddr"], "<u4")
    put(1080, recs["sport"], "<u2")
    put(1084, recs["daddr"], "<u4")
    put(1088, recs["dport"], "<u2")
    return raw.reshape(-1)


def test_protocol_bytes_on_raw_samples():
    """Every protocol byte of an eBPF sample. The sample has no flag bits: 0x41 is no Host-keyed HTTP row but an
    undefined protocol, like every byte >= 9."""
    recs = protocol_records(range(256))
    raw = to_raw(recs)
    compact = ol.compact_raw(raw)
    o = ol.Oracle()
    for tab, ips, ids in TABLES:
        for ip, i in zip(ips, ids):
            o.upsert(tab, ip, i)
    o.process(compact)
    h = handle("rec32")
    h.submit_raw(raw)
    exp, ost = o.edges(), o.stats()
    check(h, exp, {k: ost[k] for k in ist.STAT_KEYS})
    o.close()
    h.close()


def test_submit_equals_submit_packed():
    """Every protocol byte, durations on both sides of 2^32: submit(recs) and submit_packed(pack_l7(recs)) give the
    same bytes (docs/SPEC.md §10)."""
    recs = protocol_records(range(256))
    recs["duration_ns"][::3] += np.uint64(1 << 32)
    recs["daddr"][(recs["protocol"] & abi.PROTO_F_HOSTKEY) != 0] = 77
    out = []
    for packed in (False, True):
        h = handle("rec32")
        if packed:
            h.submit_packed(*capi.pack_l7(recs))
        else:
            h.submit(recs)
        out.append((h.flush(), {k: h.stats()[k] for k in ist.STAT_KEYS}))
        h.close()
    assert len(out[0][0]) > 0
    assert out[0][0].tobytes() == out[1][0].tobytes()
    assert out[0][1] == out[1][1]


# ---- the fold before a cell can wrap ---------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["forward", "reversed"])
def test_fold_before_a_cell_can_wrap(kind):
    """Packed records in device memory, all of one pair in one bucket: 2^31 - 1 events, then 2^31 + 2^20 in one
    call. Without a fold between them one pair cell would take 2^32 + 2^20 - 1 events and wrap (hot path: the u32
    cell; reversed rows, cold path: the u64 add of a cell pair would carry into the neighbouring cell). Expected:
    count = N exactly, hist = N mod 2^32, lat_sum = N * d mod 2^64. Needs ~34.4 GB of device memory."""
    import torch
    free = torch.cuda.mem_get_info()[0]
    if free < 40 << 30:
        pytest.skip(f"needs 40 GB of free device memory, {free >> 30} GB free")
    n1, n2 = (1 << 31) - 1, (1 << 31) + (1 << 20)
    d = (1 << 33) + 12345                              # bucket 50: the low cell of its pair; >= 2^32: overflow array
    assert ist.latency_bucket(d) == 50
    rec = ist.records(POD[0], SVC, d, status=503) if kind == "forward" else \
        ist.records(POD[0], POD[1], d, protocol=abi.PROTO_AMQP, method=abi.AMQP_DELIVER)
    packed, ovf = capi.pack_l7(rec)
    assert len(ovf) == 1
    h = handle("rec16")
    tile = np.tile(packed, 1 << 24)
    p = h.dev_alloc(n2 * 16)
    po = h.dev_alloc(8)
    try:
        for i in range(0, n2, len(tile)):
            h.h2d(p + i * 16, tile[: min(len(tile), n2 - i)])
        h.h2d(po, ovf)
        h.submit_packed_device(p, n1, po)
        h.submit_packed_device(p, n2, po)
        h.sync()
    finally:
        h.dev_free(p)
        h.dev_free(po)
    n = n1 + n2
    exp, est = ist.scaled_oracle(TABLES, rec, n)
    assert int(exp["count"][0]) == n and int(exp["hist"][0][50]) == n & ist.M32
    check(h, exp, est)
    h.close()
