"""GPU: one pair-dictionary slot per socket pair, and per-CTA rows for reversed pairs (alaz_b200/csrc/alz_ingest.cu).

A socket pair's forward rows and its reversed rows (AMQP DELIVER, REDIS PUSHED_EVENT) share one slot of the pair
dictionary, {key, row_fwd, row_rev}: each row word is allocated the first time an event of its kind comes. Reversed
pairs enter the hot list and get per-CTA rows like forward ones; the per-CTA index tells the two kinds of one key
apart by their fingerprints. Every case is compared per edge, bit for bit, with the oracle, and the stats counters
with the oracle's."""
import ctypes as C

import numpy as np
import pytest

import ingest_streams as ist
from alaz_b200 import abi, capi
from helpers import edges_equal, explain_diff
from test_gpu_ingest import POD, SVC, OUT, TABLES, VARIANTS, check, handle, sm_count, to_raw, two_cell_pattern, window

pytestmark = pytest.mark.gpu

PLANS = [0, abi.CFG_EAGER_JOIN, abi.CFG_NO_SMEM_CACHE]
# packed records run on the default plan only (the other plans refuse them with ALZ_E_UNSUPPORTED)
PLAN_FORMATS = [(f, fmt) for f in PLANS for fmt in ("rec32", "raw")] + [(0, "rec16")]


def reversed_(recs):
    """The same records as AMQP DELIVER: the row is reversed (the pod resolved from saddr is its To end)."""
    r = recs.copy()
    r["protocol"], r["method_flags"] = abi.PROTO_AMQP, abi.AMQP_DELIVER
    return r


def submit_host(h, fmt, recs):
    if fmt == "rec32":
        h.submit(recs)
    elif fmt == "rec16":
        h.submit_packed(*capi.pack_l7(recs))
    else:
        h.submit_raw(to_raw(recs))


def both_kinds(n_pairs, per_pair, seed):
    """Forward and reversed records of n_pairs socket pairs (pods to a service, a pod and outbound addresses)."""
    rng = np.random.default_rng(seed)
    s = np.array(POD[:10], np.uint64)[np.arange(n_pairs) % 10]
    d = np.array([SVC, POD[30], OUT] + [abi.ip("198.51.100.%d" % i) for i in range(1, 60)], np.uint64)[
        np.arange(n_pairs) // 10 % 62]
    s, d = np.repeat(s, per_pair), np.repeat(d, per_pair)
    f = ist.records(s, d, rng.integers(0, 1 << 36, len(s), dtype=np.uint64), status=rng.choice([200, 500], len(s)))
    return f, reversed_(f)


# ---- both rows of one slot --------------------------------------------------------------------------------------

@pytest.mark.parametrize("flags,fmt", PLAN_FORMATS)
@pytest.mark.parametrize("order", ["forward_first", "reversed_first", "racing"])
def test_both_kinds_one_slot(flags, fmt, order):
    """Each socket pair's forward and reversed rows are first used by separate launches in either order, or in
    one launch where every chunk holds both kinds of the same pairs, so that warps of every CTA race for the key and
    for each row word. Two windows: the second starts from a hot list that holds rows of both kinds."""
    f, r = both_kinds(200, 40, 11)
    h = handle("rec32", flags=flags)
    st = None
    for w in range(2):
        if order == "racing":
            parts = [np.stack([f, r], axis=1).reshape(-1)]
        else:
            parts = [f, r] if order == "forward_first" else [r, f]
        for p in parts:
            submit_host(h, fmt, p)
        exp, est = ist.oracle_run(TABLES, np.concatenate(parts))
        st = check(h, exp, est, before=st)
    h.close()


@pytest.mark.parametrize("flags,fmt", PLAN_FORMATS)
def test_mixed_kind_home_slot_collisions(flags, fmt):
    """Eight socket pairs that share one home slot of the pair dictionary, each with forward and reversed events,
    interleaved: the first pair's slot holds both of its rows, every other pair walks the probe chain, and a probe that
    finds a pair's key with no row of its kind yet goes down the slow path."""
    keys, _ = ist.collide_home(ist.dict_masks(1 << 12)[0], POD[20:24], 8)
    f = ist.records([k[0] for k in keys], [k[1] for k in keys], 2_000_000 + np.arange(8) * 333_333)
    pat = np.stack([reversed_(f), f], axis=1).reshape(-1)
    pat = np.tile(pat, 300)
    h = handle("rec32", max_pairs=1 << 12, flags=flags)
    st = None
    for w in range(2):
        submit_host(h, fmt, pat)
        exp, est = ist.oracle_run(TABLES, pat)
        st = check(h, exp, est, before=st)
    h.close()


@pytest.mark.parametrize("flags,fmt", PLAN_FORMATS)
def test_sentinel_key_each_kind(flags, fmt):
    """255.255.255.255 -> 255.255.255.255 from a pod equals the free marker: forward, reversed and Host-keyed each
    have their fixed row, and a slot never claims the key for either row word. (An eBPF sample has no Host-key flag,
    so the raw format leaves the Host-keyed records out.)"""
    ff = 0xFFFFFFFF
    tables = [(abi.TABLE_POD, POD + [ff], list(range(1, len(POD) + 1)) + [99]), (abi.TABLE_SVC, [SVC], [7])]
    d = np.array([300, 2_000_000, 1 << 33, 5_000_000], np.uint64)
    f = ist.records(ff, ff, d, status=500)
    host = ist.records(ff, ff, d, protocol=abi.PROTO_HTTP | abi.PROTO_F_HOSTKEY)
    pat = np.tile(np.concatenate([f, reversed_(f)] + ([host] if fmt != "raw" else []) +
                                 [ist.records(POD[0], SVC, d), reversed_(ist.records(POD[0], SVC, d))]), 500)
    h = handle("rec32", tables=tables, flags=flags)
    st = None
    for w in range(2):
        submit_host(h, fmt, pat)
        exp, est = ist.oracle_run(tables, pat)
        st = check(h, exp, est, before=st)
    h.close()


# ---- reversed pairs in the per-CTA table --------------------------------------------------------------------------

REP_ROUNDS = 1400   # as test_gpu_ingest.test_spill_replicated_row: 3 and 2 spills per replica and cell


@pytest.mark.parametrize("variant", VARIANTS)
def test_spill_reversed_tier_s(variant):
    """test_spill_replicated_row on a reversed pair: after the first flush the pair is tier S (8 rows per CTA),
    its two cells spill into the pair's reversed row and the drain adds the remainders there."""
    sms = sm_count()
    pat = reversed_(two_cell_pattern())
    h = handle(variant)
    st = window(h, variant, pat, ist.round_size(sms) // len(pat), 0)
    window(h, variant, pat, REP_ROUNDS * ist.round_size(sms) // len(pat), 1, before=st)
    h.close()


@pytest.mark.parametrize("variant", VARIANTS)
def test_spill_reversed_tier_a(variant):
    """A reversed pair below eight forward pairs of twice its count: they take tier S, it takes tier A, one row per
    CTA. 150,000 periods of 17 chunks: its chunk reaches each warp ~71 times, so each CTA's row takes ~45,000 events
    in bucket 46: a spill of 0x8000 into the reversed global row, and the rest through the drain."""
    sms = sm_count()
    rev = reversed_(two_cell_pattern())
    fwd = ist.records(np.repeat(np.array(POD[1:9], np.uint64), 128), SVC,
                      5_000_000 + 1000 * np.arange(8 * 128, dtype=np.uint64))
    pat = np.concatenate([rev, fwd])
    assert len(pat) == 17 * ist.CHUNK
    h = handle(variant)
    st = window(h, variant, pat, ist.round_size(sms) // len(pat) + 1, 0)
    window(h, variant, pat, 150_000, 1, before=st)
    h.close()


@pytest.mark.parametrize("variant", VARIANTS)
def test_unresolved_reversed_hot_row(variant):
    """A reversed tier-S pair whose source is erased from the pod table after the hot list was chosen: its events
    still hit the per-CTA rows, and the spills and the drain count them as src_unresolved."""
    sms = sm_count()
    pat = reversed_(two_cell_pattern())
    h = handle(variant)
    st = window(h, variant, pat, ist.round_size(sms) // len(pat), 0)
    h.erase(abi.TABLE_POD, POD[0])
    h.commit()
    tables = [(abi.TABLE_POD, POD[1:], list(range(2, len(POD) + 1))), (abi.TABLE_SVC, [SVC], [7])]
    window(h, variant, pat, REP_ROUNDS * ist.round_size(sms) // len(pat), 1, tables=tables, before=st)
    h.close()


# ---- row pool exhaustion between the two kinds of one pair -------------------------------------------------------

@pytest.mark.parametrize("flags", [0, abi.CFG_NO_SMEM_CACHE])
@pytest.mark.parametrize("first", ["forward", "reversed"])
def test_row_pool_exhausted_between_kinds(flags, first):
    """max_pairs rows: max_pairs - 1 other pairs, then the pair's first kind takes the last row and its second kind
    finds the pool empty. Launches run in order, so which kind is lost is fixed. The lost kind's events are counted
    as capacity_events, the flush reports ALZ_E_CAPACITY, and every edge it returns is exact."""
    max_pairs = 1024
    others = ist.records(POD[1], abi.ip("198.18.0.0") + np.arange(max_pairs - 1, dtype=np.uint64), 5000)
    f = ist.records(POD[0], SVC, 1000 + 977 * np.arange(50, dtype=np.uint64), status=503)
    a, b = (f, reversed_(f)) if first == "forward" else (reversed_(f), f)
    h = capi.Handle(max_endpoints=256, max_pairs=max_pairs, max_edges=4 * max_pairs, flags=flags)
    for tab, ips, ids in TABLES:
        h.upsert_batch(tab, np.asarray(ips, np.uint32), np.asarray(ids, np.uint32))
    h.commit()
    for p in (others, a, b, np.concatenate([b, a])):   # the last launch: the lost kind again, and a hit on the kept one
        h.submit(p)
    exp, _ = ist.oracle_run(TABLES, np.concatenate([others, a, a]))
    out = np.zeros(4 * max_pairs, dtype=abi.EDGE_OUT)
    n = C.c_size_t(0)
    rc = h.L.alz_window_flush(h.h, out.ctypes.data_as(C.c_void_p), len(out), C.byref(n))
    assert rc == abi.E_CAPACITY
    got = out[: n.value]
    assert edges_equal(got, exp), explain_diff(got, exp)
    assert h.stats()["capacity_events"] == 2 * len(b)
    h.close()
