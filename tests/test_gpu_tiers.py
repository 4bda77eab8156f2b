"""GPU: tiered history (alz_window_history_tiers, alz_window_rollup_tier*, alz_window_tier_state, docs/SPEC.md §13)
against the sequential model of tests/tier_model.py. Every tier rollup is compared with the model byte for byte,
order included, with alz_rollup_info field by field and with the tier's state; where the tables stand still also with
one oracle over all events of the covered windows."""
import threading

import numpy as np
import pytest

import oracle_lib as ol
from alaz_b200 import abi, capi
from gnn_graphs import POD_NET
from helpers import explain_diff
from rollup_model import RollupModel
from test_gpu_flush import flush_device_raw, flush_raw, oracle_edges, records
from test_gpu_rollup import (HOST_ID, LAYOUTS, N_KEYS, PA, PB, PC, SV, TABLES, by_key, rollup_raw, same_rows,
                             spec_records)
from tier_model import TierModel

pytestmark = pytest.mark.gpu


class Tiers:
    """A handle and the models, driven together: every flush that consumes its window feeds the tier model and the
    window-history model with the rows the flush returned."""

    def __init__(self, tiers, tables=(), history=None, **kw):
        kw.setdefault("max_endpoints", 1 << 14)
        kw.setdefault("max_pairs", 1 << 14)
        self.h = capi.Handle(**kw)
        self.m, self.m0 = TierModel(), RollupModel()
        for tab, ips, ids in tables:
            self.h.upsert_batch(tab, np.asarray(ips, np.uint32), np.asarray(ids, np.uint32))
        self.h.commit()
        if history:
            self.history(*history)
        self.configure(tiers)
        self.wins = []   # (rows, records) of every consumed window

    def configure(self, tiers):
        self.h.window_history_tiers(tiers)
        self.m.configure(tiers)

    def history(self, depth, arena_rows):
        self.h.window_history(depth, arena_rows)
        self.m0.history(depth, arena_rows)

    def flush(self, cap=None, path="host", epoch=None, expect=abi.OK, recs=None):
        cap = self.h.max_edges if cap is None else cap
        if path == "host":
            rc, rows, n = flush_raw(self.h, cap)
        else:
            rc, rows = flush_device_raw(self.h)
            n = len(rows)
        assert rc == expect, rc
        if n <= cap:   # one rank: only a too-small buffer keeps the window
            w = self.h.stats()["windows"]
            self.m.window(rows, w, epoch)
            self.m0.append(rows, w, epoch)
            self.wins.append((rows, recs))
        return rows

    def check(self, tier, k):
        exp, exp_info = self.m.rollup(tier, k)
        got, info = self.h.rollup_tier(tier, k)
        assert info == exp_info, (tier, k, info, exp_info)
        assert got.tobytes() == exp.tobytes(), explain_diff(got, exp)
        p, n, info_d = self.h.rollup_tier_device(tier, k)
        dev = self.h.d2h(p, n, abi.EDGE_OUT) if n else np.zeros(0, dtype=abi.EDGE_OUT)
        assert info_d == exp_info and dev.tobytes() == exp.tobytes()
        assert self.h.tier_state(tier) == self.m.state(tier), (tier, self.h.tier_state(tier), self.m.state(tier))
        return got, info

    def check_all(self, ks=(1, 2, 3)):
        for t in range(1, len(self.m.tiers) + 1):
            for k in ks:
                self.check(t, k)

    def close(self):
        self.h.close()


def covered_records(r, info):
    """the records of the windows a rollup covered (alz_stats.windows numbers them from 1)"""
    return np.concatenate([np.zeros(0, dtype=abi.L7_REC)] +
                          [rec for _, rec in r.wins[info["window_first"] - 1: info["window_last"]] if rec is not None])


# ---- constructed merge layouts ----------------------------------------------------------------------------------
MERGE_LAYOUTS = dict(LAYOUTS)
MERGE_LAYOUTS.update({
    "empty_block": [[], [0, 1, 2], [], []],                 # a window merged into an empty block, and back
    "empty_window": [[0, 5, 11], [], [3, 7], []],
    "first_key_only": [[0, 1, 2], [0], [0, 9, 10], [0]],    # the match is the block's first key
    "last_key_only": [[9, 10, 11], [11], [0, 1, 11], [11]],  # the match is the block's last key
    "all_kinds": [list(range(N_KEYS)), [11, 10, 6, 4], list(range(0, N_KEYS, 2)), [1, 3, 5, 7, 8, 9]],
})


@pytest.mark.parametrize("layout", sorted(MERGE_LAYOUTS))
def test_constructed_merge_layouts(layout):
    rng = np.random.default_rng(12)
    r = Tiers([(2, 4, 64, 16), (2, 2, 64, 16)], TABLES)
    for idx in MERGE_LAYOUTS[layout]:
        recs = spec_records(idx, rng) if idx else None
        if recs is not None:
            r.h.submit(recs)
        r.flush(recs=recs)
        r.check_all()
    for tier, k in ((1, 1), (1, 2), (2, 1)):
        got, info = r.check(tier, k)
        assert info["windows"] == 2 * k * tier
        exp = by_key(oracle_edges(TABLES, covered_records(r, info), [HOST_ID]))
        assert same_rows(got, exp), explain_diff(got, exp)
    r.close()


def test_lat_sum_wraps_past_2_64_across_a_block():
    rng = np.random.default_rng(1)
    r = Tiers([(2, 2, 8, 8)], TABLES)
    for dur in ((1 << 63) + 5, (1 << 63) + 6):
        recs = records(np.array([PA], np.uint64), np.array([SV], np.uint64), rng)
        recs["duration_ns"] = dur
        r.h.submit(recs)
        r.flush()
    got, _ = r.check(1, 1)
    assert len(got) == 1 and int(got[0]["lat_sum_ns"]) == 11 and int(got[0]["count"]) == 2
    assert int(got[0]["hist"][abi.NB - 1]) == 2
    r.close()


# ---- what feeds tier 1 ------------------------------------------------------------------------------------------
def window_of(r, idx, rng, **kw):
    if idx:
        r.h.submit(spec_records(idx, rng, per=2))
    return r.flush(**kw)


def test_zero_row_windows_and_kept_windows():
    rng = np.random.default_rng(3)
    r = Tiers([(3, 4, 64, 16)], TABLES)
    window_of(r, [], rng)
    r.h.submit(spec_records([0, 1, 2], rng))
    r.flush(cap=2, expect=abi.E_CAPACITY)                          # too small: the window stays, feeds nothing
    assert r.h.tier_state(1) == dict(entries=0, open_windows=1, dropped=0)
    r.flush()
    window_of(r, [], rng)
    assert r.h.tier_state(1) == dict(entries=1, open_windows=0, dropped=0)
    got, info = r.check(1, 1)
    assert info["windows"] == 3 and info["rows_in"] == 3 and int(got["count"].sum()) == 15
    r.close()


def test_windows_consumed_with_capacity_feed_tier_1():
    rng = np.random.default_rng(4)
    r = Tiers([(2, 3, 1 << 12, 1 << 12)], [(abi.TABLE_POD, POD_NET + np.arange(64), np.arange(64))], max_pairs=1 << 12,
              max_edges=16)
    src = POD_NET + rng.integers(0, 64, 400).astype(np.uint64)
    dst = (0x08000000 + np.arange(400)).astype(np.uint64)
    r.h.submit(records(src[:200], dst[:200], rng))
    rows = r.flush(expect=abi.E_CAPACITY)                          # more edges than max_edges
    assert len(rows) == 16
    r.h.submit(records(src[200:208], dst[200:208], rng))
    r.flush()
    r.check(1, 1)
    r.close()


# ---- tier bookkeeping -------------------------------------------------------------------------------------------
def test_block_rows_overflow_drops_and_clears_the_tiers_above():
    rng = np.random.default_rng(5)
    r = Tiers([(2, 8, 64, 4), (2, 8, 64, 64), (2, 8, 64, 64)], TABLES)
    for _ in range(8):
        window_of(r, [0, 1], rng)                                  # 2 distinct rows per block
    r.check_all((1, 4))
    assert [r.h.tier_state(t)["entries"] for t in (1, 2, 3)] == [4, 2, 1]
    window_of(r, [0, 1, 2], rng)
    window_of(r, [3, 4], rng)                                      # 5 distinct rows > 4: dropped, tier 1 cleared
    assert r.h.tier_state(1) == dict(entries=0, open_windows=0, dropped=1)
    for _ in range(6):
        window_of(r, [5], rng)
        r.check_all((1, 2))
    assert [r.h.tier_state(t)["dropped"] for t in (1, 2, 3)] == [1, 1, 1]
    r.check_all((1, 5))
    r.close()


def test_arena_overflow_drops_and_clears_the_tiers_above():
    rng = np.random.default_rng(6)
    r = Tiers([(2, 8, 4, 64), (2, 8, 64, 64)], TABLES)
    for idx in ([0], [1], [2], [3], [0, 1, 2], [3, 4], [5], [6]):   # the third block has 5 rows > arena of 4
        window_of(r, idx, rng)
        r.check_all((1, 3))
    # tier 2 retained windows 1..4, then the block of windows 5..8 contained the dropped block: cleared
    assert r.h.tier_state(1)["dropped"] == 1 and r.h.tier_state(2) == dict(entries=0, open_windows=0, dropped=1)
    r.close()


def test_ring_eviction_per_tier():
    rng = np.random.default_rng(7)
    r = Tiers([(2, 3, 7, 16), (2, 2, 9, 16)], TABLES)
    for i in range(14):
        window_of(r, [i % N_KEYS, (i + 3) % N_KEYS], rng)
        r.check_all((1, 2, 4))
    r.close()


def test_tiers_and_window_history_are_independent_in_either_order():
    rng = np.random.default_rng(8)
    for order in ("tiers_first", "history_first"):
        r = Tiers([], TABLES)
        if order == "tiers_first":
            r.configure([(2, 4, 64, 16)])
        else:
            r.history(4, 64)
        window_of(r, [0, 1], rng)
        if order == "tiers_first":
            r.history(4, 64)
        else:
            r.configure([(2, 4, 64, 16)])
        for idx in ([2], [3, 4], [5]):
            window_of(r, idx, rng)
        r.check_all((1, 2))
        exp, info = r.m0.rollup(3)
        got, ginfo = r.h.rollup(3)
        assert got.tobytes() == exp.tobytes() and ginfo == info
        assert r.h.rollup_tier(0, 3)[0].tobytes() == exp.tobytes()   # tier 0 is alz_window_rollup
        r.history(0, 0)                                            # the history off: the tiers stay
        r.check_all((1, 2))
        r.history(2, 8)
        r.configure([])                                            # the tiers off: the history stays
        window_of(r, [6], rng)
        assert r.h.rollup(1)[0].tobytes() == r.m0.rollup(1)[0].tobytes()
        rc, _, _, _ = rollup_raw(r.h, 1, 4)
        assert rc == abi.OK
        r.close()


def test_bad_values_and_states():
    r = Tiers([], TABLES)
    L, h = r.h.L, r.h
    with pytest.raises(capi.AlzError) as e:
        h.rollup_tier(1, 1)
    assert e.value.status == abi.E_STATE
    for bad in ([(1, 4, 64, 16)], [(2, 0, 64, 16)], [(2, 4, 0, 16)], [(2, 4, 64, 0)], [(2, 4, 1 << 31, 16)],
                [(2, 4, 64, 1 << 31)], [(2, 4, 64, 16)] * 5,
                [(1 << 16, 1, 64, 16), (1 << 16, 1, 64, 16)],          # an entry of 2^32 windows
                [(2, 1 << 31, 64, 16)]):                                 # retained entries covering 2^32 windows
        with pytest.raises(capi.AlzError) as e:
            h.window_history_tiers(bad)
        assert e.value.status == abi.E_INVAL
    with pytest.raises(capi.AlzError) as e:
        h.tier_state(1)
    assert e.value.status == abi.E_STATE                           # a refused call leaves the tiers off
    r.configure([(2, 4, 64, 16)])
    for tier, k in ((2, 1), (1, 0)):
        with pytest.raises(capi.AlzError) as e:
            h.rollup_tier(tier, k)
        assert e.value.status == abi.E_INVAL
    with pytest.raises(capi.AlzError) as e:
        h.tier_state(0)
    assert e.value.status == abi.E_INVAL
    r.close()


def test_a_rollup_reads_only_and_reconfiguration():
    rng = np.random.default_rng(9)
    cfg = [(3, 4, 64, 32), (2, 4, 64, 32)]
    r = Tiers(cfg, TABLES)
    for i in range(7):
        window_of(r, [i, i + 1], rng)
    before = [r.h.tier_state(t) for t in (1, 2)]
    a = [r.check(t, 4)[0].tobytes() for t in (1, 2)]
    b = [r.check(t, 4)[0].tobytes() for t in (1, 2)]               # again: nothing moved
    assert a == b and [r.h.tier_state(t) for t in (1, 2)] == before
    for i in range(5):                                              # the open blocks were not touched either
        window_of(r, [i], rng)
        r.check_all((1, 4))
    r.configure(cfg)                                               # the same values: nothing changes
    r.check_all((1, 4))
    r.configure([(2, 4, 64, 32)])                                  # other values: everything dropped
    assert r.h.tier_state(1) == dict(entries=0, open_windows=0, dropped=0)
    for i in range(3):
        window_of(r, [i], rng)
        r.check_all((1, 2))
    r.close()


# ---- clocks and threads -----------------------------------------------------------------------------------------
def test_epochs_under_a_window_clock():
    rng = np.random.default_rng(10)
    fk, fu, W = 1000, 5_000_000, 1_000_000
    r = Tiers([(2, 4, 64, 16), (2, 2, 64, 16)], TABLES, max_batch=1 << 12)
    r.h.window_clock(fk, fu, W)
    e0 = (fu - fk + 10_000) // W

    def at(idx, epoch):
        recs = spec_records(idx, rng, per=3)
        recs["write_time_ns"] = 10_000 + (epoch - e0) * W + np.arange(len(recs))
        return recs

    for i in range(4):
        r.h.submit(at([i], e0 + i))
        r.flush(epoch=e0 + i)
        r.check_all((1, 2))
    got, info = r.check(2, 1)
    assert info == dict(windows=4, clocked=1, window_first=1, window_last=4, epoch_first=e0, epoch_last=e0 + 3,
                        rows_in=4)
    r.h.window_clock(0, 0, 0)                                      # the clock goes off inside a block
    r.h.submit(at([6], e0 + 9))
    r.flush()
    r.h.submit(at([7], e0 + 9))
    r.flush()
    r.check_all((1, 2, 3))
    assert r.h.rollup_tier(1, 1)[1]["clocked"] == 0 and r.h.rollup_tier(1, 2)[1]["clocked"] == 0
    r.close()


def test_producers_submit_during_flushes_and_tier_rollups():
    t = ol.Topo(64, seed=3, mix=abi.MIX_ALL)
    h = capi.Handle(max_endpoints=4 * 4096, max_pairs=1 << 15)
    h.load_tables(t.pod_ip, t.svc_ip)
    h.window_history_tiers([(2, 64, 1 << 18, 1 << 15), (2, 64, 1 << 18, 1 << 15)])
    per, rounds, errs = 4000, 6, []
    stop = threading.Event()

    def producer(i):
        try:
            for j in range(rounds):
                h.submit(t.events((i * rounds + j) * per, per))
        except Exception as ex:   # noqa: BLE001
            errs.append(ex)

    def consumer():
        try:
            for _ in range(40):
                if stop.is_set():
                    break
                h.flush()
                for tier in (1, 2):
                    rows, info = h.rollup_tier(tier, 64)
                    assert info["rows_in"] >= len(rows)
        except Exception as ex:   # noqa: BLE001
            errs.append(ex)

    ps = [threading.Thread(target=producer, args=(i,)) for i in range(8)]
    c = threading.Thread(target=consumer)
    c.start()
    for p in ps:
        p.start()
    for p in ps:
        p.join()
    stop.set()
    c.join()
    assert not errs, errs
    h.flush()                                                      # what the producers submitted last
    while h.stats()["windows"] % 4:                                # close the open blocks with empty windows
        h.flush()
    st = h.stats()
    o = ol.Oracle()
    o.load_tables(t.pod_ip, t.svc_ip)
    o.process(t.events(0, 8 * rounds * per))
    exp = by_key(o.edges())
    o.close()
    for tier in (1, 2):
        rows, info = h.rollup_tier(tier, 64)
        assert info["windows"] == st["windows"] and info["window_first"] == 1, (tier, info, st)
        assert same_rows(rows, exp), explain_diff(rows, exp)
    h.close()
    t.close()


# ---- plans and sequences ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("flags", [0, abi.CFG_EAGER_JOIN, abi.CFG_NO_SMEM_CACHE])
def test_topo_stream_against_model_and_oracle(flags):
    t = ol.Topo(64, seed=5, mix=abi.MIX_ALL)
    per = 30_000
    r = Tiers([(2, 3, 1 << 16, 1 << 15), (3, 2, 1 << 16, 1 << 15)], max_endpoints=4 * 4096, max_pairs=1 << 15,
              flags=flags)
    r.h.load_tables(t.pod_ip, t.svc_ip)
    for w in range(12):
        recs = t.events(w * per, per)
        r.h.submit(recs)
        r.flush(path="device" if w % 2 else "host", recs=recs)
        r.check_all((1, 2, 5))
    for tier, k in ((1, 1), (1, 3), (2, 1), (2, 2)):
        got, info = r.check(tier, k)
        o = ol.Oracle()
        o.load_tables(t.pod_ip, t.svc_ip)
        o.process(covered_records(r, info))
        exp = by_key(o.edges())
        o.close()
        assert same_rows(got, exp), explain_diff(got, exp)
    r.close()
    t.close()


@pytest.mark.parametrize("seed", range(4))
def test_random_sequences_against_the_model(seed):
    rng = np.random.default_rng(200 + seed)

    def rand_tiers():
        return [(int(rng.integers(2, 4)), int(rng.integers(1, 4)), int(rng.integers(4, 30)), int(rng.integers(3, 13)))
                for _ in range(int(rng.integers(1, 4)))]

    r = Tiers(rand_tiers(), TABLES)
    for _ in range(80):
        op = rng.choice(["submit", "submit", "flush", "flush", "flush", "small", "rollup", "commit", "tiers"])
        if op == "submit":
            idx = rng.choice(N_KEYS, int(rng.integers(1, N_KEYS + 1)), replace=False).tolist()
            r.h.submit(spec_records(idx, rng, per=int(rng.integers(1, 4))))
        elif op == "flush":
            r.flush(path=str(rng.choice(["host", "device"])))
        elif op == "small":
            rc, _, n = flush_raw(r.h, 0)                          # keeps a window that has rows, consumes an empty one
            if n == 0:
                assert rc == abi.OK
                r.m.window(np.zeros(0, dtype=abi.EDGE_OUT), r.h.stats()["windows"])
        elif op == "rollup":
            tier = int(rng.integers(1, len(r.m.tiers) + 1))
            r.check(tier, int(rng.integers(1, 6)))
        elif op == "commit":
            ip = int(rng.choice([PA, PB, PC]))
            r.h.upsert(abi.TABLE_POD, ip, int(rng.integers(0, 1 << 29)))
            r.h.commit()
        else:
            r.configure(rand_tiers())
    r.flush()
    r.check_all((1, 2, 5))
    r.close()


# ---- no cost when off -------------------------------------------------------------------------------------------
def test_no_tiers_add_no_kernel_to_a_flush():
    t = ol.Topo(32, seed=9, mix=abi.MIX_ALL)
    n = []
    for mode in ("never", "configured_then_off"):
        h = capi.Handle(max_endpoints=4 * 4096, max_pairs=1 << 14)
        h.load_tables(t.pod_ip, t.svc_ip)
        if mode != "never":
            h.window_history_tiers([(2, 4, 1 << 14, 1 << 14)])
            h.window_history_tiers([])
        for w in range(3):
            h.submit(t.events(w * 5000, 5000))
            h.flush()
        n.append(h.stats()["kernel_launches"])
        h.close()
    assert n[0] == n[1]
    t.close()
