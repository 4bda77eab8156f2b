"""GPU: span rollups (alz_window_rollup_span*, docs/SPEC.md §14) against the sequential model of tests/span_model.py.
Every span is compared with the model byte for byte, order included, and alz_span_info field by field, so the plan
the device made (which pieces, hence rows_in, entries and open_blocks) is checked as well as the rows; where the
tables stand still also with one oracle over all events of the covered windows."""
import ctypes as C
import threading

import numpy as np
import pytest

import oracle_lib as ol
from alaz_b200 import abi, capi
from helpers import explain_diff
from span_model import AT_LEAST, AT_MOST, SpanModel
from test_gpu_flush import flush_device_raw, flush_raw, oracle_edges, records
from test_gpu_rollup import HOST_ID, LAYOUTS, N_KEYS, PA, SV, TABLES, by_key, same_rows, spec_records

pytestmark = pytest.mark.gpu

MODES = (AT_MOST, AT_LEAST)


def span_raw(h, N, mode, cap):
    """alz_window_rollup_span with the status instead of an exception: (status, n_out, info)."""
    out = np.zeros(max(cap, 1), dtype=abi.EDGE_OUT)
    n, info = C.c_size_t(0), abi.SpanInfo()
    rc = h.L.alz_window_rollup_span(h.h, int(N), int(mode), out.ctypes.data_as(C.c_void_p) if cap else None, cap,
                                    C.byref(n), C.byref(info))
    return rc, n.value, info.as_dict()


class Span:
    """A handle and the model, driven together: every flush that consumes its window feeds the model with the rows
    the flush returned."""

    def __init__(self, tiers=(), history=None, tables=TABLES, **kw):
        kw.setdefault("max_endpoints", 1 << 14)
        kw.setdefault("max_pairs", 1 << 14)
        self.h = capi.Handle(**kw)
        self.m = SpanModel()
        for tab, ips, ids in tables:
            self.h.upsert_batch(tab, np.asarray(ips, np.uint32), np.asarray(ids, np.uint32))
        self.h.commit()
        if history:
            self.history(*history)
        if tiers:
            self.configure(tiers)
        self.wins = {}   # alz_stats.windows -> records of that window (None: not kept)

    def configure(self, tiers):
        self.h.window_history_tiers(tiers)
        self.m.configure(tiers)

    def history(self, depth, arena_rows):
        self.h.window_history(depth, arena_rows)
        self.m.history(depth, arena_rows)

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
            self.wins[w] = recs
        return rows

    def window(self, idx, rng, per=2, **kw):
        recs = spec_records(idx, rng, per=per) if idx else None
        if recs is not None:
            self.h.submit(recs)
        return self.flush(recs=recs, **kw)

    def check(self, N, mode=AT_MOST):
        exp, exp_info = self.m.span(N, mode)
        got, info = self.h.rollup_span(N, mode)
        assert info == exp_info, (N, mode, info, exp_info)
        assert got.tobytes() == exp.tobytes(), explain_diff(got, exp)
        p, n, info_d = self.h.rollup_span_device(N, mode)
        dev = self.h.d2h(p, n, abi.EDGE_OUT) if n else np.zeros(0, dtype=abi.EDGE_OUT)
        assert info_d == exp_info and dev.tobytes() == exp.tobytes()
        return got, info

    def check_all(self, extra=2):
        """every N up to past what is retained, in both modes"""
        W = self.h.stats()["windows"]
        for N in range(1, W + 1 + extra):
            for mode in MODES:
                self.check(N, mode)

    def covered_records(self, info):
        recs = [self.wins[w] for w in range(info["window_first"], info["window_last"] + 1)]
        return np.concatenate([np.zeros(0, dtype=abi.L7_REC)] + [r for r in recs if r is not None])

    def close(self):
        self.h.close()


# ---- constructed layouts, spans at block boundaries ---------------------------------------------------------------
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_constructed_layouts_every_span_against_model_and_oracle(layout):
    rng = np.random.default_rng(31)
    r = Span([(2, 4, 64, 16), (2, 2, 64, 16)], history=(3, 64))
    for idx in LAYOUTS[layout] * 2:
        r.window(idx, rng)
        r.check_all()
    for N in (1, 2, 3, 4, 5, 7, 8):   # tier boundaries of (2, 2) at 2, 4, 8; each ± 1
        got, info = r.check(N, AT_LEAST)
        exp = by_key(oracle_edges(TABLES, r.covered_records(info), [HOST_ID]))
        assert same_rows(got, exp), explain_diff(got, exp)
    r.close()


def test_history_only_equals_the_window_rollup():
    rng = np.random.default_rng(32)
    r = Span(history=(5, 64))
    for i in range(8):
        r.window([i % N_KEYS, (i + 5) % N_KEYS], rng)
    r.check_all()
    for N in range(1, 6):
        got, info = r.h.rollup_span(N)
        exp, einfo = r.h.rollup(N)
        assert got.tobytes() == exp.tobytes() and {k: info[k] for k in einfo} == einfo
        assert info["entries"] == [N, 0, 0, 0, 0] and info["open_blocks"] == 0
    r.close()


def test_tiers_only_and_both_reach_now():
    rng = np.random.default_rng(33)
    for history in (None, (4, 64)):
        r = Span([(3, 4, 64, 32), (2, 3, 64, 32)], history=history)
        for i in range(16):
            r.window([i % N_KEYS], rng)
            r.check_all(extra=3)
        # windows 13..16: tier 1's open block holds 16 (the last block closed at 15) and tier 2's holds 13..15
        _, info = r.check(4, AT_MOST)
        assert info["windows"] == 4 and info["window_last"] == 16 and info["open_blocks"] & 2
        r.close()


# ---- open blocks left out --------------------------------------------------------------------------------------
def test_open_blocks_empty_poisoned_and_overflowed():
    rng = np.random.default_rng(34)
    r = Span([(3, 8, 64, 4), (3, 8, 64, 64)], history=(8, 64))
    r.window([0], rng)
    r.window([1], rng)
    r.window([2], rng)                                          # tier 1 closes: its open block has no input
    assert r.check(1)[1]["open_blocks"] == 0
    r.check_all()
    r.window([3, 4, 5], rng)
    r.window([6, 7], rng)                                       # 5 distinct rows > 4: tier 1's block overflowed
    assert r.m.mt.tiers[0].overflow
    r.check_all()
    _, info = r.check(2)
    assert info["open_blocks"] == 0 and info["entries"][0] == 2  # the window history takes over
    r.window([8], rng)                                          # dropped: tier 2's open block is poisoned
    assert r.m.mt.tiers[1].poisoned and r.h.tier_state(1)["dropped"] == 1
    for i in range(4):
        r.window([i], rng)
        r.check_all()
    r.close()


# ---- gaps ----------------------------------------------------------------------------------------------------------
def test_dropped_blocks_and_ring_eviction_leave_gaps():
    rng = np.random.default_rng(35)
    # tier 1's arena holds 2 entries of ~4 rows; the window history holds 2 windows
    r = Span([(2, 8, 9, 8), (3, 2, 64, 64)], history=(2, 64))
    for i in range(10):
        r.window([i % N_KEYS, (i + 1) % N_KEYS], rng)
        r.check_all(extra=4)
    r.window(list(range(9)), rng)                               # 9 distinct rows > block_rows 8: window 11's block
    r.window([0], rng)                                          # is dropped when it closes, and so is tier 2's
    r.check_all(extra=4)
    W = r.h.stats()["windows"]
    _, info = r.check(W, AT_LEAST)
    assert info["windows"] < W                                  # the gaps: less than asked, and said so
    r.close()


def test_past_everything_retained():
    rng = np.random.default_rng(36)
    r = Span([(2, 2, 64, 16)], history=(2, 64))
    for i in range(7):
        r.window([i], rng)
    for N in (8, 100, 1 << 32, (1 << 64) - 1):
        for mode in MODES:
            _, info = r.check(N, mode)
            assert info["windows"] == 5                         # tier 1 keeps [3, 4], [5, 6]; 7 is in its open block
    r.close()


# ---- the sums --------------------------------------------------------------------------------------------------
def test_sums_wrap_across_pieces():
    rng = np.random.default_rng(37)
    r = Span([(2, 4, 8, 8)], history=(4, 8))
    for dur in ((1 << 63) + 5, (1 << 63) + 6, 7):
        recs = records(np.array([PA], np.uint64), np.array([SV], np.uint64), rng)
        recs["duration_ns"] = dur
        r.h.submit(recs)
        r.flush(recs=recs)
    got, info = r.check(3)
    assert info["entries"] == [0, 1, 0, 0, 0] and info["open_blocks"] == 2
    assert len(got) == 1 and int(got[0]["lat_sum_ns"]) == 18 and int(got[0]["count"]) == 3
    r.close()


# ---- clocks ----------------------------------------------------------------------------------------------------
def test_epochs_under_a_window_clock():
    rng = np.random.default_rng(38)
    fk, fu, Wn = 1000, 5_000_000, 1_000_000
    r = Span([(2, 4, 64, 16), (2, 2, 64, 16)], history=(2, 64), max_batch=1 << 12)
    r.h.window_clock(fk, fu, Wn)
    e0 = (fu - fk + 10_000) // Wn

    def at(idx, epoch):
        recs = spec_records(idx, rng, per=3)
        recs["write_time_ns"] = 10_000 + (epoch - e0) * Wn + np.arange(len(recs))
        return recs

    for i in range(5):
        recs = at([i], e0 + i)
        r.h.submit(recs)
        r.flush(epoch=e0 + i, recs=recs)
        r.check_all()
    _, info = r.check(5)
    assert info["clocked"] == 1 and (info["epoch_first"], info["epoch_last"]) == (e0, e0 + 4)
    r.h.window_clock(0, 0, 0)                                   # the clock goes off inside a block
    recs = at([6], e0 + 9)
    r.h.submit(recs)
    r.flush(recs=recs)
    r.check_all()
    assert r.h.rollup_span(1)[1]["clocked"] == 0 and r.h.rollup_span(3)[1]["clocked"] == 0
    r.close()


# ---- reads only ------------------------------------------------------------------------------------------------
def test_a_span_reads_only_against_a_twin_handle():
    rng = np.random.default_rng(39)
    cfg = [(3, 4, 64, 32), (2, 4, 64, 32)]
    a, b = Span(cfg, history=(4, 64)), Span(cfg, history=(4, 64))
    for i in range(8):
        recs = spec_records([i % N_KEYS, (i + 2) % N_KEYS], rng)
        for r in (a, b):
            r.h.submit(recs)
            r.flush(recs=recs)
        if i % 3 == 1:                                          # earlier rollups' device rows stay valid
            p0, n0, _ = a.h.rollup_device(3)
            rows0 = a.h.d2h(p0, n0, abi.EDGE_OUT).tobytes()
            p1, n1, _ = a.h.rollup_tier_device(1, 2)
            assert a.h.d2h(p0, n0, abi.EDGE_OUT).tobytes() == rows0   # a tier rollup leaves the window rollup's
            rows1 = a.h.d2h(p1, n1, abi.EDGE_OUT).tobytes()
            p0, n0, _ = a.h.rollup_device(1)
            assert a.h.d2h(p1, n1, abi.EDGE_OUT).tobytes() == rows1   # and a window rollup the tier rollup's
            before = (a.h.d2h(p0, n0, abi.EDGE_OUT).tobytes(), rows1)
            a.check_all()
            assert (a.h.d2h(p0, n0, abi.EDGE_OUT).tobytes(), a.h.d2h(p1, n1, abi.EDGE_OUT).tobytes()) == before
    recs = spec_records([0, 5, 9], rng)
    for r in (a, b):
        r.h.submit(recs)
        r.flush()
    assert a.h.stats()["windows"] == b.h.stats()["windows"]
    for tier in (1, 2):
        assert a.h.tier_state(tier) == b.h.tier_state(tier)
        for k in (1, 4):
            (ra, ia), (rb, ib) = a.h.rollup_tier(tier, k), b.h.rollup_tier(tier, k)
            assert ra.tobytes() == rb.tobytes() and ia == ib
    for k in (1, 4):
        assert a.h.rollup(k)[0].tobytes() == b.h.rollup(k)[0].tobytes()
    for N in range(1, 12):                                      # the open blocks too
        assert a.h.rollup_span(N)[0].tobytes() == b.h.rollup_span(N)[0].tobytes()
    a.check_all()
    a.close()
    b.close()


def test_a_flush_enqueues_what_it_did_before():
    t = ol.Topo(32, seed=9, mix=abi.MIX_ALL)
    per_flush = []
    for spans in (False, True):
        h = capi.Handle(max_endpoints=4 * 4096, max_pairs=1 << 14)
        h.load_tables(t.pod_ip, t.svc_ip)
        h.window_history(4, 1 << 14)
        h.window_history_tiers([(2, 4, 1 << 14, 1 << 14), (2, 4, 1 << 14, 1 << 14)])
        d = []
        for w in range(6):
            h.submit(t.events(w * 5000, 5000))
            before = h.stats()["kernel_launches"]
            h.flush()
            d.append(h.stats()["kernel_launches"] - before)
            if spans:
                h.rollup_span(w + 1)
                h.rollup_span(3, AT_LEAST)
        per_flush.append(d)
        h.close()
    assert per_flush[0] == per_flush[1]
    t.close()


def test_bad_values_and_states():
    rng = np.random.default_rng(40)
    r = Span()
    for N, mode in ((1, AT_MOST), (0, AT_MOST), (1, 2)):       # neither the history nor the tiers: ALZ_E_STATE
        assert span_raw(r.h, N, mode, 0)[0] == abi.E_STATE
    r.configure([(2, 4, 64, 16)])
    for N, mode in ((0, AT_MOST), (0, AT_LEAST), (1, 2), (1, 0xFFFFFFFF)):
        assert span_raw(r.h, N, mode, 0)[0] == abi.E_INVAL
    rc, n, info = span_raw(r.h, 3, AT_MOST, 0)                 # nothing consumed yet: an empty span
    assert rc == abi.OK and n == 0 and info["windows"] == 0
    for i in range(3):
        r.window([i, i + 1], rng)
    exp, einfo = r.m.span(3, AT_MOST)
    rc, n, info = span_raw(r.h, 3, AT_MOST, 1)                 # too small: n_out set, nothing written
    assert rc == abi.E_CAPACITY and n == len(exp) and info == einfo
    r.check_all()
    r.configure([])
    assert span_raw(r.h, 3, AT_MOST, 0)[0] == abi.E_STATE
    r.history(2, 64)
    r.window([0], rng)
    r.check_all()
    r.close()


# ---- threads ---------------------------------------------------------------------------------------------------
def test_producers_submit_while_a_thread_flushes_and_queries():
    t = ol.Topo(64, seed=3, mix=abi.MIX_ALL)
    h = capi.Handle(max_endpoints=4 * 4096, max_pairs=1 << 15)
    h.load_tables(t.pod_ip, t.svc_ip)
    h.window_history(4, 1 << 17)
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
                for N, mode in ((3, AT_MOST), (1 << 20, AT_LEAST)):
                    rows, info = h.rollup_span(N, mode)
                    assert info["rows_in"] >= len(rows) and info["window_last"] == h.stats()["windows"]
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
    h.flush()                                                   # what the producers submitted last
    st = h.stats()
    o = ol.Oracle()
    o.load_tables(t.pod_ip, t.svc_ip)
    o.process(t.events(0, 8 * rounds * per))
    exp = by_key(o.edges())
    o.close()
    rows, info = h.rollup_span(st["windows"], AT_LEAST)
    assert info["windows"] == st["windows"] and info["window_first"] == 1, (info, st)
    assert same_rows(rows, exp), explain_diff(rows, exp)
    h.close()
    t.close()


# ---- streams and sequences -------------------------------------------------------------------------------------
def test_topo_stream_against_model_and_oracle():
    t = ol.Topo(64, seed=5, mix=abi.MIX_ALL)
    per = 30_000
    r = Span([(2, 3, 1 << 16, 1 << 15), (3, 2, 1 << 16, 1 << 15)], history=(3, 1 << 16), tables=(),
             max_endpoints=4 * 4096, max_pairs=1 << 15)
    r.h.load_tables(t.pod_ip, t.svc_ip)
    for w in range(14):
        recs = t.events(w * per, per)
        r.h.submit(recs)
        r.flush(path="device" if w % 2 else "host", recs=recs)
        for N in (1, 2, 5, 6, 7, 13):
            r.check(N, AT_MOST)
            r.check(N, AT_LEAST)
    for N in (4, 9, 14):
        got, info = r.check(N, AT_LEAST)
        o = ol.Oracle()
        o.load_tables(t.pod_ip, t.svc_ip)
        o.process(r.covered_records(info))
        exp = by_key(o.edges())
        o.close()
        assert same_rows(got, exp), explain_diff(got, exp)
    r.close()
    t.close()


@pytest.mark.parametrize("seed", range(4))
def test_random_sequences_against_the_model(seed):
    rng = np.random.default_rng(300 + seed)

    def rand_tiers():
        return [(int(rng.integers(2, 4)), int(rng.integers(1, 4)), int(rng.integers(4, 30)), int(rng.integers(3, 13)))
                for _ in range(int(rng.integers(0, 4)))]

    r = Span(rand_tiers() or [(2, 2, 16, 8)], history=(int(rng.integers(1, 5)), int(rng.integers(4, 30))))
    for _ in range(80):
        op = rng.choice(["submit", "submit", "flush", "flush", "flush", "small", "span", "commit", "tiers", "history"])
        if op == "submit":
            idx = rng.choice(N_KEYS, int(rng.integers(1, N_KEYS + 1)), replace=False).tolist()
            r.h.submit(spec_records(idx, rng, per=int(rng.integers(1, 4))))
        elif op == "flush":
            r.flush(path=str(rng.choice(["host", "device"])))
        elif op == "small":
            rc, _, n = flush_raw(r.h, 0)                       # keeps a window that has rows, consumes an empty one
            if n == 0:
                assert rc == abi.OK
                r.m.window(np.zeros(0, dtype=abi.EDGE_OUT), r.h.stats()["windows"])
        elif op == "span":
            r.check(int(rng.integers(1, 12)), int(rng.choice(MODES)))
        elif op == "commit":
            r.h.upsert(abi.TABLE_POD, int(rng.choice([PA])), int(rng.integers(0, 1 << 29)))
            r.h.commit()
        elif op == "tiers":
            r.configure(rand_tiers())
        else:
            r.history(int(rng.integers(0, 5)), int(rng.integers(4, 30)))
        if r.h.stats()["windows"] and not (r.m.m0.depth or r.m.mt.tiers):
            r.configure([(2, 2, 16, 8)])                       # keep something on, so a span is defined
    r.flush()
    r.check_all()
    r.close()
