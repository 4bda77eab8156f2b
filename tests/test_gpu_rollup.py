"""GPU: rolling windows (alz_window_history, alz_window_rollup*, docs/SPEC.md §12) against the sequential model of
tests/rollup_model.py. Every rollup is compared with the model row for row, byte for byte, order included, and
alz_rollup_info field by field; where the tables stand still also with one oracle over the windows' events."""
import ctypes as C
import threading

import numpy as np
import pytest

import oracle_lib as ol
from alaz_b200 import abi, capi
from gnn_graphs import POD_NET, SVC_NET
from helpers import edges_equal, explain_diff
from rollup_model import RollupModel, packed_key
from test_gpu_flush import flush_device_raw, flush_raw, oracle_edges, records

pytestmark = pytest.mark.gpu


def by_key(rows):
    return rows[sorted(range(len(rows)), key=lambda i: packed_key(rows[i]))]


def same_rows(a, b):
    """Two edge lists equal row by row, every field, in this order (the oracle's rows carry no defined padding)."""
    return len(a) == len(b) and all(np.array_equal(a[f], b[f]) for f in
                                    ("from_type", "from", "to_type", "to", "count", "err5xx", "lat_sum_ns", "hist"))


def rollup_raw(h, k, cap):
    """alz_window_rollup with the status instead of an exception: (status, buffer, n_out, info)."""
    out = np.full(max(cap, 1), 0xAB, dtype=np.uint8).repeat(abi.EDGE_OUT.itemsize).view(abi.EDGE_OUT)
    n, info = C.c_size_t(0), abi.RollupInfo()
    rc = h.L.alz_window_rollup(h.h, k, out.ctypes.data_as(C.c_void_p) if cap else None, cap, C.byref(n), C.byref(info))
    return rc, out, n.value, info.as_dict()


def fetch(h):
    out = np.zeros(h.max_edges, dtype=abi.EDGE_OUT)
    n = C.c_size_t(0)
    h._ck(h.L.alz_window_fetch(h.h, out.ctypes.data_as(C.c_void_p), len(out), C.byref(n)), "alz_window_fetch")
    return out[: n.value].copy()


class Roll:
    """A handle and the model, driven together: every flush that consumes its window is appended to the model with
    the rows the flush returned."""

    def __init__(self, depth, arena_rows, tables=(), **kw):
        kw.setdefault("max_endpoints", 1 << 14)
        kw.setdefault("max_pairs", 1 << 14)
        self.h = capi.Handle(**kw)
        self.m = RollupModel()
        for tab, ips, ids in tables:
            self.h.upsert_batch(tab, np.asarray(ips, np.uint32), np.asarray(ids, np.uint32))
        self.h.commit()
        self.history(depth, arena_rows)
        self.flushed = []   # rows of every consumed window

    def history(self, depth, arena_rows):
        self.h.window_history(depth, arena_rows)
        self.m.history(depth, arena_rows)

    def flush(self, cap=None, path="host", epoch=None, expect=abi.OK):
        cap = self.h.max_edges if cap is None else cap
        if path == "host":
            rc, rows, n = flush_raw(self.h, cap)
        else:
            rc, rows = flush_device_raw(self.h)
            n = len(rows)
        assert rc == expect, rc
        if n <= cap:   # one rank: only a too-small buffer keeps the window
            self.m.append(rows, self.h.stats()["windows"], epoch)
            self.flushed.append(rows)
        return rows

    def check(self, k):
        exp, exp_info = self.m.rollup(k)
        got, info = self.h.rollup(k)
        assert info == exp_info, (info, exp_info)
        assert got.tobytes() == exp.tobytes(), explain_diff(got, exp)
        p, n, info_d = self.h.rollup_device(k)
        dev = self.h.d2h(p, n, abi.EDGE_OUT) if n else np.zeros(0, dtype=abi.EDGE_OUT)
        assert info_d == exp_info and dev.tobytes() == exp.tobytes()
        return got

    def close(self):
        self.h.close()


# ---- constructed key layouts ------------------------------------------------------------------------------------
PA, PB, PC = POD_NET + 1, POD_NET + 2, POD_NET + 3          # pod ids 0, 2^29 - 1, 7
SV = SVC_NET + 1                                             # service id 3
OUT_LO, OUT_HI = 1, 0xFFFFFFFF                               # outbound 0.0.0.1 and 255.255.255.255
HOST_ID = 1                                                  # a Host-keyed id equal to the outbound address 0.0.0.1
TABLES = [(abi.TABLE_POD, [PA, PB, PC], [0, (1 << 29) - 1, 7]), (abi.TABLE_SVC, [SV], [3])]
# (saddr, daddr, reversed, host-keyed): twelve distinct edges
SPECS = [(PA, SV, 0, 0), (PB, SV, 0, 0), (PA, SV, 1, 0), (PB, SV, 1, 0),            # pod -> svc, svc -> pod (reversed)
         (PA, OUT_LO, 0, 0), (PB, OUT_HI, 0, 0), (PA, OUT_HI, 1, 0), (PB, OUT_LO, 1, 0),   # outbound, both directions
         (PA, PB, 0, 0), (PB, PA, 0, 0),                                               # pod <-> pod, both directions
         (PC, PA, 1, 0),                                                               # reversed pod <-> pod: A -> C
         (PA, HOST_ID, 0, 1)]                                                          # Host-keyed
N_KEYS = len(SPECS)


def spec_records(idx, rng, per=5):
    s = [SPECS[i] for i in idx for _ in range(per)]
    a = np.array(s, dtype=np.uint64).reshape(-1, 4)
    return records(a[:, 0], a[:, 1], rng, reversed_=a[:, 2] != 0, host=a[:, 3] != 0)


LAYOUTS = {
    "identical": [list(range(N_KEYS))] * 4,
    "disjoint": [[0, 1, 2], [3, 4, 5], [6, 7, 8], [9, 10, 11]],
    "interleaved": [list(range(0, N_KEYS, 2)), list(range(1, N_KEYS, 2)), list(range(0, N_KEYS, 3)), [11, 0]],
    "only_oldest_only_newest": [[0, 5], [5], [5], [5, 11]],
}


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_constructed_key_layouts(layout):
    rng = np.random.default_rng(11)
    r = Roll(4, 64, TABLES)
    wins = [spec_records(idx, rng) for idx in LAYOUTS[layout]]
    for recs in wins:
        r.h.submit(recs)
        last = r.flush()
        assert r.check(1).tobytes() == last.tobytes()          # k = 1: the flush that preceded it, byte for byte
    for k in (2, 3, 4):
        got = r.check(k)
        exp = by_key(oracle_edges(TABLES, np.concatenate(wins[-k:]), [HOST_ID]))
        assert same_rows(got, exp), explain_diff(got, exp)
    assert len(r.check(4)) == len({i for idx in LAYOUTS[layout] for i in idx})
    r.close()


def test_lat_sum_wraps_past_2_64():
    rng = np.random.default_rng(1)
    r = Roll(2, 8, TABLES)
    for dur in ((1 << 63) + 5, (1 << 63) + 6):
        recs = records(np.array([PA], np.uint64), np.array([SV], np.uint64), rng)
        recs["duration_ns"] = dur
        r.h.submit(recs)
        r.flush()
    got = r.check(2)
    assert len(got) == 1 and int(got[0]["lat_sum_ns"]) == 11 and int(got[0]["count"]) == 2
    assert int(got[0]["hist"][abi.NB - 1]) == 2
    r.close()


# ---- Topo streams -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flags,packed", [(0, False), (abi.CFG_EAGER_JOIN, False), (abi.CFG_NO_SMEM_CACHE, False),
                                          (0, True)])
def test_topo_stream_against_model_and_oracle(flags, packed):
    t = ol.Topo(64, seed=5, mix=abi.MIX_ALL)
    depth, per = 6, 30_000
    r = Roll(depth, 1 << 16, max_endpoints=4 * 4096, max_pairs=1 << 15, flags=flags)
    r.h.load_tables(t.pod_ip, t.svc_ip)
    for w in range(depth + 3):
        ev = t.events(w * per, per)
        if packed:
            r.h.submit_packed(*capi.pack_l7(ev))
        else:
            r.h.submit(ev)
        last = r.flush(path="device" if w % 2 else "host")
        assert r.check(1).tobytes() == last.tobytes()
    n_win = depth + 3
    for k in (2, 3, depth, depth + 5):
        got = r.check(k)
        kk = min(k, depth)
        o = ol.Oracle()
        o.load_tables(t.pod_ip, t.svc_ip)
        o.process(t.events((n_win - kk) * per, kk * per))
        exp = by_key(o.edges())
        o.close()
        assert same_rows(got, exp), explain_diff(got, exp)
    assert r.m.rollup(depth + 5)[1]["windows"] == depth
    r.close()
    t.close()


# ---- what is retained -------------------------------------------------------------------------------------------
def window_of(r, idx, rng):
    if idx:
        r.h.submit(spec_records(idx, rng, per=2))
    return r.flush()


def test_depth_arena_and_empty_windows():
    rng = np.random.default_rng(2)
    r = Roll(5, 10, TABLES)
    with pytest.raises(capi.AlzError) as e:
        r.h.rollup(0)
    assert e.value.status == abi.E_INVAL
    got, info = r.h.rollup(4)                                   # nothing retained yet
    assert len(got) == 0 and info["windows"] == 0 and info["rows_in"] == 0
    for idx in ([0, 1, 2, 3], [], [0, 4, 5, 6], [], [1, 2, 3]):      # 0-row windows between full ones
        window_of(r, idx, rng)
        for k in (1, 2, 3, 9):
            r.check(k)
    # the last one did not fit behind row 8: it starts at row 0 and evicts the first window before depth is reached
    assert [e["first_row"] for e in r.m.entries] == [4, 4, 8, 0]
    window_of(r, [7, 8, 9, 10], rng)                               # rows 3..6: the window at rows 4..7 and all before it go
    assert [e["n"] for e in r.m.entries] == [0, 3, 4]
    r.check(5)
    window_of(r, [0, 1, 2, 3, 4, 5], rng)                          # 6 rows: behind row 7 they would pass the end -> row 0, alone
    assert [(e["first_row"], e["n"]) for e in r.m.entries] == [(0, 6)]
    r.check(2)
    window_of(r, list(range(11)), rng)                             # 11 rows: larger than the arena
    assert r.m.entries == []
    for k in (1, 3):
        r.check(k)
    window_of(r, [5], rng)
    r.history(5, 10)                                               # the same values: nothing is dropped
    assert r.check(2)["count"].sum() == 2
    r.history(2, 12)
    assert len(r.check(2)) == 0
    window_of(r, [5, 6], rng)
    r.check(2)
    r.history(0, 0)                                                # off
    rc, _, _, _ = rollup_raw(r.h, 1, 4)
    assert rc == abi.E_STATE
    window_of(r, [5], rng)                                         # flushes go on as before
    L = r.h.L
    assert L.alz_window_history(r.h.h, 4, 1 << 32) == abi.E_INVAL
    assert L.alz_window_history(r.h.h, 4, 0) == abi.E_INVAL
    assert rollup_raw(r.h, 1, 4)[0] == abi.E_STATE                 # a refused call leaves the history off
    r.close()


def test_flush_that_keeps_its_window_appends_nothing():
    rng = np.random.default_rng(3)
    r = Roll(4, 64, TABLES)
    r.h.submit(spec_records([0, 1, 2], rng))
    r.flush(cap=2, expect=abi.E_CAPACITY)                          # too small: the window stays
    assert r.m.entries == [] and r.h.rollup(1)[1]["windows"] == 0
    r.flush()
    assert len(r.m.entries) == 1 and r.check(4)["count"].sum() == 15
    r.close()


def test_windows_that_lost_events_are_retained_as_returned():
    rng = np.random.default_rng(4)
    # more socket pairs than max_pairs: the flush returns ALZ_E_CAPACITY with the rows it has
    r = Roll(3, 1 << 12, [(abi.TABLE_POD, POD_NET + np.arange(64), np.arange(64))], max_pairs=256, max_edges=1 << 10)
    src = POD_NET + rng.integers(0, 64, 4000).astype(np.uint64)
    dst = (0x08000000 + np.arange(4000)).astype(np.uint64)
    r.h.submit(records(src, dst, rng))
    rows = r.flush(expect=abi.E_CAPACITY)
    assert 0 < len(rows) and r.h.stats()["capacity_events"] > 0
    assert r.check(1).tobytes() == rows.tobytes()
    r.close()
    # more edges than max_edges
    r = Roll(3, 1 << 12, [(abi.TABLE_POD, POD_NET + np.arange(64), np.arange(64))], max_pairs=1 << 12, max_edges=16)
    r.h.submit(records(src[:200], dst[:200], rng))
    rows = r.flush(expect=abi.E_CAPACITY)
    assert len(rows) == 16 and r.check(1).tobytes() == rows.tobytes()
    r.h.submit(records(src[:8], dst[:8], rng))
    r.flush()
    r.check(2)
    r.close()


def test_table_commits_between_and_inside_windows():
    rng = np.random.default_rng(5)
    r = Roll(4, 64, TABLES)
    r.h.submit(spec_records([0, 4, 8], rng))
    r.flush()
    r.h.upsert(abi.TABLE_POD, PA, 9)                               # the address changes pod id between two windows
    r.h.commit()
    r.h.submit(spec_records([0, 4], rng))
    r.h.upsert(abi.TABLE_SVC, SV, 4)                               # and the service its id inside one
    r.h.commit()
    r.h.submit(spec_records([0, 1], rng))
    r.flush()
    got = r.check(2)
    froms = {(int(x["from"]), int(x["to_type"]), int(x["to"])) for x in got if x["from_type"] == abi.NODE_POD}
    assert {(0, abi.NODE_SVC, 3), (9, abi.NODE_SVC, 3), (9, abi.NODE_SVC, 4)} <= froms   # two nodes stay two rows
    assert int(got["count"].sum()) == sum(int(w["count"].sum()) for w in r.flushed)
    r.close()


def test_a_rollup_reads_only():
    rng = np.random.default_rng(6)
    t = ol.Topo(32, seed=9, mix=abi.MIX_ALL)
    r = Roll(4, 1 << 14, max_endpoints=4 * 4096)
    r.h.load_tables(t.pod_ip, t.svc_ip)
    for w in range(3):
        r.h.submit(t.events(w * 5000, 5000))
        r.flush()

    def scores():
        s = np.zeros(r.h.max_edges, dtype=np.float32)
        n = C.c_size_t(0)
        r.h._ck(r.h.L.alz_gnn_score(r.h.h, s.ctypes.data_as(C.c_void_p), len(s), C.byref(n)), "alz_gnn_score")
        return s[: n.value].copy()

    f0, s0 = fetch(r.h), scores()
    launches = r.h.stats()["kernel_launches"]
    ev = t.events(15000, 6000)
    r.h.submit(ev[:3000])                                          # half a window, a rollup, the other half
    full = r.check(3)
    assert r.h.stats()["kernel_launches"] > launches
    assert fetch(r.h).tobytes() == f0.tobytes() and scores().tobytes() == s0.tobytes()
    # a too-small buffer: the count, nothing written; the repeated call succeeds
    rc, buf, n, info = rollup_raw(r.h, 3, len(full) - 1)
    assert rc == abi.E_CAPACITY and n == len(full) and info["windows"] == 3
    assert np.all(buf.view(np.uint8) == 0xAB)
    rc, buf, n, _ = rollup_raw(r.h, 3, len(full))
    assert rc == abi.OK and buf[:n].tobytes() == full.tobytes()
    r.h.submit(ev[3000:])
    got = r.flush()
    o = ol.Oracle()
    o.load_tables(t.pod_ip, t.svc_ip)
    o.process(ev)
    assert edges_equal(got, o.edges()), explain_diff(got, o.edges())
    o.close()
    r.close()
    t.close()


def test_history_adds_no_kernel_to_a_flush():
    t = ol.Topo(32, seed=9, mix=abi.MIX_ALL)
    n = []
    for depth in (0, 4):
        h = capi.Handle(max_endpoints=4 * 4096, max_pairs=1 << 14)
        h.load_tables(t.pod_ip, t.svc_ip)
        if depth:
            h.window_history(depth, 1 << 14)
        for w in range(3):
            h.submit(t.events(w * 5000, 5000))
            h.flush()
        n.append(h.stats()["kernel_launches"])
        h.close()
    assert n[0] == n[1]
    t.close()


# ---- window clock -----------------------------------------------------------------------------------------------
def test_epochs_under_a_window_clock():
    rng = np.random.default_rng(7)
    fk, fu, W = 1000, 5_000_000, 1_000_000
    r = Roll(4, 64, TABLES, max_batch=1 << 12)
    r.h.window_clock(fk, fu, W)
    e0 = (fu - fk + 10_000) // W

    def at(idx, epoch, off=0):
        recs = spec_records(idx, rng, per=3)
        recs["write_time_ns"] = 10_000 + (epoch - e0) * W + off + np.arange(len(recs))
        return recs

    r.h.submit(at([0, 1], e0))
    r.h.submit(at([2, 3], e0 + 1))                                 # set aside; the roll re-ingests them
    assert r.h.window_epoch() == e0
    r.flush(epoch=e0)
    r.h.submit(at([4], e0, off=500))                               # late: reduced into the open window e0 + 1
    r.flush(epoch=e0 + 1)
    assert r.h.stats()["late_events"] == 3
    got = r.check(2)
    assert r.m.rollup(2)[1] == dict(windows=2, clocked=1, window_first=1, window_last=2, epoch_first=e0,
                                    epoch_last=e0 + 1, rows_in=5)
    assert int(got["count"].sum()) == 15
    r.h.submit(at([5], e0 + 2))
    r.flush(epoch=e0 + 2)
    r.check(3)
    r.h.window_clock(0, 0, 0)                                      # the clock goes off inside the span
    r.h.submit(at([6], e0 + 9))
    r.flush()
    r.check(2)
    assert r.m.rollup(2)[1]["clocked"] == 0
    assert r.h.rollup(1)[1]["clocked"] == 0 and r.h.rollup(4)[1]["clocked"] == 0
    r.close()


# ---- threads ----------------------------------------------------------------------------------------------------
def test_producers_submit_while_another_thread_flushes_and_rolls_up():
    t = ol.Topo(64, seed=3, mix=abi.MIX_ALL)
    h = capi.Handle(max_endpoints=4 * 4096, max_pairs=1 << 15)
    h.load_tables(t.pod_ip, t.svc_ip)
    h.window_history(64, 1 << 18)
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
            for _ in range(40):   # at most 41 windows: all of them stay in the history
                if stop.is_set():
                    break
                h.flush()
                rows, info = h.rollup(64)
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
    h.flush()
    rows, info = h.rollup(64)
    st = h.stats()
    assert info["windows"] == st["windows"] <= 64, (info, st)
    assert int(rows["count"].sum()) == st["rows_emitted"] and st["events_in"] == 8 * rounds * per
    o = ol.Oracle()
    o.load_tables(t.pod_ip, t.svc_ip)
    o.process(t.events(0, 8 * rounds * per))
    exp = by_key(o.edges())
    assert same_rows(rows, exp), explain_diff(rows, exp)
    o.close()
    h.close()
    t.close()


# ---- random sequences -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(4))
def test_random_sequences_against_the_model(seed):
    rng = np.random.default_rng(100 + seed)
    r = Roll(int(rng.integers(1, 5)), int(rng.integers(6, 30)), TABLES)
    ids = {PA: 0, PB: (1 << 29) - 1, PC: 7}
    for _ in range(60):
        op = rng.choice(["submit", "submit", "flush", "flush", "small", "rollup", "commit", "history"])
        if op == "submit":
            idx = rng.choice(N_KEYS, int(rng.integers(1, N_KEYS + 1)), replace=False).tolist()
            r.h.submit(spec_records(idx, rng, per=int(rng.integers(1, 4))))
        elif op == "flush":
            r.flush(path=str(rng.choice(["host", "device"])))
        elif op == "small":
            rc, _, n = flush_raw(r.h, 0)                          # keeps a window that has rows, consumes an empty one
            if n == 0:
                assert rc == abi.OK
                r.m.append(np.zeros(0, dtype=abi.EDGE_OUT), r.h.stats()["windows"])
        elif op == "rollup":
            r.check(int(rng.integers(1, 7)))
        elif op == "commit":
            ip = int(rng.choice([PA, PB, PC]))
            ids[ip] = int(rng.integers(0, 1 << 29))
            r.h.upsert(abi.TABLE_POD, ip, ids[ip])
            r.h.commit()
        else:
            r.history(int(rng.integers(1, 5)), int(rng.integers(6, 30)))
    r.flush()
    for k in (1, 2, 5):
        r.check(k)
    r.close()
