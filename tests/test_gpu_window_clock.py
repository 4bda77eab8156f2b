"""GPU: time-cut windows (alz_window_clock, docs/SPEC.md §8) against the sequential model of tests/window_model.py.
Every flush is compared per edge, bit for bit, and the stats after every operation."""
import ctypes as C
import threading

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings, strategies as st

import oracle_lib as ol
from alaz_b200 import abi, capi
from helpers import edges_equal, explain_diff
from test_gpu_flush import flush_device_raw, flush_raw
from test_gpu_ingest import to_raw
from window_model import WindowModel

pytestmark = pytest.mark.gpu

M64 = 1 << 64
PODS = [abi.ip(f"10.0.0.{k}") for k in range(1, 9)]          # pod ids 1..8
SVCS = [abi.ip(f"172.16.0.{k}") for k in range(1, 4)]        # service ids 11..13
STRANGERS = [abi.ip("10.0.9.1"), abi.ip("10.0.9.2")]          # neither pod nor service
ADDRS = PODS + SVCS + STRANGERS
PROTOS = [abi.PROTO_HTTP, abi.PROTO_HTTP, abi.PROTO_REDIS, abi.PROTO_AMQP, abi.PROTO_KAFKA, abi.PROTO_HTTP2,
          abi.PROTO_POSTGRES]


class Pair:
    """A handle and the model, driven together."""

    def __init__(self, fk, fu, W, max_batch=1 << 16, max_pairs=1 << 12):
        self.h = capi.Handle(max_endpoints=256, max_pairs=max_pairs, max_batch=max_batch)
        self.m = WindowModel(fk, fu, W, defer_cap=2 * max_batch)
        for k, ip in enumerate(PODS):
            self.upsert(abi.TABLE_POD, ip, k + 1)
        for k, ip in enumerate(SVCS):
            self.upsert(abi.TABLE_SVC, ip, k + 11)
        self.commit()
        self.h.window_clock(fk, fu, W)

    def upsert(self, table, ip, id_):
        self.h.upsert(table, ip, id_)
        self.m.upsert(table, ip, id_)

    def erase(self, table, ip):
        self.h.erase(table, ip)
        self.m.erase(table, ip)

    def commit(self):
        self.h.commit()
        self.m.commit()
        self.check()

    def submit(self, recs, how="host"):
        if how == "host":
            self.h.submit(recs)
        elif how == "device":
            d = self.h.dev_alloc(max(1, len(recs)) * 32)
            self.h.h2d(d, recs)
            self.h.submit_device(d, len(recs))
            self.h.sync()
            self.h.dev_free(d)
        elif how == "raw":
            self.h.submit_raw(to_raw(recs))
        self.m.submit(recs)
        self.check()

    def fold(self):
        self.h.fold()
        self.check(folded=True)

    def flush(self, what=""):
        rc, got, n = flush_raw(self.h, self.h.max_edges)
        exp = self.m.flush()
        assert rc == abi.OK, (what, rc)
        assert edges_equal(got, exp), f"{what} epoch {self.m.epoch_open - 1}: " + explain_diff(got, exp)
        self.check()
        return got

    def check(self, folded=False):
        """Stats against the model. src_unresolved is complete once the pending pairs are folded: before that only
        its sum with rows_emitted is exact."""
        got, exp = self.h.stats(), self.m.stats()
        for k in ("events_in", "late_events", "deferred_events", "capacity_events", "not_request"):
            assert got[k] == exp[k], (k, got[k], exp[k], got, exp)
        assert got["src_unresolved"] + got["rows_emitted"] == exp["src_unresolved"] + exp["rows_emitted"], (got, exp)
        if folded:
            assert (got["src_unresolved"], got["rows_emitted"]) == (exp["src_unresolved"], exp["rows_emitted"]), (got, exp)
        if self.m.epoch_open is not None and self.m.epoch_open < M64:
            assert self.h.window_epoch() == self.m.epoch_open

    def close(self):
        self.h.close()


def recs_at(wts, rng, src=None, dst=None, protos=PROTOS):
    n = len(wts)
    r = np.zeros(n, dtype=abi.L7_REC)
    r["saddr"] = src if src is not None else rng.choice(PODS + STRANGERS[:1], n)
    r["daddr"] = dst if dst is not None else rng.choice(ADDRS, n)
    r["sport"], r["dport"] = 40000, 80
    r["protocol"] = rng.choice(protos, n)
    r["method_flags"] = rng.choice([1, 2], n)
    r["status"] = rng.choice([200, 404, 500, 503], n)
    r["duration_ns"] = rng.integers(1, 1 << 34, n, dtype=np.uint64)
    r["write_time_ns"] = np.asarray(wts, dtype=np.uint64)
    return r


def wt_of(p, e, k=0):
    """Kernel write time of the k-th ns of epoch e under the pair's clock (mod 2^64)."""
    m = p.m
    return (e * m.W - (m.fu - m.fk) + k) % M64


# ---- boundaries ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("how", ["host", "device", "raw"])
def test_boundaries_within_a_warp_and_a_ragged_tail(how):
    """Write times at lo - 1, lo, lo + len - 1, lo + len and lo + k len (k = 2..5), patterned by the record index mod 64
    so that one warp and both event slots of a lane see every class; 61 chunks and a ragged tail of 37."""
    W, E = 1000, 10**12
    p = Pair(12345, 12345 + E * W + 77, W)
    rng = np.random.default_rng(1)
    first = recs_at([wt_of(p, E, 500)], rng, src=PODS[0], dst=SVCS[0], protos=[abi.PROTO_HTTP])
    p.submit(first, how)                                      # opens epoch E
    lo = wt_of(p, E)
    offs = [-1, 0, W - 1, W, 2 * W, 3 * W, 4 * W, 5 * W, W + 1, 2 * W - 1]
    n = 64 * 61 + 37
    idx = np.arange(n)
    wts = [(lo + offs[(i % 64) % len(offs)]) % M64 for i in idx]
    p.submit(recs_at(wts, rng), how)
    assert p.h.stats()["late_events"] == int(sum((i % 64) % len(offs) == 0 for i in idx))
    for k in range(7):
        got = p.flush(f"window {k}")
        if k == 6:
            assert len(got) == 0
    p.fold()
    p.close()


def test_opening_record_and_clock_reset():
    """The first record of the first batch opens the clock although the rest of its batch is older (late); a clock reset
    between windows reopens on the next record, which may lie far from the old clock."""
    W = 5000
    p = Pair(0, 10**9, W)
    rng = np.random.default_rng(2)
    e0 = (10**9 + 50_000) // W
    wts = [50_000] + list(rng.integers(0, 50_000, 3000)) + list(rng.integers(50_000 + W, 50_000 + 3 * W, 2000))
    p.submit(recs_at(wts, rng))
    assert p.m.epoch_open == e0 and p.h.stats()["late_events"] > 2000
    for k in range(4):
        p.flush(f"first clock {k}")
    p.fold()
    p.h.window_clock(7, 3, 10**6)
    p.m.clock(7, 3, 10**6)
    with pytest.raises(capi.AlzError) as e:
        p.h.window_epoch()
    assert e.value.status == abi.E_STATE
    p.submit(recs_at([5 * 10**6 + 1] + [10**6] * 100 + [7 * 10**6] * 50, rng), "raw")
    for k in range(3):
        p.flush(f"second clock {k}")
    p.close()


# ---- offsets ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("fk,fu,W,wts", [
    (10**12, 5, 1000, [10**12 + 4000, 10**12 + 3999, 10**12 + 5000, 10**12 + 7123, 0, M64 - 1]),    # offset wraps
    (0, 0, 1, [100, 99, 101, 102, 100, 0, M64 - 1, 103]),                                             # one-ns windows
    (0, 0, (1 << 63) + 1, [5, 0, M64 - 1, 1 << 63, (1 << 63) + 1, 3]),                                 # two epochs only
    (0, 0, 1000, [1000, 1500, 1000 + (1 << 63) + 5, M64 - 1, 2500]),        # 2^63 and more ahead: future, not late
    (0, M64 - 500, 1000, [0, 600, 499, 500, 5, M64 - 1]),                   # the user clock wraps: 600 is late
])
def test_clock_offsets_and_far_records(fk, fu, W, wts):
    p = Pair(fk, fu, W)
    rng = np.random.default_rng(3)
    # each write time 16 times over, patterned across lanes, with pods and strangers as sources
    recs = recs_at([wts[i % len(wts)] for i in range(16 * len(wts))], rng)
    recs[0]["write_time_ns"] = wts[0]
    p.submit(recs[:1])
    p.submit(recs[1:])
    for k in range(4):
        p.flush(f"window {k}")
    p.fold()
    p.close()


# ---- ping-pong ---------------------------------------------------------------------------------------------------

def test_ping_pong_over_consecutive_rolls():
    """Every roll re-ingests set-aside records of which some are set aside again, while new submits set records aside
    into the same buffer: nothing is lost or counted twice across five swaps of the two buffers."""
    W = 100
    p = Pair(0, 0, W)
    rng = np.random.default_rng(4)
    e = 10
    p.submit(recs_at([e * W + 1], rng))
    for k in range(6):
        wts = [(e + int(d)) * W + int(o) for d, o in zip(rng.integers(-1, 5, 3000), rng.integers(0, W, 3000))]
        p.submit(recs_at(wts, rng))
        p.flush(f"roll {k}")
        e += 1
    for k in range(5):
        p.flush(f"drain {k}")
    assert p.h.stats()["deferred_events"] == 0
    p.close()


def test_roll_sets_every_record_aside_again():
    """Every held record is set aside again at the roll, 300k resolved by a commit and 300k raw: more than the
    resident threads of the roll kernel and the chunks the ingest kernel has in flight, so the re-deferred records
    would overwrite unread ones if the roll wrote into the buffer it reads."""
    W = 1000
    p = Pair(0, 0, W, max_batch=1 << 20)
    rng = np.random.default_rng(12)
    p.submit(recs_at([4 * W + 1], rng))
    p.submit(recs_at(6 * W + rng.integers(0, W, 300_000), rng))
    p.upsert(abi.TABLE_POD, STRANGERS[1], 51)
    p.commit()
    p.submit(recs_at(6 * W + rng.integers(0, W, 300_000), rng))
    for k in range(3):
        p.flush(f"window {4 + k}")
    p.fold()
    p.close()


# ---- overflow ----------------------------------------------------------------------------------------------------

def test_defer_buffer_overflow():
    """max_batch 2^12: the buffer holds 2^13 records. 2^13 + 1000 identical records of the next epoch: 1000 are lost,
    counted once (capacity_events), reported by the flush of the window that was open when they were lost; the next
    window has the 2^13 held ones."""
    W = 1000
    p = Pair(0, 0, W, max_batch=1 << 12)
    rng = np.random.default_rng(5)
    cur = recs_at([5 * W + 3] * 50, rng)
    fut = recs_at([6 * W + 7], rng, src=PODS[1], dst=SVCS[1], protos=[abi.PROTO_HTTP])
    p.submit(cur)
    p.submit(np.repeat(fut, (1 << 13) + 1000))
    st = p.h.stats()
    assert st["deferred_events"] == 1 << 13 and st["capacity_events"] == 1000
    rc, got, n = flush_raw(p.h, p.h.max_edges)
    assert rc == abi.E_CAPACITY
    exp = p.m.flush()
    assert edges_equal(got, exp), explain_diff(got, exp)
    p.check()
    got = p.flush("after the overflow")
    assert int(got["count"].sum()) == 1 << 13
    p.fold()
    p.close()


# ---- tables (arrival-tables rule) -------------------------------------------------------------------------------

@pytest.mark.parametrize("fold_first", [False, True])
def test_commit_while_records_are_held(fold_first):
    """Set-aside records are resolved under the tables they arrived under: a commit that erases a held record's source
    pod, gives its destination a service and changes a pod id does not touch them; records submitted after it take the
    new tables. An explicit fold while records are held changes nothing."""
    W = 1000
    p = Pair(0, 0, W)
    rng = np.random.default_rng(6)
    src = np.array([PODS[0], PODS[1], PODS[2], STRANGERS[0]] * 200, dtype=np.uint32)
    dst = np.array([PODS[3], SVCS[0], PODS[4], PODS[5]] * 200, dtype=np.uint32)
    p.submit(recs_at([3 * W + 1] + [4 * W + 5] * 799, rng, src=src, dst=dst))
    p.submit(recs_at([5 * W + 9] * 400, rng, src=src[:400], dst=dst[:400]))
    if fold_first:
        p.fold()
    p.erase(abi.TABLE_POD, PODS[0])                 # a held record's source leaves the pod table
    p.upsert(abi.TABLE_SVC, PODS[3], 21)            # its destination gets a service
    p.upsert(abi.TABLE_POD, PODS[2], 31)            # another source changes its id
    p.upsert(abi.TABLE_POD, STRANGERS[0], 41)       # a stranger becomes a pod
    p.commit()
    p.submit(recs_at([4 * W + 6] * 400, rng, src=src[:400], dst=dst[:400]))
    p.flush("window 3")
    p.erase(abi.TABLE_POD, PODS[1])                 # second commit: records held twice keep their first resolution
    p.commit()
    p.fold()
    p.flush("window 4")
    p.flush("window 5")
    p.close()


# ---- clock changes ------------------------------------------------------------------------------------------------

def test_clock_change_refused_while_records_are_held():
    """submit [current, future], fold, clock change: refused (no stats call in between, which would refresh the host's
    copy of the counters), and the held record still comes out at its flush."""
    W = 1000
    p = Pair(0, 0, W)
    rng = np.random.default_rng(7)
    recs = recs_at([2 * W + 1, 3 * W + 1], rng, src=PODS[0], dst=SVCS[0], protos=[abi.PROTO_HTTP])
    p.h.submit(recs)
    p.m.submit(recs)
    p.h.fold()
    assert p.h.L.alz_window_clock(p.h.h, 0, 0, 0) == abi.E_STATE
    p.check(folded=True)
    assert p.h.L.alz_window_clock(p.h.h, 5, 5, 77) == abi.E_STATE
    p.flush("window 2")
    got = p.flush("window 3")
    assert int(got["count"].sum()) == 1
    p.h.window_clock(0, 0, 0)                        # nothing held, nothing pending: accepted
    p.close()


def test_clock_change_accepted_once_nothing_is_held():
    """A flush whose roll ingests every held record leaves nothing held; after a fold the clock may change (again no
    stats call after the flush)."""
    W = 1000
    p = Pair(0, 0, W)
    rng = np.random.default_rng(8)
    p.submit(recs_at([2 * W + 1] * 10 + [3 * W + 1] * 10, rng))
    rc, got, _ = flush_raw(p.h, p.h.max_edges)
    exp = p.m.flush()
    assert rc == abi.OK and edges_equal(got, exp), explain_diff(got, exp)
    p.h.fold()
    p.h.window_clock(0, 0, 2 * W)
    p.m.clock(0, 0, 2 * W)
    p.submit(recs_at([9 * W] * 5, rng))
    p.flush("window 4 of the new clock, with the records of the old window 3")
    p.close()


# ---- flush paths ------------------------------------------------------------------------------------------------

def test_small_buffer_keeps_the_epoch_and_the_held_records():
    W = 1000
    p = Pair(0, 0, W)
    rng = np.random.default_rng(9)
    p.submit(recs_at([7 * W + 3] + [7 * W + 5] * 2000 + [8 * W + 1] * 500 + [9 * W] * 100, rng))
    before = p.h.stats()
    rc, _, n = flush_raw(p.h, 1)
    assert rc == abi.E_CAPACITY and n > 1
    assert p.h.window_epoch() == 7 and p.h.stats()["deferred_events"] == before["deferred_events"]
    p.flush("window 7 after the refused flush")
    assert p.h.window_epoch() == 8
    p.flush("window 8")
    p.close()


def test_device_flush_gives_the_host_flush_bytes():
    W = 1000
    a, b = Pair(0, 0, W), Pair(0, 0, W)
    for k in range(3):
        recs = recs_at([(3 + k) * W + 1] + [(3 + k + d) * W + 2 for d in range(3)] * 500, np.random.default_rng(10 + k))
        a.h.submit(recs)
        b.h.submit(recs)
        rc, got, _ = flush_raw(a.h, a.h.max_edges)
        rc2, dev = flush_device_raw(b.h)
        assert rc == rc2 == abi.OK
        assert got.tobytes() == dev.tobytes()
    a.close()
    b.close()


# ---- producers ----------------------------------------------------------------------------------------------------

def test_eight_producers_three_epochs():
    W = 10_000
    p = Pair(0, 0, W)
    rng = np.random.default_rng(11)
    p.submit(recs_at([20 * W + 1], rng))
    parts = [recs_at(rng.integers(20 * W, 23 * W, 20_000), np.random.default_rng(100 + k)) for k in range(8)]

    def work(k):
        for c in np.array_split(parts[k], 5):
            p.h.submit(c)
    th = [threading.Thread(target=work, args=(k,)) for k in range(8)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for part in parts:
        p.m.submit(part)
    p.check()
    for k in range(3):
        p.flush(f"window {k}")
    p.close()


# ---- random operation sequences ---------------------------------------------------------------------------------

OFFS = [-1, 0, 1, 499, 998, 999]
op_s = st.one_of(
    st.tuples(st.just("submit"), st.integers(0, 5000), st.integers(0, 2**31)),
    st.tuples(st.just("erase"), st.sampled_from(ADDRS), st.integers(0, 1)),
    st.tuples(st.just("upsert"), st.sampled_from(ADDRS), st.integers(0, 1), st.integers(1, 60)),
    st.tuples(st.just("fold")),
    st.tuples(st.just("flush"), st.booleans()),
    st.tuples(st.just("stats")),
)


@settings(max_examples=25, deadline=None, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(ops=st.lists(op_s, min_size=1, max_size=12))
def test_random_operation_sequences(ops):
    W = 1000
    p = Pair(0, 0, W)
    try:
        for op in ops:
            if op[0] == "submit":
                rng = np.random.default_rng(op[2])
                base = p.m.epoch_open if p.m.epoch_open is not None else 50
                wts = [(base + int(d)) * W + OFFS[int(o)] for d, o in
                       zip(rng.integers(-2, 4, op[1]), rng.integers(0, len(OFFS), op[1]))]
                p.submit(recs_at(wts, rng))
            elif op[0] in ("erase", "upsert"):
                tab = abi.TABLE_POD if op[2] == 0 else abi.TABLE_SVC
                if op[0] == "erase":
                    p.erase(tab, op[1])
                else:
                    p.upsert(tab, op[1], op[3])
                p.commit()
            elif op[0] == "fold":
                p.fold()
            elif op[0] == "flush":
                if op[1]:
                    rc, _, n = flush_raw(p.h, 0)
                    assert rc == (abi.E_CAPACITY if n else abi.OK)
                    if rc == abi.OK:
                        p.m.flush()
                    p.check()
                else:
                    p.flush("random")
            else:
                p.check()
        p.fold()
    finally:
        p.close()
