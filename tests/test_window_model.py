"""CPU: the sequential model of time-cut windows (tests/window_model.py) against the oracle and by hand."""
import numpy as np

import oracle_lib as ol
from alaz_b200 import abi
from helpers import edges_equal, explain_diff, sort_edges
from window_model import WindowModel, epoch

M64 = 1 << 64


def test_epoch_equals_orc_epoch_at_the_wrap():
    rng = np.random.default_rng(7)
    cases = [(0, 0, 1), (12345, 1_700_000_000_000_000_000, 10**9), (M64 - 1, 0, 7), (0, M64 - 1, 1000),
             (5, 3, (1 << 63) + 1), (M64 - 500, 100, 1 << 63), (1 << 63, (1 << 63) - 1, 3)]
    cases += [tuple(int(x) for x in rng.integers(0, M64, 2, dtype=np.uint64)) + (int(rng.integers(1, M64, dtype=np.uint64)),)
              for _ in range(20)]
    for fk, fu, w in cases:
        wt = np.array([0, 1, M64 - 1, M64 - 2, fk, (fk - 1) % M64, (fk + w) % M64, (fk - fu) % M64,
                       (fk - fu - 1) % M64] + rng.integers(0, M64, 40, dtype=np.uint64).tolist(), dtype=np.uint64)
        got = epoch(fk, fu, w, wt)
        exp = [ol.epoch(fk, fu, w, int(t)) for t in wt]
        assert got.tolist() == exp, (fk, fu, w)


def test_commit_free_stream_is_the_oracle_grouped_by_epoch():
    """Without table changes the model is "group the records by epoch": late records go to the window that was open
    when they came."""
    S, N = 300, 60_000
    t = ol.Topo(S, seed=31, mix=abi.MIX_ALL)
    ev = t.events(0, N)
    wt = ev["write_time_ns"].astype(np.uint64)
    fk, fu = int(wt[0]) + 777, 1_700_000_000_123_456_789   # first_user - first_kernel wraps
    W = (int(wt[-1]) - int(wt[0])) // 5 + 1
    e = epoch(fk, fu, W, wt)
    assert int(e.max()) - int(e[0]) >= 4
    m = WindowModel(fk, fu, W, defer_cap=N)
    for k, v in enumerate(t.pod_ip):
        m.upsert(abi.TABLE_POD, int(v), k)
    for k, v in enumerate(t.svc_ip):
        m.upsert(abi.TABLE_SVC, int(v), k)
    m.commit()
    order = np.random.default_rng(3).permutation(N - 1) + 1      # first record first, the rest in any order
    m.submit(ev[:1])
    for part in np.array_split(order, 7):
        m.submit(ev[part])
    e0 = int(e[0])
    late = int((e < e0).sum())
    st = m.stats()
    assert st["late_events"] == late and st["deferred_events"] == int((e > e0).sum()) and st["events_in"] == N
    for k in range(int(e.max()) - e0 + 1):
        o = ol.Oracle()
        o.load_tables(t.pod_ip, t.svc_ip)
        o.process(ev[(e == e0 + k) | ((e < e0) & (k == 0))])
        got, exp = m.flush(), o.edges()
        assert edges_equal(got, exp), f"epoch {e0 + k}: " + explain_diff(got, exp)
    assert m.stats()["deferred_events"] == 0


def _rec(src, dst, wt, proto=abi.PROTO_HTTP, dur=1000):
    r = np.zeros(1, dtype=abi.L7_REC)
    r["saddr"], r["daddr"], r["write_time_ns"] = abi.ip(src), abi.ip(dst), wt
    r["protocol"], r["method_flags"], r["status"], r["duration_ns"] = proto, 1, 200, dur
    return r


def test_hand_derived_arrival_tables_and_counters():
    """window_ns = 100, offset 0; pods A = 10.0.0.1 (id 1), B = 10.0.0.2 (id 2); service S = 172.16.0.1 (id 7);
    C = 10.0.0.3 is no pod.

    submit  #1 A->S wt 150   epoch 1: opens epoch 1                        -> window 1
            #2 A->B wt 120   epoch 1                                        -> window 1
            #3 B->S wt 250   epoch 2: set aside (B is a pod now)
            #4 A->S wt 260   epoch 2, KAFKA: set aside, no row
            #5 A->B wt  90   epoch 0 < 1: late                              -> window 1
            #6 C->S wt 270   epoch 2: set aside, source no pod
    erase pod B, commit
            #7 B->S wt 280   epoch 2: set aside, source no pod (tables now)

    Before the first flush: events_in 7, late 1, deferred 4 (#3 #4 #6 #7), not_request 0, src_unresolved 0,
    rows_emitted 3 (#1 #2 #5). Flush 1: pod1->svc7 count 1, pod1->pod2 count 2.
    After it, window 2 is open: not_request 1 (#4), src_unresolved 2 (#6 #7), rows_emitted 3 + 1 (#3).
    Flush 2: pod2->svc7 count 1 (#3, resolved by the tables it arrived under)."""
    A, B, C, S = "10.0.0.1", "10.0.0.2", "10.0.0.3", "172.16.0.1"
    m = WindowModel(0, 0, 100, defer_cap=100)
    m.upsert(abi.TABLE_POD, abi.ip(A), 1)
    m.upsert(abi.TABLE_POD, abi.ip(B), 2)
    m.upsert(abi.TABLE_SVC, abi.ip(S), 7)
    m.commit()
    m.submit(np.concatenate([_rec(A, S, 150), _rec(A, B, 120), _rec(B, S, 250), _rec(A, S, 260, abi.PROTO_KAFKA),
                             _rec(A, B, 90), _rec(C, S, 270)]))
    m.erase(abi.TABLE_POD, abi.ip(B))
    m.commit()
    m.submit(_rec(B, S, 280))
    assert m.epoch_open == 1
    assert m.stats() == dict(events_in=7, late_events=1, deferred_events=4, capacity_events=0, not_request=0,
                             src_unresolved=0, rows_emitted=3)
    e1 = sort_edges(m.flush())
    assert [(int(x["from_type"]), int(x["from"]), int(x["to_type"]), int(x["to"]), int(x["count"])) for x in e1] == \
        [(abi.NODE_POD, 1, abi.NODE_POD, 2, 2), (abi.NODE_POD, 1, abi.NODE_SVC, 7, 1)]
    assert m.stats() == dict(events_in=7, late_events=1, deferred_events=0, capacity_events=0, not_request=1,
                             src_unresolved=2, rows_emitted=4)
    e2 = m.flush()
    assert [(int(x["from"]), int(x["to_type"]), int(x["to"]), int(x["count"]), int(x["lat_sum_ns"])) for x in e2] == \
        [(2, abi.NODE_SVC, 7, 1, 1000)]
    assert len(m.flush()) == 0 and m.epoch_open == 4


def test_model_overflow_counts():
    """Past defer_cap a set-aside record is lost: counted in capacity_events and not held."""
    m = WindowModel(0, 0, 100, defer_cap=5)
    m.upsert(abi.TABLE_POD, abi.ip("10.0.0.1"), 1)
    m.commit()
    m.submit(np.concatenate([_rec("10.0.0.1", "10.9.9.9", 10)] + [_rec("10.0.0.1", "10.9.9.9", 150)] * 8))
    st = m.stats()
    assert (st["deferred_events"], st["capacity_events"], st["rows_emitted"]) == (5, 3, 1)
    m.flush()
    assert int(m.flush()["count"].sum()) == 5
