"""CPU: the model of time-cut windows on several ranks (tests/window_ranks_model.py), by hand and against one
WindowModel fed the union of the ranks' streams."""
import numpy as np
from hypothesis import given, settings, strategies as st

from alaz_b200 import abi
from helpers import edges_equal, explain_diff, sort_edges
from window_model import WindowModel
from window_ranks_model import M64, STATE_ERR, RanksModel, sum_rows

A, B, C, S = "10.0.0.1", "10.0.0.2", "10.0.0.3", "172.16.0.1"
W = 100


def _rec(src, dst, wt, dur=1000):
    r = np.zeros(1, dtype=abi.L7_REC)
    r["saddr"], r["daddr"], r["write_time_ns"] = abi.ip(src), abi.ip(dst), wt
    r["protocol"], r["method_flags"], r["status"], r["duration_ns"] = abi.PROTO_HTTP, 1, 200, dur
    return r


def _model(R, fk=0, fu=0, w=W, cap=1000):
    m = RanksModel(R, cap)
    for r in range(R):
        m.upsert(r, abi.TABLE_POD, abi.ip(A), 1)
        m.upsert(r, abi.TABLE_POD, abi.ip(B), 2)
        m.upsert(r, abi.TABLE_POD, abi.ip(C), 3)
        m.upsert(r, abi.TABLE_SVC, abi.ip(S), 7)
        m.commit(r)
        m.clock(r, fk, fu, w)
    return m


def _counts(rows):
    return [(int(x["from"]), int(x["count"])) for x in sort_edges(rows)]


def test_openings_at_e_e1_e3():
    """Rank 0 opens at epoch 1, rank 1 at 2, rank 2 at 4 (each from its first record: A->S, B->S, C->S).
    Flush 1: E = 1, rank 0's row; ranks 1 and 2 keep theirs. Flush 2: E = 2, rank 1's row (rank 0 is empty at 2).
    Flush 3: E = 3, no rows, rank 2 still ahead. Flush 4: E = 4, rank 2's row. After it every rank is at 5."""
    m = _model(3)
    m.submit(0, _rec(A, S, 150))
    m.submit(1, _rec(B, S, 250))
    m.submit(2, _rec(C, S, 450))
    assert [m.epoch(r) for r in range(3)] == [1, 2, 4]
    st_, rows = m.flush()
    assert st_ == abi.OK and _counts(rows) == [(1, 1)]
    assert [m.epoch(r) for r in range(3)] == [2, 2, 4]
    assert m.stats(1)["rows_emitted"] == 1 and m.stats(2)["rows_emitted"] == 1   # kept, not flushed
    assert _counts(m.flush()[1]) == [(2, 1)]
    assert [m.epoch(r) for r in range(3)] == [3, 3, 4]
    assert len(m.flush()[1]) == 0
    assert [m.epoch(r) for r in range(3)] == [4, 4, 4]
    assert _counts(m.flush()[1]) == [(3, 1)]
    assert [m.epoch(r) for r in range(3)] == [5, 5, 5] and m.windows == [4, 4, 4]


def test_rank_empty_for_three_windows_then_late_and_deferred():
    """Rank 1 has no records: the first flush opens it at E + 1 = 2 and it follows rank 0 from there. Its first
    record, of epoch 5, is set aside (it does not open a window); one of epoch 1 is late."""
    m = _model(2)
    for e in (1, 2, 3):
        m.submit(0, _rec(A, S, e * W + 10))
    assert m.epoch(1) is None
    assert _counts(m.flush()[1]) == [(1, 1)]
    assert m.epoch(1) == 2
    assert _counts(m.flush()[1]) == [(1, 1)]
    m.submit(1, _rec(B, S, 5 * W + 1))
    m.submit(1, _rec(B, S, 1 * W + 1))
    s = m.stats(1)
    assert (s["deferred_events"], s["late_events"], m.epoch(1)) == (1, 1, 3)
    assert _counts(m.flush()[1]) == [(1, 1), (2, 1)]                   # epoch 3: rank 0's and the late record
    assert len(m.flush()[1]) == 0                                      # epoch 4
    assert _counts(m.flush()[1]) == [(2, 1)]                           # epoch 5: the set-aside record
    assert m.stats(1)["deferred_events"] == 0


def test_no_rank_open_changes_nothing():
    m = _model(3)
    st_, rows = m.flush()
    assert st_ == abi.OK and len(rows) == 0 and all(m.epoch(r) is None for r in range(3))


def test_clock_mismatch_keeps_every_window():
    """Length, offset, and clock off on one rank: the flush fails on every rank and nothing changes. The same offset
    from other first times is the same clock."""
    m = _model(2)
    m.submit(0, _rec(A, S, 150))
    m.clock(1, 0, 0, 2 * W)
    assert m.flush()[0] == STATE_ERR and m.epoch(0) == 1 and m.windows == [0, 0]
    m.clock(1, 10, 10, W)                          # offset 0 again
    assert _counts(m.flush()[1]) == [(1, 1)]
    m.clock(1, 0, 5, W)
    assert m.flush()[0] == STATE_ERR
    m2 = RanksModel(2, 10)
    m2.clock(0, 0, 0, W)
    assert m2.flush()[0] == STATE_ERR


def test_past_state_sorts_after_every_epoch():
    """window_ns 2^62 + 1: epochs 0..3, the last one ends past 2^64. Rank 0 reaches the past state on its own (a
    flush before it joins); rank 1 then opens at epoch 2. E = 2: rank 0 keeps its window, in which every record is
    late; the next flush at E = 3 moves rank 1 into the past state and then both merge every window."""
    w = (1 << 62) + 1
    m = _model(2, w=w)
    m.submit(0, _rec(A, S, 3 * w + 5))
    assert m.epoch(0) == 3
    m.solo_flush(0)                                                    # alone, before the ranks join
    assert m.key(0) == M64
    m.submit(0, _rec(A, S, 7))                                         # late in the past state
    m.submit(1, _rec(B, S, 2 * w + 1))
    assert _counts(m.flush()[1]) == [(2, 1)]
    assert m.key(0) == M64 and m.epoch(1) == 3
    assert len(m.flush()[1]) == 0 and m.key(1) == M64
    assert _counts(m.flush()[1]) == [(1, 1)]
    assert m.stats(0)["late_events"] == 1


def test_unopened_rank_enters_the_past_state_with_the_last_epoch():
    w = (1 << 62) + 1
    m = _model(2, w=w)
    m.submit(0, _rec(A, S, 3 * w))
    m.flush()
    assert m.key(0) == M64 and m.key(1) == M64
    m.submit(1, _rec(B, S, 0))
    assert m.stats(1)["late_events"] == 1
    assert _counts(m.flush()[1]) == [(2, 1)]


def test_cut_at_max_edges_counts_the_owners_rows():
    m = RanksModel(2, 100, max_edges=1)
    for r in range(2):
        m.upsert(r, abi.TABLE_POD, abi.ip(A), 1)
        m.upsert(r, abi.TABLE_POD, abi.ip(B), 2)
        m.commit(r)
        m.clock(r, 0, 0, W)
    m.submit(0, _rec(A, S, 10))
    m.submit(1, np.concatenate([_rec(B, S, 20)] * 3))
    st_, rows = m.flush()
    assert st_ == abi.E_CAPACITY and _counts(rows) == [(1, 1)]
    assert m.stats(1)["capacity_events"] == 3 and m.stats(1)["rows_emitted"] == 0


def test_sum_rows_adds_a_key_present_on_two_ranks():
    a, b = np.zeros(1, abi.EDGE_OUT), np.zeros(1, abi.EDGE_OUT)
    for x in (a, b):
        x["from_type"], x["from"], x["to_type"], x["to"] = abi.NODE_POD, 1, abi.NODE_SVC, 7
        x["count"], x["lat_sum_ns"] = 2, (1 << 63) + 1
        x["hist"][0, 3] = 0xFFFFFFFF
    rows, own = sum_rows([(0, a), (1, b)])
    assert int(rows["count"][0]) == 4 and int(rows["lat_sum_ns"][0]) == 2
    assert int(rows["hist"][0, 3]) == 0xFFFFFFFE and own == [[(0, 2), (1, 2)]]


@settings(max_examples=40, deadline=None)
@given(R=st.integers(2, 5), seed=st.integers(0, 2**32 - 1), n_flush=st.integers(1, 6))
def test_same_first_epoch_is_one_model_of_the_union(R, seed, n_flush):
    """When every rank's first record falls in one epoch, the merged windows are one WindowModel fed the union."""
    rng = np.random.default_rng(seed)
    srcs, dsts = [A, B, C], [S, A, B, "8.8.8.8"]
    e0 = int(rng.integers(3, 10))
    m, one = _model(R), WindowModel(0, 0, W, 1000)
    for k, ip in enumerate([A, B, C]):
        one.upsert(abi.TABLE_POD, abi.ip(ip), k + 1)
    one.upsert(abi.TABLE_SVC, abi.ip(S), 7)
    one.commit()
    for r in range(R):
        first = _rec(srcs[r % 3], S, e0 * W + int(rng.integers(0, W)))
        m.submit(r, first)
        one.submit(first)
    for _ in range(n_flush):
        for _ in range(int(rng.integers(0, 8))):
            r = int(rng.integers(0, R))
            e = e0 + int(rng.integers(-2, 5))
            rec = _rec(srcs[int(rng.integers(0, 3))], dsts[int(rng.integers(0, 4))], max(e, 0) * W + int(rng.integers(0, W)),
                       dur=int(rng.integers(1, 1 << 20)))
            m.submit(r, rec)
            one.submit(rec)
        st_, got = m.flush()
        exp, _ = sum_rows([(0, one.flush())])
        assert st_ == abi.OK and edges_equal(got, exp), explain_diff(got, exp)
        assert got.tobytes() == exp.tobytes()
        for k in ("late_events", "deferred_events", "rows_emitted", "events_in"):
            assert sum(m.stats(r)[k] for r in range(R)) == one.stats()[k], k
