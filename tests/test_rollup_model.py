"""CPU: the model of the rolling windows (tests/rollup_model.py) pinned by hand and against the oracle. While the
tables do not change, the sum of k windows' rows is what one oracle fed the k windows' events returns."""
import numpy as np
import pytest

import oracle_lib as ol
from alaz_b200 import abi
from helpers import sort_edges
from rollup_model import RollupModel, packed_key


def row(ft, f, tt, t, count, err=0, lat=0, hist=()):
    r = np.zeros((), dtype=abi.EDGE_OUT)
    r["from_type"], r["from"], r["to_type"], r["to"] = ft, f, tt, t
    r["count"], r["err5xx"], r["lat_sum_ns"] = count, err, lat
    for b, c in hist:
        r["hist"][b] = c
    return r


def rows(*rs):
    return np.array(list(rs), dtype=abi.EDGE_OUT)


P, S, O, H = abi.NODE_POD, abi.NODE_SVC, abi.NODE_OUTBOUND, abi.NODE_OUTBOUND_HOST


def test_packed_key_orders_rows_as_a_flush_does():
    # pod -> pod < pod -> service < pod -> outbound < pod -> host < service -> pod (reversed) < outbound -> pod
    ks = [packed_key(row(P, 5, P, 9, 1)), packed_key(row(P, 0, S, 0, 1)), packed_key(row(P, 0, O, 1, 1)),
          packed_key(row(P, (1 << 29) - 1, H, 0xFFFFFFFF, 1)), packed_key(row(S, 3, P, 0, 1)),
          packed_key(row(O, 0xFFFFFFFF, P, (1 << 29) - 1, 1))]
    assert ks == sorted(ks) and len(set(ks)) == len(ks)
    assert packed_key(row(P, 7, O, 7, 1)) != packed_key(row(P, 7, H, 7, 1))       # a host id equal to an address
    assert packed_key(row(P, 7, S, 2, 1)) != packed_key(row(S, 2, P, 7, 1))       # the rev bit


def test_three_windows_by_hand():
    m = RollupModel()
    m.history(2, 100)
    a = row(P, 1, S, 2, 3, 1, 10, [(0, 3)])
    b = row(P, 1, O, 9, 1, 0, 5, [(4, 1)])
    m.append(rows(a), 1)
    m.append(rows(row(P, 1, S, 2, (1 << 64) - 2, 0, (1 << 64) - 4, [(0, (1 << 32) - 2)]), b), 2)
    got, info = m.rollup(2)
    assert info == dict(windows=2, clocked=0, window_first=1, window_last=2, epoch_first=0, epoch_last=0, rows_in=3)
    assert [int(x) for x in got["count"]] == [1, 1]                      # 3 + 2^64 - 2 wraps to 1
    assert int(got[0]["lat_sum_ns"]) == 6 and int(got[0]["hist"][0]) == 1 and int(got[0]["err5xx"]) == 1
    assert got[1].tobytes() == b.tobytes()
    m.append(rows(), 3)                                                  # depth 2: the first window leaves
    got, info = m.rollup(5)
    assert info["windows"] == 2 and info["window_first"] == 2 and info["rows_in"] == 2 and len(got) == 2
    one, info = m.rollup(1)
    assert len(one) == 0 and info["windows"] == 1 and info["window_first"] == 3


def test_arena_placement_and_eviction():
    m = RollupModel()
    m.history(8, 10)
    mk = lambda n, base: rows(*[row(P, base + i, S, 1, 1) for i in range(n)])
    m.append(mk(4, 0), 1)
    m.append(mk(4, 10), 2)
    assert [e["first_row"] for e in m.entries] == [0, 4]
    m.append(mk(3, 20), 3)            # does not fit behind row 8: starts at row 0 and evicts the window there
    assert [(e["window"], e["first_row"]) for e in m.entries] == [(2, 4), (3, 0)]
    m.append(mk(2, 30), 4)            # rows 3..4 overlap window 2
    assert [(e["window"], e["first_row"]) for e in m.entries] == [(3, 0), (4, 3)]
    m.append(mk(11, 40), 5)           # larger than the arena: nothing is retained
    assert m.entries == []
    m.append(mk(1, 50), 6)
    m.history(8, 10)                  # the same values: kept
    assert len(m.entries) == 1
    m.history(8, 11)
    assert m.entries == []


@pytest.mark.parametrize("k", [1, 2, 5])
def test_sum_of_windows_equals_one_oracle_over_their_events(k):
    t = ol.Topo(48, seed=7, mix=abi.MIX_ALL)
    o = ol.Oracle()
    o.load_tables(t.pod_ip, t.svc_ip)
    m = RollupModel()
    m.history(5, 1 << 20)
    per = 20_000
    for w in range(5):
        o.process(t.events(w * per, per))
        m.append(sort_edges(o.edges()), w + 1)
        o.reset_window()
    o.process(t.events((5 - k) * per, k * per))
    exp = o.edges()
    got, info = m.rollup(k)
    assert info["windows"] == k and info["window_first"] == 5 - k + 1 and info["window_last"] == 5
    exp = exp[sorted(range(len(exp)), key=lambda i: packed_key(exp[i]))]
    assert got.tobytes() == exp.tobytes()
    o.close()
    t.close()
