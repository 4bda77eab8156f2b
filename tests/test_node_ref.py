"""CPU: tests/node_ref.py, the §21 reference of the node calls, against node rows, metrics and top orders derived by
hand: a self-loop, a reversed (DELIVER) row, pod 7 against service 7, outbound v against Host-keyed v, a node seen only
as a to end, cells and sums that wrap, and counts above 2^53 that tie."""
import numpy as np

import metric_ref
import node_ref as nr
from alaz_b200 import abi

POD, SVC, OUT, HOST = 0, 1, 2, 3
IN, OUTS = abi.SIDE_IN, abi.SIDE_OUT
Q = abi.METRIC_QUANTILE


def row(ft, f, tt, t, count=0, err=0, lat=0, cells=None):
    r = np.zeros(1, dtype=abi.EDGE_OUT)
    r["from_type"], r["from"], r["to_type"], r["to"] = ft, f, tt, t
    r["count"], r["err5xx"], r["lat_sum_ns"] = count, err, lat
    for b, c in (cells or {}).items():
        r["hist"][0, b] = c
    return r


def rows(*rs):
    return np.concatenate(rs)


def at(nodes, t, v):
    i = np.flatnonzero((nodes["type"] == t) & (nodes["value"] == v))
    assert len(i) == 1, (t, v)
    return int(i[0])


def test_self_loop_counts_on_both_sides():
    n = nr.group(row(POD, 3, POD, 3, count=5, err=1, lat=50, cells={4: 5}))
    assert len(n) == 1 and n["type"][0] == POD and n["value"][0] == 3
    assert n["in_edges"][0] == 1 and n["out_edges"][0] == 1
    for s in ("in", "out"):
        assert (n[s]["count"][0], n[s]["err5xx"][0], n[s]["lat_sum_ns"][0], n[s]["hist"][0, 4]) == (5, 1, 50, 5)


def test_reversed_row_is_delivered_to_its_to_end():
    # a DELIVER row: the service is the from end, the consuming pod the to end (§1.4)
    n = nr.group(rows(row(SVC, 5, POD, 2, count=4, cells={0: 4}), row(POD, 2, SVC, 9, count=1, cells={1: 1})))
    p, s = at(n, POD, 2), at(n, SVC, 5)
    assert n["in"]["count"][p] == 4 and n["out"]["count"][p] == 1
    assert n["in_edges"][p] == 1 and n["out_edges"][p] == 1
    assert n["out"]["count"][s] == 4 and n["in_edges"][s] == 0 and n["in"]["count"][s] == 0


def test_same_value_different_type_are_different_nodes_in_key_order():
    n = nr.group(rows(row(POD, 1, POD, 7, count=2), row(POD, 1, SVC, 7, count=3), row(POD, 1, OUT, 9, count=4),
                      row(POD, 1, HOST, 9, count=5)))
    assert [(int(t), int(v)) for t, v in zip(n["type"], n["value"])] == [(POD, 1), (POD, 7), (SVC, 7), (OUT, 9),
                                                                          (HOST, 9)]
    assert list(n["in"]["count"]) == [0, 2, 3, 4, 5]
    assert n["out"]["count"][0] == 14 and n["out_edges"][0] == 4
    assert list(nr.keys(rows(row(POD, 1, SVC, 7)))) == [1, (1 << 32) | 7]


def test_node_seen_only_as_to_end():
    n = nr.group(rows(row(POD, 1, SVC, 4, count=6, err=2, lat=600, cells={10: 6}),
                      row(POD, 2, SVC, 4, count=2, err=0, lat=100, cells={12: 2})))
    s = at(n, SVC, 4)
    assert n["in_edges"][s] == 2 and n["out_edges"][s] == 0
    assert (n["in"]["count"][s], n["in"]["err5xx"][s], n["in"]["lat_sum_ns"][s]) == (8, 2, 700)
    assert n["in"]["hist"][s, 10] == 6 and n["in"]["hist"][s, 12] == 2
    assert n["out"].tobytes()[s * 280:(s + 1) * 280] == bytes(280)
    v = nr.matrix(n, IN, [abi.METRIC_COUNT, abi.METRIC_ERR5XX, abi.METRIC_ERR_RATE, abi.METRIC_MEAN_NS])[s]
    assert list(v) == [8.0, 2.0, 0.25, 87.5]
    assert list(nr.matrix(n, OUTS, [abi.METRIC_COUNT, abi.METRIC_ERR_RATE, (Q, 0.99)])[s]) == [0.0, 0.0, 0.0]


def test_cells_and_sums_wrap():
    big = (1 << 64) - 1
    n = nr.group(rows(row(POD, 1, SVC, 2, count=big, err=big, lat=big, cells={0: (1 << 32) - 1, 5: 7}),
                      row(POD, 3, SVC, 2, count=3, err=2, lat=5, cells={0: 2, 5: (1 << 32) - 1})))
    s = at(n, SVC, 2)
    assert (int(n["in"]["count"][s]), int(n["in"]["err5xx"][s]), int(n["in"]["lat_sum_ns"][s])) == (2, 1, 4)
    assert n["in"]["hist"][s, 0] == 1 and n["in"]["hist"][s, 5] == 6
    # the quantile total is the sum of the wrapped cells (7), as §17 takes it for an edge row
    side = nr.side_rows(n, IN)[s:s + 1]
    assert nr.values(n, IN, (Q, 0.5))[s] == metric_ref.values(side, (Q, 0.5))[0]
    assert int(side["hist"].astype(np.uint64).sum()) == 7


def test_counts_above_2_53_tie_and_rank_by_node_index():
    a, b = 1 << 53, (1 << 53) + 1   # the same float64
    n = nr.group(rows(row(POD, 9, SVC, 1, count=b), row(POD, 8, SVC, 0, count=a), row(POD, 7, SVC, 2, count=5)))
    assert [(int(t), int(v)) for t, v in zip(n["type"], n["value"])] == [(POD, 7), (POD, 8), (POD, 9), (SVC, 0),
                                                                          (SVC, 1), (SVC, 2)]
    idx, above = nr.top(n, IN, abi.METRIC_COUNT, 2, 1.0)
    assert list(idx) == [3, 4] and above == 3
    idx, above = nr.top(n, OUTS, abi.METRIC_COUNT, 10, float(a))
    assert list(idx) == [1, 2] and above == 2
    idx, above = nr.top(n, IN, abi.METRIC_COUNT, 10, -np.inf)
    assert list(idx) == [3, 4, 5, 0, 1, 2] and above == 6


def test_empty_and_group_order_does_not_matter():
    assert len(nr.group(np.zeros(0, dtype=abi.EDGE_OUT))) == 0
    rng = np.random.default_rng(5)
    r = np.zeros(300, dtype=abi.EDGE_OUT)
    r["from_type"] = rng.integers(0, 4, 300)
    r["to_type"] = rng.integers(0, 4, 300)
    r["from"] = rng.integers(0, 20, 300)
    r["to"] = rng.integers(0, 20, 300)
    r["count"] = rng.integers(0, 1 << 63, 300, dtype=np.uint64)
    r["hist"] = rng.integers(0, 1 << 32, (300, abi.NB), dtype=np.uint64).astype(np.uint32)
    g = nr.group(r)
    assert g.tobytes() == nr.group(r[rng.permutation(300)]).tobytes()
    assert int(g["in_edges"].sum()) == 300 == int(g["out_edges"].sum())
