"""CPU: tests/node_series_ref.py, the §22 reference of the node series and node trends, against series and records
derived by hand: a node present only on OUT in one entry, a self-loop, pod 7 against service 7 and outbound v against
Host-keyed v, a service whose callers change every entry, sums and cells that wrap within one point, and caller keys
with duplicates and a node no entry holds."""
import numpy as np
import pytest

import node_series_ref as nsr
from alaz_b200 import abi

POD, SVC, OUT, HOST = 0, 1, 2, 3
IN, OUTS = abi.SIDE_IN, abi.SIDE_OUT
Q = abi.METRIC_QUANTILE
C, E, R = abi.METRIC_COUNT, abi.METRIC_ERR5XX, abi.METRIC_ERR_RATE


def row(ft, f, tt, t, count=0, err=0, lat=0, cells=None):
    r = np.zeros(1, dtype=abi.EDGE_OUT)
    r["from_type"], r["from"], r["to_type"], r["to"] = ft, f, tt, t
    r["count"], r["err5xx"], r["lat_sum_ns"] = count, err, lat
    for b, c in (cells or {}).items():
        r["hist"][0, b] = c
    return r


def rows(*rs):
    return np.concatenate(rs) if rs else np.zeros(0, dtype=abi.EDGE_OUT)


def key(t, v):
    return (t << 32) | v


def test_node_present_only_on_out_in_one_entry():
    e0 = rows(row(POD, 1, SVC, 2, count=3))                          # pod 1 calls: OUT only
    e1 = rows(row(SVC, 2, POD, 1, count=4))                          # pod 1 is called: IN only
    e2 = rows(row(POD, 1, SVC, 2, count=5), row(SVC, 9, POD, 1, count=6))
    keys = [key(POD, 1)]
    v, p = nsr.series([e0, e1, e2], keys, IN, [C])
    assert p.tolist() == [[0, 1, 1]] and v[0, :, 0].tolist() == [0.0, 4.0, 6.0]
    v, p = nsr.series([e0, e1, e2], keys, OUTS, [C])
    assert p.tolist() == [[1, 0, 1]] and v[0, :, 0].tolist() == [3.0, 0.0, 5.0]
    # k cuts the oldest entries off
    v, p = nsr.series([e0, e1, e2], keys, OUTS, [C], k=2)
    assert p.tolist() == [[0, 1]] and v[0, :, 0].tolist() == [0.0, 5.0]


def test_self_loop_counts_on_both_sides_of_its_point():
    e = rows(row(POD, 3, POD, 3, count=5, err=1, cells={4: 5}))
    for side in (IN, OUTS):
        v, p = nsr.series([e], [key(POD, 3)], side, [C, E, R])
        assert p.tolist() == [[1]] and v[0, 0].tolist() == [5.0, 1.0, 0.2]


def test_same_value_of_different_types_are_different_nodes():
    e = rows(row(POD, 7, SVC, 7, count=2), row(POD, 7, OUT, 9, count=3), row(POD, 8, HOST, 9, count=11))
    keys = [key(POD, 7), key(SVC, 7), key(OUT, 9), key(HOST, 9)]
    v, p = nsr.series([e], keys, IN, [C])
    assert p[:, 0].tolist() == [0, 1, 1, 1] and v[:, 0, 0].tolist() == [0.0, 2.0, 3.0, 11.0]
    v, p = nsr.series([e], keys, OUTS, [C])
    assert p[:, 0].tolist() == [1, 0, 0, 0] and v[:, 0, 0].tolist() == [5.0, 0.0, 0.0, 0.0]


def test_service_with_changing_callers_is_present_at_every_point():
    ents = [rows(row(POD, 100 + j, SVC, 4, count=j + 1, err=j % 2)) for j in range(5)]
    v, p = nsr.series(ents, [key(SVC, 4)], IN, [C, E])
    assert p.tolist() == [[1] * 5]
    assert v[0, :, 0].tolist() == [1.0, 2.0, 3.0, 4.0, 5.0] and v[0, :, 1].tolist() == [0.0, 1.0, 0.0, 1.0, 0.0]
    # each caller's edge is present at one point only, yet the service's slope over them is exact
    rec, y, pr = nsr.expect(ents, ents[-1], IN, C, 5, stat=abi.TREND_SLOPE)
    s = rec[list(nsr.node_keys(rec)).index(key(SVC, 4))]
    assert (s["valid"], s["used"], s["trend"]) == (1, 5, 1.0)
    caller = rec[list(nsr.node_keys(rec)).index(key(POD, 104))]
    assert (caller["valid"], caller["used"]) == (0, 0)    # the pod is never called: no IN point


def test_sums_and_cells_wrap_within_one_point():
    big = (1 << 64) - 1
    e = rows(row(POD, 1, SVC, 2, count=big, lat=big, cells={0: 0xFFFFFFFF, 63: 0x80000001}),
             row(POD, 3, SVC, 2, count=3, lat=5, cells={0: 2, 63: 0x80000001}))
    v, p = nsr.series([e], [key(SVC, 2)], IN, [C, abi.METRIC_MEAN_NS, (Q, 1.0)])
    # count 2, latency sum 4 (both mod 2^64); cell 0 holds 1 and cell 63 holds 2 (mod 2^32)
    assert p.tolist() == [[1]] and v[0, 0, 0] == 2.0 and v[0, 0, 1] == 2.0
    assert v[0, 0, 2] == float(1 << 40)        # 3 cells in all: the 1.0 quantile is the top of bucket 63


def test_caller_keys_duplicates_and_unknown_nodes():
    e0 = rows(row(POD, 1, SVC, 2, count=3))
    e1 = rows(row(POD, 1, SVC, 2, count=4), row(POD, 5, SVC, 6, count=1))
    ends = np.zeros(4, dtype=abi.NODE_ENDS)
    ends["type"] = [SVC, SVC, SVC, POD]
    ends["value"] = [2, 6, 2, 77]
    keys = nsr.ends_keys(ends)
    v, p = nsr.series([e0, e1], keys, IN, [C])
    assert p.tolist() == [[1, 1], [0, 1], [1, 1], [0, 0]]
    assert v[0].tobytes() == v[2].tobytes() and not v[3].any()
    assert v[:, :, 0].tolist() == [[3.0, 4.0], [0.0, 1.0], [3.0, 4.0], [0.0, 0.0]]


@pytest.mark.parametrize("t,v", [(4, 1), (POD, 1 << 29), (SVC, (1 << 29) + 5)])
def test_malformed_keys(t, v):
    ends = np.zeros(1, dtype=abi.NODE_ENDS)
    ends["type"], ends["value"] = t, v
    with pytest.raises(ValueError):
        nsr.ends_keys(ends)


def test_outbound_values_may_use_every_bit():
    ends = np.zeros(2, dtype=abi.NODE_ENDS)
    ends["type"], ends["value"] = [OUT, HOST], [0xFFFFFFFF, 1 << 31]
    assert nsr.ends_keys(ends).tolist() == [key(OUT, 0xFFFFFFFF), key(HOST, 1 << 31)]


def test_records_and_top_order():
    ents = [rows(row(POD, 1, SVC, 2, count=c2), row(POD, 1, SVC, 3, count=c3)) for c2, c3 in ((1, 9), (2, 9), (4, 9))]
    rec, y, p = nsr.expect(ents, ents[-1], IN, C, 3, stat=abi.TREND_SHIFT, recent=1)
    assert nsr.node_keys(rec).tolist() == [key(POD, 1), key(SVC, 2), key(SVC, 3)]
    assert rec["index"].tolist() == [0, 1, 2] and rec["valid"].tolist() == [0, 1, 1]
    assert rec["trend"].tolist() == [0.0, 2.5, 0.0] and rec["before"].tolist() == [0.0, 1.5, 9.0]
    idx, above = nsr.top(rec, 5)
    assert idx.tolist() == [1, 2] and above == 2   # ties (none here) go by index; the invalid pod is never eligible
    assert rec.itemsize == 48 and rec["_pad0"].tolist() == [0, 0, 0] and rec["_pad2"].tolist() == [0, 0, 0]
