"""CPU: tests/node_change_ref.py, the §23 reference of the node change calls, against lists derived by hand: a node on
IN only in the source and on OUT only in the baseline, a self-loop, pod 7 against service 7 and outbound v against
Host-keyed v, RATIO with a zero base and with both values zero, counts divided by windows and quantiles not, empty
sides, every presence mask and ties in the top."""
import numpy as np
import pytest

import node_change_ref as ncr
import node_ref
from alaz_b200 import abi

POD, SVC, OUT, HOST = 0, 1, 2, 3
IN, OUTS = abi.SIDE_IN, abi.SIDE_OUT
BOTH, NEW, GONE = abi.PRESENT_BOTH, abi.PRESENT_NEW, abi.PRESENT_GONE
DELTA, DROP, RATIO = abi.CHANGE_DELTA, abi.CHANGE_DROP, abi.CHANGE_RATIO
A = abi.ABSENT
EMPTY = np.zeros(0, dtype=abi.EDGE_OUT)


def rows(*spec):
    """EDGE_OUT rows from (from_type, from, to_type, to, count, err5xx[, {cell: n}]) tuples, in the given order"""
    out = np.zeros(len(spec), dtype=abi.EDGE_OUT)
    for i, s in enumerate(spec):
        out[i]["from_type"], out[i]["from"], out[i]["to_type"], out[i]["to"] = s[:4]
        out[i]["count"], out[i]["err5xx"] = s[4], s[5]
        for b, c in (s[6] if len(s) > 6 else {}).items():
            out[i]["hist"][b] = c
    return out


def recs(lst):
    """[(type, node, presence, index, base_index, value, base_value, change)]"""
    return [(int(r["type"]), int(r["node"]), int(r["presence"]), int(r["index"]), int(r["base_index"]),
             float(r["value"]), float(r["base_value"]), float(r["change"])) for r in lst]


def test_in_only_in_the_source_and_out_only_in_the_baseline():
    src = rows((POD, 1, SVC, 5, 10, 0))        # source nodes: pod 1 (OUT), service 5 (IN)
    base = rows((SVC, 5, POD, 2, 4, 0))        # baseline nodes: pod 2 (IN), service 5 (OUT)
    lst, info = ncr.changes(src, base, IN, abi.METRIC_COUNT, DELTA, 7)
    assert recs(lst) == [(POD, 2, GONE, A, 0, 0.0, 4.0, -4.0), (SVC, 5, NEW, 1, A, 10.0, 0.0, 10.0)]
    assert (info["source_rows"], info["base_rows"], info["both"], info["added"], info["gone"]) == (1, 1, 0, 1, 1)
    lst, info = ncr.changes(src, base, OUTS, abi.METRIC_COUNT, DELTA, 7)
    assert recs(lst) == [(POD, 1, NEW, 0, A, 10.0, 0.0, 10.0), (SVC, 5, GONE, A, 1, 0.0, 4.0, -4.0)]
    assert (info["both"], info["added"], info["gone"], info["listed"]) == (0, 1, 1, 2)
    assert np.all(lst["_pad0"] == 0) and np.all(lst["_pad1"] == 0) and np.all(lst["_pad2"] == 0)


def test_self_loop_is_a_member_on_both_sides():
    src, base = rows((POD, 3, POD, 3, 5, 0)), rows((POD, 3, POD, 3, 2, 0))
    for side in (IN, OUTS):
        assert recs(ncr.changes(src, base, side, abi.METRIC_COUNT, DELTA, 7)[0]) == [(POD, 3, BOTH, 0, 0, 5.0, 2.0,
                                                                                       3.0)]


def test_same_value_different_type_do_not_match():
    src = rows((POD, 1, POD, 7, 2, 0), (POD, 1, OUT, 9, 6, 0))
    base = rows((POD, 1, SVC, 7, 3, 0), (POD, 1, HOST, 9, 8, 0))
    lst, info = ncr.changes(src, base, IN, abi.METRIC_COUNT, DELTA, 7)
    assert recs(lst) == [(POD, 7, NEW, 1, A, 2.0, 0.0, 2.0), (SVC, 7, GONE, A, 1, 0.0, 3.0, -3.0),
                         (OUT, 9, NEW, 2, A, 6.0, 0.0, 6.0), (HOST, 9, GONE, A, 2, 0.0, 8.0, -8.0)]
    assert info["both"] == 0 and info["listed"] == 4
    # pod 1 sends to all four: one node, BOTH on OUT, with the sums of its rows
    assert recs(ncr.changes(src, base, OUTS, abi.METRIC_COUNT, DROP, 7)[0]) == [(POD, 1, BOTH, 0, 0, 8.0, 11.0, 3.0)]


def test_ratio_with_a_zero_base_and_with_both_zero():
    src = rows((POD, 1, SVC, 2, 10, 2), (POD, 1, SVC, 3, 10, 0))
    base = rows((POD, 1, SVC, 2, 10, 0), (POD, 1, SVC, 3, 10, 0))
    lst, _ = ncr.changes(src, base, IN, abi.METRIC_ERR5XX, RATIO, 7)
    assert [float(c) for c in lst["change"]] == [np.inf, 1.0]
    lst, _ = ncr.changes(base, src, IN, abi.METRIC_ERR5XX, RATIO, 7)
    assert [float(c) for c in lst["change"]] == [0.0, 1.0]


def test_counts_are_divided_by_windows_and_quantiles_are_not():
    src = rows((POD, 1, SVC, 2, 50, 5, {10: 50}))
    base = rows((POD, 1, SVC, 2, 600, 60, {10: 600}))
    lst, info = ncr.changes(src, base, IN, abi.METRIC_COUNT, DELTA, 7, src_windows=5, base_windows=60)
    assert (lst[0]["value"], lst[0]["base_value"], lst[0]["change"]) == (10.0, 10.0, 0.0)
    assert (info["source_windows"], info["base_windows"]) == (5, 60)
    lst, _ = ncr.changes(src, base, IN, abi.METRIC_ERR5XX, RATIO, 7, src_windows=5, base_windows=60)
    assert (lst[0]["value"], lst[0]["base_value"], lst[0]["change"]) == (1.0, 1.0, 1.0)
    q = (abi.METRIC_QUANTILE, 0.99)
    lst, _ = ncr.changes(src, base, IN, q, DELTA, 7, src_windows=5, base_windows=60)
    p99 = node_ref.values(node_ref.group(src), IN, q)[1]
    assert p99 > 0 and lst[0]["value"] == p99 and lst[0]["base_value"] == p99 and lst[0]["change"] == 0.0
    # one rounding: 7 / 3 is the float64 quotient
    lst, _ = ncr.changes(rows((POD, 1, SVC, 2, 7, 0)), base, IN, abi.METRIC_COUNT, DELTA, 7, src_windows=3)
    assert lst[0]["value"] == np.float64(7.0) / np.float64(3.0)


def test_empty_sides():
    src = rows((POD, 1, SVC, 2, 3, 0), (POD, 4, SVC, 2, 1, 0))
    lst, info = ncr.changes(EMPTY, EMPTY, IN, abi.METRIC_COUNT, DELTA, 7)
    assert len(lst) == 0 and info["listed"] == 0 and info["source_rows"] == 0
    lst, info = ncr.changes(src, EMPTY, OUTS, abi.METRIC_COUNT, DELTA, 7)
    assert recs(lst) == [(POD, 1, NEW, 0, A, 3.0, 0.0, 3.0), (POD, 4, NEW, 1, A, 1.0, 0.0, 1.0)]
    assert info["added"] == 2 and info["source_rows"] == 2
    lst, info = ncr.changes(EMPTY, src, IN, (abi.METRIC_QUANTILE, 0.5), DROP, 7)
    assert recs(lst) == [(SVC, 2, GONE, A, 2, 0.0, 0.0, 0.0)] and info["gone"] == 1 and info["base_rows"] == 1


SRC = rows((POD, 1, SVC, 2, 8, 0), (POD, 1, SVC, 3, 4, 0), (POD, 1, SVC, 4, 5, 0))
BASE = rows((POD, 1, SVC, 2, 8, 0), (POD, 1, SVC, 3, 1, 0), (POD, 1, SVC, 9, 6, 0))


@pytest.mark.parametrize("mask", range(1, 8))
def test_every_presence_mask(mask):
    lst, info = ncr.changes(SRC, BASE, IN, abi.METRIC_COUNT, DELTA, mask)
    want = {BOTH: 2, NEW: 1, GONE: 1}
    assert info["listed"] == sum(n for bit, n in want.items() if mask & bit)
    assert set(int(p) for p in lst["presence"]) == {bit for bit in want if mask & bit}
    assert (info["both"], info["added"], info["gone"]) == (2, 1, 1)   # before the filter
    assert np.all(lst["node"][1:] > lst["node"][:-1])                 # ascending key (all services)


def test_top_ranks_changes_then_list_position():
    lst, info = ncr.top(SRC, BASE, IN, abi.METRIC_COUNT, DELTA, 7, 10, -np.inf)
    assert [float(c) for c in lst["change"]] == [5.0, 3.0, 0.0, -6.0] and info["above"] == 4
    lst, info = ncr.top(SRC, BASE, IN, abi.METRIC_COUNT, DELTA, 7, 1, 0.0)
    assert list(lst["node"]) == [4] and info["above"] == 3               # +0 >= +0; -6 is not eligible
    lst, info = ncr.top(SRC, BASE, IN, abi.METRIC_COUNT, DELTA, 7, 5, np.inf)
    assert len(lst) == 0 and info["above"] == 0
    # ties: equal changes keep their list order
    src = rows(*[(POD, 1, SVC, t, 5, 0) for t in range(6)])
    lst, _ = ncr.top(src, EMPTY, IN, abi.METRIC_COUNT, DELTA, 7, 4, 0.0)
    assert list(lst["node"]) == [0, 1, 2, 3]
