"""CPU: tests/change_ref.py, the numpy reference of docs/SPEC.md §18, against vectors derived by hand: a new edge, a
gone edge, equal rows (DELTA +0, RATIO 1.0), base 0 with a current value (+inf), a 5-window source against a 60-window
baseline, every presence mask and the info counts."""
import itertools

import numpy as np
import pytest

import change_ref as cr
from alaz_b200 import abi

P, S, O = abi.NODE_POD, abi.NODE_SVC, abi.NODE_OUTBOUND
BOTH, NEW, GONE = abi.PRESENT_BOTH, abi.PRESENT_NEW, abi.PRESENT_GONE
DELTA, DROP, RATIO = abi.CHANGE_DELTA, abi.CHANGE_DROP, abi.CHANGE_RATIO


def rows(*spec):
    """EDGE_OUT rows from (from_type, from, to_type, to, count, err5xx), sorted by packed key."""
    r = np.zeros(len(spec), dtype=abi.EDGE_OUT)
    for i, (ft, f, tt, t, c, e) in enumerate(spec):
        r[i]["from_type"], r[i]["from"], r[i]["to_type"], r[i]["to"] = ft, f, tt, t
        r[i]["count"], r[i]["err5xx"] = c, e
        r[i]["hist"][10] = c
    return r[np.argsort(cr.row_keys(r), kind="stable")]


# base: pod1->svc2 (10, 1), pod1->pod3 (4, 0), svc5->pod1 (reversed; 6, 6)
# src:  pod1->svc2 (10, 1), pod1->pod3 (8, 2), pod1->out 9 (new; 3, 0)
BASE = rows((P, 1, S, 2, 10, 1), (P, 1, P, 3, 4, 0), (S, 5, P, 1, 6, 6))
SRC = rows((P, 1, S, 2, 10, 1), (P, 1, P, 3, 8, 2), (P, 1, O, 9, 3, 0))


def by_edge(lst):
    return {(int(x["from_type"]), int(x["from"]), int(x["to_type"]), int(x["to"])): x for x in lst}


def test_row_keys_are_the_spec_packing():
    k = cr.row_keys(rows((P, 1, S, 2, 1, 0), (S, 5, P, 1, 1, 0)))
    assert sorted(int(x) for x in k) == [(1 << 61) | (1 << 32) | 2, (1 << 63) | (1 << 61) | (1 << 32) | 5]


def test_new_gone_and_both_rows_with_delta():
    lst, info = cr.changes(SRC, BASE, abi.METRIC_COUNT, DELTA, BOTH | NEW | GONE)
    assert info == dict(source_rows=3, base_rows=3, both=2, added=1, gone=1, listed=4, above=0, source_windows=1,
                        base_windows=1)
    k = cr.row_keys(lst)
    assert np.all(k[1:] > k[:-1])                                              # ascending key order
    e = by_edge(lst)
    same, grew, new, gone = e[(P, 1, S, 2)], e[(P, 1, P, 3)], e[(P, 1, O, 9)], e[(S, 5, P, 1)]
    assert same["presence"] == BOTH and same["value"] == 10 and same["base_value"] == 10
    assert same["change"] == 0.0 and not np.signbit(same["change"])            # x - x is +0
    assert grew["presence"] == BOTH and grew["change"] == 4.0
    assert new["presence"] == NEW and new["base_index"] == abi.ABSENT and new["base_value"] == 0 and new["change"] == 3
    assert gone["presence"] == GONE and gone["index"] == abi.ABSENT and gone["value"] == 0 and gone["change"] == -6
    for x in lst:   # indices point at the rows the record came from
        if x["index"] != abi.ABSENT:
            assert SRC[x["index"]]["from"] == x["from"] and SRC[x["index"]]["to"] == x["to"]
        if x["base_index"] != abi.ABSENT:
            assert BASE[x["base_index"]]["from"] == x["from"] and BASE[x["base_index"]]["to"] == x["to"]


def test_drop_and_ratio():
    e = by_edge(cr.changes(SRC, BASE, abi.METRIC_COUNT, DROP, 7)[0])
    assert e[(P, 1, P, 3)]["change"] == -4.0 and e[(S, 5, P, 1)]["change"] == 6.0
    e = by_edge(cr.changes(SRC, BASE, abi.METRIC_COUNT, RATIO, 7)[0])
    assert e[(P, 1, S, 2)]["change"] == 1.0                      # equal rows
    assert e[(P, 1, P, 3)]["change"] == 2.0
    assert e[(P, 1, O, 9)]["change"] == np.inf                   # base 0, value > 0
    assert e[(S, 5, P, 1)]["change"] == 0.0                      # value 0, base > 0
    e = by_edge(cr.changes(SRC, BASE, abi.METRIC_ERR5XX, RATIO, 7)[0])
    assert e[(P, 1, O, 9)]["change"] == 1.0                      # both 0


def test_error_rate_is_not_divided_by_windows():
    e = by_edge(cr.changes(SRC, BASE, abi.METRIC_ERR_RATE, DELTA, 7, src_windows=5, base_windows=60)[0])
    assert e[(P, 1, P, 3)]["value"] == 0.25 and e[(P, 1, P, 3)]["base_value"] == 0.0
    assert e[(S, 5, P, 1)]["base_value"] == 1.0


def test_five_windows_against_sixty_compare_per_window():
    # 5 windows with 50 requests against 60 windows with 600: both 10 per window, no change
    src = rows((P, 1, S, 2, 50, 5))
    base = rows((P, 1, S, 2, 600, 60))
    lst, info = cr.changes(src, base, abi.METRIC_COUNT, DELTA, 7, src_windows=5, base_windows=60)
    assert info["source_windows"] == 5 and info["base_windows"] == 60
    assert lst[0]["value"] == 10.0 and lst[0]["base_value"] == 10.0 and lst[0]["change"] == 0.0
    lst, _ = cr.changes(src, base, abi.METRIC_ERR5XX, RATIO, 7, src_windows=5, base_windows=60)
    assert lst[0]["value"] == 1.0 and lst[0]["base_value"] == 1.0 and lst[0]["change"] == 1.0
    # one rounding: 7 / 3 is the float64 quotient, not a product with 1/3
    lst, _ = cr.changes(rows((P, 1, S, 2, 7, 0)), base, abi.METRIC_COUNT, DELTA, 7, src_windows=3, base_windows=60)
    assert lst[0]["value"] == np.float64(7.0) / np.float64(3.0)


@pytest.mark.parametrize("mask", range(1, 8))
def test_every_presence_mask(mask):
    lst, info = cr.changes(SRC, BASE, abi.METRIC_COUNT, DELTA, mask)
    want = {BOTH: 2, NEW: 1, GONE: 1}
    assert info["listed"] == sum(n for bit, n in want.items() if mask & bit)
    assert set(int(p) for p in lst["presence"]) == {bit for bit in want if mask & bit}
    assert (info["both"], info["added"], info["gone"]) == (2, 1, 1)   # before the filter


def test_empty_sides():
    e = np.zeros(0, dtype=abi.EDGE_OUT)
    lst, info = cr.changes(e, e, abi.METRIC_COUNT, DELTA, 7)
    assert len(lst) == 0 and info["listed"] == 0
    lst, info = cr.changes(SRC, e, abi.METRIC_COUNT, DELTA, 7)
    assert set(lst["presence"]) == {NEW} and info["added"] == 3
    lst, info = cr.changes(e, BASE, (abi.METRIC_QUANTILE, 0.99), DROP, 7)
    assert set(lst["presence"]) == {GONE} and info["gone"] == 3 and np.all(lst["change"] > 0)


def test_top_ranks_changes_then_list_position():
    lst, info = cr.top(SRC, BASE, abi.METRIC_COUNT, DELTA, 7, 10, -np.inf)
    assert list(lst["change"]) == [4.0, 3.0, 0.0, -6.0] and info["above"] == 4
    lst, info = cr.top(SRC, BASE, abi.METRIC_COUNT, DELTA, 7, 1, 0.0)
    assert list(lst["change"]) == [4.0] and info["above"] == 3            # +0 >= +0; -6 is not eligible
    lst, info = cr.top(SRC, BASE, abi.METRIC_COUNT, RATIO, 7, 2, 0.0)
    assert lst[0]["change"] == np.inf and lst[1]["change"] == 2.0
    # ties: equal changes keep their list order
    src = rows(*[(P, 1, S, t, 5, 0) for t in range(6)])
    lst, _ = cr.top(src, np.zeros(0, dtype=abi.EDGE_OUT), abi.METRIC_COUNT, DELTA, 7, 4, 0.0)
    assert list(lst["to"]) == [0, 1, 2, 3]


def test_random_union_against_a_dict_model():
    rng = np.random.default_rng(5)
    for trial in range(20):
        keys = rng.choice(4000, size=rng.integers(0, 300), replace=False)
        a_mask, b_mask = rng.random(len(keys)) < 0.7, rng.random(len(keys)) < 0.7
        def mk(sel):
            r = np.zeros(int(sel.sum()), dtype=abi.EDGE_OUT)
            r["from_type"] = P
            r["from"] = keys[sel] // 64
            r["to_type"] = S
            r["to"] = keys[sel] % 64
            r["count"] = rng.integers(0, 100, len(r))
            r["err5xx"] = r["count"] // 3
            return r[np.argsort(cr.row_keys(r))]
        a, b = mk(a_mask), mk(b_mask)
        wa, wb = int(rng.integers(1, 9)), int(rng.integers(1, 70))
        for spec, mode, mask in itertools.product((abi.METRIC_COUNT, abi.METRIC_ERR_RATE), (DELTA, DROP, RATIO),
                                                  (1, 5, 7)):
            lst, info = cr.changes(a, b, spec, mode, mask, wa, wb)
            da = {int(k): i for i, k in enumerate(cr.row_keys(a))}
            db = {int(k): i for i, k in enumerate(cr.row_keys(b))}
            va, vb = cr.side_values(a, spec, wa), cr.side_values(b, spec, wb)
            want = []
            for k in sorted(set(da) | set(db)):
                p = BOTH if k in da and k in db else NEW if k in da else GONE
                if p & mask:
                    x, y = (va[da[k]] if k in da else 0.0), (vb[db[k]] if k in db else 0.0)
                    want.append((p, da.get(k, abi.ABSENT), db.get(k, abi.ABSENT), x, y,
                                 float(cr.change_of(mode, x, y))))
            got = [(int(r["presence"]), int(r["index"]), int(r["base_index"]), r["value"], r["base_value"],
                    r["change"]) for r in lst]
            assert got == want, (trial, spec, mode, mask)
            assert info["both"] + info["added"] == len(a) and info["both"] + info["gone"] == len(b)
