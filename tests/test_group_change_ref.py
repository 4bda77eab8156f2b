"""CPU: tests/group_change_ref.py on hand-derived cases: a rolling deploy that only the groups survive, a group that is
a member on IN only, RATIO against a zero baseline, and ends whose node keys collide when a pair is packed into 64
bits."""
import numpy as np

import change_ref
import group_change_ref as gcr
import group_ref as gr
import metric_ref
import node_change_ref as ncr
from alaz_b200 import abi

POD, SVC, OUTB, GRP = abi.NODE_POD, abi.NODE_SVC, abi.NODE_OUTBOUND, abi.NODE_GROUP
IN, OUT = abi.SIDE_IN, abi.SIDE_OUT
Q = abi.METRIC_QUANTILE
BOTH, NEW, GONE = abi.PRESENT_BOTH, abi.PRESENT_NEW, abi.PRESENT_GONE
ALL = abi.PRESENT_ALL


def rows(*specs):
    """EDGE_OUT rows from (from_type, from, to_type, to, count, err5xx, bucket) tuples: count latencies in one bucket"""
    r = np.zeros(len(specs), dtype=abi.EDGE_OUT)
    for i, (ft, f, tt, t, c, e, b) in enumerate(specs):
        r[i]["from_type"], r[i]["from"], r[i]["to_type"], r[i]["to"] = ft, f, tt, t
        r[i]["count"], r[i]["err5xx"], r[i]["lat_sum_ns"] = c, e, 1000 * c
        r[i]["hist"][b] = c
    return r


def p99_of(*cells):
    """the §17 p99 of one row whose histogram holds (bucket, count) cells"""
    r = np.zeros(1, dtype=abi.EDGE_OUT)
    for b, c in cells:
        r[0]["hist"][b] += c
        r[0]["count"] += c
    return float(metric_ref.values(r, (Q, 0.99))[0])


# web pod 1 calls the api pods; the baseline's api-1 and api-2 (pods 10, 11) are replaced by api-3 and api-4 (12, 13)
BASE = rows((POD, 1, POD, 10, 60, 1, 3), (POD, 1, POD, 11, 40, 0, 4))
SRC = rows((POD, 1, POD, 12, 70, 5, 8), (POD, 1, POD, 13, 50, 2, 9))
DEPLOY = gr.make_map([(POD, 1), (POD, 10), (POD, 11), (POD, 12), (POD, 13)], [3, 7, 7, 7, 7])


def test_a_rolling_deploy_is_both_only_as_a_group():
    pods, _ = ncr.changes(SRC, BASE, IN, abi.METRIC_COUNT, abi.CHANGE_DELTA, ALL)
    assert sorted(pods["presence"].tolist()) == [NEW, NEW, GONE, GONE]
    lst, info = gcr.node_changes(SRC, BASE, DEPLOY, IN, (Q, 0.99), abi.CHANGE_DELTA, ALL)
    assert len(lst) == 1 and info["both"] == 1 and info["source_rows"] == info["base_rows"] == 1
    r = lst[0]
    assert (r["type"], r["node"], r["presence"], r["index"], r["base_index"]) == (GRP, 7, BOTH, 1, 1)
    assert r["value"] == p99_of((8, 70), (9, 50)) and r["base_value"] == p99_of((3, 60), (4, 40))
    assert r["change"] == r["value"] - r["base_value"] > 0
    lst, _ = gcr.node_changes(SRC, BASE, DEPLOY, IN, abi.METRIC_COUNT, abi.CHANGE_DELTA, ALL, 5, 60)
    assert lst[0]["value"] == 120 / 5 and lst[0]["base_value"] == 100 / 60
    edges, info = gcr.edge_changes(SRC, BASE, DEPLOY, abi.METRIC_ERR5XX, abi.CHANGE_DELTA, ALL)
    assert len(edges) == 1 and info == dict(source_rows=1, base_rows=1, both=1, added=0, gone=0, listed=1, above=0,
                                            source_windows=1, base_windows=1)
    e = edges[0]
    assert (e["from_type"], e["from"], e["to_type"], e["to"], e["presence"]) == (GRP, 3, GRP, 7, BOTH)
    assert (e["value"], e["base_value"], e["change"]) == (7.0, 1.0, 6.0)


def test_a_group_with_rows_on_in_only():
    # group 3 (web) only calls, group 7 (api) only serves: on OUT, 7 is no member on either side and is not listed
    lst, info = gcr.node_changes(SRC, BASE, DEPLOY, OUT, abi.METRIC_COUNT, abi.CHANGE_DELTA, ALL)
    assert lst["node"].tolist() == [3] and lst["index"].tolist() == [0] and lst["base_index"].tolist() == [0]
    assert info["source_rows"] == info["base_rows"] == 1
    # api serves only in the source: NEW on IN, and not GONE on OUT where it never had rows
    base = rows((POD, 1, SVC, 5, 10, 0, 2))
    lst, _ = gcr.node_changes(SRC, base, DEPLOY, IN, abi.METRIC_COUNT, abi.CHANGE_DELTA, ALL)
    assert [(int(x["type"]), int(x["node"]), int(x["presence"])) for x in lst] == [(SVC, 5, GONE), (GRP, 7, NEW)]
    lst, _ = gcr.node_changes(SRC, base, DEPLOY, OUT, abi.METRIC_COUNT, abi.CHANGE_DELTA, ALL)
    assert [(int(x["node"]), int(x["presence"])) for x in lst] == [(3, BOTH)]


def test_ratio_against_a_zero_baseline():
    src = rows((POD, 1, POD, 12, 70, 5, 8), (POD, 2, POD, 13, 50, 0, 9))
    base = rows((POD, 1, POD, 10, 60, 0, 3), (POD, 2, POD, 11, 40, 0, 4))
    gmap = gr.make_map([(POD, 1), (POD, 2), (POD, 10), (POD, 11), (POD, 12), (POD, 13)], [3, 4, 7, 7, 7, 7])
    lst, _ = gcr.edge_changes(src, base, gmap, abi.METRIC_ERR5XX, abi.CHANGE_RATIO, ALL)
    assert [(int(x["from"]), int(x["to"])) for x in lst] == [(3, 7), (4, 7)]
    assert lst["change"][0] == np.inf and lst["change"][1] == 1.0   # 5 / 0 and 0 / 0
    assert lst["base_value"].tolist() == [0.0, 0.0]


def test_ends_that_collide_in_64_bits_stay_apart():
    # from group 1 to outbound 5, to group 5, and to outbound 2^31 + 5: three different pairs whose to values agree in
    # their low 31 bits; a naive (from << 32 | to) packing would match them
    src = rows((POD, 1, OUTB, 5, 10, 0, 1), (POD, 1, OUTB, (1 << 31) | 5, 20, 0, 1))
    base = rows((POD, 1, POD, 9, 30, 0, 1), (POD, 1, OUTB, (1 << 31) | 5, 40, 0, 1))
    gmap = gr.make_map([(POD, 1), (POD, 9)], [1, 5])
    lst, info = gcr.edge_changes(src, base, gmap, abi.METRIC_COUNT, abi.CHANGE_DELTA, ALL)
    got = [(int(x["to_type"]), int(x["to"]), int(x["presence"]), int(x["index"]), int(x["base_index"])) for x in lst]
    assert got == [(OUTB, 5, NEW, 0, abi.ABSENT), (OUTB, (1 << 31) | 5, BOTH, 1, 0), (GRP, 5, GONE, abi.ABSENT, 1)]
    assert info["both"] == 1 and info["added"] == 1 and info["gone"] == 1
    assert lst["change"].tolist() == [10.0, -20.0, -30.0]
    # presence masks filter the same union
    for mask in range(1, 8):
        sub, _ = gcr.edge_changes(src, base, gmap, abi.METRIC_COUNT, abi.CHANGE_DELTA, mask)
        assert sub.tobytes() == lst[(lst["presence"] & mask) != 0].tobytes()


def test_an_empty_map_is_the_edge_changes_in_ends_order():
    src = rows((POD, 1, SVC, 2, 5, 0, 1), (SVC, 3, POD, 1, 7, 0, 2), (POD, 4, OUTB, 9, 1, 0, 3))
    base = rows((POD, 1, SVC, 2, 6, 0, 1), (POD, 4, OUTB, 8, 2, 0, 3))
    ka, kb = change_ref.row_keys(src), change_ref.row_keys(base)
    src, base = src[np.argsort(ka)], base[np.argsort(kb)]
    want, _ = change_ref.changes(src, base, abi.METRIC_COUNT, abi.CHANGE_DELTA, ALL)
    got, _ = gcr.edge_changes(src, base, gr.EMPTY, abi.METRIC_COUNT, abi.CHANGE_DELTA, ALL)
    f, t = gcr.ends_keys(want)
    perm = np.lexsort((t, f))
    assert got[["from_type", "to_type", "from", "to", "presence", "value", "base_value", "change"]].tolist() == \
        want[perm][["from_type", "to_type", "from", "to", "presence", "value", "base_value", "change"]].tolist()
    top, info = gcr.top(got, _, 2, -np.inf)
    assert top["change"].tolist() == sorted(got["change"].tolist(), reverse=True)[:2] and info["above"] == len(got)
