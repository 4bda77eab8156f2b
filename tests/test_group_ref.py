"""CPU: tests/group_ref.py, the §24 reference of the group calls, against group edges derived by hand: an empty map,
A -> B and B -> A of one group, pod 7 against service 7, outbound v against Host-keyed v, a group id equal to a pod id,
an unmapped end beside a mapped one, sums that wrap 2^64 and cells that wrap 2^32, and the group nodes over them."""
import numpy as np
import pytest

import group_ref as gr
import node_ref as nr
from alaz_b200 import abi

POD, SVC, OUT, HOST, GRP = 0, 1, 2, 3, abi.NODE_GROUP
IN, OUTS = abi.SIDE_IN, abi.SIDE_OUT


def row(ft, f, tt, t, count=0, err=0, lat=0, cells=None):
    r = np.zeros(1, dtype=abi.EDGE_OUT)
    r["from_type"], r["from"], r["to_type"], r["to"] = ft, f, tt, t
    r["count"], r["err5xx"], r["lat_sum_ns"] = count, err, lat
    for b, c in (cells or {}).items():
        r["hist"][0, b] = c
    return r


def rows(*rs):
    return np.concatenate(rs)


def heads(e):
    return [(int(a), int(b), int(c), int(d)) for a, b, c, d in zip(e["from_type"], e["from"], e["to_type"], e["to"])]


def test_node_group_constant():
    assert abi.NODE_GROUP == 4 and abi.NODE_GROUP > abi.NODE_OUTBOUND_HOST


def test_empty_map_reorders_packed_key_order_into_node_key_order():
    # the rows in packed-key order (§3: rev | other kind | pod | other value): every pod -> service row before every
    # pod -> outbound row, the reversed service -> pod row last. Node-key order sorts on the from end first.
    r = rows(row(POD, 3, SVC, 1, count=4), row(POD, 9, SVC, 1, count=1), row(POD, 3, OUT, 0x0A000001, count=3),
             row(SVC, 2, POD, 9, count=2))
    e, info = gr.group(r)
    assert heads(e) == [(POD, 3, SVC, 1), (POD, 3, OUT, 0x0A000001), (POD, 9, SVC, 1), (SVC, 2, POD, 9)]
    assert list(e["count"]) == [4, 3, 1, 2]
    assert info == dict(source_rows=4, mapped_ends=0, edges=4, internal=0)


def test_both_directions_of_one_group_land_on_one_internal_row():
    gmap = gr.make_map([(POD, 1), (POD, 2)], [50, 50])
    r = rows(row(POD, 1, POD, 2, count=10, err=1, lat=100, cells={3: 10}),
             row(POD, 2, POD, 1, count=5, err=2, lat=40, cells={3: 1, 9: 4}))
    e, info = gr.group(r, gmap)
    assert heads(e) == [(GRP, 50, GRP, 50)]
    assert (e["count"][0], e["err5xx"][0], e["lat_sum_ns"][0], e["hist"][0, 3], e["hist"][0, 9]) == (15, 3, 140, 11, 4)
    assert info == dict(source_rows=2, mapped_ends=4, edges=1, internal=2)
    n = nr.group(e)
    assert len(n) == 1 and n["in_edges"][0] == 1 and n["out_edges"][0] == 1   # counts on both sides
    assert n["in"]["count"][0] == n["out"]["count"][0] == 15


def test_pod_and_service_with_one_id_are_different_members():
    gmap = gr.make_map([(POD, 7), (SVC, 7)], [1, 2])
    r = rows(row(POD, 7, SVC, 7, count=3), row(POD, 8, SVC, 7, count=4), row(POD, 8, POD, 7, count=5))
    e, info = gr.group(r, gmap)
    assert heads(e) == [(POD, 8, GRP, 1), (POD, 8, GRP, 2), (GRP, 1, GRP, 2)]
    assert list(e["count"]) == [5, 4, 3]
    assert info["mapped_ends"] == 4 and info["internal"] == 0


def test_outbound_and_host_keyed_value_are_mapped_apart():
    gmap = gr.make_map([(OUT, 77), (HOST, 77)], [900, 901])
    r = rows(row(POD, 1, OUT, 77, count=1), row(POD, 1, HOST, 77, count=2), row(POD, 2, OUT, 77, count=4))
    e, _ = gr.group(r, gmap)
    assert heads(e) == [(POD, 1, GRP, 900), (POD, 1, GRP, 901), (POD, 2, GRP, 900)]
    assert list(e["count"]) == [1, 2, 4]


def test_group_id_equal_to_a_pod_id_is_a_distinct_node():
    gmap = gr.make_map([(POD, 1)], [3])
    r = rows(row(POD, 1, POD, 3, count=1), row(POD, 3, POD, 1, count=2))
    e, info = gr.group(r, gmap)
    assert heads(e) == [(POD, 3, GRP, 3), (GRP, 3, POD, 3)]
    assert info["internal"] == 0
    n = nr.group(e)
    assert [(int(t), int(v)) for t, v in zip(n["type"], n["value"])] == [(POD, 3), (GRP, 3)]   # the group is last


def test_unmapped_end_beside_a_mapped_one():
    gmap = gr.make_map([(POD, 1), (POD, 2)], [10, 10])
    r = rows(row(POD, 1, SVC, 5, count=1), row(POD, 2, SVC, 5, count=2), row(POD, 3, SVC, 5, count=4),
             row(POD, 2, SVC, 6, count=8))
    e, info = gr.group(r, gmap)
    assert heads(e) == [(POD, 3, SVC, 5), (GRP, 10, SVC, 5), (GRP, 10, SVC, 6)]
    assert list(e["count"]) == [4, 3, 8]
    assert info == dict(source_rows=4, mapped_ends=3, edges=3, internal=0)


def test_sums_wrap_2_64_and_cells_wrap_2_32():
    gmap = gr.make_map([(POD, 1), (POD, 2)], [0, 0])
    big = (1 << 64) - 5
    r = rows(row(POD, 1, SVC, 9, count=big, err=big, lat=big, cells={0: (1 << 32) - 1, 63: 7}),
             row(POD, 2, SVC, 9, count=10, err=6, lat=5, cells={0: 3, 63: (1 << 32) - 7}))
    e, _ = gr.group(r, gmap)
    assert heads(e) == [(GRP, 0, SVC, 9)]
    assert (int(e["count"][0]), int(e["err5xx"][0]), int(e["lat_sum_ns"][0])) == (5, 1, 0)
    assert (int(e["hist"][0, 0]), int(e["hist"][0, 63])) == (2, 0)


def test_group_nodes_sum_every_member_and_a_p99_of_the_summed_histogram():
    # two pods of one deployment with disjoint latency buckets: the group's p99 is neither pod's
    gmap = gr.make_map([(POD, 1), (POD, 2)], [5, 5])
    r = rows(row(POD, 9, POD, 1, count=100, cells={2: 100}), row(POD, 9, POD, 2, count=100, cells={40: 100}))
    n = gr.nodes(r, gmap)
    g = int(np.flatnonzero(n["type"] == GRP)[0])
    assert n["in"]["count"][g] == 200 and n["in_edges"][g] == 1
    spec = (abi.METRIC_QUANTILE, 0.99)
    pods = nr.values(nr.group(r), IN, spec)
    grp = nr.values(n, IN, spec)[g]
    assert grp not in set(pods.tolist())


def test_a_map_with_a_repeated_node_is_refused():
    with pytest.raises(AssertionError):
        gr.make_map([(POD, 1), (POD, 1)], [1, 2])


def test_empty_source():
    e, info = gr.group(np.zeros(0, dtype=abi.EDGE_OUT), gr.make_map([(POD, 1)], [1]))
    assert len(e) == 0 and info == dict(source_rows=0, mapped_ends=0, edges=0, internal=0)
