"""CPU: tests/group_series_ref.py, the §26 reference of the group series and group trends, against the §19 and §22
references under an empty map and against series derived by hand: a deployment whose pods are replaced mid-history,
an internal g -> g row counted on both sides of its group, a key naming a mapped pod, and the §26 key rules."""
import numpy as np

import group_ref as gr
import group_series_ref as gsr
import metric_ref as mr
import node_ref as nr
import node_series_ref as nsr
import series_ref as sr
from alaz_b200 import abi
from change_ref import row_keys

POD, SVC, OUT, GRP = abi.NODE_POD, abi.NODE_SVC, abi.NODE_OUTBOUND, abi.NODE_GROUP
IN, OUTS = abi.SIDE_IN, abi.SIDE_OUT
C, E = abi.METRIC_COUNT, abi.METRIC_ERR5XX
P99 = (abi.METRIC_QUANTILE, 0.99)


def row(ft, f, tt, t, count=0, err=0, lat=0, cells=None):
    r = np.zeros(1, dtype=abi.EDGE_OUT)
    r["from_type"], r["from"], r["to_type"], r["to"] = ft, f, tt, t
    r["count"], r["err5xx"], r["lat_sum_ns"] = count, err, lat
    for b, c in (cells or {}).items():
        r["hist"][0, b] = c
    return r


def rows(*rs):
    if not rs:
        return np.zeros(0, dtype=abi.EDGE_OUT)
    out = np.concatenate(rs)
    return out[np.argsort(row_keys(out), kind="stable")]   # an entry's rows ascend in packed key


def key(t, v):
    return (t << 32) | v


def random_entries(seed, n_entries=5, n_rows=40):
    rng = np.random.default_rng(seed)
    ents = []
    for _ in range(n_entries):
        rs = {}
        for _ in range(n_rows):
            f, t, tt = int(rng.integers(0, 12)), int(rng.integers(0, 12)), int(rng.choice([POD, SVC, OUT]))
            rs[(f, tt, t)] = row(POD, f, tt, t, count=int(rng.integers(1, 50)), err=int(rng.integers(0, 3)),
                                 cells={int(rng.integers(0, abi.NB)): int(rng.integers(1, 50))})
        ents.append(rows(*rs.values()))
    return ents


def test_empty_map_equals_the_node_and_edge_series():
    ents = random_entries(1)
    src = ents[-1]
    specs = [C, E, P99]
    keys = nr.keys(src)
    for side in (IN, OUTS):
        want = nsr.series(ents, keys, side, specs)
        got = gsr.node_series(ents, keys, side, specs)
        assert all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(got, want))
    g = gsr.source_edges(src)
    order = np.argsort(row_keys(src), kind="stable")
    # §24 order is (from key, to key); §19 order is packed-key order: the same rows, permuted
    perm = [int(np.flatnonzero(row_keys(g) == k)[0]) for k in row_keys(src)[order]]
    vs, ps = sr.series(ents, row_keys(src)[order], specs)
    vg, pg = gsr.edge_series(ents, *gsr.row_ends(g), specs)
    assert np.array_equal(vg[perm].view(np.uint64), vs.view(np.uint64)) and np.array_equal(pg[perm], ps)


def test_deployment_replaced_mid_history_is_present_at_every_point():
    # deployment 10 = pods 1, 2 in entries 0..1, then pods 3, 4 in entries 2..3; every pod calls service 9
    gmap = gr.make_map([(POD, 1), (POD, 2), (POD, 3), (POD, 4)], [10, 10, 10, 10])
    ents = [rows(row(POD, 1, SVC, 9, count=2, cells={5: 2}), row(POD, 2, SVC, 9, count=3, cells={60: 3})),
            rows(row(POD, 1, SVC, 9, count=4, cells={5: 4}), row(POD, 2, SVC, 9, count=1, cells={60: 1})),
            rows(row(POD, 3, SVC, 9, count=5, cells={5: 5}), row(POD, 4, SVC, 9, count=6, cells={60: 6})),
            rows(row(POD, 3, SVC, 9, count=7, cells={5: 7}), row(SVC, 9, POD, 4, count=8, cells={60: 8}))]
    v, p = gsr.node_series(ents, [key(GRP, 10)], OUTS, [C], gmap)
    assert p.tolist() == [[1, 1, 1, 1]] and v[0, :, 0].tolist() == [5.0, 5.0, 11.0, 7.0]
    v, p = gsr.node_series(ents, [key(GRP, 10)], IN, [C], gmap)
    assert p.tolist() == [[0, 0, 0, 1]] and v[0, :, 0].tolist() == [0.0, 0.0, 0.0, 8.0]
    # the deployment's p99 is the quantile of the summed histogram, not of any pod's
    v, _ = gsr.node_series(ents, [key(GRP, 10)], OUTS, [P99], gmap)
    for j in range(3):
        summed = gr.group(ents[j], gmap)[0]
        assert v[0, j, 0] == mr.values(summed[summed["from_type"] == GRP], P99)[0]
    # a pod's own §22 series is present only in its own entries
    _, p = nsr.series(ents, [key(POD, 1), key(POD, 3)], OUTS, [C])
    assert p.tolist() == [[1, 1, 0, 0], [0, 0, 1, 1]]
    # the group edge (g10 -> svc 9)
    v, p = gsr.edge_series(ents, [key(GRP, 10)], [key(SVC, 9)], [C], gmap)
    assert p.tolist() == [[1, 1, 1, 1]] and v[0, :, 0].tolist() == [5.0, 5.0, 11.0, 7.0]
    # with the map, the deployment is one record with four points; a slope over them is defined
    rec, y, pr = gsr.node_expect(ents, ents[-1], OUTS, C, 4, gmap, stat=abi.TREND_SLOPE)
    g = rec[nsr.node_keys(rec) == np.uint64(key(GRP, 10))][0]
    assert (g["valid"], g["used"]) == (1, 4)


def test_internal_row_counts_on_both_sides_of_its_group():
    gmap = gr.make_map([(POD, 1), (POD, 2)], [3, 3])
    ents = [rows(row(POD, 1, POD, 2, count=4, err=1))]
    for side in (IN, OUTS):
        v, p = gsr.node_series(ents, [key(GRP, 3)], side, [C, E], gmap)
        assert p.tolist() == [[1]] and v[0, 0].tolist() == [4.0, 1.0]
    v, p = gsr.edge_series(ents, [key(GRP, 3)], [key(GRP, 3)], [C], gmap)
    assert p.tolist() == [[1]] and v[0, 0, 0] == 4.0


def test_key_naming_a_mapped_pod_is_absent_everywhere():
    gmap = gr.make_map([(POD, 1)], [5])
    ents = [rows(row(POD, 1, SVC, 9, count=2)), rows(row(POD, 1, SVC, 9, count=3))]
    for side in (IN, OUTS):
        v, p = gsr.node_series(ents, [key(POD, 1)], side, [C], gmap)
        assert p.tolist() == [[0, 0]] and v.tolist() == [[[0.0], [0.0]]]
    v, p = gsr.edge_series(ents, [key(POD, 1)], [key(SVC, 9)], [C], gmap)
    assert p.tolist() == [[0, 0]]
    v, p = gsr.edge_series(ents, [key(GRP, 5), key(GRP, 5)], [key(SVC, 9), key(SVC, 9)], [C], gmap)
    assert p.tolist() == [[1, 1], [1, 1]] and v[:, :, 0].tolist() == [[2.0, 3.0], [2.0, 3.0]]


def test_key_rules():
    assert gsr.pack_node(GRP, (1 << 29) - 1) == key(GRP, (1 << 29) - 1)
    assert gsr.pack_node(GRP, 1 << 29) is None and gsr.pack_node(5, 0) is None
    assert gsr.pack_node(POD, 1 << 29) is None and gsr.pack_node(OUT, 0xFFFFFFFF) == key(OUT, 0xFFFFFFFF)
    # no group end: §19's rules (a pod end is needed)
    assert gsr.pack_edge(SVC, 1, OUT, 2) is None
    assert gsr.pack_edge(POD, 1, SVC, 2) == (key(POD, 1), key(SVC, 2))
    # a group end: two valid node keys
    assert gsr.pack_edge(GRP, 1, OUT, 2) == (key(GRP, 1), key(OUT, 2))
    assert gsr.pack_edge(GRP, 1, SVC, 1 << 29) is None and gsr.pack_edge(GRP, 1 << 29, POD, 0) is None
