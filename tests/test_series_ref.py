"""CPU: tests/series_ref.py against hand-derived series (docs/SPEC.md §19)."""
import numpy as np
import pytest

import series_ref as sr
from alaz_b200 import abi
from change_ref import row_keys

POD, SVC, OUT, HOST = abi.NODE_POD, abi.NODE_SVC, abi.NODE_OUTBOUND, abi.NODE_OUTBOUND_HOST
COUNT, ERR, RATE, MEAN = abi.METRIC_COUNT, abi.METRIC_ERR5XX, abi.METRIC_ERR_RATE, abi.METRIC_MEAN_NS


def rows(*specs):
    """EDGE_OUT rows from (from_type, from, to_type, to, count, err5xx, lat_sum_ns), sorted by packed key; all the
    row's events in bucket 10 ([2^13, 1.5 * 2^13))."""
    r = np.zeros(len(specs), dtype=abi.EDGE_OUT)
    for i, (ft, f, tt, t, c, e, lat) in enumerate(specs):
        r[i]["from_type"], r[i]["from"], r[i]["to_type"], r[i]["to"] = ft, f, tt, t
        r[i]["count"], r[i]["err5xx"], r[i]["lat_sum_ns"] = c, e, lat
        r[i]["hist"][10] = c
    return r[np.argsort(row_keys(r), kind="stable")]


def key(ft, f, tt, t):
    return sr.pack_ends(ft, f, tt, t)


def test_an_edge_absent_from_some_entries():
    a = rows((POD, 1, SVC, 2, 4, 1, 400), (POD, 3, SVC, 2, 10, 0, 50))
    b = rows((POD, 3, SVC, 2, 6, 6, 60))
    c = rows((POD, 1, SVC, 2, 8, 2, 1600))
    v, p = sr.series([a, b, c], [key(POD, 1, SVC, 2), key(POD, 3, SVC, 2)], [COUNT, ERR, RATE, MEAN])
    assert p.tolist() == [[1, 0, 1], [1, 1, 0]]
    assert v[0].tolist() == [[4, 1, 0.25, 100], [0, 0, 0, 0], [8, 2, 0.25, 200]]
    assert v[1].tolist() == [[10, 0, 0, 5], [6, 6, 1, 10], [0, 0, 0, 0]]
    assert np.signbit(v[p == 0]).sum() == 0                     # absent points are +0.0


def test_quantile_of_one_bucket():
    a = rows((POD, 1, SVC, 2, 4, 0, 0))
    v, p = sr.series([a], [key(POD, 1, SVC, 2)], [(abi.METRIC_QUANTILE, 0.5), (abi.METRIC_QUANTILE, 1.0)])
    lo, hi = float(1 << 13), 1.5 * (1 << 13)
    assert v[0, 0].tolist() == [lo + 0.5 * (hi - lo), hi] and p.tolist() == [[1]]


def test_duplicate_and_unsorted_caller_keys():
    a = rows((POD, 1, SVC, 2, 4, 0, 0), (POD, 5, SVC, 2, 7, 0, 0), (SVC, 9, POD, 0, 2, 0, 0))
    keys = [key(POD, 5, SVC, 2), key(POD, 1, SVC, 2), key(POD, 5, SVC, 2), key(POD, 6, SVC, 2), key(SVC, 9, POD, 0)]
    v, p = sr.series([a], keys, [COUNT])
    assert v[:, 0, 0].tolist() == [7, 4, 7, 0, 2]
    assert p[:, 0].tolist() == [1, 1, 1, 0, 1]


def test_every_node_kind_including_host_keyed_ends():
    specs = [(POD, 1, POD, 2), (POD, 1, SVC, 2), (POD, 1, OUT, 0xFFFFFFFF), (POD, 1, HOST, 77), (SVC, 3, POD, 1),
             (OUT, 0x08080808, POD, 1), (HOST, 5, POD, 1)]
    a = rows(*[s + (i + 1, 0, 0) for i, s in enumerate(specs)])
    for i, s in enumerate(specs):
        k = key(*s)
        # the packing is the inverse of the flush's row key
        row = a[(a["from_type"] == s[0]) & (a["from"] == s[1]) & (a["to_type"] == s[2]) & (a["to"] == s[3])]
        assert k == int(row_keys(row)[0]), s
        v, p = sr.series([a], [k], [COUNT])
        assert (v[0, 0, 0], p[0, 0]) == (i + 1, 1), s
    assert key(POD, 1, POD, 2) >> 63 == 0 and key(HOST, 5, POD, 1) >> 63 == 1


@pytest.mark.parametrize("ends", [(SVC, 1, SVC, 2), (OUT, 1, HOST, 2), (4, 1, POD, 2), (POD, 1, 4, 2),
                                  (POD, 1 << 29, SVC, 2), (POD, 1, SVC, 1 << 29), (SVC, 1 << 29, POD, 1),
                                  (POD, 1, POD, 1 << 29)])
def test_malformed_keys(ends):
    assert sr.pack_ends(*ends) is None
    e = np.zeros(1, abi.EDGE_ENDS)
    e["from_type"], e["from"], e["to_type"], e["to"] = ends
    with pytest.raises(ValueError):
        sr.ends_keys(e)


def test_large_outbound_and_host_ids_are_not_malformed():
    assert sr.pack_ends(POD, (1 << 29) - 1, OUT, 0xFFFFFFFF) is not None
    assert sr.pack_ends(HOST, 0xFFFFFFFF, POD, 3) is not None


def test_reversed_pod_pod_edge_named_both_ways():
    # a flush emits the pod <-> pod row with from = A, to = B; named (A, B) it is found, named (B, A) it is another edge
    a = rows((POD, 10, POD, 20, 3, 0, 0))
    v, p = sr.series([a], [key(POD, 10, POD, 20), key(POD, 20, POD, 10)], [COUNT])
    assert p[:, 0].tolist() == [1, 0] and v[:, 0, 0].tolist() == [3, 0]
    b = rows((POD, 10, POD, 20, 3, 0, 0), (POD, 20, POD, 10, 5, 0, 0))
    v, p = sr.series([b], [key(POD, 20, POD, 10), key(POD, 10, POD, 20)], [COUNT])
    assert v[:, 0, 0].tolist() == [5, 3] and p[:, 0].tolist() == [1, 1]


def test_k_above_the_retained_count():
    es = [rows((POD, 1, SVC, 2, c, 0, 0)) for c in (1, 2, 3)]
    k1 = key(POD, 1, SVC, 2)
    v, p = sr.series(es, [k1], [COUNT], k=10)
    assert v[0, :, 0].tolist() == [1, 2, 3] and p.shape == (1, 3)
    v, p = sr.series(es, [k1], [COUNT], k=2)
    assert v[0, :, 0].tolist() == [2, 3]
    v, p = sr.series([], [k1], [COUNT], k=5)
    assert v.shape == (1, 0, 1) and p.shape == (1, 0)


def test_empty_entries_and_no_edges():
    es = [rows(), rows((POD, 1, SVC, 2, 9, 0, 0))]
    v, p = sr.series(es, [key(POD, 1, SVC, 2)], [COUNT, ERR])
    assert p.tolist() == [[0, 1]] and v[0].tolist() == [[0, 0], [9, 0]]
    v, p = sr.series(es, [], [COUNT])
    assert v.shape == (0, 2, 1)
