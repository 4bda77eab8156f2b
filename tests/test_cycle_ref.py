"""CPU: the cycles reference (tests/cycle_ref.py, docs/SPEC.md §28) on hand-written graphs with their expected records,
rows and counts, and on generated graphs whose components are scipy's strong components and whose depths and heights
are brute-force longest paths."""
import itertools

import numpy as np
from hypothesis import given, settings, strategies as st
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import connected_components

import cycle_ref as cr
import group_ref
from alaz_b200 import abi

POD, SVC = 0, 1


def graph(pairs, err=None, count=10):
    """EDGE_OUT rows from (from pod, to pod) pairs, in the given order; err[i] the 5xx count of row i"""
    r = np.zeros(len(pairs), dtype=abi.EDGE_OUT)
    r["from_type"], r["to_type"] = POD, POD
    r["from"] = [a for a, _ in pairs]
    r["to"] = [b for _, b in pairs]
    r["count"] = count
    if err is not None:
        r["err5xx"] = err
    return r


def table(rec):
    """[(value, index, component, size, depth, height)] of the records"""
    return [tuple(int(x) for x in (t["value"], t["index"], t["component"], t["size"], t["depth"], t["height"]))
            for t in rec]


def test_a_chain():
    rec, idx, got, info = cr.cycles(graph([(3, 4), (1, 2), (2, 3)]))
    assert table(rec) == [(1, 0, 0, 1, 0, 3), (2, 1, 1, 1, 1, 2), (3, 2, 2, 1, 2, 1), (4, 3, 3, 1, 3, 0)]
    assert len(idx) == 0 and len(got) == 0
    assert info == dict(rows=3, traversable=3, self_rows=0, nodes=4, components=4, cyclic=0, cyclic_nodes=0,
                        largest=1, cycle_rows=0, depth=3)
    assert len(cr.cycles(graph([(3, 4), (1, 2), (2, 3)]), min_size=2)[0]) == 0


def test_a_diamond_takes_the_longest_path():
    # 1 -> 2 -> 4 and 1 -> 3 -> 5 -> 4: 4 sits 3 rows below 1
    rec, _, _, info = cr.cycles(graph([(1, 2), (2, 4), (1, 3), (3, 5), (5, 4)]))
    assert {int(t["value"]): (int(t["depth"]), int(t["height"])) for t in rec} == {
        1: (0, 3), 2: (1, 1), 3: (1, 2), 5: (2, 1), 4: (3, 0)}
    assert info["depth"] == 3 and info["components"] == 5


def test_two_loops_joined_by_a_row():
    # loop {1, 2} -> loop {5, 6, 7}; 9 hangs under the second
    rows = graph([(5, 6), (1, 2), (6, 7), (2, 1), (7, 5), (2, 5), (6, 9)])
    rec, idx, got, info = cr.cycles(rows)
    assert table(rec) == [(1, 0, 0, 2, 0, 2), (2, 1, 0, 2, 0, 2), (5, 2, 1, 3, 1, 1), (6, 3, 1, 3, 1, 1),
                          (7, 4, 1, 3, 1, 1), (9, 5, 2, 1, 2, 0)]
    assert idx.tolist() == [1, 3, 0, 2, 4] and got.tobytes() == rows[idx].tobytes()
    assert info == dict(rows=7, traversable=7, self_rows=0, nodes=6, components=3, cyclic=2, cyclic_nodes=5,
                        largest=3, cycle_rows=5, depth=2)
    rec2, idx2, _, info2 = cr.cycles(rows, min_size=2)
    assert table(rec2) == table(rec)[:5] and idx2.tolist() == idx.tolist() and info2 == info
    rec3, idx3, _, _ = cr.cycles(rows, min_size=3)
    assert [t[0] for t in table(rec3)] == [5, 6, 7] and idx3.tolist() == [0, 2, 4]


def test_self_rows_only():
    rows = graph([(1, 1), (2, 2), (1, 1)])
    rec, idx, _, info = cr.cycles(rows)
    assert table(rec) == [(1, 0, 0, 1, 0, 0), (2, 1, 1, 1, 0, 0)] and len(idx) == 0
    assert info == dict(rows=3, traversable=3, self_rows=3, nodes=2, components=2, cyclic=0, cyclic_nodes=0,
                        largest=1, cycle_rows=0, depth=0)


def test_a_self_row_inside_a_loop_is_not_listed():
    rows = graph([(1, 2), (2, 2), (2, 1)])
    rec, idx, _, info = cr.cycles(rows, min_size=2)
    assert [t[0] for t in table(rec)] == [1, 2] and idx.tolist() == [0, 2]
    assert info["self_rows"] == 1 and info["cycle_rows"] == 2


def test_a_filter_breaks_a_loop():
    rows = graph([(1, 2), (2, 3), (3, 1)], err=[2, 2, 0])
    assert cr.cycles(rows)[3]["cyclic"] == 1
    rec, idx, _, info = cr.cycles(rows, abi.METRIC_ERR5XX, 1.0)
    assert table(rec) == [(1, 0, 0, 1, 0, 2), (2, 1, 1, 1, 1, 1), (3, 2, 2, 1, 2, 0)] and len(idx) == 0
    assert info["traversable"] == 2 and info["cyclic"] == 0
    # a row filtered out does not count as a self row either
    assert cr.cycles(graph([(1, 1)], err=[0]), abi.METRIC_ERR5XX, 1.0)[3]["self_rows"] == 0


def test_group_internal_rows_are_self_rows():
    # pods 1, 2 in group 7 and 3, 4 in group 8: 1 -> 2 and 4 -> 4 are internal; 2 -> 3 and 4 -> 1 make a loop of
    # the groups that the pods do not have
    rows = graph([(1, 2), (2, 3), (4, 1), (4, 4)])
    gmap = group_ref.make_map([(POD, 1), (POD, 2), (POD, 3), (POD, 4)], [7, 7, 8, 8])
    assert cr.cycles(rows)[3]["cyclic"] == 0
    rec, idx, got, info = cr.group_cycles(rows, gmap, min_size=2)
    assert [(int(t["type"]), int(t["value"]), int(t["size"])) for t in rec] == [(abi.NODE_GROUP, 7, 2),
                                                                                 (abi.NODE_GROUP, 8, 2)]
    assert info["self_rows"] == 2 and info["cycle_rows"] == 2 and len(got) == 2
    assert {(int(a), int(b)) for a, b in zip(got["from"], got["to"])} == {(7, 8), (8, 7)}


def test_no_rows():
    rec, idx, got, info = cr.cycles(graph([]))
    assert len(rec) == len(idx) == len(got) == 0
    assert info == dict(rows=0, traversable=0, self_rows=0, nodes=0, components=0, cyclic=0, cyclic_nodes=0,
                        largest=0, cycle_rows=0, depth=0)


def brute_longest(nc, crow):
    """the most rows on a path ending at each component, by trying every simple path of a tiny DAG"""
    succ = {c: sorted({b for a, b in crow if a == c}) for c in range(nc)}
    best = [0] * nc

    def walk(c, d):
        best[c] = max(best[c], d)
        for b in succ[c]:
            walk(b, d + 1)

    for c in range(nc):
        walk(c, 0)
    return best


@settings(max_examples=80, deadline=None)
@given(edges=st.lists(st.tuples(st.integers(0, 11), st.integers(0, 11)), min_size=1, max_size=40),
       err=st.lists(st.integers(0, 2), min_size=40, max_size=40), filt=st.booleans(), min_size=st.integers(0, 3))
def test_components_are_scipys_and_levels_are_longest_paths(edges, err, filt, min_size):
    rows = graph(edges, err=err[:len(edges)])
    spec = abi.METRIC_ERR5XX if filt else None
    rec, idx, got, info = cr.cycles(rows, spec, 1.0, min_size)
    full, _, _, _ = cr.cycles(rows, spec, 1.0, 0)
    keys = sorted({v for e in edges for v in e})
    ix = {v: i for i, v in enumerate(keys)}
    N = len(keys)
    trav = [not filt or e >= 1 for e in err[:len(edges)]]
    kept = [(ix[a], ix[b]) for (a, b), t in zip(edges, trav) if t]
    a = np.array([x for x, _ in kept], dtype=np.int64)
    b = np.array([y for _, y in kept], dtype=np.int64)
    m = csr_matrix((np.ones(len(a)), (a, b)), shape=(N, N))
    nc, lab = connected_components(m, directed=True, connection="strong")
    assert info["components"] == nc and len(full) == N
    comp = full["component"][np.argsort(full["index"])]
    # the same partition, numbered by smallest index
    assert all((lab[i] == lab[j]) == (comp[i] == comp[j]) for i, j in itertools.combinations(range(N), 2))
    firsts = [int(np.flatnonzero(comp == c)[0]) for c in range(nc)]
    assert firsts == sorted(firsts)
    crow = sorted({(int(comp[x]), int(comp[y])) for x, y in kept if comp[x] != comp[y]})
    depth = brute_longest(nc, crow)
    height = brute_longest(nc, [(y, x) for x, y in crow])
    for t in full:
        assert (t["depth"], t["height"]) == (depth[t["component"]], height[t["component"]])
    sizes = np.bincount(comp, minlength=nc)
    assert [int(t["index"]) for t in rec] == [int(t["index"]) for t in full if sizes[t["component"]] >= min_size]
    inside = [r for r, ((x, y), t) in enumerate(zip(edges, trav)) if t and x != y and comp[ix[x]] == comp[ix[y]]]
    assert info["cycle_rows"] == len(inside)
    assert sorted(idx.tolist()) == [r for r in inside if sizes[comp[ix[edges[r][0]]]] >= min_size]
    assert got.tobytes() == rows[idx].tobytes()
    assert info["cyclic_nodes"] == int(sizes[sizes >= 2].sum()) and info["largest"] == int(sizes.max())
