"""CPU: the reach reference (tests/reach_ref.py, docs/SPEC.md §27) on hand-written graphs with their expected records,
rows and counts, and on generated graphs whose hops equal scipy's unweighted shortest paths."""
import numpy as np
from hypothesis import given, settings, strategies as st
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import shortest_path

import reach_ref as rr
from alaz_b200 import abi

DOWN, UP, ANY = abi.REACH_DOWN, abi.REACH_UP, abi.REACH_ANY
NONE = abi.REACH_NONE
POD, SVC = 0, 1


def graph(pairs, err=None):
    """EDGE_OUT rows from (from pod, to pod) pairs, in the given order; err[i] the 5xx count of row i"""
    r = np.zeros(len(pairs), dtype=abi.EDGE_OUT)
    r["from_type"], r["to_type"] = POD, POD
    r["from"] = [a for a, _ in pairs]
    r["to"] = [b for _, b in pairs]
    r["count"] = 10
    if err is not None:
        r["err5xx"] = err
    return r


def table(rec):
    """[(value, hops, index, parent, row)] of the records"""
    return [tuple(int(x) for x in (t["value"], t["hops"], t["index"], t["parent"], t["row"])) for t in rec]


def test_a_chain_down_up_and_any():
    rows = graph([(1, 2), (2, 3), (3, 4)])
    rec, idx, got, info = rr.reach(rows, [(POD, 1)], DOWN, 64)
    assert table(rec) == [(1, 0, 0, NONE, NONE), (2, 1, 1, 0, 0), (3, 2, 2, 1, 1), (4, 3, 3, 2, 2)]
    assert idx.tolist() == [0, 1, 2] and got.tobytes() == rows.tobytes()
    assert info == dict(rows=3, traversable=3, seeds_found=1, nodes=4, levels=3, cut=0)
    rec, idx, _, info = rr.reach(rows, [(POD, 1)], UP, 64)
    assert table(rec) == [(1, 0, 0, NONE, NONE)] and len(idx) == 0 and info["levels"] == 0
    rec, idx, _, info = rr.reach(rows, [(POD, 4)], UP, 2)
    assert table(rec) == [(4, 0, 3, NONE, NONE), (3, 1, 2, 0, 2), (2, 2, 1, 1, 1)]
    assert idx.tolist() == [1, 2] and info["cut"] == 1 and info["levels"] == 2
    rec, idx, _, info = rr.reach(rows, [(POD, 3)], ANY, 1)
    assert table(rec) == [(3, 0, 2, NONE, NONE), (2, 1, 1, 0, 1), (4, 1, 3, 0, 2)]
    assert idx.tolist() == [1, 2] and info["cut"] == 1   # 1 -> 2 leaves hops 1 toward a node not listed


def test_a_diamond_takes_the_parent_of_smallest_index():
    # 1 -> {3, 2} -> 4: both 2 and 3 lead to 4; the parent is 2 (index 1), whatever the row order
    rows = graph([(1, 3), (3, 4), (1, 2), (2, 4)])
    rec, idx, _, info = rr.reach(rows, [(POD, 1)], DOWN, 64)
    assert table(rec) == [(1, 0, 0, NONE, NONE), (2, 1, 1, 0, 2), (3, 1, 2, 0, 0), (4, 2, 3, 1, 3)]
    assert idx.tolist() == [0, 1, 2, 3] and info["levels"] == 2


def test_any_with_both_orientations_of_one_pair_takes_the_smallest_row():
    rows = graph([(5, 6), (6, 5), (5, 6)])
    for seed, other in ((5, 6), (6, 5)):
        rec, idx, _, info = rr.reach(rows, [(POD, seed)], ANY, 3)
        assert table(rec)[1][0] == other and table(rec)[1][4] == 0
        assert idx.tolist() == [0, 1, 2] and info == dict(rows=3, traversable=3, seeds_found=1, nodes=2, levels=1,
                                                          cut=0)
    rec, _, _, _ = rr.reach(rows, [(POD, 6)], DOWN, 3)
    assert table(rec)[1] == (5, 1, 0, 0, 1)


def test_a_cycle_and_a_self_loop():
    rows = graph([(1, 1), (1, 2), (2, 3), (3, 1)])
    rec, idx, _, info = rr.reach(rows, [(POD, 2)], DOWN, 64)
    assert table(rec) == [(2, 0, 1, NONE, NONE), (3, 1, 2, 0, 2), (1, 2, 0, 1, 3)]
    assert idx.tolist() == [0, 1, 2, 3]   # the self-loop and the row back to the seed are listed
    assert info == dict(rows=4, traversable=4, seeds_found=1, nodes=3, levels=2, cut=0)
    rec, idx, _, info = rr.reach(rows, [(POD, 1)], ANY, 64)
    assert table(rec) == [(1, 0, 0, NONE, NONE), (2, 1, 1, 0, 1), (3, 1, 2, 0, 3)]
    assert idx.tolist() == [0, 1, 2, 3]


def test_a_filter_cuts_a_path():
    rows = graph([(1, 2), (2, 3), (1, 4), (4, 3)], err=[3, 0, 1, 1])
    rec, idx, _, info = rr.reach(rows, [(POD, 1)], DOWN, 64, abi.METRIC_ERR5XX, 1.0)
    assert table(rec) == [(1, 0, 0, NONE, NONE), (2, 1, 1, 0, 0), (4, 1, 3, 0, 2), (3, 2, 2, 2, 3)]
    assert idx.tolist() == [0, 2, 3] and info["traversable"] == 3
    rec, _, _, info = rr.reach(rows, [(POD, 1)], DOWN, 64, abi.METRIC_ERR5XX, 2.0)
    assert table(rec) == [(1, 0, 0, NONE, NONE), (2, 1, 1, 0, 0)] and info["traversable"] == 1
    # -inf admits every row; a metric of +0.0 against min -0.0 is admitted, -0.0 against +0.0 is not
    assert rr.reach(rows, [(POD, 1)], DOWN, 64, abi.METRIC_ERR5XX, -np.inf)[3]["traversable"] == 4
    assert rr.reach(rows, [(POD, 1)], DOWN, 64, abi.METRIC_ERR5XX, -0.0)[3]["traversable"] == 4


def test_cut_at_the_bound():
    rows = graph([(i, i + 1) for i in range(10)] + [(2, 7)])
    hops = {0: 0, 1: 1, 2: 2, 3: 3, 7: 3, 4: 4, 8: 4, 5: 5, 9: 5, 6: 6, 10: 6}
    for k in range(1, 9):
        rec, idx, _, info = rr.reach(rows, [(POD, 0)], DOWN, k)
        assert {int(v): int(h) for v, h in zip(rec["value"], rec["hops"])} == {v: h for v, h in hops.items() if h <= k}
        listed = set(rec["value"].tolist())
        cut = sum(1 for a, b in zip(rows["from"], rows["to"])
                  if a in listed and b not in listed and rec["hops"][list(rec["value"]).index(a)] == k)
        assert info["cut"] == cut and info["levels"] == max(rec["hops"])
        assert (info["cut"] == 0) == (len(rr.reach(rows, [(POD, 0)], DOWN, k + 1)[0]) == len(rec))


def test_absent_and_duplicate_seeds():
    rows = graph([(1, 2), (2, 3)])
    rec, idx, _, info = rr.reach(rows, [(POD, 9), (SVC, 1), (POD, 2), (POD, 2), (POD, 2)], DOWN, 64)
    assert table(rec) == [(2, 0, 1, NONE, NONE), (3, 1, 2, 0, 1)] and info["seeds_found"] == 1
    rec, idx, got, info = rr.reach(rows, [(POD, 9)], DOWN, 64)
    assert len(rec) == 0 and len(idx) == 0 and info == dict(rows=2, traversable=2, seeds_found=0, nodes=0, levels=0,
                                                            cut=0)
    rec, _, _, info = rr.reach(rows[:0], [(POD, 1)], ANY, 64)
    assert len(rec) == 0 and info == dict(rows=0, traversable=0, seeds_found=0, nodes=0, levels=0, cut=0)


def test_parents_rebuild_shortest_paths():
    rng = np.random.default_rng(3)
    rows = graph([(int(a), int(b)) for a, b in rng.integers(0, 40, (150, 2))])
    for d in (DOWN, UP, ANY):
        rec, idx, got, _ = rr.reach(rows, [(POD, 0), (POD, 1)], d, 64)
        for j in range(len(rec)):
            p = rr.path(rec, j)
            assert len(p) == rec["hops"][j] + 1 and rec["hops"][p[0][0]] == 0
            for (a, _), (b, r) in zip(p, p[1:]):
                ends = {(int(rows["from"][r]), int(rows["to"][r]))}
                if d == ANY:
                    ends.add((int(rows["to"][r]), int(rows["from"][r])))
                want = (int(rec["value"][a]), int(rec["value"][b]))
                assert (want if d != UP else want[::-1]) in ends
                assert r in idx


@settings(max_examples=60, deadline=None)
@given(n=st.integers(1, 30), edges=st.lists(st.tuples(st.integers(0, 29), st.integers(0, 29)), max_size=120),
       seed=st.integers(0, 29), direction=st.sampled_from([DOWN, UP, ANY]), max_hops=st.integers(1, 8))
def test_hops_are_scipy_shortest_paths(n, edges, seed, direction, max_hops):
    edges = [(a % n, b % n) for a, b in edges]
    if not edges:
        return
    rows = graph(edges)
    keys = sorted({v for e in edges for v in e})
    ix = {v: i for i, v in enumerate(keys)}
    a = np.array([ix[x] for x, _ in edges])
    b = np.array([ix[y] for _, y in edges])
    if direction == UP:
        a, b = b, a
    m = csr_matrix((np.ones(len(a)), (a, b)), shape=(len(keys), len(keys)))
    dist = shortest_path(m, directed=direction != ANY, unweighted=True)
    s = keys[seed % len(keys)]
    rec, _, _, info = rr.reach(rows, [(POD, s)], direction, max_hops)
    want = {keys[i]: int(dd) for i, dd in enumerate(dist[ix[s]]) if np.isfinite(dd) and dd <= max_hops}
    assert {int(v): int(h) for v, h in zip(rec["value"], rec["hops"])} == want
    assert [(int(h), int(i)) for h, i in zip(rec["hops"], rec["index"])] == sorted(
        (want[keys[i]], i) for i in range(len(keys)) if keys[i] in want)
    beyond = {keys[i] for i, dd in enumerate(dist[ix[s]]) if np.isfinite(dd) and dd > max_hops}
    assert (info["cut"] > 0) == bool(beyond)
