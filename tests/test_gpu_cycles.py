"""GPU: cycles (alz_cycles*, alz_group_cycles*, alz_debug_cycles_rows, docs/SPEC.md §28).

Records, row positions, rows and info of the host and device forms are compared as bytes against tests/cycle_ref.py
over the rows of each source (grouped by the map in force for the group form). Windows come from the Modelled stream
of tests/test_gpu_edge_series.py; the hook lists build layouts ingest cannot make: a chain and a ring of 2^16 nodes in
descending key order, a hub with 2^20 callers it calls back, 2^18 disjoint 2- and 3-cycles, a random graph of 2^20
rows, layered DAGs, a chain of 2-node loops whose indices fall downstream and every type byte."""
import ctypes as C

import numpy as np
import pytest

import cycle_ref as cr
import group_ref as gr
import metric_ref
from alaz_b200 import abi, capi
from test_gpu_edge_series import Modelled, make_source
from test_gpu_gnn_rollup import universe
from test_gpu_group_series import namespaces_map
from test_gpu_groups import owners_map

pytestmark = pytest.mark.gpu
WINDOW, WIN, TIER, SPAN = abi.SOURCE_WINDOW, abi.ROLLUP_WINDOWS, abi.ROLLUP_TIER, abi.ROLLUP_SPAN
Q = abi.METRIC_QUANTILE
POD, SVC = 0, 1


def dump(rec, idx, rows, info):
    return rec.tobytes(), idx.tobytes(), rows.tobytes(), info


def check(h, group, source, rows, gmap, spec=None, min_value=0.0, min_size=1):
    """host and device forms of one call against the reference; returns the reference's result"""
    kw = dict(spec=spec, min_value=min_value, min_size=min_size)
    exp = cr.group_cycles(rows, gmap, **kw) if group else cr.cycles(rows, **kw)
    got = (h.group_cycles if group else h.cycles)(source, **kw)
    what = (group, source, spec, min_value, min_size)
    if dump(*got) != dump(*exp):
        raise AssertionError((what, got[3], exp[3], len(got[0]), len(exp[0])))
    pn, nn, pi, pr, nrows, info = (h.group_cycles_device if group else h.cycles_device)(source, **kw)
    assert (nn, nrows, info) == (len(exp[0]), len(exp[1]), exp[3]), what
    assert h.d2h(pn, nn, abi.CYCLE_NODE).tobytes() == exp[0].tobytes(), what
    assert h.d2h(pi, nrows, np.uint32).tobytes() == exp[1].tobytes(), what
    assert h.d2h(pr, nrows, abi.EDGE_OUT).tobytes() == exp[2].tobytes(), what
    return exp


@pytest.fixture(scope="module")
def mod():
    m = Modelled(universe(seed=53), history=(6, 1 << 15), tiers=[(2, 4, 1 << 15, 1 << 13)])
    m.random_windows(12, seed=531, lo=0.2, hi=0.7)
    m.last = m.window(np.flatnonzero(np.random.default_rng(532).random(m.s.g.n_edges) < 0.5))
    yield m
    m.h.group_set([], [])
    m.close()


def count_threshold(rows):
    v = metric_ref.values(rows, abi.METRIC_COUNT)
    return float(np.quantile(v, 0.5)) if len(v) else 0.0


@pytest.mark.parametrize("source", [WINDOW, WIN, TIER, SPAN])
def test_every_source_form_map_filter_and_min_size(mod, source):
    h = mod.h
    rows = make_source(mod, source)
    filters = [(None, 0.0), (abi.METRIC_ERR5XX, 1.0), (abi.METRIC_COUNT, count_threshold(rows))]
    maps = [("node", None), ("empty", ([], [])), ("owners", owners_map(rows)), ("namespaces", namespaces_map(rows))]
    nodes = 0
    for name, mp in maps:
        group = mp is not None
        if group:
            h.group_set(*mp)
            gmap = gr.make_map(*mp) if len(mp[0]) else gr.EMPTY
        else:
            gmap = gr.EMPTY
        for spec, mv in filters:
            for min_size in (1, 2):
                exp = check(h, group, source, rows, gmap, spec, mv, min_size)
                nodes = max(nodes, exp[3]["nodes"])
    assert nodes > 10, source
    h.group_set([], [])


@pytest.fixture(scope="module")
def hh():
    h = capi.Handle(device=0, max_endpoints=1 << 10, max_pairs=1 << 12)
    yield h
    h.close()


def hook_rows(pairs, types=(POD, POD)):
    r = np.zeros(len(pairs), dtype=abi.EDGE_OUT)
    r["from_type"], r["to_type"] = types
    if len(pairs):
        r["from"], r["to"] = np.asarray(pairs, dtype=np.uint64).T
    r["count"] = 1
    return r


def check_hook(h, rows, spec=None, min_value=0.0, min_size=1):
    exp = cr.cycles(rows, spec, min_value, min_size)
    got = h.debug_cycles_rows(rows, spec, min_value, min_size)
    if dump(*got) != dump(*exp):
        raise AssertionError((spec, min_value, min_size, got[3], exp[3]))
    return exp


def test_a_chain_and_a_ring_of_2_16_nodes_in_descending_key_order(hh):
    n = 1 << 16
    chain = [(i + 1, i) for i in range(n - 1)][::-1]
    exp = check_hook(hh, hook_rows(chain))
    assert exp[3]["components"] == n and exp[3]["depth"] == n - 1 and exp[3]["cyclic"] == 0
    ring = hook_rows(chain + [(0, n - 1)])
    exp = check_hook(hh, ring, min_size=2)
    assert exp[3]["components"] == 1 and exp[3]["largest"] == n and len(exp[1]) == n and exp[3]["depth"] == 0
    # the other way round the ring, and the ring cut by a filter into the chain again
    check_hook(hh, hook_rows([(b, a) for a, b in chain] + [(n - 1, 0)]), min_size=2)
    ring["err5xx"] = 1
    ring["err5xx"][-1] = 0
    exp = check_hook(hh, ring, abi.METRIC_ERR5XX, 1.0)
    assert exp[3]["cyclic"] == 0 and exp[3]["depth"] == n - 1


def test_chains_of_2_node_loops_whose_indices_fall_or_rise_downstream(hh):
    # colouring one way settles one loop per iteration on such a chain (about N^2 / 4 rounds for N nodes); the other
    # way settles every loop at once, and iterations alternate. 512 nodes per chain keep even the slow way quick.
    k = 256
    falling = [(2 * (k - 1 - i), 2 * (k - 1 - i) + 1) for i in range(k)]   # loop i, upstream first
    rising = [(2 * i + 2 * k, 2 * i + 2 * k + 1) for i in range(k)]
    chain = lambda loops: [p for a, b in loops for p in ((a, b), (b, a))] + \
        [(loops[i][1], loops[i + 1][0]) for i in range(k - 1)]
    for pairs, loops in ((chain(falling), k), (chain(rising), k), (chain(falling) + chain(rising), 2 * k)):
        rows = hook_rows(pairs)[np.random.default_rng(99).permutation(len(pairs))]
        exp = check_hook(hh, rows, min_size=2)
        assert exp[3]["cyclic"] == loops and exp[3]["components"] == loops and exp[3]["depth"] == k - 1


def test_a_hub_with_2_20_callers_it_calls_back(hh):
    n = 1 << 20
    calls = hook_rows([(i, 5) for i in range(n)], types=(POD, SVC))
    back = hook_rows([(5, i) for i in range(n)], types=(SVC, POD))
    rows = np.concatenate([calls, back])[np.random.default_rng(95).permutation(2 * n)]
    exp = check_hook(hh, rows, min_size=2)
    assert exp[3]["components"] == 1 and exp[3]["largest"] == n + 1 and len(exp[1]) == 2 * n
    exp = check_hook(hh, calls)   # the callers alone: a star of depth 1
    assert exp[3]["components"] == n + 1 and exp[3]["depth"] == 1


def test_2_18_disjoint_2_and_3_cycles(hh):
    rng = np.random.default_rng(96)
    k = 1 << 18
    ids = rng.permutation(1 << 22)
    pairs, at = [], 0
    for j in range(k):
        s = 2 + (j & 1)
        c = ids[at:at + s].tolist()
        at += s
        pairs += [(c[i], c[(i + 1) % s]) for i in range(s)]
    rows = hook_rows(pairs)[rng.permutation(len(pairs))]
    rows["err5xx"] = rng.integers(0, 8, len(rows)) > 0
    exp = check_hook(hh, rows, min_size=2)
    assert exp[3]["cyclic"] == k and exp[3]["cyclic_nodes"] == at and exp[3]["depth"] == 0
    exp = check_hook(hh, rows, abi.METRIC_ERR5XX, 1.0, min_size=2)
    assert 0 < exp[3]["cyclic"] < k


def test_a_random_graph_of_2_20_rows(hh):
    rng = np.random.default_rng(97)
    n = 1 << 20
    rows = hook_rows(rng.integers(0, 1 << 19, (n, 2)))
    rows["err5xx"] = rng.integers(0, 3, n)
    rows["count"] = rng.integers(1, 100, n)
    exp = check_hook(hh, rows, min_size=2)
    assert exp[3]["cyclic"] >= 1
    check_hook(hh, rows, abi.METRIC_ERR5XX, 1.0)
    check_hook(hh, rows, abi.METRIC_COUNT, 90.0, min_size=2)


@pytest.mark.parametrize("layers,width", [(2, 1000), (10, 3000), (200, 50)])
def test_layered_dags_with_known_depth_and_height(hh, layers, width):
    rng = np.random.default_rng(layers)
    node = lambda i, j: i * width + j
    pairs = []
    for i in range(layers - 1):
        for j in range(width):   # every node has a caller in the layer above and a callee in the layer below
            pairs.append((node(i, int(rng.integers(width))), node(i + 1, j)))
            pairs.append((node(i, j), node(i + 1, int(rng.integers(width)))))
        for _ in range(width):   # rows that skip layers do not lengthen a path
            a = int(rng.integers(i + 1, layers))
            pairs.append((node(i, int(rng.integers(width))), node(a, int(rng.integers(width)))))
    ids = rng.permutation(1 << 24)[:layers * width]
    rows = hook_rows([(ids[a], ids[b]) for a, b in pairs])[rng.permutation(len(pairs))]
    rec, _, _, info = check_hook(hh, rows)
    assert info["components"] == layers * width and info["depth"] == layers - 1
    where = {int(ids[v]): v // width for v in range(layers * width)}
    for t in rec:
        assert (t["depth"], t["height"]) == (where[int(t["value"])], layers - 1 - where[int(t["value"])])


def test_every_type_byte_and_repeated_ends(hh):
    rng = np.random.default_rng(98)
    n = 4096
    rows = np.zeros(n, dtype=abi.EDGE_OUT)
    rows["from_type"] = rng.integers(0, 256, n)
    rows["to_type"] = rng.integers(0, 256, n)
    rows["from"] = rng.integers(0, 4, n)
    rows["to"] = rng.integers(0, 4, n)
    rows["count"] = 1
    rows = np.concatenate([rows, rows[:500], rows[:100][::-1]])
    for min_size in (0, 1, 2):
        exp = check_hook(hh, rows, min_size=min_size)
    assert exp[3]["cyclic"] >= 1 and exp[3]["self_rows"] >= 1
    assert set(range(256)) <= set(rows["from_type"].tolist()) | set(rows["to_type"].tolist())


def call(h, fn, *args, m=None, mv=0.0, min_size=1, node_cap=0, nodes=None, row_cap=0, ri=None, rows=None,
         n_nodes=True, n_rows=True):
    nn, nr_, info = C.c_size_t(77), C.c_size_t(77), abi.CycleInfo()
    ptr = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    rc = getattr(h.L, fn)(h.h, *args, m, mv, min_size, ptr(nodes), node_cap, C.byref(nn) if n_nodes else None,
                          ptr(ri), ptr(rows), row_cap, C.byref(nr_) if n_rows else None, C.byref(info))
    return rc, nn.value, nr_.value, info.as_dict()


def test_errors_capacity_and_zero_rows(mod):
    h = mod.h
    h.group_set(*owners_map(make_source(mod, WINDOW)))
    rows = make_source(mod, WINDOW)
    gmap = gr.make_map(*owners_map(rows))
    m1 = abi.metrics(abi.METRIC_ERR5XX)
    E = abi.E_INVAL
    for fn in ("alz_cycles", "alz_group_cycles"):
        exp = cr.cycles(rows) if fn == "alz_cycles" else cr.group_cycles(rows, gmap)
        assert len(exp[0]) > 1
        assert call(h, fn, WINDOW)[0] == 0
        for src in (3, 7, 0xFFFFFFFE):
            assert call(h, fn, src)[:3] == (E, 0, 0)
        assert call(h, fn, WINDOW, n_nodes=False)[0] == E
        assert call(h, fn, WINDOW, n_rows=False)[0] == E
        for bad in (abi.metrics((9, 0.0)), abi.metrics((Q, 1.5)), abi.metrics((Q, float("nan")))):
            assert call(h, fn, WINDOW, m=bad)[0] == E
        assert call(h, fn, WINDOW, m=m1, mv=float("nan"))[0] == E
        assert call(h, fn, WINDOW, m=None, mv=float("nan"))[0] == 0   # ignored without a metric
        # capacity: counts set, nothing written
        out = np.zeros(len(exp[0]), dtype=abi.CYCLE_NODE)
        rc, nn, nrows, info = call(h, fn, WINDOW, nodes=out, node_cap=len(exp[0]) - 1)
        assert (rc, nn, nrows, info) == (abi.E_CAPACITY, len(exp[0]), len(exp[1]), exp[3])
        assert not out.view(np.uint8).any()
        if len(exp[1]):
            ri = np.zeros(len(exp[1]), dtype=np.uint32)
            rc, nn, nrows, _ = call(h, fn, WINDOW, nodes=out, node_cap=len(out), ri=ri, row_cap=len(ri) - 1)
            assert (rc, nn, nrows) == (abi.E_CAPACITY, len(exp[0]), len(exp[1])) and not ri.any()
            assert not out.view(np.uint8).any()
            assert call(h, fn, WINDOW, ri=ri, row_cap=len(ri))[0] == 0 and ri.tobytes() == exp[1].tobytes()
        rc, nn, nrows, info = call(h, fn, WINDOW, nodes=out, node_cap=len(out))
        assert rc == 0 and out.tobytes() == exp[0].tobytes()
        nn = C.c_size_t(5)
        assert getattr(h.L, fn + "_device")(h.h, WINDOW, None, 0.0, 1, None, C.byref(nn), None, None, None,
                                            None) == E and nn.value == 0
    h.group_set([], [])
    assert call(h, "alz_debug_cycles_rows", C.c_void_p(8), 1 << 29)[0] == abi.E_CAPACITY
    assert call(h, "alz_debug_cycles_rows", None, 4)[0] == E
    got = h.debug_cycles_rows(np.zeros(0, dtype=abi.EDGE_OUT))
    assert len(got[0]) == 0 and got[3] == dict(rows=0, traversable=0, self_rows=0, nodes=0, components=0, cyclic=0,
                                               cyclic_nodes=0, largest=0, cycle_rows=0, depth=0)


def test_rollup_sources_without_rows_and_an_empty_window():
    h = capi.Handle(device=0, max_endpoints=1 << 10, max_pairs=1 << 12)
    try:
        for fn in ("alz_cycles", "alz_group_cycles"):
            for s in (WIN, TIER, SPAN):
                assert call(h, fn, s)[:3] == (abi.E_STATE, 0, 0)
            rc, nn, nrows, info = call(h, fn, WINDOW)
            assert (rc, nn, nrows) == (0, 0, 0) and info["rows"] == 0
    finally:
        h.close()


def test_reads_only(mod):
    """the window, every rollup's rows, the map and other families' device results (reach's among them) keep their
    bytes, and a flush after the calls gives the rows the model expects"""
    h = mod.h
    for s in (WIN, TIER, SPAN):
        make_source(mod, s)
    rows = make_source(mod, SPAN)
    h.group_set(*owners_map(rows))

    def fetch():
        out, n = np.zeros(h.max_edges, dtype=abi.EDGE_OUT), C.c_size_t(0)
        h._ck(h.L.alz_window_fetch(h.h, out.ctypes.data_as(C.c_void_p), len(out), C.byref(n)), "alz_window_fetch")
        return out[: n.value].tobytes()

    ALL = [abi.METRIC_COUNT, (Q, 0.99)]
    stored = lambda: [fetch(), h.edge_metrics(*ALL).tobytes(), h.group_edges(SPAN)[0].tobytes()] + \
        [h.edge_metrics_rollup(s, *ALL).tobytes() for s in (WIN, TIER, SPAN)]
    rows_before = stored()
    p_node, n_node = h.node_rows_device(SPAN)
    p_ge, n_ge, _ = h.group_edges_device(SPAN)
    p_gn, n_gn = h.group_nodes_device(SPAN)
    p_met, n_met = h.edge_metrics_rollup_device(SPAN, *ALL)
    seeds = np.zeros(20, dtype=abi.NODE_ENDS)
    import node_ref
    keys = node_ref.keys(rows)[:20]
    seeds["type"], seeds["value"] = (keys >> np.uint64(32)).astype(np.uint8), (keys & np.uint64(0xFFFFFFFF))
    p_rn, n_rn, p_ri, p_rr, n_rr, _ = h.reach_device(SPAN, seeds, abi.REACH_ANY, 64)

    def snap():
        return [h.d2h(p_node, n_node, abi.NODE_OUT).tobytes(), h.d2h(p_ge, n_ge, abi.EDGE_OUT).tobytes(),
                h.d2h(p_gn, n_gn, abi.NODE_OUT).tobytes(), h.d2h(p_met, n_met * len(ALL), np.float64).tobytes(),
                h.d2h(p_rn, n_rn, abi.REACH_NODE).tobytes(), h.d2h(p_ri, n_rr, np.uint32).tobytes(),
                h.d2h(p_rr, n_rr, abi.EDGE_OUT).tobytes()]

    before = snap()
    for s in (WINDOW, WIN, TIER, SPAN):
        h.cycles(s)
        h.group_cycles(s, abi.METRIC_ERR5XX, 1.0, 2)
        h.cycles_device(s, (Q, 0.99), 1e6)
    assert snap() == before
    assert stored() == rows_before
    want = mod.window(np.flatnonzero(np.random.default_rng(533).random(mod.s.g.n_edges) < 0.5))
    assert fetch() == want.tobytes()
    mod.last = want
    h.group_set([], [])
