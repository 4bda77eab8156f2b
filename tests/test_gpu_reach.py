"""GPU: reach (alz_reach*, alz_group_reach*, alz_debug_reach_rows, docs/SPEC.md §27).

Records, row positions, rows and info of the host and device forms are compared as bytes against tests/reach_ref.py
over the rows of each source (grouped by the map in force for the group form). Windows come from the Modelled stream
of tests/test_gpu_edge_series.py; the hook lists build layouts ingest cannot make: chains around max_hops 64, a hub
of 2^20 callers, 2^20 seeds into one node, a random graph of 2^20 rows and every type byte."""
import ctypes as C
import itertools

import numpy as np
import pytest

import group_ref as gr
import node_ref as nr
import reach_ref as rr
from alaz_b200 import abi, capi
from test_gpu_edge_series import Modelled, make_source
from test_gpu_gnn_rollup import universe
from test_gpu_group_series import namespaces_map
from test_gpu_groups import ends, owners_map

pytestmark = pytest.mark.gpu
WINDOW, WIN, TIER, SPAN = abi.SOURCE_WINDOW, abi.ROLLUP_WINDOWS, abi.ROLLUP_TIER, abi.ROLLUP_SPAN
DOWN, UP, ANY = abi.REACH_DOWN, abi.REACH_UP, abi.REACH_ANY
Q = abi.METRIC_QUANTILE
POD, SVC, OUTB, HOST, GRP = 0, 1, 2, 3, abi.NODE_GROUP
NONE = abi.REACH_NONE


def dump(rec, idx, rows, info):
    return rec.tobytes(), idx.tobytes(), rows.tobytes(), info


def check(h, group, source, rows, gmap, seeds, direction, max_hops, spec=None, min_value=0.0):
    """host and device forms of one call against the reference; returns the reference's result"""
    kw = dict(direction=direction, max_hops=max_hops, spec=spec, min_value=min_value)
    exp = rr.group_reach(rows, seeds, gmap, **kw) if group else rr.reach(rows, seeds, **kw)
    got = (h.group_reach if group else h.reach)(source, seeds, **kw)
    what = (group, source, direction, max_hops, spec, min_value, len(seeds))
    if dump(*got) != dump(*exp):
        raise AssertionError((what, got[3], exp[3], len(got[0]), len(exp[0])))
    pn, nn, pi, pr, nrows, info = (h.group_reach_device if group else h.reach_device)(source, seeds, **kw)
    assert (nn, nrows, info) == (len(exp[0]), len(exp[1]), exp[3]), what
    assert h.d2h(pn, nn, abi.REACH_NODE).tobytes() == exp[0].tobytes(), what
    assert h.d2h(pi, nrows, np.uint32).tobytes() == exp[1].tobytes(), what
    assert h.d2h(pr, nrows, abi.EDGE_OUT).tobytes() == exp[2].tobytes(), what
    return exp


@pytest.fixture(scope="module")
def mod():
    m = Modelled(universe(seed=47), history=(6, 1 << 15), tiers=[(2, 4, 1 << 15, 1 << 13)])
    m.random_windows(12, seed=471, lo=0.2, hi=0.7)
    m.last = m.window(np.flatnonzero(np.random.default_rng(472).random(m.s.g.n_edges) < 0.5))
    yield m
    m.h.group_set([], [])
    m.close()


def seed_sets(keys, rng):
    """one seed, 100 seeds, duplicates, absent seeds, outbound and Host-keyed seeds"""
    e = ends(keys)
    pods = e[e["type"] == POD]
    if len(pods) < 3:   # a map that holds every pod: its groups
        pods = e[e["type"] == GRP]
    sets = [e[:1], pods[rng.permutation(len(pods))[:100]], np.concatenate([pods[:3], pods[:3], pods[1:2]])]
    absent = ends(np.array([(POD << 32) | 999_999, (SVC << 32) | 77_777, (HOST << 32) | 0xFFFFFFFF], np.uint64))
    sets.append(np.concatenate([absent, pods[-2:]]))
    far = e[(e["type"] == OUTB) | (e["type"] == HOST)]
    sets.append(np.concatenate([far, absent[:1]]) if len(far) else absent)
    return sets


def p99_threshold(rows):
    import metric_ref
    v = metric_ref.values(rows, (Q, 0.99))
    return float(np.quantile(v, 0.5)) if len(v) else 0.0


@pytest.mark.parametrize("source", [WINDOW, WIN, TIER, SPAN])
def test_every_source_form_direction_and_bound(mod, source):
    h = mod.h
    rows = make_source(mod, source)
    rng = np.random.default_rng(source & 0xFF)
    filters = [(None, 0.0), (abi.METRIC_ERR5XX, 1.0), ((Q, 0.99), p99_threshold(rows))]
    maps = [("node", None), ("empty", ([], [])), ("owners", owners_map(rows)), ("namespaces", namespaces_map(rows))]
    for name, mp in maps:
        group = mp is not None
        if group:
            h.group_set(*mp)
            gmap = gr.make_map(*mp) if len(mp[0]) else gr.EMPTY
            keys = nr.keys(gr.group(rows, gmap)[0])
        else:
            gmap, keys = gr.EMPTY, nr.keys(rows)
        sets = seed_sets(keys, rng)
        if group:
            gkeys = keys[(keys >> np.uint64(32)) == GRP]
            sets.append(ends(gkeys[:5]) if len(gkeys) else ends(np.array([(GRP << 32) | 12345], np.uint64)))
        levels = 0
        for j, (d, k, (spec, mv)) in enumerate(itertools.product((DOWN, UP, ANY), (1, 2, 64), filters)):
            exp = check(h, group, source, rows, gmap, sets[j % len(sets)], d, k, spec, mv)
            levels = max(levels, exp[3]["levels"])
        assert levels >= 2, (source, name)   # the graphs reach past one hop
    h.group_set([], [])


@pytest.mark.parametrize("source", [WINDOW, SPAN])
def test_an_empty_map_is_node_reach_up_to_row_positions(mod, source):
    h = mod.h
    h.group_set([], [])
    rows = make_source(mod, source)
    gedges = gr.group(rows, gr.EMPTY)[0]
    seeds = ends(nr.keys(rows)[:20])
    for d in (DOWN, UP, ANY):
        a = h.reach(source, seeds, d, 3)
        b = h.group_reach(source, seeds, d, 3)
        for f in ("type", "value", "hops", "index", "parent"):
            assert (a[0][f] == b[0][f]).all(), (d, f)
        assert a[3] == b[3] and sorted(a[2].tobytes()[i * 296:(i + 1) * 296] for i in range(len(a[2]))) == \
            sorted(b[2].tobytes()[i * 296:(i + 1) * 296] for i in range(len(b[2])))
        if d != ANY:
            hopped = a[0]["row"] != NONE
            assert hopped.sum() > 0
            assert rows[a[0]["row"][hopped]].tobytes() == gedges[b[0]["row"][hopped]].tobytes(), d


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


def check_hook(h, rows, seeds, direction, max_hops, spec=None, min_value=0.0):
    exp = rr.reach(rows, seeds, direction, max_hops, spec, min_value)
    got = h.debug_reach_rows(rows, seeds, direction, max_hops, spec, min_value)
    if dump(*got) != dump(*exp):
        raise AssertionError((direction, max_hops, got[3], exp[3]))
    return exp


def test_chains_around_max_hops_64(hh):
    rng = np.random.default_rng(91)
    for n_nodes, levels, cut in ((64, 63, 0), (65, 64, 0), (66, 64, 1)):
        ids = rng.permutation(1 << 20)[:n_nodes]
        pairs = [(int(ids[i]), int(ids[i + 1])) for i in range(n_nodes - 1)]
        rows = hook_rows(pairs)[rng.permutation(n_nodes - 1)]
        exp = check_hook(hh, rows, [(POD, int(ids[0]))], DOWN, 64)
        assert (exp[3]["nodes"], exp[3]["levels"], exp[3]["cut"]) == (min(n_nodes, 65), levels, cut)
        mid = int(ids[n_nodes // 2])
        exp = check_hook(hh, rows, [(POD, mid)], ANY, 64)
        assert exp[3]["nodes"] == n_nodes
        check_hook(hh, rows, [(POD, mid)], ANY, 7)
        check_hook(hh, rows, [(POD, int(ids[-1]))], UP, 64)


def test_a_hub_of_2_20_callers(hh):
    n = 1 << 20
    rows = hook_rows([(i, 5) for i in range(n)], types=(POD, SVC))
    rows = rows[np.random.default_rng(92).permutation(n)]
    exp = check_hook(hh, rows, [(SVC, 5)], UP, 3)
    assert exp[3]["nodes"] == n + 1 and exp[3]["levels"] == 1 and len(exp[1]) == n
    exp = check_hook(hh, rows, [(POD, 77)], DOWN, 3)
    assert exp[3]["nodes"] == 2
    exp = check_hook(hh, rows, [(POD, 77)], ANY, 2)
    assert exp[3]["nodes"] == n + 1 and exp[3]["levels"] == 2
    # 2^20 seeds, every caller, into the one node
    seeds = np.zeros(n, dtype=abi.NODE_ENDS)
    seeds["value"] = np.arange(n)
    exp = check_hook(hh, rows, seeds, DOWN, 64)
    assert exp[3]["seeds_found"] == n and exp[3]["nodes"] == n + 1 and exp[3]["levels"] == 1


def test_a_random_graph_of_2_20_rows(hh):
    rng = np.random.default_rng(93)
    n = 1 << 20
    rows = hook_rows(rng.integers(0, 1 << 19, (n, 2)))
    rows["err5xx"] = rng.integers(0, 3, n)
    seeds = [(POD, int(v)) for v in rng.integers(0, 1 << 19, 10)]
    for d, k in ((DOWN, 64), (UP, 3), (ANY, 2)):
        check_hook(hh, rows, seeds, d, k)
    check_hook(hh, rows, seeds, DOWN, 64, abi.METRIC_ERR5XX, 1.0)


def test_every_type_byte(hh):
    rng = np.random.default_rng(94)
    n = 4096
    rows = np.zeros(n, dtype=abi.EDGE_OUT)
    rows["from_type"] = rng.integers(0, 256, n)
    rows["to_type"] = rng.integers(0, 256, n)
    rows["from"] = rng.integers(0, 4, n)
    rows["to"] = rng.integers(0, 4, n)
    rows["count"] = 1
    for d in (DOWN, UP, ANY):
        exp = check_hook(hh, rows, [(t, v) for t in range(4) for v in range(4)], d, 64)
        assert exp[3]["nodes"] > 16
    assert set(range(256)) <= set(rows["from_type"].tolist()) | set(rows["to_type"].tolist())


def call(h, fn, *args, seeds=None, n_seeds=None, dir=DOWN, hops=3, m=None, mv=0.0, node_cap=0, nodes=None,
         row_cap=0, ri=None, rows=None, n_nodes=True, n_rows=True):
    nn, nr_, info = C.c_size_t(77), C.c_size_t(77), abi.ReachInfo()
    sp = None if seeds is None else seeds.ctypes.data_as(C.c_void_p)
    n_s = (0 if seeds is None else len(seeds)) if n_seeds is None else n_seeds
    ptr = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    rc = getattr(h.L, fn)(h.h, *args, sp, n_s, dir, hops, m, mv, ptr(nodes), node_cap,
                          C.byref(nn) if n_nodes else None, ptr(ri), ptr(rows), row_cap,
                          C.byref(nr_) if n_rows else None, C.byref(info))
    return rc, nn.value, nr_.value, info.as_dict()


def test_errors_capacity_and_zero_rows(mod):
    h = mod.h
    h.group_set([], [])
    rows = make_source(mod, WINDOW)
    keys = nr.keys(rows)
    good = ends(keys[:4])
    m1 = abi.metrics(abi.METRIC_ERR5XX)
    for fn in ("alz_reach", "alz_group_reach"):
        exp = rr.reach(rows, good, DOWN, 3) if fn == "alz_reach" else rr.group_reach(rows, good, gr.EMPTY,
                                                                                      direction=DOWN, max_hops=3)
        assert len(exp[0]) > 1 and len(exp[1]) > 1
        E = abi.E_INVAL
        assert call(h, fn, WINDOW, seeds=good)[0] == 0
        for src in (3, 7, 0xFFFFFFFE):
            assert call(h, fn, src, seeds=good)[:3] == (E, 0, 0)
        assert call(h, fn, WINDOW, seeds=good, dir=3)[0] == E
        for hops in (0, 65, 1 << 31):
            assert call(h, fn, WINDOW, seeds=good, hops=hops)[0] == E
        assert call(h, fn, WINDOW, seeds=good, hops=64)[0] == 0
        assert call(h, fn, WINDOW, seeds=good, n_seeds=0)[0] == E
        assert call(h, fn, WINDOW, seeds=None, n_seeds=3)[0] == E
        assert call(h, fn, WINDOW, seeds=good, n_nodes=False)[0] == E
        assert call(h, fn, WINDOW, seeds=good, n_rows=False)[0] == E
        for bad in (abi.metrics((9, 0.0)), abi.metrics((Q, 1.5)), abi.metrics((Q, float("nan")))):
            assert call(h, fn, WINDOW, seeds=good, m=bad)[0] == E
        assert call(h, fn, WINDOW, seeds=good, m=m1, mv=float("nan"))[0] == E
        assert call(h, fn, WINDOW, seeds=good, m=None, mv=float("nan"))[0] == 0   # ignored without a metric
        for bad in ((5 << 32) | 1, 1 << 29, (1 << 32) | (1 << 29)):
            assert call(h, fn, WINDOW, seeds=np.concatenate([good, ends(np.array([bad], np.uint64))]))[0] == E
        grp = ends(np.array([(GRP << 32) | 7], np.uint64))
        assert call(h, fn, WINDOW, seeds=grp)[0] == (E if fn == "alz_reach" else 0)
        assert call(h, fn, WINDOW, seeds=ends(np.array([(GRP << 32) | (1 << 29)], np.uint64)))[0] == E
        # capacity: counts set, nothing written
        out = np.zeros(len(exp[0]), dtype=abi.REACH_NODE)
        rc, nn, nrows, info = call(h, fn, WINDOW, seeds=good, nodes=out, node_cap=len(exp[0]) - 1)
        assert (rc, nn, nrows, info) == (abi.E_CAPACITY, len(exp[0]), len(exp[1]), exp[3])
        assert not out.view(np.uint8).any()
        ri = np.zeros(len(exp[1]), dtype=np.uint32)
        rc, nn, nrows, _ = call(h, fn, WINDOW, seeds=good, nodes=out, node_cap=len(out), ri=ri,
                                row_cap=len(ri) - 1)
        assert (rc, nn, nrows) == (abi.E_CAPACITY, len(exp[0]), len(exp[1])) and not ri.any()
        assert not out.view(np.uint8).any()
        rr_ = np.zeros(len(exp[1]), dtype=abi.EDGE_OUT)
        assert call(h, fn, WINDOW, seeds=good, rows=rr_, row_cap=len(ri) - 1)[0] == abi.E_CAPACITY
        # a cap is checked only where its array is given
        assert call(h, fn, WINDOW, seeds=good, ri=ri, row_cap=len(ri))[0] == 0
        assert ri.tobytes() == exp[1].tobytes()
        rc, nn, nrows, info = call(h, fn, WINDOW, seeds=good, nodes=out, node_cap=len(out))
        assert rc == 0 and out.tobytes() == exp[0].tobytes()
        # device: the same validation
        nn = C.c_size_t(5)
        assert getattr(h.L, fn + "_device")(h.h, WINDOW, None, 2, DOWN, 3, None, 0.0, None, C.byref(nn), None, None,
                                            None, None) == E and nn.value == 0
    # more than 2^29 - 1 rows through the hook, more than 2^30 - 1 seeds
    assert call(h, "alz_debug_reach_rows", C.c_void_p(8), 1 << 29, seeds=good)[0] == abi.E_CAPACITY
    assert call(h, "alz_debug_reach_rows", None, 4, seeds=good)[0] == abi.E_INVAL
    many = np.zeros(1 << 30, dtype=abi.NODE_ENDS)   # 8 GB of untouched zero pages: every seed is (POD, 0)
    assert call(h, "alz_reach", WINDOW, seeds=many)[0] == abi.E_CAPACITY
    del many
    # zero rows
    got = h.debug_reach_rows(np.zeros(0, dtype=abi.EDGE_OUT), [(POD, 1)], ANY, 5)
    assert len(got[0]) == 0 and got[3] == dict(rows=0, traversable=0, seeds_found=0, nodes=0, levels=0, cut=0)


def test_rollup_sources_without_rows_and_an_empty_window():
    h = capi.Handle(device=0, max_endpoints=1 << 10, max_pairs=1 << 12)
    try:
        seeds = ends(np.array([1], np.uint64))
        for fn in ("alz_reach", "alz_group_reach"):
            for s in (WIN, TIER, SPAN):
                assert call(h, fn, s, seeds=seeds)[:3] == (abi.E_STATE, 0, 0)
            rc, nn, nrows, info = call(h, fn, WINDOW, seeds=seeds)
            assert (rc, nn, nrows) == (0, 0, 0) and info["rows"] == 0
    finally:
        h.close()


def test_reads_only(mod):
    """the window, every rollup's rows, the baseline, the map and every other family's device results keep their
    bytes, and a flush after a reach gives the rows the model expects"""
    h = mod.h
    for s in (WIN, TIER, SPAN):
        make_source(mod, s)
    h.baseline_pin(SPAN)
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
    p_top = h.edge_top_rollup_device(SPAN, abi.METRIC_COUNT, 50)
    p_ch, n_ch, _ = h.node_changes_device(abi.SIDE_IN, abi.METRIC_COUNT, source=WINDOW)
    p_gch, n_gch, _ = h.group_edge_changes_device(abi.METRIC_COUNT, source=WINDOW)
    p_ser = h.node_series_device(SPAN, abi.SIDE_IN, 0, 4, *ALL)
    p_tr = h.edge_trends_device(SPAN, 0, 4, abi.METRIC_COUNT, abi.Trend(stat=abi.TREND_SLOPE, recent=1, min_points=2))
    try:
        p_gnn = h.gnn_score_rollup_device(SPAN)
    except capi.AlzError as e:   # built without the GNN pass
        assert e.status == abi.E_UNSUPPORTED
        p_gnn = (0, 0)

    def snap():
        return [h.d2h(p_node, n_node, abi.NODE_OUT).tobytes(), h.d2h(p_ge, n_ge, abi.EDGE_OUT).tobytes(),
                h.d2h(p_gn, n_gn, abi.NODE_OUT).tobytes(), h.d2h(p_met, n_met * len(ALL), np.float64).tobytes(),
                h.d2h(p_top[0], p_top[3], abi.EDGE_OUT).tobytes(), h.d2h(p_ch, n_ch, abi.NODE_CHANGE).tobytes(),
                h.d2h(p_gch, n_gch, abi.EDGE_CHANGE).tobytes(),
                h.d2h(p_ser[0], p_ser[2] * p_ser[3] * len(ALL), np.float64).tobytes(),
                h.d2h(p_tr[0], p_tr[1], abi.EDGE_TREND).tobytes(),
                h.d2h(p_gnn[0], p_gnn[1], np.float32).tobytes() if p_gnn[1] else b""]

    before = snap()
    seeds = ends(nr.keys(rows)[:50])
    gseeds = ends(nr.keys(gr.group(rows, gr.make_map(*owners_map(rows)))[0])[:50])
    for s in (WINDOW, WIN, TIER, SPAN):
        for d in (DOWN, UP, ANY):
            h.reach(s, seeds, d, 64)
            h.group_reach(s, gseeds, d, 64, abi.METRIC_ERR5XX, 1.0)
            h.reach_device(s, seeds, d, 2, (Q, 0.99), 1e6)
    assert snap() == before
    assert stored() == rows_before
    base = h.edge_changes(abi.METRIC_COUNT, source=SPAN)[0]
    assert (base["presence"] == abi.PRESENT_BOTH).all()   # the span against its own pin: the baseline is intact
    # a flush after the calls flushes what the model expects
    want = mod.window(np.flatnonzero(np.random.default_rng(473).random(mod.s.g.n_edges) < 0.5))
    assert fetch() == want.tobytes()
    mod.last = want
    h.group_set([], [])
