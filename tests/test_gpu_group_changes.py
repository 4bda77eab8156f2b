"""GPU: group changes against a pinned baseline (alz_group_edge_changes*, alz_group_node_changes*,
alz_debug_group_edge_changes_rows, docs/SPEC.md §25).

The expected lists and top results are tests/group_change_ref.py over the same rows and map, compared as bytes.
Windows and rollups come from the Stream of tests/test_gpu_gnn_rollup.py; the hook runs the join over layouts ingest
cannot make: ends whose node keys collide in 64 bits, lists that differ only in the to end, one group edge on 2^20
rows, cells of 2^32 - 1 and lists of 2^20 + 3 rows."""
import ctypes as C
import itertools

import numpy as np
import pytest

import group_change_ref as gcr
import group_ref as gr
import metric_ref
import node_change_ref as ncr
import node_ref as nr
from alaz_b200 import abi, capi
from test_gpu_edge_changes import Sources
from test_gpu_gnn_rollup import Stream, universe
from test_gpu_groups import edge_rows, ends, owners_map

pytestmark = pytest.mark.gpu
WINDOW, WIN, TIER, SPAN = abi.SOURCE_WINDOW, abi.ROLLUP_WINDOWS, abi.ROLLUP_TIER, abi.ROLLUP_SPAN
IN, OUT = abi.SIDE_IN, abi.SIDE_OUT
Q = abi.METRIC_QUANTILE
SPECS = [abi.METRIC_COUNT, abi.METRIC_ERR5XX, abi.METRIC_ERR_RATE, abi.METRIC_MEAN_NS, (Q, 0.0), (Q, 0.5), (Q, 0.99),
         (Q, 1.0)]
MODES = [abi.CHANGE_DELTA, abi.CHANGE_DROP, abi.CHANGE_RATIO]
MASKS = list(range(1, 8))
POD, SVC, OUTB, GRP = abi.NODE_POD, abi.NODE_SVC, abi.NODE_OUTBOUND, abi.NODE_GROUP
BOTH, NEW, GONE = abi.PRESENT_BOTH, abi.PRESENT_NEW, abi.PRESENT_GONE
PARAM = {WINDOW: 5, WIN: 3, TIER: 1, SPAN: 3}


def namespaces_map(rows):
    """every pod and service into one of 100 namespaces by its id; outbound ends stay as they are"""
    keys = nr.keys(rows)
    keys = keys[(keys >> np.uint64(32)) <= SVC]
    return ends(keys), ((keys & np.uint64(0xFFFFFFFF)) % np.uint64(100)).astype(np.uint32)


def set_map(h, nodes, groups):
    h.group_set(nodes, groups)
    return gr.make_map(nodes, groups) if len(nodes) else gr.EMPTY


def same(got, want, what):
    got_l, got_i = got
    want_l, want_i = want
    assert got_i == want_i, (what, got_i, want_i)
    assert got_l.tobytes() == want_l.tobytes(), (what, len(got_l), len(want_l),
                                                 np.flatnonzero(got_l != want_l)[:5] if len(got_l) == len(want_l)
                                                 else None)


def cuts(lst):
    fin = lst["change"][np.isfinite(lst["change"])]
    mid = float(np.median(fin)) if len(fin) else 0.0
    n = max(len(lst), 1)
    return itertools.product((1, n, n + 5) if n > 1 else (1, 6), (-np.inf, mid, np.inf))


def check_all(h, src_rows, src_w, base_rows, base_w, source, gmap, what, full=True):
    """every group change call of `source` against the reference, both levels and sides"""
    ga, gb = gr.group(src_rows, gmap)[0], gr.group(base_rows, gmap)[0]
    na, nb = nr.group(ga), nr.group(gb)
    specs = SPECS if full else [abi.METRIC_COUNT, (Q, 0.99)]
    for spec, mode in itertools.product(specs, MODES):
        want = gcr.edge_changes_of(ga, gb, spec, mode, 7, src_w, base_w)
        same(h.group_edge_changes(spec, mode, 7, source=source), want, (what, "edges", spec, mode))
        for side in (IN, OUT):
            want = ncr.changes_of_nodes(na, nb, side, spec, mode, 7, src_w, base_w)
            same(h.group_node_changes(side, spec, mode, 7, source=source), want, (what, "nodes", side, spec, mode))
    for mask in MASKS:
        spec, mode = SPECS[mask], MODES[mask % 3]
        same(h.group_edge_changes(spec, mode, mask, source=source),
             gcr.edge_changes_of(ga, gb, spec, mode, mask, src_w, base_w), (what, "edges", mask))
        for side in (IN, OUT):
            same(h.group_node_changes(side, spec, mode, mask, source=source),
                 ncr.changes_of_nodes(na, nb, side, spec, mode, mask, src_w, base_w), (what, "nodes", side, mask))
    for (spec, mode), mask in itertools.product(((abi.METRIC_COUNT, abi.CHANGE_DELTA), ((Q, 0.99), abi.CHANGE_RATIO),
                                                 (abi.METRIC_ERR_RATE, abi.CHANGE_DROP)), (7, 5)):
        lst, info = gcr.edge_changes_of(ga, gb, spec, mode, mask, src_w, base_w)
        for k, mn in cuts(lst):
            same(h.group_edge_changes_top(spec, k, mn, mode, mask, source=source), gcr.top(lst, info, k, mn),
                 (what, "edge top", spec, mode, mask, k, mn))
        for side in (IN, OUT):
            lst, info = ncr.changes_of_nodes(na, nb, side, spec, mode, mask, src_w, base_w)
            for k, mn in cuts(lst):
                same(h.group_node_changes_top(side, spec, k, mn, mode, mask, source=source),
                     gcr.top(lst, info, k, mn), (what, "node top", side, spec, mode, mask, k, mn))


@pytest.fixture(scope="module")
def stream():
    s = Stream(universe(seed=24), history=(6, 1 << 15), tiers=[(2, 4, 1 << 15, 1 << 13)])
    s.random_windows(9, seed=241, lo=0.2, hi=0.6)
    yield s
    s.h.group_set([], [])
    s.close()


@pytest.mark.parametrize("base_kind", [WINDOW, WIN, TIER, SPAN])
def test_every_source_against_every_baseline_kind_and_map(stream, base_kind):
    src = Sources(stream)
    h = stream.h
    base_rows, _ = src.make(base_kind, {WINDOW: 1, WIN: 4, TIER: 2, SPAN: 6}[base_kind])
    pinned = h.baseline_pin(base_kind)
    stream.random_windows(2, seed=242 + base_kind % 7, lo=0.2, hi=0.6)   # the baseline survives flushes
    for kind in (WINDOW, WIN, TIER, SPAN):
        rows, _ = src.make(kind, PARAM[kind])
        both = np.concatenate([rows, base_rows])
        for name, mk in (("owners", owners_map), ("namespaces", namespaces_map), ("empty", None)):
            gmap = set_map(h, *mk(both)) if mk else set_map(h, [], [])
            check_all(h, rows, src.windows[kind], base_rows, pinned["windows"], kind, gmap, (base_kind, kind, name),
                      full=name == "owners")
    h.group_set([], [])


def test_an_empty_map_gives_the_node_and_edge_changes(stream):
    h = stream.h
    set_map(h, [], [])
    src = Sources(stream)
    src.make(WIN, 4)
    h.baseline_pin(WIN)
    stream.random_windows(1, seed=251)
    for source in (WINDOW, SPAN):
        rows, _ = src.make(source, PARAM[source])
        base_rows = src.rows[WIN]
        for spec, mode in itertools.product((abi.METRIC_COUNT, (Q, 0.99), abi.METRIC_ERR_RATE), MODES):
            for side in (IN, OUT):
                want = h.node_changes(side, spec, mode, 7, source=source)
                same(h.group_node_changes(side, spec, mode, 7, source=source), want, (source, side, spec, mode))
            lst, info = h.edge_changes(spec, mode, 7, source=source)
            inv_a = np.argsort(np.lexsort(gcr.ends_keys(rows)[::-1]))
            inv_b = np.argsort(np.lexsort(gcr.ends_keys(base_rows)[::-1]))
            f, t = gcr.ends_keys(lst)
            want = lst[np.lexsort((t, f))].copy()
            has_a, has_b = want["index"] != abi.ABSENT, want["base_index"] != abi.ABSENT
            want["index"][has_a] = inv_a[want["index"][has_a]]
            want["base_index"][has_b] = inv_b[want["base_index"][has_b]]
            same(h.group_edge_changes(spec, mode, 7, source=source), (want, info), (source, "edges", spec, mode))


def test_a_source_against_itself_and_values_are_the_group_metrics(stream):
    h = stream.h
    rows, info = h.rollup_span(4)
    set_map(h, *owners_map(rows))
    h.baseline_pin(SPAN)
    w = info["windows"]
    for spec in SPECS:
        lst, ci = h.group_edge_changes(spec, abi.CHANGE_DELTA, source=SPAN)
        assert np.all(lst["presence"] == BOTH) and ci["added"] == ci["gone"] == 0
        assert np.all(lst["index"] == lst["base_index"]) and np.all(lst["change"].view(np.uint64) == 0)
        assert np.all(h.group_edge_changes(spec, abi.CHANGE_RATIO, source=SPAN)[0]["change"] == 1.0)
        vals = h.group_edge_metrics(SPAN, spec).reshape(-1)[lst["index"]]
        if spec in (abi.METRIC_COUNT, abi.METRIC_ERR5XX):
            vals = vals / np.float64(w)
        assert lst["value"].tobytes() == vals.tobytes(), spec
        for side in (IN, OUT):
            lst, ci = h.group_node_changes(side, spec, abi.CHANGE_DELTA, source=SPAN)
            assert np.all(lst["presence"] == BOTH) and np.all(lst["change"].view(np.uint64) == 0)
            assert np.all(h.group_node_changes(side, spec, abi.CHANGE_RATIO, source=SPAN)[0]["change"] == 1.0)
            vals = h.group_node_metrics(SPAN, side, spec).reshape(-1)[lst["index"]]
            if spec in (abi.METRIC_COUNT, abi.METRIC_ERR5XX):
                vals = vals / np.float64(w)
            assert lst["value"].tobytes() == vals.tobytes(), (side, spec)
    h.group_set([], [])


def test_device_variants_equal_host(stream):
    h = stream.h
    rows, _ = h.rollup(3)
    set_map(h, *owners_map(rows))
    h.baseline_pin(WIN)
    stream.random_windows(1, seed=261)
    for spec in (abi.METRIC_COUNT, (Q, 0.99)):
        lst, info = h.group_edge_changes(spec, abi.CHANGE_RATIO, 7)
        p, n, dinfo = h.group_edge_changes_device(spec, abi.CHANGE_RATIO, 7)
        assert n == len(lst) and dinfo == info and h.d2h(p, n, abi.EDGE_CHANGE).tobytes() == lst.tobytes()
        top, tinfo = h.group_edge_changes_top(spec, 20, 0.0, abi.CHANGE_RATIO, 7)
        p, n, dinfo = h.group_edge_changes_top_device(spec, 20, 0.0, abi.CHANGE_RATIO, 7)
        assert n == len(top) and dinfo == tinfo and h.d2h(p, n, abi.EDGE_CHANGE).tobytes() == top.tobytes()
        for side in (IN, OUT):
            lst, info = h.group_node_changes(side, spec, abi.CHANGE_RATIO, 7)
            p, n, dinfo = h.group_node_changes_device(side, spec, abi.CHANGE_RATIO, 7)
            assert n == len(lst) and dinfo == info and h.d2h(p, n, abi.NODE_CHANGE).tobytes() == lst.tobytes()
            top, tinfo = h.group_node_changes_top(side, spec, 20, 0.0, abi.CHANGE_RATIO, 7)
            p, n, dinfo = h.group_node_changes_top_device(side, spec, 20, 0.0, abi.CHANGE_RATIO, 7)
            assert n == len(top) and dinfo == tinfo and h.d2h(p, n, abi.NODE_CHANGE).tobytes() == top.tobytes()
    h.group_set([], [])


def test_a_rolling_deploy_is_both_only_as_a_group():
    """api-1 and api-2 serve before, api-3 and api-4 after: pods NEW and GONE, the deployment BOTH"""
    s = Stream(universe(seed=27), history=(4, 1 << 15))
    h, g = s.h, s.g
    try:
        into = (g.tt == POD) & (g.ft == POD) & ~g.rev
        pods, cnt = np.unique(g.tv[into], return_counts=True)
        api = pods[np.argsort(-cnt, kind="stable")[:4]]
        before = np.flatnonzero(into & np.isin(g.tv, api[:2]))
        after = np.flatnonzero(into & np.isin(g.tv, api[2:]))
        base_rows = s.window(before)
        h.baseline_pin(WINDOW)
        src_rows = s.window(after)
        pods_ch, _ = h.node_changes(IN, (Q, 0.99))
        api_pods = pods_ch[np.isin(pods_ch["node"], api) & (pods_ch["type"] == POD)]
        assert len(api_pods) == 4 and set(api_pods["presence"].tolist()) == {NEW, GONE}
        gmap = set_map(h, ends(api.astype(np.uint64)), np.full(4, 42, np.uint32))
        lst, info = h.group_node_changes(IN, (Q, 0.99))
        same((lst, info), gcr.node_changes(src_rows, base_rows, gmap, IN, (Q, 0.99), abi.CHANGE_DELTA, 7), "deploy")
        grp = lst[lst["type"] == GRP]
        assert len(grp) == 1 and grp[0]["node"] == 42 and grp[0]["presence"] == BOTH
        want = []
        for r in (src_rows, base_rows):   # the p99 of the histograms summed over every row into the four pods
            into_api = r[(r["to_type"] == POD) & np.isin(r["to"], api)].copy()
            summed = np.zeros(1, dtype=abi.EDGE_OUT)
            for f in ("count", "err5xx", "lat_sum_ns"):
                summed[f] = into_api[f].sum()
            summed["hist"] = into_api["hist"].sum(axis=0, dtype=np.uint32)
            want.append(float(metric_ref.values(summed, (Q, 0.99))[0]))
        assert [grp[0]["value"], grp[0]["base_value"]] == want
        pod_p99 = [x["value"] or x["base_value"] for x in api_pods]
        assert grp[0]["change"] == grp[0]["value"] - grp[0]["base_value"] and len(pod_p99) == 4
        edges, _ = h.group_edge_changes(abi.METRIC_COUNT)
        into_grp = edges[(edges["to_type"] == GRP) & (edges["to"] == 42)]
        assert len(into_grp) and np.all(into_grp["presence"] != 0)
    finally:
        s.close()


def test_the_cached_baseline_follows_pins_and_maps():
    s = Stream(universe(seed=28), history=(4, 1 << 15))
    h = s.h
    try:
        r1 = s.window(np.arange(0, 1500))
        h.baseline_pin(WINDOW)
        src = s.window(np.arange(500, 2500))

        def check(base_rows, gmap, what):
            for side in (IN, OUT):
                same(h.group_node_changes(side, (Q, 0.99), abi.CHANGE_DELTA),
                     gcr.node_changes(src, base_rows, gmap, side, (Q, 0.99), abi.CHANGE_DELTA, 7), (what, side))
            same(h.group_edge_changes(abi.METRIC_COUNT, abi.CHANGE_DELTA),
                 gcr.edge_changes(src, base_rows, gmap, abi.METRIC_COUNT, abi.CHANGE_DELTA, 7), what)

        m1 = set_map(h, *owners_map(np.concatenate([r1, src])))
        check(r1, m1, "first")
        m2 = set_map(h, *namespaces_map(np.concatenate([r1, src])))
        check(r1, m2, "new map")
        bad = ends(np.array([3, 4, 3], np.uint64))
        assert h.L.alz_group_set(h.h, bad.ctypes.data_as(C.c_void_p),
                                 np.array([1, 2, 3], np.uint32).ctypes.data_as(C.c_void_p), 3) == abi.E_INVAL
        check(r1, m2, "refused set")
        h.baseline_pin(WINDOW)   # the source window itself
        check(src, m2, "new pin")
        h.baseline_clear()
        assert h.L.alz_group_edge_changes(h.h, WINDOW, abi.metrics(abi.METRIC_COUNT), 0, 7, None, 0,
                                          C.byref(C.c_size_t()), None) == abi.E_STATE
        r3 = s.window(np.arange(2000, 3000))
        h.baseline_pin(WINDOW)
        src = s.window(np.arange(100, 2600))
        check(r3, m2, "clear and re-pin")
        check(r3, set_map(h, [], []), "map cleared")
    finally:
        s.close()


def test_reads_only(stream):
    """the device results of the group, edge change and node change calls keep their bytes"""
    h = stream.h
    rows, _ = h.rollup_span(5)
    h.baseline_pin(SPAN)
    stream.random_windows(1, seed=271)
    rows, _ = h.rollup_span(3)
    set_map(h, *owners_map(rows))
    p_ge, n_ge, _ = h.group_edges_device(SPAN)
    p_nc, n_nc, _ = h.node_changes_device(IN, (Q, 0.99), source=SPAN)
    p_ec, n_ec, _ = h.edge_changes_device(abi.METRIC_COUNT, source=SPAN)
    p_gn, n_gn = h.group_nodes_device(SPAN)

    def snap():
        return [h.d2h(p_ge, n_ge, abi.EDGE_OUT).tobytes(), h.d2h(p_nc, n_nc, abi.NODE_CHANGE).tobytes(),
                h.d2h(p_ec, n_ec, abi.EDGE_CHANGE).tobytes(), h.d2h(p_gn, n_gn, abi.NODE_OUT).tobytes()]

    before = snap()
    for source in (WINDOW, WIN, SPAN):
        h.group_edge_changes((Q, 0.99), source=source)
        h.group_edge_changes_top(abi.METRIC_COUNT, 10, source=source)
        h.group_node_changes(OUT, abi.METRIC_ERR_RATE, source=source)
        h.group_node_changes_top(IN, (Q, 0.99), 10, source=source)
    assert snap() == before
    assert h.edge_changes(abi.METRIC_COUNT, source=SPAN)[0].tobytes() == h.d2h(p_ec, n_ec, abi.EDGE_CHANGE).tobytes()
    h.group_set([], [])


def test_every_error_code_sets_n():
    h = capi.Handle(device=0, max_endpoints=1 << 10, max_pairs=1 << 12)
    try:
        L, hp, m1 = h.L, h.h, abi.metrics(abi.METRIC_COUNT)
        n, pp, ci = C.c_size_t(77), C.c_void_p(), abi.ChangeInfo()

        def edge(src=WINDOW, m=m1, mode=0, pres=7, out=None, cap=0):
            n.value = 77
            return L.alz_group_edge_changes(hp, src, m, mode, pres, out, cap, C.byref(n), C.byref(ci))

        def node(src=WINDOW, side=IN, m=m1, mode=0, pres=7, k=None, mn=0.0):
            n.value = 77
            if k is None:
                return L.alz_group_node_changes(hp, src, side, m, mode, pres, None, 0, C.byref(n), C.byref(ci))
            return L.alz_group_node_changes_top(hp, src, side, m, mode, pres, k, mn, None, 0, C.byref(n), C.byref(ci))

        assert edge() == abi.E_STATE and n.value == 0   # no baseline
        assert node() == abi.E_STATE and n.value == 0
        h.flush()
        h.baseline_pin(WINDOW)
        for s in (WIN, TIER, SPAN):
            assert edge(src=s) == abi.E_STATE and n.value == 0   # a rollup source with no rows
            assert node(src=s) == abi.E_STATE and n.value == 0
        for bad in (dict(src=3), dict(src=0xFFFFFFFE), dict(mode=3), dict(pres=0), dict(pres=8),
                    dict(m=abi.metrics((9, 0.0))), dict(m=abi.metrics((Q, 1.5))), dict(out=None, cap=4)):
            assert edge(**bad) == abi.E_INVAL and n.value == 0, bad
        for bad in (dict(side=2), dict(src=3), dict(mode=7), dict(pres=9), dict(k=0), dict(k=3, mn=float("nan"))):
            assert node(**bad) == abi.E_INVAL and n.value == 0, bad
        assert L.alz_group_edge_changes_device(hp, WINDOW, m1, 0, 7, None, C.byref(n), None) == abi.E_INVAL
        assert L.alz_group_node_changes_top_device(hp, WINDOW, IN, m1, 0, 7, 3, 0.0, None, C.byref(n),
                                                   None) == abi.E_INVAL and n.value == 0
        assert L.alz_group_edge_changes(hp, WINDOW, m1, 0, 7, None, 0, None, None) == abi.E_INVAL
        # capacity: a host cap below the list, *n set, nothing written
        rng = np.random.default_rng(5)
        r = edge_rows(40, rng)
        r["from"], r["to"] = np.arange(40), 7
        src = r.copy()
        src["to"] = 8
        lst, _ = h.debug_group_edge_changes_rows(src, r, abi.METRIC_COUNT)
        assert len(lst) == 80
        ps, pb = h.dev_alloc(src.nbytes), h.dev_alloc(r.nbytes)
        try:
            h.h2d(ps, src)
            h.h2d(pb, r)
            out = np.zeros(80, dtype=abi.EDGE_CHANGE)
            assert L.alz_debug_group_edge_changes_rows(hp, C.c_void_p(ps), 40, 1, C.c_void_p(pb), 40, 1, m1, 0, 7,
                                                       out.ctypes.data_as(C.c_void_p), 79, C.byref(n),
                                                       C.byref(ci)) == abi.E_CAPACITY
            assert n.value == 80 and not out.view(np.uint8).any()
            assert L.alz_debug_group_edge_changes_rows(hp, C.c_void_p(ps), 1 << 29, 1, C.c_void_p(pb), 40, 1, m1, 0,
                                                       7, None, 0, C.byref(n), None) == abi.E_CAPACITY and n.value == 0
            assert L.alz_debug_group_edge_changes_rows(hp, C.c_void_p(ps), 40, 0, C.c_void_p(pb), 40, 1, m1, 0, 7,
                                                       None, 0, C.byref(n), None) == abi.E_INVAL
        finally:
            h.dev_free(ps)
            h.dev_free(pb)
    finally:
        h.close()


# ---- hook lists: layouts ingest cannot make --------------------------------------------------------------------

@pytest.fixture(scope="module")
def hh():
    h = capi.Handle(device=0, max_endpoints=1 << 10, max_pairs=1 << 12)
    yield h
    h.close()


def check_hook(h, src, base, gmap, what, specs=(abi.METRIC_COUNT, (Q, 0.99)), windows=(3, 7)):
    """the hook against the reference; returns the reference's full list by COUNT, DELTA"""
    ga, gb = gr.group(src, gmap)[0], gr.group(base, gmap)[0]
    for spec, mode in itertools.product(specs, MODES):
        for mask in (7, 3, 4):
            got = h.debug_group_edge_changes_rows(src, base, spec, mode, mask, *windows)
            same(got, gcr.edge_changes_of(ga, gb, spec, mode, mask, *windows), (what, spec, mode, mask))
    return gcr.edge_changes_of(ga, gb, abi.METRIC_COUNT, abi.CHANGE_DELTA, 7, *windows)[0]


def test_ends_that_collide_in_64_bits(hh):
    rng = np.random.default_rng(91)
    gmap = set_map(hh, ends(np.arange(64, dtype=np.uint64)), (np.arange(64) % 4).astype(np.uint32))
    n = 64
    src = edge_rows(n, rng)
    src["from"] = np.arange(n)
    src["to_type"], src["to"] = OUTB, np.arange(n) % 4
    base = edge_rows(n, rng)
    base["from"] = np.arange(n)
    base["to_type"], base["to"] = POD, np.arange(n) % 4   # pods 0..3 are groups 0..3: group vs outbound, one value
    lst = check_hook(hh, src, base, gmap, "group vs outbound")
    assert len(lst) == 8 and not np.any(lst["presence"] == BOTH)   # (g, outbound g) NEW, (g, group g) GONE
    src["to"] = (np.arange(n) % 8) | (1 << 31)           # outbound values past 2^31 ...
    base["to_type"], base["to"] = OUTB, np.arange(n) % 8  # ... against the same low 31 bits
    lst = check_hook(hh, src, base, gmap, "bit 31")
    assert not np.any(lst["presence"] == BOTH)
    base["to"] = src["to"]
    lst = check_hook(hh, src, base, gmap, "equal")
    assert np.all(lst["presence"] == BOTH)


def test_lists_that_differ_only_in_the_to_end(hh):
    rng = np.random.default_rng(92)
    gmap = set_map(hh, ends(np.arange(1000, dtype=np.uint64)), (np.arange(1000) // 10).astype(np.uint32))
    src = edge_rows(3000, rng)
    src["from"] = rng.integers(0, 1000, 3000)
    src["to"] = rng.integers(0, 50, 3000)
    base = src.copy()
    base["to"] = rng.integers(25, 75, 3000)
    lst = check_hook(hh, src, base, gmap, "to end", specs=SPECS)
    assert set(lst["presence"].tolist()) <= {BOTH, NEW, GONE}


def test_one_group_edge_on_2_20_rows_wrapping_cells_and_long_lists(hh):
    rng = np.random.default_rng(93)
    n = 1 << 20
    one = set_map(hh, ends(np.arange(1 << 16, dtype=np.uint64)), np.zeros(1 << 16, np.uint32))
    r = edge_rows(n, rng)
    r["from"], r["to"] = rng.integers(0, 1 << 16, n), 5
    base = r[: n // 2].copy()
    lst = check_hook(hh, r, base, one, "one group edge")
    assert len(lst) == 1 and lst[0]["presence"] == BOTH
    r["hist"], r["count"] = 0xFFFFFFFF, np.uint64((1 << 64) - 1)
    check_hook(hh, r, base, one, "wrapping cells")
    m = n + 3
    gmap = set_map(hh, ends(np.arange(1 << 16, dtype=np.uint64)), (np.arange(1 << 16) // 4).astype(np.uint32))
    a = edge_rows(m, rng)
    a["from"], a["to"] = rng.integers(0, 1 << 16, m), rng.integers(0, 1 << 12, m)
    b = edge_rows(m, rng)
    b["from"], b["to"] = rng.integers(0, 1 << 16, m), rng.integers(0, 1 << 12, m)
    lst = check_hook(hh, a, b, gmap, "2^20 + 3", specs=((Q, 0.99),))
    assert len(lst) > n // 2
    hh.group_set([], [])
