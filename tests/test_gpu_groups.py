"""GPU: groups (alz_group_set, alz_group_edges*, alz_group_edge_metrics*, alz_group_edge_top*, alz_group_nodes*,
alz_group_node_metrics*, alz_group_node_top*, alz_debug_group_edges, docs/SPEC.md §24).

Group edges, node rows, values, top indices and info are compared as bytes against tests/group_ref.py over the rows of
each source. Windows come from the Modelled stream of tests/test_gpu_edge_series.py; the hook lists build layouts
ingest cannot make: runs of every length around the reduce's warp chunk (64 rows) and block (512 rows), one group edge
on 2^20 rows, cells of 2^32 - 1."""
import ctypes as C

import numpy as np
import pytest

import group_ref as gr
import node_ref as nr
from alaz_b200 import abi, capi
from test_gpu_edge_series import Modelled, make_source
from test_gpu_gnn_rollup import universe

pytestmark = pytest.mark.gpu
WINDOW, WIN, TIER, SPAN = abi.SOURCE_WINDOW, abi.ROLLUP_WINDOWS, abi.ROLLUP_TIER, abi.ROLLUP_SPAN
IN, OUT = abi.SIDE_IN, abi.SIDE_OUT
Q = abi.METRIC_QUANTILE
ALL = [abi.METRIC_COUNT, abi.METRIC_ERR5XX, abi.METRIC_ERR_RATE, abi.METRIC_MEAN_NS, (Q, 0.5), (Q, 0.99), (Q, 1.0)]
POD, SVC, OUTB, HOST, GRP = 0, 1, 2, 3, abi.NODE_GROUP


def ends(keys):
    """NODE_ENDS of uint64 node keys"""
    e = np.zeros(len(keys), dtype=abi.NODE_ENDS)
    e["type"] = (keys >> np.uint64(32)).astype(np.uint8)
    e["value"] = (keys & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    return e


def owners_map(rows):
    """pods two per owner, each service to the owner group of its id, outbound ends to one external group"""
    keys = nr.keys(rows)
    t, v = keys >> np.uint64(32), keys & np.uint64(0xFFFFFFFF)
    g = np.where(t == POD, v // 2, np.where(t == SVC, v, 1 << 20)).astype(np.uint32)
    return ends(keys), g


def big_map(rows, n=1_000_000):
    """n entries: every node of the rows (pods by tens, the rest one group each), the keys just beside them that no
    row holds, and pods far past the universe"""
    keys = nr.keys(rows)
    near = np.unique(np.concatenate([keys - np.uint64(1), keys + np.uint64(1)]))
    near = near[~np.isin(near, keys)]
    near = near[((near >> np.uint64(32)) <= HOST) & ~(((near >> np.uint64(32)) <= SVC) &
                                                     ((near & np.uint64(0xFFFFFFFF)) >= (1 << 29)))]
    fill = np.arange(1 << 20, (1 << 20) + n - len(keys) - len(near), dtype=np.uint64)   # pods 2^20 and up
    allk = np.concatenate([keys, near, fill])
    t, v = allk >> np.uint64(32), allk & np.uint64(0xFFFFFFFF)
    g = np.where(t == POD, v // 10, (v * 7 + t) % (1 << 29)).astype(np.uint32)
    perm = np.random.default_rng(5).permutation(len(allk))
    return ends(allk[perm]), g[perm]


def set_map(h, nodes, groups):
    h.group_set(nodes, groups)
    return gr.make_map(nodes, groups) if len(nodes) else gr.EMPTY


def check_source(h, source, rows, gmap, full=True):
    """every group call of `source` against the reference over its rows, host and device forms"""
    exp, einfo = gr.group(rows, gmap)
    got, info = h.group_edges(source)
    assert info == einfo, (source, info, einfo)
    assert got.tobytes() == exp.tobytes(), (source, len(got), len(exp))
    p, n, dinfo = h.group_edges_device(source)
    assert n == len(exp) and dinfo == einfo and h.d2h(p, n, abi.EDGE_OUT).tobytes() == exp.tobytes(), source
    want = gr.edge_matrix(exp, ALL)
    assert h.group_edge_metrics(source, *ALL).tobytes() == want.tobytes(), source
    p, n = h.group_edge_metrics_device(source, *ALL)
    assert n == len(exp) and h.d2h(p, n * len(ALL), np.float64).tobytes() == want.tobytes(), source
    for spec in (ALL if full else [(Q, 0.99)]):
        for k, mv in ((17, 0.0), (len(exp) + 3, -np.inf)):
            idx, above = gr.edge_top(exp, spec, k, mv)
            rows_t, vals, index, tinfo = h.group_edge_top(source, spec, k, mv)
            what = (source, spec, k, mv)
            assert index.tobytes() == idx.tobytes(), what
            assert rows_t.tobytes() == exp[idx].tobytes(), what
            assert vals.tobytes() == want[idx, ALL.index(spec)].tobytes(), what
            assert tinfo == dict(scored=len(exp), above=above), what
            pr, pv, pi, m, di = h.group_edge_top_device(source, spec, k, mv)
            assert m == len(idx) and di == tinfo and h.d2h(pi, m, np.uint32).tobytes() == idx.tobytes(), what
            assert h.d2h(pr, m, abi.EDGE_OUT).tobytes() == exp[idx].tobytes(), what
    nodes = nr.group(exp)
    assert h.group_nodes(source).tobytes() == nodes.tobytes(), source
    p, n = h.group_nodes_device(source)
    assert n == len(nodes) and h.d2h(p, n, abi.NODE_OUT).tobytes() == nodes.tobytes(), source
    for side in (IN, OUT):
        want = nr.matrix(nodes, side, ALL)
        assert h.group_node_metrics(source, side, *ALL).tobytes() == want.tobytes(), (source, side)
        p, n = h.group_node_metrics_device(source, side, *ALL)
        assert n == len(nodes) and h.d2h(p, n * len(ALL), np.float64).tobytes() == want.tobytes(), (source, side)
        for spec in (ALL if full else [abi.METRIC_COUNT, (Q, 0.99)]):
            v = nr.values(nodes, side, spec)
            for k, mv in ((20, 0.0), (len(nodes) + 3, -np.inf)):
                idx, above = nr.top(nodes, side, spec, k, mv)
                got_n, vals, index, tinfo = h.group_node_top(source, side, spec, k, mv)
                what = (source, side, spec, k, mv)
                assert index.tobytes() == idx.tobytes(), what
                assert got_n.tobytes() == nodes[idx].tobytes() and vals.tobytes() == v[idx].tobytes(), what
                assert tinfo == dict(scored=len(nodes), above=above), what
                pn, pv, pi, m, di = h.group_node_top_device(source, side, spec, k, mv)
                assert m == len(idx) and di == tinfo, what
                assert h.d2h(pn, m, abi.NODE_OUT).tobytes() == nodes[idx].tobytes(), what
                assert h.d2h(pv, m, np.float64).tobytes() == v[idx].tobytes(), what
    return exp, nodes


@pytest.fixture(scope="module")
def mod():
    m = Modelled(universe(seed=44), history=(6, 1 << 15), tiers=[(2, 4, 1 << 15, 1 << 13)])
    m.random_windows(12, seed=441, lo=0.2, hi=0.7)
    m.last = m.window(np.flatnonzero(np.random.default_rng(442).random(m.s.g.n_edges) < 0.5))
    yield m
    m.h.group_set([], [])
    m.close()


@pytest.mark.parametrize("source", [WINDOW, WIN, TIER, SPAN])
def test_every_source_every_map(mod, source):
    h = mod.h
    rows = make_source(mod, source)
    keys = nr.keys(rows)
    # the empty map: the source's rows in node-key order, and the group nodes are the §21 nodes
    exp, nodes = check_source(h, source, rows, set_map(h, [], []))
    assert len(exp) == len(rows) and nodes.tobytes() == nr.group(rows).tobytes()
    # one entry: the first service alone in its group
    svc = keys[(keys >> np.uint64(32)) == SVC][:1]
    check_source(h, source, rows, set_map(h, ends(svc), [123]), full=False)
    # owners: pods two per owner, services to their owner's group, outbound ends to one external group
    exp, nodes = check_source(h, source, rows, set_map(h, *owners_map(rows)))
    assert (exp["from_type"] == GRP).all() and (exp["to_type"] == GRP).all()
    assert len(exp) < len(rows)
    # every pod in one group: one group that every pod row runs into
    pods = keys[(keys >> np.uint64(32)) == POD]
    exp, _ = check_source(h, source, rows, set_map(h, ends(pods), np.full(len(pods), 9, np.uint32)), full=False)
    assert ((exp["from_type"] == GRP) & (exp["to_type"] == GRP)).sum() == 1


def test_a_map_of_a_million_entries(mod):
    h = mod.h
    for source in (WINDOW, SPAN):
        rows = make_source(mod, source)
        exp, _ = check_source(h, source, rows, set_map(h, *big_map(rows)), full=False)
        assert (exp["from_type"] == GRP).any() and (exp["to_type"] == GRP).any()


def test_results_are_byte_identical_on_repeated_calls(mod):
    h = mod.h
    rows = make_source(mod, SPAN)
    set_map(h, *owners_map(rows))
    first = [h.group_edges(SPAN)[0].tobytes(), h.group_nodes(SPAN).tobytes(),
             h.group_node_metrics(SPAN, IN, *ALL).tobytes()]
    for _ in range(3):
        assert [h.group_edges(SPAN)[0].tobytes(), h.group_nodes(SPAN).tobytes(),
                h.group_node_metrics(SPAN, IN, *ALL).tobytes()] == first


def edge_rows(n, rng, cells_hi=1 << 8):
    r = np.zeros(n, dtype=abi.EDGE_OUT)
    r["from_type"], r["to_type"] = POD, SVC
    r["count"] = rng.integers(0, 1 << 40, n, dtype=np.uint64)
    r["err5xx"] = rng.integers(0, 1 << 20, n, dtype=np.uint64)
    r["lat_sum_ns"] = rng.integers(0, 1 << 62, n, dtype=np.uint64)
    r["hist"] = rng.integers(0, cells_hi, (n, abi.NB), dtype=np.uint64).astype(np.uint32)
    return r


def check_hook(h, rows, gmap, what):
    exp, einfo = gr.group(rows, gmap)
    got, info = h.debug_group_edges(rows)
    if got.tobytes() != exp.tobytes():
        bad = np.flatnonzero((got.view(np.uint8).reshape(-1, 296) != exp.view(np.uint8).reshape(-1, 296)).any(1)) \
            if len(got) == len(exp) else []
        raise AssertionError((what, len(got), len(exp), bad[:5]))
    assert info == einfo, (what, info, einfo)
    return exp


@pytest.fixture(scope="module")
def hh():
    h = capi.Handle(device=0, max_endpoints=1 << 10, max_pairs=1 << 12)
    yield h
    h.close()


def test_run_lengths_around_the_warp_chunk_and_the_block(hh):
    rng = np.random.default_rng(81)
    lengths = [31, 32, 33, 63, 64, 65, 127, 128, 129, 511, 512, 513, 1023, 1024, 1025, 4095, 4096, 4097, 1, 2, 3]
    lengths += list(range(1, 140, 3))
    # pods 0..4999 by hundreds into groups 0..49; run j: the pods of group j % 50 calling service j
    gmap = set_map(hh, ends(np.arange(5000, dtype=np.uint64)), (np.arange(5000) // 100).astype(np.uint32))
    parts = []
    for j, L in enumerate(lengths):
        r = edge_rows(L, rng)
        r["from"] = (j % 50) * 100 + rng.integers(0, 100, L)
        r["to"] = j
        parts.append(r)
    rows = np.concatenate(parts)
    exp = check_hook(hh, rows[rng.permutation(len(rows))], gmap, "runs")
    assert sorted(exp["count"].tolist()) == sorted(int(p["count"].sum()) for p in parts)
    # runs laid end to end in sorted order, each at an offset that puts its ends on every side of a boundary
    for L in lengths[:18]:
        for lead in (0, 1, 63, 64, 65, 511, 512, 513):
            a = edge_rows(lead, rng)
            a["from"] = rng.integers(0, 100, lead)        # group 0 -> service 0: sorts first
            a["to"] = 0
            b = edge_rows(L, rng)
            b["from"] = 100 + rng.integers(0, 100, L)     # group 1 -> service 0: the run under test
            b["to"] = 0
            c = edge_rows(70, rng)
            c["from"] = 200 + rng.integers(0, 100, 70)    # group 2 -> service 0 after it
            c["to"] = 0
            check_hook(hh, np.concatenate([a, b, c]), gmap, ("run", L, lead))


def test_lists_of_2_20_rows_uniform_one_group_edge_and_wrapping_cells(hh):
    rng = np.random.default_rng(82)
    n = 1 << 20
    r = edge_rows(n, rng)
    r["from"] = rng.integers(0, 1 << 16, n)
    r["to"] = rng.integers(0, 1 << 10, n)
    gmap = set_map(hh, ends(np.arange(1 << 16, dtype=np.uint64)), (np.arange(1 << 16) // 4).astype(np.uint32))
    exp = check_hook(hh, r, gmap, "uniform")
    assert len(exp) > n // 2
    one = set_map(hh, ends(np.arange(1 << 16, dtype=np.uint64)), np.zeros(1 << 16, np.uint32))
    r["to"] = 5
    exp = check_hook(hh, r, one, "one group edge")
    assert len(exp) == 1
    r["hist"] = 0xFFFFFFFF
    r["count"] = np.uint64((1 << 64) - 1)
    exp = check_hook(hh, r, one, "wrapping cells")
    assert int(exp["hist"][0, 0]) == (n * 0xFFFFFFFF) % (1 << 32)
    assert int(exp["count"][0]) == ((1 << 64) - n) % (1 << 64)
    assert len(hh.debug_group_edges(np.zeros(0, dtype=abi.EDGE_OUT))[0]) == 0


def raw_set(h, nodes, groups, n=None):
    nodes = np.ascontiguousarray(nodes, dtype=abi.NODE_ENDS)
    groups = np.ascontiguousarray(groups, dtype=np.uint32)
    return h.L.alz_group_set(h.h, nodes.ctypes.data_as(C.c_void_p), groups.ctypes.data_as(C.c_void_p),
                             len(nodes) if n is None else n)


def test_every_error_code_and_a_failed_set_keeps_the_map(mod):
    h = mod.h
    L, hp, n = h.L, h.h, C.c_size_t(77)
    rows = make_source(mod, WINDOW)
    gmap = set_map(h, *owners_map(rows))
    before = h.group_edges(WINDOW)[0].tobytes()
    assert before == gr.group(rows, gmap)[0].tobytes()
    good = ends(np.array([1, 2], np.uint64))
    for nodes, groups in ((ends(np.array([(5 << 32) | 1], np.uint64)), [1]),          # type above HOST
                          (ends(np.array([1 << 29], np.uint64)), [1]),                # pod id >= 2^29
                          (ends(np.array([(1 << 32) | (1 << 29)], np.uint64)), [1]),  # service id >= 2^29
                          (good, [1, 1 << 29]),                                       # group >= 2^29
                          (ends(np.array([3, 4, 3], np.uint64)), [1, 2, 3])):         # one node twice
        assert raw_set(h, nodes, groups) == abi.E_INVAL
        assert h.group_edges(WINDOW)[0].tobytes() == before
    assert L.alz_group_set(hp, None, None, 3) == abi.E_INVAL
    assert raw_set(h, good, [1, 2], n=1 << 30) == abi.E_CAPACITY
    assert h.group_edges(WINDOW)[0].tobytes() == before
    # host outbound and Host-keyed ends with values past 2^29 are members like any other
    assert raw_set(h, ends(np.array([(2 << 32) | 0xFFFFFFFF, (3 << 32) | 0xFFFFFFFF], np.uint64)), [0, 1]) == 0
    m1 = abi.metrics(abi.METRIC_COUNT)
    info, ginfo = abi.TopInfo(), abi.GroupInfo()
    pp = C.c_void_p()
    for src in (3, 7, 0xFFFFFFFE):
        assert L.alz_group_edges(hp, src, None, 0, C.byref(n), C.byref(ginfo)) == abi.E_INVAL and n.value == 0
        assert L.alz_group_nodes(hp, src, None, 0, C.byref(n)) == abi.E_INVAL and n.value == 0
        assert L.alz_group_edge_metrics(hp, src, m1, 1, None, 0, C.byref(n)) == abi.E_INVAL
        assert L.alz_group_node_metrics(hp, src, IN, m1, 1, None, 0, C.byref(n)) == abi.E_INVAL
    assert L.alz_group_node_metrics(hp, WINDOW, 2, m1, 1, None, 0, C.byref(n)) == abi.E_INVAL
    assert L.alz_group_node_top(hp, WINDOW, 2, m1, 3, 0.0, None, None, None, 0, C.byref(n), None) == abi.E_INVAL
    for nm in (0, 9):
        assert L.alz_group_edge_metrics(hp, WINDOW, abi.metrics(*([0] * max(nm, 1))), nm, None, 0,
                                        C.byref(n)) == abi.E_INVAL
    for bad in (abi.metrics((9, 0.0)), abi.metrics((Q, 1.5)), abi.metrics((Q, float("nan")))):
        assert L.alz_group_edge_metrics(hp, WINDOW, bad, 1, None, 0, C.byref(n)) == abi.E_INVAL
        assert L.alz_group_edge_top(hp, WINDOW, bad, 3, 0.0, None, None, None, 0, C.byref(n), None) == abi.E_INVAL
    assert L.alz_group_edge_top(hp, WINDOW, m1, 0, 0.0, None, None, None, 0, C.byref(n), None) == abi.E_INVAL
    assert L.alz_group_node_top(hp, WINDOW, IN, m1, 3, float("nan"), None, None, None, 0, C.byref(n),
                                None) == abi.E_INVAL
    assert L.alz_group_edges(hp, WINDOW, None, 0, None, None) == abi.E_INVAL
    assert L.alz_group_edges(hp, WINDOW, None, 5, C.byref(n), None) == abi.E_INVAL
    assert L.alz_group_edges_device(hp, WINDOW, None, C.byref(n), None) == abi.E_INVAL and n.value == 0
    assert L.alz_group_nodes_device(hp, WINDOW, None, C.byref(n)) == abi.E_INVAL
    assert L.alz_group_edge_metrics_device(hp, WINDOW, m1, 1, None, C.byref(n)) == abi.E_INVAL
    assert L.alz_debug_group_edges(hp, None, 4, None, 0, C.byref(n), None) == abi.E_INVAL
    # capacity: *n set, nothing written
    exp = gr.group(rows, gr.EMPTY)[0]
    h.group_set([], [])
    out = np.zeros(len(exp), dtype=abi.EDGE_OUT)
    assert L.alz_group_edges(hp, WINDOW, out.ctypes.data_as(C.c_void_p), len(exp) - 1, C.byref(n),
                             C.byref(ginfo)) == abi.E_CAPACITY
    assert n.value == len(exp) and not out.view(np.uint8).any() and ginfo.edges == len(exp)
    nodes = nr.group(exp)
    assert L.alz_group_nodes(hp, WINDOW, None, 0, C.byref(n)) == abi.E_CAPACITY and n.value == len(nodes)
    assert L.alz_group_node_metrics(hp, WINDOW, IN, m1, 1, None, 0, C.byref(n)) == abi.E_CAPACITY
    assert L.alz_group_edge_top(hp, WINDOW, m1, 5, 0.0, None, None, None, 2, C.byref(n), C.byref(info)) == \
        abi.E_CAPACITY and n.value == 5
    assert L.alz_group_edges_device(hp, WINDOW, C.byref(pp), C.byref(n), None) == 0 and n.value == len(exp)


def test_rollup_sources_without_rows_and_an_empty_window():
    h = capi.Handle(device=0, max_endpoints=1 << 10, max_pairs=1 << 12)
    try:
        L, n, m1 = h.L, C.c_size_t(77), abi.metrics(abi.METRIC_COUNT)
        h.group_set([(POD, 1)], [1])
        for s in (WIN, TIER, SPAN):
            assert L.alz_group_edges(h.h, s, None, 0, C.byref(n), None) == abi.E_STATE and n.value == 0
            assert L.alz_group_nodes(h.h, s, None, 0, C.byref(n)) == abi.E_STATE
            assert L.alz_group_node_top(h.h, s, IN, m1, 3, 0.0, None, None, None, 0, C.byref(n), None) == abi.E_STATE
        got, info = h.group_edges(WINDOW)
        assert len(got) == 0 and info == dict(source_rows=0, mapped_ends=0, edges=0, internal=0)
        assert len(h.group_nodes(WINDOW)) == 0
        assert len(h.group_node_top(WINDOW, IN, abi.METRIC_COUNT, 5)[0]) == 0
    finally:
        h.close()


def test_reads_only(mod):
    """the window, every rollup's rows, the baseline and every other family's device results keep their bytes"""
    h = mod.h
    h.group_set([], [])
    for s in (WIN, TIER, SPAN):
        make_source(mod, s)
    h.baseline_pin(SPAN)
    def fetch():
        out, n = np.zeros(len(mod.last) + 1, dtype=abi.EDGE_OUT), C.c_size_t(0)
        h._ck(h.L.alz_window_fetch(h.h, out.ctypes.data_as(C.c_void_p), len(out), C.byref(n)), "alz_window_fetch")
        return out[: n.value].tobytes()

    stored = lambda: [fetch(), h.edge_metrics(*ALL).tobytes()] + [h.edge_metrics_rollup(s, *ALL).tobytes()
                                                                   for s in (WIN, TIER, SPAN)]
    rows_before = stored()
    p_node, n_node = h.node_rows_device(SPAN)
    p_met, n_met = h.edge_metrics_rollup_device(SPAN, *ALL)
    p_top = h.edge_top_rollup_device(SPAN, abi.METRIC_COUNT, 50)
    p_ch, n_ch, _ = h.node_changes_device(IN, abi.METRIC_COUNT, source=WINDOW)
    p_ser = h.node_series_device(SPAN, IN, 0, 4, *ALL)
    p_tr = h.edge_trends_device(SPAN, 0, 4, abi.METRIC_COUNT, abi.Trend(stat=abi.TREND_SLOPE, recent=1, min_points=2))
    try:
        p_gnn = h.gnn_score_rollup_device(SPAN)
    except capi.AlzError as e:   # built without the GNN pass
        assert e.status == abi.E_UNSUPPORTED
        p_gnn = (0, 0)

    def snap():
        return [h.d2h(p_node, n_node, abi.NODE_OUT).tobytes(), h.d2h(p_met, n_met * len(ALL), np.float64).tobytes(),
                h.d2h(p_top[0], p_top[3], abi.EDGE_OUT).tobytes(), h.d2h(p_ch, n_ch, abi.NODE_CHANGE).tobytes(),
                h.d2h(p_ser[0], p_ser[2] * p_ser[3] * len(ALL), np.float64).tobytes(),
                h.d2h(p_tr[0], p_tr[1], abi.EDGE_TREND).tobytes(),
                h.d2h(p_gnn[0], p_gnn[1], np.float32).tobytes() if p_gnn[1] else b""]

    before = snap()
    set_map(h, *owners_map(make_source(mod, SPAN)))
    for s in (WINDOW, WIN, TIER, SPAN):
        h.group_edges(s)
        h.group_edge_metrics(s, *ALL)
        h.group_node_top(s, IN, (Q, 0.99), 10)
        h.group_edge_top(s, abi.METRIC_COUNT, 10)
    assert snap() == before
    base = h.edge_changes(abi.METRIC_COUNT, source=SPAN)[0]
    assert (base["presence"] == abi.PRESENT_BOTH).all()   # the span against its own pin: the baseline is intact
    assert stored() == rows_before
    h.group_set([], [])
