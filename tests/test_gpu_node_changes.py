"""GPU: node changes against a pinned baseline (alz_node_changes*, alz_node_changes_top*, alz_debug_node_changes_rows,
docs/SPEC.md §23).

The expected lists and top results are tests/node_change_ref.py over the same rows, compared as bytes: node, indices,
presence, padding and the bits of value, base value and change. Windows and rollups come from the Stream of
tests/test_gpu_gnn_rollup.py; the hook runs the join over layouts ingest cannot make."""
import ctypes as C
import itertools

import numpy as np
import pytest

import metric_ref
import node_change_ref as ncr
import node_ref as nr
from alaz_b200 import abi, capi
from test_gpu_edge_changes import Sources
from test_gpu_gnn_rollup import Stream, universe
from test_gpu_node_metrics import edge_rows

pytestmark = pytest.mark.gpu
WINDOW, WIN, TIER, SPAN = abi.SOURCE_WINDOW, abi.ROLLUP_WINDOWS, abi.ROLLUP_TIER, abi.ROLLUP_SPAN
IN, OUT = abi.SIDE_IN, abi.SIDE_OUT
Q = abi.METRIC_QUANTILE
SPECS = [abi.METRIC_COUNT, abi.METRIC_ERR5XX, abi.METRIC_ERR_RATE, abi.METRIC_MEAN_NS, (Q, 0.0), (Q, 0.5), (Q, 0.99),
         (Q, 1.0)]
MODES = [abi.CHANGE_DELTA, abi.CHANGE_DROP, abi.CHANGE_RATIO]
MASKS = list(range(1, 8))
POD, SVC = abi.NODE_POD, abi.NODE_SVC


def same(got, want, what):
    got_l, got_i = got
    want_l, want_i = want
    assert got_i == want_i, (what, got_i, want_i)
    assert got_l.tobytes() == want_l.tobytes(), (what, len(got_l), len(want_l),
                                                 np.flatnonzero(got_l != want_l)[:5] if len(got_l) == len(want_l)
                                                 else None)


def top_of(lst, info, k, mn):
    idx, above = metric_ref.top(lst["change"], k, mn)
    return lst[idx], dict(info, above=above)


def check_all(h, src_rows, src_w, base_rows, base_w, source, what):
    na, nb = nr.group(src_rows), nr.group(base_rows)
    for side in (IN, OUT):
        for spec, mode in itertools.product(SPECS, MODES):
            want = ncr.changes_of_nodes(na, nb, side, spec, mode, 7, src_w, base_w)
            same(h.node_changes(side, spec, mode, 7, source=source), want, (what, side, spec, mode))
        for mask in MASKS:
            spec, mode = SPECS[mask], MODES[mask % 3]
            want = ncr.changes_of_nodes(na, nb, side, spec, mode, mask, src_w, base_w)
            same(h.node_changes(side, spec, mode, mask, source=source), want, (what, side, spec, mode, mask))
        for (spec, mode), mask in itertools.product(((abi.METRIC_COUNT, abi.CHANGE_DELTA), ((Q, 0.99), abi.CHANGE_RATIO),
                                                     (abi.METRIC_ERR_RATE, abi.CHANGE_DROP)), (7, 5)):
            lst, info = ncr.changes_of_nodes(na, nb, side, spec, mode, mask, src_w, base_w)
            fin = lst["change"][np.isfinite(lst["change"])]
            mid = float(np.median(fin)) if len(fin) else 0.0
            for k, mn in itertools.product((1, 100, len(lst) + 5), (-np.inf, mid, np.inf)):
                got = h.node_changes_top(side, spec, k, mn, mode, mask, source=source)
                same(got, top_of(lst, info, k, mn), (what, "top", side, spec, mode, mask, k, mn))


@pytest.fixture(scope="module")
def stream():
    s = Stream(universe(seed=14), history=(6, 1 << 15), tiers=[(2, 4, 1 << 15, 1 << 13)])
    s.random_windows(9, seed=141, lo=0.2, hi=0.6)
    yield s
    s.close()


@pytest.mark.parametrize("base_kind", [WINDOW, WIN, TIER, SPAN])
def test_every_source_against_every_baseline_kind(stream, base_kind):
    src = Sources(stream)
    h = stream.h
    base_rows, _ = src.make(base_kind, {WINDOW: 1, WIN: 4, TIER: 2, SPAN: 6}[base_kind])
    pinned = h.baseline_pin(base_kind)
    stream.random_windows(2, seed=142 + base_kind % 7, lo=0.2, hi=0.6)   # the baseline survives flushes
    for kind, param in ((WINDOW, 5), (WIN, 3), (TIER, 1), (SPAN, 3)):
        rows, _ = src.make(kind, param)
        check_all(h, rows, src.windows[kind], base_rows, pinned["windows"], kind, (base_kind, kind))


@pytest.mark.parametrize("source", [WINDOW, WIN, SPAN])
def test_values_are_the_node_metrics_of_the_source(stream, source):
    h = stream.h
    src = Sources(stream)
    src.make(WIN, 5)
    h.baseline_pin(WIN)
    rows, _ = src.make(source, {WINDOW: 9, WIN: 2, SPAN: 4}[source])
    w = src.windows[source]
    for side, spec in itertools.product((IN, OUT), SPECS):
        vals = h.node_metrics(source, side, spec).reshape(-1)
        lst, _ = h.node_changes(side, spec, abi.CHANGE_DELTA, abi.PRESENT_BOTH | abi.PRESENT_NEW, source=source)
        assert len(lst) and np.all(lst["index"] != abi.ABSENT)
        want = vals[lst["index"]]
        if spec in (abi.METRIC_COUNT, abi.METRIC_ERR5XX):
            want = want / np.float64(w)
        assert lst["value"].tobytes() == want.tobytes(), (source, side, spec)
        nodes = h.node_rows(source)[lst["index"]]
        assert np.all(nodes["type"] == lst["type"]) and np.all(nodes["value"] == lst["node"])


def test_a_source_against_itself_is_all_both_with_no_change(stream):
    h = stream.h
    for source, param in ((WIN, 3), (SPAN, 5)):
        rows, _ = (h.rollup(param) if source == WIN else h.rollup_span(param))
        h.baseline_pin(source)
        for side, spec in itertools.product((IN, OUT), SPECS):
            lst, info = h.node_changes(side, spec, abi.CHANGE_DELTA, source=source)
            assert np.all(lst["presence"] == abi.PRESENT_BOTH) and info["added"] == info["gone"] == 0
            assert np.all(lst["index"] == lst["base_index"])
            assert np.all(lst["change"].view(np.uint64) == 0), (source, side, spec)   # +0.0
            lst, _ = h.node_changes(side, spec, abi.CHANGE_RATIO, source=source)
            assert np.all(lst["change"] == 1.0)
            nodes = nr.group(rows)
            assert info["source_rows"] == int((nodes["in_edges" if side == IN else "out_edges"] > 0).sum())


def test_device_variants_equal_host(stream):
    h = stream.h
    h.baseline_pin(WINDOW)
    stream.random_windows(1, seed=17)
    for side, spec in itertools.product((IN, OUT), (abi.METRIC_COUNT, (Q, 0.99))):
        lst, info = h.node_changes(side, spec, abi.CHANGE_RATIO, 7)
        p, n, dinfo = h.node_changes_device(side, spec, abi.CHANGE_RATIO, 7)
        assert n == len(lst) and dinfo == info
        assert h.d2h(p, n, abi.NODE_CHANGE).tobytes() == lst.tobytes()
        top, tinfo = h.node_changes_top(side, spec, 20, 0.0, abi.CHANGE_RATIO, 7)
        p, n, dinfo = h.node_changes_top_device(side, spec, 20, 0.0, abi.CHANGE_RATIO, 7)
        assert n == len(top) and dinfo == tinfo
        assert h.d2h(p, n, abi.NODE_CHANGE).tobytes() == top.tobytes()


def test_a_re_pin_replaces_the_cached_baseline_nodes_and_clear_removes_them():
    s = Stream(universe(seed=15), history=(4, 1 << 15))
    h = s.h
    try:
        s.random_windows(3, seed=151)
        base1, i1 = h.rollup(2)
        h.baseline_pin(WIN)
        cur = s.window(np.arange(0, 700))
        first = h.node_changes(IN, abi.METRIC_COUNT)
        same(first, ncr.changes(cur, base1, IN, abi.METRIC_COUNT, abi.CHANGE_DELTA, 7, 1, i1["windows"]), "first")
        same(h.node_changes(IN, abi.METRIC_COUNT), first, "cached")
        base2 = s.window(np.arange(300, 1500))
        h.baseline_pin(WINDOW)
        second = h.node_changes(IN, abi.METRIC_COUNT)
        assert second[0].tobytes() != first[0].tobytes()
        same(second, ncr.changes(base2, base2, IN, abi.METRIC_COUNT, abi.CHANGE_DELTA, 7), "re-pinned")
        # the hook groups its own lists and leaves the next call to regroup the baseline
        h.debug_node_changes_rows(cur, base1, OUT, abi.METRIC_COUNT)
        same(h.node_changes(OUT, (Q, 0.5)), ncr.changes(base2, base2, OUT, (Q, 0.5), abi.CHANGE_DELTA, 7), "after hook")
        h.baseline_clear()
        with pytest.raises(capi.AlzError) as e:
            h.node_changes(IN, abi.METRIC_COUNT)
        assert e.value.status == abi.E_STATE
        h.baseline_pin(WINDOW)
        same(h.node_changes(OUT, abi.METRIC_ERR_RATE),
             ncr.changes(base2, base2, OUT, abi.METRIC_ERR_RATE, abi.CHANGE_DELTA, 7), "pinned after clear")
    finally:
        s.close()


def test_reads_only():
    s = Stream(universe(seed=16), history=(5, 1 << 15), tiers=[(2, 3, 1 << 15, 1 << 13)])
    h = s.h
    try:
        s.random_windows(8, seed=161, lo=0.2, hi=0.6)
        h.rollup(3)
        h.baseline_pin(WIN)
        s.random_windows(2, seed=162)
        span_rows = h.rollup_span(5)[0]
        h.rollup(2)
        base = h.edge_changes(abi.METRIC_COUNT)
        nr_p, nr_n = h.node_rows_device(SPAN)
        nm_p, nm_n = h.node_metrics_device(WIN, IN, (Q, 0.99))
        ns_v, ns_p, ns_n, ns_P, _, _ = h.node_series_device(SPAN, OUT, 0, 4, abi.METRIC_COUNT)
        ec_p, ec_n, _ = h.edge_changes_device((Q, 0.99), abi.CHANGE_RATIO)
        em_p, em_n = h.edge_metrics_rollup_device(SPAN, abi.METRIC_COUNT)
        g_p, g_n = h.gnn_score_rollup_device(WIN)

        def snapshot():
            return dict(nodes=h.d2h(nr_p, nr_n, abi.NODE_OUT), node_metrics=h.d2h(nm_p, nm_n, np.float64),
                        series=h.d2h(ns_v, ns_n * ns_P, np.float64), series_p=h.d2h(ns_p, ns_n * ns_P, np.uint8),
                        changes=h.d2h(ec_p, ec_n, abi.EDGE_CHANGE), metrics=h.d2h(em_p, em_n, np.float64),
                        gnn=h.d2h(g_p, g_n, np.float32))

        before = snapshot()
        for src in (WINDOW, WIN, SPAN):
            for side in (IN, OUT):
                h.node_changes(side, (Q, 0.99), abi.CHANGE_RATIO, source=src)
                h.node_changes_top_device(side, abi.METRIC_COUNT, 5, source=src)
        h.debug_node_changes_rows(span_rows, span_rows[::3], IN, abi.METRIC_COUNT)
        after = snapshot()
        for k in before:
            assert before[k].tobytes() == after[k].tobytes(), k
        same(h.edge_changes(abi.METRIC_COUNT), base, "edge changes")
        assert h.rollup_span(5)[0].tobytes() == span_rows.tobytes()
    finally:
        s.close()


def raw(h, fn, *args):
    """(status, n_out) of fn with a null output."""
    n = C.c_size_t(777)
    info = abi.ChangeInfo()
    rc = getattr(h.L, fn)(h.h, *args, C.byref(n), C.byref(info))
    return rc, n.value


def test_every_error_code():
    s = Stream(universe(seed=17, n_edges=400), history=(3, 1 << 14))
    h = s.h
    try:
        m = abi.metrics(abi.METRIC_COUNT)
        bad_q = abi.metrics((Q, 1.5))
        bad_kind = (abi.Metric * 1)(abi.Metric(9, 0, 0.0))
        fn, top = "alz_node_changes", "alz_node_changes_top"
        # no baseline
        assert raw(h, fn, WINDOW, IN, m, 0, 7, None, 0)[0] == abi.E_STATE
        assert raw(h, top, WINDOW, IN, m, 0, 7, 5, 0.0, None, 0)[0] == abi.E_STATE
        s.random_windows(2, seed=1)
        assert h.L.alz_baseline_pin(h.h, WINDOW, None) == 0
        # no rollup rows
        for kind in (WIN, TIER, SPAN):
            assert raw(h, fn, kind, OUT, m, 0, 7, None, 0)[0] == abi.E_STATE
        # invalid arguments
        assert raw(h, fn, 3, IN, m, 0, 7, None, 0)[0] == abi.E_INVAL                    # unknown source
        assert raw(h, fn, WINDOW, 2, m, 0, 7, None, 0)[0] == abi.E_INVAL                # unknown side
        assert raw(h, fn, WINDOW, IN, bad_kind, 0, 7, None, 0)[0] == abi.E_INVAL
        assert raw(h, fn, WINDOW, IN, bad_q, 0, 7, None, 0)[0] == abi.E_INVAL
        assert raw(h, fn, WINDOW, IN, None, 0, 7, None, 0)[0] == abi.E_INVAL
        assert raw(h, fn, WINDOW, IN, m, 3, 7, None, 0)[0] == abi.E_INVAL                # unknown mode
        assert raw(h, fn, WINDOW, IN, m, 0, 0, None, 0)[0] == abi.E_INVAL                # presence 0
        assert raw(h, fn, WINDOW, IN, m, 0, 8, None, 0)[0] == abi.E_INVAL                # presence above 7
        assert raw(h, fn, WINDOW, IN, m, 0, 7, None, 5)[0] == abi.E_INVAL                # null out with cap
        assert raw(h, top, WINDOW, IN, m, 0, 7, 0, 0.0, None, 0)[0] == abi.E_INVAL       # k = 0
        assert raw(h, top, WINDOW, IN, m, 0, 7, 5, float("nan"), None, 0)[0] == abi.E_INVAL
        assert h.L.alz_node_changes_device(h.h, WINDOW, IN, m, 0, 7, None, None, None) == abi.E_INVAL
        assert h.L.alz_node_changes_top_device(h.h, WINDOW, IN, m, 0, 7, 5, 0.0, None, None, None) == abi.E_INVAL
        assert h.L.alz_node_changes(None, WINDOW, IN, m, 0, 7, None, 0, None, None) == abi.E_INVAL
        # capacity: *n_out set, nothing written
        rc, n = raw(h, fn, WINDOW, IN, m, 0, 7, None, 0)
        assert rc == abi.E_CAPACITY and n > 0
        out = np.zeros(n - 1, abi.NODE_CHANGE)
        out.view(np.uint8)[:] = 0xAB
        nn, info = C.c_size_t(0), abi.ChangeInfo()
        assert h.L.alz_node_changes(h.h, WINDOW, IN, m, 0, 7, out.ctypes.data_as(C.c_void_p), n - 1, C.byref(nn),
                                    C.byref(info)) == abi.E_CAPACITY
        assert nn.value == n and np.all(out.view(np.uint8) == 0xAB) and info.listed == n
        rc, n = raw(h, top, WINDOW, OUT, m, 0, 7, 3, -np.inf, None, 0)
        assert rc == abi.E_CAPACITY and n == 3
        # the hook: windows 0, null rows, a side above the 2^29 - 1 row limit (refused before anything is read)
        hook = "alz_debug_node_changes_rows"
        assert raw(h, hook, None, 0, 0, None, 0, 1, IN, m, 0, 7, None, 0)[0] == abi.E_INVAL
        assert raw(h, hook, None, 5, 1, None, 0, 1, IN, m, 0, 7, None, 0)[0] == abi.E_INVAL
        assert raw(h, hook, None, 0, 1, None, 0, 1, 2, m, 0, 7, None, 0)[0] == abi.E_INVAL
        assert raw(h, hook, None, 0, 1, None, 0, 1, IN, m, 0, 7, None, 0) == (0, 0)
        assert raw(h, hook, C.c_void_p(16), 1 << 29, 1, None, 0, 1, IN, m, 0, 7, None, 0)[0] == abi.E_CAPACITY
        assert raw(h, hook, None, 0, 1, C.c_void_p(16), 1 << 29, 1, OUT, m, 0, 7, None, 0)[0] == abi.E_CAPACITY
        # an empty source and an empty baseline are valid
        s.window(np.zeros(0, dtype=np.int64))
        lst, info = h.node_changes(IN, abi.METRIC_COUNT)
        assert info["source_rows"] == 0 and info["gone"] == info["base_rows"] == len(lst) > 0
        assert h.baseline_pin(WINDOW)["rows_in"] == 0
        s.random_windows(1, seed=3)
        lst, info = h.node_changes(OUT, abi.METRIC_COUNT)
        assert info["base_rows"] == 0 and info["added"] == info["source_rows"] == len(lst) > 0
    finally:
        s.close()


# ---- constructed layouts through the hook -------------------------------------------------------------------------

@pytest.fixture(scope="module")
def hh():
    h = capi.Handle(device=0, max_endpoints=1 << 10, max_pairs=1 << 12)
    yield h
    h.close()


def hook_check(h, a, b, what, specs=(abi.METRIC_COUNT, (Q, 0.99)), modes=MODES, masks=(7, 1, 6), wa=5, wb=60):
    na, nb = nr.group(a), nr.group(b)
    for side, spec, mode, mask in itertools.product((IN, OUT), specs, modes, masks):
        got = h.debug_node_changes_rows(a, b, side, spec, mode, mask, wa, wb)
        same(got, ncr.changes_of_nodes(na, nb, side, spec, mode, mask, wa, wb), (what, side, spec, mode, mask))


def test_hub_of_2_20_callers(hh):
    rng = np.random.default_rng(81)
    n = 1 << 20
    a = edge_rows(n, rng)
    a["from"] = rng.permutation(n)   # 2^20 pods calling service 5
    a["to"] = 5
    b = edge_rows(n // 2, rng)
    b["from"] = rng.permutation(n)[: n // 2]
    b["to"] = np.where(rng.random(n // 2) < 0.5, 5, 6)
    hook_check(hh, a, b, "hub", specs=((Q, 0.99),), modes=(abi.CHANGE_RATIO,), masks=(7,))


def test_members_on_one_side_only(hh):
    rng = np.random.default_rng(82)
    n = 3000
    # pods 0..999 only call in the source and are only called in the baseline, services the other way round
    a = edge_rows(n, rng, from_type=POD, to_type=SVC)
    a["from"], a["to"] = rng.integers(0, 1000, n), rng.integers(0, 50, n)
    b = edge_rows(n, rng, from_type=SVC, to_type=POD)
    b["from"], b["to"] = rng.integers(0, 50, n), rng.integers(0, 1000, n)
    hook_check(hh, a, b, "one side")
    lst, info = hh.debug_node_changes_rows(a, b, IN, abi.METRIC_COUNT)
    assert info["both"] == 0 and set(lst["presence"]) == {abi.PRESENT_NEW, abi.PRESENT_GONE}


@pytest.mark.parametrize("n", [1, 15, 16, 17, 31, 32, 33, 63, 64, 65, 4095, 4096, 4097])
def test_lists_around_tile_boundaries(hh, n):
    # n rows pod i -> service i: 2n nodes, so node lists of 2n and pair runs ending at every tile offset
    rng = np.random.default_rng(n)
    a = edge_rows(n, rng)
    a["from"] = np.arange(n)
    a["to"] = np.arange(n)
    b = edge_rows(n + 1, rng)
    b["from"] = np.arange(n + 1) + n // 2
    b["to"] = np.arange(n + 1) // 2
    hook_check(hh, a, b, ("tiles", n))


def test_2_20_plus_3_rows(hh):
    rng = np.random.default_rng(83)
    n = (1 << 20) + 3
    a = edge_rows(n, rng)
    a["from_type"], a["to_type"] = rng.integers(0, 2, n), rng.integers(0, 4, n)
    a["from"], a["to"] = rng.integers(0, 1 << 17, n), rng.integers(0, 1 << 16, n)
    b = a[rng.permutation(n)[: n // 2]].copy()
    b["count"] = rng.integers(0, 1 << 40, len(b), dtype=np.uint64)
    b["to"] = b["to"] + np.uint32(7)
    hook_check(hh, a, b, "large", specs=(abi.METRIC_ERR5XX, (Q, 0.5)), modes=(abi.CHANGE_DELTA,), masks=(7, 2))
