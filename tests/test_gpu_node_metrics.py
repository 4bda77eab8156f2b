"""GPU: node metrics (alz_node_rows*, alz_node_metrics*, alz_node_top*, alz_debug_node_rows, docs/SPEC.md §21).

Node rows, values, top indices and info are compared as bytes against tests/node_ref.py over the rows of each source.
Windows come from the Modelled stream of tests/test_gpu_edge_series.py; the hook lists build layouts ingest cannot
make: a hub of 2^20 callers, every run length around the reduce's tile boundaries, wrapping cells split over tiles."""
import ctypes as C

import numpy as np
import pytest

import node_ref as nr
from alaz_b200 import abi, capi
from test_gpu_edge_series import Modelled, make_source
from test_gpu_gnn_rollup import Stream, universe

pytestmark = pytest.mark.gpu
WINDOW, WIN, TIER, SPAN = abi.SOURCE_WINDOW, abi.ROLLUP_WINDOWS, abi.ROLLUP_TIER, abi.ROLLUP_SPAN
IN, OUT = abi.SIDE_IN, abi.SIDE_OUT
Q = abi.METRIC_QUANTILE
ALL = [abi.METRIC_COUNT, abi.METRIC_ERR5XX, abi.METRIC_ERR_RATE, abi.METRIC_MEAN_NS, (Q, 0.5), (Q, 0.99), (Q, 1.0)]
SUMS = [abi.METRIC_MEAN_NS, abi.METRIC_COUNT, abi.METRIC_ERR_RATE]
POD, SVC, OUTB, HOST = 0, 1, 2, 3


@pytest.fixture(scope="module")
def mod():
    m = Modelled(universe(seed=34), history=(6, 1 << 15), tiers=[(2, 4, 1 << 15, 1 << 13)])
    m.random_windows(12, seed=341, lo=0.2, hi=0.7)
    m.last = m.window(np.flatnonzero(np.random.default_rng(342).random(m.s.g.n_edges) < 0.5))
    yield m
    m.close()


def check_source(h, source, rows):
    """every node call of `source` against the reference over its rows, host and device forms"""
    exp = nr.group(rows)
    got = h.node_rows(source)
    assert got.tobytes() == exp.tobytes(), (source, len(got), len(exp))
    p, n = h.node_rows_device(source)
    assert n == len(exp) and h.d2h(p, n, abi.NODE_OUT).tobytes() == exp.tobytes(), source
    for side in (IN, OUT):
        for specs in (ALL, SUMS, [(Q, 0.99)]):
            want = nr.matrix(exp, side, specs)
            assert h.node_metrics(source, side, *specs).tobytes() == want.tobytes(), (source, side, specs)
            p, n = h.node_metrics_device(source, side, *specs)
            assert n == len(exp) and h.d2h(p, n * len(specs), np.float64).tobytes() == want.tobytes(), (source, side)
        for spec in ALL:
            v = nr.values(exp, side, spec)
            for k, mv in ((17, 0.0), (len(exp) + 3, -np.inf), (5, float(np.median(v)) if len(v) else 0.0)):
                idx, above = nr.top(exp, side, spec, k, mv)
                nodes, vals, index, info = h.node_top(source, side, spec, k, mv)
                what = (source, side, spec, k, mv)
                assert index.tobytes() == idx.tobytes(), (what, index[:8], idx[:8])
                assert nodes.tobytes() == exp[idx].tobytes() and vals.tobytes() == v[idx].tobytes(), what
                assert info == dict(scored=len(exp), above=above), (what, info)
                pn, pv, pi, m, dinfo = h.node_top_device(source, side, spec, k, mv)
                assert m == len(idx) and dinfo == info, what
                assert h.d2h(pn, m, abi.NODE_OUT).tobytes() == exp[idx].tobytes(), what
                assert h.d2h(pv, m, np.float64).tobytes() == v[idx].tobytes(), what
                assert h.d2h(pi, m, np.uint32).tobytes() == idx.tobytes(), what
    return exp


@pytest.mark.parametrize("source", [WINDOW, WIN, TIER, SPAN])
def test_every_source_both_sides_every_metric(mod, source):
    exp = check_source(mod.h, source, make_source(mod, source))
    assert len(exp) > 100 and (exp["in_edges"] > 0).any() and (exp["out_edges"] > 0).any()
    assert len(np.unique(exp["type"])) >= 3


def gnn_node_keys(h):
    keys = np.zeros(1 << 16, dtype=np.uint64)
    h2 = np.zeros((1 << 16, 64), dtype=np.float32)
    nv = C.c_size_t(0)
    h._ck(h.L.alz_gnn_nodes(h.h, keys.ctypes.data_as(C.c_void_p), h2.ctypes.data_as(C.c_void_p), len(keys),
                            C.byref(nv)), "alz_gnn_nodes")
    return keys[: nv.value]


@pytest.mark.parametrize("source", [WINDOW, SPAN])
def test_node_keys_equal_the_gnn_node_set(mod, source):
    h = mod.h
    rows = make_source(mod, source)
    if source == WINDOW:
        scores = np.zeros(len(rows), dtype=np.float32)
        n = C.c_size_t(0)
        rc = h.L.alz_gnn_score(h.h, scores.ctypes.data_as(C.c_void_p), len(scores), C.byref(n))
        if rc == abi.E_UNSUPPORTED:
            pytest.skip("built without the GNN pass")
        assert rc == 0
    else:
        h.gnn_score_rollup(source)
    got = h.node_rows(source)
    keys = (got["type"].astype(np.uint64) << np.uint64(32)) | got["value"].astype(np.uint64)
    assert keys.tobytes() == gnn_node_keys(h).tobytes() == nr.keys(rows).tobytes()


def edge_rows(n, rng, from_type=POD, to_type=SVC, cells_hi=1 << 8):
    r = np.zeros(n, dtype=abi.EDGE_OUT)
    r["from_type"], r["to_type"] = from_type, to_type
    r["count"] = rng.integers(0, 1 << 40, n, dtype=np.uint64)
    r["err5xx"] = rng.integers(0, 1 << 20, n, dtype=np.uint64)
    r["lat_sum_ns"] = rng.integers(0, 1 << 62, n, dtype=np.uint64)
    r["hist"] = rng.integers(0, cells_hi, (n, abi.NB), dtype=np.uint64).astype(np.uint32)
    return r


def check_hook(h, rows, what):
    exp = nr.group(rows)
    got = h.debug_node_rows(rows)
    if got.tobytes() != exp.tobytes():
        bad = np.flatnonzero((got.view(np.uint8).reshape(-1, 576) != exp.view(np.uint8).reshape(-1, 576)).any(1)) \
            if len(got) == len(exp) else []
        raise AssertionError((what, len(got), len(exp), bad[:5]))
    return exp


@pytest.fixture(scope="module")
def hh():
    h = capi.Handle(device=0, max_endpoints=1 << 10, max_pairs=1 << 12)
    yield h
    h.close()


def test_hub_of_2_20_callers(hh):
    rng = np.random.default_rng(71)
    n = 1 << 20
    rows = edge_rows(n, rng)
    rows["from"] = rng.permutation(n)   # 2^20 distinct pods, every one calling service 5
    rows["to"] = 5
    exp = check_hook(hh, rows, "hub")
    hub = exp[(exp["type"] == SVC) & (exp["value"] == 5)]
    assert len(exp) == n + 1 and hub["in_edges"][0] == n and hub["out_edges"][0] == 0


def test_run_lengths_across_tile_boundaries(hh):
    rng = np.random.default_rng(72)
    lengths = list(range(1, 4098, 7)) + [4097] + list(range(1, 130))
    lengths += [x for p in range(1, 17) for x in (2 ** p - 1, 2 ** p, 2 ** p + 1)]
    parts = []
    for j, L in enumerate(lengths):   # node (SVC, j) on L rows, from pods that repeat across runs
        r = edge_rows(L, rng)
        r["from"] = rng.integers(0, 5000, L)
        r["to"] = j
        parts.append(r)
    rows = np.concatenate(parts)
    rows = rows[rng.permutation(len(rows))]
    exp = check_hook(hh, rows, "runs")
    svc = exp[exp["type"] == SVC]
    assert list(svc["in_edges"]) == lengths
    for p in (17, 18, 19, 20):
        for L in (2 ** p - 1, 2 ** p, 2 ** p + 1):
            r = edge_rows(L, rng, cells_hi=4)
            r["from"] = rng.integers(0, 1 << 12, L)
            r["from_type"] = rng.integers(0, 2, L)
            r["to"] = 3
            check_hook(hh, r, ("run", L))


def test_wrapping_cells_across_a_tile_boundary(hh):
    rng = np.random.default_rng(73)
    for n in (31, 32, 33, 64, 100, 1000):
        r = edge_rows(n, rng)
        r["from"] = np.arange(n)
        r["to"] = 1
        r["hist"][:, 0] = 0xFFFFFFFF
        r["hist"][:, 63] = 0x80000001
        r["count"] = np.uint64((1 << 64) - 1)
        exp = check_hook(hh, r, ("wrap", n))
        s = exp[exp["type"] == SVC][0]
        assert s["in"]["hist"][0] == (n * 0xFFFFFFFF) % (1 << 32) and int(s["in"]["count"]) == ((1 << 64) - n) % (1 << 64)


def test_mixed_layouts_self_loops_and_empty(hh):
    rng = np.random.default_rng(74)
    assert len(hh.debug_node_rows(np.zeros(0, dtype=abi.EDGE_OUT))) == 0
    n = 50_000
    r = edge_rows(n, rng, cells_hi=1 << 32)
    r["from_type"] = rng.integers(0, 4, n)
    r["to_type"] = rng.integers(0, 4, n)
    r["from"] = rng.integers(0, 300, n)
    r["to"] = np.where(rng.random(n) < 0.1, r["from"], rng.integers(0, 300, n))
    r["to_type"] = np.where(r["to"] == r["from"], r["from_type"], r["to_type"])
    r["count"] = rng.integers(0, 1 << 64, n, dtype=np.uint64)
    exp = check_hook(hh, r, "mixed")
    assert int(exp["in_edges"].sum()) == n == int(exp["out_edges"].sum())
    # the same rows in another order give the same bytes
    assert hh.debug_node_rows(r[::-1]).tobytes() == exp.tobytes()


def test_errors_and_capacity():
    h = capi.Handle(device=0, max_endpoints=1 << 10, max_pairs=1 << 12)
    try:
        L, n = h.L, C.c_size_t(77)
        m1 = abi.metrics(abi.METRIC_COUNT)
        info = abi.TopInfo()
        # no rollup yet: STATE; no window yet: 0 nodes
        for s in (WIN, TIER, SPAN):
            assert L.alz_node_rows(h.h, s, None, 0, C.byref(n)) == abi.E_STATE and n.value == 0
            assert L.alz_node_metrics(h.h, s, IN, m1, 1, None, 0, C.byref(n)) == abi.E_STATE
            assert L.alz_node_top(h.h, s, IN, m1, 3, 0.0, None, None, None, 0, C.byref(n), C.byref(info)) == abi.E_STATE
        assert L.alz_node_rows(h.h, WINDOW, None, 0, C.byref(n)) == 0 and n.value == 0
        assert L.alz_node_top(h.h, WINDOW, OUT, m1, 3, 0.0, None, None, None, 0, C.byref(n), C.byref(info)) == 0
        assert n.value == 0 and (info.scored, info.above) == (0, 0)
        # a window of a few edges
        s = Stream(universe(n_edges=40, seed=5))
        try:
            hs = s.h
            rows = s.window(np.arange(40))
            exp = nr.group(rows)
            k = len(exp)
            Ls, hp = hs.L, hs.h
            m2 = abi.metrics(abi.METRIC_COUNT, (Q, 0.5))
            bad = [abi.metrics((9, 0.0)), abi.metrics((Q, 1.5)), abi.metrics((Q, float("nan")))]
            for src in (3, 7, 0xFFFFFFFE):
                assert Ls.alz_node_rows(hp, src, None, 0, C.byref(n)) == abi.E_INVAL and n.value == 0
                assert Ls.alz_node_metrics(hp, src, IN, m1, 1, None, 0, C.byref(n)) == abi.E_INVAL
            assert Ls.alz_node_metrics(hp, WINDOW, 2, m1, 1, None, 0, C.byref(n)) == abi.E_INVAL
            assert Ls.alz_node_top(hp, WINDOW, 2, m1, 3, 0.0, None, None, None, 0, C.byref(n), None) == abi.E_INVAL
            for nm in (0, 9):
                assert Ls.alz_node_metrics(hp, WINDOW, IN, abi.metrics(*([abi.METRIC_COUNT] * 9)), nm, None, 0,
                                           C.byref(n)) == abi.E_INVAL
            for m in bad:
                assert Ls.alz_node_metrics(hp, WINDOW, IN, m, 1, None, 0, C.byref(n)) == abi.E_INVAL
                assert Ls.alz_node_top(hp, WINDOW, IN, m, 3, 0.0, None, None, None, 0, C.byref(n), None) == abi.E_INVAL
            assert Ls.alz_node_top(hp, WINDOW, IN, m1, 0, 0.0, None, None, None, 0, C.byref(n), None) == abi.E_INVAL
            assert Ls.alz_node_top(hp, WINDOW, IN, m1, 3, float("nan"), None, None, None, 0, C.byref(n),
                                   None) == abi.E_INVAL
            # null required pointers
            assert Ls.alz_node_rows(hp, WINDOW, None, 5, C.byref(n)) == abi.E_INVAL
            assert Ls.alz_node_rows(hp, WINDOW, None, 0, None) == abi.E_INVAL
            assert Ls.alz_node_rows_device(hp, WINDOW, None, C.byref(n)) == abi.E_INVAL
            assert Ls.alz_node_metrics(hp, WINDOW, IN, None, 1, None, 0, C.byref(n)) == abi.E_INVAL
            assert Ls.alz_node_metrics(hp, WINDOW, IN, m1, 1, None, 5, C.byref(n)) == abi.E_INVAL
            assert Ls.alz_node_metrics_device(hp, WINDOW, IN, m1, 1, None, C.byref(n)) == abi.E_INVAL
            assert Ls.alz_node_rows(None, WINDOW, None, 0, C.byref(n)) == abi.E_INVAL
            assert Ls.alz_debug_node_rows(hp, None, 5, None, 0, C.byref(n)) == abi.E_INVAL
            # a cap below the nodes: ALZ_E_CAPACITY, *n_out set, nothing written
            out = np.frombuffer(b"\xab" * (576 * (k - 1)), dtype=abi.NODE_OUT).copy()
            keep = out.tobytes()
            rc = Ls.alz_node_rows(hp, WINDOW, out.ctypes.data_as(C.c_void_p), k - 1, C.byref(n))
            assert rc == abi.E_CAPACITY and n.value == k and out.tobytes() == keep
            vals = np.full((k - 1) * 2, 7.0)
            rc = Ls.alz_node_metrics(hp, WINDOW, OUT, m2, 2, vals.ctypes.data_as(C.c_void_p), k - 1, C.byref(n))
            assert rc == abi.E_CAPACITY and n.value == k and (vals == 7.0).all()
            tv, ti = np.full(2, 7.0), np.full(2, 9, dtype=np.uint32)
            tn = np.frombuffer(b"\xab" * (576 * 2), dtype=abi.NODE_OUT).copy()
            keep = tn.tobytes()
            rc = Ls.alz_node_top(hp, WINDOW, IN, m1, 5, -np.inf, tn.ctypes.data_as(C.c_void_p),
                                 tv.ctypes.data_as(C.c_void_p), ti.ctypes.data_as(C.c_void_p), 2, C.byref(n),
                                 C.byref(info))
            assert rc == abi.E_CAPACITY and n.value == min(5, k) and tn.tobytes() == keep
            assert (tv == 7.0).all() and (ti == 9).all() and (info.scored, info.above) == (k, k)
            # the exact cap works
            assert hs.node_rows(WINDOW).tobytes() == exp.tobytes()
        finally:
            s.close()
    finally:
        h.close()


def test_reads_only():
    m = Modelled(universe(seed=35), history=(5, 1 << 15), tiers=[(2, 3, 1 << 15, 1 << 13)])
    try:
        m.random_windows(8, seed=351, lo=0.2, hi=0.6)
        h = m.h
        h.rollup(3)
        h.baseline_pin(WIN)
        m.random_windows(2, seed=352)
        h.rollup_tier(1, 2)
        h.rollup_span(5)
        span_rows = h.rollup_span(5)[0]
        h.rollup(2)
        specs = [abi.METRIC_COUNT, (Q, 0.99), abi.METRIC_ERR_RATE]
        T = capi.Handle.trend

        def gnn_nodes():
            keys = np.zeros(1 << 16, dtype=np.uint64)
            emb = np.zeros((1 << 16, 64), dtype=np.float32)
            nv = C.c_size_t(0)
            h._ck(h.L.alz_gnn_nodes(h.h, keys.ctypes.data_as(C.c_void_p), emb.ctypes.data_as(C.c_void_p), len(keys),
                                    C.byref(nv)), "alz_gnn_nodes")
            return np.concatenate([keys[: nv.value].view(np.uint8), emb[: nv.value].view(np.uint8).ravel()])

        held = {kind: h.gnn_score_rollup(kind) for kind in (WIN, TIER, SPAN)}
        sv, spp, sn, sp_, _, _ = h.edge_series_device(WIN, 0, 4, *specs)
        mv, mn = h.edge_metrics_rollup_device(TIER, *specs)
        tr_, tv, ti, tn, _ = h.edge_top_rollup_device(SPAN, (Q, 0.99), 9)
        cv, cn, _ = h.edge_changes_device((Q, 0.99), abi.CHANGE_RATIO)
        trd, trn, trp, _, _ = h.edge_trends_device(SPAN, 0, 4, (Q, 0.99), T(abi.TREND_SLOPE, recent=1))
        gv, gn = h.gnn_score_rollup_device(WIN)

        def snapshot():
            return dict(series=h.d2h(sv, sn * sp_ * len(specs), np.float64), series_p=h.d2h(spp, sn * sp_, np.uint8),
                        metrics=h.d2h(mv, mn * len(specs), np.float64), top=h.d2h(tv, tn, np.float64),
                        top_i=h.d2h(ti, tn, np.uint32), top_r=h.d2h(tr_, tn, abi.EDGE_OUT),
                        changes=h.d2h(cv, cn, abi.EDGE_CHANGE), trends=h.d2h(trd, trn, abi.EDGE_TREND),
                        gnn=h.d2h(gv, gn, np.float32), nodes=gnn_nodes(),
                        stats={k: v for k, v in h.stats().items() if k != "kernel_launches"})

        before = snapshot()
        for src in (WINDOW, WIN, TIER, SPAN):
            h.node_rows(src)
            h.node_rows_device(src)
            for side in (IN, OUT):
                h.node_metrics(src, side, *specs)
                h.node_metrics_device(src, side, (Q, 0.5))
                h.node_top(src, side, (Q, 0.99), 7)
                h.node_top_device(src, side, abi.METRIC_COUNT, 3)
        h.debug_node_rows(span_rows)
        after = snapshot()
        assert before.pop("stats") == after.pop("stats")
        for k in before:
            assert np.asarray(before[k]).tobytes() == np.asarray(after[k]).tobytes(), k
        # the rollups' rows are still there and score as before
        for kind in (WIN, TIER, SPAN):
            assert h.gnn_score_rollup(kind).tobytes() == held[kind].tobytes(), kind
        assert h.rollup_span(5)[0].tobytes() == span_rows.tobytes()
        assert h.node_rows(SPAN).tobytes() == nr.group(span_rows).tobytes()
    finally:
        m.close()
