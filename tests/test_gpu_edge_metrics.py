"""GPU: the edge metrics (alz_edge_metrics*, alz_debug_edge_metrics_rows, docs/SPEC.md §17).

The expected values are tests/metric_ref.py over the same rows, bit for bit; quantiles also equal alz_edge_quantiles
row by row. The debug hook runs the kernel over constructed rows the ingest path cannot make: cells of 2^32 - 1,
count = 0 with a non-empty histogram, latency sums near 2^64."""
import ctypes as C

import numpy as np
import pytest

import metric_ref as mr
from alaz_b200 import abi, capi
from test_gnn_quantiles import BIG, QS, _hists
from test_gpu_gnn_rollup import Stream, nodes, universe

pytestmark = pytest.mark.gpu
WIN, TIER, SPAN = abi.ROLLUP_WINDOWS, abi.ROLLUP_TIER, abi.ROLLUP_SPAN
Q = abi.METRIC_QUANTILE
ALL = [abi.METRIC_COUNT, abi.METRIC_ERR5XX, abi.METRIC_ERR_RATE, abi.METRIC_MEAN_NS, (Q, 0.5), (Q, 0.99), (Q, 0.0),
       (Q, 1.0)]


@pytest.fixture(scope="module")
def hh():
    h = capi.Handle(max_endpoints=64, max_pairs=1 << 12)
    yield h
    h.close()


def hook(h, rows, specs, cap=None):
    """alz_debug_edge_metrics_rows over `rows` copied to the device: (status, values [cap x nm], n_out)."""
    rows = np.ascontiguousarray(rows, dtype=abi.EDGE_OUT)
    d = h.dev_alloc(max(rows.nbytes, 8))
    try:
        h.h2d(d, rows)
        cap = len(rows) if cap is None else cap
        out = np.full((max(cap, 1), max(len(specs), 1)), 7.5)
        n = C.c_size_t(12345)
        rc = h.L.alz_debug_edge_metrics_rows(h.h, C.c_void_p(d), len(rows), abi.metrics(*specs), len(specs),
                                             out.ctypes.data_as(C.c_void_p), cap, C.byref(n))
    finally:
        h.dev_free(d)
    return rc, out, n.value


def constructed_rows():
    """The adversarial histograms of test_gnn_quantiles.py, with counts, 5xx and latency sums at their extremes."""
    hs = _hists()
    rng = np.random.default_rng(17)
    rows = np.zeros(len(hs), dtype=abi.EDGE_OUT)
    rows["hist"] = hs
    rows["count"] = hs.astype(np.uint64).sum(axis=1)
    rows["count"][::7] = 0                                                   # count = 0, histogram non-empty
    rows["count"][3::11] = np.uint64((1 << 64) - 1)
    rows["err5xx"] = rng.integers(0, 1 << 40, len(rows), dtype=np.uint64)
    rows["err5xx"][5::13] = np.uint64((1 << 64) - 1)
    rows["lat_sum_ns"] = rng.integers(0, 1 << 63, len(rows), dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    rows["lat_sum_ns"][1::9] = np.uint64((1 << 64) - 1)
    rows["lat_sum_ns"][2::9] = np.uint64((1 << 64) - 2048)
    return rows


def host_quantile(row, q):
    out, qa = np.zeros(1), np.array([q])
    assert capi.load().alz_edge_quantiles(row.ctypes.data_as(C.c_void_p), qa.ctypes.data_as(C.c_void_p), 1,
                                          out.ctypes.data_as(C.c_void_p)) == 0
    return out[0]


def test_hook_constructed_rows_bitwise(hh):
    rows = constructed_rows()
    for specs in (ALL, [(Q, q) for q in QS], [abi.METRIC_MEAN_NS, abi.METRIC_ERR_RATE], [(Q, 1e-300)],
                  [abi.METRIC_COUNT]):
        rc, got, n = hook(hh, rows, specs)
        assert rc == 0 and n == len(rows), (rc, n)
        want = mr.matrix(rows, specs)
        assert got[:n].tobytes() == want.tobytes(), (specs, np.argwhere(got[:n] != want)[:5])
    rc, got, n = hook(hh, rows, [(Q, q) for q in QS])
    for i in range(len(rows)):
        for j, q in enumerate(QS):
            assert got[i, j].tobytes() == np.float64(host_quantile(rows[i:i + 1], q)).tobytes(), (i, q)


def test_hook_bucket_ends_and_small_q(hh):
    """Targets exactly on a bucket's end and q = 1e-300: the cases a fused multiply-add rounds differently."""
    rows = np.zeros(64 * 3, dtype=abi.EDGE_OUT)
    for b in range(64):
        rows["hist"][3 * b, b] = 2
        rows["hist"][3 * b, (b + 5) % 64] = 2
        rows["hist"][3 * b + 1, b] = 99
        rows["hist"][3 * b + 1, (b + 1) % 64] = 1
        rows["hist"][3 * b + 2, b] = BIG
        rows["hist"][3 * b + 2, 63 - b] = 3
    specs = [(Q, 0.5), (Q, 0.99), (Q, 1e-300), (Q, 0.0), (Q, 1.0), (Q, 0.3), (Q, 0.7), (Q, 0.999)]
    rc, got, n = hook(hh, rows, specs)
    assert rc == 0 and n == len(rows)
    assert got[:n].tobytes() == mr.matrix(rows, specs).tobytes()


def test_hook_random_histograms_every_shape(hh):
    rng = np.random.default_rng(5)
    for n in (1, 31, 32, 33, 1000, 70_001):
        rows = np.zeros(n, dtype=abi.EDGE_OUT)
        rows["hist"] = np.where(rng.random((n, 64)) < rng.uniform(0.02, 0.5), rng.integers(0, 1 << 32, (n, 64)),
                                0).astype(np.uint32)
        rows["count"] = rng.integers(0, 1 << 40, n, dtype=np.uint64)
        rows["err5xx"] = rng.integers(0, 1 << 30, n, dtype=np.uint64)
        rows["lat_sum_ns"] = rng.integers(0, 1 << 63, n, dtype=np.uint64)
        specs = [(Q, float(rng.random())), abi.METRIC_ERR_RATE, (Q, 0.99), abi.METRIC_MEAN_NS]
        rc, got, nn = hook(hh, rows, specs)
        assert rc == 0 and nn == n
        assert got[:n].tobytes() == mr.matrix(rows, specs).tobytes(), n


def test_hook_rules(hh):
    rows = constructed_rows()[:50]
    rc, got, n = hook(hh, rows, ALL, cap=49)                                 # cap counts rows
    assert rc == abi.E_CAPACITY and n == 50 and np.all(got == 7.5)
    rc, _, n = hook(hh, rows[:0], ALL)
    assert rc == 0 and n == 0
    assert hook(hh, rows, [])[0] == abi.E_INVAL
    assert hook(hh, rows, [abi.METRIC_COUNT] * 9)[0] == abi.E_INVAL
    assert hook(hh, rows, [abi.METRIC_COUNT] * 8)[0] == 0
    for bad in ([5], [(Q, -0.1)], [(Q, 1.5)], [(Q, float("nan"))], [abi.METRIC_COUNT, (Q, float("inf"))]):
        assert hook(hh, rows, bad)[0] == abi.E_INVAL, bad
    assert hook(hh, rows, [(abi.METRIC_COUNT, float("nan"))])[0] == 0     # q is ignored for the other kinds


# ---- real sources -------------------------------------------------------------------------------------------------

def test_window_and_rollup_sources():
    s = Stream(universe(seed=21), history=(4, 1 << 15), tiers=[(2, 4, 1 << 15, 1 << 13)])
    s.random_windows(6, seed=211, lo=0.2, hi=0.6)
    last = s.window(np.arange(200, 2800))
    h = s.h
    got = h.edge_metrics(*ALL)
    assert got.tobytes() == mr.matrix(last, ALL).tobytes()
    p, n = h.edge_metrics_device(*ALL)
    h.sync()
    assert n == len(last) and h.d2h(p, n * len(ALL), np.float64).tobytes() == got.tobytes()
    for kind, roll in ((WIN, lambda: h.rollup(3)[0]), (WIN, lambda: h.rollup(1)[0]),
                       (TIER, lambda: h.rollup_tier(1, 2)[0]), (SPAN, lambda: h.rollup_span(6, abi.SPAN_AT_LEAST)[0])):
        rows = roll()
        assert len(rows) > 0
        for specs in (ALL, [abi.METRIC_COUNT, abi.METRIC_ERR5XX], [(Q, 0.95)]):
            got = h.edge_metrics_rollup(kind, *specs)
            assert got.tobytes() == mr.matrix(rows, specs).tobytes(), (kind, specs)
            p, n = h.edge_metrics_rollup_device(kind, *specs)
            h.sync()
            assert n == len(rows) and h.d2h(p, n * len(specs), np.float64).tobytes() == got.tobytes()
    s.close()


def raw_metrics(h, kind, specs, cap, values=True, m_ptr=True):
    """alz_edge_metrics (kind None) or alz_edge_metrics_rollup with a sentinel buffer: (status, values, n_out)."""
    out = np.full((max(cap, 1), max(len(specs), 1)), 7.5)
    n = C.c_size_t(12345)
    m = abi.metrics(*specs) if m_ptr else None
    v = out.ctypes.data_as(C.c_void_p) if values else None
    if kind is None:
        rc = h.L.alz_edge_metrics(h.h, m, len(specs), v, cap, C.byref(n))
    else:
        rc = h.L.alz_edge_metrics_rollup(h.h, int(kind), m, len(specs), v, cap, C.byref(n))
    return rc, out, n.value


def test_errors_capacity_and_states():
    s = Stream(universe(seed=22, n_edges=800), history=(3, 1 << 14))
    h = s.h
    rc, _, n = raw_metrics(h, None, ALL, 0)                                  # no window yet: 0 rows
    assert rc == 0 and n == 0
    for kind in (WIN, TIER, SPAN):
        rc, _, n = raw_metrics(h, kind, ALL, 5)
        assert rc == abi.E_STATE and n == 0, kind
    rows = s.window(np.arange(0, 600))
    assert raw_metrics(h, 3, ALL, 5)[0] == abi.E_INVAL
    assert raw_metrics(h, 0xFFFFFFFF, ALL, 5)[0] == abi.E_INVAL
    assert raw_metrics(h, None, [], 5)[0] == abi.E_INVAL
    assert raw_metrics(h, None, ALL + [abi.METRIC_COUNT], len(rows))[0] == abi.E_INVAL
    assert raw_metrics(h, None, [(Q, 2.0)], len(rows))[0] == abi.E_INVAL
    assert raw_metrics(h, None, [7], len(rows))[0] == abi.E_INVAL
    assert raw_metrics(h, None, ALL, len(rows), m_ptr=False)[0] == abi.E_INVAL
    assert raw_metrics(h, None, ALL, 5, values=False)[0] == abi.E_INVAL
    rc, out, n = raw_metrics(h, None, ALL, len(rows) - 1)
    assert rc == abi.E_CAPACITY and n == len(rows) and np.all(out == 7.5)
    rc, _, n = raw_metrics(h, None, ALL, 0, values=False)
    assert rc == abi.E_CAPACITY and n == len(rows)
    rc, out, n = raw_metrics(h, None, ALL, len(rows))
    assert rc == 0 and out[:n].tobytes() == mr.matrix(rows, ALL).tobytes()
    p, nn = C.c_void_p(), C.c_size_t(9)
    assert h.L.alz_edge_metrics_device(h.h, abi.metrics(*ALL), 0, C.byref(p), C.byref(nn)) == abi.E_INVAL
    assert nn.value == 0
    assert h.L.alz_edge_metrics_device(h.h, abi.metrics(*ALL), 1, None, C.byref(nn)) == abi.E_INVAL
    h.rollup(2)
    assert raw_metrics(h, WIN, ALL, 10_000)[0] == 0
    rc = h.L.alz_window_rollup(h.h, 0, None, 0, C.byref(nn), None)          # k = 0: leaves nothing to read
    assert rc == abi.E_INVAL
    assert raw_metrics(h, WIN, ALL, 10_000)[0] == abi.E_STATE
    s.close()


def test_zero_row_sources():
    s = Stream(universe(seed=23, n_edges=300), history=(3, 1 << 14))
    s.window(np.array([], np.int64))
    rows, _ = s.h.rollup(1)
    assert len(rows) == 0
    assert s.h.edge_metrics_rollup(WIN, *ALL).shape == (0, len(ALL))
    assert s.h.edge_metrics(*ALL).shape == (0, len(ALL))
    s.close()


def gnn_scores(h, n):
    scores = np.zeros(max(n, 1), np.float32)
    nn = C.c_size_t(0)
    h._ck(h.L.alz_gnn_score(h.h, scores.ctypes.data_as(C.c_void_p), len(scores), C.byref(nn)), "alz_gnn_score")
    return scores[: nn.value]


def test_reads_only_gnn_state_unchanged():
    """A metric or metric-top call runs no GNN pass: the GNN's device scores, top results and alz_gnn_nodes are the
    same bytes before and after it, and the source rows stay scorable."""
    s = Stream(universe(seed=24), history=(4, 1 << 15))
    s.random_windows(3, seed=241)
    h = s.h
    last = s.window(np.arange(100, 2500))
    n = len(last)
    dev = C.c_void_p()
    nn = C.c_size_t(0)
    h._ck(h.L.alz_gnn_score_device(h.h, C.byref(dev), C.byref(nn)), "alz_gnn_score_device")
    h.sync()
    before_scores = h.d2h(dev.value, n, np.float32)
    pr, pv, pi, m, _ = h.gnn_top_device(50, 0.0)
    h.sync()
    before_top = [h.d2h(pr, m, abi.EDGE_OUT), h.d2h(pv, m, np.float32), h.d2h(pi, m, np.uint32)]
    keys, h2 = nodes(h, n)
    h.edge_metrics(*ALL)
    h.edge_top((Q, 0.99), 100)
    h.rollup(2)
    h.edge_metrics_rollup(WIN, *ALL)
    h.edge_top_rollup(WIN, abi.METRIC_ERR5XX, 100)
    h.sync()
    assert h.d2h(dev.value, n, np.float32).tobytes() == before_scores.tobytes()
    after_top = [h.d2h(pr, m, abi.EDGE_OUT), h.d2h(pv, m, np.float32), h.d2h(pi, m, np.uint32)]
    assert all(a.tobytes() == b.tobytes() for a, b in zip(before_top, after_top))
    k2, h22 = nodes(h, n)
    assert k2.tobytes() == keys.tobytes() and h22.tobytes() == h2.tobytes()
    assert gnn_scores(h, n).tobytes() == before_scores.tobytes()            # the window is still scorable
    assert len(h.gnn_score_rollup(WIN)) > 0                                  # so is the rollup
    s.close()


def test_metric_calls_allocate_no_gnn_state():
    """On a fresh handle, metric calls work without ever creating the GNN state: alz_gnn_nodes still says none."""
    s = Stream(universe(seed=25, n_edges=500), history=(2, 1 << 14))
    rows = s.window(np.arange(0, 400))
    assert s.h.edge_metrics(abi.METRIC_COUNT).shape == (len(rows), 1)
    s.h.edge_top(abi.METRIC_COUNT, 10)
    n = C.c_size_t(0)
    assert s.h.L.alz_gnn_nodes(s.h.h, None, None, 0, C.byref(n)) == abi.E_STATE
    s.close()
