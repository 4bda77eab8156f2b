"""GPU: edge changes against a pinned baseline (alz_baseline_pin, alz_edge_changes*, alz_edge_changes_top*,
alz_debug_edge_changes_rows, docs/SPEC.md §18).

The expected lists and top results are tests/change_ref.py over the same rows, compared as bytes: key fields,
indices, presence and the bits of value, base value and change. Windows and rollups come from the Stream of
tests/test_gpu_gnn_rollup.py; the hook runs the join over constructed layouts."""
import ctypes as C
import itertools

import numpy as np
import pytest

import change_ref as cr
from alaz_b200 import abi, capi
from test_gpu_edge_metrics import constructed_rows
from test_gpu_gnn_rollup import Stream, universe

pytestmark = pytest.mark.gpu
WINDOW, WIN, TIER, SPAN = abi.SOURCE_WINDOW, abi.ROLLUP_WINDOWS, abi.ROLLUP_TIER, abi.ROLLUP_SPAN
Q = abi.METRIC_QUANTILE
SPECS = [abi.METRIC_COUNT, abi.METRIC_ERR5XX, abi.METRIC_ERR_RATE, abi.METRIC_MEAN_NS, (Q, 0.5), (Q, 0.99), (Q, 1.0)]
MODES = [abi.CHANGE_DELTA, abi.CHANGE_DROP, abi.CHANGE_RATIO]
MASKS = list(range(1, 8))
INFO_KEYS = ("windows", "clocked", "window_first", "window_last", "epoch_first", "epoch_last", "rows_in")


def same(got, want, what):
    got_l, got_i = got
    want_l, want_i = want
    assert got_i == want_i, (what, got_i, want_i)
    assert got_l.tobytes() == want_l.tobytes(), (what, len(got_l), len(want_l),
                                                 np.flatnonzero(got_l != want_l)[:5] if len(got_l) == len(want_l)
                                                 else None)


def rollup_info(info):
    return {k: info[k] for k in INFO_KEYS}


class Sources:
    """The rows and windows of each source kind, as the last call of that kind returned them."""

    def __init__(self, s):
        self.s, self.rows, self.windows, self.info = s, {}, {}, {}

    def make(self, kind, param):
        h = self.s.h
        if kind == WINDOW:
            rng = np.random.default_rng(param)
            rows = self.s.window(np.flatnonzero(rng.random(self.s.g.n_edges) < rng.uniform(0.2, 0.7)))
            info = dict(windows=1)
        elif kind == WIN:
            rows, info = h.rollup(param)
        elif kind == TIER:
            rows, info = h.rollup_tier(1, param)
        else:
            rows, info = h.rollup_span(param)
        self.rows[kind], self.windows[kind], self.info[kind] = rows, info["windows"], info
        return rows, info


def check_all(h, src_rows, src_w, base_rows, base_w, source, what, masks=MASKS, top_masks=(7, 5)):
    for spec, mode in itertools.product(SPECS, MODES):
        for mask in masks:
            got = h.edge_changes(spec, mode, mask, source=source)
            want = cr.changes(src_rows, base_rows, spec, mode, mask, src_w, base_w)
            same(got, want, (what, spec, mode, mask))
        for mask, k, mn in itertools.product(top_masks, (1, 50), (0.0, -np.inf)):
            got = h.edge_changes_top(spec, k, mn, mode, mask, source=source)
            want = cr.top(src_rows, base_rows, spec, mode, mask, k, mn, src_w, base_w)
            same(got, want, (what, "top", spec, mode, mask, k, mn))


@pytest.fixture(scope="module")
def stream():
    s = Stream(universe(seed=4), history=(6, 1 << 15), tiers=[(2, 4, 1 << 15, 1 << 13)])
    s.random_windows(9, seed=41, lo=0.2, hi=0.6)
    yield s
    s.close()


@pytest.mark.parametrize("base_kind", [WINDOW, WIN, TIER, SPAN])
def test_every_source_against_every_baseline_kind(stream, base_kind):
    src = Sources(stream)
    h = stream.h
    base_rows, base_info = src.make(base_kind, {WINDOW: 1, WIN: 4, TIER: 2, SPAN: 6}[base_kind])
    pinned = h.baseline_pin(base_kind)
    if base_kind == WINDOW:   # what a k = 1 window rollup reports for that window
        assert pinned == rollup_info(h.rollup(1)[1])
        assert pinned["windows"] == 1 and pinned["rows_in"] == len(base_rows)
    else:
        assert pinned == rollup_info(base_info)
    stream.random_windows(2, seed=42 + base_kind % 7, lo=0.2, hi=0.6)   # the baseline survives flushes
    for kind, param in ((WINDOW, 5), (WIN, 3), (TIER, 1), (SPAN, 3)):
        rows, _ = src.make(kind, param)
        check_all(h, rows, src.windows[kind], base_rows, pinned["windows"], kind, (base_kind, kind))


def test_window_info_is_a_k1_rollup_after_every_flush(stream):
    h = stream.h
    for seed in range(3):
        stream.random_windows(1, seed=100 + seed)
        assert h.baseline_pin(WINDOW) == rollup_info(h.rollup(1)[1])


def test_device_variants_equal_host(stream):
    h = stream.h
    h.baseline_pin(WINDOW)
    stream.random_windows(1, seed=7)
    for spec in (abi.METRIC_COUNT, (Q, 0.99)):
        lst, info = h.edge_changes(spec, abi.CHANGE_RATIO, 7)
        p, n, dinfo = h.edge_changes_device(spec, abi.CHANGE_RATIO, 7)
        assert n == len(lst) and dinfo == info
        assert h.d2h(p, n, abi.EDGE_CHANGE).tobytes() == lst.tobytes()
        top, tinfo = h.edge_changes_top(spec, 20, 0.0, abi.CHANGE_RATIO, 7)
        p, n, dinfo = h.edge_changes_top_device(spec, 20, 0.0, abi.CHANGE_RATIO, 7)
        assert n == len(top) and dinfo == tinfo
        assert h.d2h(p, n, abi.EDGE_CHANGE).tobytes() == top.tobytes()


def test_reads_only(stream):
    h = stream.h
    stream.random_windows(2, seed=55)
    h.rollup(3)
    h.baseline_pin(WIN)
    stream.random_windows(1, seed=56)
    rows_w, _ = h.rollup(2)
    span_rows, _ = h.rollup_span(4)
    before = dict(metrics_w=h.edge_metrics(*SPECS), metrics_r=h.edge_metrics_rollup(WIN, *SPECS),
                  gnn=h.gnn_score_rollup(SPAN), gnn_w=h.gnn_top(5)[1], top_m=h.edge_top(abi.METRIC_COUNT, 5)[0])
    pm, nm = h.edge_metrics_device(abi.METRIC_COUNT)
    dev_m = h.d2h(pm, nm, np.float64)
    for source in (WINDOW, WIN, SPAN):
        for spec in SPECS:
            h.edge_changes(spec, abi.CHANGE_DELTA, 7, source=source)
            h.edge_changes_top(spec, 9, 0.0, abi.CHANGE_DROP, 7, source=source)
    assert h.d2h(pm, nm, np.float64).tobytes() == dev_m.tobytes()      # metric device results untouched
    assert h.rollup_span(4)[0].tobytes() == span_rows.tobytes()
    after = dict(metrics_w=h.edge_metrics(*SPECS), metrics_r=h.edge_metrics_rollup(WIN, *SPECS),
                 gnn=h.gnn_score_rollup(SPAN), gnn_w=h.gnn_top(5)[1], top_m=h.edge_top(abi.METRIC_COUNT, 5)[0])
    for k in before:
        assert before[k].tobytes() == after[k].tobytes(), k
    assert h.rollup(2)[0].tobytes() == rows_w.tobytes()


def test_baseline_survives_reconfiguration_and_goes_with_clear():
    s = Stream(universe(seed=5), history=(4, 1 << 15), tiers=[(2, 3, 1 << 15, 1 << 13)])
    h = s.h
    s.random_windows(5, seed=61)
    base, info = h.rollup(3)
    assert h.baseline_pin(WIN) == rollup_info(info)
    h.window_history(5, 1 << 15)                                    # other values: the window rollup rows go
    h.window_history_tiers([(3, 2, 1 << 15, 1 << 13)])
    s.random_windows(4, seed=62)
    h.rollup(2)
    h.rollup_tier(1, 1)
    h.rollup_span(3)
    h.gnn_score_rollup(WIN)
    h.edge_top(abi.METRIC_COUNT, 5)
    rows = s.window(np.arange(0, 500))
    same(h.edge_changes(abi.METRIC_COUNT, abi.CHANGE_DELTA, 7), cr.changes(rows, base, abi.METRIC_COUNT,
                                                                           abi.CHANGE_DELTA, 7, 1, 3), "reconfigured")
    # a re-pin replaces it
    span, sinfo = h.rollup_span(2)
    assert h.baseline_pin(SPAN) == rollup_info(sinfo)
    same(h.edge_changes((Q, 0.99), abi.CHANGE_RATIO, 7), cr.changes(rows, span, (Q, 0.99), abi.CHANGE_RATIO, 7, 1,
                                                                    sinfo["windows"]), "re-pinned")
    h.baseline_clear()
    with pytest.raises(capi.AlzError) as e:
        h.edge_changes(abi.METRIC_COUNT)
    assert e.value.status == abi.E_STATE
    s.close()


def raw(h, fn, *args):
    """(status, n_out) of fn with a null output."""
    n = C.c_size_t(777)
    info = abi.ChangeInfo()
    rc = getattr(h.L, fn)(h.h, *args, C.byref(n), C.byref(info))
    return rc, n.value


def test_every_error_code():
    s = Stream(universe(seed=6, n_edges=400), history=(3, 1 << 14))
    h = s.h
    m = abi.metrics(abi.METRIC_COUNT)
    bad_q = abi.metrics((Q, 1.5))
    bad_kind = (abi.Metric * 1)(abi.Metric(9, 0, 0.0))
    fn = "alz_edge_changes"
    # no baseline
    assert raw(h, fn, WINDOW, m, 0, 7, None, 0)[0] == abi.E_STATE
    assert raw(h, "alz_edge_changes_top", WINDOW, m, 0, 7, 5, 0.0, None, 0)[0] == abi.E_STATE
    # no rollup rows to pin or compare
    assert h.L.alz_baseline_pin(h.h, WIN, None) == abi.E_STATE
    assert h.L.alz_baseline_pin(h.h, 7, None) == abi.E_INVAL
    s.random_windows(2, seed=1)
    assert h.L.alz_baseline_pin(h.h, WINDOW, None) == 0
    assert raw(h, fn, WIN, m, 0, 7, None, 0)[0] == abi.E_STATE
    assert raw(h, fn, TIER, m, 0, 7, None, 0)[0] == abi.E_STATE
    # invalid arguments
    assert raw(h, fn, 3, m, 0, 7, None, 0)[0] == abi.E_INVAL                    # unknown source
    assert raw(h, fn, WINDOW, bad_kind, 0, 7, None, 0)[0] == abi.E_INVAL
    assert raw(h, fn, WINDOW, bad_q, 0, 7, None, 0)[0] == abi.E_INVAL
    assert raw(h, fn, WINDOW, None, 0, 7, None, 0)[0] == abi.E_INVAL
    assert raw(h, fn, WINDOW, m, 3, 7, None, 0)[0] == abi.E_INVAL                # unknown mode
    assert raw(h, fn, WINDOW, m, 0, 0, None, 0)[0] == abi.E_INVAL                # presence 0
    assert raw(h, fn, WINDOW, m, 0, 8, None, 0)[0] == abi.E_INVAL                # presence above 7
    assert raw(h, fn, WINDOW, m, 0, 7, None, 5)[0] == abi.E_INVAL                # null out with cap
    assert raw(h, "alz_edge_changes_top", WINDOW, m, 0, 7, 0, 0.0, None, 0)[0] == abi.E_INVAL          # k = 0
    assert raw(h, "alz_edge_changes_top", WINDOW, m, 0, 7, 5, float("nan"), None, 0)[0] == abi.E_INVAL
    assert h.L.alz_edge_changes_device(h.h, WINDOW, m, 0, 7, None, None, None) == abi.E_INVAL
    assert h.L.alz_edge_changes(None, WINDOW, m, 0, 7, None, 0, None, None) == abi.E_INVAL
    # capacity: *n_out set, nothing written
    rc, n = raw(h, fn, WINDOW, m, 0, 7, None, 0)
    assert rc == abi.E_CAPACITY and n > 0
    out = np.zeros(n - 1, abi.EDGE_CHANGE)
    out.view(np.uint8)[:] = 0xAB
    nn, info = C.c_size_t(0), abi.ChangeInfo()
    assert h.L.alz_edge_changes(h.h, WINDOW, m, 0, 7, out.ctypes.data_as(C.c_void_p), n - 1, C.byref(nn),
                                C.byref(info)) == abi.E_CAPACITY
    assert nn.value == n and np.all(out.view(np.uint8) == 0xAB)
    rc, n = raw(h, "alz_edge_changes_top", WINDOW, m, 0, 7, 3, 0.0, None, 0)
    assert rc == abi.E_CAPACITY and n == 3
    # the hook: windows 0, null rows
    assert raw(h, "alz_debug_edge_changes_rows", None, 0, 0, None, 0, 1, m, 0, 7, None, 0)[0] == abi.E_INVAL
    assert raw(h, "alz_debug_edge_changes_rows", None, 5, 1, None, 0, 1, m, 0, 7, None, 0)[0] == abi.E_INVAL
    assert raw(h, "alz_debug_edge_changes_rows", None, 0, 1, None, 0, 1, m, 0, 7, None, 0)[0] == 0
    # an empty source and an empty baseline are valid
    s.window(np.zeros(0, dtype=np.int64))
    lst, info = h.edge_changes(abi.METRIC_COUNT)
    assert info["source_rows"] == 0 and info["gone"] == info["base_rows"] == len(lst)
    assert h.baseline_pin(WINDOW)["rows_in"] == 0
    s.random_windows(1, seed=3)
    lst, info = h.edge_changes(abi.METRIC_COUNT)
    assert info["base_rows"] == 0 and info["added"] == info["source_rows"] == len(lst)
    s.close()


# ---- constructed layouts through the hook -------------------------------------------------------------------------

def keyed_rows(keys, seed):
    """EDGE_OUT rows pod (key >> 32) -> service (key & 0xFFFFFFFF) in ascending key order, with the extreme
    histograms and sums of test_gpu_edge_metrics.constructed_rows."""
    keys = np.sort(np.asarray(keys, dtype=np.uint64))
    pool = constructed_rows()
    rng = np.random.default_rng(seed)
    r = pool[rng.integers(0, len(pool), len(keys))].copy() if len(keys) else np.zeros(0, abi.EDGE_OUT)
    r["from_type"] = abi.NODE_POD
    r["to_type"] = abi.NODE_SVC
    r["from"] = (keys >> np.uint64(32)).astype(np.uint32)
    r["to"] = (keys & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    k = cr.row_keys(r)
    assert np.all(k[1:] > k[:-1])
    return r


def hook_check(h, a, b, what, specs=SPECS, wa=1, wb=1):
    for spec, mode in itertools.product(specs, MODES):
        for mask in MASKS:
            got = h.debug_edge_changes_rows(a, b, spec, mode, mask, wa, wb)
            same(got, cr.changes(a, b, spec, mode, mask, wa, wb), (what, spec, mode, mask))


@pytest.fixture(scope="module")
def hh():
    h = capi.Handle(max_endpoints=64, max_pairs=1 << 12)
    yield h
    h.close()


def layouts():
    k = lambda *xs: np.array(xs, dtype=np.uint64)
    r = np.arange(1, 600, dtype=np.uint64) * np.uint64(7919)
    yield "both empty", k(), k()
    yield "source empty", k(), r[:100]
    yield "baseline empty", r[:100], k()
    yield "identical", r[:300], r[:300]
    yield "disjoint ranges", r[:200], r[300:500]
    yield "disjoint reversed", r[300:500], r[:200]
    yield "interleaved", r[0::2], r[1::2]
    yield "one shared key first", np.concatenate([r[:1], r[1::2]]), np.concatenate([r[:1], r[2::2]])
    yield "one shared key last", np.concatenate([r[1:-1:2], r[-1:]]), np.concatenate([r[2:-1:2], r[-1:]])
    yield "high keys", k(1 << 60, (1 << 60) + 1, 0x1FFFFFFF_FFFFFFFF), k(0x1FFFFFFF_FFFFFFFF, 5)


@pytest.mark.parametrize("case", list(range(10)))
def test_hook_layouts(hh, case):
    name, ka, kb = list(layouts())[case]
    hook_check(hh, keyed_rows(ka, 1), keyed_rows(kb, 2), name)


@pytest.mark.parametrize("n", [1, 255, 256, 257, 4095, 4096, 4097])
def test_hook_sizes_around_tiles(hh, n):
    rng = np.random.default_rng(n)
    keys = rng.choice(1 << 40, size=2 * n, replace=False).astype(np.uint64)
    both = keys[: n // 2]
    a = np.concatenate([both, keys[n // 2: n]])
    b = np.concatenate([both, keys[n: n + n // 3 + 1]])
    hook_check(hh, keyed_rows(a, 3), keyed_rows(b, 4), f"n={n}", specs=[abi.METRIC_COUNT, (Q, 0.99)], wa=5, wb=60)


def test_hook_large(hh):
    n = (1 << 20) + 3
    rng = np.random.default_rng(9)
    keys = np.unique(rng.integers(0, 1 << 44, int(n * 1.6), dtype=np.uint64))
    rng.shuffle(keys)
    a = np.sort(keys[:n])
    b = np.sort(np.concatenate([keys[: n // 2], keys[n: n + n // 2]]))
    ra, rb = keyed_rows(a, 5), keyed_rows(b, 6)
    for spec, mode, mask in ((abi.METRIC_ERR5XX, abi.CHANGE_DELTA, 7), ((Q, 0.5), abi.CHANGE_RATIO, 5),
                             (abi.METRIC_MEAN_NS, abi.CHANGE_DROP, 6)):
        same(hh.debug_edge_changes_rows(ra, rb, spec, mode, mask, 5, 60),
             cr.changes(ra, rb, spec, mode, mask, 5, 60), ("large", spec, mode, mask))
