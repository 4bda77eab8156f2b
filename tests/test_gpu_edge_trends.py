"""GPU: edge trends (alz_edge_trends*, docs/SPEC.md §20).

The expected records, top order, series, presence, points and info are tests/trend_ref.py over the entries that
tests/rollup_model.py and tests/tier_model.py say the rings retain, compared as bytes. Windows come from the Modelled
stream of tests/test_gpu_edge_series.py."""
import ctypes as C

import numpy as np
import pytest

import trend_ref as tr
from alaz_b200 import abi, capi
from test_gpu_edge_series import DEPTH, TIER_DEPTH, Modelled, make_source
from test_gpu_gnn_rollup import universe

pytestmark = pytest.mark.gpu
WINDOW, WIN, TIER, SPAN = abi.SOURCE_WINDOW, abi.ROLLUP_WINDOWS, abi.ROLLUP_TIER, abi.ROLLUP_SPAN
Q = abi.METRIC_QUANTILE
STATS = [abi.TREND_SLOPE, abi.TREND_SHIFT, abi.TREND_RATIO, abi.TREND_ZSCORE]
T = capi.Handle.trend


def spec_of(t):
    return dict(stat=t.stat, direction=t.direction, absent=t.absent, recent=t.recent, min_points=t.min_points)


def expect(m, rows, tier, k, spec, t):
    ents, pts = m.entries(tier)
    rec, y, p = tr.expect(ents, rows, spec, k, **spec_of(t))
    take = pts[max(len(pts) - k, 0):]
    info = dict(edges=len(rows), rows_in=sum(x["rows_in"] for x in take), valid=int(rec["valid"].sum()), above=0,
                points=len(take), tier=tier)
    return rec, y, p, take, info


def check(m, rows, source, tier, k, spec, t, top=None, min_trend=-np.inf, what=None):
    """the full list and the top call of (source, tier, k, spec, t) against the reference, as bytes"""
    h = m.h
    what = what or (source, tier, k, spec, spec_of(t))
    rec, y, p, pts, info = expect(m, rows, tier, k, spec, t)
    got, gpts, ginfo = h.edge_trends(source, tier, k, spec, t)
    assert got.tobytes() == rec.tobytes(), (what, np.flatnonzero(got.view(np.uint8).reshape(-1, 48).any(1)
                                                                    != rec.view(np.uint8).reshape(-1, 48).any(1))[:5])
    assert gpts == pts and ginfo == info, (what, ginfo, info)
    top = top or max(len(rows) // 4, 1)
    idx, above = tr.top(rec, top, min_trend)
    trec, trows, ts, tp, tpts, tinfo = h.edge_trends_top(source, tier, k, spec, t, top, min_trend)
    assert trec.tobytes() == rec[idx].tobytes(), (what, trec["index"][:8], idx[:8])
    assert trows.tobytes() == rows[idx].tobytes(), what
    assert ts.tobytes() == y[idx].tobytes() and tp.tobytes() == p[idx].tobytes(), what
    assert tpts == pts and tinfo == dict(info, above=above), (what, tinfo)
    return rec, idx


@pytest.fixture(scope="module")
def mod():
    m = Modelled(universe(seed=24), history=(DEPTH, 1 << 15), tiers=[(2, TIER_DEPTH, 1 << 15, 1 << 13)])
    m.random_windows(12, seed=241, lo=0.2, hi=0.7)
    m.last = m.window(np.flatnonzero(np.random.default_rng(242).random(m.s.g.n_edges) < 0.5))
    assert len(m.rm.entries) == DEPTH and len(m.tm.tiers[0].ring.entries) == TIER_DEPTH
    yield m
    m.close()


@pytest.mark.parametrize("tier", [0, 1])
@pytest.mark.parametrize("source", [WINDOW, WIN, TIER, SPAN])
def test_every_source_stat_direction_and_absent_mode(mod, tier, source):
    rows = make_source(mod, source)
    depth = DEPTH if tier == 0 else TIER_DEPTH
    cases = [(depth, 1, (Q, 0.99)), (depth + 4, 2, abi.METRIC_COUNT), (3, 2, abi.METRIC_ERR_RATE),
             (2, 1, abi.METRIC_MEAN_NS), (depth, depth - 1, abi.METRIC_ERR5XX)]
    valid = 0
    for stat in STATS:
        for direction in (abi.TREND_RISING, abi.TREND_FALLING):
            for absent in (abi.TREND_ABSENT_SKIP, abi.TREND_ABSENT_ZERO):
                for k, r, spec in cases:
                    rec, _ = check(mod, rows, source, tier, k, spec, T(stat, direction, absent, r))
                    valid += int(rec["valid"].sum())
    assert valid > 0


def test_min_points_and_min_trend_cuts(mod):
    rows = mod.last
    for mp in (0, 3, DEPTH - 1, DEPTH, DEPTH + 1):
        rec, _ = check(mod, rows, WINDOW, 0, DEPTH, (Q, 0.99), T(abi.TREND_SLOPE, recent=2, min_points=mp))
        assert (rec["valid"] == 1).sum() == ((rec["used"] >= max(mp, 2)).sum())
    t = T(abi.TREND_SHIFT, recent=2)
    rec, _, _, _, _ = expect(mod, rows, 0, DEPTH, (Q, 0.99), t)
    vals = np.sort(rec["trend"][rec["valid"] == 1])
    for cut in (vals[len(vals) // 2], vals[-1], vals[-1] + 1.0, 0.0, -0.0, -np.inf, np.inf):
        _, idx = check(mod, rows, WINDOW, 0, DEPTH, (Q, 0.99), t, top=len(rows), min_trend=cut, what=cut)
        assert np.all(rec["trend"][idx] >= cut)


def test_infinite_trends_rank_first_and_ties_go_by_index(mod):
    rows = mod.last
    t = T(abi.TREND_RATIO, absent=abi.TREND_ABSENT_ZERO, recent=1)    # new edges: before 0, recent > 0 -> +inf
    rec, idx = check(mod, rows, WINDOW, 0, 3, abi.METRIC_COUNT, t, top=len(rows))
    inf = np.flatnonzero(rec["trend"] == np.inf)
    assert len(inf) > 10 and idx[: len(inf)].tolist() == inf.tolist()
    # ZSCORE over zeros before: +inf rising, first; -inf falling, last of the valid rows
    for direction, first in ((abi.TREND_RISING, True), (abi.TREND_FALLING, False)):
        t = T(abi.TREND_ZSCORE, direction=direction, absent=abi.TREND_ABSENT_ZERO, recent=1)
        rec, idx = check(mod, rows, WINDOW, 0, DEPTH, abi.METRIC_COUNT, t, top=len(rows), what=("zscore", direction))
        inf = np.flatnonzero(np.isinf(rec["trend"]))
        assert len(inf) > 10 and len(idx) == rec["valid"].sum()
        assert (idx[: len(inf)] if first else idx[len(idx) - len(inf):]).tolist() == inf.tolist()


def test_identical_series_tie_in_index_order():
    m = Modelled(universe(n_edges=500, seed=25), history=(6, 1 << 13))
    for _ in range(5):
        m.window(np.arange(500))
    rows = m.window(np.arange(500))
    for t in (T(abi.TREND_SLOPE), T(abi.TREND_SHIFT, recent=2), T(abi.TREND_RATIO, recent=3)):
        rec, idx = check(m, rows, WINDOW, 0, 6, abi.METRIC_COUNT, t, top=100)
        assert np.all(rec["valid"] == 1) and len(np.unique(rec["trend"])) == 1
        assert idx.tolist() == list(range(100))
    m.close()


@pytest.mark.parametrize("tier", [0, 1])
def test_top_series_are_the_series_rows_and_device_equals_host(mod, tier):
    h = mod.h
    rows = mod.last
    t = T(abi.TREND_ZSCORE, recent=1)
    spec = (Q, 0.5)
    k = DEPTH if tier == 0 else TIER_DEPTH
    trec, trows, ts, tp, tpts, tinfo = h.edge_trends_top(WINDOW, tier, k, spec, t, 50)
    sv, sp, spts, _ = h.edge_series(WINDOW, tier, k, spec)
    assert len(trec) == 50
    assert ts.tobytes() == sv[trec["index"], :, 0].tobytes() and tp.tobytes() == sp[trec["index"]].tobytes()
    assert tpts == spts
    got, pts, info = h.edge_trends(WINDOW, tier, k, spec, t)
    d, n, P, dpts, dinfo = h.edge_trends_device(WINDOW, tier, k, spec, t)
    assert (n, P, dpts, dinfo) == (len(got), len(pts), pts, info)
    assert h.d2h(d, n, abi.EDGE_TREND).tobytes() == got.tobytes()
    pr, pw, ps, pp, m, P, dpts, dinfo = h.edge_trends_top_device(WINDOW, tier, k, spec, t, 50)
    assert (m, P, dpts, dinfo) == (50, len(tpts), tpts, tinfo)
    assert h.d2h(pr, m, abi.EDGE_TREND).tobytes() == trec.tobytes()
    assert h.d2h(pw, m, abi.EDGE_OUT).tobytes() == trows.tobytes()
    assert h.d2h(ps, m * P, np.float64).tobytes() == ts.tobytes()
    assert h.d2h(pp, m * P, np.uint8).tobytes() == tp.tobytes()


def test_no_retained_entry_and_reconfiguration():
    m = Modelled(universe(n_edges=400, seed=26), history=(4, 1 << 13), tiers=[(2, 2, 1 << 13, 1 << 12)])
    m.random_windows(5, seed=261)
    t = T(abi.TREND_SHIFT, recent=1)
    win = m.window(np.arange(300))
    check(m, win, WINDOW, 0, 4, abi.METRIC_COUNT, t)
    m.h.window_history(5, 1 << 12)                      # reconfiguring drops the history: P = 0
    m.rm.history(5, 1 << 12)
    got, pts, info = m.h.edge_trends(WINDOW, 0, 4, abi.METRIC_COUNT, t)
    assert len(got) == len(win) == info["edges"] and got["index"].tolist() == list(range(len(win)))
    assert pts == [] and info["points"] == 0 and info["valid"] == 0 and not got["valid"].any()
    assert not got["used"].any() and not got["trend"].view(np.uint64).any()
    trec, trows, ts, tp, tpts, tinfo = m.h.edge_trends_top(WINDOW, 0, 4, abi.METRIC_COUNT, t, 10)
    assert len(trec) == 0 and ts.shape == (0, 0) and tinfo["above"] == 0 and tinfo["points"] == 0
    for n in (120, 0, 250, 200):                       # the new history, an empty window among them
        last = m.window(np.arange(n) if n else np.zeros(0, np.int64))
    for k, r in ((2, 1), (4, 3), (9, 2)):
        for stat in STATS:
            check(m, last, WINDOW, 0, k, (Q, 0.9), T(stat, recent=r), what=("after", k, r, stat))
    check(m, last, WINDOW, 1, 3, abi.METRIC_COUNT, T(abi.TREND_SLOPE, recent=1), what="tier")
    m.close()


# ---- errors ------------------------------------------------------------------------------------------------------

def raw(h, source, tier, k, m, t, out=None, cap=0):
    n, p, info = C.c_size_t(777), C.c_uint32(777), abi.TrendInfo()
    rc = h.L.alz_edge_trends(h.h, source, tier, k, m, C.byref(t) if t is not None else None, out, cap, C.byref(n),
                             C.byref(p), None, C.byref(info))
    return rc, n.value, p.value


def raw_top(h, source, tier, k, m, t, top, min_trend, cap=0, out=None):
    n, p, info = C.c_size_t(777), C.c_uint32(777), abi.TrendInfo()
    rc = h.L.alz_edge_trends_top(h.h, source, tier, k, m, C.byref(t), top, min_trend, out, None, None, None, cap,
                                 C.byref(n), C.byref(p), None, C.byref(info))
    return rc, n.value, p.value


def test_every_error_code():
    m = Modelled(universe(n_edges=400, seed=27), history=(3, 1 << 14), tiers=[(2, 2, 1 << 14, 1 << 12)])
    h = m.h
    cm = abi.metrics(abi.METRIC_COUNT)
    m.random_windows(5, seed=271)
    ok = T(abi.TREND_SHIFT, recent=1)
    rc, n, P = raw(h, WINDOW, 0, 3, cm, ok)
    assert rc == abi.E_CAPACITY and n > 0 and P == 3                               # cap 0 below the rows
    # invalid arguments
    assert raw(h, WINDOW, 0, 1, cm, T(recent=1))[0] == abi.E_INVAL                 # k < 2
    assert raw(h, WINDOW, 0, 0, cm, T(recent=1))[0] == abi.E_INVAL
    for bad in (T(recent=0), T(recent=3), T(stat=4, recent=1), T(direction=2, recent=1), T(absent=2, recent=1)):
        assert raw(h, WINDOW, 0, 3, cm, bad)[0] == abi.E_INVAL, spec_of(bad)
    assert raw(h, WINDOW, 0, 4, cm, T(recent=3))[0] == abi.E_CAPACITY             # r = k - 1 is fine
    assert raw(h, WINDOW, 2, 3, cm, ok)[0] == abi.E_INVAL                          # tier above the tiers
    assert raw(h, WINDOW, 0, 3, (abi.Metric * 1)(abi.Metric(9, 0, 0.0)), ok)[0] == abi.E_INVAL
    for q in (1.5, -0.1, float("nan")):
        assert raw(h, WINDOW, 0, 3, abi.metrics((Q, q)), ok)[0] == abi.E_INVAL
    assert raw(h, 3, 0, 3, cm, ok)[0] == abi.E_INVAL                               # unknown source
    assert raw(h, WINDOW, 0, 3, None, ok)[0] == abi.E_INVAL                        # null metric
    assert raw(h, WINDOW, 0, 3, cm, None)[0] == abi.E_INVAL                        # null trend
    assert raw(h, WINDOW, 0, 3, cm, ok, cap=5)[0] == abi.E_INVAL                   # null out with cap
    assert raw_top(h, WINDOW, 0, 3, cm, ok, 0, 0.0)[0] == abi.E_INVAL              # top = 0
    assert raw_top(h, WINDOW, 0, 3, cm, ok, 5, float("nan"))[0] == abi.E_INVAL
    n, p_ = C.c_size_t(0), C.c_uint32(0)
    assert h.L.alz_edge_trends(h.h, WINDOW, 0, 3, cm, C.byref(ok), None, 0, None, C.byref(p_), None,
                               None) == abi.E_INVAL
    assert h.L.alz_edge_trends(h.h, WINDOW, 0, 3, cm, C.byref(ok), None, 0, C.byref(n), None, None,
                               None) == abi.E_INVAL
    assert h.L.alz_edge_trends(None, WINDOW, 0, 3, cm, C.byref(ok), None, 0, C.byref(n), C.byref(p_), None,
                               None) == abi.E_INVAL
    assert h.L.alz_edge_trends_device(h.h, WINDOW, 0, 3, cm, C.byref(ok), None, C.byref(n), C.byref(p_), None,
                                      None) == abi.E_INVAL                          # null dev_out
    assert h.L.alz_edge_trends_top_device(h.h, WINDOW, 0, 3, cm, C.byref(ok), 5, 0.0, None, None, None, None,
                                          C.byref(n), C.byref(p_), None, None) == abi.E_INVAL
    # state: no rows of a rollup source; no tiers, no history
    for src in (WIN, TIER, SPAN):
        assert raw(h, src, 0, 3, cm, ok)[0] == abi.E_STATE
        assert raw_top(h, src, 0, 3, cm, ok, 5, 0.0)[0] == abi.E_STATE
    t = Modelled(universe(n_edges=200, seed=28), tiers=[(2, 2, 1 << 13, 1 << 12)])
    t.random_windows(2, seed=281)
    assert raw(t.h, WINDOW, 0, 3, cm, ok)[0] == abi.E_STATE
    t.close()
    w = Modelled(universe(n_edges=200, seed=29), history=(2, 1 << 13))
    w.random_windows(1, seed=291)
    assert raw(w.h, WINDOW, 1, 3, cm, ok)[0] == abi.E_STATE
    w.close()
    # capacity: a host cap below the rows, or below the top rows, writes nothing
    rc, n_rows, P = raw(h, WINDOW, 0, 3, cm, ok)
    buf = np.full(n_rows * 48, 0x5A, np.uint8)
    rc, n2, P2 = raw(h, WINDOW, 0, 3, cm, ok, out=buf.ctypes.data_as(C.c_void_p), cap=n_rows - 1)
    assert (rc, n2, P2) == (abi.E_CAPACITY, n_rows, 3) and np.all(buf == 0x5A)
    rc, m_top, _ = raw_top(h, WINDOW, 0, 3, cm, ok, 40, -np.inf, cap=10, out=buf.ctypes.data_as(C.c_void_p))
    assert (rc, m_top) == (abi.E_CAPACITY, 40) and np.all(buf == 0x5A)
    m.close()


def test_more_than_2_30_slots_is_a_capacity_error():
    """2^14 rows over 2^16 points (empty windows, then the source window) are 2^30 slots: refused before anything
    runs; 2^12 points fit."""
    m = Modelled(universe(n_pods=3000, n_edges=1 << 14, seed=30), history=(1 << 16, 1 << 15))
    for _ in range((1 << 16) - 1):
        m.h.flush()
    rows = m.s.window(np.arange(1 << 14))
    assert len(rows) == 1 << 14
    cm = abi.metrics(abi.METRIC_COUNT)
    n, p_, d = C.c_size_t(0), C.c_uint32(0), C.c_void_p()
    t = T(recent=1)
    rc = m.h.L.alz_edge_trends_device(m.h.h, WINDOW, 0, 1 << 16, cm, C.byref(t), C.byref(d), C.byref(n),
                                      C.byref(p_), None, None)
    assert (rc, n.value, p_.value) == (abi.E_CAPACITY, 1 << 14, 1 << 16)
    rc = m.h.L.alz_edge_trends_top_device(m.h.h, WINDOW, 0, 1 << 16, cm, C.byref(t), 5, 0.0, C.byref(d), None, None,
                                          None, C.byref(n), C.byref(p_), None, None)
    assert (rc, n.value, p_.value) == (abi.E_CAPACITY, 0, 1 << 16)
    got, pts, info = m.h.edge_trends(WINDOW, 0, 1 << 12, abi.METRIC_COUNT, t)
    assert info["points"] == 1 << 12 and info["valid"] == 0 and np.all(got["used"] == 1)   # SKIP: one point each
    m.close()


# ---- reads only ----------------------------------------------------------------------------------------------------

def test_reads_only():
    m = Modelled(universe(seed=31), history=(5, 1 << 15), tiers=[(2, 3, 1 << 15, 1 << 13)])
    m.random_windows(8, seed=311, lo=0.2, hi=0.6)
    h = m.h
    h.rollup(3)
    h.baseline_pin(WIN)
    m.random_windows(2, seed=312)
    h.rollup_tier(1, 2)
    h.rollup_span(5)
    h.rollup(2)
    ALL = [abi.METRIC_COUNT, (Q, 0.99), abi.METRIC_ERR_RATE]

    def snapshot():
        return dict(series=h.d2h(sv, sn * sp_ * len(ALL), np.float64), series_p=h.d2h(spp, sn * sp_, np.uint8),
                    metrics=h.d2h(mv, mn, np.float64), top=h.d2h(tv, tn, np.float64), top_i=h.d2h(ti, tn, np.uint32),
                    top_r=h.d2h(tr_, tn, abi.EDGE_OUT), changes=h.d2h(cv, cn, abi.EDGE_CHANGE),
                    gnn=h.d2h(gv, gn, np.float32), nodes=nodes())

    def nodes():
        keys = np.zeros(1 << 16, dtype=np.uint64)
        emb = np.zeros((1 << 16, 64), dtype=np.float32)
        nv = C.c_size_t(0)
        h._ck(h.L.alz_gnn_nodes(h.h, keys.ctypes.data_as(C.c_void_p), emb.ctypes.data_as(C.c_void_p), len(keys),
                                C.byref(nv)), "alz_gnn_nodes")
        return np.concatenate([keys[: nv.value].view(np.uint8), emb[: nv.value].view(np.uint8).ravel()])

    held = {kind: h.gnn_score_rollup(kind) for kind in (WIN, TIER, SPAN)}
    changes = h.edge_changes((Q, 0.99), abi.CHANGE_DELTA, source=SPAN)[0]
    stats = h.stats()
    sv, spp, sn, sp_, _, _ = h.edge_series_device(WIN, 0, 4, *ALL)
    mv, mn = h.edge_metrics_rollup_device(TIER, *ALL)
    tr_, tv, ti, tn, _ = h.edge_top_rollup_device(SPAN, (Q, 0.99), 9)
    cv, cn, _ = h.edge_changes_device((Q, 0.99), abi.CHANGE_RATIO)
    gv, gn = h.gnn_score_rollup_device(WIN)
    before = snapshot()
    for tier in (0, 1):
        for src in (WINDOW, WIN, TIER, SPAN):
            for stat in STATS:
                t = T(stat, recent=1, absent=abi.TREND_ABSENT_ZERO)
                h.edge_trends(src, tier, 9, (Q, 0.99), t)
                h.edge_trends_top(src, tier, 4, abi.METRIC_COUNT, t, 17)
                h.edge_trends_device(src, tier, 3, abi.METRIC_ERR5XX, t)
                h.edge_trends_top_device(src, tier, 9, (Q, 0.5), t, 5)
    after = snapshot()
    for k in before:
        assert np.asarray(before[k]).tobytes() == np.asarray(after[k]).tobytes(), k
    for kind in (WIN, TIER, SPAN):
        assert h.gnn_score_rollup(kind).tobytes() == held[kind].tobytes(), kind
    assert h.edge_changes((Q, 0.99), abi.CHANGE_DELTA, source=SPAN)[0].tobytes() == changes.tobytes()
    assert h.stats()["windows"] == stats["windows"]
    m.close()
