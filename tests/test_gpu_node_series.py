"""GPU: node series and node trends (alz_node_series*, alz_node_series_keys*, alz_node_trends*, docs/SPEC.md §22).

Values, presence, records, top order, node rows, points and info are compared as bytes against tests/node_series_ref.py
over the entries that tests/rollup_model.py and tests/tier_model.py say the rings retain. Windows come from the
Modelled stream of tests/test_gpu_edge_series.py."""
import ctypes as C

import numpy as np
import pytest

import node_ref as nr
import node_series_ref as nsr
from alaz_b200 import abi, capi
from test_gpu_edge_series import DEPTH, TIER_DEPTH, Modelled, make_source
from test_gpu_gnn_rollup import universe

pytestmark = pytest.mark.gpu
WINDOW, WIN, TIER, SPAN = abi.SOURCE_WINDOW, abi.ROLLUP_WINDOWS, abi.ROLLUP_TIER, abi.ROLLUP_SPAN
IN, OUT = abi.SIDE_IN, abi.SIDE_OUT
Q = abi.METRIC_QUANTILE
SPECS = ([abi.METRIC_COUNT], [(Q, 0.99)], [(Q, 0.5), (Q, 0.99), abi.METRIC_ERR_RATE])
STATS = [abi.TREND_SLOPE, abi.TREND_SHIFT, abi.TREND_RATIO, abi.TREND_ZSCORE]
T = capi.Handle.trend
POD, SVC, OUTB, HOST = 0, 1, 2, 3


@pytest.fixture(scope="module")
def mod():
    m = Modelled(universe(seed=44), history=(DEPTH, 1 << 15), tiers=[(2, TIER_DEPTH, 1 << 15, 1 << 13)])
    m.random_windows(12, seed=441, lo=0.2, hi=0.7)
    m.last = m.window(np.flatnonzero(np.random.default_rng(442).random(m.s.g.n_edges) < 0.5))
    assert len(m.rm.entries) == DEPTH and len(m.tm.tiers[0].ring.entries) == TIER_DEPTH
    yield m
    m.close()


def expect(m, tier, k, keys, side, specs):
    ents, pts = m.entries(tier)
    v, p = nsr.series(ents, keys, side, specs, k)
    take = pts[max(len(pts) - k, 0):]
    return v, p, take, sum(x["rows_in"] for x in take)


def same(got, want, what):
    v, p, pts, info = got
    wv, wp, wpts, rows_in = want
    assert v.shape == wv.shape and p.shape == wp.shape, (what, v.shape, wv.shape)
    assert p.tobytes() == wp.tobytes(), (what, np.argwhere(p != wp)[:5])
    assert v.tobytes() == wv.tobytes(), (what, np.argwhere(v.view(np.uint64) != wv.view(np.uint64))[:5])
    assert pts == wpts, (what, pts, wpts)
    assert info["points"] == len(wpts) and info["edges"] == len(p) and info["rows_in"] == rows_in, (what, info)


def same_device(h, got, dev, nm, what):
    v, p, pts, info = got
    pv, pp, n, P, dpts, dinfo = dev
    assert (n, P, dpts, dinfo) == (v.shape[0], v.shape[1], pts, info), what
    assert h.d2h(pv, n * P * nm, np.float64).tobytes() == v.tobytes(), what
    assert h.d2h(pp, n * P, np.uint8).tobytes() == p.tobytes(), what


# ---- series ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("tier", [0, 1])
@pytest.mark.parametrize("source", [WINDOW, WIN, TIER, SPAN])
def test_every_source_side_ring_and_metric_set(mod, tier, source):
    h = mod.h
    keys = nr.keys(make_source(mod, source))
    depth = DEPTH if tier == 0 else TIER_DEPTH
    absent_some = present_some = False
    for side in (IN, OUT):
        for k in (1, 3, depth + 5):
            for specs in SPECS:
                got = h.node_series(source, side, tier, k, *specs)
                same(got, expect(mod, tier, k, keys, side, specs), (source, side, tier, k, specs))
                absent_some |= not got[1].all()
                present_some |= bool(got[1].any())
        specs = SPECS[2]
        same_device(h, h.node_series(source, side, tier, 3, *specs), h.node_series_device(source, side, tier, 3, *specs),
                    len(specs), (source, side, tier))
    assert absent_some and present_some


@pytest.mark.parametrize("tier", [0, 1])
def test_caller_keys_host_and_device(mod, tier):
    h = mod.h
    rng = np.random.default_rng(tier)
    seen = nr.keys(np.concatenate(mod.entries(tier)[0]))
    pick = seen[rng.choice(len(seen), 200, replace=False)]
    nodes = [(int(k >> np.uint64(32)), int(k & np.uint64(0xFFFFFFFF))) for k in pick]
    nodes += nodes[:9] + [(POD, 123456), (SVC, (1 << 29) - 1), (OUTB, 0xFFFFFFFF), (HOST, 7)]   # duplicates, unknown
    ends = capi.Handle.node_ends(nodes)
    keys = nsr.ends_keys(ends)
    for side in (IN, OUT):
        for k in (1, 3, 50):
            for specs in SPECS:
                got = h.node_series_keys(ends, side, tier, k, *specs)
                same(got, expect(mod, tier, k, keys, side, specs), ("keys", side, tier, k, specs))
            same_device(h, got, h.node_series_keys_device(ends, side, tier, k, *specs), len(specs), ("keys", side, k))
        v, p, _, _ = h.node_series_keys(ends, side, tier, 50, *SPECS[2])
        assert v[:9].tobytes() == v[200:209].tobytes() and p[:9].tobytes() == p[200:209].tobytes()


@pytest.mark.parametrize("tier", [0, 1])
def test_newest_point_is_the_k1_rollup_node_metrics(mod, tier):
    h = mod.h
    kind = WIN if tier == 0 else TIER
    (h.rollup if tier == 0 else (lambda k: h.rollup_tier(1, k)))(1)
    nodes = h.node_rows(kind)
    for side in (IN, OUT):
        specs = [abi.METRIC_COUNT, abi.METRIC_ERR_RATE, (Q, 0.5), (Q, 0.99), abi.METRIC_MEAN_NS]
        want = h.node_metrics(kind, side, *specs)
        on = nodes["in_edges" if side == IN else "out_edges"] > 0
        v, p, _, _ = h.node_series_keys(nodes, side, tier, 3, *specs)
        assert p[:, -1].tobytes() == on.astype(np.uint8).tobytes()
        assert v[on, -1, :].tobytes() == want[on].tobytes() and not v[~on, -1, :].any()
        v, p, _, _ = h.node_series(kind, side, tier, 1, *specs)
        assert v[on, 0, :].tobytes() == want[on].tobytes()


def key_index(keys, t, v):
    i = np.flatnonzero(keys == np.uint64((t << 32) | v))
    assert len(i) == 1
    return int(i[0])


def test_hub_service_called_by_thousands_of_pods_in_every_window():
    m = Modelled(universe(n_pods=6000, n_svcs=1, n_edges=12000, seed=45), history=(4, 1 << 16))
    try:
        m.random_windows(5, seed=451, lo=0.6, hi=0.8)
        rows = m.h.rollup(4)[0]
        keys = nr.keys(rows)
        hub = key_index(keys, SVC, 0)
        for ent in m.entries(0)[0]:
            callers = ent[(ent["to_type"] == SVC) & (ent["to"] == 0)]
            assert len(np.unique(callers["from"])) >= 1000
        for side in (IN, OUT):
            for specs in SPECS:
                got = m.h.node_series(WIN, side, 0, 4, *specs)
                same(got, expect(m, 0, 4, keys, side, specs), ("hub", side, specs))
        v, p, _, _ = m.h.node_series(WIN, IN, 0, 4, abi.METRIC_COUNT)
        assert p[hub].all() and (v[hub, :, 0] > 1000).all()
    finally:
        m.close()


def test_no_points_and_empty_sources():
    m = Modelled(universe(n_edges=300, seed=46), history=(4, 1 << 13))
    try:
        h = m.h
        rows = m.window(np.arange(300))
        n = len(nr.keys(rows))
        h.window_history(5, 1 << 12)                 # reconfigured: no retained entry, P = 0
        m.rm.history(5, 1 << 12)
        v, p, pts, info = h.node_series(WINDOW, IN, 0, 3, *SPECS[2])
        assert v.shape == (n, 0, 3) and p.shape == (n, 0) and pts == [] and info["points"] == 0
        rec, pts, info = h.node_trends(WINDOW, IN, 0, 3, abi.METRIC_COUNT, T(abi.TREND_SLOPE))
        assert len(rec) == n and not rec["valid"].any() and info["valid"] == 0
        trec, tn, ts, tp, tpts, tinfo = h.node_trends_top(WINDOW, IN, 0, 3, abi.METRIC_COUNT, T(abi.TREND_SLOPE), 5)
        assert len(trec) == 0 and tinfo["edges"] == n and tinfo["above"] == 0
        m.window(np.zeros(0, np.int64))              # an empty window: a source of no nodes, one empty entry
        v, p, pts, info = h.node_series(WINDOW, OUT, 0, 3, abi.METRIC_COUNT)
        assert v.shape == (0, 1, 1) and len(pts) == 1 and info["rows_in"] == 0
        v, p, pts, info = h.node_series_keys(capi.Handle.node_ends([(SVC, 1)]), IN, 0, 3, abi.METRIC_COUNT)
        assert v.shape == (1, 1, 1) and not p.any() and not v.any()
    finally:
        m.close()


# ---- trends ----------------------------------------------------------------------------------------------------------

def spec_of(t):
    return dict(stat=t.stat, direction=t.direction, absent=t.absent, recent=t.recent, min_points=t.min_points)


def check_trends(m, rows, source, side, tier, k, spec, t, top=None, min_trend=-np.inf, what=None):
    """the full list and the top call of the node trends against the reference, as bytes"""
    h = m.h
    what = what or (source, side, tier, k, spec, spec_of(t))
    ents, pts = m.entries(tier)
    rec, y, p = nsr.expect(ents, rows, side, spec, k, **spec_of(t))
    nodes = nr.group(rows)
    take = pts[max(len(pts) - k, 0):]
    info = dict(edges=len(nodes), rows_in=sum(x["rows_in"] for x in take), valid=int(rec["valid"].sum()), above=0,
                points=len(take), tier=tier)
    got, gpts, ginfo = h.node_trends(source, side, tier, k, spec, t)
    assert got.tobytes() == rec.tobytes(), (what, np.flatnonzero((got.view(np.uint8).reshape(-1, 48)
                                                                  != rec.view(np.uint8).reshape(-1, 48)).any(1))[:5])
    assert gpts == take and ginfo == info, (what, ginfo, info)
    top = top or max(len(nodes) // 4, 1)
    idx, above = nsr.top(rec, top, min_trend)
    trec, tnodes, ts, tp, tpts, tinfo = h.node_trends_top(source, side, tier, k, spec, t, top, min_trend)
    assert trec.tobytes() == rec[idx].tobytes(), (what, trec["index"][:8], idx[:8])
    assert tnodes.tobytes() == nodes[idx].tobytes(), what
    assert ts.tobytes() == y[idx].tobytes() and tp.tobytes() == p[idx].tobytes(), what
    assert tpts == take and tinfo == dict(info, above=above), (what, tinfo)
    return rec, idx


@pytest.mark.parametrize("side", [IN, OUT])
@pytest.mark.parametrize("source", [WINDOW, SPAN])
def test_trends_every_stat_direction_and_absent_mode(mod, source, side):
    rows = make_source(mod, source)
    valid = 0
    for stat in STATS:
        for direction in (abi.TREND_RISING, abi.TREND_FALLING):
            for absent in (abi.TREND_ABSENT_SKIP, abi.TREND_ABSENT_ZERO):
                for tier, k, r, spec in ((0, DEPTH, 1, (Q, 0.99)), (0, 3, 2, abi.METRIC_COUNT),
                                         (1, TIER_DEPTH + 2, 1, abi.METRIC_ERR_RATE)):
                    rec, _ = check_trends(mod, rows, source, side, tier, k, spec, T(stat, direction, absent, r))
                    valid += int(rec["valid"].sum())
    assert valid > 0


@pytest.mark.parametrize("source", [WIN, TIER])
def test_trends_rollup_sources(mod, source):
    rows = make_source(mod, source)
    for side in (IN, OUT):
        check_trends(mod, rows, source, side, 0, DEPTH, (Q, 0.5), T(abi.TREND_ZSCORE, recent=2))
        check_trends(mod, rows, source, side, 1, TIER_DEPTH, abi.METRIC_MEAN_NS, T(abi.TREND_SLOPE))


def test_trend_cuts_infinities_and_index_ties(mod):
    rows = mod.last
    for mp in (0, 3, DEPTH, DEPTH + 1):
        rec, _ = check_trends(mod, rows, WINDOW, IN, 0, DEPTH, (Q, 0.99), T(abi.TREND_SLOPE, recent=2, min_points=mp))
        assert (rec["valid"] == 1).sum() == (rec["used"] >= max(mp, 2)).sum()
    t = T(abi.TREND_SHIFT, recent=2)
    rec, _, _ = nsr.expect(mod.entries(0)[0], rows, IN, (Q, 0.99), DEPTH, **spec_of(t))
    vals = np.sort(rec["trend"][rec["valid"] == 1])
    n = len(rec)
    for cut in (vals[len(vals) // 2], vals[-1], vals[-1] + 1.0, 0.0, -0.0, -np.inf, np.inf):
        _, idx = check_trends(mod, rows, WINDOW, IN, 0, DEPTH, (Q, 0.99), t, top=n, min_trend=cut, what=cut)
        assert np.all(rec["trend"][idx] >= cut)
    # nodes new in the last window: before 0, recent > 0 -> RATIO +inf, ranked first in index order
    rec, idx = check_trends(mod, rows, WINDOW, OUT, 0, 3, abi.METRIC_COUNT,
                            T(abi.TREND_RATIO, absent=abi.TREND_ABSENT_ZERO, recent=1), top=n)
    inf = np.flatnonzero(rec["trend"] == np.inf)
    assert len(inf) > 0 and idx[: len(inf)].tolist() == inf.tolist()
    for direction, first in ((abi.TREND_RISING, True), (abi.TREND_FALLING, False)):
        t = T(abi.TREND_ZSCORE, direction=direction, absent=abi.TREND_ABSENT_ZERO, recent=1)
        rec, idx = check_trends(mod, rows, WINDOW, IN, 0, DEPTH, abi.METRIC_COUNT, t, top=n, what=("z", direction))
        inf = np.flatnonzero(np.isinf(rec["trend"]))
        assert len(idx) == rec["valid"].sum()
        assert (idx[: len(inf)] if first else idx[len(idx) - len(inf):]).tolist() == inf.tolist()


def test_identical_node_series_tie_in_index_order():
    m = Modelled(universe(n_edges=500, seed=47), history=(6, 1 << 13))
    try:
        for _ in range(5):
            m.window(np.arange(500))
        rows = m.window(np.arange(500))
        n = len(nr.keys(rows))
        rec, idx = check_trends(m, rows, WINDOW, OUT, 0, 6, abi.METRIC_COUNT, T(abi.TREND_SHIFT, recent=2), top=n)
        on = np.flatnonzero(rec["valid"] == 1)
        assert len(on) > 50 and np.all(rec["trend"][on] == 0.0) and idx.tolist() == on.tolist()
    finally:
        m.close()


@pytest.mark.parametrize("tier", [0, 1])
def test_trend_top_series_are_node_series_and_device_equals_host(mod, tier):
    h = mod.h
    t = T(abi.TREND_ZSCORE, recent=1)
    spec = (Q, 0.99)
    k = DEPTH if tier == 0 else TIER_DEPTH
    trec, tnodes, ts, tp, tpts, tinfo = h.node_trends_top(SPAN, IN, tier, k, spec, t, 40)
    sv, sp, spts, _ = h.node_series(SPAN, IN, tier, k, spec)
    assert len(trec) == 40 and tpts == spts
    assert ts.tobytes() == sv[trec["index"], :, 0].tobytes() and tp.tobytes() == sp[trec["index"]].tobytes()
    assert tnodes.tobytes() == h.node_rows(SPAN)[trec["index"]].tobytes()
    got, pts, info = h.node_trends(SPAN, IN, tier, k, spec, t)
    d, n, P, dpts, dinfo = h.node_trends_device(SPAN, IN, tier, k, spec, t)
    assert (n, P, dpts, dinfo) == (len(got), len(pts), pts, info)
    assert h.d2h(d, n, abi.NODE_TREND).tobytes() == got.tobytes()
    pr, pn, ps, pp, m, P, dpts, dinfo = h.node_trends_top_device(SPAN, IN, tier, k, spec, t, 40)
    assert (m, P, dpts, dinfo) == (40, len(tpts), tpts, tinfo)
    assert h.d2h(pr, m, abi.NODE_TREND).tobytes() == trec.tobytes()
    assert h.d2h(pn, m, abi.NODE_OUT).tobytes() == tnodes.tobytes()
    assert h.d2h(ps, m * P, np.float64).tobytes() == ts.tobytes()
    assert h.d2h(pp, m * P, np.uint8).tobytes() == tp.tobytes()


# ---- errors ------------------------------------------------------------------------------------------------------

def raw(h, *args, fn="alz_node_series", out=None, present=None, cap=0, points=None):
    n, p, info = C.c_size_t(777), C.c_uint32(777), abi.SeriesInfo()
    rc = getattr(h.L, fn)(h.h, *args, out, present, cap, C.byref(n), C.byref(p), points, C.byref(info))
    return rc, n.value, p.value


def raw_trends(h, *args, fn="alz_node_trends", cap=0):
    n, p, info = C.c_size_t(777), C.c_uint32(777), abi.TrendInfo()
    rc = getattr(h.L, fn)(h.h, *args, None, cap, C.byref(n), C.byref(p), None, C.byref(info))
    return rc, n.value, p.value


def test_every_error_code():
    m = Modelled(universe(n_edges=400, seed=48), history=(3, 1 << 14), tiers=[(2, 2, 1 << 14, 1 << 12)])
    h = m.h
    cm = abi.metrics(abi.METRIC_COUNT)
    nodes = len(nr.keys(m.random_windows(5, seed=481)[-1]))
    ok = raw(h, WINDOW, IN, 0, 3, cm, 1)
    assert ok == (abi.E_CAPACITY, nodes, 3)
    assert raw(h, WINDOW, 2, 0, 3, cm, 1)[0] == abi.E_INVAL                                 # unknown side
    assert raw(h, WINDOW, IN, 0, 0, cm, 1)[0] == abi.E_INVAL                                # k = 0
    assert raw(h, WINDOW, IN, 2, 1, cm, 1)[0] == abi.E_INVAL                                # tier above the tiers
    assert raw(h, WINDOW, IN, 0, 1, cm, 0)[0] == abi.E_INVAL                                # nm = 0
    assert raw(h, WINDOW, IN, 0, 1, abi.metrics(*[abi.METRIC_COUNT] * 9), 9)[0] == abi.E_INVAL
    for q in (1.5, float("nan")):
        assert raw(h, WINDOW, IN, 0, 1, abi.metrics((Q, q)), 1)[0] == abi.E_INVAL
    assert raw(h, 3, IN, 0, 1, cm, 1)[0] == abi.E_INVAL                                     # unknown source
    assert raw(h, WINDOW, IN, 0, 1, None, 1)[0] == abi.E_INVAL                              # null metrics
    assert raw(h, WINDOW, IN, 0, 1, cm, 1, cap=5)[0] == abi.E_INVAL                         # null values with cap
    n, p_ = C.c_size_t(0), C.c_uint32(0)
    assert h.L.alz_node_series(h.h, WINDOW, IN, 0, 1, cm, 1, None, None, 0, None, None, None, None) == abi.E_INVAL
    assert h.L.alz_node_series(None, WINDOW, IN, 0, 1, cm, 1, None, None, 0, C.byref(n), C.byref(p_), None,
                               None) == abi.E_INVAL
    assert h.L.alz_node_series_device(h.h, WINDOW, IN, 0, 1, cm, 1, None, None, C.byref(n), C.byref(p_), None,
                                      None) == abi.E_INVAL                                  # null dev_values
    buf = np.zeros(64).ctypes.data_as(C.c_void_p)
    for bad in ((4, 1), (POD, 1 << 29), (SVC, 1 << 29)):
        e = capi.Handle.node_ends([(SVC, 2), bad])
        assert raw(h, e.ctypes.data_as(C.c_void_p), 2, IN, 0, 1, cm, 1, fn="alz_node_series_keys", cap=2,
                   out=buf)[0] == abi.E_INVAL, bad
        assert raw(h, e.ctypes.data_as(C.c_void_p), 2, IN, 0, 1, cm, 1, fn="alz_node_series_keys")[0] == \
            abi.E_INVAL, bad                                                                # before the cap of 0
    assert raw(h, None, 3, IN, 0, 1, cm, 1, fn="alz_node_series_keys")[0] == abi.E_INVAL    # null keys
    assert raw(h, None, 0, IN, 0, 1, cm, 1, fn="alz_node_series_keys")[:2] == (0, 0)        # no keys: fine
    # trends: k < 2, recent out of range, unknown stat / side, top = 0, NaN min_trend, null dev_out
    tr_ok = T(abi.TREND_SLOPE)
    assert raw_trends(h, WINDOW, IN, 0, 1, cm, C.byref(tr_ok))[0] == abi.E_INVAL
    assert raw_trends(h, WINDOW, IN, 0, 3, cm, C.byref(T(abi.TREND_SLOPE, recent=3)))[0] == abi.E_INVAL
    assert raw_trends(h, WINDOW, IN, 0, 3, cm, C.byref(T(4)))[0] == abi.E_INVAL
    assert raw_trends(h, WINDOW, 2, 0, 3, cm, C.byref(tr_ok))[0] == abi.E_INVAL
    assert raw_trends(h, WINDOW, IN, 0, 3, cm, C.byref(tr_ok))[:2] == (abi.E_CAPACITY, nodes)
    info = abi.TrendInfo()
    for top, mt in ((0, 0.0), (3, float("nan"))):
        assert h.L.alz_node_trends_top(h.h, WINDOW, IN, 0, 3, cm, C.byref(tr_ok), top, mt, None, None, None, None, 0,
                                       C.byref(n), C.byref(p_), None, C.byref(info)) == abi.E_INVAL
    assert h.L.alz_node_trends_device(h.h, WINDOW, IN, 0, 3, cm, C.byref(tr_ok), None, C.byref(n), C.byref(p_), None,
                                      None) == abi.E_INVAL
    # state: no rows of a rollup source; no tiers, no history
    for src in (WIN, TIER, SPAN):
        assert raw(h, src, IN, 0, 1, cm, 1)[0] == abi.E_STATE
        assert raw_trends(h, src, OUT, 0, 2, cm, C.byref(tr_ok))[0] == abi.E_STATE
    t = Modelled(universe(n_edges=200, seed=49), tiers=[(2, 2, 1 << 13, 1 << 12)])
    t.random_windows(2, seed=491)
    assert raw(t.h, WINDOW, IN, 0, 1, cm, 1)[0] == abi.E_STATE
    assert raw_trends(t.h, WINDOW, IN, 0, 2, cm, C.byref(tr_ok))[0] == abi.E_STATE
    t.close()
    w = Modelled(universe(n_edges=200, seed=50), history=(2, 1 << 13))
    w.random_windows(1, seed=501)
    assert raw(w.h, WINDOW, IN, 1, 1, cm, 1)[0] == abi.E_STATE
    w.close()
    # capacity: a cap below the nodes writes nothing but sets *n_out and *n_points
    vals = np.full((nodes, 2), 7.0)
    pres = np.full((nodes, 2), 9, np.uint8)
    pts = (abi.RollupInfo * 2)()
    rc = raw(h, WINDOW, OUT, 0, 2, cm, 1, out=vals.ctypes.data_as(C.c_void_p),
             present=pres.ctypes.data_as(C.c_void_p), cap=nodes - 1, points=pts)
    assert rc == (abi.E_CAPACITY, nodes, 2)
    assert np.all(vals == 7.0) and np.all(pres == 9) and pts[0].windows == 0
    m.close()


def test_more_than_2_30_slots_is_a_capacity_error():
    """64 points x 2^24 keys = 2^30 slots: the size is refused after the keys are checked and before they are sorted,
    copied to the device or matched against the entries."""
    h = capi.Handle(max_endpoints=64, max_pairs=1 << 12)
    try:
        h.window_history(64, 1 << 10)
        for _ in range(64):
            h.flush()
        big = np.zeros(1 << 24, dtype=abi.NODE_ENDS)
        cm = abi.metrics(abi.METRIC_COUNT)
        n, p_ = C.c_size_t(0), C.c_uint32(0)
        pv, pp = C.c_void_p(), C.c_void_p()
        rc = h.L.alz_node_series_keys_device(h.h, big.ctypes.data_as(C.c_void_p), len(big), IN, 0, 64, cm, 1,
                                             C.byref(pv), C.byref(pp), C.byref(n), C.byref(p_), None, None)
        assert (rc, n.value, p_.value) == (abi.E_CAPACITY, len(big), 64)
        rc = h.L.alz_node_series_keys_device(h.h, big.ctypes.data_as(C.c_void_p), len(big) - 1, IN, 0, 64, cm, 1,
                                             C.byref(pv), C.byref(pp), C.byref(n), C.byref(p_), None, None)
        assert (rc, n.value, p_.value) == (abi.OK, len(big) - 1, 64)   # 2^30 - 64 slots, every one absent
        assert not h.d2h(pp.value, 1 << 20, np.uint8).any()
    finally:
        h.close()


# ---- reads only ----------------------------------------------------------------------------------------------------

def test_reads_only_both_ways():
    m = Modelled(universe(seed=51), history=(5, 1 << 15), tiers=[(2, 3, 1 << 15, 1 << 13)])
    try:
        m.random_windows(8, seed=511, lo=0.2, hi=0.6)
        h = m.h
        h.rollup(3)
        h.baseline_pin(WIN)
        m.random_windows(2, seed=512)
        h.rollup_tier(1, 2)
        span_rows = h.rollup_span(5)[0]
        h.rollup(2)
        specs = [abi.METRIC_COUNT, (Q, 0.99), abi.METRIC_ERR_RATE]
        held = {kind: h.gnn_score_rollup(kind) for kind in (WIN, TIER, SPAN)}
        named = {src: h.node_rows(src)[:50] for src in (WINDOW, WIN, TIER, SPAN)}
        tn, tv, ti, tm, _ = h.node_top_device(TIER, OUT, (Q, 0.99), 9)   # the node family's last device results
        sv, spp, sn, sp_, _, _ = h.edge_series_device(WIN, 0, 4, *specs)
        trd, trn, _, _, _ = h.edge_trends_device(SPAN, 0, 4, (Q, 0.99), T(abi.TREND_SLOPE))
        ev, en = h.edge_metrics_rollup_device(TIER, *specs)
        gv, gn = h.gnn_score_rollup_device(WIN)

        def snapshot():
            return dict(ntop=h.d2h(tn, tm, abi.NODE_OUT), ntop_v=h.d2h(tv, tm, np.float64),
                        ntop_i=h.d2h(ti, tm, np.uint32), series=h.d2h(sv, sn * sp_ * len(specs), np.float64),
                        series_p=h.d2h(spp, sn * sp_, np.uint8), trends=h.d2h(trd, trn, abi.EDGE_TREND),
                        metrics=h.d2h(ev, en * len(specs), np.float64), gnn=h.d2h(gv, gn, np.float32),
                        stats={k: v for k, v in h.stats().items() if k != "kernel_launches"})

        before = snapshot()
        for src in (WINDOW, WIN, TIER, SPAN):
            for side in (IN, OUT):
                for tier in (0, 1):
                    h.node_series(src, side, tier, 9, *specs)
                    h.node_series_device(src, side, tier, 2, abi.METRIC_COUNT)
                    h.node_trends(src, side, tier, 3, (Q, 0.99), T(abi.TREND_SHIFT))
                    h.node_trends_top_device(src, side, tier, 3, abi.METRIC_COUNT, T(abi.TREND_SLOPE), 5)
            h.node_series_keys(named[src], IN, 0, 3, *specs)
        after = snapshot()
        assert before.pop("stats") == after.pop("stats")
        for k in before:
            assert np.asarray(before[k]).tobytes() == np.asarray(after[k]).tobytes(), k
        for kind in (WIN, TIER, SPAN):
            assert h.gnn_score_rollup(kind).tobytes() == held[kind].tobytes(), kind
        assert h.rollup_span(5)[0].tobytes() == span_rows.tobytes()
        # the other way: node series and node trend device results keep their bytes across the other families
        dv, dp, dn, dP, _, _ = h.node_series_device(SPAN, IN, 0, 4, *specs)
        ndv, ndn, _, _, _ = h.node_trends_device(SPAN, OUT, 0, 4, (Q, 0.99), T(abi.TREND_SLOPE))
        keep = (h.d2h(dv, dn * dP * len(specs), np.float64), h.d2h(dp, dn * dP, np.uint8),
                h.d2h(ndv, ndn, abi.NODE_TREND))
        for src in (WINDOW, SPAN):
            h.node_rows(src)
            h.node_metrics(src, IN, *specs)
            h.node_top(src, OUT, (Q, 0.5), 4)
            h.edge_series(src, 0, 3, *specs)
            h.edge_trends_top(src, 0, 3, abi.METRIC_COUNT, T(abi.TREND_SHIFT), 5)
            h.edge_metrics_rollup(SPAN, *specs)
        again = (h.d2h(dv, dn * dP * len(specs), np.float64), h.d2h(dp, dn * dP, np.uint8),
                 h.d2h(ndv, ndn, abi.NODE_TREND))
        assert all(x.tobytes() == y.tobytes() for x, y in zip(keep, again))
        # between the two families with their own states: a node series result across node trend calls, then a node
        # trend top result across node series calls
        for src in (WINDOW, SPAN):
            h.node_trends(src, IN, 0, 5, (Q, 0.99), T(abi.TREND_SHIFT, recent=2))
            h.node_trends_top(src, OUT, 1, 3, abi.METRIC_COUNT, T(abi.TREND_SLOPE), 7)
        assert h.d2h(dv, dn * dP * len(specs), np.float64).tobytes() == keep[0].tobytes()
        assert h.d2h(dp, dn * dP, np.uint8).tobytes() == keep[1].tobytes()
        pr, pn, ps, pq, tm2, tP, _, _ = h.node_trends_top_device(SPAN, IN, 0, 4, (Q, 0.99),
                                                                 T(abi.TREND_ZSCORE, recent=1), 20)

        def top_results():
            return (h.d2h(pr, tm2, abi.NODE_TREND), h.d2h(pn, tm2, abi.NODE_OUT), h.d2h(ps, tm2 * tP, np.float64),
                    h.d2h(pq, tm2 * tP, np.uint8))

        held_top = top_results()
        assert tm2 > 0
        for src in (WINDOW, WIN, TIER, SPAN):
            h.node_series(src, OUT, 0, 9, *specs)
            h.node_series_device(src, IN, 1, 3, abi.METRIC_COUNT)
            h.node_series_keys(named[src], IN, 1, 3, *specs)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(held_top, top_results()))
    finally:
        m.close()
