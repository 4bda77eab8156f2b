"""GPU: group series and group trends (alz_group_edge_series*, alz_group_node_series*, alz_group_*_series_keys*,
alz_group_edge_trends*, alz_group_node_trends*, docs/SPEC.md §26).

Values, presence, records, top order, top rows, points and info are compared as bytes against
tests/group_series_ref.py over the entries that tests/rollup_model.py and tests/tier_model.py say the rings retain,
each grouped by the map in force. Windows come from the Modelled stream of tests/test_gpu_edge_series.py."""
import ctypes as C

import numpy as np
import pytest

import group_ref as gr
import group_series_ref as gsr
import node_ref as nr
import node_series_ref as nsr
from alaz_b200 import abi, capi
from change_ref import row_keys
from test_gpu_edge_series import DEPTH, TIER_DEPTH, Modelled, make_source
from test_gpu_gnn_rollup import universe
from test_gpu_groups import ends, owners_map

pytestmark = pytest.mark.gpu
WINDOW, WIN, TIER, SPAN = abi.SOURCE_WINDOW, abi.ROLLUP_WINDOWS, abi.ROLLUP_TIER, abi.ROLLUP_SPAN
IN, OUT = abi.SIDE_IN, abi.SIDE_OUT
Q = abi.METRIC_QUANTILE
SPECS = ([abi.METRIC_COUNT], [(Q, 0.99)], [(Q, 0.5), (Q, 0.99), abi.METRIC_ERR_RATE])
STATS = [abi.TREND_SLOPE, abi.TREND_SHIFT, abi.TREND_RATIO, abi.TREND_ZSCORE]
T = capi.Handle.trend
POD, SVC, OUTB, HOST, GRP = 0, 1, 2, 3, abi.NODE_GROUP


def namespaces_map(rows):
    """pods and services into 100 namespaces by id, outbound ends to one external group"""
    keys = nr.keys(rows)
    t, v = keys >> np.uint64(32), keys & np.uint64(0xFFFFFFFF)
    g = np.where(t <= SVC, v % 100, 1 << 20).astype(np.uint32)
    return ends(keys), g


MAPS = ("empty", "owners", "namespaces")


def use_map(m, which):
    """set the map `which` over every node the stream's universe can produce; the reference form of it"""
    if which == "empty":
        m.h.group_set(np.zeros(0, abi.NODE_ENDS), np.zeros(0, np.uint32))
        return gr.EMPTY
    rows = np.concatenate([e for e in m.entries(0)[0]] + [e for e in m.entries(1)[0]] + [m.last])
    nodes, groups = (owners_map if which == "owners" else namespaces_map)(rows)
    m.h.group_set(nodes, groups)
    return gr.make_map(nodes, groups)


@pytest.fixture(scope="module")
def mod():
    m = Modelled(universe(seed=64), history=(DEPTH, 1 << 15), tiers=[(2, TIER_DEPTH, 1 << 15, 1 << 13)])
    m.random_windows(12, seed=641, lo=0.2, hi=0.7)
    m.last = m.window(np.flatnonzero(np.random.default_rng(642).random(m.s.g.n_edges) < 0.5))
    assert len(m.rm.entries) == DEPTH and len(m.tm.tiers[0].ring.entries) == TIER_DEPTH
    yield m
    m.close()


def take_of(m, tier, k):
    ents, pts = m.entries(tier)
    take = pts[max(len(pts) - k, 0):]
    return ents, take, sum(x["rows_in"] for x in take)


def same(got, want, take, rows_in, what):
    v, p, pts, info = got
    wv, wp = want
    assert v.shape == wv.shape and p.shape == wp.shape, (what, v.shape, wv.shape)
    assert p.tobytes() == wp.tobytes(), (what, np.argwhere(p != wp)[:5])
    assert v.tobytes() == wv.tobytes(), (what, np.argwhere(v.view(np.uint64) != wv.view(np.uint64))[:5])
    assert pts == take, (what, pts, take)
    assert info["points"] == len(take) and info["edges"] == len(p) and info["rows_in"] == rows_in, (what, info)


def same_device(h, got, dev, nm, what):
    v, p, pts, info = got
    pv, pp, n, P, dpts, dinfo = dev
    assert (n, P, dpts, dinfo) == (v.shape[0], v.shape[1], pts, info), what
    assert h.d2h(pv, n * P * nm, np.float64).tobytes() == v.tobytes(), what
    assert h.d2h(pp, n * P, np.uint8).tobytes() == p.tobytes(), what


# ---- series ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("which", MAPS)
@pytest.mark.parametrize("tier", [0, 1])
@pytest.mark.parametrize("source", [WINDOW, WIN, TIER, SPAN])
def test_every_source_ring_map_side_and_metric_set(mod, source, tier, which):
    h = mod.h
    gmap = use_map(mod, which)
    rows = make_source(mod, source)
    ge = gsr.source_edges(rows, gmap)
    gkeys = nr.keys(ge)
    assert h.group_edges(source)[0].tobytes() == ge.tobytes()
    depth = DEPTH if tier == 0 else TIER_DEPTH
    present_some = absent_some = False
    for k in (1, 3, depth + 5):
        ents, take, rows_in = take_of(mod, tier, k)
        for specs in SPECS:
            got = h.group_edge_series(source, tier, k, *specs)
            same(got, gsr.edge_series(ents, *gsr.row_ends(ge), specs, gmap, k), take, rows_in,
                 ("edges", source, tier, which, k, specs))
            for side in (IN, OUT):
                got = h.group_node_series(source, side, tier, k, *specs)
                same(got, gsr.node_series(ents, gkeys, side, specs, gmap, k), take, rows_in,
                     ("nodes", source, tier, which, side, k, specs))
                present_some |= bool(got[1].any())
                absent_some |= not got[1].all()
    specs = SPECS[2]
    same_device(h, h.group_edge_series(source, tier, 3, *specs), h.group_edge_series_device(source, tier, 3, *specs),
                len(specs), ("edges device", source, tier, which))
    for side in (IN, OUT):
        same_device(h, h.group_node_series(source, side, tier, 3, *specs),
                    h.group_node_series_device(source, side, tier, 3, *specs), len(specs),
                    ("nodes device", source, tier, which, side))
    assert present_some and absent_some


@pytest.mark.parametrize("tier", [0, 1])
def test_caller_keys_host_and_device(mod, tier):
    h = mod.h
    gmap = use_map(mod, "owners")
    rng = np.random.default_rng(tier)
    ents = mod.entries(tier)[0]
    seen = nr.keys(np.concatenate([gr.group(e, gmap)[0] for e in ents]))
    pick = [(int(k >> np.uint64(32)), int(k & np.uint64(0xFFFFFFFF))) for k in seen[rng.choice(len(seen), 150,
                                                                                                  replace=False)]]
    mapped = [(int(t), int(v)) for t, v in zip(*[x.astype(np.int64) for x in (np.asarray(
        gmap[0] >> np.uint64(32)), np.asarray(gmap[0] & np.uint64(0xFFFFFFFF)))])][:20]   # pods the map holds
    nodes = pick + pick[:7] + mapped + [(GRP, 0), (GRP, (1 << 29) - 1), (SVC, (1 << 29) - 1), (OUTB, 0xFFFFFFFF)]
    ne = capi.Handle.node_ends(nodes)
    nkeys = gsr.node_ends_keys(ne)
    ge = np.concatenate([gr.group(e, gmap)[0] for e in ents])
    sel = ge[rng.choice(len(ge), 150, replace=False)]
    edges = [(int(r["from_type"]), int(r["from"]), int(r["to_type"]), int(r["to"])) for r in sel]
    edges += edges[:5] + [(POD, int(v), SVC, 3) for _, v in mapped[:5]] + [(GRP, 1, GRP, 1), (GRP, 7, OUTB, 9)]
    ee = capi.Handle.edge_ends(edges)
    kf, kt = gsr.edge_ends_keys(ee)
    for k in (1, 3, 50):
        ents_k, take, rows_in = take_of(mod, tier, k)
        for specs in SPECS:
            got = h.group_edge_series_keys(ee, tier, k, *specs)
            same(got, gsr.edge_series(ents_k, kf, kt, specs, gmap, k), take, rows_in, ("edge keys", tier, k, specs))
            for side in (IN, OUT):
                got_n = h.group_node_series_keys(ne, side, tier, k, *specs)
                same(got_n, gsr.node_series(ents_k, nkeys, side, specs, gmap, k), take, rows_in,
                     ("node keys", tier, side, k, specs))
        same_device(h, got, h.group_edge_series_keys_device(ee, tier, k, *specs), len(specs), ("edge keys dev", k))
        same_device(h, got_n, h.group_node_series_keys_device(ne, OUT, tier, k, *specs), len(specs),
                    ("node keys dev", k))
    v, p, _, _ = h.group_node_series_keys(ne, OUT, tier, 50, *SPECS[2])
    assert v[:7].tobytes() == v[150:157].tobytes() and p[:7].tobytes() == p[150:157].tobytes()
    assert not p[157:177].any() and not v[157:177].any()        # mapped pods: absent everywhere
    v, p, _, _ = h.group_edge_series_keys(ee, tier, 50, *SPECS[2])
    assert v[:5].tobytes() == v[150:155].tobytes() and not p[155:160].any()


@pytest.mark.parametrize("tier", [0, 1])
def test_empty_map_equals_node_and_edge_series(mod, tier):
    h = mod.h
    use_map(mod, "empty")
    for source in (WINDOW, SPAN):
        rows = make_source(mod, source)
        specs = SPECS[2]
        for side in (IN, OUT):
            a, b = h.group_node_series(source, side, tier, 4, *specs), h.node_series(source, side, tier, 4, *specs)
            assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes() and a[2:] == b[2:]
            da = h.group_node_series_device(source, side, tier, 4, *specs)
            assert h.d2h(da[0], da[2] * da[3] * 3, np.float64).tobytes() == b[0].tobytes()
        ge = h.group_edges(source)[0]
        perm = np.argsort(row_keys(ge), kind="stable")      # §24 order -> packed-key order
        assert row_keys(ge)[perm].tobytes() == row_keys(rows).tobytes()
        a, b = h.group_edge_series(source, tier, 4, *specs), h.edge_series(source, tier, 4, *specs)
        assert a[0][perm].tobytes() == b[0].tobytes() and a[1][perm].tobytes() == b[1].tobytes() and a[2:] == b[2:]


@pytest.mark.parametrize("which", MAPS)
@pytest.mark.parametrize("tier", [0, 1])
def test_newest_point_is_the_k1_rollup_group_metrics(mod, tier, which):
    h = mod.h
    use_map(mod, which)
    kind = WIN if tier == 0 else TIER
    (h.rollup if tier == 0 else (lambda k: h.rollup_tier(1, k)))(1)
    specs = [abi.METRIC_COUNT, abi.METRIC_ERR_RATE, (Q, 0.5), (Q, 0.99), abi.METRIC_MEAN_NS]
    ge = h.group_edges(kind)[0]
    v, p, _, _ = h.group_edge_series_keys(ge, tier, 3, *specs)
    assert p[:, -1].all() and v[:, -1, :].tobytes() == h.group_edge_metrics(kind, *specs).tobytes()
    v, p, _, _ = h.group_edge_series(kind, tier, 1, *specs)
    assert p.all() and v[:, 0, :].tobytes() == h.group_edge_metrics(kind, *specs).tobytes()
    nodes = h.group_nodes(kind)
    for side in (IN, OUT):
        want = h.group_node_metrics(kind, side, *specs)
        on = nodes["in_edges" if side == IN else "out_edges"] > 0
        v, p, _, _ = h.group_node_series_keys(nodes, side, tier, 3, *specs)
        assert p[:, -1].tobytes() == on.astype(np.uint8).tobytes()
        assert v[on, -1, :].tobytes() == want[on].tobytes() and not v[~on, -1, :].any()
        v, p, _, _ = h.group_node_series(kind, side, tier, 1, *specs)
        assert v[on, 0, :].tobytes() == want[on].tobytes()


def test_rolling_deploy_through_the_stream():
    """window j carries the edges of pods with id % 4 == j % 4; deployment d holds pods 8d .. 8d + 7, so every
    deployment is present at every point while each pod is present at every fourth"""
    m = Modelled(universe(n_pods=400, n_svcs=20, n_edges=3000, seed=65), history=(8, 1 << 15))
    try:
        g = m.s.g
        pod_of = np.where(g.ft == POD, g.fv, g.tv)
        for j in range(8):
            m.window(np.flatnonzero(pod_of % 4 == j % 4))
        ents = m.entries(0)[0]
        pods = np.unique(nr.keys(np.concatenate(ents)))
        pods = pods[(pods >> np.uint64(32)) == POD]
        pv = (pods & np.uint64(0xFFFFFFFF)).astype(np.uint32)
        m.h.group_set(ends(pods), (pv // 8).astype(np.uint32))
        gmap = gr.make_map(ends(pods), (pv // 8).astype(np.uint32))
        for side in (IN, OUT):
            got = m.h.group_node_series(WINDOW, side, 0, 8, abi.METRIC_COUNT, (Q, 0.99))
            _, take, rows_in = take_of(m, 0, 8)
            want = gsr.node_series(ents, nr.keys(gsr.source_edges(ents[-1], gmap)), side,
                                   [abi.METRIC_COUNT, (Q, 0.99)], gmap, 8)
            same(got, want, take, rows_in, ("rolling", side))
        v, p, _, _ = m.h.group_node_series_keys(capi.Handle.node_ends([(GRP, d) for d in range(10)]), OUT, 0, 8,
                                                abi.METRIC_COUNT)
        assert p.all()                                   # every deployment in every window
        for j, e in enumerate(ents):                     # with its members' summed counts
            for d in range(10):
                mine = (e["from_type"] == POD) & (e["from"] // 8 == d)
                assert v[d, j, 0] == float(e["count"][mine].sum())
        v, p, _, _ = m.h.node_series_keys(capi.Handle.node_ends([(POD, int(x)) for x in pv[:40]]), OUT, 0, 8,
                                          abi.METRIC_COUNT)
        assert not p.all(axis=1).any() and p.any()       # no pod in every window
    finally:
        m.close()


def test_hub_group_of_thousands_of_pods_in_every_window():
    m = Modelled(universe(n_pods=6000, n_svcs=1, n_edges=12000, seed=66), history=(4, 1 << 16))
    try:
        m.random_windows(5, seed=661, lo=0.6, hi=0.8)
        rows = m.h.rollup(4)[0]
        keys = nr.keys(rows)
        pods = keys[(keys >> np.uint64(32)) == POD]
        m.h.group_set(ends(pods), np.zeros(len(pods), np.uint32))      # every pod into group 0
        gmap = gr.make_map(ends(pods), np.zeros(len(pods), np.uint32))
        ents, take, rows_in = take_of(m, 0, 4)
        for e in ents:
            assert len(np.unique(e["from"][e["from_type"] == POD])) >= 1000
        ge = gsr.source_edges(rows, gmap)
        for specs in SPECS:
            same(m.h.group_edge_series(WIN, 0, 4, *specs), gsr.edge_series(ents, *gsr.row_ends(ge), specs, gmap, 4),
                 take, rows_in, ("hub edges", specs))
            for side in (IN, OUT):
                same(m.h.group_node_series(WIN, side, 0, 4, *specs),
                     gsr.node_series(ents, nr.keys(ge), side, specs, gmap, 4), take, rows_in, ("hub", side, specs))
        v, p, _, _ = m.h.group_node_series_keys(capi.Handle.node_ends([(GRP, 0)]), OUT, 0, 4, abi.METRIC_COUNT)
        assert p.all() and (v[0, :, 0] > 1000).all()
    finally:
        m.close()


# ---- trends ----------------------------------------------------------------------------------------------------------

def spec_of(t):
    return dict(stat=t.stat, direction=t.direction, absent=t.absent, recent=t.recent, min_points=t.min_points)


def check_trends(m, rows, gmap, source, nodes, side, tier, k, spec, t, top=None, min_trend=-np.inf, what=None):
    """the full list and the top call of the group edge or node trends against the reference, as bytes"""
    h = m.h
    what = what or (source, nodes, side, tier, k, spec, spec_of(t))
    ents, take, rows_in = take_of(m, tier, k)
    if nodes:
        rec, y, p = gsr.node_expect(ents, rows, side, spec, k, gmap, **spec_of(t))
        srows = gsr.source_nodes(rows, gmap)
        got, gpts, ginfo = h.group_node_trends(source, side, tier, k, spec, t)
    else:
        rec, y, p = gsr.edge_expect(ents, rows, spec, k, gmap, **spec_of(t))
        srows = gsr.source_edges(rows, gmap)
        got, gpts, ginfo = h.group_edge_trends(source, tier, k, spec, t)
    info = dict(edges=len(srows), rows_in=rows_in, valid=int(rec["valid"].sum()), above=0, points=len(take),
                tier=tier)
    assert got.tobytes() == rec.tobytes(), what
    assert gpts == take and ginfo == info, (what, ginfo, info)
    top = top or max(len(srows) // 4, 1)
    idx, above = gsr.top(rec, top, min_trend)
    if nodes:
        trec, trows, ts, tp, tpts, tinfo = h.group_node_trends_top(source, side, tier, k, spec, t, top, min_trend)
    else:
        trec, trows, ts, tp, tpts, tinfo = h.group_edge_trends_top(source, tier, k, spec, t, top, min_trend)
    assert trec.tobytes() == rec[idx].tobytes(), (what, trec["index"][:8], idx[:8])
    assert trows.tobytes() == srows[idx].tobytes(), what
    assert ts.tobytes() == y[idx].tobytes() and tp.tobytes() == p[idx].tobytes(), what
    assert tpts == take and tinfo == dict(info, above=above), (what, tinfo)
    return rec, idx


@pytest.mark.parametrize("which", ["owners", "namespaces"])
@pytest.mark.parametrize("source", [WINDOW, SPAN])
def test_trends_every_stat_direction_and_absent_mode(mod, source, which):
    gmap = use_map(mod, which)
    rows = make_source(mod, source)
    valid = 0
    for stat in STATS:
        for direction in (abi.TREND_RISING, abi.TREND_FALLING):
            for absent in (abi.TREND_ABSENT_SKIP, abi.TREND_ABSENT_ZERO):
                for nodes, side, tier, k, r, spec in ((False, IN, 0, DEPTH, 1, (Q, 0.99)),
                                                      (True, IN, 0, 3, 2, abi.METRIC_COUNT),
                                                      (True, OUT, 1, TIER_DEPTH + 2, 1, abi.METRIC_ERR_RATE)):
                    rec, _ = check_trends(mod, rows, gmap, source, nodes, side, tier, k, spec,
                                          T(stat, direction, absent, r))
                    valid += int(rec["valid"].sum())
    assert valid > 0


def test_trend_cuts_infinities_and_index_ties(mod):
    gmap = use_map(mod, "owners")
    rows = mod.last
    t = T(abi.TREND_SHIFT, recent=2)
    for nodes in (False, True):
        rec, _, _ = (gsr.node_expect(mod.entries(0)[0], rows, IN, (Q, 0.99), DEPTH, gmap, **spec_of(t)) if nodes else
                     gsr.edge_expect(mod.entries(0)[0], rows, (Q, 0.99), DEPTH, gmap, **spec_of(t)))
        vals = np.sort(rec["trend"][rec["valid"] == 1])
        n = len(rec)
        for cut in (vals[len(vals) // 2], vals[-1], vals[-1] + 1.0, 0.0, -0.0, -np.inf, np.inf):
            _, idx = check_trends(mod, rows, gmap, WINDOW, nodes, IN, 0, DEPTH, (Q, 0.99), t, top=n, min_trend=cut,
                                  what=(nodes, cut))
            assert np.all(rec["trend"][idx] >= cut)
        rec, idx = check_trends(mod, rows, gmap, WINDOW, nodes, OUT, 0, 3, abi.METRIC_COUNT,
                                T(abi.TREND_RATIO, absent=abi.TREND_ABSENT_ZERO, recent=1), top=n)
        inf = np.flatnonzero(rec["trend"] == np.inf)
        assert idx[: len(inf)].tolist() == inf.tolist()     # +inf first, in index order


@pytest.mark.parametrize("tier", [0, 1])
def test_trend_top_series_are_group_series_and_device_equals_host(mod, tier):
    h = mod.h
    use_map(mod, "namespaces")
    t = T(abi.TREND_ZSCORE, recent=1)
    spec = (Q, 0.99)
    k = DEPTH if tier == 0 else TIER_DEPTH
    trec, tn, ts, tp, tpts, tinfo = h.group_node_trends_top(SPAN, IN, tier, k, spec, t, 40)
    sv, sp, spts, _ = h.group_node_series(SPAN, IN, tier, k, spec)
    assert len(trec) > 0 and tpts == spts
    assert ts.tobytes() == sv[trec["index"], :, 0].tobytes() and tp.tobytes() == sp[trec["index"]].tobytes()
    assert tn.tobytes() == h.group_nodes(SPAN)[trec["index"]].tobytes()
    got, pts, info = h.group_node_trends(SPAN, IN, tier, k, spec, t)
    d, n, P, dpts, dinfo = h.group_node_trends_device(SPAN, IN, tier, k, spec, t)
    assert (n, P, dpts, dinfo) == (len(got), len(pts), pts, info)
    assert h.d2h(d, n, abi.NODE_TREND).tobytes() == got.tobytes()
    pr, pn, ps, pp, m, P, dpts, dinfo = h.group_node_trends_top_device(SPAN, IN, tier, k, spec, t, 40)
    assert (m, P, dpts, dinfo) == (len(trec), len(tpts), tpts, tinfo)
    assert h.d2h(pr, m, abi.NODE_TREND).tobytes() == trec.tobytes()
    assert h.d2h(pn, m, abi.NODE_OUT).tobytes() == tn.tobytes()
    assert h.d2h(ps, m * P, np.float64).tobytes() == ts.tobytes() and h.d2h(pp, m * P, np.uint8).tobytes() == tp.tobytes()
    erec, er, es, ep, epts, einfo = h.group_edge_trends_top(SPAN, tier, k, spec, t, 40)
    ev, epr, _, _ = h.group_edge_series(SPAN, tier, k, spec)
    assert len(erec) > 0 and es.tobytes() == ev[erec["index"], :, 0].tobytes()
    assert ep.tobytes() == epr[erec["index"]].tobytes()
    assert er.tobytes() == h.group_edges(SPAN)[0][erec["index"]].tobytes()
    assert (erec["from_type"] == GRP).any()
    got, pts, info = h.group_edge_trends(SPAN, tier, k, spec, t)
    d, n, P, dpts, dinfo = h.group_edge_trends_device(SPAN, tier, k, spec, t)
    assert (n, dpts, dinfo) == (len(got), pts, info) and h.d2h(d, n, abi.EDGE_TREND).tobytes() == got.tobytes()
    pr, pw, ps, pp, m, P, dpts, dinfo = h.group_edge_trends_top_device(SPAN, tier, k, spec, t, 40)
    assert (m, dpts, dinfo) == (len(erec), epts, einfo)
    assert h.d2h(pr, m, abi.EDGE_TREND).tobytes() == erec.tobytes()
    assert h.d2h(pw, m, abi.EDGE_OUT).tobytes() == er.tobytes()
    assert h.d2h(ps, m * P, np.float64).tobytes() == es.tobytes() and h.d2h(pp, m * P, np.uint8).tobytes() == ep.tobytes()


# ---- errors ------------------------------------------------------------------------------------------------------

def raw(h, *args, fn="alz_group_node_series", out=None, present=None, cap=0, points=None):
    n, p, info = C.c_size_t(777), C.c_uint32(777), abi.SeriesInfo()
    rc = getattr(h.L, fn)(h.h, *args, out, present, cap, C.byref(n), C.byref(p), points, C.byref(info))
    return rc, n.value, p.value


def raw_trends(h, *args, fn="alz_group_node_trends", cap=0):
    n, p, info = C.c_size_t(777), C.c_uint32(777), abi.TrendInfo()
    rc = getattr(h.L, fn)(h.h, *args, None, cap, C.byref(n), C.byref(p), None, C.byref(info))
    return rc, n.value, p.value


def test_every_error_code():
    m = Modelled(universe(n_edges=400, seed=68), history=(3, 1 << 14), tiers=[(2, 2, 1 << 14, 1 << 12)])
    h = m.h
    cm = abi.metrics(abi.METRIC_COUNT)
    last = m.random_windows(5, seed=681)[-1]
    nodes, groups = owners_map(last)
    h.group_set(nodes, groups)
    gmap = gr.make_map(nodes, groups)
    n_nodes, n_edges = len(gsr.source_nodes(last, gmap)), len(gsr.source_edges(last, gmap))
    assert raw(h, WINDOW, IN, 0, 3, cm, 1) == (abi.E_CAPACITY, n_nodes, 3)
    assert raw(h, WINDOW, 0, 3, cm, 1, fn="alz_group_edge_series") == (abi.E_CAPACITY, n_edges, 3)
    assert raw(h, WINDOW, 2, 0, 3, cm, 1)[0] == abi.E_INVAL                                 # unknown side
    assert raw(h, WINDOW, IN, 0, 0, cm, 1) == (abi.E_INVAL, 0, 0)                           # k = 0
    assert raw(h, WINDOW, IN, 2, 1, cm, 1)[0] == abi.E_INVAL                                # tier above the tiers
    assert raw(h, WINDOW, IN, 0, 1, cm, 0)[0] == abi.E_INVAL                                # nm = 0
    assert raw(h, WINDOW, IN, 0, 1, abi.metrics((Q, 1.5)), 1)[0] == abi.E_INVAL
    assert raw(h, 3, IN, 0, 1, cm, 1)[0] == abi.E_INVAL                                     # unknown source
    assert raw(h, 3, 0, 1, cm, 1, fn="alz_group_edge_series")[0] == abi.E_INVAL
    assert raw(h, WINDOW, IN, 0, 1, cm, 1, cap=5)[0] == abi.E_INVAL                         # null values with cap
    n, p_ = C.c_size_t(0), C.c_uint32(0)
    assert h.L.alz_group_node_series(h.h, WINDOW, IN, 0, 1, cm, 1, None, None, 0, None, None, None, None) == abi.E_INVAL
    assert h.L.alz_group_edge_series_device(h.h, WINDOW, 0, 1, cm, 1, None, None, C.byref(n), C.byref(p_), None,
                                            None) == abi.E_INVAL                            # null dev_values
    buf = np.zeros(64).ctypes.data_as(C.c_void_p)
    for bad in ((5, 1), (GRP, 1 << 29), (POD, 1 << 29), (SVC, 1 << 29)):
        e = capi.Handle.node_ends([(SVC, 2), bad])
        assert raw(h, e.ctypes.data_as(C.c_void_p), 2, IN, 0, 1, cm, 1, fn="alz_group_node_series_keys", cap=2,
                   out=buf)[0] == abi.E_INVAL, bad
        assert raw(h, e.ctypes.data_as(C.c_void_p), 2, IN, 0, 1, cm, 1, fn="alz_group_node_series_keys")[0] == \
            abi.E_INVAL, bad                                                                # before the cap of 0
    for bad in ((SVC, 1, OUTB, 2), (GRP, 1 << 29, SVC, 1), (GRP, 1, 5, 1), (POD, 1 << 29, SVC, 1)):
        e = capi.Handle.edge_ends([(POD, 1, SVC, 2), bad])
        assert raw(h, e.ctypes.data_as(C.c_void_p), 2, 0, 1, cm, 1, fn="alz_group_edge_series_keys")[0] == \
            abi.E_INVAL, bad
    ok = capi.Handle.edge_ends([(GRP, 1, OUTB, 2), (GRP, 3, GRP, 3)])
    assert raw(h, ok.ctypes.data_as(C.c_void_p), 2, 0, 1, cm, 1, fn="alz_group_edge_series_keys") == \
        (abi.E_CAPACITY, 2, 1)
    assert raw(h, None, 3, IN, 0, 1, cm, 1, fn="alz_group_node_series_keys")[0] == abi.E_INVAL   # null keys
    assert raw(h, None, 0, 0, 1, cm, 1, fn="alz_group_edge_series_keys")[:2] == (0, 0)           # no keys: fine
    tr_ok = T(abi.TREND_SLOPE)
    assert raw_trends(h, WINDOW, IN, 0, 1, cm, C.byref(tr_ok))[0] == abi.E_INVAL             # k < 2
    assert raw_trends(h, WINDOW, IN, 0, 3, cm, C.byref(T(abi.TREND_SLOPE, recent=3)))[0] == abi.E_INVAL
    assert raw_trends(h, WINDOW, 2, 0, 3, cm, C.byref(tr_ok))[0] == abi.E_INVAL
    assert raw_trends(h, WINDOW, IN, 0, 3, cm, C.byref(tr_ok))[:2] == (abi.E_CAPACITY, n_nodes)
    assert raw_trends(h, WINDOW, 0, 3, cm, C.byref(tr_ok), fn="alz_group_edge_trends")[:2] == (abi.E_CAPACITY, n_edges)
    info = abi.TrendInfo()
    for top, mt in ((0, 0.0), (3, float("nan"))):
        assert h.L.alz_group_node_trends_top(h.h, WINDOW, IN, 0, 3, cm, C.byref(tr_ok), top, mt, None, None, None,
                                             None, 0, C.byref(n), C.byref(p_), None, C.byref(info)) == abi.E_INVAL
        assert h.L.alz_group_edge_trends_top(h.h, WINDOW, 0, 3, cm, C.byref(tr_ok), top, mt, None, None, None,
                                             None, 0, C.byref(n), C.byref(p_), None, C.byref(info)) == abi.E_INVAL
    for src in (WIN, TIER, SPAN):
        assert raw(h, src, IN, 0, 1, cm, 1)[0] == abi.E_STATE
        assert raw(h, src, 0, 1, cm, 1, fn="alz_group_edge_series")[0] == abi.E_STATE
        assert raw_trends(h, src, 0, 2, cm, C.byref(tr_ok), fn="alz_group_edge_trends")[0] == abi.E_STATE
    t = Modelled(universe(n_edges=200, seed=69), tiers=[(2, 2, 1 << 13, 1 << 12)])
    t.random_windows(2, seed=691)
    assert raw(t.h, WINDOW, IN, 0, 1, cm, 1)[0] == abi.E_STATE                              # no window history
    assert raw(t.h, WINDOW, 0, 1, cm, 1, fn="alz_group_edge_series")[0] == abi.E_STATE
    t.close()
    vals = np.full((n_nodes, 2), 7.0)
    pres = np.full((n_nodes, 2), 9, np.uint8)
    pts = (abi.RollupInfo * 2)()
    rc = raw(h, WINDOW, OUT, 0, 2, cm, 1, out=vals.ctypes.data_as(C.c_void_p),
             present=pres.ctypes.data_as(C.c_void_p), cap=n_nodes - 1, points=pts)
    assert rc == (abi.E_CAPACITY, n_nodes, 2)
    assert np.all(vals == 7.0) and np.all(pres == 9) and pts[0].windows == 0
    m.close()


def test_more_than_2_30_slots_is_a_capacity_error():
    """64 points x 2^24 keys = 2^30 slots: refused after the keys are checked and before they are sorted"""
    h = capi.Handle(max_endpoints=64, max_pairs=1 << 12)
    try:
        h.window_history(64, 1 << 10)
        for _ in range(64):
            h.flush()
        cm = abi.metrics(abi.METRIC_COUNT)
        n, p_ = C.c_size_t(0), C.c_uint32(0)
        pv, pp = C.c_void_p(), C.c_void_p()
        big = np.zeros(1 << 24, dtype=abi.NODE_ENDS)
        big["type"] = GRP
        for fn, arr in (("alz_group_node_series_keys_device", big),):
            rc = getattr(h.L, fn)(h.h, arr.ctypes.data_as(C.c_void_p), len(arr), IN, 0, 64, cm, 1, C.byref(pv),
                                  C.byref(pp), C.byref(n), C.byref(p_), None, None)
            assert (rc, n.value, p_.value) == (abi.E_CAPACITY, len(arr), 64)
        edges = np.zeros(1 << 24, dtype=abi.EDGE_ENDS)
        edges["from_type"], edges["to_type"] = GRP, GRP
        rc = h.L.alz_group_edge_series_keys_device(h.h, edges.ctypes.data_as(C.c_void_p), len(edges), 0, 64, cm, 1,
                                                   C.byref(pv), C.byref(pp), C.byref(n), C.byref(p_), None, None)
        assert (rc, n.value, p_.value) == (abi.E_CAPACITY, len(edges), 64)
        rc = h.L.alz_group_edge_series_keys_device(h.h, edges.ctypes.data_as(C.c_void_p), len(edges) - 1, 0, 64, cm,
                                                   1, C.byref(pv), C.byref(pp), C.byref(n), C.byref(p_), None, None)
        assert (rc, n.value, p_.value) == (abi.OK, len(edges) - 1, 64)
        assert not h.d2h(pp.value, 1 << 20, np.uint8).any()
    finally:
        h.close()


# ---- reads only ----------------------------------------------------------------------------------------------------

def test_reads_only_both_ways():
    m = Modelled(universe(seed=71), history=(5, 1 << 15), tiers=[(2, 3, 1 << 15, 1 << 13)])
    try:
        m.random_windows(8, seed=711, lo=0.2, hi=0.6)
        h = m.h
        m.last = m.window(np.flatnonzero(np.random.default_rng(712).random(m.s.g.n_edges) < 0.5))
        nodes, groups = owners_map(np.concatenate(m.entries(0)[0] + m.entries(1)[0]))
        h.group_set(nodes, groups)
        h.rollup(3)
        h.baseline_pin(WIN)
        h.rollup_tier(1, 2)
        span_rows = h.rollup_span(5)[0]
        specs = [abi.METRIC_COUNT, (Q, 0.99), abi.METRIC_ERR_RATE]
        named = {src: h.group_nodes(src)[:50] for src in (WINDOW, WIN, TIER, SPAN)}   # before the results held below
        # the group family's device results: node rows, top, edge metrics and edge rows all of TIER, so that each call
        # leaves the earlier ones' buffers and bytes as they were
        gn_p, gn_n = h.group_nodes_device(TIER)
        gt = h.group_node_top_device(TIER, OUT, (Q, 0.99), 9)
        gm_p, gm_n = h.group_edge_metrics_device(TIER, *specs)
        ge_p, ge_n, _ = h.group_edges_device(TIER)
        gc_p, gc_n, _ = h.group_edge_changes_device((Q, 0.99), source=SPAN)
        nv, npp, nn, nP, _, _ = h.node_series_device(WIN, IN, 0, 4, *specs)
        trd, trn, _, _, _ = h.node_trends_device(SPAN, OUT, 0, 4, (Q, 0.99), T(abi.TREND_SLOPE))
        sv, spp, sn, sP, _, _ = h.edge_series_device(WIN, 0, 4, *specs)
        held_gnn = h.gnn_score_rollup(SPAN)

        def snapshot():
            return dict(gn=h.d2h(gn_p, gn_n, abi.NODE_OUT), gm=h.d2h(gm_p, gm_n * 3, np.float64),
                        ge=h.d2h(ge_p, ge_n, abi.EDGE_OUT), gt=h.d2h(gt[0], gt[3], abi.NODE_OUT),
                        gt_v=h.d2h(gt[1], gt[3], np.float64),
                        gt_i=h.d2h(gt[2], gt[3], np.uint32),
                        gc=h.d2h(gc_p, gc_n, abi.EDGE_CHANGE), ns=h.d2h(nv, nn * nP * 3, np.float64),
                        nsp=h.d2h(npp, nn * nP, np.uint8), nt=h.d2h(trd, trn, abi.NODE_TREND),
                        es=h.d2h(sv, sn * sP * 3, np.float64), esp=h.d2h(spp, sn * sP, np.uint8),
                        stats={k: v for k, v in h.stats().items() if k != "kernel_launches"})

        before = snapshot()
        cached = h.group_edge_changes((Q, 0.99), source=SPAN)

        def launches_of(call):
            n0 = h.stats()["kernel_launches"]
            call()
            return h.stats()["kernel_launches"] - n0

        cached_launches = launches_of(lambda: h.group_edge_changes_device((Q, 0.99), source=SPAN))
        for src in (WINDOW, WIN, TIER, SPAN):
            for tier in (0, 1):
                h.group_edge_series(src, tier, 9, *specs)
                h.group_edge_trends_top_device(src, tier, 3, abi.METRIC_COUNT, T(abi.TREND_SLOPE), 5)
                for side in (IN, OUT):
                    h.group_node_series(src, side, tier, 9, *specs)
                    h.group_node_series_device(src, side, tier, 2, abi.METRIC_COUNT)
                    h.group_node_trends(src, side, tier, 3, (Q, 0.99), T(abi.TREND_SHIFT))
            h.group_node_series_keys(named[src], IN, 0, 3, *specs)
        after = snapshot()
        assert before.pop("stats") == after.pop("stats")
        for k in before:
            assert np.asarray(before[k]).tobytes() == np.asarray(after[k]).tobytes(), k
        assert h.group_edges_device(TIER)[0] == ge_p and h.group_nodes_device(TIER)[0] == gn_p
        # the baseline's cached groups are used as they were, not grouped again: the same launches as before
        assert launches_of(lambda: h.group_edge_changes_device((Q, 0.99), source=SPAN)) == cached_launches
        assert h.group_edge_changes((Q, 0.99), source=SPAN)[0].tobytes() == cached[0].tobytes()
        assert h.gnn_score_rollup(SPAN).tobytes() == held_gnn.tobytes()
        assert h.rollup_span(5)[0].tobytes() == span_rows.tobytes()
        # the other way: group series and group trend device results keep their bytes across every other family
        dv, dp, dn, dP, _, _ = h.group_node_series_device(SPAN, IN, 0, 4, *specs)
        pr, pn, ps, pq, tm, tP, _, _ = h.group_edge_trends_top_device(SPAN, 0, 4, (Q, 0.99),
                                                                      T(abi.TREND_ZSCORE, recent=1), 20)

        def held():
            return (h.d2h(dv, dn * dP * 3, np.float64), h.d2h(dp, dn * dP, np.uint8), h.d2h(pr, tm, abi.EDGE_TREND),
                    h.d2h(pn, tm, abi.EDGE_OUT), h.d2h(ps, tm * tP, np.float64))

        keep = held()
        assert tm > 0
        for src in (WINDOW, SPAN):
            h.group_edges(src)
            h.group_node_metrics(src, IN, *specs)
            h.group_node_top(src, OUT, (Q, 0.5), 4)
            h.group_node_changes(IN, (Q, 0.99), source=src)
            h.node_series(src, IN, 0, 3, *specs)
            h.node_trends_top(src, OUT, 0, 3, abi.METRIC_COUNT, T(abi.TREND_SHIFT), 5)
            h.edge_series(src, 0, 3, *specs)
            h.edge_trends_top(src, 0, 3, abi.METRIC_COUNT, T(abi.TREND_SHIFT), 5)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(keep, held()))
        # and each of the two group families across the other: the series across group trend calls, then a trend
        # top result across group series calls
        h.group_node_trends_top(SPAN, OUT, 1, 3, abi.METRIC_COUNT, T(abi.TREND_SLOPE), 7)
        h.group_edge_trends(WINDOW, 0, 3, (Q, 0.99), T(abi.TREND_SHIFT))
        assert all(x.tobytes() == y.tobytes() for x, y in zip(keep[:2], held()[:2]))
        pr, pn, ps, pq, tm, tP, _, _ = h.group_edge_trends_top_device(SPAN, 0, 4, (Q, 0.99),
                                                                      T(abi.TREND_ZSCORE, recent=1), 20)
        keep = held()
        h.group_edge_series(WINDOW, 0, 3, *specs)
        h.group_node_series_keys(capi.Handle.node_ends([(GRP, 1)]), OUT, 1, 3, abi.METRIC_COUNT)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(keep[2:], held()[2:]))
    finally:
        m.close()
