"""GPU: correlations (alz_edge_correlations*, alz_node_correlations*, alz_group_edge_correlations*,
alz_group_node_correlations*, alz_debug_corr_series, docs/SPEC.md §29).

Records, top order, top rows, series, points and info are compared as bytes against tests/corr_ref.py over the
candidate series that tests/series_ref.py, node_series_ref.py and group_series_ref.py give for the entries that
tests/rollup_model.py and tests/tier_model.py say the rings retain. Windows come from the Modelled stream of
tests/test_gpu_edge_series.py."""
import ctypes as C

import numpy as np
import pytest

import corr_ref as cr
import group_ref as gr
import group_series_ref as gsr
import node_ref as nr
import node_series_ref as nsr
import series_ref as sr
from alaz_b200 import abi, capi
from change_ref import row_keys
from test_gpu_edge_series import DEPTH, TIER_DEPTH, Modelled, make_source
from test_gpu_gnn_rollup import universe
from test_gpu_group_series import use_map

pytestmark = pytest.mark.gpu
WINDOW, WIN, TIER, SPAN = abi.SOURCE_WINDOW, abi.ROLLUP_WINDOWS, abi.ROLLUP_TIER, abi.ROLLUP_SPAN
IN, OUT = abi.SIDE_IN, abi.SIDE_OUT
Q = abi.METRIC_QUANTILE
POS, NEG, ABS = abi.CORR_POSITIVE, abi.CORR_NEGATIVE, abi.CORR_ABS
SKIP, ZERO = abi.CORR_ABSENT_SKIP, abi.CORR_ABSENT_ZERO
K = capi.Handle.corr
Target = capi.Handle.Target
LEVELS = ("edge", "node", "group_edge", "group_node")


def spec_of(c):
    return dict(direction=c.direction, absent=c.absent, max_lag=c.max_lag, min_points=c.min_points)


@pytest.fixture(scope="module")
def mod():
    m = Modelled(universe(seed=84), history=(DEPTH, 1 << 15), tiers=[(2, TIER_DEPTH, 1 << 15, 1 << 13)])
    m.random_windows(12, seed=841, lo=0.2, hi=0.7)
    m.last = m.window(np.flatnonzero(np.random.default_rng(842).random(m.s.g.n_edges) < 0.5))
    assert len(m.rm.entries) == DEPTH and len(m.tm.tiers[0].ring.entries) == TIER_DEPTH
    yield m
    m.close()


def candidates(m, level, rows, side, tier, k, spec, gmap):
    """(heads for corr_ref.records, node?, the top call's rows, y [n, P], p [n, P]) of a level's candidates"""
    gmap = gr.EMPTY if gmap is None else gmap
    ents, _ = m.entries(tier)
    if level == "edge":
        v, p = sr.series(ents, row_keys(rows), [spec], k)
        return rows, False, rows, v[:, :, 0], p
    if level == "node":
        keys = nr.keys(rows)
        v, p = nsr.series(ents, keys, side, [spec], k)
        return keys, True, nr.group(rows), v[:, :, 0], p
    g = gsr.source_edges(rows, gmap)
    if level == "group_edge":
        v, p = gsr.edge_series(ents, *gsr.row_ends(g), [spec], gmap, k)
        return g, False, g, v[:, :, 0], p
    keys = nr.keys(g)
    v, p = gsr.node_series(ents, keys, side, [spec], gmap, k)
    return keys, True, gsr.source_nodes(rows, gmap), v[:, :, 0], p


def take_of(m, tier, k):
    _, pts = m.entries(tier)
    take = pts[max(len(pts) - k, 0):]
    return take, sum(x["rows_in"] for x in take)


def synthetic(m, tier, k, seed, holes=True):
    """a target of random values (some absent) aligned to the ring"""
    take, _ = take_of(m, tier, k)
    rng = np.random.default_rng(seed)
    P = len(take)
    pres = (rng.random(P) < 0.85).astype(np.uint8) if holes else None
    return Target(rng.normal(size=P) * 1e3, pres, take[-1]["window_last"] if P else 0)


def keys_target(m, level, rows, side, tier, k, spec, gmap, pick=0):
    """the target a one-key series-keys call of the level gives for candidate `pick`"""
    h = m.h
    gmap = gr.EMPTY if gmap is None else gmap
    if level == "edge":
        v, p, pts, _ = h.edge_series_keys(rows[pick:pick + 1], tier, k, spec)
    elif level == "node":
        v, p, pts, _ = h.node_series_keys(nr.group(rows)[pick:pick + 1], side, tier, k, spec)
    elif level == "group_edge":
        g = gsr.source_edges(rows, gmap)
        v, p, pts, _ = h.group_edge_series_keys(g[pick:pick + 1], tier, k, spec)
    else:
        v, p, pts, _ = h.group_node_series_keys(gsr.source_nodes(rows, gmap)[pick:pick + 1], side, tier, k, spec)
    return Target(v[0, :, 0], p[0], pts[-1]["window_last"] if pts else 0)


def check(m, level, source, tier, k, spec, corr, target, side=IN, gmap=None, top=None, min_score=-np.inf,
          what=None):
    """the full list, the top call and both device forms of one call against the reference, as bytes"""
    h = m.h
    what = what or (level, source, tier, k, spec, side, spec_of(corr))
    rows = make_source(m, source)
    heads, node, trows_all, y, p = candidates(m, level, rows, side, tier, k, spec, gmap)
    rec = cr.records(heads, y, p, target.values, target.present, node=node, **spec_of(corr))
    take, rows_in = take_of(m, tier, k)
    tp = np.ones(len(target.values), np.uint8) if target.present is None else target.present
    info = dict(rows=len(rec), rows_in=rows_in, valid=int(rec["valid"].sum()), above=0, points=len(take), tier=tier,
                target_used=int((tp != 0).sum()))
    got, gpts, ginfo = h.correlations(level, source, tier, k, spec, corr, target, side=side)
    assert got.tobytes() == rec.tobytes(), (what, np.flatnonzero(got.view(np.uint8).reshape(-1, 48).any(1) !=
                                                                 rec.view(np.uint8).reshape(-1, 48).any(1))[:5])
    assert gpts == take and ginfo == info, (what, ginfo, info)
    d, n, P, dpts, dinfo = h.correlations_device(level, source, tier, k, spec, corr, target, side=side)
    assert (n, P, dpts, dinfo) == (len(rec), len(take), take, info), what
    assert h.d2h(d, n, rec.dtype).tobytes() == rec.tobytes(), what
    top = top or max(len(rec) // 4, 1)
    idx, above = cr.top(rec, top, min_score)
    trec, trows, ts, tpp, tpts, tinfo = h.correlations_top(level, source, tier, k, spec, corr, target, top, min_score,
                                                           side=side)
    assert trec.tobytes() == rec[idx].tobytes(), (what, trec["index"][:8], idx[:8])
    assert trows.tobytes() == trows_all[idx].tobytes(), what
    assert ts.tobytes() == y[idx].tobytes() and tpp.tobytes() == p[idx].tobytes(), what
    assert tpts == take and tinfo == dict(info, above=above), (what, tinfo)
    pr, pw, ps, pq, mm, P, dpts, dinfo = h.correlations_top_device(level, source, tier, k, spec, corr, target, top,
                                                                    min_score, side=side)
    assert (mm, dinfo) == (len(idx), tinfo), what
    if mm:
        assert h.d2h(pr, mm, rec.dtype).tobytes() == trec.tobytes(), what
        assert h.d2h(pw, mm, trows.dtype).tobytes() == trows.tobytes(), what
        assert h.d2h(ps, mm * P, np.float64).tobytes() == ts.tobytes(), what
    return rec, idx


@pytest.mark.parametrize("tier", [0, 1])
@pytest.mark.parametrize("source", [WINDOW, WIN, TIER, SPAN])
def test_every_source_direction_and_absent_mode_edges(mod, source, tier):
    depth = DEPTH if tier == 0 else TIER_DEPTH
    valid = 0
    for spec in ((Q, 0.99), abi.METRIC_COUNT):
        for direction in (POS, NEG, ABS):
            for absent in (SKIP, ZERO):
                for max_lag in (0, 1, depth - 1):
                    c = K(direction, absent, max_lag, 3)
                    rows = make_source(mod, source)
                    t = keys_target(mod, "edge", rows, IN, tier, depth, spec, None, pick=len(rows) // 3)
                    rec, _ = check(mod, "edge", source, tier, depth, spec, c, t)
                    valid += int(rec["valid"].sum())
                    check(mod, "edge", source, tier, depth, spec, c, synthetic(mod, tier, depth, seed=max_lag))
    assert valid > 0


@pytest.mark.parametrize("which", ["empty", "owners", "namespaces"])
@pytest.mark.parametrize("level", LEVELS[1:])
def test_node_and_group_levels_both_sides_every_map(mod, level, which):
    gmap = use_map(mod, which)
    for source in (WINDOW, SPAN):
        for tier, k in ((0, DEPTH), (1, TIER_DEPTH)):
            for side in ((IN, OUT) if level != "group_edge" else (IN,)):
                rows = make_source(mod, source)
                for spec, c in (((Q, 0.99), K(POS, SKIP, 1, 3)), (abi.METRIC_ERR_RATE, K(ABS, ZERO, k - 1, 3)),
                                (abi.METRIC_COUNT, K(NEG, SKIP, 0, 4))):
                    t = keys_target(mod, level, rows, side, tier, k, spec, gmap, pick=1)
                    check(mod, level, source, tier, k, spec, c, t, side=side, gmap=gmap, what=(level, which, source,
                                                                                             tier, side, spec))
                    check(mod, level, source, tier, k, spec, c, synthetic(mod, tier, k, seed=7), side=side, gmap=gmap)


def test_a_candidate_correlates_with_itself_and_min_score_cuts(mod):
    rows = mod.last
    spec = (Q, 0.99)
    _, _, _, y, p = candidates(mod, "edge", rows, IN, 0, DEPTH, spec, None)
    varied = [i for i in range(len(rows)) if p[i].sum() >= 4 and np.ptp(y[i][p[i] == 1]) > 0]
    pick = varied[0]
    t = keys_target(mod, "edge", rows, IN, 0, DEPTH, spec, None, pick=pick)
    for mp in (3, 4, DEPTH):
        rec, _ = check(mod, "edge", WINDOW, 0, DEPTH, spec, K(POS, SKIP, 0, mp), t)
        assert np.all(rec["used"][rec["valid"] == 1] >= mp)
    rec, _ = check(mod, "edge", WINDOW, 0, DEPTH, spec, K(POS, SKIP, 0, 3), t)
    assert rec["valid"][pick] == 1 and abs(rec["r"][pick] - 1.0) < 1e-12
    vals = np.sort(rec["score"][rec["valid"] == 1])
    for cut in (vals[len(vals) // 2], vals[-1], 0.0, -0.0, 2.0, -np.inf):
        _, idx = check(mod, "edge", WINDOW, 0, DEPTH, spec, K(POS, SKIP, 0, 3), t, top=len(rows), min_score=cut,
                       what=cut)
        assert np.all(rec["score"][idx] >= cut)


def raw(h, fn, head, k, corr, target, m=None):
    """the status of the device form of fn, (n_out, n_points)"""
    d, n, p, info = C.c_void_p(), C.c_size_t(7), C.c_uint32(7), abi.CorrInfo()
    m = abi.metrics(abi.METRIC_COUNT) if m is None else m
    rc = getattr(h.L, fn + "_device")(h.h, *head, k, m, None if corr is None else C.byref(corr),
                                      None if target is None else C.byref(target.s), C.byref(d), C.byref(n),
                                      C.byref(p), None, C.byref(info))
    return rc, n.value, p.value


def test_stale_targets_and_every_invalid_argument(mod):
    h = mod.h
    rows = mod.last
    t = keys_target(mod, "edge", rows, IN, 0, DEPTH, abi.METRIC_COUNT, None)
    ok = K(POS, SKIP, 2, 3)
    head = (WINDOW, 0)
    assert raw(h, "alz_edge_correlations", head, DEPTH, ok, t)[0] == abi.OK
    short = Target(t.values[1:], t.present[1:], t.s.window_last)
    assert raw(h, "alz_edge_correlations", head, DEPTH, ok, short)[0] == abi.E_STATE   # n != P
    old = Target(t.values, t.present, t.s.window_last - 1)
    assert raw(h, "alz_edge_correlations", head, DEPTH, ok, old)[0] == abi.E_STATE     # not the newest entry's
    bad = [
        (DEPTH, None, t), (DEPTH, ok, None), (0, ok, t),
        (DEPTH, K(3, SKIP, 0, 3), t), (DEPTH, K(POS, 2, 0, 3), t), (DEPTH, K(POS, SKIP, 33, 3), t),
        (2, K(POS, SKIP, 2, 3), t), (DEPTH, K(POS, SKIP, 0, 2), t),
        (DEPTH, ok, Target(np.where(np.arange(DEPTH) == 2, np.nan, 1.0), None, t.s.window_last)),
        (DEPTH, ok, Target(np.where(np.arange(DEPTH) == 2, np.inf, 1.0), None, t.s.window_last)),
        (DEPTH, ok, Target(np.where(np.arange(DEPTH) == 2, 2.0 ** 64 * 1.0000001, 1.0), None, t.s.window_last)),
        (DEPTH, ok, Target(np.zeros(0), None, t.s.window_last, n=DEPTH)),
    ]
    for k, c, tt in bad:
        assert raw(h, "alz_edge_correlations", head, k, c, tt)[0] == abi.E_INVAL, (k, c and spec_of(c))
    # an absent NaN and a present 2^64 are accepted
    vals = np.where(np.arange(DEPTH) == 2, np.nan, 2.0 ** 64)
    pres = (np.arange(DEPTH) != 2).astype(np.uint8)
    rec, _ = check(mod, "edge", WINDOW, 0, DEPTH, abi.METRIC_COUNT, ok, Target(vals, pres, t.s.window_last))
    n, p = C.c_size_t(0), C.c_uint32(0)
    assert h.L.alz_edge_correlations(h.h, WINDOW, 0, DEPTH, abi.metrics(abi.METRIC_COUNT), C.byref(ok), C.byref(t.s),
                                     None, 0, C.byref(n), C.byref(p), None, None) == abi.E_CAPACITY   # cap 0
    assert n.value == len(rows) and p.value == DEPTH
    assert raw(h, "alz_node_correlations", (WINDOW, 2, 0), DEPTH, ok, t)[0] == abi.E_INVAL     # side
    assert raw(h, "alz_edge_correlations", (99, 0), DEPTH, ok, t)[0] == abi.E_INVAL           # source
    assert raw(h, "alz_edge_correlations", (WINDOW, 7), DEPTH, ok, t)[0] == abi.E_INVAL       # tier
    f = h.L.alz_edge_correlations_top
    n, p = C.c_size_t(0), C.c_uint32(0)
    for top, ms in ((0, 0.0), (5, float("nan"))):
        assert f(h.h, WINDOW, 0, DEPTH, abi.metrics(abi.METRIC_COUNT), C.byref(ok), C.byref(t.s), top, ms, None, None,
                 None, None, 0, C.byref(n), C.byref(p), None, None) == abi.E_INVAL


def test_a_flush_makes_the_target_stale_and_nothing_else_moves():
    m = Modelled(universe(n_edges=400, seed=85), history=(5, 1 << 13), tiers=[(2, 3, 1 << 13, 1 << 12)])
    m.random_windows(6, seed=851)
    m.last = m.window(np.arange(400))
    h = m.h
    rows = m.last
    spec = abi.METRIC_COUNT
    t = keys_target(m, "edge", rows, IN, 0, 5, spec, None, pick=3)
    c = K(ABS, SKIP, 2, 3)
    targets = {level: keys_target(m, level, rows, IN, 0, 5, spec, None, pick=1) for level in LEVELS}
    # other families' device results keep their bytes across correlation calls
    d_tr, n_tr, _, _, _ = h.edge_trends_device(WINDOW, 0, 5, spec, capi.Handle.trend(abi.TREND_SLOPE))
    before_tr = h.d2h(d_tr, n_tr, abi.EDGE_TREND).tobytes()
    pv, pp, ns, Ps, _, _ = h._series_device("alz_edge_series_device", (WINDOW,), (0, 5), (spec,))
    before_sv = h.d2h(pv, ns * Ps, np.float64).tobytes()
    for level in LEVELS:
        check(m, level, WINDOW, 0, 5, spec, c, targets[level])
    assert h.d2h(d_tr, n_tr, abi.EDGE_TREND).tobytes() == before_tr
    assert h.d2h(pv, ns * Ps, np.float64).tobytes() == before_sv
    # the next flush moves the ring: the same target is now stale, a fresh one works
    m.last = m.window(np.arange(200))
    assert raw(h, "alz_edge_correlations", (WINDOW, 0), 5, c, t)[0] == abi.E_STATE
    check(m, "edge", WINDOW, 0, 5, spec, c, keys_target(m, "edge", m.last, IN, 0, 5, spec, None, pick=3))
    m.close()


def test_zero_retained_entries():
    m = Modelled(universe(n_edges=50, seed=86), history=(4, 1 << 12))
    h = m.h
    c = K(POS, SKIP, 2, 3)
    for level in LEVELS:   # no flush yet: a 0-row window, P = 0
        got, pts, info = h.correlations(level, WINDOW, 0, 4, abi.METRIC_COUNT, c, Target(np.zeros(0), None, 0))
        assert len(got) == 0 and pts == [] and info["points"] == 0 and info["target_used"] == 0
    m.last = m.window(np.arange(50))
    assert raw(h, "alz_edge_correlations", (WINDOW, 0), 4, c, Target(np.zeros(0), None, 0))[0] == abi.E_STATE
    rec, _ = check(m, "edge", WINDOW, 0, 4, abi.METRIC_COUNT, c, synthetic(m, 0, 4, seed=1))
    assert rec["valid"].sum() == 0   # one point: no lag has 3 pairs
    m.close()


def hook_check(h, x, px, y, py, corr, top=0, min_score=-np.inf, what=None, offset=0):
    rec = cr.records(None, x, px, y, py, **spec_of(corr))
    got, idx, valid, above = h.debug_corr_series(x, px, Target(y, py), corr, top, min_score, offset=offset)
    if top:
        widx, wabove = cr.top(rec, top, min_score)
        assert idx.tolist() == widx.tolist() and above == wabove, what
        assert got.tobytes() == rec[widx].tobytes(), what
    else:
        assert got.tobytes() == rec.tobytes(), (what, np.flatnonzero((got != rec))[:5])
    assert valid == int(rec["valid"].sum()), what
    return rec


@pytest.fixture(scope="module")
def hh():
    h = capi.Handle(device=0, max_endpoints=1 << 10, max_pairs=1 << 12)
    yield h
    h.close()


@pytest.mark.parametrize("P", [1, 2, 3, 31, 63, 64, 65, 100, 127, 128, 129, 333, 1000])
def test_hook_tiles_over_j(hh, P):
    rng = np.random.default_rng(P)
    n = 301
    y = rng.normal(size=P) * 50
    x = y[None, :] * rng.normal(size=(n, 1)) + rng.normal(size=(n, P)) * 20
    for L in (1, 7):   # some rows lead the target
        x[L::37, L:] = y[None, : P - L] if P > L else x[L::37, L:]
    px = (rng.random((n, P)) < 0.9).astype(np.uint8)
    py = (rng.random(P) < 0.9).astype(np.uint8)
    for c in (K(POS, SKIP, 0, 3), K(ABS, ZERO, 8, 3), K(NEG, SKIP, 32, 5)):
        hook_check(hh, x, px, y, py, c, what=(P, spec_of(c)))
        hook_check(hh, x, px, y, py, c, top=40, what=(P, spec_of(c), "top"))
    # series one element past a 16-byte boundary: the whole-row loads start with their unaligned head
    hook_check(hh, x, px, y, py, K(ABS, SKIP, 8, 3), what=(P, "offset"), offset=1)


def test_max_lag_32_through_a_deep_history():
    m = Modelled(universe(n_edges=1500, seed=87), history=(40, 1 << 15))
    m.random_windows(39, seed=871, lo=0.3, hi=0.9)
    m.last = m.window(np.flatnonzero(np.random.default_rng(872).random(1500) < 0.6))
    assert len(m.rm.entries) == 40
    rows = m.last
    for spec in ((Q, 0.99), abi.METRIC_COUNT):
        for c in (K(ABS, SKIP, 32, 3), K(POS, ZERO, 8, 5), K(NEG, SKIP, 32, 8)):
            check(m, "edge", WINDOW, 0, 40, spec, c, keys_target(m, "edge", rows, IN, 0, 40, spec, None, pick=7))
            check(m, "edge", WINDOW, 0, 40, spec, c, synthetic(m, 0, 40, seed=3))
        check(m, "node", WINDOW, 0, 40, spec, K(ABS, SKIP, 32, 3),
              keys_target(m, "node", rows, OUT, 0, 40, spec, None, pick=2), side=OUT)
    m.close()


def test_hook_million_rows(hh):
    rng = np.random.default_rng(3)
    n, P = 1 << 20, 12
    y = rng.normal(size=P)
    x = rng.normal(size=(n, P))
    x[::1000] = y * 3.0
    px = np.ones((n, P), np.uint8)
    px[::7, ::5] = 0
    rec = hook_check(hh, x, px, y, None, K(POS, SKIP, 4, 3), top=1000)
    assert rec["valid"].sum() > n * 0.99


def test_hook_constant_rows_constant_target_and_large_values(hh):
    P = 20
    rng = np.random.default_rng(4)
    y = rng.normal(size=P)
    x = np.stack([np.full(P, 5.0), np.zeros(P), y * 2.0 ** 63, -y * 2.0 ** 64 / 4, y + 2.0 ** 63,
                  np.full(P, 2.0 ** 64), np.where(np.arange(P) % 2 == 0, 2.0 ** 64, -2.0 ** 64)])
    px = np.ones_like(x, dtype=np.uint8)
    for c in (K(POS, SKIP, 3, 3), K(ABS, ZERO, 3, 3)):
        rec = hook_check(hh, x, px, y, None, c, what=spec_of(c))
        assert rec["valid"][0] == 0 and rec["valid"][1] == 0 and rec["valid"][5] == 0
        assert rec["valid"][2] == 1
        rec = hook_check(hh, x, px, np.full(P, 3.0), None, c)
        assert rec["valid"].sum() == 0
        hook_check(hh, x, px, np.where(np.arange(P) % 3 == 0, 2.0 ** 64, -2.0 ** 64), None, c)


def test_hook_r_rounds_past_one_and_ties(hh):
    rng = np.random.default_rng(11)
    P, n = 7, 400
    y = rng.normal(size=(n, P)) * 10.0 ** rng.integers(-3, 4, size=(n, 1))
    # scaled copies of one target each: r is 1 in exact arithmetic, and the roundings take some of them past 1
    past, clamped = 0, 0
    for i in range(0, 400, 8):
        xs = y[i][None, :] * np.array([3.0, 0.1, 7.0, 1e-3, 1.0, 5.0, 0.3, 11.0])[:, None]
        raw = cr.correlations(xs, np.ones_like(xs, np.uint8), y[i], clamp=False)["r"]
        past += int((raw > 1.0).sum())
        rec = hook_check(hh, xs, np.ones_like(xs, np.uint8), y[i], None, K(POS, SKIP, 0, 3))
        assert np.all(rec["r"] <= 1.0)
        clamped += int(((raw > 1.0) & (rec["r"] == 1.0)).sum())
    assert past > 0 and clamped == past
    # period-2 rows and a target absent at j < 3: lags 0 / 2 and 1 / 3 tie bit for bit; identical rows tie by row
    y2 = np.tile([0.0, 1.0], 8) + np.repeat(rng.normal(size=8) * 1e-3, 2)
    x2 = np.tile(np.tile([3.0, 5.0], 8), (50, 1))
    py2 = np.array([0, 0, 0] + [1] * 13, np.uint8)
    for c in (K(POS, SKIP, 3, 3), K(NEG, SKIP, 3, 3), K(ABS, SKIP, 3, 3)):
        rec = hook_check(hh, x2, np.ones_like(x2, np.uint8), y2, py2, c, top=20)
        assert len(np.unique(rec["lag"])) == 1
        _, idx, _, _ = hh.debug_corr_series(x2, np.ones_like(x2, np.uint8), Target(y2, py2), c, 20)
        assert idx.tolist() == list(range(20))
