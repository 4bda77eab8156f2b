"""GPU: edge series (alz_edge_series*, alz_edge_series_keys*, docs/SPEC.md §19).

The expected values and presence are tests/series_ref.py over the entries tests/rollup_model.py and tests/tier_model.py
say the rings retain, compared as bytes; the expected points are what those models report for a rollup of each entry
alone. Windows come from the Stream of tests/test_gpu_gnn_rollup.py."""
import ctypes as C

import numpy as np
import pytest

import series_ref as sr
from alaz_b200 import abi, capi
from change_ref import row_keys
from rollup_model import RollupModel
from test_gpu_gnn_rollup import Stream, universe
from tier_model import TierModel, rows_of

pytestmark = pytest.mark.gpu
WINDOW, WIN, TIER, SPAN = abi.SOURCE_WINDOW, abi.ROLLUP_WINDOWS, abi.ROLLUP_TIER, abi.ROLLUP_SPAN
Q = abi.METRIC_QUANTILE
ALL = [abi.METRIC_COUNT, abi.METRIC_ERR5XX, abi.METRIC_ERR_RATE, abi.METRIC_MEAN_NS, (Q, 0.5), (Q, 0.99), (Q, 1.0)]
SUMS = [abi.METRIC_MEAN_NS, abi.METRIC_COUNT, abi.METRIC_ERR_RATE, abi.METRIC_ERR5XX]
DEPTH, TIER_DEPTH = 6, 4


class Modelled:
    """A Stream whose flushes also feed a RollupModel and a TierModel."""

    def __init__(self, g, history=None, tiers=(), **kw):
        self.s = Stream(g, history=history, tiers=tiers, **kw)
        self.h = self.s.h
        self.rm, self.tm = RollupModel(), TierModel()
        if history:
            self.rm.history(*history)
        if tiers:
            self.tm.configure(tiers)

    def window(self, edges):
        rows = self.s.window(edges)
        w = self.h.stats()["windows"]
        self.rm.append(rows, w)
        self.tm.window(rows, w)
        return rows

    def random_windows(self, n, seed, lo=0.3, hi=0.8):
        rng = np.random.default_rng(seed)
        return [self.window(np.flatnonzero(rng.random(self.s.g.n_edges) < rng.uniform(lo, hi))) for _ in range(n)]

    def entries(self, tier):
        """(rows of each retained entry, the info a rollup of it alone reports), oldest first"""
        if tier == 0:
            return ([rows_of(e["rows"]) for e in self.rm.entries],
                    [dict(windows=1, clocked=0, window_first=e["window"], window_last=e["window"], epoch_first=0,
                          epoch_last=0, rows_in=e["n"]) for e in self.rm.entries])
        ring = self.tm.tiers[tier - 1].ring
        return ([rows_of(e["rows"]) for e in ring.entries],
                [dict(windows=e["windows"], clocked=0, window_first=e["window_first"], window_last=e["window"],
                      epoch_first=0, epoch_last=0, rows_in=e["n"]) for e in ring.entries])

    def close(self):
        self.s.close()


def expect(m, tier, k, keys, specs):
    ents, pts = m.entries(tier)
    v, p = sr.series(ents, keys, specs, k)
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


def make_source(m, kind):
    h = m.h
    if kind == WINDOW:
        return m.last
    if kind == WIN:
        return h.rollup(3)[0]
    if kind == TIER:
        return h.rollup_tier(1, 2)[0]
    return h.rollup_span(5)[0]


@pytest.fixture(scope="module")
def mod():
    m = Modelled(universe(seed=14), history=(DEPTH, 1 << 15), tiers=[(2, TIER_DEPTH, 1 << 15, 1 << 13)])
    m.random_windows(12, seed=141, lo=0.2, hi=0.6)
    m.last = m.window(np.flatnonzero(np.random.default_rng(142).random(m.s.g.n_edges) < 0.5))
    assert len(m.rm.entries) == DEPTH and len(m.tm.tiers[0].ring.entries) == TIER_DEPTH
    yield m
    m.close()


@pytest.mark.parametrize("tier", [0, 1])
@pytest.mark.parametrize("source", [WINDOW, WIN, TIER, SPAN])
def test_every_source_every_k_every_metric(mod, tier, source):
    h = mod.h
    rows = make_source(mod, source)
    keys = row_keys(rows)
    depth = DEPTH if tier == 0 else TIER_DEPTH
    for k in (1, 3, depth, depth + 5):
        for specs in (ALL, SUMS, [(Q, 0.99)]):
            same(h.edge_series(source, tier, k, *specs), expect(mod, tier, k, keys, specs), (source, tier, k, specs))


@pytest.mark.parametrize("tier", [0, 1])
def test_caller_keys_host_and_device(mod, tier):
    h = mod.h
    rng = np.random.default_rng(tier)
    seen = np.concatenate(mod.entries(tier)[0])
    seen = seen[np.unique(row_keys(seen), return_index=True)[1]]
    ends = [(int(r["from_type"]), int(r["from"]), int(r["to_type"]), int(r["to"]))
            for r in seen[rng.choice(len(seen), 300, replace=False)]]
    ends += ends[:7] + [(abi.NODE_POD, 123456, abi.NODE_SVC, 99999)]   # duplicates and an edge no entry holds
    rev = [e for e in ends if e[0] == abi.NODE_POD and e[2] == abi.NODE_POD][:5]
    ends += [(e[2], e[3], e[0], e[1]) for e in rev]                   # pod <-> pod edges named the other way
    keys_arr = capi.Handle.edge_ends(ends)
    keys = sr.ends_keys(keys_arr)
    for k in (1, 3, 50):
        want = expect(mod, tier, k, keys, ALL)
        got = h.edge_series_keys(keys_arr, tier, k, *ALL)
        same(got, want, ("keys", tier, k))
        pv, pp, n, P, pts, info = h.edge_series_keys_device(keys_arr, tier, k, *ALL)
        assert (n, P, pts, info) == (len(ends), got[1].shape[1], got[2], got[3])
        assert h.d2h(pv, n * P * len(ALL), np.float64).tobytes() == got[0].tobytes()
        assert h.d2h(pp, n * P, np.uint8).tobytes() == got[1].tobytes()
    # the source device form too
    v, p, pts, info = h.edge_series(WINDOW, tier, 3, *ALL)
    pv, pp, n, P, dpts, dinfo = h.edge_series_device(WINDOW, tier, 3, *ALL)
    assert (n, P, dpts, dinfo) == (v.shape[0], v.shape[1], pts, info)
    assert h.d2h(pv, v.size, np.float64).tobytes() == v.tobytes()
    assert h.d2h(pp, p.size, np.uint8).tobytes() == p.tobytes()


def test_unknown_edge_is_all_absent_and_duplicates_agree(mod):
    h = mod.h
    r = mod.last[:3]
    ends = capi.Handle.edge_ends(np.concatenate([r, r[::-1]]))
    extra = capi.Handle.edge_ends([(abi.NODE_POD, (1 << 29) - 1, abi.NODE_OUTBOUND_HOST, 5)])
    v, p, _, _ = h.edge_series_keys(np.concatenate([ends, extra]), 0, DEPTH, *ALL)
    assert v[:3].tobytes() == v[3:6][::-1].tobytes() and p[:3].tobytes() == p[3:6][::-1].tobytes()
    assert not p[6].any() and not v[6].view(np.uint64).any()
    assert p[:3, -1].all()                                        # the last window holds them


@pytest.mark.parametrize("tier", [0, 1])
def test_newest_point_is_the_k1_rollup_metrics(mod, tier):
    h = mod.h
    rows, _ = h.rollup_tier(tier, 1)
    kind = WIN if tier == 0 else TIER
    want = h.edge_metrics_rollup(kind, *ALL)
    v, p, pts, _ = h.edge_series_keys(rows, tier, 2, *ALL)
    assert p[:, -1].all()
    assert v[:, -1, :].tobytes() == want.tobytes()
    v, p, _, _ = h.edge_series(kind, tier, 1, *ALL)
    assert v[:, 0, :].tobytes() == want.tobytes() and p.all()
    info = (h.rollup if tier == 0 else (lambda k: h.rollup_tier(1, k)))(1)[1]
    assert pts[-1] == {x: info[x] for x in pts[-1]}


# ---- ring layouts ----------------------------------------------------------------------------------------------

def test_wrapping_arena_empty_window_oversized_window_and_reconfiguration():
    m = Modelled(universe(n_edges=400, seed=15), history=(4, 350))
    rng = np.random.default_rng(151)
    wrapped = had_empty = False
    for w in range(14):
        n = [250, 120, 300, 0, 200, 260, 90, 310, 0, 150, 240, 280, 60, 130][w]
        rows = m.window(rng.choice(400, n, replace=False) if n else np.zeros(0, np.int64))
        firsts = [e["first_row"] for e in m.rm.entries]
        wrapped |= len(firsts) > 1 and firsts[-1] == 0
        had_empty |= len(m.rm.entries) > 1 and any(e["n"] == 0 for e in m.rm.entries[:-1])
        if len(m.rm.entries) > 1:
            union = np.concatenate([rows_of(e["rows"]) for e in m.rm.entries])
            union = union[np.unique(row_keys(union), return_index=True)[1]]
            for k in (1, 2, 4, 9):
                for specs in (ALL, SUMS):
                    same(m.h.edge_series(WINDOW, 0, k, *specs), expect(m, 0, k, row_keys(rows), specs), (w, k))
                    same(m.h.edge_series_keys(union, 0, k, *specs), expect(m, 0, k, row_keys(union), specs),
                         ("keys", w, k))
    assert wrapped and had_empty
    # a window larger than the arena clears the history: P shrinks to what came after it
    big = m.window(np.arange(400))
    assert len(big) > 350 and len(m.rm.entries) == 0
    v, p, pts, info = m.h.edge_series(WINDOW, 0, 4, abi.METRIC_COUNT)
    assert v.shape == (len(big), 0, 1) and pts == [] and info["points"] == 0
    last = m.window(np.arange(100))
    same(m.h.edge_series(WINDOW, 0, 4, *ALL), expect(m, 0, 4, row_keys(rows_of(m.rm.entries[-1]["rows"])), ALL),
         "after the clear")
    # reconfiguring: P = 0
    m.h.window_history(5, 1 << 12)
    m.rm.history(5, 1 << 12)
    v, p, pts, info = m.h.edge_series(WINDOW, 0, 3, *ALL)
    assert v.shape == (len(last), 0, len(ALL)) and p.shape == (len(last), 0) and pts == []
    m.close()


def test_empty_entry_in_the_middle():
    m = Modelled(universe(n_edges=300, seed=16), history=(5, 1 << 12), tiers=[(2, 3, 1 << 12, 1 << 11)])
    m.window(np.arange(0, 200))
    m.window(np.zeros(0, np.int64))
    m.window(np.arange(100, 300))
    m.window(np.zeros(0, np.int64))
    keys = row_keys(m.h.rollup(4)[0])
    for tier, k in ((0, 4), (0, 2), (1, 2)):
        same(m.h.edge_series(WIN, tier, k, *ALL), expect(m, tier, k, keys, ALL), (tier, k))
    m.close()


def test_more_than_2_24_slots_and_2_20_entry_rows():
    g = universe(n_pods=30000, n_svcs=200, n_edges=60000, seed=17)
    m = Modelled(g, history=(22, 1 << 21), max_pairs=1 << 17)
    m.random_windows(22, seed=171, lo=0.9, hi=0.95)
    rows_in = sum(e["n"] for e in m.rm.entries)
    assert rows_in > (1 << 20)
    rng = np.random.default_rng(172)
    known = capi.Handle.edge_ends(rows_of(m.rm.entries[-1]["rows"]))
    idx = rng.integers(0, len(known), 780_000)
    ends = known[idx]
    absent = rng.random(len(ends)) < 0.1
    ends["from"][absent & (ends["from_type"] == abi.NODE_POD)] = (1 << 29) - 7   # no such pod
    assert len(ends) * 22 > (1 << 24)
    keys = sr.ends_keys(ends)
    for specs in ([abi.METRIC_COUNT], [(Q, 0.99), abi.METRIC_ERR_RATE]):
        same(m.h.edge_series_keys(ends, 0, 22, *specs), expect(m, 0, 22, keys, specs), ("large", specs))
    m.close()


# ---- errors ------------------------------------------------------------------------------------------------------

def raw(h, *args, fn="alz_edge_series", out=None, present=None, cap=0, points=None):
    n, p, info = C.c_size_t(777), C.c_uint32(777), abi.SeriesInfo()
    rc = getattr(h.L, fn)(h.h, *args, out, present, cap, C.byref(n), C.byref(p), points, C.byref(info))
    return rc, n.value, p.value


def test_every_error_code():
    m = Modelled(universe(n_edges=400, seed=18), history=(3, 1 << 14), tiers=[(2, 2, 1 << 14, 1 << 12)])
    h = m.h
    cm = abi.metrics(abi.METRIC_COUNT)
    m.random_windows(5, seed=181)
    ok = raw(h, WINDOW, 0, 3, cm, 1)
    assert ok[0] == abi.E_CAPACITY and ok[1] > 0 and ok[2] == 3
    # invalid arguments
    assert raw(h, WINDOW, 0, 0, cm, 1)[0] == abi.E_INVAL                                    # k = 0
    assert raw(h, WINDOW, 2, 1, cm, 1)[0] == abi.E_INVAL                                    # tier above the tiers
    assert raw(h, WINDOW, 0, 1, cm, 0)[0] == abi.E_INVAL                                    # nm = 0
    assert raw(h, WINDOW, 0, 1, abi.metrics(*[abi.METRIC_COUNT] * 9), 9)[0] == abi.E_INVAL  # nm = 9
    assert raw(h, WINDOW, 0, 1, (abi.Metric * 1)(abi.Metric(9, 0, 0.0)), 1)[0] == abi.E_INVAL
    for q in (1.5, -0.1, float("nan")):
        assert raw(h, WINDOW, 0, 1, abi.metrics((Q, q)), 1)[0] == abi.E_INVAL
    assert raw(h, 3, 0, 1, cm, 1)[0] == abi.E_INVAL                                         # unknown source
    assert raw(h, WINDOW, 0, 1, None, 1)[0] == abi.E_INVAL                                  # null metrics
    assert raw(h, WINDOW, 0, 1, cm, 1, cap=5)[0] == abi.E_INVAL                             # null values with cap
    assert h.L.alz_edge_series(h.h, WINDOW, 0, 1, cm, 1, None, None, 0, None, None, None, None) == abi.E_INVAL
    n = C.c_size_t(0)
    assert h.L.alz_edge_series(h.h, WINDOW, 0, 1, cm, 1, None, None, 0, C.byref(n), None, None, None) == abi.E_INVAL
    assert h.L.alz_edge_series(None, WINDOW, 0, 1, cm, 1, None, None, 0, None, None, None, None) == abi.E_INVAL
    p_ = C.c_uint32(0)
    assert h.L.alz_edge_series_device(h.h, WINDOW, 0, 1, cm, 1, None, None, C.byref(n), C.byref(p_), None,
                                      None) == abi.E_INVAL                                  # null dev_values
    for bad in ((abi.NODE_SVC, 1, abi.NODE_SVC, 2), (4, 1, abi.NODE_POD, 2), (abi.NODE_POD, 1 << 29, abi.NODE_SVC, 1),
                (abi.NODE_POD, 1, abi.NODE_SVC, 1 << 29)):
        e = capi.Handle.edge_ends([(abi.NODE_POD, 1, abi.NODE_SVC, 2), bad])
        assert raw(h, e.ctypes.data_as(C.c_void_p), 2, 0, 1, cm, 1, fn="alz_edge_series_keys", cap=2,
                   out=np.zeros(64).ctypes.data_as(C.c_void_p))[0] == abi.E_INVAL, bad
    assert raw(h, None, 3, 0, 1, cm, 1, fn="alz_edge_series_keys")[0] == abi.E_INVAL        # null keys
    assert raw(h, None, 0, 0, 1, cm, 1, fn="alz_edge_series_keys")[:2] == (0, 0)            # no keys: fine
    # state: no rows of a rollup source; no tiers, no history
    for src in (WIN, TIER, SPAN):
        assert raw(h, src, 0, 1, cm, 1)[0] == abi.E_STATE
    t = Modelled(universe(n_edges=200, seed=19), tiers=[(2, 2, 1 << 13, 1 << 12)])
    t.random_windows(2, seed=191)
    assert raw(t.h, WINDOW, 0, 1, cm, 1)[0] == abi.E_STATE
    assert raw(t.h, WINDOW, 1, 1, cm, 1)[0] == abi.E_CAPACITY                               # cap 0 below the rows
    t.close()
    w = Modelled(universe(n_edges=200, seed=20), history=(2, 1 << 13))
    w.random_windows(1, seed=201)
    assert raw(w.h, WINDOW, 1, 1, cm, 1)[0] == abi.E_STATE
    w.close()
    # capacity: cap below the rows writes nothing but sets *n_out and *n_points
    rc, n_rows, P = raw(h, WINDOW, 0, 2, cm, 1)
    assert rc == abi.E_CAPACITY and P == 2
    vals = np.full((n_rows, P), 7.0)
    pres = np.full((n_rows, P), 9, np.uint8)
    pts = (abi.RollupInfo * 2)()
    rc, n2, P2 = raw(h, WINDOW, 0, 2, cm, 1, out=vals.ctypes.data_as(C.c_void_p),
                     present=pres.ctypes.data_as(C.c_void_p), cap=n_rows - 1, points=pts)
    assert (rc, n2, P2) == (abi.E_CAPACITY, n_rows, 2)
    assert np.all(vals == 7.0) and np.all(pres == 9) and pts[0].windows == 0
    m.close()


def test_more_than_2_30_slots_is_a_capacity_error():
    """64 points x 2^24 keys = 2^30 slots. The keys are zero pages that the call never reads: the size is refused
    before the keys are packed."""
    h = capi.Handle(max_endpoints=64, max_pairs=1 << 12)
    h.window_history(64, 1 << 10)
    for _ in range(64):
        h.flush()
    big = np.zeros(1 << 24, dtype=abi.EDGE_ENDS)
    cm = abi.metrics(abi.METRIC_COUNT)
    n, p_ = C.c_size_t(0), C.c_uint32(0)
    pv, pp = C.c_void_p(), C.c_void_p()
    rc = h.L.alz_edge_series_keys_device(h.h, big.ctypes.data_as(C.c_void_p), len(big), 0, 64, cm, 1, C.byref(pv),
                                         C.byref(pp), C.byref(n), C.byref(p_), None, None)
    assert (rc, n.value, p_.value) == (abi.E_CAPACITY, len(big), 64)
    rc = h.L.alz_edge_series_keys_device(h.h, big.ctypes.data_as(C.c_void_p), len(big) - 1, 0, 64, cm, 1,
                                         C.byref(pv), C.byref(pp), C.byref(n), C.byref(p_), None, None)
    assert (rc, n.value, p_.value) == (abi.OK, len(big) - 1, 64)   # 2^30 - 64 slots, every one absent
    assert not h.d2h(pp.value, 1 << 20, np.uint8).any()
    h.close()


# ---- reads only ----------------------------------------------------------------------------------------------------

def test_reads_only_against_a_twin_handle():
    cfg = dict(history=(4, 1 << 15), tiers=[(2, 3, 1 << 15, 1 << 13)])
    a, b = Modelled(universe(seed=21), **cfg), Modelled(universe(seed=21), **cfg)
    for m in (a, b):
        m.random_windows(7, seed=211, lo=0.2, hi=0.6)
        m.h.rollup(3)
        m.h.baseline_pin(WIN)
        m.random_windows(1, seed=212)
        m.h.rollup_tier(1, 2)
        m.h.rollup_span(5)
        m.h.rollup(2)
        m.keys = capi.Handle.edge_ends(m.random_windows(1, seed=214)[0])
    h = a.h

    def state(hh):
        return dict(metrics_w=hh.edge_metrics(*ALL), metrics_r=hh.edge_metrics_rollup(TIER, *ALL),
                    gnn=hh.gnn_score_rollup(SPAN), top=hh.edge_top((Q, 0.99), 7)[0],
                    changes=hh.edge_changes((Q, 0.99), abi.CHANGE_RATIO)[0])

    pm, nm_ = h.edge_metrics_device(abi.METRIC_COUNT)
    dev_m = h.d2h(pm, nm_, np.float64)
    pg, ng = h.gnn_score_rollup_device(WIN)
    dev_g = h.d2h(pg, ng, np.float32)
    for tier in (0, 1):
        for src in (WINDOW, WIN, TIER, SPAN):
            h.edge_series(src, tier, 9, *ALL)
            h.edge_series_device(src, tier, 2, *SUMS)
        h.edge_series_keys(a.keys, tier, 3, *ALL)
    assert h.d2h(pm, nm_, np.float64).tobytes() == dev_m.tobytes()
    assert h.d2h(pg, ng, np.float32).tobytes() == dev_g.tobytes()
    sa, sb = state(a.h), state(b.h)
    for k in sa:
        assert sa[k].tobytes() == sb[k].tobytes(), k
    # the held rollups, then the next flush and rollups of every kind
    for kind in (WIN, TIER, SPAN):
        assert a.h.gnn_score_rollup(kind).tobytes() == b.h.gnn_score_rollup(kind).tobytes(), kind
    ra, rb = a.random_windows(2, seed=213), b.random_windows(2, seed=213)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(ra, rb))
    for call in (lambda m: m.h.rollup(4), lambda m: m.h.rollup_tier(1, 3), lambda m: m.h.rollup_span(9),
                 lambda m: m.h.rollup_span(3, abi.SPAN_AT_LEAST)):
        (x, xi), (y, yi) = call(a), call(b)
        assert x.tobytes() == y.tobytes() and xi == yi
    assert a.h.stats()["windows"] == b.h.stats()["windows"]
    a.close()
    b.close()
