"""GPU: the GNN anomaly pass over a window, tier or span rollup's rows (alz_gnn_score_rollup*, docs/SPEC.md §15).

The oracle is tests/gnn_ref.py run on the rollup's own rows, with the tolerances of tests/test_gpu_gnn.py (check(),
GAMMA); node keys and h2 come from alz_gnn_nodes. Every case runs on both layer paths (the `path` fixture). Windows
are cut from one universe of edges (tests/gnn_graphs.py) whose tables are loaded once: each window submits the
records of a subset of the edges, so edge sets overlap, appear and vanish from window to window."""
import ctypes as C

import numpy as np
import pytest

import gnn_graphs as gg
from alaz_b200 import abi, capi
from test_gpu_gnn import _star, check, path  # noqa: F401  (path is a fixture)
from test_gpu_rollup import rollup_raw

pytestmark = pytest.mark.gpu
WIN, TIER, SPAN = abi.ROLLUP_WINDOWS, abi.ROLLUP_TIER, abi.ROLLUP_SPAN
AT_MOST, AT_LEAST = abi.SPAN_AT_MOST, abi.SPAN_AT_LEAST


def score_raw(h, kind, cap):
    """alz_gnn_score_rollup with the status instead of an exception: (status, scores, n_out)."""
    out = np.zeros(max(cap, 1), dtype=np.float32)
    n = C.c_size_t(12345)
    rc = h.L.alz_gnn_score_rollup(h.h, int(kind), out.ctypes.data_as(C.c_void_p) if cap else None, cap, C.byref(n))
    return rc, out, n.value


def nodes(h, n_rows):
    """alz_gnn_nodes of the last GNN pass: (node keys, h2)."""
    keys = np.zeros(max(2 * n_rows, 1), dtype=np.uint64)
    h2 = np.zeros((len(keys), 64), dtype=np.float32)
    nv = C.c_size_t(0)
    h._ck(h.L.alz_gnn_nodes(h.h, keys.ctypes.data_as(C.c_void_p), h2.ctypes.data_as(C.c_void_p), len(keys),
                            C.byref(nv)), "alz_gnn_nodes")
    return keys[: nv.value], h2[: nv.value]


def score_and_check(h, kind, rows, what):
    """Scores of the last rollup of `kind` against gnn_ref on its rows; returns the scores."""
    scores = h.gnn_score_rollup(kind)
    assert len(scores) == len(rows), (what, len(scores), len(rows))
    keys, h2 = nodes(h, len(rows))
    check(rows, scores, keys, h2, what)
    return scores


def universe(n_pods=700, n_svcs=24, n_out=6, n_edges=3000, seed=0):
    """Distinct edges pod -> pod (some reversed), pod -> service, service -> pod, pod -> outbound; 1..3 events each,
    lognormal durations, 1 in 8 with status 500."""
    rng = np.random.default_rng(seed)
    outs = np.array([abi.ip("8.8.8.8"), abi.ip("203.0.113.7"), 1, 0xFFFFFFFE, 0xFFFFFFFF, abi.ip("198.51.100.9")])
    items = set()
    while len(items) < n_edges:
        k = rng.integers(0, 10)
        p, q = int(rng.integers(0, n_pods)), int(rng.integers(0, n_pods))
        if k < 5:
            items.add(((gg.POD, p), (gg.POD, q), k == 0))
        elif k < 8:
            items.add(((gg.POD, p), (gg.SVC, int(rng.integers(0, n_svcs))), False))
        elif k < 9:
            items.add(((gg.SVC, int(rng.integers(0, n_svcs))), (gg.POD, q), False))
        else:
            items.add(((gg.POD, p), (gg.OUT, int(outs[rng.integers(0, n_out)])), False))
    edges = sorted(items)
    ft = np.array([a[0] for a, _, _ in edges], np.uint8)
    fv = np.array([a[1] for a, _, _ in edges], np.uint64)
    tt = np.array([b[0] for _, b, _ in edges], np.uint8)
    tv = np.array([b[1] for _, b, _ in edges], np.uint64)
    cnt = 1 + rng.integers(0, 3, len(edges))
    ee = np.repeat(np.arange(len(edges)), cnt)
    dur = np.exp(rng.normal(np.log(2e6), 1.0, len(ee))).astype(np.uint64)
    status = np.where(rng.random(len(ee)) < 0.125, 500, 200)
    return gg.Graph(ft, fv, tt, tv, ee, dur, status, rev=np.array([r for _, _, r in edges]))


class Stream:
    """One handle with the universe's tables: window(edges) submits the records of those edges, with durations scaled
    per window so that no two windows carry the same histograms, and flushes."""

    def __init__(self, g, history=None, tiers=(), **kw):
        self.g, self.b = g, gg.Built(g)
        kw.setdefault("max_endpoints", len(self.b.pod_ip) + len(self.b.svc_ip) + 16)
        kw.setdefault("max_pairs", 1 << max(12, int(np.ceil(np.log2(2 * g.n_edges)))))
        self.h = capi.Handle(**kw)
        gg.load(self.h, self.b)
        if history:
            self.h.window_history(*history)
        if tiers:
            self.h.window_history_tiers(tiers)
        self.rng = np.random.default_rng(7)

    def window(self, edges):
        recs = self.b.recs[np.isin(self.g.ev_edge, edges)].copy()
        recs["duration_ns"] = (recs["duration_ns"] * self.rng.uniform(0.5, 4.0)).astype(np.uint64)
        if len(recs):
            self.h.submit(recs)
        return self.h.flush()

    def random_windows(self, n, seed, lo=0.3, hi=0.8):
        rng = np.random.default_rng(seed)
        return [self.window(np.flatnonzero(rng.random(self.g.n_edges) < rng.uniform(lo, hi))) for _ in range(n)]

    def close(self):
        self.h.close()


# ---- the three kinds against gnn_ref ---------------------------------------------------------------------------

def test_window_rollups_every_k(path):
    s = Stream(universe(seed=1), history=(5, 1 << 15))
    s.random_windows(3, seed=11)
    s.window(np.arange(0, 40))                                   # a small window: most edges vanish, then come back
    s.random_windows(3, seed=12)
    for k in range(1, 7):                                        # 6 > depth: every retained window
        rows, info = s.h.rollup(k)
        assert info["windows"] == min(k, 5)
        score_and_check(s.h, WIN, rows, f"window rollup k={k}")
    s.close()


def test_tier_rollups_with_a_tier_2_entry(path):
    s = Stream(universe(seed=2), tiers=[(2, 4, 1 << 15, 1 << 13), (2, 2, 1 << 15, 1 << 14)])
    s.random_windows(9, seed=21, lo=0.1, hi=0.5)
    assert s.h.tier_state(2)["entries"] == 2
    for tier, k in ((1, 1), (1, 3), (1, 4), (2, 1), (2, 2)):
        rows, info = s.h.rollup_tier(tier, k)
        assert info["windows"] == k * (2 if tier == 1 else 4)
        score_and_check(s.h, TIER, rows, f"tier {tier} k={k}")
    s.close()


def test_span_rollups_of_history_tier_entries_and_an_open_block(path):
    s = Stream(universe(seed=3), history=(3, 1 << 15), tiers=[(2, 4, 1 << 15, 1 << 13), (2, 2, 1 << 15, 1 << 14)])
    s.random_windows(11, seed=31, lo=0.1, hi=0.5)
    kinds = set()
    for N, mode in ((1, AT_MOST), (2, AT_MOST), (3, AT_LEAST), (5, AT_MOST), (7, AT_LEAST), (11, AT_MOST),
                    (100, AT_LEAST)):
        rows, info = s.h.rollup_span(N, mode)
        kinds |= {("history" if t == 0 else "tier") for t, e in enumerate(info["entries"]) if e}
        kinds |= {"open"} if info["open_blocks"] else set()
        score_and_check(s.h, SPAN, rows, f"span {N} {mode}")
    assert kinds == {"history", "tier", "open"}, kinds
    s.close()


def test_hub_in_degree_built_up_over_windows(path):
    """10^5 identical clients of one service, a tenth of them in each of 10 windows: the hub's float64 neighbour sum
    over 10^5 rows is only reached in the rollup."""
    g = _star(100_000, 2, 1_500_000)
    b = gg.Built(g)
    h = capi.Handle(max_endpoints=len(b.pod_ip) + len(b.svc_ip) + 16, max_pairs=1 << 15)
    gg.load(h, b)
    h.window_history(10, 1 << 17)
    for w in range(10):
        h.submit(b.recs[g.ev_edge % 10 == w])
        assert len(h.flush()) == 10_000
    rows, _ = h.rollup(10)
    assert len(rows) == 100_000
    score_and_check(h, WIN, rows, "hub over 10 windows")
    h.close()


# ---- bit for bit -------------------------------------------------------------------------------------------------

def test_one_window_rollup_scores_as_the_window(path):
    s = Stream(universe(seed=4), history=(3, 1 << 15))
    for w in range(4):
        flushed = s.random_windows(1, seed=41 + w)[0]
        win_scores, keys, h2 = gg.gnn(s.h, len(flushed))
        rows, _ = s.h.rollup(1)
        assert rows.tobytes() == flushed.tobytes()
        roll_scores = s.h.gnn_score_rollup(WIN)
        assert roll_scores.tobytes() == win_scores.tobytes(), w
        rkeys, rh2 = nodes(s.h, len(rows))
        assert rkeys.tobytes() == keys.tobytes() and rh2.tobytes() == h2.tobytes()
    s.close()


def test_history_span_scores_as_the_window_rollup(path):
    s = Stream(universe(seed=5), history=(6, 1 << 15))
    s.random_windows(6, seed=51)
    for N in (1, 2, 4, 6):
        span_rows, info = s.h.rollup_span(N, AT_MOST)
        assert info["windows"] == N and info["entries"][0] == N
        span_scores = s.h.gnn_score_rollup(SPAN)
        rows, _ = s.h.rollup(N)
        assert rows.tobytes() == span_rows.tobytes()
        assert s.h.gnn_score_rollup(WIN).tobytes() == span_scores.tobytes(), N
    s.close()


def test_two_scorings_and_host_and_device_agree_on_a_tiered_handle(path):
    s = Stream(universe(seed=6), history=(4, 1 << 15), tiers=[(2, 4, 1 << 15, 1 << 13), (3, 2, 1 << 15, 1 << 14)])
    s.random_windows(8, seed=61, lo=0.1, hi=0.5)
    for kind, call in ((WIN, lambda: s.h.rollup(3)), (TIER, lambda: s.h.rollup_tier(2, 1)),
                       (SPAN, lambda: s.h.rollup_span(7, AT_LEAST))):
        rows, _ = call()
        a = score_and_check(s.h, kind, rows, f"kind {kind}")
        b = s.h.gnn_score_rollup(kind)
        p, n = s.h.gnn_score_rollup_device(kind)
        assert n == len(rows)
        s.h.sync()
        c = s.h.d2h(p, n, np.float32)
        assert a.tobytes() == b.tobytes() == c.tobytes(), kind
        again, _ = call()                                       # the call read only: the rows are still the same
        assert again.tobytes() == rows.tobytes()
    s.close()


# ---- growth above max_edges --------------------------------------------------------------------------------------

def test_rollup_above_max_edges_then_a_window_then_a_smaller_rollup(path):
    """max_edges = 1024: 20 windows of 1000 disjoint edges make a 20,000-row rollup. The GNN state grows for it; a
    window and a smaller rollup scored after it must see none of the grown buffers' stale rows or nodes."""
    g = universe(n_pods=9000, n_svcs=40, n_edges=20_000, seed=7)
    s = Stream(g, history=(20, 1 << 15), max_pairs=1 << 13, max_edges=1024)
    rng = np.random.default_rng(71)
    perm = rng.permutation(g.n_edges)
    for w in range(20):
        assert len(s.window(perm[w * 1000:(w + 1) * 1000])) == 1000
    rows, _ = s.h.rollup(20)
    assert len(rows) == 20_000
    score_and_check(s.h, WIN, rows, "20k rows on max_edges 1024")
    flushed = s.window(perm[:600])
    scores, keys, h2 = gg.gnn(s.h, len(flushed))
    check(flushed, scores, keys, h2, "window after the growth")
    rows, _ = s.h.rollup(2)
    assert len(rows) == 1000 + 600 - len(np.intersect1d(perm[:600], perm[19_000:]))
    score_and_check(s.h, WIN, rows, "smaller rollup after the growth")
    rows, _ = s.h.rollup(20)                                     # and the grown state once more
    score_and_check(s.h, WIN, rows, "20 windows again")
    s.close()


# ---- states --------------------------------------------------------------------------------------------------------

def test_no_rows_before_a_rollup_and_after_a_failed_one():
    s = Stream(universe(n_edges=400, seed=8), history=(3, 1 << 14), tiers=[(2, 3, 1 << 14, 1 << 12)])
    for kind in (WIN, TIER, SPAN):
        assert score_raw(s.h, kind, 0)[0] == abi.E_STATE, kind
    s.random_windows(4, seed=81)
    assert score_raw(s.h, WIN, 0)[0] == abi.E_STATE              # flushes alone leave nothing to score
    # window kind: a host rollup that returned ALZ_E_CAPACITY, then k = 0
    rows, _ = s.h.rollup(2)
    score_and_check(s.h, WIN, rows, "window")
    rc, _, n, _ = rollup_raw(s.h, 2, 1)
    assert rc == abi.E_CAPACITY and n == len(rows)
    assert score_raw(s.h, WIN, 0)[0] == abi.E_STATE
    s.h.rollup(2)
    assert score_raw(s.h, WIN, 0)[0] == abi.E_CAPACITY
    assert rollup_raw(s.h, 0, 0)[0] == abi.E_INVAL
    assert score_raw(s.h, WIN, 0)[0] == abi.E_STATE
    # tier kind: too small, k = 0 and a tier above the configured ones
    for bad in ((1, 1, 1), (1, 0, 0), (2, 1, 0)):
        rows, _ = s.h.rollup_tier(1, 2)
        assert len(s.h.gnn_score_rollup(TIER)) == len(rows)
        out = np.zeros(1, dtype=abi.EDGE_OUT)
        n = C.c_size_t(0)
        rc = s.h.L.alz_window_rollup_tier(s.h.h, bad[0], bad[1], out.ctypes.data_as(C.c_void_p) if bad[2] else None,
                                          bad[2], C.byref(n), None)
        assert rc in (abi.E_CAPACITY, abi.E_INVAL), rc
        assert score_raw(s.h, TIER, 0)[0] == abi.E_STATE, bad
    # span kind: too small, N = 0
    for N, cap in ((4, 1), (0, 0)):
        rows, _ = s.h.rollup_span(4, AT_LEAST)
        assert len(s.h.gnn_score_rollup(SPAN)) == len(rows)
        out = np.zeros(1, dtype=abi.EDGE_OUT)
        n, info = C.c_size_t(0), abi.SpanInfo()
        rc = s.h.L.alz_window_rollup_span(s.h.h, N, AT_LEAST, out.ctypes.data_as(C.c_void_p) if cap else None, cap,
                                          C.byref(n), C.byref(info))
        assert rc in (abi.E_CAPACITY, abi.E_INVAL), rc
        assert score_raw(s.h, SPAN, 0)[0] == abi.E_STATE, N
    s.close()


def test_reconfiguring_drops_its_own_kind_only(path):
    hist, tiers = (3, 1 << 14), [(2, 3, 1 << 14, 1 << 12)]
    s = Stream(universe(n_edges=500, seed=9), history=hist, tiers=tiers)
    s.random_windows(5, seed=91)
    wrows, _ = s.h.rollup(3)
    trows, _ = s.h.rollup_tier(1, 2)
    srows, _ = s.h.rollup_span(5, AT_LEAST)
    before = {k: s.h.gnn_score_rollup(k).tobytes() for k in (WIN, TIER, SPAN)}
    s.h.window_history(*hist)                                    # the current values change nothing
    s.h.window_history_tiers(tiers)
    assert {k: s.h.gnn_score_rollup(k).tobytes() for k in (WIN, TIER, SPAN)} == before
    score_and_check(s.h, WIN, wrows, "window after the same history")
    score_and_check(s.h, TIER, trows, "tier after the same tiers")
    s.h.window_history(4, 1 << 14)                               # other values: the window rows go
    assert score_raw(s.h, WIN, 0)[0] == abi.E_STATE
    assert s.h.gnn_score_rollup(TIER).tobytes() == before[TIER]
    s.h.window_history_tiers([(3, 3, 1 << 14, 1 << 12)])         # and the tier rows
    assert score_raw(s.h, TIER, 0)[0] == abi.E_STATE
    assert s.h.gnn_score_rollup(SPAN).tobytes() == before[SPAN]  # span rows survive both
    score_and_check(s.h, SPAN, srows, "span after both reconfigurations")
    s.close()


def test_window_and_tier_kinds_do_not_see_each_others_rows(path):
    s = Stream(universe(n_edges=800, seed=10), history=(4, 1 << 14), tiers=[(2, 3, 1 << 14, 1 << 12)])
    s.random_windows(6, seed=101, lo=0.1, hi=0.3)
    trows, _ = s.h.rollup_tier(1, 3)
    assert score_raw(s.h, WIN, 0)[0] == abi.E_STATE              # a tier rollup is not a window rollup
    score_and_check(s.h, TIER, trows, "tier")
    wrows, _ = s.h.rollup(1)
    assert len(wrows) != len(trows)
    score_and_check(s.h, WIN, wrows, "window after a tier rollup")
    score_and_check(s.h, TIER, trows, "tier after a window rollup")
    w0, _ = s.h.rollup_tier(0, 2)                                # tier 0 is the window history: the window kind
    score_and_check(s.h, WIN, w0, "tier 0")
    score_and_check(s.h, TIER, trows, "tier after tier 0")
    s.close()


def test_empty_span_small_cap_and_unknown_kind():
    s = Stream(universe(n_edges=300, seed=12), tiers=[(2, 3, 1 << 14, 1 << 12)])
    s.random_windows(2, seed=121)
    rows, info = s.h.rollup_span(1, AT_MOST)                     # one closed entry of 2 windows, an empty open block
    assert len(rows) == 0 and info["windows"] == 0
    rc, _, n = score_raw(s.h, SPAN, 0)
    assert rc == abi.OK and n == 0
    p, n = s.h.gnn_score_rollup_device(SPAN)
    assert n == 0
    keys, _ = nodes(s.h, 0)
    assert len(keys) == 0
    rows, _ = s.h.rollup_span(2, AT_MOST)
    assert len(rows) > 1
    rc, out, n = score_raw(s.h, SPAN, len(rows) - 1)
    assert rc == abi.E_CAPACITY and n == len(rows) and not out.any()
    rc, out, n = score_raw(s.h, SPAN, len(rows))
    assert rc == abi.OK and n == len(rows)
    for kind in (3, 0xFFFFFFFF):
        assert score_raw(s.h, kind, 0)[:3:2] == (abi.E_INVAL, 0)
        p, n = C.c_void_p(), C.c_size_t(7)
        assert s.h.L.alz_gnn_score_rollup_device(s.h.h, kind, C.byref(p), C.byref(n)) == abi.E_INVAL and n.value == 0
    s.close()
