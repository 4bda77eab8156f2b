"""GPU: the top anomalous rows (alz_gnn_top*, alz_debug_top_scores, docs/SPEC.md §16).

The expected result is tests/top_ref.py over the scores alz_gnn_score* returns for the same rows, and it must match
exactly: row bytes, score bits and indices. The selection alone is driven through alz_debug_top_scores with score
distributions the GNN never produces: ties of every size at the threshold, keys that differ in one digit only, the
IEEE specials."""
import ctypes as C

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings, strategies as st

import gnn_graphs as gg
import oracle_lib as ol
import top_ref
from alaz_b200 import abi, capi
from test_gpu_gnn import _star, path, pod_graph  # noqa: F401  (path is a fixture)
from test_gpu_gnn_rollup import Stream, nodes, universe

pytestmark = pytest.mark.gpu
WIN, TIER, SPAN = abi.ROLLUP_WINDOWS, abi.ROLLUP_TIER, abi.ROLLUP_SPAN
F = np.float32
SPECIALS = np.array([0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x007FFFFF, 0x3F800000, 0x7F800000, 0xFF800000,
                     0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFFFFFFF], np.uint32).view(F)


@pytest.fixture(scope="module")
def hh():
    h = capi.Handle(max_endpoints=64, max_pairs=1 << 12)
    yield h
    h.close()


def hook(h, scores, k, min_score, cap=None, with_index=True):
    """alz_debug_top_scores over `scores` copied to the device: (status, index, n_out, above)."""
    scores = np.ascontiguousarray(scores, dtype=F)
    d = h.dev_alloc(max(scores.nbytes, 4))
    try:
        h.h2d(d, scores)
        cap = min(int(k), len(scores)) if cap is None else cap
        index = np.full(max(cap, 1), 0xDEADBEEF, np.uint32)
        n, above = C.c_size_t(12345), C.c_uint64(777)
        rc = h.L.alz_debug_top_scores(h.h, C.c_void_p(d), len(scores), int(k), float(min_score),
                                      index.ctypes.data_as(C.c_void_p) if with_index else None, cap, C.byref(n),
                                      C.byref(above))
    finally:
        h.dev_free(d)
    return rc, index, n.value, above.value


def check_hook(h, scores, k, min_score, what=""):
    rc, index, n, above = hook(h, scores, k, min_score)
    assert rc == 0, (what, rc)
    exp, exp_above = top_ref.top(scores, k, min_score)
    assert above == exp_above, (what, above, exp_above)
    assert n == len(exp), (what, n, len(exp))
    assert np.array_equal(index[:n], exp), (what, index[:n][:20], exp[:20])
    return n


# ---- the selection alone ----------------------------------------------------------------------------------------

def distributions(n, rng):
    """name -> scores of length n."""
    u = np.arange(n, dtype=np.uint32)
    out = {
        "equal": np.full(n, 0.75, F),
        "ascending": (u.astype(np.float64) / max(n, 1)).astype(F),
        "descending": ((n - u).astype(np.float64) / max(n, 1)).astype(F),
        "low_digit": (np.uint32(0x3F000000) | (rng.integers(0, 1 << 10, n).astype(np.uint32))).view(F),
        "high_digit": ((rng.integers(0, 1 << 11, n).astype(np.uint32) << np.uint32(21)) | np.uint32(0x1234)).view(F),
        "two_values": np.where(rng.random(n) < 0.5, F(0.25), F(0.5)).astype(F),
        "specials": rng.choice(SPECIALS, n),
        "random": rng.random(n).astype(F),
    }
    return out


@pytest.mark.parametrize("n", [1, 2, 4095, 4096, 4097, 100_003])
def test_hook_adversarial_distributions(hh, n):
    rng = np.random.default_rng(n)
    for name, s in distributions(n, rng).items():
        present = float(s[rng.integers(0, n)])
        mins = [float("-inf"), 0.0, present, 0.6, 2.0]
        if np.isnan(present):
            mins[2] = 0.5
        for k in sorted({1, 2, 2048, max(n - 1, 1), n, n + 5}):
            for ms in mins:
                check_hook(hh, s, k, ms, f"{name} n={n} k={k} min={ms}")


def test_hook_min_score_positions(hh):
    s = np.array([0.1, 0.3, 0.3, 0.7, 0.9, 0.0, -0.0], F)
    assert check_hook(hh, s, 10, 0.3) == 4                  # equal to a present value
    assert check_hook(hh, s, 10, 0.5) == 2                  # between two values
    rc, _, n, above = hook(hh, s, 10, 0.95)                 # above all of them
    assert (rc, n, above) == (0, 0, 0)
    assert check_hook(hh, s, 10, -1.0) == 7                 # below all of them
    assert check_hook(hh, s, 10, 0.0) == 6                  # +0 is eligible, -0 is not


def test_hook_large(hh):
    n = 1 << 26
    rng = np.random.default_rng(26)
    s = (rng.integers(0, 1 << 24, n, dtype=np.uint32) | np.uint32(0x3E000000)).view(F)   # many ties among 2^26
    for k in (1, 1000, 100_000):
        check_hook(hh, s, k, 0.0, f"2^26 k={k}")
    check_hook(hh, np.full(n, 0.5, F), 100_000, 0.5, "2^26 equal")


@settings(max_examples=60, deadline=None, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(st.lists(st.sampled_from([0.0, -0.0, 0.25, 0.5, 0.5000001, 1.0, float("inf"), float("-inf"), float("nan"),
                                 1e-45, -1e-45]), min_size=1, max_size=300),
       st.integers(1, 320), st.sampled_from([float("-inf"), 0.0, -0.0, 0.25, 0.5, 2.0]))
def test_hook_property_small_arrays(hh, vals, k, ms):
    check_hook(hh, np.array(vals, F), k, ms)


def test_hook_contract(hh):
    s = np.random.default_rng(1).random(5000).astype(F)
    rc, index, n, above = hook(hh, s, 100, 0.0, cap=99)     # cap too small: n set, nothing written
    assert rc == abi.E_CAPACITY and n == 100 and above == 5000 and np.all(index == 0xDEADBEEF)
    rc, _, n, above = hook(hh, s, 100, 0.0, cap=0, with_index=False)
    assert rc == abi.E_CAPACITY and n == 100
    rc, _, n, _ = hook(hh, s, 100, 0.0, with_index=False)
    assert rc == 0 and n == 100
    assert hook(hh, s, 0, 0.0)[0] == abi.E_INVAL
    assert hook(hh, s, 1, float("nan"))[0] == abi.E_INVAL
    n_out, above = C.c_size_t(5), C.c_uint64(5)
    assert hh.L.alz_debug_top_scores(hh.h, None, 0, 3, 0.0, None, 0, C.byref(n_out), C.byref(above)) == 0
    assert n_out.value == 0 and above.value == 0
    rc = hh.L.alz_debug_top_scores(hh.h, C.c_void_p(16), 1 << 30, 3, 0.0, None, 0, C.byref(n_out), None)
    assert rc == abi.E_CAPACITY


# ---- through the GNN pass ----------------------------------------------------------------------------------------

def expect(rows, scores, k, min_score, got, what=""):
    """got = (rows, scores, index, info) of a top call over `rows` whose pass scored `scores`."""
    g_rows, g_scores, g_index, info = got
    idx, above = top_ref.top(scores, k, min_score)
    assert info == {"scored": len(rows), "above": above}, (what, info, above)
    assert np.array_equal(g_index, idx), (what, g_index[:10], idx[:10])
    assert g_scores.view(np.uint32).tobytes() == scores[idx].view(np.uint32).tobytes(), what
    assert g_rows.tobytes() == rows[idx].tobytes(), what


def window_scores(h, n):
    scores = np.zeros(max(n, 1), F)
    nn = C.c_size_t(0)
    h._ck(h.L.alz_gnn_score(h.h, scores.ctypes.data_as(C.c_void_p), len(scores), C.byref(nn)), "alz_gnn_score")
    return scores[: nn.value]


def test_window_source_synthetic_stream(path):
    t = ol.Topo(300, seed=1300, mix=abi.MIX_ALL)
    h = capi.Handle(max_endpoints=1200, max_pairs=1 << 17)
    h.load_tables(t.pod_ip, t.svc_ip)
    h.submit(t.events(0, 400_000))
    rows = h.flush()
    n = len(rows)
    assert n > 2000
    scores = window_scores(h, n)
    for k in (1, 10, 1000, n, n + 5):
        for ms in (0.0, float(np.median(scores))):
            expect(rows, scores, k, ms, h.gnn_top(k, ms), f"window k={k} min={ms}")
    fetched = np.zeros(n, dtype=abi.EDGE_OUT)
    nf = C.c_size_t(0)
    h._ck(h.L.alz_window_fetch(h.h, fetched.ctypes.data_as(C.c_void_p), n, C.byref(nf)), "alz_window_fetch")
    assert nf.value == n and fetched.tobytes() == rows.tobytes()
    h.close()


def test_rollup_sources(path):
    s = Stream(universe(seed=5), history=(4, 1 << 15), tiers=[(2, 4, 1 << 15, 1 << 13)])
    s.random_windows(7, seed=51, lo=0.2, hi=0.6)
    cases = [(WIN, lambda: s.h.rollup(3)[0]), (WIN, lambda: s.h.rollup(1)[0]), (TIER, lambda: s.h.rollup_tier(1, 3)[0]),
             (SPAN, lambda: s.h.rollup_span(6, abi.SPAN_AT_LEAST)[0])]
    for kind, roll in cases:
        rows = roll()
        scores = s.h.gnn_score_rollup(kind)
        for k in (1, 10, 1000, len(rows) + 5):
            for ms in (0.0, 0.5):
                expect(rows, scores, k, ms, s.h.gnn_top_rollup(kind, k, ms), f"kind {kind} k={k} min={ms}")
    s.close()


def test_rollup_above_max_edges_grows(path):
    s = Stream(universe(seed=6, n_edges=3000), history=(6, 1 << 14), max_edges=1024, max_pairs=1 << 13)
    for j in range(6):
        s.window(np.arange(j * 500, j * 500 + 500))
    rows, _ = s.h.rollup(6)
    assert len(rows) > 1024
    top = s.h.gnn_top_rollup(WIN, 50, 0.0)                  # first GNN call: the state grows here
    scores = s.h.gnn_score_rollup(WIN)
    expect(rows, scores, 50, 0.0, top, "grown")
    expect(rows, scores, 3000, 0.0, s.h.gnn_top_rollup(WIN, 3000, 0.0), "grown, all")
    s.close()


def _ties(g, ks):
    b = gg.Built(g)
    h = gg.handle_for(b)
    gg.load(h, b)
    rows = gg.ingest(h, b, check=False)
    scores = window_scores(h, len(rows))
    assert len(np.unique(scores)) < len(scores)                       # the pass itself made ties
    for k in ks:
        got = h.gnn_top(k, 0.0)
        expect(rows, scores, k, 0.0, got, f"ties k={k}")
        eq = np.diff(got[1].view(np.uint32).astype(np.int64)) == 0
        assert np.all(np.diff(got[2].astype(np.int64))[eq] > 0)       # equal scores: index order
    h.close()


def test_ties_perfect_matching(path):
    n_e = 100_000
    _ties(pod_graph(2 * np.arange(n_e), 2 * np.arange(n_e) + 1, seed=3), (1, 777, 50_000, n_e))


def test_ties_hub_of_identical_clients(path):
    _ties(_star(50_000, 3, 1_500_000), (1, 10, 30_000, 50_001))


# ---- the contract --------------------------------------------------------------------------------------------------

def raw_top(h, kind, k, ms, cap, rows=True, scores=True, index=True, info=True):
    """alz_gnn_top (kind None) or alz_gnn_top_rollup with sentinel buffers: (status, rows, scores, index, n, info)."""
    rr = np.frombuffer(bytearray(b"\xab" * (max(cap, 1) * abi.EDGE_OUT.itemsize)), dtype=abi.EDGE_OUT)
    ss = np.full(max(cap, 1), 0x7F7F7F7F, np.uint32).view(F)
    ii = np.full(max(cap, 1), 0xDEADBEEF, np.uint32)
    n, inf = C.c_size_t(12345), abi.TopInfo(7, 7)
    p = lambda a, on: a.ctypes.data_as(C.c_void_p) if on else None  # noqa: E731
    args = (int(k), float(ms), p(rr, rows), p(ss, scores), p(ii, index), cap, C.byref(n), C.byref(inf) if info else None)
    rc = h.L.alz_gnn_top(h.h, *args) if kind is None else h.L.alz_gnn_top_rollup(h.h, int(kind), *args)
    return rc, rr, ss, ii, n.value, inf.as_dict()


def test_errors_and_capacity():
    s = Stream(universe(seed=8, n_edges=800), history=(3, 1 << 14))
    h = s.h
    assert raw_top(h, None, 5, 0.0, 5)[0] == 0 and raw_top(h, None, 5, 0.0, 5)[4] == 0     # no window yet: 0 rows
    for kind in (WIN, TIER, SPAN):
        rc, _, _, _, n, _ = raw_top(h, kind, 5, 0.0, 5)
        assert rc == abi.E_STATE and n == 0, kind
    rows = s.window(np.arange(0, 600))
    assert raw_top(h, None, 0, 0.0, 5)[0] == abi.E_INVAL
    assert raw_top(h, None, 5, float("nan"), 5)[0] == abi.E_INVAL
    assert raw_top(h, 3, 5, 0.0, 5)[0] == abi.E_INVAL
    assert raw_top(h, 0xFFFFFFFF, 5, 0.0, 5)[0] == abi.E_INVAL
    rc, rr, ss, ii, n, _ = raw_top(h, None, 20, 0.0, 19)                     # cap too small
    assert rc == abi.E_CAPACITY and n == 20
    assert set(rr.view(np.uint8).tolist()) == {0xAB} and np.all(ss.view(np.uint32) == 0x7F7F7F7F)
    assert np.all(ii == 0xDEADBEEF)
    rc, _, _, _, n, _ = raw_top(h, None, 20, 0.0, 0, rows=False, scores=False, index=False, info=False)
    assert rc == abi.E_CAPACITY and n == 20
    full = raw_top(h, None, 20, 0.0, 20)
    for flags in ((False, True, True), (True, False, True), (True, True, False), (False, False, False)):
        rc, rr, ss, ii, n, inf = raw_top(h, None, 20, 0.0, 20, *flags, info=False)
        assert rc == 0 and n == 20, flags
        for got, want, on in ((rr, full[1], flags[0]), (ss, full[2], flags[1]), (ii, full[3], flags[2])):
            if on:
                assert got[:20].tobytes() == want[:20].tobytes(), flags
    assert full[5] == {"scored": len(rows), "above": len(rows)}
    h.rollup(2)
    assert h.gnn_top_rollup(WIN, 5)[3]["scored"] > 0
    s.close()


def test_zero_row_rollup_and_window():
    s = Stream(universe(seed=9, n_edges=300), history=(3, 1 << 14))
    s.window(np.array([], np.int64))
    rows, info = s.h.rollup(1)
    assert len(rows) == 0
    r = s.h.gnn_top_rollup(WIN, 5)
    assert len(r[0]) == 0 and r[3] == {"scored": 0, "above": 0}
    r = s.h.gnn_top(5)
    assert len(r[0]) == 0 and r[3] == {"scored": 0, "above": 0}
    s.close()


def test_device_variant_repeats_nodes_and_reads_only(path):
    s = Stream(universe(seed=10), history=(4, 1 << 15), tiers=[(2, 3, 1 << 15, 1 << 13)])
    s.random_windows(5, seed=101)
    h = s.h
    last = s.window(np.arange(100, 2500))
    for kind, roll in ((None, None), (WIN, lambda: h.rollup(3)[0]), (TIER, lambda: h.rollup_tier(1, 2)[0]),
                       (SPAN, lambda: h.rollup_span(5, abi.SPAN_AT_MOST)[0])):
        rows = last if kind is None else roll()
        k = 300
        host = h.gnn_top(k, 0.2) if kind is None else h.gnn_top_rollup(kind, k, 0.2)
        again = h.gnn_top(k, 0.2) if kind is None else h.gnn_top_rollup(kind, k, 0.2)
        for a, b in zip(host[:3], again[:3]):
            assert a.tobytes() == b.tobytes(), kind                       # repeated calls: bitwise identical
        keys_top, h2_top = nodes(h, len(rows))                             # alz_gnn_nodes refers to the top call's pass
        pr, ps, pi, n, info = h.gnn_top_device(k, 0.2) if kind is None else h.gnn_top_rollup_device(kind, k, 0.2)
        assert n == len(host[0]) and info == host[3]
        h.sync()
        assert h.d2h(pr, n, abi.EDGE_OUT).tobytes() == host[0].tobytes()
        assert h.d2h(ps, n, F).tobytes() == host[1].tobytes()
        assert h.d2h(pi, n, np.uint32).tobytes() == host[2].tobytes()
        scores = window_scores(h, len(rows)) if kind is None else h.gnn_score_rollup(kind)   # still scorable
        keys, h2 = nodes(h, len(rows))
        assert keys.tobytes() == keys_top.tobytes() and h2.tobytes() == h2_top.tobytes(), kind
        expect(rows, scores, k, 0.2, host, f"kind {kind}")
    fetched = np.zeros(len(last), dtype=abi.EDGE_OUT)
    nf = C.c_size_t(0)
    h._ck(h.L.alz_window_fetch(h.h, fetched.ctypes.data_as(C.c_void_p), len(last), C.byref(nf)), "alz_window_fetch")
    assert fetched[: nf.value].tobytes() == last.tobytes()
    s.close()


def test_next_flush_unchanged_by_top_calls():
    """Two handles fed the same windows; one runs top calls between flushes: the flushes are identical."""
    a = Stream(universe(seed=12), history=(3, 1 << 15))
    b = Stream(universe(seed=12), history=(3, 1 << 15))
    rng = np.random.default_rng(3)
    for j in range(4):
        edges = np.flatnonzero(rng.random(a.g.n_edges) < 0.5)
        ra, rb = a.window(edges), b.window(edges)
        assert ra.tobytes() == rb.tobytes(), j
        a.h.gnn_top(25, 0.1)
        a.h.rollup(2)
        a.h.gnn_top_rollup(WIN, 25)
    a.close()
    b.close()
