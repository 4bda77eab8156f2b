"""GPU: the top edges by a metric (alz_edge_top*, alz_debug_top_keys64, docs/SPEC.md §17).

The expected result is tests/metric_ref.py: its values of the same rows and its rank order, and it must match
exactly: row bytes, value bits and indices. The 64-bit selection alone is driven through alz_debug_top_keys64 with
value distributions no metric produces: keys that differ in one digit of each of the six digit passes, or only in the
lowest bit, n-way ties, the IEEE specials."""
import ctypes as C

import numpy as np
import pytest

import metric_ref as mr
from alaz_b200 import abi, capi
from test_gpu_gnn_rollup import Stream, universe

pytestmark = pytest.mark.gpu
WIN, TIER, SPAN = abi.ROLLUP_WINDOWS, abi.ROLLUP_TIER, abi.ROLLUP_SPAN
Q = abi.METRIC_QUANTILE
KINDS = [abi.METRIC_COUNT, abi.METRIC_ERR5XX, abi.METRIC_ERR_RATE, abi.METRIC_MEAN_NS, (Q, 0.5), (Q, 0.99), (Q, 1.0)]
SPECIALS = np.array([0x0, 1 << 63, 0x1, 0x000FFFFFFFFFFFFF, 0x3FF0000000000000, 0x7FF0000000000000,
                     0x7FEFFFFFFFFFFFFF, 0x8000000000000001, 0xFFF0000000000000], np.uint64).view(np.float64)


@pytest.fixture(scope="module")
def hh():
    h = capi.Handle(max_endpoints=64, max_pairs=1 << 12)
    yield h
    h.close()


def hook(h, values, k, min_value, cap=None, with_index=True):
    """alz_debug_top_keys64 over `values` copied to the device: (status, index, n_out, above)."""
    values = np.ascontiguousarray(values, dtype=np.float64)
    d = h.dev_alloc(max(values.nbytes, 8))
    try:
        h.h2d(d, values)
        cap = min(int(k), len(values)) if cap is None else cap
        index = np.full(max(cap, 1), 0xDEADBEEF, np.uint32)
        n, above = C.c_size_t(12345), C.c_uint64(777)
        rc = h.L.alz_debug_top_keys64(h.h, C.c_void_p(d), len(values), int(k), float(min_value),
                                      index.ctypes.data_as(C.c_void_p) if with_index else None, cap, C.byref(n),
                                      C.byref(above))
    finally:
        h.dev_free(d)
    return rc, index, n.value, above.value


def check_hook(h, values, k, min_value, what=""):
    rc, index, n, above = hook(h, values, k, min_value)
    assert rc == 0, (what, rc)
    exp, exp_above = mr.top(values, k, min_value)
    assert above == exp_above, (what, above, exp_above)
    assert n == len(exp), (what, n, len(exp))
    assert np.array_equal(index[:n], exp), (what, index[:n][:20], exp[:20])
    return n


def distributions(n, rng):
    """name -> float64 values of length n."""
    u = np.arange(n, dtype=np.uint64)
    base = np.uint64(0x4000000000000000)
    out = {
        "equal": np.full(n, 0.75),
        "ascending": u.astype(np.float64) / max(n, 1),
        "descending": (n - u).astype(np.float64) / max(n, 1),
        "lowest_bit": (base | rng.integers(0, 2, n, dtype=np.uint64)).view(np.float64),
        "two_values": np.where(rng.random(n) < 0.5, 0.25, 0.5),
        "specials": rng.choice(SPECIALS, n),
        "random": rng.random(n),
    }
    for d, (shift, bits) in enumerate(((53, 10), (42, 11), (31, 11), (20, 11), (10, 10), (0, 10))):
        # only digit d differs (pass 0's top bit stays clear: positive values)
        out[f"digit{d}"] = ((rng.integers(0, 1 << bits, n, dtype=np.uint64) << np.uint64(shift)) |
                            np.uint64(0x0000000000012345 if shift else 0x0010000000000000)).view(np.float64)
    return out


@pytest.mark.parametrize("n", [1, 2, 4095, 4096, 4097, 100_003])
def test_hook_adversarial_distributions(hh, n):
    rng = np.random.default_rng(n)
    for name, v in distributions(n, rng).items():
        present = float(v[rng.integers(0, n)])
        for k in sorted({1, 2, 2048, max(n - 1, 1), n, n + 5}):
            for ms in (float("-inf"), -0.0, 0.0, present, 0.6, float("inf")):
                check_hook(hh, v, k, ms, f"{name} n={n} k={k} min={ms}")


def test_hook_min_value_positions_and_zero_signs(hh):
    v = np.array([0.1, 0.3, 0.3, 0.7, 0.9, 0.0, -0.0, 5e-324, np.inf])
    assert check_hook(hh, v, 20, 0.3) == 5                  # equal to a present value
    assert check_hook(hh, v, 20, 0.5) == 3                  # between two values
    assert check_hook(hh, v, 20, np.inf) == 1               # +inf only
    assert check_hook(hh, v, 20, -1.0) == 9                 # below all of them
    assert check_hook(hh, v, 20, 0.0) == 8                  # +0 is eligible, -0 is not
    assert check_hook(hh, v, 20, -0.0) == 9
    assert check_hook(hh, v, 20, 5e-324) == 7               # the smallest denormal


def test_hook_large(hh):
    n = 1 << 26
    rng = np.random.default_rng(26)
    v = (rng.integers(0, 1 << 20, n, dtype=np.uint64) << np.uint64(30) | np.uint64(0x3E00000000000000)).view(np.float64)
    for k in (1, 100_000):
        check_hook(hh, v, k, 0.0, f"2^26 k={k}")
    check_hook(hh, np.full(n, 0.5), 100_000, 0.5, "2^26 equal")


def test_hook_contract(hh):
    v = np.random.default_rng(1).random(5000)
    rc, index, n, above = hook(hh, v, 100, 0.0, cap=99)     # cap too small: n set, nothing written
    assert rc == abi.E_CAPACITY and n == 100 and above == 5000 and np.all(index == 0xDEADBEEF)
    rc, _, n, _ = hook(hh, v, 100, 0.0, with_index=False)
    assert rc == 0 and n == 100
    assert hook(hh, v, 0, 0.0)[0] == abi.E_INVAL
    assert hook(hh, v, 1, float("nan"))[0] == abi.E_INVAL
    n_out, above = C.c_size_t(5), C.c_uint64(5)
    assert hh.L.alz_debug_top_keys64(hh.h, None, 0, 3, 0.0, None, 0, C.byref(n_out), C.byref(above)) == 0
    assert n_out.value == 0 and above.value == 0
    assert hh.L.alz_debug_top_keys64(hh.h, C.c_void_p(16), 1 << 30, 3, 0.0, None, 0, C.byref(n_out),
                                     None) == abi.E_CAPACITY


# ---- real sources --------------------------------------------------------------------------------------------------

def expect(rows, spec, k, min_value, got, what=""):
    """got = (rows, values, index, info) of a top call by `spec` over `rows`."""
    g_rows, g_values, g_index, info = got
    v = mr.values(rows, spec)
    idx, above = mr.top(v, k, min_value)
    assert info == {"scored": len(rows), "above": above}, (what, info, above)
    assert np.array_equal(g_index, idx), (what, g_index[:10], idx[:10])
    assert g_values.tobytes() == v[idx].tobytes(), what
    assert g_rows.tobytes() == rows[idx].tobytes(), what


def test_window_source_every_metric():
    s = Stream(universe(seed=31), history=(4, 1 << 15))
    s.random_windows(2, seed=311)
    rows = s.window(np.arange(0, 2900))
    h = s.h
    for spec in KINDS:
        v = mr.values(rows, spec)
        for k in (1, 10, 1000, len(rows), len(rows) + 5):
            for ms in (0.0, float(np.median(v))):
                expect(rows, spec, k, ms, h.edge_top(spec, k, ms), f"{spec} k={k} min={ms}")
    pr, pv, pi, n, info = h.edge_top_device((Q, 0.99), 77)
    host = h.edge_top((Q, 0.99), 77)
    h.sync()
    assert n == 77 and info == host[3]
    pr, pv, pi, n, info = h.edge_top_device((Q, 0.99), 77)
    h.sync()
    assert h.d2h(pr, n, abi.EDGE_OUT).tobytes() == host[0].tobytes()
    assert h.d2h(pv, n, np.float64).tobytes() == host[1].tobytes()
    assert h.d2h(pi, n, np.uint32).tobytes() == host[2].tobytes()
    s.close()


def test_rollup_sources_every_metric():
    s = Stream(universe(seed=32), history=(4, 1 << 15), tiers=[(2, 4, 1 << 15, 1 << 13)])
    s.random_windows(7, seed=321, lo=0.2, hi=0.6)
    h = s.h
    for kind, roll in ((WIN, lambda: h.rollup(3)[0]), (TIER, lambda: h.rollup_tier(1, 3)[0]),
                       (SPAN, lambda: h.rollup_span(6, abi.SPAN_AT_LEAST)[0])):
        rows = roll()
        assert len(rows) > 0
        for spec in KINDS:
            for k in (1, 100, len(rows) + 5):
                expect(rows, spec, k, 0.0, h.edge_top_rollup(kind, spec, k, 0.0), f"kind {kind} {spec} k={k}")
        pr, pv, pi, n, info = h.edge_top_rollup_device(kind, abi.METRIC_ERR5XX, 50)
        h.sync()
        expect(rows, abi.METRIC_ERR5XX, 50, 0.0, (h.d2h(pr, n, abi.EDGE_OUT), h.d2h(pv, n, np.float64),
                                                 h.d2h(pi, n, np.uint32), info), f"device kind {kind}")
    s.close()


def raw_top(h, kind, spec, k, ms, cap, rows=True, values=True, index=True, info=True, m_ptr=True):
    """alz_edge_top (kind None) or alz_edge_top_rollup with sentinel buffers: (status, rows, values, index, n, info)."""
    rr = np.frombuffer(bytearray(b"\xab" * (max(cap, 1) * abi.EDGE_OUT.itemsize)), dtype=abi.EDGE_OUT)
    vv = np.full(max(cap, 1), 7.5)
    ii = np.full(max(cap, 1), 0xDEADBEEF, np.uint32)
    n, inf = C.c_size_t(12345), abi.TopInfo(7, 7)
    p = lambda a, on: a.ctypes.data_as(C.c_void_p) if on else None  # noqa: E731
    m = abi.metrics(spec) if m_ptr else None
    args = (m, int(k), float(ms), p(rr, rows), p(vv, values), p(ii, index), cap, C.byref(n),
            C.byref(inf) if info else None)
    rc = h.L.alz_edge_top(h.h, *args) if kind is None else h.L.alz_edge_top_rollup(h.h, int(kind), *args)
    return rc, rr, vv, ii, n.value, inf.as_dict()


def test_errors_and_capacity():
    s = Stream(universe(seed=33, n_edges=800), history=(3, 1 << 14))
    h = s.h
    rc, *_, n, _ = raw_top(h, None, abi.METRIC_COUNT, 5, 0.0, 5)               # no window yet: 0 rows
    assert rc == 0 and n == 0
    for kind in (WIN, TIER, SPAN):
        rc, *_, n, _ = raw_top(h, kind, abi.METRIC_COUNT, 5, 0.0, 5)
        assert rc == abi.E_STATE and n == 0, kind
    rows = s.window(np.arange(0, 600))
    assert raw_top(h, None, abi.METRIC_COUNT, 0, 0.0, 5)[0] == abi.E_INVAL
    assert raw_top(h, None, abi.METRIC_COUNT, 5, float("nan"), 5)[0] == abi.E_INVAL
    assert raw_top(h, None, 9, 5, 0.0, 5)[0] == abi.E_INVAL
    assert raw_top(h, None, (Q, -0.5), 5, 0.0, 5)[0] == abi.E_INVAL
    assert raw_top(h, None, abi.METRIC_COUNT, 5, 0.0, 5, m_ptr=False)[0] == abi.E_INVAL
    assert raw_top(h, 3, abi.METRIC_COUNT, 5, 0.0, 5)[0] == abi.E_INVAL
    rc, rr, vv, ii, n, _ = raw_top(h, None, abi.METRIC_COUNT, 20, 0.0, 19)    # cap too small
    assert rc == abi.E_CAPACITY and n == 20
    assert set(rr.view(np.uint8).tolist()) == {0xAB} and np.all(vv == 7.5) and np.all(ii == 0xDEADBEEF)
    full = raw_top(h, None, (Q, 0.9), 20, 0.0, 20)
    for flags in ((False, True, True), (True, False, True), (True, True, False), (False, False, False)):
        rc, rr, vv, ii, n, _ = raw_top(h, None, (Q, 0.9), 20, 0.0, 20, *flags, info=False)
        assert rc == 0 and n == 20, flags
        for got, want, on in ((rr, full[1], flags[0]), (vv, full[2], flags[1]), (ii, full[3], flags[2])):
            if on:
                assert got[:20].tobytes() == want[:20].tobytes(), flags
    assert full[5] == {"scored": len(rows), "above": len(rows)}
    rc, *_, n, inf = raw_top(h, None, abi.METRIC_COUNT, 5, 1e30, 5)             # nothing eligible
    assert rc == 0 and n == 0 and inf == {"scored": len(rows), "above": 0}
    s.close()


def test_zero_row_sources():
    s = Stream(universe(seed=34, n_edges=300), history=(3, 1 << 14))
    s.window(np.array([], np.int64))
    rows, _ = s.h.rollup(1)
    assert len(rows) == 0
    r = s.h.edge_top_rollup(WIN, abi.METRIC_COUNT, 5)
    assert len(r[0]) == 0 and r[3] == {"scored": 0, "above": 0}
    r = s.h.edge_top(abi.METRIC_COUNT, 5)
    assert len(r[0]) == 0 and r[3] == {"scored": 0, "above": 0}
    s.close()
