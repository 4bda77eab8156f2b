"""CPU: tests/metric_ref.py, the reference of the edge metrics and the top edges (docs/SPEC.md §17). Its quantile
agrees bit for bit with alz_edge_quantiles and the oracle's orc_quantile on the adversarial histograms of
test_gnn_quantiles.py; its key and rank order agree with the definition: ±0, ties, count = 0."""
import ctypes as C

import numpy as np

import metric_ref as mr
import oracle_lib as ol
from alaz_b200 import abi, capi
from test_gnn_quantiles import BIG, QS, _hists

Q = abi.METRIC_QUANTILE


def _rows(hists):
    rows = np.zeros(len(hists), dtype=abi.EDGE_OUT)
    rows["hist"] = hists
    return rows


def test_quantile_matches_host_function_and_oracle():
    hs = _hists()
    rows = _rows(hs)
    L = capi.load()
    for q in QS:
        got = mr.values(rows, (Q, q))
        qa = np.array([q])
        for i in range(len(rows)):
            host = np.zeros(1)
            assert L.alz_edge_quantiles(rows[i:i + 1].ctypes.data_as(C.c_void_p), qa.ctypes.data_as(C.c_void_p), 1,
                                        host.ctypes.data_as(C.c_void_p)) == 0
            assert got[i].tobytes() == host[0].tobytes(), (q, i, got[i], host[0])
            assert got[i].tobytes() == np.float64(ol.quantile(hs[i], q)).tobytes(), (q, i)


def test_scalar_metrics_and_count_zero():
    rows = np.zeros(4, dtype=abi.EDGE_OUT)
    rows["count"] = [0, 3, (1 << 64) - 1, 7]
    rows["err5xx"] = [5, 1, 1 << 63, 0]
    rows["lat_sum_ns"] = [9, 10, (1 << 64) - 1, 1]
    rows["hist"][0, 4] = BIG                                   # count = 0 with a non-empty histogram
    assert mr.values(rows, abi.METRIC_COUNT).tolist() == [0.0, 3.0, float(2 ** 64), 7.0]
    assert mr.values(rows, abi.METRIC_ERR5XX).tolist() == [5.0, 1.0, float(2 ** 63), 0.0]
    rate = mr.values(rows, abi.METRIC_ERR_RATE)
    assert rate[0] == 0.0 and rate[1] == 1.0 / 3.0 and rate[2] == 0.5 and rate[3] == 0.0
    mean = mr.values(rows, abi.METRIC_MEAN_NS)
    assert mean[0] == 0.0 and mean[1] == 10.0 / 3.0 and mean[2] == 1.0 and mean[3] == 1.0 / 7.0
    assert mr.values(rows, (Q, 0.5))[0] > 0.0                 # the quantile reads the histogram, not count
    m = mr.matrix(rows, [abi.METRIC_COUNT, (Q, 0.5)])
    assert m.shape == (4, 2) and m[1, 0] == 3.0


def _lexsort_top(v, k, min_value):
    """The definition with Python integers: sort by (-key, index), keep key >= key(min)."""
    keys = [int(x) for x in mr.order_key(v)]
    kmin = int(mr.order_key(min_value)[0])
    order = sorted(range(len(v)), key=lambda i: (-keys[i], i))
    elig = [i for i in order if keys[i] >= kmin]
    return elig[:k], len(elig)


def test_order_key_total_order():
    v = np.array([-np.inf, -1.0, -5e-324, -0.0, 0.0, 5e-324, 1.0, np.inf])
    k = mr.order_key(v)
    assert np.all(np.diff(k.astype(object)) > 0)              # strictly increasing in IEEE total order
    assert mr.order_key(0.0)[0] == np.uint64(1 << 63) and mr.order_key(-0.0)[0] == np.uint64((1 << 63) - 1)


def test_top_ties_zero_signs_and_min_positions():
    v = np.array([0.5, 0.0, -0.0, 0.5, 1.0, 0.25, 0.5, 0.0])
    for k in (1, 2, 3, 5, 8, 100):
        for ms in (-np.inf, -0.0, 0.0, 0.25, 0.3, 0.5, 1.0, 2.0):
            idx, above = mr.top(v, k, ms)
            want, want_above = _lexsort_top(v, k, ms)
            assert idx.tolist() == want and above == want_above, (k, ms)
    assert mr.top(v, 10, 0.0)[1] == 7 and mr.top(v, 10, -0.0)[1] == 8   # -0 is eligible only from min -0 down
    assert mr.top(v, 3, 0.0)[0].tolist() == [4, 0, 3]                    # ties: lower index first


def test_top_random_against_definition():
    rng = np.random.default_rng(4)
    for n in (1, 7, 300):
        v = rng.choice([0.0, -0.0, 1e-310, 0.5, 2.0, np.inf, 3.0], n)
        for k in (1, 3, n, n + 2):
            for ms in (0.0, 0.5, float(v[0])):
                idx, above = mr.top(v, k, ms)
                want, want_above = _lexsort_top(v, k, ms)
                assert idx.tolist() == want and above == want_above


def _fma(a, b, c):
    """a * b + c rounded once, as a fused multiply-add does (exact rational arithmetic, then one rounding)."""
    from fractions import Fraction
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def _quantile_contracted(hist, q):
    """SPEC §5 with the two contractions nvcc makes by default: (target - cum) as fma(q, total, -cum) and
    lo + f * (hi - lo) as fma(f, hi - lo, lo)."""
    import gnn_ref
    total = float(int(np.sum(hist.astype(np.uint64))))
    if total == 0.0:
        return 0.0
    target, cum = q * total, 0.0
    for b in range(64):
        c = float(hist[b])
        if c > 0.0 and cum + c >= target:
            f = max(_fma(q, total, -cum) / c, 0.0)
            lo, hi = gnn_ref.bucket_lo(b), gnn_ref.bucket_hi(b)
            return _fma(f, hi - lo, lo)
        cum += c
    return gnn_ref.bucket_hi(63)


def test_contracted_quantile_would_fail_the_gpu_cases():
    """The mutation the metric kernel guards against with its round-to-nearest intrinsics: a quantile compiled with
    fused multiply-adds differs from the reference on cases that tests/test_gpu_edge_metrics.py runs, so such a
    kernel fails them."""
    hs = _hists()
    rows = _rows(hs)
    diff = 0
    for q in QS:
        want = mr.values(rows, (Q, q))
        diff += sum(np.float64(_quantile_contracted(hs[i], q)).tobytes() != want[i].tobytes() for i in range(len(hs)))
    assert diff > 0
