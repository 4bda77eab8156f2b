"""CPU: the four restatements of the SPEC §5 quantile agree bit for bit on adversarial histograms: the library's host
function (alz_edge_quantiles, the same float64 arithmetic as the GNN's edge features), the oracle's orc_quantile and
tests/gnn_ref.py's scalar and vectorised versions (the GNN reference). Cells reach 2^32 - 1, which no test stream
can fill through the ingest path."""
import ctypes as C

import numpy as np

import gnn_ref
import oracle_lib as ol
from alaz_b200 import abi, capi

QS = [0.0, 1e-300, 0.25, 0.5, 0.75, 0.99, 0.999, 1.0]
BIG = (1 << 32) - 1


def _hists():
    hs = []

    def h(cells):
        x = np.zeros(64, np.uint32)
        for b, c in cells.items():
            x[b] = c
        hs.append(x)
    h({})                                                       # empty: 0
    for b in (0, 1, 2, 31, 32, 62, 63):
        h({b: 1}); h({b: BIG})                                  # all mass in one bucket
    h({5: 2, 9: 2}); h({3: 3, 4: 3}); h({7: 5, 12: 5})           # p50 on a bucket's end, across 2l+1 | 2l+2
    h({0: 1, 5: 1}); h({0: 1, 63: 1}); h({62: 1, 63: 1})
    h({10: 99, 20: 1}); h({11: 198, 14: 2}); h({61: 297, 63: 3})  # p99 exactly on a bucket's end
    h({1: BIG, 2: BIG}); h({0: BIG, 63: 1}); h({0: 1, 63: BIG})
    h({b: BIG for b in range(64)})                              # total 64 (2^32 - 1) > 2^37
    h({b: BIG if b % 2 else 1 for b in range(64)})
    h({31: BIG, 32: BIG, 33: 1})                                # the middle lane boundary, huge counts
    rng = np.random.default_rng(7)
    for _ in range(200):
        x = np.zeros(64, np.uint32)
        k = rng.integers(1, 6)
        x[rng.choice(64, k, replace=False)] = rng.choice([1, 2, 3, 99, 100, 1 << 31, BIG - 1, BIG], k)
        hs.append(x)
    return np.array(hs)


def _lib_quantiles(hist, qs):
    L = capi.load()
    e = np.zeros(1, dtype=abi.EDGE_OUT)
    e["hist"][0] = hist
    q = np.array(qs, dtype=np.float64)
    out = np.zeros(len(qs))
    assert L.alz_edge_quantiles(e.ctypes.data_as(C.c_void_p), q.ctypes.data_as(C.c_void_p), len(qs),
                                out.ctypes.data_as(C.c_void_p)) == 0
    return out


def test_quantile_restatements_agree_bitwise():
    hs = _hists()
    for q in QS:
        vec = gnn_ref.quantiles_vec(hs, q)
        for i, x in enumerate(hs):
            want = gnn_ref.quantile(x, q)
            got = [float(_lib_quantiles(x, [q])[0]), ol.quantile(x, q), float(vec[i])]
            assert all(np.float64(g).tobytes() == np.float64(want).tobytes() for g in got), \
                (q, {b: int(c) for b, c in enumerate(x) if c}, want, got)


def test_quantile_hand_values():
    """Spot values: a tie on a bucket's end takes that bucket's upper bound; p0 sits at the first non-empty
    bucket's lower bound; cells of 2^32 - 1 lose nothing."""
    lo, hi = gnn_ref.bucket_lo, gnn_ref.bucket_hi
    x = np.zeros(64, np.uint32); x[5] = 2; x[9] = 2
    assert gnn_ref.quantile(x, 0.5) == hi(5)
    x = np.zeros(64, np.uint32); x[10] = 99; x[20] = 1
    assert gnn_ref.quantile(x, 0.99) == hi(10)
    assert gnn_ref.quantile(x, 0.0) == lo(10)
    x = np.zeros(64, np.uint32); x[0] = BIG; x[63] = BIG
    assert gnn_ref.quantile(x, 0.5) == hi(0)
    assert gnn_ref.quantile(x, 1.0) == float(1 << 40)
