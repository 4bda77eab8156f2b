"""CPU: the wrapping stream of tests/wrap_layout.py through the models and the quantile references. The models'
sums of the layout's windows equal the closed form (cells mod 2^32, u64 sums mod 2^64) on their own, before any GPU
test compares a kernel with them; and the quantile of a wrapped row takes its total from the cells (docs/SPEC.md §5),
the same in metric_ref, gnn_ref, alz_edge_quantiles and the oracle's orc_quantile."""
import ctypes as C

import numpy as np

import gnn_ref
import metric_ref as mr
import oracle_lib as ol
import wrap_layout as wl
from alaz_b200 import abi, capi
from rollup_model import RollupModel
from span_model import AT_LEAST, AT_MOST, SpanModel
from tier_model import TierModel

Q = abi.METRIC_QUANTILE


def test_one_window_is_the_oracle_of_one_tile_scaled():
    e, st = wl.window_edges()
    assert len(e) == 4 and st["events_in"] == 8200 * wl.TILES
    wl.check_closed_form(e, 1)
    assert wl.HOT * wl.TILES * wl.W == (1 << 32) + (1 << 20)


def test_models_sum_the_windows_to_the_closed_form():
    e, _ = wl.window_edges()
    m = RollupModel()
    m.history(16, 64)
    t2, t16 = TierModel(), TierModel()
    t2.configure([(2, 8, 64, 16), (2, 4, 64, 16), (2, 2, 64, 16), (2, 1, 64, 16)])
    t16.configure([(16, 2, 64, 16)])
    for w in range(1, wl.W + 1):
        m.append(e, w)
        t2.window(e, w)
        t16.window(e, w)
    rows, info = m.rollup(16)
    assert info["windows"] == 16
    wl.check_closed_form(rows, 16)
    a, b = wl.row_a(rows), wl.row_b(rows)
    assert int(a["hist"][50]) == 1 << 20 and int(b["hist"][8]) == 1 << 20
    assert int(a["count"]) == (1 << 32) + 3 * (1 << 20)
    wl.check_closed_form(m.rollup(15)[0], 15)
    assert int(wl.row_a(m.rollup(15)[0])["hist"][50]) == 15 * 4097 << 16
    for model, tier, k in ((t2, 4, 1), (t2, 3, 2), (t2, 1, 8), (t16, 1, 1)):
        rows, info = model.rollup(tier, k)
        assert info["windows"] == 16
        assert rows.tobytes() == m.rollup(16)[0].tobytes()


def test_span_model_wraps_over_tier_entries_and_an_open_block():
    e, _ = wl.window_edges()
    s = SpanModel()
    s.history(4, 64)
    s.configure([(4, 4, 64, 16)])
    for w in range(1, 19):
        s.window(e, w)
    rows, info = s.span(16, AT_LEAST)
    assert info["windows"] == 18 and info["entries"] == [0, 4, 0, 0, 0] and info["open_blocks"] == 2
    wl.check_closed_form(rows, 18)
    assert int(wl.row_a(rows)["hist"][50]) == (18 * 4097 << 16) - (1 << 32)
    rows, info = s.span(16, AT_MOST)
    assert info["windows"] == 14
    wl.check_closed_form(rows, 14)


def test_quantiles_of_a_wrapped_row_take_the_total_from_the_cells():
    e, _ = wl.window_edges()
    m = RollupModel()
    m.history(16, 64)
    for w in range(1, wl.W + 1):
        m.append(e, w)
    rows, _ = m.rollup(16)
    a = wl.row_a(rows)
    assert int(a["hist"].astype(np.uint64).sum()) == 3 << 20 < int(a["count"])
    i = int(np.flatnonzero(rows["to_type"] == abi.NODE_SVC)[0])
    L = capi.load()
    for q in (0.0, 0.5, 0.99, 1.0):
        want = mr.values(rows, (Q, q))
        assert want.tobytes() == gnn_ref.quantiles_vec(rows["hist"], q).tobytes()
        for j in range(len(rows)):
            host = np.zeros(1)
            qa = np.array([q])
            assert L.alz_edge_quantiles(rows[j:j + 1].ctypes.data_as(C.c_void_p), qa.ctypes.data_as(C.c_void_p), 1,
                                        host.ctypes.data_as(C.c_void_p)) == 0
            assert host.tobytes() == want[j:j + 1].tobytes(), (q, j)
            assert np.float64(ol.quantile(rows["hist"][j], q)).tobytes() == want[j:j + 1].tobytes(), (q, j)
    # halfway into bucket 50 [2^33, 1.5 * 2^33); q * count would lie past every cell and give bucket 63's end, 2^40
    assert mr.values(rows, (Q, 0.5))[i] == float((1 << 33) + (1 << 31))
    assert 0.5 * float(a["count"]) > float(a["hist"].astype(np.uint64).sum())
