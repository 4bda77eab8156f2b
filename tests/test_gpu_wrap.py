"""GPU: histogram cells that wrap modulo 2^32 (docs/SPEC.md §3) in the sums that add rows: window rollups, tier blocks
and tier rollups, spans over several buffers, and the general path of the multi-rank merge; and the readers of the
wrapped rows (§15 GNN scores, §17 metrics and top edges, §18 changes, §19 series).

The stream is tests/wrap_layout.py: a window of 537M packed records whose hot cells hold 4097 * 2^16 events, so
that a sum of 16 windows passes 2^32 in two cells (bucket 50 of a pod -> service row, bucket 8 of a reversed
pod <-> pod row) and a sum of 15 does not. It goes through the real ingest and flush: one device buffer of 2^13
tiles, uploaded once per module and submitted SUBMITS times per window. Every window is compared with the oracle
(`scaled_oracle`) before anything sums it, so that an ingest fault shows as one. Every sum is compared with the
models (tests/rollup_model.py, tier_model.py, span_model.py: rows byte for byte, info field by field, host and device
forms) and with the closed form of wrap_layout, so that a model error cannot hide a kernel error."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import ingest_streams as ist
import loopback_ranks as lr
import metric_ref as mr
import wrap_layout as wl
from alaz_b200 import abi, capi
from change_ref import row_keys
from helpers import edges_equal, explain_diff
from rollup_model import RollupModel
from span_model import AT_LEAST, AT_MOST
from test_gpu_edge_changes import check_all as check_changes
from test_gpu_edge_metrics import host_quantile
from test_gpu_edge_series import Modelled, expect as expect_series, same as same_series
from test_gpu_edge_top import expect as expect_top
from test_gpu_gnn_rollup import score_and_check
from test_gpu_loopback_ranks import HERE, ROOT, SMALL, shim  # noqa: F401  (shim is a fixture)
from test_gpu_span import Span
from test_gpu_tiers import Tiers

pytestmark = pytest.mark.gpu
WINDOW, WIN, TIER = abi.SOURCE_WINDOW, abi.ROLLUP_WINDOWS, abi.ROLLUP_TIER
Q = abi.METRIC_QUANTILE
ALL = [abi.METRIC_COUNT, abi.METRIC_ERR5XX, abi.METRIC_ERR_RATE, abi.METRIC_MEAN_NS, (Q, 0.0), (Q, 0.5), (Q, 0.99),
       (Q, 1.0)]
HANDLE = dict(max_endpoints=256, max_pairs=1 << 12)
NEED = 4 << 30          # the 1.07 GB buffer, the handles and the parent's own CUDA context, with room to spare


def free_device_memory():
    import torch
    return torch.cuda.mem_get_info()[0]


class Buffer:
    """The packed tile repeated BUF_TILES times in device memory, its overflow array, and the oracle's window."""

    def __init__(self):
        packed, ovf = capi.pack_l7(wl.tile())
        self.tile, self.ovf = packed, ovf
        self.n = len(packed) * wl.BUF_TILES
        self.owner = capi.Handle(max_endpoints=64, max_pairs=1 << 10)
        self.p = self.owner.dev_alloc(self.n * packed.itemsize)
        self.po = self.owner.dev_alloc(max(ovf.nbytes, 8))
        step = 1 << 9
        block = np.tile(packed, step)
        for t in range(0, wl.BUF_TILES, step):
            self.owner.h2d(self.p + t * packed.nbytes, block)
        self.owner.h2d(self.po, ovf)
        self.owner.sync()
        self.exp, self.est = wl.window_edges()

    def window(self, h, flush):
        """One window of the stream into h, flushed by flush(); its rows checked against the oracle."""
        before = h.stats()
        for _ in range(wl.SUBMITS):
            h.submit_packed_device(self.p, self.n, self.po)
        rows = flush()
        assert edges_equal(rows, self.exp), explain_diff(rows, self.exp)
        st = h.stats()
        for k in ist.STAT_KEYS:
            assert st[k] - before[k] == self.est[k], (k, st[k] - before[k], self.est[k])
        return rows

    def close(self):
        self.owner.dev_free(self.p)
        self.owner.dev_free(self.po)
        self.owner.close()


@pytest.fixture(scope="module")
def buf():
    free = free_device_memory()
    if free < NEED:
        pytest.skip(f"needs {NEED >> 30} GB of free device memory, {free >> 30} GB free")
    b = Buffer()
    yield b
    b.close()


def check_window_rollup(r, k):
    """alz_window_rollup(k), host and device, against the window-history model of a Tiers."""
    exp, exp_info = r.m0.rollup(k)
    got, info = r.h.rollup(k)
    assert info == exp_info, (k, info, exp_info)
    assert got.tobytes() == exp.tobytes(), explain_diff(got, exp)
    p, n, info_d = r.h.rollup_device(k)
    assert info_d == exp_info and r.h.d2h(p, n, abi.EDGE_OUT).tobytes() == exp.tobytes()
    return got


# ---- window history and one tier of factor 16 over the same 16 windows ------------------------------------------------

@pytest.fixture(scope="module")
def hist16(buf):
    """History depth 16 and one tier (factor 16): 16 windows. The baseline is pinned after window 1."""
    r = Tiers([(16, 2, 64, 16)], wl.TABLES, history=(16, 64), **HANDLE)
    r.states = []
    for w in range(wl.W):
        rows = buf.window(r.h, r.flush)
        if w == 0:
            r.base_rows, r.base_info = rows, r.h.baseline_pin(WINDOW)
        r.states.append(r.h.tier_state(1))
        assert r.states[-1] == r.m.state(1), (w, r.states[-1], r.m.state(1))
    yield r
    r.close()


def test_window_rollup_of_16_wraps_and_of_15_does_not(hist16):
    got = check_window_rollup(hist16, 16)
    wl.check_closed_form(got, 16)
    a, b = wl.row_a(got), wl.row_b(got)
    assert int(a["hist"][50]) == 1 << 20 and int(a["hist"][51]) == 1 << 20 and int(a["hist"][10]) == 1 << 20
    assert int(a["count"]) == int(a["err5xx"]) == (1 << 32) + 3 * (1 << 20)
    assert int(b["hist"][8]) == 1 << 20 and int(b["hist"][7]) == int(b["hist"][9]) == 1 << 20
    assert int(a["lat_sum_ns"]) < 16 * (4097 * wl.A_DUR[50] << 16)    # lat_sum_ns passed 2^64 as well
    got = check_window_rollup(hist16, 15)
    wl.check_closed_form(got, 15)
    assert int(wl.row_a(got)["hist"][50]) == 15 * 4097 << 16 < 1 << 32   # one window less: no wrap
    wl.check_closed_form(check_window_rollup(hist16, 1), 1)


def test_tier_of_factor_16_wraps_in_its_open_block(hist16):
    assert hist16.states[14] == dict(entries=0, open_windows=15, dropped=0)
    assert hist16.states[15] == dict(entries=1, open_windows=0, dropped=0)
    for k in (1, 2):
        got, info = hist16.check(1, k)
        assert info["windows"] == 16 and info["rows_in"] == 4
        wl.check_closed_form(got, 16)


def test_metrics_of_the_wrapped_rows(hist16):
    h = hist16.h
    for kind, rows in ((WIN, h.rollup(16)[0]), (TIER, h.rollup_tier(1, 1)[0])):
        got = h.edge_metrics_rollup(kind, *ALL)
        assert got.tobytes() == mr.matrix(rows, ALL).tobytes(), (kind, got, mr.matrix(rows, ALL))
        p, n = h.edge_metrics_rollup_device(kind, *ALL)
        h.sync()
        assert n == len(rows) and h.d2h(p, n * len(ALL), np.float64).tobytes() == got.tobytes()
        for i in range(len(rows)):
            for j, spec in enumerate(ALL[4:], 4):
                assert got[i, j].tobytes() == np.float64(host_quantile(rows[i:i + 1], spec[1])).tobytes(), (i, spec)
        # SPEC §5: row A's total is the sum of its cells, 3 * 2^20; its p50 lies halfway into bucket 50
        a = int(np.flatnonzero(rows["to_type"] == abi.NODE_SVC)[0])
        assert got[a, ALL.index((Q, 0.5))] == float((1 << 33) + (1 << 31))
        assert got[a, ALL.index(abi.METRIC_COUNT)] == float((1 << 32) + 3 * (1 << 20))


def test_top_edges_of_the_wrapped_rows(hist16):
    h = hist16.h
    rows = h.rollup(16)[0]
    for spec in (abi.METRIC_COUNT, (Q, 0.5)):
        for k in (1, 2, len(rows) + 1):
            expect_top(rows, spec, k, 0.0, h.edge_top_rollup(WIN, spec, k), (spec, k))


def test_changes_of_the_wrapped_rollup_against_a_pinned_window(hist16):
    h = hist16.h
    assert hist16.base_info["windows"] == 1 and hist16.base_info["window_first"] == 1
    rows, info = h.rollup(16)
    check_changes(h, rows, info["windows"], hist16.base_rows, 1, WIN, "wrap")


class _Entries:
    """The retained entries of the window history and the tier, as the series tests' expectation reads them."""
    entries = Modelled.entries

    def __init__(self, r):
        self.rm, self.tm = r.m0, r.m


def test_series_of_the_wrapped_tier_entry(hist16):
    h = hist16.h
    m = _Entries(hist16)
    for tier, kind, roll in ((1, TIER, lambda: h.rollup_tier(1, 1)), (0, WIN, lambda: h.rollup(16))):
        rows, _ = roll()
        keys = row_keys(rows)
        for k in (1, 16):
            same_series(h.edge_series(kind, tier, k, *ALL), expect_series(m, tier, k, keys, ALL), (tier, k))
    v, p, _, _ = h.edge_series(TIER, 1, 1, (Q, 0.5))
    a = int(np.flatnonzero(h.rollup_tier(1, 1)[0]["to_type"] == abi.NODE_SVC)[0])
    assert p[a, 0] and v[a, 0, 0] == float((1 << 33) + (1 << 31))


def test_gnn_scores_of_the_wrapped_rollup(hist16):
    rows = hist16.h.rollup(16)[0]
    score_and_check(hist16.h, WIN, rows, "rollup of 16 wrapped windows")


# ---- tiers of factor 2: the wrap in tier 4's merge, and tier rollups over several entries ----------------------------

def test_tiers_of_factor_2_wrap_in_tier_4_and_in_tier_rollups(buf):
    r = Tiers([(2, 8, 64, 16), (2, 4, 64, 16), (2, 2, 64, 16), (2, 1, 64, 16)], wl.TABLES, **HANDLE)
    for w in range(wl.W):
        buf.window(r.h, r.flush)
        for t in (1, 2, 3, 4):
            assert r.h.tier_state(t) == r.m.state(t), (w, t, r.h.tier_state(t), r.m.state(t))
    # tier 4's one entry: its block wrapped when it merged its second input (two tier-3 blocks of 8 windows)
    for tier, k, m in ((4, 1, 16), (3, 1, 8), (3, 2, 16), (2, 4, 16), (1, 8, 16), (1, 7, 14), (1, 1, 2)):
        got, info = r.check(tier, k)
        assert info["windows"] == m, (tier, k, info)
        wl.check_closed_form(got, m)
    r.close()


# ---- spans over the tier arena and an open block ---------------------------------------------------------------------

def test_spans_over_tier_entries_and_an_open_block(buf):
    """Tier 1 of factor 4 keeps 4 entries (16 windows), window history 4: after 18 windows the entries cover 1..16,
    the open block 17..18 and the history 15..18. Spans of 14 and 18 windows can be made, the one of 18 wraps and
    takes 4 tier entries and the open block: two buffers, rows mapped through the virtual-row lookup."""
    r = Span([(4, 4, 64, 16)], history=(4, 64), tables=wl.TABLES, **HANDLE)
    for _ in range(18):
        buf.window(r.h, r.flush)
    for N in (2, 14, 15, 16, 17, 18, 19):
        for mode in (AT_MOST, AT_LEAST):
            got, info = r.check(N, mode)
            if info["windows"]:
                wl.check_closed_form(got, info["windows"])
    for N, mode, m in ((16, AT_LEAST, 18), (18, AT_MOST, 18), (19, AT_MOST, 18), (16, AT_MOST, 14)):
        got, info = r.check(N, mode)
        assert info["windows"] == m, (N, mode, info)
        if m == 18:
            assert info["entries"] == [0, 4, 0, 0, 0] and info["open_blocks"] == 1 << 1, info
            assert int(wl.row_a(got)["hist"][50]) == 18 * 4097 << 16 & wl.M32
        else:
            assert info["entries"] == [0, 3, 0, 0, 0] and info["open_blocks"] == 1 << 1, info
    r.close()


# ---- the general path of the multi-rank merge --------------------------------------------------------------------------

def test_sixteen_ranks_wrap_in_the_general_path(buf, shim, tmp_path):  # noqa: F811
    """16 ranks of one process on one GPU (tests/loopback_wrap_ranks.py) each submit one window of the stream, so
    every key is on every rank and the merge takes the general path: cells widened to u64, all-reduced, cut back to
    u32. The merged window is 16 windows' worth, so cells 50 and 8 wrap in the cut. Two such windows, then a window
    rollup of both on every rank."""
    R, windows = 16, 2
    spec = {"nranks": R, "cfg": SMALL, "buf_tiles": wl.BUF_TILES, "submits": wl.SUBMITS, "windows": windows,
            "history": [2, 64]}
    tab = [(t, ip, i) for t, ips, ids in wl.TABLES for ip, i in zip(ips, ids)]
    sp, ip_, op = (str(tmp_path / x) for x in ("spec.json", "in.npz", "out.npz"))
    with open(sp, "w") as f:
        json.dump(spec, f)
    np.savez(ip_, tab0=np.asarray(tab, np.int64), tile=buf.tile, ovf=buf.ovf)
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = os.path.dirname(shim) + os.pathsep + env.get("LD_LIBRARY_PATH", "")
    env["LOOPBACK_NCCL_TIMEOUT_S"] = "120"
    p = subprocess.run([sys.executable, os.path.join(HERE, "loopback_wrap_ranks.py"), sp, ip_, op], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    z = np.load(op)
    meta = json.loads(str(z["meta"]))
    assert not meta["errors"], meta["errors"]
    assert meta["maps"] == [shim], meta["maps"]
    rank = lambda r: meta["ranks"][str(r)]
    exp, est = ist.scaled_oracle(wl.TABLES, wl.tile(), R * wl.TILES)
    m = RollupModel()
    m.history(2, 64)
    keys = ("events_in", "rows_emitted", "capacity_events")
    before = [{k: 0 for k in keys} for _ in range(R)]
    for j in range(windows):
        rows0 = z[f"rows_{j}_0"]
        for r in range(R):
            d = rank(r)[j]
            assert d["rc"] == abi.OK and d["n_out"] == len(rows0), (r, j, d["rc"], d["n_out"])
            assert z[f"rows_{j}_{r}"].tobytes() == rows0.tobytes(), f"rank {r} differs from rank 0 in window {j}"
            assert lr.OP_ALLREDUCE in [op_ for op_, _ in d["log"]], (r, j, d["log"])
        assert edges_equal(rows0, exp), explain_diff(rows0, exp)
        wl.check_closed_form(rows0, R)
        assert int(wl.row_a(rows0)["hist"][50]) == 1 << 20 and int(wl.row_b(rows0)["hist"][8]) == 1 << 20
        delta = {k: sum(rank(r)[j]["stats"][k] - before[r][k] for r in range(R)) for k in keys}
        assert delta == dict(events_in=est["events_in"], rows_emitted=int(exp["count"].sum()), capacity_events=0)
        before = [rank(r)[j]["stats"] for r in range(R)]
        m.append(rows0, rank(0)[j]["stats"]["windows"])
    want, want_info = m.rollup(windows)
    assert want_info["windows"] == windows
    wl.check_closed_form(want, R * windows)
    for r in range(R):
        assert meta["rollup"][str(r)] == want_info, (r, meta["rollup"][str(r)], want_info)
        assert z[f"rollup_{r}"].tobytes() == want.tobytes(), r
