"""CPU: the model of span rollups (tests/span_model.py) pinned by hand on small configurations, and its planner against
a brute-force enumeration of every set of disjoint retained pieces, with gaps, dropped blocks and evicted windows."""
import itertools

import numpy as np
import pytest

from rollup_model import RollupModel
from span_model import AT_LEAST, AT_MOST, SpanModel, choose, cost, coverable
from test_tier_model import win


def feed(m, n, start=1, keys=lambda w: (w % 4, 10)):
    for w in range(start, start + n):
        m.window(win(*keys(w)), w, epoch=100 + w)


def test_tiers_only_spans_at_block_boundaries():
    m = SpanModel()
    m.configure([(2, 4, 100, 100)])
    feed(m, 5)                                      # tier 1: [1, 2], [3, 4]; open block: [5]
    assert sorted(coverable(m.units(), 5)) == [0, 1, 3, 5]
    assert m.span(2, AT_MOST)[1]["windows"] == 1 and m.span(2, AT_LEAST)[1]["windows"] == 3
    rows, info = m.span(3)
    assert info == dict(windows=3, clocked=1, window_first=3, window_last=5, epoch_first=103, epoch_last=105,
                        rows_in=5, entries=[0, 1, 0, 0, 0], open_blocks=2)
    assert [int(x) for x in rows["count"]] == [1, 1, 1, 3]   # pods 0, 1, 3 once; pod 10 in every window
    assert m.span(9, AT_LEAST)[1]["windows"] == 5             # past everything retained: the largest there is
    assert m.span(9, AT_MOST)[1]["windows"] == 5
    m.window(win(7), 6)                                       # the block [5, 6] closes; no open block
    assert sorted(coverable(m.units(), 6)) == [0, 2, 4, 6]
    rows, info = m.span(1, AT_MOST)
    assert info["windows"] == 0 and len(rows) == 0 and info["entries"] == [0] * 5 and info["window_first"] == 0


def test_history_only_equals_the_window_rollup():
    rng = np.random.default_rng(1)
    m, flat = SpanModel(), RollupModel()
    m.history(5, 1000)
    flat.history(5, 1000)
    for w in range(1, 9):
        r = win(*rng.choice(30, int(rng.integers(0, 6)), replace=False).tolist(), count=int(rng.integers(1, 4)))
        m.window(r, w)
        flat.append(r, w)
    for N in range(1, 8):
        rows, info = m.span(N)
        exp, einfo = flat.rollup(N)
        assert rows.tobytes() == exp.tobytes()
        assert {k: info[k] for k in einfo} == einfo and info["entries"][0] == min(N, 5)


def test_fewest_rows_then_fewest_pieces_then_the_coarser_piece():
    m = SpanModel()
    m.history(8, 1000)
    m.configure([(2, 8, 100, 100), (2, 8, 100, 100)])
    feed(m, 2, keys=lambda w: (1,))                 # one row per window: tier-1 [1, 2] has 1 row, the windows 2
    _, info = m.span(2)
    # tier-1 entry [1, 2] and tier-2's open block [1, 2] both have 1 row: the coarser one is taken
    assert info["rows_in"] == 1 and info["entries"] == [0, 0, 0, 0, 0] and info["open_blocks"] == 4
    m.window(win(1), 3)
    _, info = m.span(3)                             # [1, 2] as one piece; window 3 from tier 1's open block, which
    assert info["rows_in"] == 2 and info["open_blocks"] == 6 and info["entries"] == [0] * 5   # ties the history's
    m2 = SpanModel()
    m2.history(8, 1000)
    m2.configure([(2, 8, 100, 100)])
    feed(m2, 2, keys=lambda w: (w,))                # distinct rows: the tier entry has as many rows as the windows
    _, info = m2.span(2)
    assert info["rows_in"] == 2 and info["entries"] == [0, 1, 0, 0, 0]   # fewer pieces


def test_overflowed_and_poisoned_open_blocks_are_left_out():
    m = SpanModel()
    m.history(8, 1000)
    m.configure([(4, 8, 100, 3), (2, 8, 100, 100)])
    m.window(win(1, 2), 1)
    m.window(win(3, 4), 2)                          # 4 distinct rows > 3: tier 1's open block overflowed
    _, info = m.span(2)
    assert info["windows"] == 2 and info["entries"] == [2, 0, 0, 0, 0] and info["open_blocks"] == 0
    feed(m, 2, start=3)                             # the block closes and is dropped: tier 2's block is poisoned
    assert m.mt.tiers[1].poisoned
    feed(m, 1, start=5)
    _, info = m.span(5, AT_LEAST)
    assert info["windows"] == 5 and info["open_blocks"] == 2 and info["entries"] == [4, 0, 0, 0, 0]


def test_gaps_fall_back_under_at_least():
    m = SpanModel()
    m.configure([(2, 8, 100, 100)])
    m.history(2, 1000)
    feed(m, 6)                                      # tier 1: [1, 2], [3, 4], [5, 6]; history: 5, 6
    m.configure([(2, 8, 100, 100), (2, 8, 100, 100)])   # other values: every tier entry dropped
    feed(m, 1, start=7)                             # tier 1's open block [7]; history 6, 7
    assert sorted(coverable(m.units(), 7)) == [0, 1, 2]
    assert m.span(5, AT_LEAST)[1]["windows"] == 2 and m.span(5, AT_MOST)[1]["windows"] == 2


def brute(units, W):
    """{m: the best plan} by enumerating every set of units"""
    out = {}
    for k in range(len(units) + 1):
        for pick in itertools.combinations(range(len(units)), k):
            ws = sorted(w for i in pick for w in range(units[i]["window_first"], units[i]["window_last"] + 1))
            if len(ws) != len(set(ws)) or (ws and ws != list(range(W - len(ws) + 1, W + 1))):
                continue
            plan = sorted(pick, key=lambda i: units[i]["window_first"])
            m = len(ws)
            if m not in out or cost(plan, units) < cost(out[m], units):
                out[m] = plan
    return out


@pytest.mark.parametrize("seed", range(12))
def test_planner_against_brute_force(seed):
    rng = np.random.default_rng(40 + seed)
    m = SpanModel()
    m.history(int(rng.integers(1, 5)), int(rng.integers(3, 12)))
    m.configure([(int(rng.integers(2, 4)), int(rng.integers(1, 4)), int(rng.integers(3, 12)), int(rng.integers(2, 8)))
                 for _ in range(int(rng.integers(1, 4)))])
    W = 0
    for _ in range(int(rng.integers(4, 30))):
        W += 1
        m.window(win(*rng.choice(12, int(rng.integers(0, 5)), replace=False).tolist()), W)
        units = m.units()
        if len(units) > 14:
            continue
        got, exp = coverable(units, W), brute(units, W)
        assert sorted(got) == sorted(exp)
        for k in got:
            assert cost(got[k], units) == cost(exp[k], units)
            assert got[k] == exp[k]
        for N in range(1, W + 3):
            assert choose(got, N, AT_MOST) == max([k for k in exp if k <= N])
            above = [k for k in exp if k >= N]
            assert choose(got, N, AT_LEAST) == (min(above) if above else max(exp))
