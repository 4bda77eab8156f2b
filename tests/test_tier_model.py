"""CPU: the model of the tiered history (tests/tier_model.py) pinned by hand: cascades with factors 2 and 3 over three
tiers, dropped blocks and the clearing of the tiers above, reconfiguration, and every tier entry equal to the
rolling-window model's sum of the windows it covers."""
import numpy as np

from alaz_b200 import abi
from rollup_model import RollupModel
from test_rollup_model import P, S, row, rows
from tier_model import TierModel


def win(*keys, count=1):
    """A window with one row per pod id in keys, pod -> service 1."""
    return rows(*[row(P, k, S, 1, count, 0, 10 * count, [(k % abi.NB, count)]) for k in sorted(keys)])


def test_cascade_factors_2_and_3_over_three_tiers():
    m = TierModel()
    m.configure([(2, 4, 100, 100), (3, 4, 100, 100), (2, 4, 100, 100)])
    for w in range(1, 13):
        m.window(win(w % 4, 10), w, epoch=100 + w)
        # tier 1 closes after windows 2, 4, ...; tier 2 after 6, 12; tier 3 after 12
        assert m.state(1) == dict(entries=min(w // 2, 4), open_windows=w % 2, dropped=0)
        assert m.state(2)["entries"] == w // 6 and m.state(2)["open_windows"] == 2 * ((w // 2) % 3)
        assert m.state(3)["entries"] == w // 12 and m.state(3)["open_windows"] == 6 * ((w // 6) % 2)
    got, info = m.rollup(1, 1)                      # windows 11 and 12: pods 3, 0 and 10 twice
    assert [int(x) for x in got["from"]] == [0, 3, 10] and [int(x) for x in got["count"]] == [1, 1, 2]
    assert info == dict(windows=2, clocked=1, window_first=11, window_last=12, epoch_first=111, epoch_last=112,
                        rows_in=3)
    got, info = m.rollup(2, 2)                      # windows 1..12: two entries of 5 rows
    assert info == dict(windows=12, clocked=1, window_first=1, window_last=12, epoch_first=101, epoch_last=112,
                        rows_in=10)
    assert [int(x) for x in got["count"]] == [3, 3, 3, 3, 12]
    top, info3 = m.rollup(3, 5)
    assert top.tobytes() == got.tobytes() and info3 == dict(info, rows_in=5)   # one entry of the same 5 rows
    assert m.rollup(1, 9)[1]["windows"] == 8        # depth 4 of tier 1: windows 5..12
    m.window(win(1), 13)                            # not clocked: the open block of every tier is unclocked
    m.window(win(1), 14, epoch=114)
    assert m.rollup(1, 1)[1]["clocked"] == 0 and m.rollup(1, 2)[1]["clocked"] == 0


def test_each_entry_is_the_sum_of_the_windows_it_covers():
    rng = np.random.default_rng(3)
    m, flat = TierModel(), RollupModel()
    m.configure([(3, 8, 1000, 1000), (2, 8, 1000, 1000)])
    flat.history(64, 1 << 20)
    for w in range(1, 25):
        r = win(*rng.choice(40, int(rng.integers(0, 12)), replace=False).tolist(), count=int(rng.integers(1, 5)))
        m.window(r, w)
        flat.append(r, w)
    for tier, per in ((1, 3), (2, 6)):
        for k in (1, 2, 3):
            got, info = m.rollup(tier, k)
            exp, _ = flat.rollup(k * per)
            assert got.tobytes() == exp.tobytes() and info["windows"] == k * per and info["window_last"] == 24


def test_a_block_over_block_rows_is_dropped_and_the_tiers_above_drop_the_blocks_that_contain_it():
    m = TierModel()
    m.configure([(2, 8, 100, 3), (2, 8, 100, 100), (2, 8, 100, 100)])
    for w in range(1, 9):
        m.window(win(w), w)                         # two distinct rows per tier-1 block: fits
    assert [m.state(t)["entries"] for t in (1, 2, 3)] == [4, 2, 1]
    m.window(win(1, 2), 9)
    m.window(win(3, 4), 10)                         # 4 distinct rows > 3: dropped, tier 1 cleared
    assert m.state(1) == dict(entries=0, open_windows=0, dropped=1)
    assert m.state(2)["entries"] == 2               # tier 2 keeps its entries until the poisoned block closes
    m.window(win(5), 11)
    m.window(win(6), 12)                            # tier 2's block of windows 9..12 closes: dropped, cleared
    assert m.state(1)["entries"] == 1 and m.state(2) == dict(entries=0, open_windows=0, dropped=1)
    for w in range(13, 17):
        m.window(win(w), w)                         # tier 3's block of windows 9..16 closes: dropped, cleared
    assert m.state(3) == dict(entries=0, open_windows=0, dropped=1)
    assert m.state(2)["entries"] == 1 and m.rollup(2, 4)[1]["window_first"] == 13


def test_a_block_over_the_arena_is_dropped_but_fits_its_block():
    m = TierModel()
    m.configure([(2, 8, 3, 100), (2, 8, 100, 100)])
    m.window(win(1), 1)
    m.window(win(2), 2)
    m.window(win(1, 2), 3)
    m.window(win(3, 4), 4)                          # 4 rows > arena of 3
    assert m.state(1) == dict(entries=0, open_windows=0, dropped=1)
    assert m.state(2) == dict(entries=0, open_windows=0, dropped=1)


def test_ring_eviction_per_tier():
    m = TierModel()
    m.configure([(2, 2, 100, 100)])
    for w in range(1, 9):
        m.window(win(w), w)
    assert m.state(1)["entries"] == 2 and m.rollup(1, 5)[1]["window_first"] == 5
    m.configure([(2, 8, 5, 100)])                   # arena of 5 rows, 2-row blocks: the third wraps to row 0
    for w in range(1, 7):
        m.window(win(w), w)
    assert [(e["first_row"], e["n"]) for e in m.tiers[0].ring.entries] == [(2, 2), (0, 2)]


def test_reconfiguration():
    m = TierModel()
    cfg = [(2, 4, 100, 100), (2, 4, 100, 100)]
    m.configure(cfg)
    for w in range(1, 4):
        m.window(win(w), w)
    m.configure(cfg)                                # the same values: nothing changes
    assert m.state(1) == dict(entries=1, open_windows=1, dropped=0)
    m.configure([(3, 4, 100, 100), (2, 4, 100, 100)])
    assert m.state(1) == dict(entries=0, open_windows=0, dropped=0)
    for w in range(4, 7):                           # boundaries counted from the configuring call
        m.window(win(w), w)
    assert m.rollup(1, 1)[1]["window_first"] == 4 and m.state(2)["open_windows"] == 3
    m.configure([])
    assert m.tiers == []
    m.window(win(1), 7)                             # tiers off: nothing to feed
