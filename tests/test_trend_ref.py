"""CPU: tests/trend_ref.py against hand-derived trends (docs/SPEC.md §20)."""
import numpy as np
import pytest

import trend_ref as tr
from alaz_b200 import abi

SLOPE, SHIFT, RATIO, ZSCORE = abi.TREND_SLOPE, abi.TREND_SHIFT, abi.TREND_RATIO, abi.TREND_ZSCORE
RISING, FALLING = abi.TREND_RISING, abi.TREND_FALLING
SKIP, ZERO = abi.TREND_ABSENT_SKIP, abi.TREND_ABSENT_ZERO


def one(y, p=None, **spec):
    """the trend dict of one row, as Python scalars"""
    y = np.asarray([y], dtype=np.float64)
    p = np.ones_like(y, dtype=np.uint8) if p is None else np.asarray([p], dtype=np.uint8)
    return {k: v[0].item() for k, v in tr.trends(y, p, **spec).items()}


def test_a_linear_series_gives_its_exact_slope():
    for a, b, P in ((3.0, 2.0, 6), (100.0, -0.5, 11), (0.0, 0.25, 60)):
        y = [a + b * j for j in range(P)]
        t = one(y, stat=SLOPE)
        assert t["trend"] == b and t["valid"] == 1 and t["used"] == P
        assert one(y, stat=SLOPE, direction=FALLING)["trend"] == -b


def test_slope_over_the_present_points_uses_their_indices():
    y, p = [1.0, 0.0, 5.0, 7.0], [1, 0, 1, 1]            # points 0, 2, 3: x mean 5/3, y mean 13/3
    xm, ym = 5.0 / 3, 13.0 / 3
    sxy = ((0.0 + (0 - xm) * (1.0 - ym)) + (2 - xm) * (5.0 - ym)) + (3 - xm) * (7.0 - ym)
    sxx = ((0.0 + (0 - xm) * (0 - xm)) + (2 - xm) * (2 - xm)) + (3 - xm) * (3 - xm)
    t = one(y, p, stat=SLOPE)
    assert t["trend"] == sxy / sxx and t["used"] == 3
    z = one(y, p, stat=SLOPE, absent=ZERO)                # the hole is a 0 at x = 1
    assert z["used"] == 4 and z["trend"] != t["trend"]


def test_skip_and_zero_differ_on_series_with_holes():
    y, p = [4.0, 0.0, 4.0, 0.0, 8.0], [1, 0, 1, 0, 1]
    s = one(y, p, stat=SHIFT, recent=2)                   # B = {0, 2}, R = {4}
    assert (s["before"], s["recent"], s["trend"], s["used"]) == (4.0, 8.0, 4.0, 3)
    z = one(y, p, stat=SHIFT, recent=2, absent=ZERO)      # B = {0, 1, 2}, R = {3, 4}
    assert (z["before"], z["recent"], z["trend"], z["used"]) == (8.0 / 3, 4.0, 4.0 - 8.0 / 3, 5)
    r = one(y, p, stat=RATIO, recent=2, absent=ZERO)
    assert r["trend"] == 4.0 / (8.0 / 3)
    # a row with no recent point: SHIFT is not defined under SKIP, is under ZERO
    y, p = [2.0, 3.0, 0.0], [1, 1, 0]
    assert one(y, p, stat=SHIFT)["valid"] == 0
    z = one(y, p, stat=SHIFT, absent=ZERO)
    assert z["valid"] == 1 and z["trend"] == -2.5


@pytest.mark.parametrize("stat", [SHIFT, RATIO, ZSCORE])
def test_recent_at_or_above_P_leaves_the_comparisons_invalid(stat):
    y = [1.0, 2.0, 3.0]
    for r in (3, 4, 9):
        t = one(y, stat=stat, recent=r)
        assert t["valid"] == 0 and t["trend"] == 0.0 and not np.signbit(t["trend"])
        assert (t["before"], t["recent"], t["used"]) == (0.0, 2.0, 3)
    assert one(y, stat=SLOPE, recent=9)["trend"] == 1.0      # the slope has no recent part


def test_zscore_of_a_flat_baseline_is_infinite_or_zero():
    base = [5.0, 5.0, 5.0, 5.0]
    up, down, same = one(base + [6.0], stat=ZSCORE), one(base + [4.0], stat=ZSCORE), one(base + [5.0], stat=ZSCORE)
    assert up["trend"] == np.inf and down["trend"] == -np.inf
    assert same["trend"] == 0.0 and not np.signbit(same["trend"]) and same["valid"] == 1
    assert one(base + [4.0], stat=ZSCORE, direction=FALLING)["trend"] == np.inf
    # one earlier point is not enough for a deviation
    assert one([5.0, 6.0], stat=ZSCORE)["valid"] == 0
    # the population deviation: B = 2, 4, 6 has mean 4, sd sqrt(8 / 3)
    t = one([2.0, 4.0, 6.0, 9.0], stat=ZSCORE)
    ss = ((0.0 + (2.0 - 4.0) * (2.0 - 4.0)) + 0.0) + (6.0 - 4.0) * (6.0 - 4.0)
    assert t["trend"] == (9.0 - 4.0) / np.sqrt(ss / 3)


def test_ratio_follows_the_zero_before_rule():
    assert one([0.0, 0.0, 3.0], stat=RATIO)["trend"] == np.inf
    assert one([0.0, 0.0, 0.0], stat=RATIO)["trend"] == 1.0
    assert one([2.0, 2.0, 3.0], stat=RATIO)["trend"] == 1.5
    assert one([2.0, 2.0, 0.0], stat=RATIO)["trend"] == 0.0
    assert one([2.0, 2.0, 0.0], stat=RATIO, direction=FALLING)["trend"] == np.inf     # roles swapped
    assert one([0.0, 0.0, 0.0], stat=RATIO, direction=FALLING)["trend"] == 1.0
    assert one([2.0, 2.0, 8.0], stat=RATIO, direction=FALLING)["trend"] == 0.25


def test_falling_mirrors_rising():
    rng = np.random.default_rng(3)
    y = rng.gamma(2.0, 50.0, (200, 12))
    p = (rng.random((200, 12)) < 0.8).astype(np.uint8)
    for stat in (SLOPE, SHIFT, ZSCORE):
        for absent in (SKIP, ZERO):
            r = tr.trends(y, p, stat, RISING, absent, 4)
            f = tr.trends(y, p, stat, FALLING, absent, 4)
            assert np.array_equal(r["valid"], f["valid"])
            assert np.array_equal(f["trend"], np.where(r["valid"] == 1, 0.0 - r["trend"], 0.0))
            for k in ("used", "recent", "before"):
                assert np.array_equal(r[k], f[k])
    r = tr.trends(y, p, RATIO, RISING, SKIP, 4)
    f = tr.trends(y, p, RATIO, FALLING, SKIP, 4)
    ok = (r["valid"] == 1) & (r["recent"] > 0)
    assert np.array_equal(f["trend"][ok], r["before"][ok] / r["recent"][ok])


def test_min_points():
    y, p = [1.0, 2.0, 0.0, 4.0, 5.0], [1, 1, 0, 1, 1]
    for mp, valid in ((0, 1), (3, 1), (4, 1), (5, 0), (99, 0)):
        t = one(y, p, stat=SHIFT, recent=2, min_points=mp)
        assert t["valid"] == valid and t["used"] == 4
        assert t["trend"] == (4.5 - 1.5 if valid else 0.0)
    assert one(y, p, stat=SHIFT, recent=2, min_points=5, absent=ZERO)["valid"] == 1


def test_counts_above_2_53():
    big = float(1 << 60)                                       # the float64 ulp here is 2^8
    y = [big, big, big + 512.0, big + 1024.0]
    s = one(y, stat=SHIFT, recent=2)
    assert s["before"] == big and s["recent"] == big + 768.0 and s["trend"] == 768.0
    # the sum of all four rounds up to 2^62 + 2048, so ym = big + 512 (not big + 384); Sxy stays 1792, Sxx 5
    assert one(y, stat=SLOPE)["trend"] == 1792.0 / 5.0
    z = one([big, big + 512.0, big, big + 4096.0], stat=ZSCORE)   # B's mean big + 512 / 3 rounds to big + 256
    assert z["before"] == big + 256.0 and z["trend"] == 3840.0 / 256.0


def test_sums_are_sequential_in_ascending_j():
    """2^53 + 1 + 1 sums to 2^53 one add at a time, to 2^53 + 2 pairwise: the mean pins the order."""
    y = [2.0 ** 53, 1.0, 1.0, 0.0]
    t = one(y, stat=SHIFT, recent=1)
    assert t["before"] == 2.0 ** 53 / 3 and t["before"] != (2.0 ** 53 + 2.0) / 3
    t = one([1.0, 1.0, 2.0 ** 53, 0.0], stat=SHIFT, recent=1)   # the other order keeps the ones
    assert t["before"] == (2.0 ** 53 + 2.0) / 3


def test_records_and_top_order():
    rows = np.zeros(6, dtype=abi.EDGE_OUT)
    rows["from_type"], rows["from"], rows["to_type"], rows["to"] = abi.NODE_POD, np.arange(6), abi.NODE_SVC, 7
    y = np.array([[1, 2, 3], [1, 1, 1], [3, 2, 1], [1, 2, 3], [0, 0, 5], [0, 0, 0]], dtype=np.float64)
    p = np.array([[1, 1, 1], [1, 1, 1], [1, 1, 1], [1, 1, 1], [0, 0, 1], [0, 0, 0]], dtype=np.uint8)
    rec = tr.records(rows, y, p, stat=SLOPE)
    assert rec["index"].tolist() == list(range(6)) and rec["from"].tolist() == list(range(6))
    assert rec["valid"].tolist() == [1, 1, 1, 1, 0, 0] and rec["used"].tolist() == [3, 3, 3, 3, 1, 0]
    idx, above = tr.top(rec, 10)
    assert idx.tolist() == [0, 3, 1, 2] and above == 4           # ties in index order; invalid rows never eligible
    idx, above = tr.top(rec, 1, 0.0)
    assert idx.tolist() == [0] and above == 3
    rec = tr.records(rows, y, p, stat=ZSCORE, absent=ZERO)       # B = [0, 0] for row 4: sd 0, d > 0
    idx, _ = tr.top(rec, 2)
    assert idx.tolist() == [4, 0] and rec["trend"][4] == np.inf
