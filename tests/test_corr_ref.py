"""CPU: tests/corr_ref.py against hand-worked correlations (docs/SPEC.md §29), a scalar Python loop (bit for bit) and
np.corrcoef."""
import math

import numpy as np
from hypothesis import given, settings, strategies as st

import corr_ref as cr
from alaz_b200 import abi

POS, NEG, ABS = abi.CORR_POSITIVE, abi.CORR_NEGATIVE, abi.CORR_ABS
SKIP, ZERO = abi.CORR_ABSENT_SKIP, abi.CORR_ABSENT_ZERO


def one(x, y, px=None, py=None, **corr):
    """the correlation dict of one candidate, as Python scalars"""
    x = np.asarray([x], dtype=np.float64)
    px = np.ones_like(x, dtype=np.uint8) if px is None else np.asarray([px], dtype=np.uint8)
    return {k: v[0].item() for k, v in cr.correlations(x, px, y, py, **corr).items()}


def scalar(x, px, y, py, direction, absent, max_lag, min_points):
    """The SPEC statistic of one candidate with Python floats, one lag and one j at a time."""
    P = len(y)
    x = [x[a] if px[a] else 0.0 for a in range(P)]
    y = [y[j] if py[j] else 0.0 for j in range(P)]
    best = None
    used0, r0 = 0, 0.0
    for L in range(max_lag + 1):
        pairs = [(x[j - L], y[j]) for j in range(L, P) if absent == ZERO or (px[j - L] and py[j])]
        u = len(pairs)
        sx = sy = 0.0
        for a, b in pairs:
            sx += a
            sy += b
        mx, my = (sx / u, sy / u) if u else (0.0, 0.0)
        sxx = syy = sxy = 0.0
        for a, b in pairs:
            dx, dy = a - mx, b - my
            sxx += dx * dx
            syy += dy * dy
            sxy += dx * dy
        den = math.sqrt(sxx) * math.sqrt(syy)
        defined = u >= min_points and den > 0
        r = min(max(sxy / den, -1.0), 1.0) if defined else 0.0
        if L == 0:
            used0, r0 = u, r
        if defined:
            s = r if direction == POS else (0.0 - r if direction == NEG else abs(r))
            if best is None or s > best[3]:
                best = (L, u, r, s)
    if best is None:
        return dict(valid=0, lag=0, used=used0, r=0.0, score=0.0, r0=r0)
    return dict(valid=1, lag=best[0], used=best[1], r=best[2], score=best[3], r0=r0)


def test_a_scaled_copy_correlates_exactly():
    y = [0.0, 2.0, 0.0, 2.0]          # deviations +-1 and +-3: every sum and square root is exact
    c = one([3 * v + 10 for v in y], y)
    assert c["valid"] == 1 and c["lag"] == 0 and c["used"] == 4
    assert c["r"] == 1.0 == c["score"] == c["r0"]
    n = one([-v for v in y], y)
    assert n["r"] == -1.0 and n["score"] == -1.0
    assert one([-v for v in y], y, direction=NEG)["score"] == 1.0
    assert one([-v for v in y], y, direction=ABS)["score"] == 1.0


def test_hand_worked_r_with_its_roundings():
    x, y = [1.0, 2.0, 4.0], [1.0, 3.0, 2.0]
    mx, my = 7.0 / 3, 2.0
    dx = [v - mx for v in x]
    dy = [v - my for v in y]
    sxx = ((0.0 + dx[0] * dx[0]) + dx[1] * dx[1]) + dx[2] * dx[2]
    syy = ((0.0 + dy[0] * dy[0]) + dy[1] * dy[1]) + dy[2] * dy[2]
    sxy = ((0.0 + dx[0] * dy[0]) + dx[1] * dy[1]) + dx[2] * dy[2]
    c = one(x, y)
    assert c["r"] == sxy / (math.sqrt(sxx) * math.sqrt(syy)) and c["used"] == 3


def test_a_leading_candidate_is_found_at_its_lag():
    rng = np.random.default_rng(5)
    base = rng.normal(size=40)
    x = base[3:]                     # the target follows the candidate three points later: y[j] = x[j - 3]
    y = base[:-3]
    c = one(x, y, max_lag=8)
    assert c["lag"] == 3 and abs(c["r"] - 1.0) < 1e-15 and c["used"] == len(y) - 3
    assert c["r0"] < 0.9


def test_ties_take_the_smallest_lag():
    # period-2 series and a target absent at j < 3: lags 0 and 2 use the same pairs in the same order, and so do lags
    # 1 and 3, so their scores tie bit for bit
    rng = np.random.default_rng(2)
    y = np.tile([0.0, 1.0], 8) + np.repeat(rng.normal(size=8) * 1e-3, 2)
    x = np.tile([3.0, 5.0], 8)
    py = [0, 0, 0] + [1] * 13
    full = cr.correlations(np.stack([x]), np.ones((1, 16), np.uint8), y, py, max_lag=3)
    c = one(x, y, py=py, max_lag=3)
    assert c["lag"] == 0 and c["r"] > 0.99
    assert one(x, y, py=py, max_lag=3, direction=NEG)["lag"] == 1
    per_lag = [one(x, y, py=py, max_lag=L)["score"] for L in range(4)]
    assert full["score"][0] == per_lag[3] and c["r"] == one(x[2:], y[2:], py=py[2:])["r"]


def test_constant_series_and_min_points_leave_lags_undefined():
    y = [1.0, 2.0, 3.0, 4.0]
    assert one([5.0] * 4, y)["valid"] == 0
    assert one(y, [7.0] * 4)["valid"] == 0
    c = one(y, y, min_points=5)
    assert c["valid"] == 0 and c["used"] == 4 and c["r"] == 0.0 == c["r0"] == c["score"]
    assert one(y, y, max_lag=1, min_points=4)["lag"] == 0
    assert one(y[1:] + [0.0], y, max_lag=1, min_points=3)["lag"] == 1


def test_skip_and_zero_treat_holes_differently():
    x, px = [1.0, 9.0, 3.0, 4.0, 5.0], [1, 0, 1, 1, 1]
    y = [1.0, 2.0, 3.0, 4.0, 5.0]
    s = one(x, y, px)
    assert s["used"] == 4 and s["r"] == 1.0
    z = one(x, y, px, absent=ZERO)
    assert z["used"] == 5 and z["r"] < 1.0
    t = one(y, y, py=[1, 1, 0, 1, 1])
    assert t["used"] == 4 and abs(t["r"] - 1.0) < 1e-15


def test_r_past_one_is_clamped():
    rng = np.random.default_rng(11)
    hit = False
    for _ in range(2000):
        y = rng.normal(size=7) * 10.0 ** rng.integers(-3, 4)
        x = y * rng.choice([3.0, 0.1, 7.0, 1e-3])
        c = one(x, y)
        s = scalar(list(x), [1] * 7, list(y), [1] * 7, POS, SKIP, 0, 3)
        assert c["r"] <= 1.0 and c["r"] == s["r"]
        hit |= (np.dot(x - x.mean(), y - y.mean()) > 0 and c["r"] == 1.0)
    assert hit


def test_top_ranks_by_score_then_row():
    y = np.arange(8.0)
    x = np.stack([y, -y, y * y, y, np.full(8, 2.0)])
    rec = cr.records(None, x, np.ones_like(x, np.uint8), y)
    idx, above = cr.top(rec, 10)
    assert above == 4 and list(idx) == [0, 3, 2, 1]
    idx, above = cr.top(rec, 10, min_score=0.5)
    assert list(idx) == [0, 3, 2] and above == 3


series = st.integers(3, 24).flatmap(lambda P: st.tuples(
    st.lists(st.floats(-1e6, 1e6, allow_nan=False), min_size=P, max_size=P),
    st.lists(st.integers(0, 1), min_size=P, max_size=P),
    st.lists(st.floats(-1e6, 1e6, allow_nan=False), min_size=P, max_size=P),
    st.lists(st.integers(0, 1), min_size=P, max_size=P)))


@settings(max_examples=300, deadline=None)
@given(series, st.sampled_from([POS, NEG, ABS]), st.sampled_from([SKIP, ZERO]), st.integers(0, 6),
       st.integers(3, 6))
def test_matches_a_scalar_loop_bit_for_bit(s, direction, absent, max_lag, min_points):
    x, px, y, py = s
    c = one(x, y, px, py, direction=direction, absent=absent, max_lag=max_lag, min_points=min_points)
    e = scalar(x, px, y, py, direction, absent, max_lag, min_points)
    for k in ("valid", "lag", "used"):
        assert c[k] == e[k], k
    for k in ("r", "score", "r0"):
        assert np.float64(c[k]).tobytes() == np.float64(e[k]).tobytes(), k


@settings(max_examples=200, deadline=None)
@given(st.integers(4, 60), st.integers(0, 2 ** 32 - 1))
def test_matches_corrcoef(P, seed):
    rng = np.random.default_rng(seed)
    y = rng.normal(size=P) * 100.0
    x = 0.5 * y + rng.normal(size=P) * 50.0
    c = one(x, y)
    assert abs(c["r"] - np.corrcoef(x, y)[0, 1]) < 1e-12
