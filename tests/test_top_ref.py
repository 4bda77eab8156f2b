"""CPU: the numpy reference of the top anomalous rows (tests/top_ref.py, docs/SPEC.md §16) on hand-written cases. The
GPU tests trust it, so its key function and its order are pinned here."""
import numpy as np
import pytest

import top_ref

F = np.float32
NAN_POS, NAN_NEG = np.uint32(0x7FC00000).view(F), np.uint32(0xFFC00000).view(F)


def test_order_key_is_ieee_total_order():
    vals = np.array([NAN_NEG, -np.inf, -1.0, np.uint32(0x80000001).view(F), -0.0, 0.0,
                     np.uint32(0x00000001).view(F), 0.5, 1.0, np.inf, NAN_POS], dtype=F)
    keys = top_ref.order_key(vals)
    assert np.all(np.diff(keys.astype(np.int64)) > 0), keys
    assert int(top_ref.order_key(F(-0.0))) == 0x7FFFFFFF and int(top_ref.order_key(F(0.0))) == 0x80000000
    assert int(top_ref.order_key(F(1.0))) == 0x3F800000 ^ 0x80000000


def test_hand_written_cases():
    s = np.array([0.5, 0.9, 0.5, -0.0, 0.0, 0.9, NAN_POS, 0.1], dtype=F)
    # NaN (positive sign) ranks first; 0.9 twice: index 1 before 5; then 0.5 at 0 before 2; +0 before -0
    idx, above = top_ref.top(s, 100, float("-inf"))
    assert idx.tolist() == [6, 1, 5, 0, 2, 7, 4, 3] and above == 8
    idx, above = top_ref.top(s, 3, 0.5)              # eligible: NaN, 0.9, 0.9, 0.5, 0.5
    assert idx.tolist() == [6, 1, 5] and above == 5
    idx, above = top_ref.top(s, 10, 0.0)             # +0 is eligible, -0 is not
    assert idx.tolist() == [6, 1, 5, 0, 2, 7, 4] and above == 7
    idx, above = top_ref.top(s, 10, -0.0)
    assert idx.tolist() == [6, 1, 5, 0, 2, 7, 4, 3] and above == 8
    idx, above = top_ref.top(s, 10, float(NAN_POS))  # only the NaN itself
    assert idx.tolist() == [6] and above == 1
    idx, above = top_ref.top(np.full(5, 0.25, F), 3, 0.25)   # a 5-way tie: lowest indices first
    assert idx.tolist() == [0, 1, 2] and above == 5
    idx, above = top_ref.top(s, 4, 2.0)
    assert idx.tolist() == [6] and above == 1         # +NaN is above every number
    idx, above = top_ref.top(np.zeros(0, F), 4, 0.0)
    assert len(idx) == 0 and above == 0


@pytest.mark.parametrize("seed", range(6))
def test_partial_sort_equals_the_definition(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 3000))
    pool = rng.choice(np.array([0.0, -0.0, 0.25, 0.5, 1.0, np.inf, -np.inf, NAN_POS, NAN_NEG], F), 6)
    s = np.where(rng.random(n) < 0.5, rng.choice(pool, n), rng.random(n).astype(F)).astype(F)
    for k in (1, 2, n // 2 + 1, n, n + 5):
        for ms in (float("-inf"), 0.0, -0.0, 0.5, float(s[0]), 2.0):
            a, b = top_ref.top(s, k, ms), top_ref.top_lexsort(s, k, ms)
            assert a[0].tolist() == b[0].tolist() and a[1] == b[1], (k, ms)
