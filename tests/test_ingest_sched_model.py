"""CPU: the ingest kernel's chunk schedule (static rounds, then chunks claimed from a cursor) on its host model
(sched_model.py). A chunk taken twice would count its records twice, one never taken would drop them, and a warp
whose sequence went down again would wait on a copy it never requested: each case runs every warp of a launch to
its end in random interleavings and checks that every chunk is read exactly once, each warp's in increasing order."""
import random

import pytest

import sched_model as sm

H100_SMS = 132
ROUND = H100_SMS * sm.WARPS * sm.CHUNK          # records in one round of chunks on an H100


def boundary_sizes(sms):
    """Record counts around the first claimed chunk: the last static chunk, the first and second claimed ones."""
    stride = sms * sm.WARPS
    out = []
    for rounds in (3, 8, 11, 200):
        st = rounds - rounds * sm.DYN_EIGHTHS // 8
        d0 = st * stride
        for nc in (d0 - 1, d0, d0 + 1, d0 + 2):
            if (nc + stride - 1) // stride == rounds:   # the split is the one computed for `rounds`
                out.append(nc * sm.CHUNK)
    return out


def test_split_rule():
    """Up to two rounds, nothing is claimed; the static part is the first 5/8 of the rounds, rounded up."""
    stride = H100_SMS * sm.WARPS
    assert sm.split(1, H100_SMS) == (1, stride)
    assert sm.split(2 * ROUND, H100_SMS) == (2, 2 * stride)
    assert sm.split(2 * ROUND + 1, H100_SMS) == (2, 2 * stride)   # 3 rounds: the third is claimed
    assert sm.split(200 * ROUND, H100_SMS) == (125, 125 * stride)
    assert sm.split(100_000_000, H100_SMS) == (463, 463 * stride)  # config 2: 740 rounds, 277 claimed


@pytest.mark.parametrize("n", [1, 63, 64, 65, 127, 128, 129, ROUND - 1, ROUND, ROUND + 1, 2 * ROUND + 1,
                               3 * ROUND - 1, 3 * ROUND])
def test_ragged_sizes_h100_grid(n):
    for seed in range(3):
        sm.check(n, H100_SMS, random.Random(seed))


@pytest.mark.parametrize("n", boundary_sizes(H100_SMS))
def test_static_claimed_boundary(n):
    sm.check(n, H100_SMS, random.Random(n))


@pytest.mark.parametrize("sms", [1, 2, 3, 5])
def test_every_size_small_grids(sms):
    """Every chunk count up to 14 rounds on small grids, partial last chunks included: every static/claimed
    boundary, a partial chunk in either part, and warps that get no chunk at all."""
    stride = sms * sm.WARPS
    rng = random.Random(sms)
    for nc in range(1, 14 * stride + 2):
        sm.check(nc * sm.CHUNK - rng.randrange(sm.CHUNK), sms, rng)


def test_partial_last_chunk_claimed():
    n = 11 * ROUND - 5 * sm.CHUNK - 17
    st, d0 = sm.split(n, H100_SMS)
    assert sm.n_chunks(n) - 1 >= d0 and n % sm.CHUNK
    sm.check(n, H100_SMS, random.Random(1))


def test_more_warps_than_chunks():
    for n in (1, 5 * sm.CHUNK + 1, (H100_SMS * sm.WARPS - 1) * sm.CHUNK):
        taken = sm.check(n, H100_SMS, random.Random(n))
        assert sum(1 for t in taken if t) == sm.n_chunks(n)


def test_fast_ctas_take_more():
    """CTAs that run twice as fast take about twice as many of the claimed chunks; the static ones stay put."""
    sms = 4
    n = 64 * sms * sm.WARPS * sm.CHUNK
    speed = [2.0, 1.0, 1.0, 1.0]
    taken = sm.check(n, sms, random.Random(7), speed)
    st, d0 = sm.split(n, sms)
    per_cta = [sum(1 for t in taken[b * sm.WARPS:(b + 1) * sm.WARPS] for c in t if c >= d0) for b in range(sms)]
    static = [sum(1 for t in taken[b * sm.WARPS:(b + 1) * sm.WARPS] for c in t if c < d0) for b in range(sms)]
    assert static == [st * sm.WARPS] * sms
    assert per_cta[0] > 1.5 * max(per_cta[1:])
