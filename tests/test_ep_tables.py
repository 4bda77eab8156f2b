"""CPU: the constructors and models of tests/ep_tables.py. The numpy hash32 and filter bits must equal the header's,
the constructors must deliver the homes and bits they promise, and the mirror model must keep the probing invariants,
or the endpoint-table tests would check the wrong layouts."""
import os
import subprocess

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import ep_tables as et
from alaz_b200 import abi
from test_ingest_streams import ROOT, _nvcc

_PROG = r"""
#include <cstdio>
#include <cstdlib>
#include "alaz_b200/csrc/alz_device.cuh"
int main(int argc, char** argv) {
  for (int i = 1; i < argc; ++i) {
    const uint32_t h = alz::hash32((uint32_t)strtoul(argv[i], nullptr, 0));
    // the filter bits as bloom_update (alz_api.cu) and maybe_pod (alz_ingest.cu) take them
    printf("%u %u %u\n", h, h & (ALZ_BLOOM_WORDS * 32u - 1u), (h >> 15) & (ALZ_BLOOM_WORDS * 32u - 1u));
  }
  return 0;
}
"""

EDGE_IPS = [0, 1, 2, 0xFFFF, 0x10000, 0x7FFFFFFF, 0x80000000, et.M32, et.HOST_DADDR]


def test_hash32_and_filter_bits_match_header(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    src, exe = tmp_path / "h32.cu", tmp_path / "h32"
    src.write_text(_PROG)
    subprocess.run([nvcc, "-std=c++17", "-I", ROOT, str(src), "-o", str(exe)], check=True, capture_output=True)
    ips = np.concatenate([np.random.default_rng(7).integers(0, 1 << 32, 300, dtype=np.uint64),
                          np.array(EDGE_IPS, np.uint64)]).astype(np.uint32)
    out = subprocess.run([str(exe)] + [str(int(x)) for x in ips], check=True, capture_output=True, text=True).stdout
    got = np.array([[int(v) for v in line.split()] for line in out.splitlines()], np.int64)
    b1, b2 = et.filter_bits(ips)
    assert got[:, 0].tolist() == et.hash32(ips).tolist()
    assert got[:, 1].tolist() == b1.tolist() and got[:, 2].tolist() == b2.tolist()


def test_unhash32_round_trip():
    rng = np.random.default_rng(1)
    xs = np.concatenate([rng.integers(0, 1 << 32, 100_000, dtype=np.uint64), np.array(EDGE_IPS, np.uint64)])
    xs = xs.astype(np.uint32)
    assert np.array_equal(et.unhash32(et.hash32(xs)), xs)
    assert np.array_equal(et.hash32(et.unhash32(xs)), xs)


def test_ep_cap():
    assert [et.ep_cap(n) for n in (1, 2, 3, 32, 33, 64, 1 << 20, 1 << 30, (1 << 30) + 1, 1 << 31)] == \
        [2, 4, 8, 64, 128, 128, 1 << 21, 1 << 31, 1 << 31, 1 << 31]


@pytest.mark.parametrize("cap", [64, 128, 1 << 14, 1 << 21])
def test_with_home(cap):
    for slot in (0, 1, cap - 4, cap - 1):
        a = et.with_home(cap, slot, 40, seed=slot)
        assert len(set(a)) == 40 and not set(a) & set(et.SPECIAL)
        assert np.all(et.home(a, cap) == slot)
        assert len({int(b) for b in et.filter_bits(a)[0]}) > 1 or cap >= et.BLOOM_BITS


def test_filter_bit_constructors():
    x = 0x1ABCD
    a = et.with_b1(x, 20)
    assert np.all(et.filter_bits(a)[0] == x) and len(set(et.filter_bits(a)[1].tolist())) == 20
    assert np.all(et.home(a, 128) == x & 127) and np.all(et.home(a, 1 << 17) == x)   # same b1 => same home
    b = et.with_b2(x, 20)
    assert np.all(et.filter_bits(b)[1] == x) and len(set(et.filter_bits(b)[0].tolist())) == 20
    c = et.equal_bits(10)
    b1, b2 = et.filter_bits(c)
    assert np.array_equal(b1, b2) and len(set(b1.tolist())) == 10
    y = et.with_bits(0x2ABC0 & et.BLOOM_MASK | (1 << 15), 0x12345 & ~3 | 1)
    assert [int(v) for v in et.filter_bits(y)] == [0x2ABC0 & et.BLOOM_MASK | (1 << 15), 0x12345 & ~3 | 1]


def test_false_positives_pass_the_filter_and_are_not_pods():
    pods = et.random_addrs(300, seed=3)
    fp = et.false_positives(pods, 50)
    m = et.FilterModel()
    for p in pods:
        m.update(p, +1)
    bits = m.bitmap()
    assert not set(fp) & set(pods)
    for a in fp:
        assert all(bits[int(b)] for b in et.filter_bits(a))
    # a pod set of two, built around an address: the address passes and is not one of them
    h = 0x5A5A1234
    b1, b2 = h & et.BLOOM_MASK, (h >> 15) & et.BLOOM_MASK
    pa, pb = et.with_b1(b1, 1, avoid=[et.unhash32(h)])[0], et.with_b2(b2, 1, avoid=[et.unhash32(h)])[0]
    assert int(et.unhash32(h)) in et.false_positives([pa, pb], 5)


def test_filter_model_saturates_and_counts_back():
    m = et.FilterModel()
    a = et.with_b2(77, 300)
    for x in a:
        m.update(x, +1)
    assert m.cnt[77] == 255
    for x in a[:299]:
        m.update(x, -1)
    assert m.cnt[77] == 255 and m.bitmap().sum() == 1 + 1   # the saturated bit and the last address's b1
    c = et.with_b1(5, 2)
    m.update(c[0], +1), m.update(c[1], +1), m.update(c[0], -1)
    assert m.cnt[5] == 1


def test_wrapped_chain_layout():
    """The layout of the GPU test's chain across the end: entries homed at cap - 4 fill the last four slots and run on
    from slot 0, entries homed at 0..3 land behind them; deleting an entry before the wrap moves later ones back
    across it."""
    m = et.MirrorModel(32)
    cap = m.cap
    chain, low, order = et.wrapped_chain(cap)
    for k, ip in enumerate(order):
        assert m.upsert(abi.TABLE_POD, ip, k) == abi.OK
    m.commit()
    m.check()
    assert [m.slot_of(x) for x in chain] == [cap - 4, cap - 3, cap - 2, cap - 1, 1, 2, 4, 5, 6, 8, 9, 10]
    assert [m.slot_of(x) for x in low] == [0, 11, 7, 3]
    absent = et.with_home(cap, cap - 4, 13, seed=1)[12]
    assert m.probes(absent) == 17                                     # 16 occupied slots, then slot 12
    m.erase(abi.TABLE_POD, chain[1])
    m.commit()
    m.check()
    assert m.slot_of(chain[4]) == cap - 1                              # moved back across the end
    assert m.slot_of(low[0]) == 0 and m.slot_of(low[3]) == 3           # stay at their homes
    assert m.slot_of(chain[6]) == 2                                    # jumps over low[3]
    assert m.slot_of(low[1]) == 10 and not m.occ[11]


def test_merged_chains_layout():
    m = et.MirrorModel(32)
    a, b, order = et.merged_chains(m.cap, 20, 4)
    for k, ip in enumerate(order):
        m.upsert(abi.TABLE_SVC, ip, k)
    m.commit()
    assert [m.slot_of(x) for x in order] == list(range(20, 28))
    m.erase(abi.TABLE_SVC, a[0])
    m.commit()
    m.check()
    assert m.slot_of(b[0]) == 21 and m.slot_of(a[1]) == 20 and m.slot_of(b[1]) == 22   # b[0] stays at its home


_ops = st.lists(st.tuples(st.sampled_from("uuuec"), st.integers(0, 47), st.integers(0, 1)), max_size=120)


@settings(max_examples=300, deadline=None)
@given(_ops)
def test_mirror_model_invariants(ops):
    """Random upserts, erases and commits on a 48-address universe homed into three adjacent slots near the end of a
    64-slot table of 32 endpoints: keys stay reachable, occupied slots equal keys, absent lookups stop at a free slot,
    and the mirror equals the host map at every commit."""
    m = et.MirrorModel(32)
    U = [a for s in (60, 61, 62) for a in et.with_home(m.cap, s, 16, seed=s)]
    for op, k, t in ops:
        if op == "u":
            exp = abi.OK if U[k] in m.host or len(m.host) < 32 else abi.E_CAPACITY
            assert m.upsert(t, U[k], k) == exp
        elif op == "e":
            m.erase(t, U[k])
        else:
            m.commit()
            m.check()
            assert m.occ.sum() == len(m.host) <= 32
            assert m.committed() == {ip: tuple(v) for ip, v in m.host.items()}
            for a in U:
                n = m.probes(a)
                s = (m.home(a) + n - 1) & m.mask
                assert (m.slot_of(a) == s) if a in m.host else not m.occ[s]
