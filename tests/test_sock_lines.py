"""CPU: the socket-timeline builders of tests/sock_lines.py, and the hand-derived boundary lines on the C restatement
against the Python one. The GPU tests aim at the device's index and pool with these builders and compare against the
C restatement, so both must be right first."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import oracle_lib as ol
import sock_lines as sl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import ref_py  # noqa: E402

_PROG = r"""
#include <cstdio>
#include <cstdlib>
#include "alaz_b200/csrc/alz_device.cuh"
int main(int argc, char** argv) {
  for (int i = 1; i + 1 < argc; i += 2) {
    const unsigned long long x = strtoull(argv[i], nullptr, 0), fd = strtoull(argv[i + 1], nullptr, 0);
    const uint32_t pid = (uint32_t)x;   // alz_sock.cu line_slot: ((uint64_t)pid << 40) ^ fd ^ golden
    printf("%llu %llu\n", (unsigned long long)alz::hash64(x),
           (unsigned long long)alz::hash64(((uint64_t)pid << 40) ^ fd ^ 0x9E3779B97F4A7C15ull));
  }
  return 0;
}
"""


def _nvcc():
    return shutil.which("nvcc") or next((p for p in [os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"),
                                                                  "bin", "nvcc")] if os.path.exists(p)), None)


def test_hash64_matches_header(tmp_path):
    """The numpy hash64 against the header's __host__ __device__ one, compiled for the host; and the line hash input."""
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    src, exe = tmp_path / "h64.cu", tmp_path / "h64"
    src.write_text(_PROG)
    subprocess.run([nvcc, "-std=c++17", "-I", ROOT, str(src), "-o", str(exe)], check=True, capture_output=True)
    rng = np.random.default_rng(6)
    xs = [int(v) for v in rng.integers(0, 1 << 63, 100, dtype=np.uint64) * np.uint64(2) + np.uint64(1)]
    xs += [0, 1, 1 << 40, (1 << 64) - 1, 1 << 24, (1 << 24) + 5, (1 << 32) - 1, 0xFFFFFF]
    fds = [int(v) for v in rng.integers(0, 1 << 63, len(xs), dtype=np.uint64)]
    fds[-8:] = [0, 7, (1 << 64) - 1, 1 << 40, 3, 3, 9, 0]
    args = [str(a) for x, f in zip(xs, fds) for a in (x, f)]
    out = subprocess.run([str(exe)] + args, check=True, capture_output=True, text=True).stdout.split()
    got_h = [int(v) for v in out[0::2]]
    got_line = [int(v) for v in out[1::2]]
    assert got_h == sl.hash64(np.array(xs, dtype=np.uint64)).tolist()
    pids = [x & 0xFFFFFFFF for x in xs]
    assert got_line == sl.hash64(sl.line_key(np.array(pids, np.uint64), np.array(fds, np.uint64))).tolist()


@pytest.mark.parametrize("mask", [15, 31, 511, 4095])
def test_keys_with_one_home(mask):
    keys = sl.keys_with_home(mask, 5, 64)
    assert len(set(keys)) == 64
    assert all(int(sl.line_slot(p, f, mask)) == 5 for p, f in keys)


@pytest.mark.parametrize("mask", [31, 511])
def test_wrap_chain(mask):
    keys = sl.wrap_chain(mask, 5)
    assert len(set(keys)) == 6
    assert [int(sl.line_slot(p, f, mask)) for p, f in keys] == [mask - 1] * 5 + [0]


def test_alias_pairs_share_the_hash_input():
    for pid, fd in [(0x123, 0x45), (1, 0), ((1 << 24) - 1, (1 << 64) - 1)]:
        for a, b in sl.alias_pairs(pid, fd):
            assert a != b
            assert int(sl.line_key(*a)) == int(sl.line_key(*b))
    # bits 24..31 of the pid never reach the hash
    assert int(sl.line_key(0xFF000123, 9)) == int(sl.line_key(0x123, 9))


def test_index_and_segment_rules():
    assert [sl.index_cap_for(n) for n in (1, 8, 9, 33, 64)] == [16, 64, 64, 256, 512]
    assert sl.index_cap_for(8, 16) == 16 and sl.index_cap_for(9, 16) == 64
    assert [sl.seg_cap_for(n) for n in (0, 1, 10, 11, 12, 16, 17, 40000)] == [16, 16, 16, 16, 32, 32, 32, 65536]


@settings(max_examples=200, deadline=None)
@given(steps=st.lists(st.lists(st.tuples(st.integers(0, 40), st.integers(1, 3000)), max_size=12), max_size=12))
def test_pool_garbage_stays_below_the_live_segments(steps):
    """A moved segment is at least twice the one it leaves, so a line's dead segments add up to less than its live one,
    and the garbage clause of the repool rule (garbage > used / 2) cannot fire on its own: only a full pool re-lays."""
    m = sl.SyncModel()
    lens = {}
    for step in steps:
        for line, grow in step:
            lens[(line, 3)] = lens.get((line, 3), 0) + grow
        m.sync(dict(lens))
        assert m.garbage * 2 <= m.used
    assert m.garbage_repools == 0


# ---- the C restatement against the Python one on hand-derived lines -----------------------------------------------

class _C:
    def __init__(self):
        self.o = ol.SockMaps()

    def op(self, op):
        self.o.process(sl.script_rec(op))

    def get(self, key, ts, now):
        r = self.o.lookup(sl.query(key[0], key[1], ts), now_ns=now)[0]
        return sl.found_k(r["saddr"]) if r["found"] else None

    def gc(self):
        self.o.gc()

    def records(self):
        return self.o.records()


class _Py:
    def __init__(self):
        self.p = ref_py.SocketMaps()

    def op(self, op):
        r = sl.script_rec(op)[0]
        self.p.process_tcp(int(r["type"]), int(r["pid"]), int(r["fd"]), int(r["timestamp_ns"]), int(r["saddr"]),
                           int(r["daddr"]), int(r["sport"]), int(r["dport"]))

    def get(self, key, ts, now):
        r = self.p.lookup(key[0], key[1], ts, now)
        return None if r is None else sl.found_k(r[0])

    def gc(self):
        self.p.gc()

    def records(self):
        return sum(len(ln.values) for ln in self.p.lines.values())


def run_script(side, ops):
    out = []
    for op in ops:
        if op[0] in ("o", "c"):
            side.op(op)
        elif op[0] == "get":
            out.append(side.get(*op[1:]))
        else:
            side.gc()
            out.append(side.records())
    return out


@pytest.mark.parametrize("name", sorted(sl.BOUNDARY))
def test_boundary_lines_on_both_restatements(name):
    ops, expected = sl.BOUNDARY[name]
    assert run_script(_C(), ops) == expected
    assert run_script(_Py(), ops) == expected


@pytest.mark.parametrize("d", [-1, 0, 1])
def test_five_minute_test_wraps_mod_2_64(d):
    """Go adds LastMatch + 5 min in uint64: a stamp within five minutes of 2^64 wraps to a small sum, so its own pair is
    dropped although it holds the largest stamp. Both restatements must agree (C: 1 record; before the Python one
    masked the sum, it kept 3)."""
    x = (1 << 64) - 5 * sl.MINUTE + d
    for stamp in (x, sl.M64):
        ops, expected = sl._near_wrap(stamp)
        c, p = run_script(_C(), ops), run_script(_Py(), ops)
        assert c == p == expected, (stamp, c, p)
    # the case as reported: open@10, close@20, open@30, close@40, open@50, open@60, lookups at 15 and 35
    c, p = _C(), _Py()
    for ts, k in ((10, 1), (20, None), (30, 2), (40, None), (50, 3), (60, 4)):
        op = ("o", sl.K, ts, k) if k else ("c", sl.K, ts)
        c.op(op)
        p.op(op)
    for side in (c, p):
        side.get(sl.K, 15, sl.M64)
        side.get(sl.K, 35, 10**9)
        side.gc()
    assert c.records() == p.records() == 1
