"""CPU: the stream builders of tests/ingest_streams.py. scaled_oracle must equal the oracle on the tiled stream, and
the numpy hashes must equal the ones the kernels use, or the ingest tier tests would check the wrong thing."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import ingest_streams as ist
import oracle_lib as ol
from alaz_b200 import abi
from helpers import edges_equal, explain_diff

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POD, POD2, SVC = abi.ip("10.0.0.1"), abi.ip("10.0.0.2"), abi.ip("172.16.0.1")
TABLES = [(abi.TABLE_POD, [POD, POD2], [1, 2]), (abi.TABLE_SVC, [SVC], [7])]


def _pattern(kind, rng):
    n = 40
    if kind == "mixed":      # forward, reversed, host-keyed, unresolved, not-a-request rows, 5xx
        r = ist.records(np.where(np.arange(n) % 5 == 4, abi.ip("9.9.9.9"), POD), SVC,
                        rng.integers(0, 1 << 42, n), status=rng.choice([200, 500, 503], n))
        r["protocol"][::7] = abi.PROTO_KAFKA
        r["protocol"][1::6] = abi.PROTO_AMQP
        r["method_flags"][1::6] = abi.AMQP_DELIVER
        r["protocol"][2::9] |= abi.PROTO_F_HOSTKEY
        r["daddr"][2::9] = 77
        return r
    if kind == "wrapping":   # lat sums past 2^64 within a few periods
        return ist.records(POD, SVC, np.array([(1 << 64) - 1, (1 << 63) + 12345, 1 << 62, 999], np.uint64))
    return ist.records(POD2, POD, 3_000_000, status=503)   # one record


@pytest.mark.parametrize("kind", ["mixed", "wrapping", "single"])
@pytest.mark.parametrize("reps", [1, 3, 17])
@pytest.mark.parametrize("with_prefix", [False, True])
def test_scaled_oracle_equals_oracle_on_tiled_stream(kind, reps, with_prefix):
    rng = np.random.default_rng(reps)
    pat = _pattern(kind, rng)
    prefix = _pattern("wrapping", rng)[::-1].copy() if with_prefix else None
    got, gst = ist.scaled_oracle(TABLES, pat, reps, prefix)
    stream = np.concatenate(([prefix] if with_prefix else []) + [np.tile(pat, reps)])
    exp, est = ist.oracle_run(TABLES, stream)
    assert edges_equal(got, exp), explain_diff(got, exp)
    assert gst == est
    if kind == "wrapping" and reps > 1:
        assert int(exp["lat_sum_ns"].max()) < sum(int(d) for d in pat["duration_ns"]) * reps   # it did wrap


def test_hist_cells_wrap_mod_2_32():
    """A cell times reps past 2^32 wraps, count does not."""
    got, st = ist.scaled_oracle(TABLES, ist.records(POD, SVC, 1000), (1 << 32) + 5)
    assert len(got) == 1
    assert int(got["count"][0]) == (1 << 32) + 5 and int(got["hist"][0][ist.latency_bucket(1000)]) == 5
    assert st["rows_emitted"] == (1 << 32) + 5


def test_latency_bucket_matches_oracle():
    ds = [0, 1, 255, 256, 383, 384, 511, 512, (1 << 32) - 1, 1 << 32, (1 << 40) - 1, 1 << 40, (1 << 64) - 1]
    ds += [ist.bucket_lo(b) + k for b in range(1, 64) for k in (-1, 0)]
    for d in ds:
        assert ist.latency_bucket(d) == ol.bucket(d), d


def test_table_collisions_by_construction():
    """collide_table gives a second source the same hash (bucket and fingerprint); daddr_for_table_hash a chosen
    one."""
    d2 = ist.collide_table(POD, SVC, POD2)
    h1, h2 = ist.table_hash(ist.pair_key(POD, SVC)), ist.table_hash(ist.pair_key(POD2, d2))
    assert h1 == h2 and ist.tab_fp(h1) == ist.tab_fp(h2) and ist.tab_idx1(h1) == ist.tab_idx1(h2)
    h = 0xDEAD0000 | 0x1234
    assert int(ist.table_hash(ist.pair_key(POD, ist.daddr_for_table_hash(POD, h)))) == h


def test_collide_home():
    for mask in ist.dict_masks(1 << 12):
        keys, slot = ist.collide_home(mask, [POD, POD2], 8)
        assert len(set(keys)) == 8
        k = ist.pair_key([s for s, _ in keys], [d for _, d in keys])
        assert np.all(ist.pair_hash(k) & np.uint32(mask) == slot)


def test_chunk_ownership():
    sms = 132
    n = ist.round_size(sms) + 65
    c = ist.per_cta_counts(n, sms)
    assert c.sum() == n and c[0] == 16 * 64 + 65 and np.all(c[1:] == 16 * 64)
    assert ist.replica_of_record(np.arange(64)).tolist() == [i % 8 for i in range(64)]


_PROG = r"""
#include <cstdio>
#include <cstdlib>
#include "alaz_b200/csrc/alz_device.cuh"
int main(int argc, char** argv) {
  for (int i = 1; i < argc; ++i) printf("%u\n", alz::pair_hash(strtoull(argv[i], nullptr, 0)));
  return 0;
}
"""


def _nvcc():
    return shutil.which("nvcc") or next((p for p in [os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"),
                                                                  "bin", "nvcc")] if os.path.exists(p)), None)


def test_pair_hash_matches_header(tmp_path):
    """The numpy pair_hash against the header's __host__ __device__ one, compiled for the host."""
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    src, exe = tmp_path / "ph.cu", tmp_path / "ph"
    src.write_text(_PROG)
    subprocess.run([nvcc, "-std=c++17", "-I", ROOT, str(src), "-o", str(exe)], check=True, capture_output=True)
    rng = np.random.default_rng(5)
    keys = np.concatenate([rng.integers(0, 1 << 63, 200, dtype=np.uint64) * np.uint64(2) + np.uint64(1),
                           np.array([0, 1, (1 << 32) - 1, 1 << 32, (1 << 64) - 1], np.uint64)])
    out = subprocess.run([str(exe)] + [str(int(k)) for k in keys], check=True, capture_output=True, text=True).stdout
    assert [int(x) for x in out.split()] == ist.pair_hash(keys).tolist()
