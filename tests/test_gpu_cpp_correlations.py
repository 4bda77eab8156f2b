"""GPU: the C++ host adapter's correlations (tests/cpp/corr_adapter_test.cc, built with g++ against libalazgpu.so):
Correlations, NodeCorrelations, GroupCorrelations and GroupNodeCorrelations on a small service map where a
dependency's p99 leads its caller's by one window."""
import os
import subprocess

import pytest

from alaz_b200 import build

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_correlations_through_cpp_adapter(tmp_path):
    lib = build.build()
    exe = str(tmp_path / "corr_adapter_test")
    srcs = [os.path.join(ROOT, "tests", "cpp", "corr_adapter_test.cc"),
            os.path.join(ROOT, "alaz_b200", "host", "alaz_aggregator.cc")]
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror"] + srcs +
                   ["-L" + os.path.dirname(lib), "-lalazgpu", "-Wl,-rpath," + os.path.dirname(lib), "-o", exe],
                   check=True, capture_output=True, text=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "corr adapter ok" in r.stdout
