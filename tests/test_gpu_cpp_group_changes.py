"""GPU: the C++ host adapter's group changes (tests/cpp/group_changes_adapter_test.cc, built with g++ against
libalazgpu.so): GroupChanges and GroupNodeChanges through a rolling deploy against a pinned window, with NodeChanges
listing the replaced pods as GONE and NEW."""
import os
import subprocess

import pytest

from alaz_b200 import build

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_group_changes_through_cpp_adapter(tmp_path):
    lib = build.build()
    exe = str(tmp_path / "group_changes_adapter_test")
    srcs = [os.path.join(ROOT, "tests", "cpp", "group_changes_adapter_test.cc"),
            os.path.join(ROOT, "alaz_b200", "host", "alaz_aggregator.cc")]
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror"] + srcs +
                   ["-L" + os.path.dirname(lib), "-lalazgpu", "-Wl,-rpath," + os.path.dirname(lib), "-o", exe],
                   check=True, capture_output=True, text=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "group changes adapter ok" in r.stdout
