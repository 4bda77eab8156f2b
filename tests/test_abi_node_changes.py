"""CPU: the layout of alz_node_change (include/alazgpu.h, docs/SPEC.md §23) matches the Python mirror in
alaz_b200/abi.py, it shares alz_edge_change's offsets from presence on (the gather of the top records serves both),
its node value sits where alz_node_trend's does, and the node change entry points are declared, exported by the
library and bound."""
import os
import re
import subprocess

from alaz_b200 import abi, build, capi
from test_abi_nodes import _layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ["alz_node_changes", "alz_node_changes_device", "alz_node_changes_top", "alz_node_changes_top_device"]
SHARED = ["presence", "index", "base_index", "value", "base_value", "change"]


def test_node_change_layout():
    got = _layout("alz_node_change", list(abi.NODE_CHANGE.names))
    assert got[0] == abi.NODE_CHANGE.itemsize == 48
    assert got[1:] == [abi.NODE_CHANGE.fields[f][1] for f in abi.NODE_CHANGE.names] == \
        [0, 1, 2, 3, 8, 12, 16, 20, 24, 32, 40]


def test_node_change_shares_the_edge_change_offsets():
    assert _layout("alz_node_change", SHARED) == _layout("alz_edge_change", SHARED)
    assert [abi.NODE_CHANGE.fields[f][1] for f in SHARED] == [abi.EDGE_CHANGE.fields[f][1] for f in SHARED]
    assert _layout("alz_node_change", ["type", "node"])[1:] == _layout("alz_node_trend", ["type", "value"])[1:]


def test_node_changes_symbols_are_declared_exported_and_bound():
    header = open(os.path.join(ROOT, "include", "alazgpu.h")).read()
    synth = open(os.path.join(ROOT, "include", "alazgpu_synth.h")).read()
    for s in SYMBOLS:
        assert re.search(r"\bint " + s + r"\(", header), s
        assert s in capi.EXPORTS, s
    assert re.search(r"\bint alz_debug_node_changes_rows\(", synth)
    bound = SYMBOLS + ["alz_debug_node_changes_rows"]
    if os.path.exists(build.LIB):
        syms = subprocess.check_output(["nm", "-D", "--defined-only", build.LIB], text=True)
        for s in bound:
            assert re.search(r"\bT " + s + r"$", syms, re.M), s
    src = open(os.path.join(ROOT, "alaz_b200", "capi.py")).read()
    for s in bound:
        assert f'"{s}": (' in src, s
