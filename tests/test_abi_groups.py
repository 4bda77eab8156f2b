"""CPU: the layout of alz_group_info (include/alazgpu.h, docs/SPEC.md §24) matches the Python mirror in alaz_b200/abi.py,
ALZ_NODE_GROUP follows the flushed node types, and the group entry points are declared, exported by the library and
bound."""
import ctypes as C
import os
import re
import subprocess

from alaz_b200 import abi, build, capi
from test_abi_changes import _run
from test_abi_nodes import _layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INFO_FIELDS = ["source_rows", "mapped_ends", "edges", "internal"]
SYMBOLS = ["alz_group_set", "alz_group_edges", "alz_group_edges_device", "alz_group_edge_metrics",
           "alz_group_edge_metrics_device", "alz_group_edge_top", "alz_group_edge_top_device", "alz_group_nodes",
           "alz_group_nodes_device", "alz_group_node_metrics", "alz_group_node_metrics_device", "alz_group_node_top",
           "alz_group_node_top_device"]
HOOK = "alz_debug_group_edges"


def test_group_info_layout():
    got = _layout("alz_group_info", INFO_FIELDS)
    assert got[0] == C.sizeof(abi.GROUP_INFO) == 32
    assert got[1:] == [getattr(abi.GROUP_INFO, f).offset for f in INFO_FIELDS] == [0, 8, 16, 24]


def test_node_group_constant():
    got = _run("""
    #include <stdio.h>
    #include "alazgpu.h"
    int main(void){ printf("%d %d ", (int)ALZ_NODE_GROUP, (int)ALZ_NODE_OUTBOUND_HOST); return 0; }
    """)
    assert got == [abi.NODE_GROUP, abi.NODE_OUTBOUND_HOST] == [4, 3]


def test_group_symbols_are_declared_exported_and_bound():
    header = open(os.path.join(ROOT, "include", "alazgpu.h")).read()
    synth = open(os.path.join(ROOT, "include", "alazgpu_synth.h")).read()
    for s in SYMBOLS:
        assert re.search(r"\bint " + s + r"\(", header), s
        assert s in capi.EXPORTS, s
    assert re.search(r"\bint " + HOOK + r"\(", synth)
    if os.path.exists(build.LIB):
        syms = subprocess.check_output(["nm", "-D", "--defined-only", build.LIB], text=True)
        for s in SYMBOLS + [HOOK]:
            assert re.search(r"\bT " + s + r"$", syms, re.M), s
    src = open(os.path.join(ROOT, "alaz_b200", "capi.py")).read()
    for s in SYMBOLS + [HOOK]:
        assert f'"{s}": (' in src, s
