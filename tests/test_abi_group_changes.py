"""CPU: the group change entry points (docs/SPEC.md §25) are declared in include/alazgpu.h, exported by the library and
bound, and their test hook is declared in include/alazgpu_synth.h. They reuse alz_edge_change, alz_node_change and
alz_change_info, whose layouts tests/test_abi_changes.py and tests/test_abi_node_changes.py check."""
import os
import re
import subprocess

from alaz_b200 import build, capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ["alz_group_edge_changes", "alz_group_edge_changes_device", "alz_group_edge_changes_top",
           "alz_group_edge_changes_top_device", "alz_group_node_changes", "alz_group_node_changes_device",
           "alz_group_node_changes_top", "alz_group_node_changes_top_device"]
HOOK = "alz_debug_group_edge_changes_rows"


def test_group_change_symbols_are_declared_exported_and_bound():
    header = open(os.path.join(ROOT, "include", "alazgpu.h")).read()
    synth = open(os.path.join(ROOT, "include", "alazgpu_synth.h")).read()
    for s in SYMBOLS:
        assert re.search(r"\bint " + s + r"\(", header), s
        assert s in capi.EXPORTS, s
    assert re.search(r"\bint " + HOOK + r"\(", synth)
    assert HOOK not in header
    if os.path.exists(build.LIB):
        syms = subprocess.check_output(["nm", "-D", "--defined-only", build.LIB], text=True)
        for s in SYMBOLS + [HOOK]:
            assert re.search(r"\bT " + s + r"$", syms, re.M), s
    src = open(os.path.join(ROOT, "alaz_b200", "capi.py")).read()
    for s in SYMBOLS + [HOOK]:
        assert f'"{s}": (' in src, s
    for m in ("group_edge_changes", "group_edge_changes_device", "group_edge_changes_top",
              "group_edge_changes_top_device", "group_node_changes", "group_node_changes_device",
              "group_node_changes_top", "group_node_changes_top_device", "debug_group_edge_changes_rows"):
        assert callable(getattr(capi.Handle, m)), m
