"""CPU: the group series and group trend entry points (docs/SPEC.md §26) are declared in include/alazgpu.h, exported by
the library and bound. They reuse alz_edge_ends, alz_node_ends, alz_edge_trend, alz_node_trend, alz_series_info,
alz_trend_info and alz_rollup_info, whose layouts the edge and node series ABI tests check."""
import os
import re
import subprocess

from alaz_b200 import build, capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ["alz_group_edge_series", "alz_group_edge_series_device", "alz_group_edge_series_keys",
           "alz_group_edge_series_keys_device", "alz_group_node_series", "alz_group_node_series_device",
           "alz_group_node_series_keys", "alz_group_node_series_keys_device", "alz_group_edge_trends",
           "alz_group_edge_trends_device", "alz_group_edge_trends_top", "alz_group_edge_trends_top_device",
           "alz_group_node_trends", "alz_group_node_trends_device", "alz_group_node_trends_top",
           "alz_group_node_trends_top_device"]


def test_group_series_symbols_are_declared_exported_and_bound():
    assert len(SYMBOLS) == 16
    header = open(os.path.join(ROOT, "include", "alazgpu.h")).read()
    for s in SYMBOLS:
        assert re.search(r"\bint " + s + r"\(", header), s
        assert s in capi.EXPORTS, s
    if os.path.exists(build.LIB):
        syms = subprocess.check_output(["nm", "-D", "--defined-only", build.LIB], text=True)
        for s in SYMBOLS:
            assert re.search(r"\bT " + s + r"$", syms, re.M), s
    src = open(os.path.join(ROOT, "alaz_b200", "capi.py")).read()
    for s in SYMBOLS:
        assert f'"{s}": (' in src, s
    for s in SYMBOLS:
        assert callable(getattr(capi.Handle, s[len("alz_"):])), s
