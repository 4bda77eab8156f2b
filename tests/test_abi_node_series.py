"""CPU: the layouts of alz_node_ends and alz_node_trend (include/alazgpu.h, docs/SPEC.md §22) match the Python mirror
in alaz_b200/abi.py, alz_node_ends is the head of alz_node_out, alz_node_trend is laid out as alz_edge_trend from
`valid` on (the trend kernel writes both), and the node series and trend entry points are declared, exported by the
library and bound."""
import os
import re
import subprocess

from alaz_b200 import abi, build, capi
from test_abi_nodes import _layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ["alz_node_series", "alz_node_series_device", "alz_node_series_keys", "alz_node_series_keys_device",
           "alz_node_trends", "alz_node_trends_device", "alz_node_trends_top", "alz_node_trends_top_device"]
SHARED = ["valid", "index", "used", "trend", "recent", "before"]


def test_node_ends_layout_is_the_head_of_a_node_row():
    got = _layout("alz_node_ends", list(abi.NODE_ENDS.names))
    assert got[0] == abi.NODE_ENDS.itemsize == 8
    assert got[1:] == [abi.NODE_ENDS.fields[f][1] for f in abi.NODE_ENDS.names] == [0, 1, 4]
    assert _layout("alz_node_out", ["type", "value"])[1:] == got[1:2] + got[3:]


def test_node_trend_layout():
    got = _layout("alz_node_trend", list(abi.NODE_TREND.names))
    assert got[0] == abi.NODE_TREND.itemsize == 48
    assert got[1:] == [abi.NODE_TREND.fields[f][1] for f in abi.NODE_TREND.names] == \
        [0, 1, 2, 3, 8, 12, 16, 20, 24, 32, 40]


def test_node_trend_shares_the_edge_trend_layout_from_valid_on():
    node = _layout("alz_node_trend", SHARED + ["value"])
    edge = _layout("alz_edge_trend", SHARED + ["from"])
    assert node == edge
    assert [abi.NODE_TREND.fields[f][1] for f in SHARED] == [abi.EDGE_TREND.fields[f][1] for f in SHARED]


def test_node_series_symbols_are_declared_exported_and_bound():
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
