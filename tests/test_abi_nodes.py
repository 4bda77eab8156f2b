"""CPU: the layouts of alz_node_sums and alz_node_out (include/alazgpu.h, docs/SPEC.md §21) match the Python mirror in
alaz_b200/abi.py, side IN's sums sit where alz_edge_out's do (so a node side reads in place as an edge row), the side
constants agree, and the node entry points are declared, exported by the library and bound."""
import os
import re
import subprocess

from alaz_b200 import abi, build, capi
from test_abi_changes import _run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SUMS_FIELDS = list(abi.NODE_SUMS.names)
NODE_FIELDS = list(abi.NODE_OUT.names)
SYMBOLS = ["alz_node_rows", "alz_node_rows_device", "alz_node_metrics", "alz_node_metrics_device", "alz_node_top",
           "alz_node_top_device"]


def _layout(struct, fields, header="alazgpu.h"):
    offs = " ".join(f'printf("%zu ", offsetof({struct}, {f}));' for f in fields)
    return _run(f"""
    #include <stdio.h>
    #include <stddef.h>
    #include "{header}"
    int main(void){{ printf("%zu ", sizeof({struct})); {offs} return 0; }}
    """)


def test_node_sums_layout():
    got = _layout("alz_node_sums", SUMS_FIELDS)
    assert got[0] == abi.NODE_SUMS.itemsize == 280
    assert got[1:] == [abi.NODE_SUMS.fields[f][1] for f in SUMS_FIELDS] == [0, 8, 16, 24]


def test_node_out_layout():
    got = _layout("alz_node_out", NODE_FIELDS)
    assert got[0] == abi.NODE_OUT.itemsize == 576
    assert got[1:] == [abi.NODE_OUT.fields[f][1] for f in NODE_FIELDS] == [0, 1, 4, 8, 12, 16, 296]


def test_each_side_is_laid_out_as_the_tail_of_an_edge_row():
    edge = _layout("alz_edge_out", ["count", "err5xx", "lat_sum_ns", "hist"])[1:]
    sums = [abi.NODE_SUMS.fields[f][1] for f in SUMS_FIELDS]
    inside = _layout("alz_node_out", ["in.count", "in.err5xx", "in.lat_sum_ns", "in.hist"])[1:]
    outside = _layout("alz_node_out", ["out.count", "out.err5xx", "out.lat_sum_ns", "out.hist"])[1:]
    assert inside == edge == [16, 24, 32, 40]                      # in.count at 16, as alz_edge_out.count
    assert outside == [x + 280 for x in edge]                       # side OUT reads as a row 280 bytes further on
    assert [x - 16 for x in edge] == sums
    assert abi.EDGE_OUT.itemsize - abi.EDGE_OUT.fields["count"][1] == abi.NODE_SUMS.itemsize


def test_side_constants():
    got = _run("""
    #include <stdio.h>
    #include "alazgpu.h"
    int main(void){ printf("%u %u ", (unsigned)ALZ_SIDE_IN, (unsigned)ALZ_SIDE_OUT); return 0; }
    """)
    assert got == [abi.SIDE_IN, abi.SIDE_OUT] == [0, 1]


def test_node_symbols_are_declared_exported_and_bound():
    header = open(os.path.join(ROOT, "include", "alazgpu.h")).read()
    synth = open(os.path.join(ROOT, "include", "alazgpu_synth.h")).read()
    for s in SYMBOLS:
        assert re.search(r"\bint " + s + r"\(", header), s
        assert s in capi.EXPORTS, s
    assert re.search(r"\bint alz_debug_node_rows\(", synth)
    if os.path.exists(build.LIB):
        syms = subprocess.check_output(["nm", "-D", "--defined-only", build.LIB], text=True)
        for s in SYMBOLS + ["alz_debug_node_rows"]:
            assert re.search(r"\bT " + s + r"$", syms, re.M), s
    src = open(os.path.join(ROOT, "alaz_b200", "capi.py")).read()
    for s in SYMBOLS + ["alz_debug_node_rows"]:
        assert f'"{s}": (' in src, s
