"""CPU: the layouts of alz_edge_ends and alz_series_info (include/alazgpu.h, docs/SPEC.md §19) match the Python mirror
in alaz_b200/abi.py, and the series entry points are declared and bound."""
import ctypes as C
import os
import re

from alaz_b200 import abi, capi
from test_abi_changes import _run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENDS_FIELDS = ["from_type", "to_type", "_pad", "from", "to"]
INFO_FIELDS = [n for n, _ in abi.SeriesInfo._fields_]
SYMBOLS = ["alz_edge_series", "alz_edge_series_device", "alz_edge_series_keys", "alz_edge_series_keys_device"]


def test_edge_ends_layout_is_the_head_of_edge_out():
    offs = " ".join(f'printf("%zu ", offsetof(alz_edge_ends, {f}));' for f in ENDS_FIELDS)
    heads = " ".join(f'printf("%zu ", offsetof(alz_edge_out, {f}));' for f in ENDS_FIELDS)
    got = _run(f"""
    #include <stdio.h>
    #include <stddef.h>
    #include "alazgpu.h"
    int main(void){{ printf("%zu ", sizeof(alz_edge_ends)); {offs} {heads} return 0; }}
    """)
    assert got[0] == 16 == abi.EDGE_ENDS.itemsize == C.sizeof(abi.EdgeEnds)
    assert got[1:6] == [abi.EDGE_ENDS.fields[f][1] for f in ENDS_FIELDS] == [0, 1, 2, 8, 12]
    assert got[6:] == got[1:6]
    assert [abi.EDGE_OUT.fields[f][1] for f in ENDS_FIELDS] == got[1:6]
    assert abi.EdgeEnds.from_.offset == 8 and abi.EdgeEnds.to.offset == 12


def test_series_info_layout():
    offs = " ".join(f'printf("%zu ", offsetof(alz_series_info, {f}));' for f in INFO_FIELDS)
    got = _run(f"""
    #include <stdio.h>
    #include <stddef.h>
    #include "alazgpu.h"
    int main(void){{ printf("%zu ", sizeof(alz_series_info)); {offs} return 0; }}
    """)
    assert got[0] == C.sizeof(abi.SeriesInfo) == 24
    assert got[1:] == [getattr(abi.SeriesInfo, f).offset for f in INFO_FIELDS] == [0, 8, 16, 20]


def test_series_symbols_are_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "alazgpu.h")).read()
    for s in SYMBOLS:
        assert re.search(r"\bint " + s + r"\(", header), s
        assert s in capi.EXPORTS, s
