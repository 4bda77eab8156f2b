"""CPU: the layouts of alz_trend, alz_edge_trend and alz_trend_info (include/alazgpu.h, docs/SPEC.md §20) match the
Python mirror in alaz_b200/abi.py, the record's head is laid out as alz_edge_ends, the constants agree, and the trend
entry points are declared and bound."""
import ctypes as C
import os
import re

from alaz_b200 import abi, capi
from test_abi_changes import _run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TREND_FIELDS = [n for n, _ in abi.Trend._fields_]
REC_FIELDS = list(abi.EDGE_TREND.names)
INFO_FIELDS = [n for n, _ in abi.TrendInfo._fields_]
HEAD = ["from_type", "to_type", "from", "to"]
SYMBOLS = ["alz_edge_trends", "alz_edge_trends_device", "alz_edge_trends_top", "alz_edge_trends_top_device"]
CONSTANTS = {"ALZ_TREND_SLOPE": abi.TREND_SLOPE, "ALZ_TREND_SHIFT": abi.TREND_SHIFT,
             "ALZ_TREND_RATIO": abi.TREND_RATIO, "ALZ_TREND_ZSCORE": abi.TREND_ZSCORE,
             "ALZ_TREND_RISING": abi.TREND_RISING, "ALZ_TREND_FALLING": abi.TREND_FALLING,
             "ALZ_TREND_ABSENT_SKIP": abi.TREND_ABSENT_SKIP, "ALZ_TREND_ABSENT_ZERO": abi.TREND_ABSENT_ZERO}


def _layout(struct, fields):
    offs = " ".join(f'printf("%zu ", offsetof({struct}, {f}));' for f in fields)
    return _run(f"""
    #include <stdio.h>
    #include <stddef.h>
    #include "alazgpu.h"
    int main(void){{ printf("%zu ", sizeof({struct})); {offs} return 0; }}
    """)


def test_trend_spec_layout():
    got = _layout("alz_trend", TREND_FIELDS)
    assert got[0] == C.sizeof(abi.Trend) == 24
    assert got[1:] == [getattr(abi.Trend, f).offset for f in TREND_FIELDS] == [0, 4, 8, 12, 16, 20]


def test_edge_trend_layout_and_its_head():
    got = _layout("alz_edge_trend", REC_FIELDS)
    assert got[0] == abi.EDGE_TREND.itemsize == 48
    assert got[1:] == [abi.EDGE_TREND.fields[f][1] for f in REC_FIELDS] == [0, 1, 2, 3, 8, 12, 16, 20, 24, 32, 40]
    head = _layout("alz_edge_ends", HEAD)[1:]
    assert [abi.EDGE_TREND.fields[f][1] for f in HEAD] == head == [abi.EDGE_CHANGE.fields[f][1] for f in HEAD]


def test_trend_info_layout():
    got = _layout("alz_trend_info", INFO_FIELDS)
    assert got[0] == C.sizeof(abi.TrendInfo) == 40
    assert got[1:] == [getattr(abi.TrendInfo, f).offset for f in INFO_FIELDS] == [0, 8, 16, 24, 32, 36]


def test_trend_constants():
    body = " ".join(f'printf("%u ", (unsigned){c});' for c in CONSTANTS)
    got = _run(f"""
    #include <stdio.h>
    #include "alazgpu.h"
    int main(void){{ {body} return 0; }}
    """)
    assert got == list(CONSTANTS.values()) == [0, 1, 2, 3, 0, 1, 0, 1]


def test_trend_symbols_are_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "alazgpu.h")).read()
    for s in SYMBOLS:
        assert re.search(r"\bint " + s + r"\(", header), s
        assert s in capi.EXPORTS, s
