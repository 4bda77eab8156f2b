"""CPU: the layouts of alz_corr, alz_corr_target, alz_edge_corr, alz_node_corr and alz_corr_info (include/alazgpu.h,
docs/SPEC.md §29) match the Python mirror in alaz_b200/abi.py, the records' heads are laid out as the trend records',
the constants agree, and the correlation entry points are declared and bound."""
import ctypes as C
import os
import re

from alaz_b200 import abi, capi
from test_abi_changes import _run
from test_abi_trends import _layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEVELS = ("edge", "node", "group_edge", "group_node")
SYMBOLS = [f"alz_{lv}_correlations{s}" for lv in LEVELS for s in ("", "_device", "_top", "_top_device")]
CONSTANTS = {"ALZ_CORR_POSITIVE": abi.CORR_POSITIVE, "ALZ_CORR_NEGATIVE": abi.CORR_NEGATIVE,
             "ALZ_CORR_ABS": abi.CORR_ABS, "ALZ_CORR_ABSENT_SKIP": abi.CORR_ABSENT_SKIP,
             "ALZ_CORR_ABSENT_ZERO": abi.CORR_ABSENT_ZERO, "ALZ_CORR_MAX_LAG": abi.CORR_MAX_LAG}


def test_corr_spec_and_target_layout():
    f = [n for n, _ in abi.Corr._fields_]
    got = _layout("alz_corr", f)
    assert got[0] == C.sizeof(abi.Corr) == 16 and got[1:] == [getattr(abi.Corr, n).offset for n in f] == [0, 4, 8, 12]
    f = [n for n, _ in abi.CorrTarget._fields_]
    got = _layout("alz_corr_target", f)
    assert got[0] == C.sizeof(abi.CorrTarget) == 32
    assert got[1:] == [getattr(abi.CorrTarget, n).offset for n in f] == [0, 8, 16, 24]


def test_records_and_their_heads():
    for struct, dt, trend in (("alz_edge_corr", abi.EDGE_CORR, abi.EDGE_TREND),
                              ("alz_node_corr", abi.NODE_CORR, abi.NODE_TREND)):
        names = list(dt.names)
        got = _layout(struct, names)
        assert got[0] == dt.itemsize == 48
        assert got[1:] == [dt.fields[n][1] for n in names]
        for n in ("valid", "index", "used"):
            assert dt.fields[n][1] == trend.fields[n][1], (struct, n)
        assert dt.fields["lag"][1] == 3 and dt.fields["r"][1] == 24 and dt.fields["r0"][1] == 40
    for n in ("from_type", "to_type", "from", "to"):
        assert abi.EDGE_CORR.fields[n][1] == abi.EDGE_TREND.fields[n][1]
    assert abi.NODE_CORR.fields["value"][1] == abi.NODE_TREND.fields["value"][1]


def test_corr_info_layout():
    f = [n for n, _ in abi.CorrInfo._fields_]
    got = _layout("alz_corr_info", f)
    assert got[0] == C.sizeof(abi.CorrInfo) == 48
    assert got[1:] == [getattr(abi.CorrInfo, n).offset for n in f] == [0, 8, 16, 24, 32, 36, 40, 44]


def test_corr_constants():
    body = " ".join(f'printf("%u ", (unsigned){c});' for c in CONSTANTS)
    got = _run(f"""
    #include <stdio.h>
    #include "alazgpu.h"
    int main(void){{ {body} return 0; }}
    """)
    assert got == list(CONSTANTS.values()) == [0, 1, 2, 0, 1, 32]


def test_corr_symbols_are_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "alazgpu.h")).read()
    for s in SYMBOLS:
        assert re.search(r"\bint " + s + r"\(", header), s
        assert s in capi.EXPORTS, s
    synth = open(os.path.join(ROOT, "include", "alazgpu_synth.h")).read()
    assert re.search(r"\bint alz_debug_corr_series\(", synth)
