"""CPU: the layouts of alz_edge_change and alz_change_info (include/alazgpu.h, docs/SPEC.md §18) match the Python
mirror in alaz_b200/abi.py, and the constants agree."""
import ctypes as C
import os
import subprocess
import tempfile

from alaz_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHANGE_FIELDS = ["from_type", "to_type", "presence", "_pad", "from", "to", "index", "base_index", "value",
                 "base_value", "change"]
INFO_FIELDS = [n for n, _ in abi.ChangeInfo._fields_]


def _run(prog):
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(prog)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        return [int(x) for x in subprocess.check_output([exe], text=True).split()]


def test_edge_change_layout():
    offs = " ".join(f'printf("%zu ", offsetof(alz_edge_change, {f}));' for f in CHANGE_FIELDS)
    got = _run(f"""
    #include <stdio.h>
    #include <stddef.h>
    #include "alazgpu.h"
    int main(void){{ printf("%zu ", sizeof(alz_edge_change)); {offs} return 0; }}
    """)
    assert got[0] == 48 == abi.EDGE_CHANGE.itemsize
    assert got[1:] == [abi.EDGE_CHANGE.fields[f][1] for f in CHANGE_FIELDS]
    assert got[1:] == [0, 1, 2, 3, 8, 12, 16, 20, 24, 32, 40]


def test_change_info_layout():
    offs = " ".join(f'printf("%zu ", offsetof(alz_change_info, {f}));' for f in INFO_FIELDS)
    got = _run(f"""
    #include <stdio.h>
    #include <stddef.h>
    #include "alazgpu.h"
    int main(void){{ printf("%zu ", sizeof(alz_change_info)); {offs} return 0; }}
    """)
    assert got[0] == C.sizeof(abi.ChangeInfo) == 64
    assert got[1:] == [getattr(abi.ChangeInfo, f).offset for f in INFO_FIELDS]


def test_constants():
    names = ["ALZ_SOURCE_WINDOW", "ALZ_CHANGE_DELTA", "ALZ_CHANGE_DROP", "ALZ_CHANGE_RATIO", "ALZ_PRESENT_BOTH",
             "ALZ_PRESENT_NEW", "ALZ_PRESENT_GONE", "ALZ_ABI_VERSION"]
    got = _run("""
    #include <stdio.h>
    #include "alazgpu.h"
    int main(void){ printf("%u %u %u %u %u %u %u %u", ALZ_SOURCE_WINDOW, ALZ_CHANGE_DELTA, ALZ_CHANGE_DROP,
                           ALZ_CHANGE_RATIO, ALZ_PRESENT_BOTH, ALZ_PRESENT_NEW, ALZ_PRESENT_GONE,
                           (unsigned)ALZ_ABI_VERSION); return 0; }
    """)
    assert dict(zip(names, got)) == dict(
        ALZ_SOURCE_WINDOW=abi.SOURCE_WINDOW, ALZ_CHANGE_DELTA=abi.CHANGE_DELTA, ALZ_CHANGE_DROP=abi.CHANGE_DROP,
        ALZ_CHANGE_RATIO=abi.CHANGE_RATIO, ALZ_PRESENT_BOTH=abi.PRESENT_BOTH, ALZ_PRESENT_NEW=abi.PRESENT_NEW,
        ALZ_PRESENT_GONE=abi.PRESENT_GONE, ALZ_ABI_VERSION=2)
