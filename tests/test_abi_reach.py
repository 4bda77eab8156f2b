"""CPU: the reach entry points (docs/SPEC.md §27) are declared in include/alazgpu.h (the hook in alazgpu_synth.h),
exported by the library and bound; alz_reach_node and alz_reach_info match their numpy and ctypes layouts, and the
constants match the header."""
import ctypes as C
import os
import re
import subprocess

from alaz_b200 import abi, build, capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PUBLIC = ["alz_reach", "alz_reach_device", "alz_group_reach", "alz_group_reach_device"]
HOOK = "alz_debug_reach_rows"


def header(name):
    return open(os.path.join(ROOT, "include", name)).read()


def test_reach_symbols_are_declared_exported_and_bound():
    pub, synth = header("alazgpu.h"), header("alazgpu_synth.h")
    for s in PUBLIC:
        assert re.search(r"\bint " + s + r"\(", pub), s
        assert s in capi.EXPORTS, s
    assert re.search(r"\bint " + HOOK + r"\(", synth) and HOOK not in capi.EXPORTS
    if os.path.exists(build.LIB):
        syms = subprocess.check_output(["nm", "-D", "--defined-only", build.LIB], text=True)
        for s in PUBLIC + [HOOK]:
            assert re.search(r"\bT " + s + r"$", syms, re.M), s
    src = open(os.path.join(ROOT, "alaz_b200", "capi.py")).read()
    for s in PUBLIC + [HOOK]:
        assert f'"{s}": (' in src, s
        assert callable(getattr(capi.Handle, s[len("alz_"):])), s
    assert "alz_reach.cu" in build.SOURCES


def test_record_and_info_layouts():
    assert abi.REACH_NODE.itemsize == 24
    assert [(f, abi.REACH_NODE.fields[f][1]) for f in ("type", "value", "hops", "index", "parent", "row")] == \
        [("type", 0), ("value", 4), ("hops", 8), ("index", 12), ("parent", 16), ("row", 20)]
    assert abi.REACH_NODE.fields["value"][1] == abi.NODE_ENDS.fields["value"][1]
    assert C.sizeof(abi.ReachInfo) == 48
    assert [n for n, _ in abi.ReachInfo._fields_] == ["rows", "traversable", "seeds_found", "nodes", "levels", "cut"]
    assert [getattr(abi.ReachInfo, n).offset for n, _ in abi.ReachInfo._fields_] == [0, 8, 16, 24, 32, 40]
    pub = header("alazgpu.h")
    body = re.search(r"typedef struct alz_reach_node \{(.*?)\} alz_reach_node;", pub, re.S).group(1)
    assert re.findall(r"(uint\d+_t) (\w+)", body) == [("uint8_t", "type"), ("uint8_t", "_pad"), ("uint32_t", "value"),
                                                      ("uint32_t", "hops"), ("uint32_t", "index"),
                                                      ("uint32_t", "parent"), ("uint32_t", "row")]
    body = re.search(r"typedef struct alz_reach_info \{(.*?)\} alz_reach_info;", pub, re.S).group(1)
    assert [n for _, n in re.findall(r"(uint64_t) (\w+);", body)] == [n for n, _ in abi.ReachInfo._fields_]


def test_constants():
    pub = header("alazgpu.h")
    for name, v in (("ALZ_REACH_DOWN", abi.REACH_DOWN), ("ALZ_REACH_UP", abi.REACH_UP),
                    ("ALZ_REACH_ANY", abi.REACH_ANY), ("ALZ_REACH_MAX_HOPS", abi.REACH_MAX_HOPS)):
        assert int(re.search(r"#define " + name + r"\s+(\d+)u", pub).group(1)) == v, name
    assert (abi.REACH_DOWN, abi.REACH_UP, abi.REACH_ANY, abi.REACH_MAX_HOPS) == (0, 1, 2, 64)
    assert abi.REACH_NONE == 0xFFFFFFFF
