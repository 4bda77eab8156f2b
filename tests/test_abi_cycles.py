"""CPU: the cycles entry points (docs/SPEC.md §28) are declared in include/alazgpu.h (the hook in alazgpu_synth.h),
exported by the library and bound; alz_cycle_node and alz_cycle_info match their numpy and ctypes layouts."""
import ctypes as C
import os
import re
import subprocess

from alaz_b200 import abi, build, capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PUBLIC = ["alz_cycles", "alz_cycles_device", "alz_group_cycles", "alz_group_cycles_device"]
HOOK = "alz_debug_cycles_rows"
INFO = ["rows", "traversable", "self_rows", "nodes", "components", "cyclic", "cyclic_nodes", "largest", "cycle_rows",
        "depth"]


def header(name):
    return open(os.path.join(ROOT, "include", name)).read()


def test_cycles_symbols_are_declared_exported_and_bound():
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
    assert "alz_cycles.cu" in build.SOURCES


def test_record_and_info_layouts():
    assert abi.CYCLE_NODE.itemsize == 28
    assert [(f, abi.CYCLE_NODE.fields[f][1]) for f in ("type", "value", "index", "component", "size", "depth",
                                                        "height")] == \
        [("type", 0), ("value", 4), ("index", 8), ("component", 12), ("size", 16), ("depth", 20), ("height", 24)]
    assert abi.CYCLE_NODE.fields["value"][1] == abi.NODE_ENDS.fields["value"][1]
    assert C.sizeof(abi.CycleInfo) == 80
    assert [n for n, _ in abi.CycleInfo._fields_] == INFO
    assert [getattr(abi.CycleInfo, n).offset for n in INFO] == list(range(0, 80, 8))
    pub = header("alazgpu.h")
    body = re.search(r"typedef struct alz_cycle_node \{(.*?)\} alz_cycle_node;", pub, re.S).group(1)
    assert re.findall(r"(uint\d+_t) (\w+)", body) == [("uint8_t", "type"), ("uint8_t", "_pad"), ("uint32_t", "value"),
                                                      ("uint32_t", "index"), ("uint32_t", "component"),
                                                      ("uint32_t", "size"), ("uint32_t", "depth"),
                                                      ("uint32_t", "height")]
    body = re.search(r"typedef struct alz_cycle_info \{(.*?)\} alz_cycle_info;", pub, re.S).group(1)
    assert [n for _, n in re.findall(r"(uint64_t) (\w+);", body)] == INFO


def test_the_calls_take_the_same_arguments():
    pub, synth = header("alazgpu.h"), header("alazgpu_synth.h")

    def args(text, name):
        return re.sub(r"\s+", " ", re.search(r"\bint " + name + r"\((.*?)\);", text, re.S).group(1))

    assert args(pub, "alz_cycles") == args(pub, "alz_group_cycles")
    assert args(pub, "alz_cycles_device") == args(pub, "alz_group_cycles_device")
    assert args(synth, HOOK).replace("const alz_edge_out* dev_rows, size_t n", "uint32_t source") == \
        args(pub, "alz_cycles")
