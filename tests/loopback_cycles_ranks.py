"""Cycles on several ranks in ONE process on ONE GPU, over the loopback collective (tests/loopback_nccl.cu): the child
process of tests/test_gpu_cycles_ranks.py (`python loopback_cycles_ranks.py SPEC.json IN.npz OUT.npz`). Like
tests/loopback_ranks.py it must never import torch, whose libnccl.so.2 would take the place of the loopback library
that LD_LIBRARY_PATH names. One thread per rank builds a handle on device 0, joins the communicator, sets the group
map of IN.npz, configures the window history and runs the windows: submit, flush, a rollup of the last `rollup`
windows, then the node and group cycles of the window and of the rollup under every filter of FILTERS.

SPEC.json: {"nranks": R, "cfg": {Handle keywords}, "history": [depth, arena_rows], "windows": J, "rollup": k}
IN.npz: tab0 = (table, ip, id) rows; w{j}_r{r} = the L7 records rank r submits in window j; map_types / map_values /
map_groups (the group map).
OUT.npz: win_{j}_{r} (the flushed rows), roll_{j}_{r} (the rollup's rows), and for form f (n: node, g: group), source
s (0: window, 1: rollup) and filter case c (an index into FILTERS): {f}rec{s}{c}_{j}_{r}, {f}idx{s}{c}_{j}_{r},
{f}rows{s}{c}_{j}_{r} and {f}info{s}{c}_{j}_{r} (the info's ten counts); meta = {"errors", "maps"}.
"""
import ctypes as C
import json
import sys
import threading

import numpy as np

import loopback_ranks as lr
from alaz_b200 import abi

# (metric, min_value, min_size)
FILTERS = ((None, 0.0, 1), (abi.METRIC_ERR5XX, 1.0, 2), (abi.METRIC_COUNT, 2.0, 2))
INFO = ("rows", "traversable", "self_rows", "nodes", "components", "cyclic", "cyclic_nodes", "largest", "cycle_rows",
        "depth")


def main(spec_path, in_path, out_path):
    from alaz_b200 import capi
    spec = json.load(open(spec_path))
    with np.load(in_path) as z:     # read every array now: the rank threads must not share the zip file
        inp = {k: z[k] for k in z.files}
    L = capi.load()
    R = int(spec["nranks"])
    out, meta = {}, {"errors": []}
    shim = C.CDLL("libnccl.so.2")      # the library LD_LIBRARY_PATH names (the one the product's dlopen gets)
    shim.loopback_fault_block_status.argtypes = [C.c_int, C.c_long, C.c_int]
    shim.loopback_fault_block_status(-1, 0, 0)
    shim.loopback_log_clear()
    idbuf = (C.c_uint8 * abi.COMM_ID_BYTES)()
    assert L.alz_comm_unique_id(idbuf) == 0
    bar = threading.Barrier(R, timeout=300)
    lock = threading.Lock()

    def rank_main(r):
        try:
            h = capi.Handle(device=0, **spec["cfg"])
            rc = L.alz_comm_init(h.h, R, r, idbuf)
            if rc != 0:
                raise RuntimeError(f"alz_comm_init: {rc}")
            if r == 0:
                meta["maps"] = lr._libnccl_maps()
            tab = inp["tab0"]
            for t in (abi.TABLE_POD, abi.TABLE_SVC):
                m = tab[:, 0] == t
                if m.any():
                    h.upsert_batch(t, tab[m, 1].astype(np.uint32), tab[m, 2].astype(np.uint32))
            h.commit()
            h.group_set(h.node_ends(list(zip(inp["map_types"].tolist(), inp["map_values"].tolist()))),
                        inp["map_groups"])
            h.window_history(*spec["history"])
            res = {}
            for j in range(int(spec["windows"])):
                recs = inp[f"w{j}_r{r}"]
                if len(recs):
                    h.submit(recs)
                h.sync()
                bar.wait()
                res[f"win_{j}_{r}"] = h.flush()
                res[f"roll_{j}_{r}"] = h.rollup(int(spec["rollup"]))[0]
                for s, src in enumerate((abi.SOURCE_WINDOW, abi.ROLLUP_WINDOWS)):
                    for c, (m, mv, ms) in enumerate(FILTERS):
                        for f, call in (("n", h.cycles), ("g", h.group_cycles)):
                            rec, idx, rows, info = call(src, m, mv, ms)
                            res[f"{f}rec{s}{c}_{j}_{r}"], res[f"{f}idx{s}{c}_{j}_{r}"] = rec, idx
                            res[f"{f}rows{s}{c}_{j}_{r}"] = rows
                            res[f"{f}info{s}{c}_{j}_{r}"] = np.array([info[k] for k in INFO], np.uint64)
                bar.wait()
            with lock:
                out.update(res)
            bar.wait()
            h.close()
        except Exception as e:  # noqa: BLE001
            with lock:
                meta["errors"].append([r, repr(e)])
            bar.abort()

    th = [threading.Thread(target=rank_main, args=(r,)) for r in range(R)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    out["meta"] = np.array(json.dumps(meta))
    np.savez(out_path, **out)
    return 0


if __name__ == "__main__":
    sys.exit(main(*sys.argv[1:4]))
