"""Groups on several ranks in ONE process on ONE GPU, over the loopback collective (tests/loopback_nccl.cu): the child
process of tests/test_gpu_groups_ranks.py (`python loopback_groups_ranks.py SPEC.json IN.npz OUT.npz`).
Like tests/loopback_ranks.py it must never import torch, whose libnccl.so.2 would take the place of the loopback
library that LD_LIBRARY_PATH names. One thread per rank builds a handle on device 0, joins the communicator,
sets the same group map, configures the window history and runs the windows: submit, flush, a rollup of the last
`rollup` windows, then the group edges, their metrics and top rows, and the group nodes with both sides' metrics and
top nodes, of the window and of the rollup.

SPEC.json: {"nranks": R, "cfg": {Handle keywords}, "history": [depth, arena_rows], "windows": J, "rollup": k,
            "top": N}
IN.npz: tab0 = (table, ip, id) rows; map_nodes, map_groups = the group map; w{j}_r{r} = the L7 records rank r submits
in window j.
OUT.npz: win_{j}_{r} (the flushed rows), roll_{j}_{r} (the rollup's rows), and for source s (0: window, 1: rollup):
edges{s}_{j}_{r}, einfo{s}_{j}_{r}, emet{s}_{j}_{r}, etop{s}_{j}_{r}, eidx{s}_{j}_{r}, nodes{s}_{j}_{r},
val{s}{side}_{j}_{r}, top{s}{side}_{j}_{r}, tval{s}{side}_{j}_{r}, tidx{s}{side}_{j}_{r}; meta = {"errors", "maps"}.
"""
import ctypes as C
import json
import sys
import threading

import numpy as np

import loopback_ranks as lr
from alaz_b200 import abi

SPECS = [(abi.METRIC_QUANTILE, 0.99), abi.METRIC_COUNT, abi.METRIC_ERR_RATE]   # SPECS[side] ranks the top nodes,
                                                                                 # SPECS[0] the top group edges


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
            h.group_set(inp["map_nodes"], inp["map_groups"])
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
                    edges, info = h.group_edges(src)
                    res[f"edges{s}_{j}_{r}"] = edges
                    res[f"einfo{s}_{j}_{r}"] = np.array([info[k] for k in sorted(info)], np.uint64)
                    res[f"emet{s}_{j}_{r}"] = h.group_edge_metrics(src, *SPECS)
                    res[f"etop{s}_{j}_{r}"], _, res[f"eidx{s}_{j}_{r}"], _ = h.group_edge_top(src, SPECS[0],
                                                                                             spec["top"], -np.inf)
                    res[f"nodes{s}_{j}_{r}"] = h.group_nodes(src)
                    for side in (abi.SIDE_IN, abi.SIDE_OUT):
                        res[f"val{s}{side}_{j}_{r}"] = h.group_node_metrics(src, side, *SPECS)
                        nodes, vals, idx, _ = h.group_node_top(src, side, SPECS[side], spec["top"], -np.inf)
                        res[f"top{s}{side}_{j}_{r}"], res[f"tval{s}{side}_{j}_{r}"] = nodes, vals
                        res[f"tidx{s}{side}_{j}_{r}"] = idx
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
