"""Group changes against a pinned baseline on several ranks in ONE process on ONE GPU, over the loopback collective
(tests/loopback_nccl.cu): the child process of tests/test_gpu_group_changes_ranks.py (`python
loopback_group_changes_ranks.py SPEC.json IN.npz OUT.npz`). Like tests/loopback_ranks.py it must never import torch,
whose libnccl.so.2 would take the place of the loopback library that LD_LIBRARY_PATH names. One thread per rank builds
a handle on device 0, joins the communicator, sets the group map of IN.npz, configures the window history and the
tiers and runs the windows: submit, flush; after window `pin_after` it pins the baseline the spec names, and after
every later window it takes alz_group_edge_changes, alz_group_node_changes and their top calls of the window and of
every rollup of the spec.

SPEC.json: as tests/loopback_changes_ranks.py's. IN.npz: as there, and map_types / map_values / map_groups (the group map).
OUT.npz: base_{r} (the pinned rows), basew_{r} (their windows), rows_{j}_{r}_{s}, win_{j}_{r}_{s} (the source's rows
and windows), list{c}_{j}_{r}_{s}, top{c}_{j}_{r}_{s} and their info{c}_{j}_{r}_{s} / tinfo{c}_{j}_{r}_{s} for each
case c of CASES (side None: the group edges); s = 0 is the window, s >= 1 rollup s - 1; meta = {"errors", "maps"}.
"""
import ctypes as C
import json
import sys
import threading

import numpy as np

import loopback_ranks as lr
from alaz_b200 import abi
from loopback_changes_ranks import INFO, run_rollup

Q = abi.METRIC_QUANTILE
# (side, metric, mode, presence); side None: the group edge changes
CASES = ((None, (Q, 0.99), abi.CHANGE_DELTA, 7), (None, abi.METRIC_ERR5XX, abi.CHANGE_RATIO, 3),
         (abi.SIDE_IN, (Q, 0.99), abi.CHANGE_DELTA, 7), (abi.SIDE_OUT, abi.METRIC_COUNT, abi.CHANGE_DROP, 5),
         (abi.SIDE_IN, abi.METRIC_ERR_RATE, abi.CHANGE_RATIO, 6))


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
            h.window_history_tiers(spec["tiers"])
            res = {}
            k, mc = int(spec["k"]), float(spec["min_change"])
            for j in range(int(spec["windows"])):
                recs = inp[f"w{j}_r{r}"]
                if len(recs):
                    h.submit(recs)
                h.sync()
                bar.wait()
                win = h.flush()
                if j == int(spec["pin_after"]):
                    if spec["pin"][0] == "window":
                        res[f"base_{r}"], source = win, abi.SOURCE_WINDOW
                    else:
                        res[f"base_{r}"], _, source = run_rollup(h, spec["pin"])
                    res[f"basew_{r}"] = np.array([h.baseline_pin(source)["windows"]], np.uint64)
                elif j > int(spec["pin_after"]):
                    # one rollup per kind, so each stays the last of its kind while it is compared
                    sources = [(win, 1, abi.SOURCE_WINDOW)] + [run_rollup(h, roll) for roll in spec["rollups"]]
                    for s, (rows, w, source) in enumerate(sources):
                        res[f"rows_{j}_{r}_{s}"], res[f"win_{j}_{r}_{s}"] = rows, np.array([w], np.uint64)
                        for c, (side, metric, mode, presence) in enumerate(CASES):
                            if side is None:
                                lst, info = h.group_edge_changes(metric, mode, presence, source)
                                top, tinfo = h.group_edge_changes_top(metric, k, mc, mode, presence, source)
                            else:
                                lst, info = h.group_node_changes(side, metric, mode, presence, source)
                                top, tinfo = h.group_node_changes_top(side, metric, k, mc, mode, presence, source)
                            res[f"list{c}_{j}_{r}_{s}"], res[f"top{c}_{j}_{r}_{s}"] = lst, top
                            res[f"info{c}_{j}_{r}_{s}"] = np.array([info[x] for x in INFO], np.uint64)
                            res[f"tinfo{c}_{j}_{r}_{s}"] = np.array([tinfo[x] for x in INFO], np.uint64)
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
