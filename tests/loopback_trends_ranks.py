"""Edge trends on several ranks in ONE process on ONE GPU, over the loopback collective (tests/loopback_nccl.cu): the
child process of tests/test_gpu_edge_trends_ranks.py (`python loopback_trends_ranks.py SPEC.json IN.npz OUT.npz`).
Like tests/loopback_ranks.py it must never import torch, whose libnccl.so.2 would take the place of the loopback
library that LD_LIBRARY_PATH names. One thread per rank builds a handle on device 0, joins the communicator,
configures the window history and the tiers and runs the windows: submit, flush, then alz_edge_trends and
alz_edge_trends_top of the window on every ring and every trend of the spec.

SPEC.json: {"nranks": R, "cfg": {Handle keywords}, "history": [depth, arena_rows],
            "tiers": [[factor, depth, arena_rows, block_rows], ...], "windows": J, "rings": [[tier, k], ...],
            "trends": [[stat, direction, absent, recent, min_points], ...], "top": N}
IN.npz: tab0 = (table, ip, id) rows; w{j}_r{r} = the L7 records rank r submits in window j.
OUT.npz: win_{j}_{r} (the flushed rows), and for ring c and trend t: rec{c}_{t}_{j}_{r}, pts{c}_{t}_{j}_{r} (the
records, points as RollupInfo dicts in JSON), top{c}_{t}_{j}_{r}, trow{c}_{t}_{j}_{r}, tser{c}_{t}_{j}_{r},
tpre{c}_{t}_{j}_{r} (the top call's records, rows, series and presence); meta = {"errors", "maps"}.
"""
import ctypes as C
import json
import sys
import threading

import numpy as np

import loopback_ranks as lr
from alaz_b200 import abi

SPEC = (abi.METRIC_QUANTILE, 0.99)


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
            h.window_history(*spec["history"])
            h.window_history_tiers(spec["tiers"])
            res = {}
            for j in range(int(spec["windows"])):
                recs = inp[f"w{j}_r{r}"]
                if len(recs):
                    h.submit(recs)
                h.sync()
                bar.wait()
                win = h.flush()
                res[f"win_{j}_{r}"] = win
                for c, (tier, k) in enumerate(spec["rings"]):
                    for t, ts in enumerate(spec["trends"]):
                        tt = capi.Handle.trend(*ts)
                        rec, pts, _ = h.edge_trends(abi.SOURCE_WINDOW, tier, k, SPEC, tt)
                        res[f"rec{c}_{t}_{j}_{r}"], res[f"pts{c}_{t}_{j}_{r}"] = rec, np.array(json.dumps(pts))
                        tr_, rows, ser, pre, _, _ = h.edge_trends_top(abi.SOURCE_WINDOW, tier, k, SPEC, tt, spec["top"])
                        res[f"top{c}_{t}_{j}_{r}"], res[f"trow{c}_{t}_{j}_{r}"] = tr_, rows
                        res[f"tser{c}_{t}_{j}_{r}"], res[f"tpre{c}_{t}_{j}_{r}"] = ser, pre
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
