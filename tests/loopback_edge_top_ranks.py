"""Edge metrics and top edges on several ranks in ONE process on ONE GPU, over the loopback collective
(tests/loopback_nccl.cu): the child process of tests/test_gpu_edge_top_ranks.py (`python loopback_edge_top_ranks.py
SPEC.json IN.npz OUT.npz`). Like tests/loopback_ranks.py it must never import torch, whose libnccl.so.2 would take the
place of the loopback library that LD_LIBRARY_PATH names. One thread per rank builds a handle on device 0, joins the
communicator, configures the window history and the tiers and runs the windows: submit, flush, alz_edge_metrics and
alz_edge_top over the window, then for every rollup of the spec the rollup, alz_edge_metrics_rollup and
alz_edge_top_rollup of its kind.

SPEC.json: {"nranks": R, "cfg": {Handle keywords}, "history": [depth, arena_rows],
            "tiers": [[factor, depth, arena_rows, block_rows], ...], "windows": J,
            "rollups": [["window", k] | ["tier", tier, k] | ["span", N, mode], ...], "k": k, "min_value": m}
IN.npz: tab0 = (table, ip, id) rows; w{j}_r{r} = the L7 records rank r submits in window j.
OUT.npz: rows_{j}_{r}_{s} (the source's rows), values_{j}_{r}_{s} (its metrics), top{t}_{j}_{r}_{s}_{rows|values|index}
and info{t}_{j}_{r}_{s} for each top metric t; s = 0 is the window, s >= 1 rollup s - 1; meta = {"errors", "maps"}.
"""
import ctypes as C
import json
import sys
import threading

import numpy as np

import loopback_ranks as lr
from alaz_b200 import abi

Q = abi.METRIC_QUANTILE
METRICS = (abi.METRIC_COUNT, abi.METRIC_ERR5XX, abi.METRIC_ERR_RATE, abi.METRIC_MEAN_NS, (Q, 0.5), (Q, 0.99))
TOPS = ((Q, 0.99), abi.METRIC_ERR5XX, abi.METRIC_MEAN_NS)


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
                k, ms = int(spec["k"]), float(spec["min_value"])

                def record(s, rows, metrics, top):
                    res[f"rows_{j}_{r}_{s}"] = rows
                    res[f"values_{j}_{r}_{s}"] = metrics(*METRICS)
                    for t, spec_t in enumerate(TOPS):
                        got = top(spec_t, k, ms)
                        for part, x in zip(("rows", "values", "index"), got[:3]):
                            res[f"top{t}_{j}_{r}_{s}_{part}"] = x
                        res[f"info{t}_{j}_{r}_{s}"] = np.array([got[3]["scored"], got[3]["above"]], np.uint64)
                record(0, win, h.edge_metrics, h.edge_top)
                for s, roll in enumerate(spec["rollups"], start=1):
                    if roll[0] == "window":
                        rows, _ = h.rollup(roll[1])
                        kind = abi.ROLLUP_WINDOWS
                    elif roll[0] == "tier":
                        rows, _ = h.rollup_tier(roll[1], roll[2])
                        kind = abi.ROLLUP_TIER
                    else:
                        rows, _ = h.rollup_span(roll[1], roll[2])
                        kind = abi.ROLLUP_SPAN
                    record(s, rows, lambda *m, kind=kind: h.edge_metrics_rollup(kind, *m),
                           lambda *a, kind=kind: h.edge_top_rollup(kind, *a))
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
