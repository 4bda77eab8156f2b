"""Top anomalous rows on several ranks in ONE process on ONE GPU, over the loopback collective
(tests/loopback_nccl.cu): the child process of tests/test_gpu_gnn_top_ranks.py (`python loopback_gnn_top_ranks.py
SPEC.json IN.npz OUT.npz`). Like tests/loopback_ranks.py it must never import torch, whose libnccl.so.2 would take the
place of the loopback library that LD_LIBRARY_PATH names. One thread per rank builds a handle on device 0, joins the
communicator, configures the window history and the tiers and runs the windows: submit, flush, alz_gnn_top over the
window, then for every rollup of the spec the rollup, alz_gnn_top_rollup of its kind and alz_gnn_score_rollup.

SPEC.json: {"nranks": R, "cfg": {Handle keywords}, "history": [depth, arena_rows],
            "tiers": [[factor, depth, arena_rows, block_rows], ...], "windows": J,
            "rollups": [["window", k] | ["tier", tier, k] | ["span", N, mode], ...], "k": k, "min_score": m}
IN.npz: tab0 = (table, ip, id) rows; w{j}_r{r} = the L7 records rank r submits in window j.
OUT.npz: rows_{j}_{r}_{s} (the source's rows), scores_{j}_{r}_{s} (its scores), top_{j}_{r}_{s}_{rows|scores|index}
and info_{j}_{r}_{s}; s = 0 is the window, s >= 1 rollup s - 1; meta = {"errors", "maps"}.
"""
import ctypes as C
import json
import sys
import threading

import numpy as np

import loopback_ranks as lr
from alaz_b200 import abi


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
                k, ms = int(spec["k"]), float(spec["min_score"])
                res[f"rows_{j}_{r}_0"] = win
                top = h.gnn_top(k, ms)
                sc = np.zeros(max(len(win), 1), np.float32)
                n = C.c_size_t(0)
                h._ck(L.alz_gnn_score(h.h, sc.ctypes.data_as(C.c_void_p), len(sc), C.byref(n)), "alz_gnn_score")
                res[f"scores_{j}_{r}_0"] = sc[: n.value]
                for part, x in zip(("rows", "scores", "index"), top[:3]):
                    res[f"top_{j}_{r}_0_{part}"] = x
                res[f"info_{j}_{r}_0"] = np.array([top[3]["scored"], top[3]["above"]], np.uint64)
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
                    top = h.gnn_top_rollup(kind, k, ms)
                    res[f"rows_{j}_{r}_{s}"] = rows
                    res[f"scores_{j}_{r}_{s}"] = h.gnn_score_rollup(kind)
                    for part, x in zip(("rows", "scores", "index"), top[:3]):
                        res[f"top_{j}_{r}_{s}_{part}"] = x
                    res[f"info_{j}_{r}_{s}"] = np.array([top[3]["scored"], top[3]["above"]], np.uint64)
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
