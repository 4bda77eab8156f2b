"""Correlations on several ranks in ONE process on ONE GPU, over the loopback collective (tests/loopback_nccl.cu): the
child process of tests/test_gpu_correlations_ranks.py (`python loopback_corr_ranks.py SPEC.json IN.npz OUT.npz`).
Like tests/loopback_ranks.py it must never import torch, whose libnccl.so.2 would take the place of the loopback
library that LD_LIBRARY_PATH names. One thread per rank builds a handle on device 0, joins the communicator,
configures the window history, the tiers and a group map, and runs the windows: submit, flush, then for every ring,
target and correlation spec the full list and the top call of the edge, node (both sides), group-edge and group-node
correlations of the window.

SPEC.json: {"nranks": R, "cfg": {Handle keywords}, "history": [depth, arena_rows],
            "tiers": [[factor, depth, arena_rows, block_rows], ...], "windows": J, "rings": [[tier, k], ...],
            "corrs": [[direction, absent, max_lag, min_points], ...], "top": N, "groups": G}
IN.npz: tab0 = (table, ip, id) rows; w{j}_r{r} = the L7 records rank r submits in window j.
OUT.npz: win_{j}_{r} (the flushed rows); for ring c, target g (0: the first row's series, 1: a synthetic series), spec
s and call name q (LEVEL_SIDE): rec/top/trow/tser/tpre{c}_{g}_{s}_{q}_{j}_{r}, and tgt{c}_{g}_{j}_{r} (the target's
values, presence and window_last); meta = {"errors", "maps"}.
"""
import ctypes as C
import json
import sys
import threading

import numpy as np

import loopback_ranks as lr
from alaz_b200 import abi

SPEC = (abi.METRIC_QUANTILE, 0.99)
CALLS = [("edge", abi.SIDE_IN), ("node", abi.SIDE_IN), ("node", abi.SIDE_OUT), ("group_edge", abi.SIDE_IN),
         ("group_node", abi.SIDE_IN), ("group_node", abi.SIDE_OUT)]


def targets(h, win, tier, k, j, c):
    """the targets of ring (tier, k) after window j: the first row's series and a synthetic series, both aligned"""
    from alaz_b200 import capi
    v, p, pts, _ = h.edge_series_keys(win[:1], tier, k, SPEC)
    last = pts[-1]["window_last"] if pts else 0
    rng = np.random.default_rng(1000 * j + c)
    P = v.shape[1]
    return [capi.Handle.Target(v[0, :, 0], p[0], last),
            capi.Handle.Target(rng.normal(size=P) * 1e6, (rng.random(P) < 0.9).astype(np.uint8), last)]


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
            pods = np.unique(tab[tab[:, 0] == abi.TABLE_POD, 2]).astype(np.uint32)
            h.group_set([(abi.NODE_POD, int(v)) for v in pods], (pods % int(spec["groups"])).astype(np.uint32))
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
                    for g, tg in enumerate(targets(h, win, tier, k, j, c)):
                        res[f"tgt{c}_{g}_{j}_{r}"] = np.array(json.dumps(
                            [tg.values.tolist(), tg.present.tolist(), int(tg.s.window_last)]))
                        for s, cs in enumerate(spec["corrs"]):
                            corr = capi.Handle.corr(*cs)
                            for level, side in CALLS:
                                q = f"{level}_{side}"
                                rec, _, _ = h.correlations(level, abi.SOURCE_WINDOW, tier, k, SPEC, corr, tg,
                                                           side=side)
                                top_, rows, ser, pre, _, _ = h.correlations_top(level, abi.SOURCE_WINDOW, tier, k,
                                                                                SPEC, corr, tg, spec["top"],
                                                                                side=side)
                                key = f"{c}_{g}_{s}_{q}_{j}_{r}"
                                res["rec" + key], res["top" + key], res["trow" + key] = rec, top_, rows
                                res["tser" + key], res["tpre" + key] = ser, pre
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
