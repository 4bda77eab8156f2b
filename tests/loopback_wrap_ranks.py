"""Histogram cells that wrap in the general path of the multi-rank merge, on several ranks in ONE process on ONE GPU
over the loopback collective (tests/loopback_nccl.cu): the child process of tests/test_gpu_wrap.py
(`python loopback_wrap_ranks.py SPEC.json IN.npz OUT.npz`). Like tests/loopback_ranks.py it must never import torch,
whose libnccl.so.2 would take the place of the loopback library that LD_LIBRARY_PATH names.

Rank 0 allocates one device buffer with its handle's dev_alloc and fills it with buf_tiles copies of the packed tile;
every rank submits that buffer `submits` times per window, so every rank holds every key. One thread per rank builds a
handle on device 0, joins the communicator, sets the history and runs the windows: submit, flush; then one window
rollup of all of them. Rank 0 frees the buffer after the last barrier.

SPEC.json: {"nranks": R, "cfg": {Handle keywords}, "buf_tiles": T, "submits": S, "windows": J, "history": [d, a]}
IN.npz: tab0 = (table, ip, id) rows; tile = the packed records (alz_l7_rec16); ovf = their overflow durations.
OUT.npz: rows_{j}_{r}, rollup_{r}; meta = {"ranks": {r: [{rc, n_out, log, stats}]}, "rollup": {r: info}, "errors",
"maps"}.
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
    R, windows = int(spec["nranks"]), int(spec["windows"])
    out, meta = {}, {"ranks": {}, "rollup": {}, "errors": []}
    shim = C.CDLL("libnccl.so.2")      # the library LD_LIBRARY_PATH names (the one the product's dlopen gets)
    shim.loopback_log_entry.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_ulonglong)]
    shim.loopback_fault_block_status.argtypes = [C.c_int, C.c_long, C.c_int]
    shim.loopback_fault_block_status(-1, 0, 0)
    shim.loopback_log_clear()
    idbuf = (C.c_uint8 * abi.COMM_ID_BYTES)()
    assert L.alz_comm_unique_id(idbuf) == 0
    bar = threading.Barrier(R, timeout=600)
    lock = threading.Lock()
    tile, ovf = inp["tile"], inp["ovf"]
    n_buf = len(tile) * int(spec["buf_tiles"])
    buf = {}

    def fill(h):
        buf["p"] = h.dev_alloc(n_buf * tile.itemsize)
        buf["po"] = h.dev_alloc(max(ovf.nbytes, 8))
        step = 1 << 9
        block = np.tile(tile, step)
        for t in range(0, int(spec["buf_tiles"]), step):
            h.h2d(buf["p"] + t * tile.nbytes, block)
        h.h2d(buf["po"], ovf)
        h.sync()

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
            if r == 0:
                fill(h)
            bar.wait()
            res = []
            for j in range(windows):
                for _ in range(int(spec["submits"])):
                    h.submit_packed_device(buf["p"], n_buf, buf["po"])
                h.sync()
                bar.wait()
                n0 = shim.loopback_log_count(r)
                rows = lr._edge_array(h.max_edges)
                n = C.c_size_t(0)
                d = {"rc": L.alz_window_flush(h.h, rows.ctypes.data_as(C.c_void_p), h.max_edges, C.byref(n))}
                d["n_out"] = n.value
                d["log"] = lr._log_slice(shim, r, n0)
                d["stats"] = h.stats()
                out[f"rows_{j}_{r}"] = rows[: n.value].copy()
                res.append(d)
                bar.wait()
            out[f"rollup_{r}"], info = h.rollup(windows)
            with lock:
                meta["ranks"][str(r)] = res
                meta["rollup"][str(r)] = info
            bar.wait()
            if r == 0:
                h.dev_free(buf.pop("p"))
                h.dev_free(buf.pop("po"))
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
