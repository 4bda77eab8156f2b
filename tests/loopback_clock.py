"""Child process of tests/test_gpu_loopback_clock.py: ranks with a window clock, in ONE process on ONE GPU over the
loopback collective (tests/loopback_nccl.cu), driven by a list of operations. It uses the helpers of
tests/loopback_ranks.py and, like it, must never import torch.

`python loopback_clock.py SPEC.json IN.npz OUT.npz`

SPEC.json: {"nranks": R, "cfg": {Handle keywords}, "ops": [op, ...], "solo": bool}
  op = {"op": "clock", "r": r, "args": [first_kernel, first_user, window_ns]}
     | {"op": "submit", "r": r, "key": name, "how": "host" | "device"}
     | {"op": "commit", "r": r, "key": name}          upserts IN[name] = (table, ip, id) rows, then commits
     | {"op": "fold", "r": r}
     | {"op": "join"}                                  every rank joins the communicator
     | {"op": "flush", "how": "host" | "device", "cap": rows | null, "fetch": bool}   every rank, or
     | {"op": "flush", "r": r}                         rank r alone, before it joins
IN.npz: tables = (table, ip, id) rows every rank loads first; the arrays the ops name.
OUT.npz: meta = JSON {"ranks": {r: [after each op: {"stats", "epoch": [rc, value], and for a flush "rc", "n_out",
         "log", "fetch_rc"}]}, "solo": [...], "errors"}; rows_{i}_{r} / fetch_{i}_{r} / rows_{i}_solo.
"""
import ctypes as C
import json
import os
import sys
import threading

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import loopback_ranks as lr  # noqa: E402  (puts the repository root on sys.path)

from alaz_b200 import abi  # noqa: E402


def _epoch(h):
    e = C.c_uint64(0)
    rc = h.L.alz_window_epoch(h.h, C.byref(e))
    return [rc, e.value if rc == abi.OK else None]


def _upsert_rows(h, rows):
    for tab in (abi.TABLE_POD, abi.TABLE_SVC):
        m = rows[:, 0] == tab
        if m.any():
            h.upsert_batch(tab, rows[m, 1].astype(np.uint32), rows[m, 2].astype(np.uint32))


def _flush(h, op):
    """one flush as the caller makes it: (record, rows, fetched rows or None)"""
    d = {}
    if op.get("how", "host") == "host":
        cap = h.max_edges if op.get("cap") is None else int(op["cap"])
        buf = lr._edge_array(cap)
        n = C.c_size_t(0)
        d["rc"] = h.L.alz_window_flush(h.h, buf.ctypes.data_as(C.c_void_p), cap, C.byref(n))
        ok = d["rc"] == abi.OK or (d["rc"] == abi.E_CAPACITY and n.value <= cap)
        rows = buf[: n.value].copy() if ok else buf[:0].copy()
    else:
        p, n = C.c_void_p(), C.c_size_t(0)
        d["rc"] = h.L.alz_window_flush_device(h.h, C.byref(p), C.byref(n))
        rows = h.d2h(p.value, n.value, abi.EDGE_OUT) if (n.value and p.value) else lr._edge_array(0)[:0]
    d["n_out"] = n.value
    fetched = None
    if op.get("fetch"):
        buf = lr._edge_array(h.max_edges)
        m = C.c_size_t(0)
        d["fetch_rc"] = h.L.alz_window_fetch(h.h, buf.ctypes.data_as(C.c_void_p), h.max_edges, C.byref(m))
        fetched = buf[: m.value].copy()
    return d, rows, fetched


def main(spec_path, in_path, out_path):
    from alaz_b200 import capi
    spec = json.load(open(spec_path))
    with np.load(in_path) as z:     # read every array now: the rank threads must not share the zip file
        inp = {k: z[k] for k in z.files}
    L = capi.load()
    R = int(spec["nranks"])
    ops = spec["ops"]
    out, meta = {}, {"ranks": {}, "errors": []}
    shim = C.CDLL("libnccl.so.2")      # the library LD_LIBRARY_PATH names (the one the product's dlopen gets)
    shim.loopback_log_entry.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_ulonglong)]
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
            _upsert_rows(h, inp["tables"])
            h.commit()
            res = []
            for i, op in enumerate(ops):
                kind, mine = op["op"], op.get("r", r) == r
                d = {}
                n0 = shim.loopback_log_count(r)
                if kind == "join":
                    if L.alz_comm_init(h.h, R, r, idbuf) != 0:
                        raise RuntimeError("alz_comm_init")
                elif kind == "flush" and mine:
                    d, rows, fetched = _flush(h, op)
                    out[f"rows_{i}_{r}"] = rows
                    if fetched is not None:
                        out[f"fetch_{i}_{r}"] = fetched
                    d["log"] = lr._log_slice(shim, r, n0)
                elif mine and kind == "clock":
                    d["rc"] = h.L.alz_window_clock(h.h, *[C.c_uint64(int(x)) for x in op["args"]])
                elif mine and kind == "submit":
                    recs = np.ascontiguousarray(inp[op["key"]], dtype=abi.L7_REC)
                    if op.get("how", "host") == "device":
                        p = h.dev_alloc(max(1, len(recs)) * recs.itemsize)
                        h.h2d(p, recs)
                        h.submit_device(p, len(recs))
                        h.sync()
                        h.dev_free(p)
                    else:
                        h.submit(recs)
                elif mine and kind == "commit":
                    _upsert_rows(h, inp[op["key"]])
                    h.commit()
                elif mine and kind == "fold":
                    h.fold()
                h.sync()
                d["stats"] = h.stats()
                d["epoch"] = _epoch(h)
                res.append(d)
                bar.wait()
            with lock:
                meta["ranks"][str(r)] = res
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

    if spec.get("solo") and not meta["errors"]:
        # one handle: rank 0's clock, every rank's records, the ranks' flushes
        h = capi.Handle(device=0, **spec["cfg"])
        _upsert_rows(h, inp["tables"])
        h.commit()
        solo = []
        for i, op in enumerate(ops):
            if op["op"] == "clock" and op["r"] == 0:
                h.window_clock(*op["args"])
            elif op["op"] == "submit":
                h.submit(inp[op["key"]])
            elif op["op"] == "commit" and op["r"] == 0:
                _upsert_rows(h, inp[op["key"]])
                h.commit()
            elif op["op"] == "flush" and "r" not in op:
                d, rows, _ = _flush(h, {})
                out[f"rows_{i}_solo"] = rows
                solo.append(d)
        meta["solo"] = solo
        h.close()
    meta["maps"] = lr._libnccl_maps()
    out["meta"] = np.array(json.dumps(meta))
    np.savez(out_path, **out)
    return 0


if __name__ == "__main__":
    sys.exit(main(*sys.argv[1:4]))
