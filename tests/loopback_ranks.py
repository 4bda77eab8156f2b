"""Several ranks of the multi-rank window merge in ONE process on ONE GPU, over the loopback collective
(tests/loopback_nccl.cu), plus numpy restatements of the merge's host-side rules.

As a program (`python loopback_ranks.py SPEC.json IN.npz OUT.npz`) it is the child process of
tests/test_gpu_loopback_ranks.py: it must never import torch, whose libnccl.so.2 would take the place of the
loopback library that LD_LIBRARY_PATH names. One thread per rank builds a handle on device 0, joins the
communicator and runs the windows the spec describes; a handle without a communicator (the "solo" handle) runs
every window's records of all ranks on its own. Everything each rank returned goes to OUT.npz.

SPEC.json: {"nranks": R, "cfg": {Handle keywords}, "cfg_rank": {"r": {keywords for rank r}},
            "tables": K, "windows": [{"flush": "host" | "device", "cap": rows | null, "fetch": bool,
                                      "gnn": bool, "commit": bool}], "fault": [rank, kth, status] | null,
            "solo": bool, "init_only": bool}
IN.npz: tab{k} = (table, ip, id) rows; w{j}_r{r} = the L7 records rank r submits in window j; with "commit",
        rank r submits the first half, upserts commit{j} = (table, ip, id) rows, commits, then submits the rest.
"""
import ctypes as C
import json
import os
import sys
import threading

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from alaz_b200 import abi  # noqa: E402

ROW_BYTES = 296                # sizeof(alz_edge_out)
OP_ALLGATHER, OP_ALLREDUCE = 1, 2


# ---- numpy restatements of alz_device.cuh / alz_comm.cu -------------------------------------------------
def hash32(x):
    x = np.asarray(x, dtype=np.uint64) & 0xFFFFFFFF
    x ^= x >> 16
    x = (x * 0x85EBCA6B) & 0xFFFFFFFF
    x ^= x >> 13
    x = (x * 0xC2B2AE35) & 0xFFFFFFFF
    x ^= x >> 16
    return x


def owner_rank(saddr, nranks):
    """alz_owner_rank: the rank of an event, a function of its source address only."""
    if nranks <= 1:
        return np.zeros(np.shape(saddr), dtype=np.uint64)
    h = hash32(np.asarray(saddr, dtype=np.uint64) ^ 0xA1A2B200)
    return (h * np.uint64(nranks)) >> np.uint64(32)


def block_rows_for(max_count):
    """Rows of one rank's block in the merge's all-gather: the largest rank's count + 25 %, in steps of 1024."""
    want = int(max_count) + int(max_count) // 4 + 1024
    return (want + 1023) // 1024 * 1024


def make_edge_key(pod_id, other_type, other, rev):
    """Packed edge key (the canonical order of merged rows is ascending key)."""
    if rev and other_type == abi.NODE_POD:
        pod_id, other, rev = other, pod_id, False
    return (int(rev) << 63) | (int(other_type) << 61) | ((int(pod_id) & 0x1FFFFFFF) << 32) | (int(other) & 0xFFFFFFFF)


def row_key_of(row):
    """Packed key of an alz_edge_out row (alz_comm.cu row_key_of)."""
    if int(row["from_type"]) == abi.NODE_POD:
        return make_edge_key(int(row["from"]), int(row["to_type"]), int(row["to"]), False)
    return make_edge_key(int(row["to"]), int(row["from_type"]), int(row["from"]), True)


def canonical(rows):
    """rows in the merge's canonical order."""
    keys = [row_key_of(r) for r in rows]
    return rows[np.argsort(np.array(keys, dtype=np.uint64), kind="stable")]


# ---- the child process --------------------------------------------------------------------------------------
def _libnccl_maps():
    with open("/proc/self/maps") as f:
        return sorted({ln.split()[-1] for ln in f if "libnccl" in ln and "/" in ln})


def _edge_array(n):
    return np.zeros(max(int(n), 1), dtype=abi.EDGE_OUT)


def main(spec_path, in_path, out_path):
    from alaz_b200 import capi
    spec = json.load(open(spec_path))
    with np.load(in_path) as z:     # read every array now: the rank threads must not share the zip file
        inp = {k: z[k] for k in z.files}
    L = capi.load()
    R = int(spec["nranks"])
    out, meta = {}, {"ranks": {}, "errors": []}

    if spec.get("init_only"):
        # alz_comm_init's argument checks: the rejected ones must not even load NCCL
        h = capi.Handle(device=0, max_endpoints=1 << 10, max_pairs=1 << 12, max_batch=1 << 12)
        idbuf = (C.c_uint8 * abi.COMM_ID_BYTES)()
        meta["rc_65"] = L.alz_comm_init(h.h, 65, 0, idbuf)
        meta["rc_100"] = L.alz_comm_init(h.h, 100, 99, idbuf)
        meta["rc_rank_high"] = L.alz_comm_init(h.h, 4, 4, idbuf)
        meta["rc_rank_neg"] = L.alz_comm_init(h.h, 4, -1, idbuf)
        meta["rc_zero"] = L.alz_comm_init(h.h, 0, 0, idbuf)
        meta["loaded_before"] = _libnccl_maps()
        assert L.alz_comm_unique_id(idbuf) == 0
        meta["rc_one"] = L.alz_comm_init(h.h, 1, 0, idbuf)
        meta["rc_again"] = L.alz_comm_init(h.h, 1, 0, idbuf)
        meta["maps"] = _libnccl_maps()
        h.close()
        np.savez(out_path, meta=np.array(json.dumps(meta)))
        return 0

    shim = C.CDLL("libnccl.so.2")      # the library LD_LIBRARY_PATH names (the one the product's dlopen gets)
    shim.loopback_log_entry.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_ulonglong)]
    shim.loopback_fault_block_status.argtypes = [C.c_int, C.c_long, C.c_int]
    if spec.get("fault"):
        shim.loopback_fault_block_status(*[int(x) for x in spec["fault"]])
    else:
        shim.loopback_fault_block_status(-1, 0, 0)
    shim.loopback_log_clear()
    tables = [inp[f"tab{k}"] for k in range(int(spec.get("tables", 0)))]
    windows = spec["windows"]
    idbuf = (C.c_uint8 * abi.COMM_ID_BYTES)()
    assert L.alz_comm_unique_id(idbuf) == 0
    bar = threading.Barrier(R, timeout=300)
    lock = threading.Lock()

    def upsert_rows(h, rows):
        for tab in (abi.TABLE_POD, abi.TABLE_SVC):
            m = rows[:, 0] == tab
            if m.any():
                h.upsert_batch(tab, rows[m, 1].astype(np.uint32), rows[m, 2].astype(np.uint32))

    def run_windows(h, r, recs_of, log_of):
        res = []
        for j, w in enumerate(windows):
            recs = recs_of(j)
            if w.get("commit"):
                h.submit(recs[: len(recs) // 2])
                upsert_rows(h, inp[f"commit{j}"])
                h.commit()
                h.submit(recs[len(recs) // 2:])
            elif len(recs):
                h.submit(recs)
            h.sync()
            if log_of:
                bar.wait()
            n0 = log_of() if log_of else 0
            d = {}
            if w.get("flush", "host") == "host":
                cap = h.max_edges if w.get("cap") is None else int(w["cap"])
                buf = _edge_array(cap)
                n = C.c_size_t(0)
                d["rc"] = h.L.alz_window_flush(h.h, buf.ctypes.data_as(C.c_void_p), cap, C.byref(n))
                d["n_out"] = n.value
                ok = d["rc"] == abi.OK or (d["rc"] == abi.E_CAPACITY and n.value <= cap)
                rows = buf[: n.value].copy() if ok else buf[:0].copy()
            else:
                p, n = C.c_void_p(), C.c_size_t(0)
                d["rc"] = h.L.alz_window_flush_device(h.h, C.byref(p), C.byref(n))
                d["n_out"] = n.value
                d["dev_null"] = not p.value
                rows = h.d2h(p.value, n.value, abi.EDGE_OUT) if (n.value and p.value) else _edge_array(0)[:0]
            if log_of:
                d["log"] = _log_slice(shim, r, n0)
            if w.get("fetch"):
                buf = _edge_array(h.max_edges)
                n = C.c_size_t(0)
                d["fetch_rc"] = h.L.alz_window_fetch(h.h, buf.ctypes.data_as(C.c_void_p), h.max_edges, C.byref(n))
                out[f"fetch_{j}_{r}"] = buf[: n.value].copy()
            if w.get("gnn"):
                sc = np.zeros(max(h.max_edges, 1), np.float32)
                n = C.c_size_t(0)
                d["gnn_rc"] = h.L.alz_gnn_score(h.h, sc.ctypes.data_as(C.c_void_p), h.max_edges, C.byref(n))
                out[f"gnn_{j}_{r}"] = sc[: n.value].copy()
            d["stats"] = h.stats()
            out[f"rows_{j}_{r}"] = rows
            res.append(d)
            if log_of:
                bar.wait()
        return res

    def rank_main(r):
        try:
            kw = dict(spec["cfg"])
            kw.update(spec.get("cfg_rank", {}).get(str(r), {}))
            h = capi.Handle(device=0, **kw)
            rc = L.alz_comm_init(h.h, R, r, idbuf)
            if rc != 0:
                raise RuntimeError(f"alz_comm_init: {rc}")
            if r == 0:
                meta["maps"] = _libnccl_maps()
            for t in tables:
                upsert_rows(h, t)
            h.commit()
            res = run_windows(h, r, lambda j: inp[f"w{j}_r{r}"], lambda: shim.loopback_log_count(r))
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
        kw = dict(spec["cfg"])
        h = capi.Handle(device=0, **kw)
        for t in tables:
            upsert_rows(h, t)
        h.commit()
        allrecs = lambda j: np.concatenate([inp[f"w{j}_r{r}"] for r in range(R)])
        meta["solo"] = run_windows(h, "solo", allrecs, None)
        h.close()
    meta["maps_end"] = _libnccl_maps()
    out["meta"] = np.array(json.dumps(meta))
    np.savez(out_path, **out)
    return 0


def _log_slice(shim, r, n0):
    res = []
    for i in range(n0, shim.loopback_log_count(r)):
        op, b = C.c_int(0), C.c_ulonglong(0)
        shim.loopback_log_entry(r, i, C.byref(op), C.byref(b))
        res.append([op.value, b.value])
    return res


if __name__ == "__main__":
    sys.exit(main(*sys.argv[1:4]))
