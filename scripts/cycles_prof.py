#!/usr/bin/env python
"""What do the cycles calls (docs/SPEC.md §28) cost? At bench.py config-2 sizes (Topo(10_000), --events
device-resident events per window, --buffers distinct event buffers taken in turn): the window history keeps --windows
windows. Two sources: the last window, and a span rollup of all of them. Three forms: the node form, and the group
form under group_prof.py's two maps (owners, namespaces). Two filters: none, and ERR5XX >= 1. min_size 2.
Per call: device events around the whole call (alz_cycles_device / alz_group_cycles_device), median and min-max over
--reps after two warm-ups, calls alternated; with the components, cyclic components, largest component, depth and
rows listed. Once per source and form, for scale, the host route: the traversed rows copied to the host and their
strong components found there by scipy (node keys by np.unique, then connected_components(connection="strong")).
Then the hook's worst cases: a chain and a ring of 2^16 nodes in descending key order, about one round per node, and
chains of 512 and 2048 nodes in two-node loops whose indices fall downstream, about N^2 / 4 rounds.
Prints one JSON line per case and a last one with everything, with the card (name, power limit, SM clock now and max).
Usage (GPU box): python scripts/cycles_prof.py [--reps R] [--events N] [--buffers B] [--windows W]
"""
import argparse
import ctypes as C
import itertools
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from alaz_b200 import abi  # noqa: E402
from edge_series_prof import card  # noqa: E402
from edge_top_prof import timed  # noqa: E402
from gnn_top_prof import handle_for  # noqa: E402
from group_prof import maps  # noqa: E402

W, S = abi.SOURCE_WINDOW, abi.ROLLUP_SPAN


def host_route(h, p, n, reps=3):
    """ms per call (host clock): the traversed rows copied to the host and their strong components found by scipy"""
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import connected_components
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        rows = h.d2h(p, n, abi.EDGE_OUT)
        kf = (rows["from_type"].astype(np.uint64) << np.uint64(32)) | rows["from"].astype(np.uint64)
        kt = (rows["to_type"].astype(np.uint64) << np.uint64(32)) | rows["to"].astype(np.uint64)
        keys, inv = np.unique(np.concatenate([kf, kt]), return_inverse=True)
        m = csr_matrix((np.ones(n), (inv[:n], inv[n:])), shape=(len(keys), len(keys)))
        connected_components(m, directed=True, connection="strong")
        out.append((time.perf_counter() - t0) * 1e3)
    return round(sorted(out)[len(out) // 2], 1)


def ring_rows(n, closed):
    """a chain n - 1 -> n - 2 -> ... -> 0 (closed: and 0 -> n - 1), as pod rows"""
    r = np.zeros(n - 1 + closed, dtype=abi.EDGE_OUT)
    r["from"][: n - 1] = np.arange(n - 1, 0, -1)
    r["to"][: n - 1] = np.arange(n - 2, -1, -1)
    if closed:
        r["from"][-1], r["to"][-1] = 0, n - 1
    r["count"] = 1
    return r


def loop_chain_rows(n):
    """n / 2 two-node loops in a chain, upstream loops holding the larger indices: the colouring's quadratic case"""
    k = n // 2
    loops = [(2 * (k - 1 - i), 2 * (k - 1 - i) + 1) for i in range(k)]
    pairs = [p for a, b in loops for p in ((a, b), (b, a))] + [(loops[i][1], loops[i + 1][0]) for i in range(k - 1)]
    r = np.zeros(len(pairs), dtype=abi.EDGE_OUT)
    r["from"], r["to"] = np.asarray(pairs, dtype=np.uint32).T
    r["count"] = 1
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--buffers", type=int, default=4)
    ap.add_argument("--windows", type=int, default=60)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("cycles_prof.py: no CUDA device")
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    result = {"card": card(), "cases": []}
    print(json.dumps({"card": result["card"]}), flush=True)

    h, bufs, _ = handle_for(torch, stream, 10_000, a.events, a.buffers)
    h.submit_device(bufs[0], a.events)
    first = h.flush_device()[1]                                       # sizes the history
    h.window_history(a.windows, a.windows * (first + first // 2))
    for w in range(a.windows):
        h.submit_device(bufs[w % len(bufs)], a.events)
        h.flush_device()
    ps, ns, info_s = h.rollup_span_device(a.windows)
    span_rows = h.d2h(ps, ns, abi.EDGE_OUT)
    result["source"] = {"span_rows": ns, "span_windows": info_s["windows"]}
    forms = [("node", None)] + [(name, (ends, groups)) for name, ends, groups in maps(span_rows)]
    for (src_name, src), (form, mp) in itertools.product((("window", W), ("span", S)), forms):
        group = mp is not None
        h.group_set(*(mp if group else ([], [])))
        if group:
            p, n, _ = h.group_edges_device(src)
        elif src == S:
            p, n = ps, ns
        else:   # the last window's rows, fetched and put back on the device for the host route's copy
            fetched, m = np.zeros(h.max_edges, dtype=abi.EDGE_OUT), C.c_size_t(0)
            h._ck(h.L.alz_window_fetch(h.h, fetched.ctypes.data_as(C.c_void_p), len(fetched), C.byref(m)),
                  "alz_window_fetch")
            fetched = fetched[: m.value]
            p, n = h.dev_alloc(max(fetched.nbytes, 1)), len(fetched)
            h.h2d(p, fetched)
        fn = h.group_cycles_device if group else h.cycles_device
        calls, meta = {}, {}
        for filt in ("none", "err5xx>=1"):
            spec, mv = (None, 0.0) if filt == "none" else (abi.METRIC_ERR5XX, 1.0)
            calls[filt] = lambda fn=fn, spec=spec, mv=mv: fn(src, spec, mv, 2)
            r = calls[filt]()
            meta[filt] = {k: r[5][k] for k in ("traversable", "self_rows", "nodes", "components", "cyclic",
                                                "cyclic_nodes", "largest", "cycle_rows", "depth")}
        ms = timed(torch, stream, h, calls, a.reps)
        host_ms = host_route(h, p, n)
        if not group and src == W:
            h.dev_free(p)
        for name in calls:
            case = {"source": src_name, "form": form, "traversed_rows": n, "filter": name, "call_ms": ms[name],
                    **meta[name]}
            result["cases"].append(case)
            print(json.dumps(case), flush=True)
        hr = {"source": src_name, "form": form, "traversed_rows": n, "host_route_ms": host_ms}
        result["cases"].append(hr)
        print(json.dumps(hr), flush=True)
    h.group_set([], [])
    # the worst cases: a chain and a ring, about one round per node; a chain of two-node loops, about N^2 / 4 rounds
    for name, rows in (("chain_2^16", ring_rows(1 << 16, False)), ("ring_2^16", ring_rows(1 << 16, True)),
                       ("loop_chain_512", loop_chain_rows(512)), ("loop_chain_2048", loop_chain_rows(2048))):
        p = h.dev_alloc(rows.nbytes)
        h.h2d(p, rows)
        nn, nr, info = C.c_size_t(0), C.c_size_t(0), abi.CycleInfo()

        def hook(p=p, n=len(rows)):
            h._ck(h.L.alz_debug_cycles_rows(h.h, C.c_void_p(p), n, None, 0.0, 2, None, 0, C.byref(nn), None, None, 0,
                                            C.byref(nr), C.byref(info)), "alz_debug_cycles_rows")

        ms = timed(torch, stream, h, {name: hook}, max(3, a.reps // 3))
        h.dev_free(p)
        case = {"case": name, "rows": len(rows), "call_ms": ms[name], **info.as_dict()}
        result["cases"].append(case)
        print(json.dumps(case), flush=True)
    result["card_after"] = card()
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
