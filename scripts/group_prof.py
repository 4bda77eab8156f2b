#!/usr/bin/env python
"""What do the group calls (docs/SPEC.md §24) cost? At bench.py config-2 sizes (Topo(10_000), --events device-resident
events per window, --buffers distinct event buffers taken in turn): the window history keeps --windows windows, and a
span rollup of all of them is the source. Two maps over its nodes:
  owners      pods two per owner (group = pod id / 2), each service to the owner group of its own id
  namespaces  the same owners folded into 100 namespaces (group = owner % 100)
Timed, as device calls, for each map:
  edges            alz_group_edges_device
  node_metrics     alz_group_node_metrics_device, IN, {count, 5xx rate, p99}
  node_top100_p99  alz_group_node_top_device, IN, top 100 by p99
Per call: device events around the whole call, median and min-max over --reps after two warm-ups, calls alternated.
Per kernel: device time from torch.profiler over the same calls, summed per kernel name and divided by the calls.
Once, for scale, the host route: the span's rows copied to the host, grouped with tests/group_ref.py, the group nodes'
IN p99 computed in numpy.
Then the reduce on hook lists of 2^20 rows (alz_debug_group_edges): uniform (2^16 pods in fours to 2^10 services)
against one group edge (every row into one), per kernel from torch.profiler.
Prints one JSON line per case and a last one with everything, with the card (name, power limit, SM clock now and max).
Usage (GPU box): python scripts/group_prof.py [--reps R] [--events N] [--buffers B] [--windows W]
"""
import argparse
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
from edge_changes_prof import kernel_times  # noqa: E402
from edge_series_prof import card  # noqa: E402
from edge_top_prof import timed  # noqa: E402
from gnn_top_prof import handle_for  # noqa: E402

Q = abi.METRIC_QUANTILE
IN, S = abi.SIDE_IN, abi.ROLLUP_SPAN
P99 = (Q, 0.99)
PANEL = [abi.METRIC_COUNT, abi.METRIC_ERR_RATE, P99]


def maps(rows):
    """(name, NODE_ENDS, groups) of the two maps over the nodes of the rows"""
    import node_ref
    keys = node_ref.keys(rows)
    t, v = keys >> np.uint64(32), keys & np.uint64(0xFFFFFFFF)
    keep = t <= abi.NODE_SVC
    ends = np.zeros(int(keep.sum()), dtype=abi.NODE_ENDS)
    ends["type"], ends["value"] = t[keep], v[keep]
    owner = np.where(t[keep] == abi.NODE_POD, v[keep] // 2, v[keep]).astype(np.uint32)
    return [("owners", ends, owner), ("namespaces", ends, owner % 100)]


def host_route(h, p, n, gmap, reps=3):
    """(ms per call, host clock): the rows copied to the host, grouped, every group node's IN p99"""
    import group_ref
    import node_ref
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        rows = h.d2h(p, n, abi.EDGE_OUT)
        node_ref.values(group_ref.nodes(rows, gmap), IN, P99)
        out.append((time.perf_counter() - t0) * 1e3)
    return round(sorted(out)[len(out) // 2], 1)


def hook_lists(torch, h):
    """per-kernel ms of alz_debug_group_edges on 2^20 rows, uniform against one group edge"""
    import ctypes as C
    rng = np.random.default_rng(3)
    n = 1 << 20
    r = np.zeros(n, dtype=abi.EDGE_OUT)
    r["from_type"], r["to_type"] = abi.NODE_POD, abi.NODE_SVC
    r["from"] = rng.integers(0, 1 << 16, n)
    r["to"] = rng.integers(0, 1 << 10, n)
    r["count"] = rng.integers(0, 1 << 20, n)
    r["hist"] = rng.integers(0, 1 << 8, (n, abi.NB))
    pods = np.zeros(1 << 16, dtype=abi.NODE_ENDS)
    pods["value"] = np.arange(1 << 16)
    out = {}
    for name, groups, to in (("uniform", np.arange(1 << 16) // 4, r["to"].copy()),
                             ("one_group_edge", np.zeros(1 << 16), np.full(n, 5))):
        r["to"] = to
        h.group_set(pods, groups.astype(np.uint32))
        p = h.dev_alloc(r.nbytes)
        h.h2d(p, r)
        res = np.zeros(n, dtype=abi.EDGE_OUT)
        m = C.c_size_t(0)

        def call():
            h._ck(h.L.alz_debug_group_edges(h.h, C.c_void_p(p), n, res.ctypes.data_as(C.c_void_p), n, C.byref(m),
                                            None), "alz_debug_group_edges")
        call()
        out[name] = {"edges": m.value, "kernels_ms": kernel_times(torch, h, [call], 5)}
        h.dev_free(p)
    h.group_set([], [])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=12)
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--buffers", type=int, default=4)
    ap.add_argument("--windows", type=int, default=60)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("group_prof.py: no CUDA device")
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
    rows = h.d2h(ps, ns, abi.EDGE_OUT)
    result["source"] = {"rows": ns, "windows": info_s["windows"]}
    import group_ref
    for name, ends, groups in maps(rows):
        h.group_set(ends, groups)
        gmap = group_ref.make_map(ends, groups)
        _, n_edges, ginfo = h.group_edges_device(S)
        _, n_nodes = h.group_nodes_device(S)
        cases = {"edges": lambda: h.group_edges_device(S),
                 "node_metrics": lambda: h.group_node_metrics_device(S, IN, *PANEL),
                 "node_top100_p99": lambda: h.group_node_top_device(S, IN, P99, 100, float("-inf"))}
        ms = timed(torch, stream, h, cases, a.reps)
        m = {"map": name, "entries": len(ends), "group_edges": n_edges, "group_nodes": n_nodes, "info": ginfo,
             "calls": {}}
        for case, f in cases.items():
            m["calls"][case] = {"call_ms": ms[case], "kernels_ms": kernel_times(torch, h, [f], 5)}
        m["host_route_ms"] = host_route(h, ps, ns, gmap)
        result["cases"].append(m)
        print(json.dumps(m), flush=True)
    result["hook_2_20"] = hook_lists(torch, h)
    print(json.dumps({"hook_2_20": result["hook_2_20"]}), flush=True)
    h.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
