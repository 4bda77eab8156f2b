#!/usr/bin/env python
"""What do the node calls (docs/SPEC.md §21) cost? At bench.py config-2 sizes (Topo(10_000), --events device-resident
events per window, --buffers distinct event buffers taken in turn): the window history keeps --windows windows and the
source is a span rollup of all of them. Timed, as device calls:
  (a) alz_node_rows_device: every node's row
  (b) alz_node_metrics_device of {count, 5xx rate, p99} on the IN side
  (c) alz_node_top_device: the top 100 nodes by IN-side p99
  (d) alz_node_top_device: the top 100 nodes by OUT-side count
and, through alz_debug_node_rows (which adds a host copy of the result, so the hook lists are timed on the device
kernels alone), two lists of 2^20 rows: uniform (about 4 rows per node) and one hub (every row into one service, one
run of 2^20 IN-side contributions). Once, for scale, the host alternative: the span's rows copied to the host, grouped
in numpy (tests/node_ref.py) and the p99 of every node's IN side computed there.

Per call: device events around the whole call, median and min-max over --reps after two warm-ups, calls alternated.
Per kernel: device time from torch.profiler over the same calls, summed per kernel name and divided by the calls.
Bytes: the keys pass reads 16 B and writes 24 B per row; the sort moves 12 B per pair per pass (five passes); the
reduce reads 296 B of each row twice (once per end) and writes 576 B per node.
Prints one JSON line per case and a last one with everything, with the card (name, power limit, SM clock now and max).
Usage (GPU box): python scripts/node_prof.py [--reps R] [--events N] [--buffers B] [--windows W]
"""
import argparse
import json
import os
import sys
import time

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
TOP = 100


def host_alternative(h, reps=3):
    """the span's rows copied to the host, grouped by node and every IN side's p99 in numpy: ms per call"""
    import node_ref as nr
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        rows = h.rollup_span(h.last_span)[0]
        nodes = nr.group(rows)
        nr.values(nodes, abi.SIDE_IN, (Q, 0.99))
        out.append((time.perf_counter() - t0) * 1e3)
    return round(sorted(out)[len(out) // 2], 1)


def hook_lists(np, n):
    """(uniform, hub): n rows each; uniform spreads their 2n ends over about n / 2 nodes (4 per node)"""
    rng = np.random.default_rng(11)
    lists = []
    for hub in (False, True):
        r = np.zeros(n, dtype=abi.EDGE_OUT)
        r["count"] = rng.integers(1, 1 << 20, n, dtype=np.uint64)
        r["err5xx"] = rng.integers(0, 1 << 10, n, dtype=np.uint64)
        r["lat_sum_ns"] = rng.integers(0, 1 << 40, n, dtype=np.uint64)
        r["hist"] = rng.integers(0, 1 << 16, (n, abi.NB), dtype=np.uint64).astype(np.uint32)
        r["from_type"] = 0
        r["from"] = rng.permutation(n) if hub else rng.integers(0, n // 4, n)
        r["to_type"] = 1 if hub else rng.integers(0, 4, n)
        r["to"] = 0 if hub else rng.integers(0, n // 16, n)
        lists.append(r)
    return lists


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=12)
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--buffers", type=int, default=4)
    ap.add_argument("--windows", type=int, default=60)
    ap.add_argument("--hook-rows", type=int, default=1 << 20)
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("node_prof.py: no CUDA device")
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    result = {"card": card(), "cases": []}

    h, bufs, _ = handle_for(torch, stream, 10_000, a.events, a.buffers)
    h.submit_device(bufs[0], a.events)
    first = h.flush_device()[1]                                       # sizes the history
    W = a.windows
    h.window_history(W, W * (first + first // 2))
    for w in range(W):
        h.submit_device(bufs[w % len(bufs)], a.events)
        h.flush_device()
    _, n, span = h.rollup_span_device(W)
    h.last_span = W
    S = abi.ROLLUP_SPAN
    nodes = h.node_rows_device(S)[1]
    result["rows"] = {"span": n, "span_windows": span["windows"], "window_rows": first, "nodes": nodes}
    p99 = (Q, 0.99)
    cases = {
        "a_node_rows": lambda: h.node_rows_device(S),
        "b_metrics_in_count_5xx_rate_p99": lambda: h.node_metrics_device(S, abi.SIDE_IN, abi.METRIC_COUNT,
                                                                          abi.METRIC_ERR_RATE, p99),
        f"c_top{TOP}_in_p99": lambda: h.node_top_device(S, abi.SIDE_IN, p99, TOP),
        f"d_top{TOP}_out_count": lambda: h.node_top_device(S, abi.SIDE_OUT, abi.METRIC_COUNT, TOP),
    }
    ms = timed(torch, stream, h, cases, a.reps)
    for name, f in cases.items():
        c = {"case": name, "rows": n, "nodes": nodes, "call_ms": ms[name], "kernels_ms": kernel_times(torch, h, [f], 5)}
        result["cases"].append(c)
        print(json.dumps(c), flush=True)
    host = host_alternative(h)
    result["host_alternative_ms"] = host
    print(json.dumps({"host_alternative_ms": host}), flush=True)

    # the hook lists: the rows stay on the device; the call copies its node rows to the host, so the comparison is
    # the device time of its kernels
    import ctypes as C
    hook = {}
    for name, rows in zip(("uniform", "hub"), hook_lists(np, a.hook_rows)):
        p = h.dev_alloc(rows.nbytes)
        h.h2d(p, rows)
        cnt = C.c_size_t(0)
        h._ck(h.L.alz_debug_node_rows(h.h, C.c_void_p(p), len(rows), None, 0, C.byref(cnt)), "alz_debug_node_rows",
              allow=(abi.E_CAPACITY,))
        out = np.zeros(cnt.value, dtype=abi.NODE_OUT)

        def f(p=p, m=len(rows), out=out, cnt=cnt):
            h._ck(h.L.alz_debug_node_rows(h.h, C.c_void_p(p), m, out.ctypes.data_as(C.c_void_p), len(out),
                                          C.byref(cnt)), "alz_debug_node_rows")
        ms = timed(torch, stream, h, {name: f}, a.reps)[name]
        kt = kernel_times(torch, h, [f], 5)
        ours = {k: v for k, v in kt.items() if "node_" in k or "Radix" in k or "Scan" in k or "scan" in k}
        c = {"case": f"hook_{name}", "rows": len(rows), "nodes": cnt.value, "call_ms": ms, "kernels_ms": kt,
             "device_ms": round(sum(ours.values()), 4)}
        hook[name] = c
        print(json.dumps(c), flush=True)
        h.dev_free(p)
    result["hook"] = hook
    h.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
