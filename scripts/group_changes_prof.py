#!/usr/bin/env python
"""What do group changes against a pinned baseline (docs/SPEC.md §25) cost? At bench.py config-2 sizes
(Topo(10_000), --events device-resident events per window, --buffers distinct event buffers taken in turn): the window
history keeps --base-windows + --source-windows windows; a span rollup of the first --base-windows windows is pinned,
and a span rollup of the last --source-windows windows is compared against it. Two maps over the nodes of both sides
(scripts/group_prof.py's): owners (pods two per owner, each service to the owner group of its id) and namespaces (the
owners folded into 100). Timed, as device calls, for each map:
  edges_p99 / edges_top100_p99   alz_group_edge_changes[_top]_device by p99, DELTA, every presence (top: 100, -inf)
  nodes_in_p99 / nodes_top100    alz_group_node_changes[_top]_device, IN side, the same
  *_cached                       the calls above with the baseline's groups kept from the previous call
  *_after_map                    the call right after an alz_group_set of the same map, which makes it group the
                                 baseline's rows again, as the first call after a pin does (each rep sets the map,
                                 waits, then times the call alone)
Per call: device events around the whole call, median and min-max over --reps after two warm-ups, calls alternated.
Per kernel: device time from torch.profiler over the same calls, summed per kernel name and divided by the calls.
Once, for scale, the host route: both sides' rows copied to the host, grouped, and the group edge and IN group node
changes by p99 computed in numpy (tests/group_change_ref.py).
Prints one JSON line per case and a last one with everything, with the card (name, power limit, SM clock now and max).
Usage (GPU box): python scripts/group_changes_prof.py [--reps R] [--events N] [--buffers B]
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
from gnn_top_prof import handle_for, summary  # noqa: E402
from group_prof import maps  # noqa: E402

Q = abi.METRIC_QUANTILE
TOP = 100
IN, S = abi.SIDE_IN, abi.ROLLUP_SPAN
ALL, DELTA = abi.PRESENT_ALL, abi.CHANGE_DELTA
P99 = (Q, 0.99)


def first_after(torch, stream, h, before, call, reps):
    """device ms of `call` right after `before` (a pin or a map set), which makes it group the baseline again"""
    ms = []
    for _ in range(reps + 2):
        before()
        h.sync()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        call()
        e1.record(stream)
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return summary(ms[2:])


def host_route(h, src, base, gmap, reps=3):
    """(ms per call, host clock): both sides' rows copied to the host, grouped, both change lists by p99"""
    import group_change_ref as gcr
    (ps, ns, ws), (pb, nb, wb) = src, base
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        rs, rb = h.d2h(ps, ns, abi.EDGE_OUT), h.d2h(pb, nb, abi.EDGE_OUT)
        gcr.edge_changes(rs, rb, gmap, P99, DELTA, ALL, ws, wb)
        gcr.node_changes(rs, rb, gmap, IN, P99, DELTA, ALL, ws, wb)
        out.append((time.perf_counter() - t0) * 1e3)
    return round(sorted(out)[len(out) // 2], 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=12)
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--buffers", type=int, default=4)
    ap.add_argument("--base-windows", type=int, default=60)
    ap.add_argument("--source-windows", type=int, default=5)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("group_changes_prof.py: no CUDA device")
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    result = {"card": card(), "cases": []}
    print(json.dumps({"card": result["card"]}), flush=True)

    h, bufs, _ = handle_for(torch, stream, 10_000, a.events, a.buffers)
    h.submit_device(bufs[0], a.events)
    first = h.flush_device()[1]                                       # sizes the history
    depth = a.base_windows + a.source_windows
    h.window_history(depth, depth * (first + first // 2))
    for w in range(a.base_windows):
        h.submit_device(bufs[w % len(bufs)], a.events)
        h.flush_device()
    pb, nb, _ = h.rollup_span_device(a.base_windows)
    base_rows = h.d2h(pb, nb, abi.EDGE_OUT)
    pinned = h.baseline_pin(S)
    for w in range(a.source_windows):
        h.submit_device(bufs[(w + 1) % len(bufs)], a.events)
        h.flush_device()
    ps, ns, info_s = h.rollup_span_device(a.source_windows)
    src_rows = h.d2h(ps, ns, abi.EDGE_OUT)
    # the host route reads the baseline from a copy: the span rollup's rows are now the source's
    pb2 = h.dev_alloc(base_rows.nbytes)
    h.h2d(pb2, base_rows)
    result["rows"] = {"source": ns, "source_windows": info_s["windows"], "baseline": nb,
                      "baseline_windows": pinned["windows"]}
    print(json.dumps(result["rows"]), flush=True)
    import group_ref
    for name, ends, groups in maps(np.concatenate([src_rows, base_rows])):
        h.group_set(ends, groups)
        gmap = group_ref.make_map(ends, groups)
        _, listed_e, ce = h.group_edge_changes_device(P99, DELTA, ALL, S)
        _, listed_n, cn = h.group_node_changes_device(IN, P99, DELTA, ALL, S)
        m = {"map": name, "entries": len(ends), "edges": dict(ce, listed=listed_e), "nodes_in": dict(cn,
                                                                                                    listed=listed_n),
             "calls": {}}
        cases = {"edges_p99_cached": lambda: h.group_edge_changes_device(P99, DELTA, ALL, S),
                 f"edges_top{TOP}_p99_cached": lambda: h.group_edge_changes_top_device(P99, TOP, float("-inf"), DELTA,
                                                                                       ALL, S),
                 "nodes_in_p99_cached": lambda: h.group_node_changes_device(IN, P99, DELTA, ALL, S),
                 f"nodes_top{TOP}_in_p99_cached": lambda: h.group_node_changes_top_device(IN, P99, TOP, float("-inf"),
                                                                                          DELTA, ALL, S)}
        ms = timed(torch, stream, h, cases, a.reps)
        for case, f in cases.items():
            m["calls"][case] = {"call_ms": ms[case], "kernels_ms": kernel_times(torch, h, [f], 5)}
        for case, call in (("edges_p99", cases["edges_p99_cached"]), ("nodes_in_p99", cases["nodes_in_p99_cached"]),
                           (f"edges_top{TOP}_p99", cases[f"edges_top{TOP}_p99_cached"]),
                           (f"nodes_top{TOP}_in_p99", cases[f"nodes_top{TOP}_in_p99_cached"])):
            m["calls"][case + "_after_map"] = {"call_ms": first_after(torch, stream, h,
                                                                      lambda: h.group_set(ends, groups), call,
                                                                      a.reps)}
        m["calls"]["edges_p99_after_map"]["kernels_ms"] = kernel_times(
            torch, h, [lambda: (h.group_set(ends, groups), cases["edges_p99_cached"]())], 5)
        m["calls"]["edges_p99_after_map"]["kernels_ms_note"] = "includes the map's sort and duplicate check"
        m["host_route_ms"] = host_route(h, (ps, ns, info_s["windows"]), (pb2, nb, pinned["windows"]), gmap)
        result["cases"].append(m)
        print(json.dumps(m), flush=True)
    h.dev_free(pb2)
    h.group_set([], [])
    h.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
