#!/usr/bin/env python
"""What do group series and group trends (docs/SPEC.md §26) cost? At bench.py config-2 sizes (Topo(10_000), --events
device-resident events per window, --buffers distinct event buffers taken in turn): the window history keeps 60
windows; the source is a span rollup of the last 60 windows. For each of scripts/group_prof.py's two maps (owners:
pods two per owner, each service to the owner group of its id; namespaces: the owners folded into 100), timed as
device calls:
  (a) alz_group_node_series_device: every group node x 60 points, {count, 5xx rate, p99} of the IN side
  (b) alz_group_node_series_keys_device: 10 groups named by the caller x 60 points, {p99} of the IN side
  (c) alz_group_node_trends_top_device: the top 100 group nodes by IN p99 ZSCORE (the last 5 points against the 55)
  (d) alz_group_edge_series_device: every group edge x 60 points, {count, 5xx rate, p99}
and, for the scale of the map lookups, alz_node_series_device over the same source and points (the same path with no
map). Once, the host route the calls replace: each retained window alone as rollup(j) - rollup(j - 1) copied
to the host, grouped by the map, and every group node's IN p99 computed in numpy (tests/group_ref.py).
Per call: device events around the whole call, median and min-max over --reps after two warm-ups, calls alternated.
Per kernel: device time from torch.profiler over the same calls, summed per kernel name and divided by the calls.
Prints one JSON line per case and a last one with everything, with the card (name, power limit, SM clock now and max).
Usage (GPU box): python scripts/group_series_prof.py [--reps R] [--events N] [--buffers B] [--windows W]
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
from alaz_b200 import abi, capi  # noqa: E402
from edge_changes_prof import kernel_times  # noqa: E402
from edge_series_prof import card  # noqa: E402
from edge_top_prof import timed  # noqa: E402
from gnn_top_prof import handle_for  # noqa: E402
from group_prof import maps  # noqa: E402

Q = abi.METRIC_QUANTILE
TOP = 100
P99 = (Q, 0.99)


def host_route(h, W, gmap):
    """every retained window alone as rollup(j) - rollup(j - 1) on the host, grouped by the map, every group node's
    IN p99: ms (host clock)"""
    import group_ref
    import node_ref
    from change_ref import row_keys
    t0 = time.perf_counter()
    prev = np.zeros(0, dtype=abi.EDGE_OUT)
    for j in range(1, W + 1):
        cur = h.rollup(j)[0]
        pos = np.searchsorted(row_keys(cur), row_keys(prev))   # a rollup's rows are ascending; prev's keys are in cur
        d = cur.copy()
        for f in ("count", "err5xx", "lat_sum_ns", "hist"):
            d[f][pos] -= prev[f]
        node_ref.values(group_ref.nodes(d[d["count"] > 0], gmap), abi.SIDE_IN, P99)
        prev = cur
    return round((time.perf_counter() - t0) * 1e3, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=12)
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--buffers", type=int, default=4)
    ap.add_argument("--windows", type=int, default=60)
    ap.add_argument("--no-host", action="store_true", help="skip the host route")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("group_series_prof.py: no CUDA device")
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    result = {"card": card(), "cases": []}
    print(json.dumps({"card": result["card"]}), flush=True)

    h, bufs, _ = handle_for(torch, stream, 10_000, a.events, a.buffers)
    h.submit_device(bufs[0], a.events)
    first = h.flush_device()[1]                                       # sizes the history
    W = a.windows
    h.window_history(W, W * (first + first // 2))
    for w in range(W):
        h.submit_device(bufs[w % len(bufs)], a.events)
        h.flush_device()
    ps, n, span = h.rollup_span_device(W)
    S, IN = abi.ROLLUP_SPAN, abi.SIDE_IN
    rows = h.d2h(ps, n, abi.EDGE_OUT)
    result["rows"] = {"span": n, "span_windows": span["windows"], "window_rows": first}
    print(json.dumps(result["rows"]), flush=True)
    three = (abi.METRIC_COUNT, abi.METRIC_ERR_RATE, P99)
    T = capi.Handle.trend
    import group_ref
    for name, ends, groups in maps(rows):
        h.group_set(ends, groups)
        gmap = group_ref.make_map(ends, groups)
        gnodes = h.group_nodes(S)
        named = gnodes[gnodes["type"] == abi.NODE_GROUP][:10]
        m = {"map": name, "entries": len(ends), "group_nodes": len(gnodes), "group_edges": h.group_edges_device(S)[1],
             "calls": {}}
        cases = {
            f"a_all_group_nodes_x{W}_count_5xx_rate_p99_in": lambda: h.group_node_series_device(S, IN, 0, W, *three),
            f"b_10_groups_x{W}_p99_in": lambda: h.group_node_series_keys_device(named, IN, 0, W, P99),
            f"c_top{TOP}_group_nodes_in_p99_zscore_x{W}": lambda: h.group_node_trends_top_device(
                S, IN, 0, W, P99, T(abi.TREND_ZSCORE, recent=5), TOP),
            f"d_all_group_edges_x{W}_count_5xx_rate_p99": lambda: h.group_edge_series_device(S, 0, W, *three),
            f"node_series_all_nodes_x{W}_count_5xx_rate_p99_in": lambda: h.node_series_device(S, IN, 0, W, *three),
        }
        ms = timed(torch, stream, h, cases, a.reps)
        for case, f in cases.items():
            info = f()[-1]
            c = {"series_rows": info["edges"], "points": info["points"], "rows_in": info["rows_in"],
                 "call_ms": ms[case], "kernels_ms": kernel_times(torch, h, [f], 5)}
            if "valid" in info:
                c.update(valid=info["valid"], above=info["above"])
            m["calls"][case] = c
        if not a.no_host and name == "owners":   # once: the route does not depend on the map's size much
            m["host_route_ms"] = host_route(h, W, gmap)
        result["cases"].append(m)
        print(json.dumps(m), flush=True)
    h.group_set([], [])
    h.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
