#!/usr/bin/env python
"""What do node series and node trends (docs/SPEC.md §22) cost? At bench.py config-2 sizes (Topo(10_000), --events
device-resident events per window, --buffers distinct event buffers taken in turn): the window history keeps 60
windows and a tier of factor 5 keeps 12 entries. The source is a span rollup of the last 60 windows. Timed, as device
calls:
  (a) alz_node_series_device: every source node x 60 points, {count, 5xx rate, p99} of the IN side
  (b) alz_node_series_keys_device: 10 services named by the caller x 60 points, {p99} of the IN side
  (c) alz_node_trends_top_device: the top 100 nodes by IN p99 ZSCORE (the last 5 points against the 55 before)
  (d) alz_node_series_device: every source node x the tier's 12 points, {count, 5xx rate, p99} of the IN side
and once, for scale, the host route the calls replace: each retained window alone as the difference of two window
rollups (rollup(j) - rollup(j - 1), copied to the host), grouped by node and its IN p99 computed in numpy
(tests/node_ref.py).

Per call: device events around the whole call, median and min-max over --reps after two warm-ups, calls alternated.
Per kernel: device time from torch.profiler over the same calls, summed per kernel name and divided by the calls.
Scratch of a call: 8 + 4 B of keys and values per entry row in and out of the sort, 8 B of heads and run numbers per
entry row, the sort's temporary storage, and 576 B per present (node, entry) slot; the present slots of (a) are counted
from its presence bytes (a host call of the same series), so the scratch is printed for the run's own data.
Prints one JSON line per case and a last one with everything, with the card (name, power limit, SM clock now and max).
Usage (GPU box): python scripts/node_series_prof.py [--reps R] [--events N] [--buffers B] [--windows W] [--factor F]
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
from alaz_b200 import abi, capi  # noqa: E402
from edge_changes_prof import kernel_times  # noqa: E402
from edge_series_prof import card  # noqa: E402
from edge_top_prof import timed  # noqa: E402
from gnn_top_prof import handle_for  # noqa: E402

Q = abi.METRIC_QUANTILE
TOP = 100


def host_route(h, W):
    """every retained window alone as rollup(j) - rollup(j - 1) on the host, grouped by node, IN p99: ms (host clock)"""
    import numpy as np
    import node_ref as nr
    from change_ref import row_keys
    t0 = time.perf_counter()
    prev = np.zeros(0, dtype=abi.EDGE_OUT)
    copied = 0
    for j in range(1, W + 1):
        cur = h.rollup(j)[0]
        copied += cur.nbytes
        pos = np.searchsorted(row_keys(cur), row_keys(prev))   # a rollup's rows are ascending; prev's keys are in cur
        d = cur.copy()
        for f in ("count", "err5xx", "lat_sum_ns", "hist"):
            d[f][pos] -= prev[f]
        nr.values(nr.group(d[d["count"] > 0]), abi.SIDE_IN, (Q, 0.99))
        prev = cur
    return round((time.perf_counter() - t0) * 1e3, 1), copied


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=12)
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--buffers", type=int, default=4)
    ap.add_argument("--windows", type=int, default=60)
    ap.add_argument("--factor", type=int, default=5)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("node_series_prof.py: no CUDA device")
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    result = {"card": card(), "cases": []}

    h, bufs, _ = handle_for(torch, stream, 10_000, a.events, a.buffers)
    h.submit_device(bufs[0], a.events)
    first = h.flush_device()[1]                                       # sizes the history
    W = a.windows
    h.window_history(W, W * (first + first // 2))
    tier_depth = W // a.factor
    h.window_history_tiers([(a.factor, tier_depth, tier_depth * 2 * first, 2 * first)])
    for w in range(W):
        h.submit_device(bufs[w % len(bufs)], a.events)
        h.flush_device()
    _, n, span = h.rollup_span_device(W)
    S, IN = abi.ROLLUP_SPAN, abi.SIDE_IN
    nodes = h.node_rows(S)
    services = nodes[nodes["type"] == abi.NODE_SVC][:10]
    result["rows"] = {"span": n, "span_windows": span["windows"], "window_rows": first, "nodes": len(nodes)}
    p99 = (Q, 0.99)
    three = (abi.METRIC_COUNT, abi.METRIC_ERR_RATE, p99)
    T = capi.Handle.trend
    cases = {
        f"a_all_nodes_x{W}_count_5xx_rate_p99_in": lambda: h.node_series_device(S, IN, 0, W, *three),
        f"b_10_services_x{W}_p99_in": lambda: h.node_series_keys_device(services, IN, 0, W, p99),
        f"c_top{TOP}_in_p99_zscore_x{W}": lambda: h.node_trends_top_device(S, IN, 0, W, p99,
                                                                         T(abi.TREND_ZSCORE, recent=5), TOP),
        f"d_all_nodes_tier1_x{tier_depth}_count_5xx_rate_p99_in": lambda: h.node_series_device(S, IN, 1, tier_depth,
                                                                                              *three),
    }
    ms = timed(torch, stream, h, cases, a.reps)
    for name, f in cases.items():
        info = f()[-1]
        c = {"case": name, "series_rows": info["edges"], "points": info["points"], "rows_in": info["rows_in"],
             "call_ms": ms[name], "kernels_ms": kernel_times(torch, h, [f], 5)}
        if "valid" in info:
            c.update(valid=info["valid"], above=info["above"])
        result["cases"].append(c)
        print(json.dumps(c), flush=True)
    # the scratch of (a): the pair arrays per entry row, and one compact node row per present slot
    present = int(h.node_series(S, IN, 0, W, abi.METRIC_COUNT)[1].sum())
    rows_in = result["cases"][0]["rows_in"]
    result["scratch_a"] = {"present_slots": present, "slot_rows_bytes": present * abi.NODE_OUT.itemsize,
                           "pair_bytes": rows_in * (8 + 8 + 4 + 4 + 4 + 4)}
    print(json.dumps(result["scratch_a"]), flush=True)
    host_ms, copied = host_route(h, W)
    result["host_route"] = {"ms": host_ms, "bytes_copied": copied}
    print(json.dumps(result["host_route"]), flush=True)
    h.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
