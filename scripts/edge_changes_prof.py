#!/usr/bin/env python
"""What does the change list against a pinned baseline (docs/SPEC.md §18) cost? At bench.py config-2 sizes
(Topo(10_000), --events device-resident events per window, --buffers distinct event buffers taken in turn): the window
history keeps 64 windows, a span rollup of 60 windows is pinned, and a span rollup of the last 5 windows is compared
against it, by p99, by 5xx rate and by count, as the full list (alz_edge_changes_device) and as the top 100
(alz_edge_changes_top_device, min_change -inf).

Per call: device events around the whole call, median and min-max over --reps after two warm-ups, calls alternated.
Per kernel: device time from torch.profiler over the same calls, summed per kernel name and divided by the calls.
Bytes the join must move, from the row counts (n_s source rows, n_b baseline rows, L listed records):
  keys    16 B read + 8 B written per source row
  match   8 B per row of either side, plus the lower-bound probes (not counted), 12 B written per row
  scans   4 B read + 4 B written per row of either side
  values  the §17 pass: 256 B (quantile) or 24 B (sums) read and 8 B written per row of either side
  emit    per row of either side: 16 B of its row, 12 B of flags and scans, 8 B of value; 48 B (+ 8 B for the top
          call) written per listed record
and the share of 3.35 TB/s (the H100 SXM's HBM3 peak) that this gives over the whole call's median.
Prints one JSON line per call group and a last one with everything, with the card (name, power limit, SM clock).
Usage (GPU box): python scripts/edge_changes_prof.py [--reps R] [--events N] [--buffers B]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from alaz_b200 import abi  # noqa: E402
from edge_top_prof import timed  # noqa: E402
from flush_prof import card  # noqa: E402
from gnn_top_prof import handle_for  # noqa: E402

PEAK_TBS = 3.35
Q = abi.METRIC_QUANTILE
METRICS = (("p99", (Q, 0.99), 256), ("err_rate", abi.METRIC_ERR_RATE, 24), ("count", abi.METRIC_COUNT, 24))


def join_bytes(n_s, n_b, listed, value_bytes, top):
    n = n_s + n_b
    return (n_s * 24 + n * (8 + 12) + n * 8 + n * (value_bytes + 8) + n * (16 + 12 + 8) +
            listed * (48 + (8 if top else 0)))


def kernel_times(torch, h, calls, reps):
    """device ms per call of every kernel the calls launch (torch.profiler), by kernel name"""
    from torch.profiler import ProfilerActivity, profile
    h.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            for f in calls:
                f()
        h.sync()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = getattr(e, "cuda_time_total", 0)
        if t:
            out[e.key[:80]] = round(t / 1000.0 / reps, 4)
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--buffers", type=int, default=4)
    ap.add_argument("--base-windows", type=int, default=60)
    ap.add_argument("--source-windows", type=int, default=5)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("edge_changes_prof.py: no CUDA device")
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    result = {"card": card(), "groups": []}

    h, bufs, _ = handle_for(torch, stream, 10_000, a.events, a.buffers)
    h.submit_device(bufs[0], a.events)
    first = h.flush_device()[1]                                       # sizes the history
    depth = a.base_windows + a.source_windows - 1
    h.window_history(depth, depth * (first + first // 2))
    for w in range(a.base_windows):
        h.submit_device(bufs[w % len(bufs)], a.events)
        h.flush_device()
    _, n_b, info_b = h.rollup_span_device(a.base_windows)
    pinned = h.baseline_pin(abi.ROLLUP_SPAN)
    for w in range(a.source_windows):
        h.submit_device(bufs[(w + 1) % len(bufs)], a.events)
        h.flush_device()
    _, n_s, info_s = h.rollup_span_device(a.source_windows)
    result["rows"] = {"source": n_s, "source_windows": info_s["windows"], "baseline": n_b,
                      "baseline_windows": pinned["windows"]}
    S = abi.ROLLUP_SPAN
    for name, spec, vb in METRICS:
        listed = h.edge_changes_device(spec, abi.CHANGE_DELTA, abi.PRESENT_ALL, S)[1]
        calls = {f"list_{name}": lambda spec=spec: h.edge_changes_device(spec, abi.CHANGE_DELTA, abi.PRESENT_ALL, S),
                 f"top100_{name}": lambda spec=spec: h.edge_changes_top_device(spec, 100, float("-inf"),
                                                                              abi.CHANGE_DELTA, abi.PRESENT_ALL, S)}
        ms = timed(torch, stream, h, calls, a.reps)
        g = {"metric": name, "listed": listed, "calls_ms": ms, "kernels_ms": {}, "bytes": {}, "share_of_peak": {}}
        for cname, f in calls.items():
            top = cname.startswith("top")
            g["kernels_ms"][cname] = kernel_times(torch, h, [f], 5)
            b = join_bytes(n_s, n_b, listed, vb, top)
            g["bytes"][cname] = b
            g["share_of_peak"][cname] = round(b / (ms[cname]["median"] * 1e-3) / (PEAK_TBS * 1e12), 4)
        result["groups"].append(g)
        print(json.dumps(g), flush=True)
    h.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
