#!/usr/bin/env python
"""What do node changes against a pinned baseline (docs/SPEC.md §23) cost? At bench.py config-2 sizes
(Topo(10_000), --events device-resident events per window, --buffers distinct event buffers taken in turn): the window
history keeps --base-windows + --source-windows windows; a window rollup of the first --base-windows windows is pinned,
and a span rollup of the last --source-windows windows is compared against it. Timed, as device calls:
  list_in_p99 / list_in_count     alz_node_changes_device, IN side, DELTA, every presence
  top100_in_p99 / top100_in_count alz_node_changes_top_device, the same, top 100 with min_change -inf
  first_after_pin_in_p99          the list call right after a re-pin of the same baseline, so it groups the baseline's
                                  rows too (each rep pins, waits, then times the call alone)
Per call: device events around the whole call, median and min-max over --reps after two warm-ups, calls alternated.
Per kernel: device time from torch.profiler over the same calls, summed per kernel name and divided by the calls.
Once, for scale, the host alternative: both sides' rows copied to the host, grouped by node, every IN side's p99
computed and the two node lists joined in numpy (tests/node_change_ref.py).
Prints one JSON line per case and a last one with everything, with the card (name, power limit, SM clock now and max).
Usage (GPU box): python scripts/node_changes_prof.py [--reps R] [--events N] [--buffers B]
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
from gnn_top_prof import handle_for, summary  # noqa: E402

Q = abi.METRIC_QUANTILE
TOP = 100
IN, S, WIN = abi.SIDE_IN, abi.ROLLUP_SPAN, abi.ROLLUP_WINDOWS
ALL, DELTA = abi.PRESENT_ALL, abi.CHANGE_DELTA


def first_after_pin(torch, stream, h, spec, reps):
    """device ms of the list call right after a re-pin, which groups the baseline's rows again"""
    ms = []
    for _ in range(reps + 2):
        h.baseline_pin(WIN)
        h.sync()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        h.node_changes_device(IN, spec, DELTA, ALL, S)
        e1.record(stream)
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return summary(ms[2:])


def host_alternative(h, src, base, reps=3):
    """(ms per call, host clock): both sides' rows copied to the host, grouped, IN p99 of every node, joined"""
    import node_change_ref as ncr
    (ps, ns, ws), (pb, nb, wb) = src, base
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        rs, rb = h.d2h(ps, ns, abi.EDGE_OUT), h.d2h(pb, nb, abi.EDGE_OUT)
        ncr.changes(rs, rb, IN, (Q, 0.99), DELTA, ALL, ws, wb)
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
        raise SystemExit("node_changes_prof.py: no CUDA device")
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    result = {"card": card(), "cases": []}

    h, bufs, _ = handle_for(torch, stream, 10_000, a.events, a.buffers)
    h.submit_device(bufs[0], a.events)
    first = h.flush_device()[1]                                       # sizes the history
    depth = a.base_windows + a.source_windows
    h.window_history(depth, depth * (first + first // 2))
    for w in range(a.base_windows):
        h.submit_device(bufs[w % len(bufs)], a.events)
        h.flush_device()
    pb, nb, _ = h.rollup_device(a.base_windows)                       # stays the last window rollup's rows
    pinned = h.baseline_pin(WIN)
    for w in range(a.source_windows):
        h.submit_device(bufs[(w + 1) % len(bufs)], a.events)
        h.flush_device()
    ps, ns, info_s = h.rollup_span_device(a.source_windows)
    p99 = (Q, 0.99)
    _, listed, ci = h.node_changes_device(IN, p99, DELTA, ALL, S)
    result["rows"] = {"source": ns, "source_windows": info_s["windows"], "baseline": nb,
                      "baseline_windows": pinned["windows"], "source_nodes_in": ci["source_rows"],
                      "baseline_nodes_in": ci["base_rows"], "listed_in": listed, "both": ci["both"],
                      "added": ci["added"], "gone": ci["gone"]}
    print(json.dumps(result["rows"]), flush=True)
    cases = {}
    for name, spec in (("p99", p99), ("count", abi.METRIC_COUNT)):
        cases[f"list_in_{name}"] = lambda spec=spec: h.node_changes_device(IN, spec, DELTA, ALL, S)
        cases[f"top{TOP}_in_{name}"] = lambda spec=spec: h.node_changes_top_device(IN, spec, TOP, float("-inf"),
                                                                                   DELTA, ALL, S)
    ms = timed(torch, stream, h, cases, a.reps)
    for name, f in cases.items():
        c = {"case": name, "call_ms": ms[name], "kernels_ms": kernel_times(torch, h, [f], 5)}
        result["cases"].append(c)
        print(json.dumps(c), flush=True)
    c = {"case": "first_after_pin_in_p99", "call_ms": first_after_pin(torch, stream, h, p99, a.reps)}
    h.baseline_pin(WIN)
    h.sync()
    c["kernels_ms"] = kernel_times(torch, h, [lambda: (h.baseline_pin(WIN),
                                                       h.node_changes_device(IN, p99, DELTA, ALL, S))], 5)
    c["kernels_ms_note"] = "includes the pin's copy and key kernel"
    result["cases"].append(c)
    print(json.dumps(c), flush=True)
    host = host_alternative(h, (ps, ns, info_s["windows"]), (pb, nb, pinned["windows"]))
    result["host_alternative_ms"] = host
    print(json.dumps({"host_alternative_ms": host}), flush=True)
    h.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
