#!/usr/bin/env python
"""What does an edge series (docs/SPEC.md §19) cost? At bench.py config-2 sizes (Topo(10_000), --events device-resident
events per window, --buffers distinct event buffers taken in turn): the window history keeps 60 windows and a tier of
factor 5 keeps 12 entries. The source is a span rollup of the last 60 windows. Timed, as device calls:
  (a) every row of the span x the 60 history points, for {count}, {p99} and {p50, p99, 5xx rate}
  (b) 100 caller keys x the 60 history points, for {p99}
  (c) every row of the span x the tier's 12 points, for {p99}
and once, for scale, the host alternative: point j as rollup(j) - rollup(j - 1), i.e. 60 window rollups of growing
size copied to the host (host clock; the subtraction itself not counted).

Per call: device events around the whole call, median and min-max over --reps after two warm-ups, calls alternated.
Per kernel: device time from torch.profiler over the same calls, summed per kernel name and divided by the calls.
Bytes a series must move, from the row counts (n series rows, u distinct keys, E entry rows read, P points, H present
slots, nm metrics):
  keys    a source: 16 B read + 8 B written per row; caller keys: 8 B per distinct key and 4 B per row copied in
  match   4 B per slot of u x P set, 16 B read per entry row (the lower-bound probes into the keys, L2-resident, are
          not counted), 4 B written per hit
  values  4 B (+ 4 B of map) read per slot, 256 B (quantile) or 24 B (sums) per present slot, 8 nm + 1 B written per
          slot
and the share of 3.35 TB/s (the H100 SXM's HBM3 peak) that this gives over the whole call's median.
Prints one JSON line per case and a last one with everything, with the card (name, power limit, SM clock now and max).
Usage (GPU box): python scripts/edge_series_prof.py [--reps R] [--events N] [--buffers B]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from alaz_b200 import abi, capi  # noqa: E402
from edge_changes_prof import kernel_times  # noqa: E402
from edge_top_prof import timed  # noqa: E402
from gnn_top_prof import handle_for  # noqa: E402

PEAK_TBS = 3.35
Q = abi.METRIC_QUANTILE
SETS = (("count", [abi.METRIC_COUNT]), ("p99", [(Q, 0.99)]),
        ("p50_p99_err_rate", [(Q, 0.5), (Q, 0.99), abi.METRIC_ERR_RATE]))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def series_bytes(n, u, rows_in, P, present, specs, source):
    quant = any(isinstance(s, tuple) for s in specs)
    slots = n * P
    keys = n * 24 if source else u * 8 + n * 4
    match = u * P * 4 + rows_in * 16 + present * 4
    values = slots * (4 + (0 if source else 4)) + present * (256 if quant else 24) + slots * (8 * len(specs) + 1)
    return keys + match + values


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--buffers", type=int, default=4)
    ap.add_argument("--windows", type=int, default=60)
    ap.add_argument("--factor", type=int, default=5)
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("edge_series_prof.py: no CUDA device")
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
    result["rows"] = {"span": n, "span_windows": span["windows"], "window_rows": first}
    S = abi.ROLLUP_SPAN
    rng = np.random.default_rng(5)
    span_rows = h.d2h(h.rollup_span_device(W)[0], n, abi.EDGE_OUT)
    keys = capi.Handle.edge_ends(span_rows[np.sort(rng.choice(n, 100, replace=False))])

    cases = []
    for name, specs in SETS:
        cases.append((f"a_rows_x{W}_{name}", specs, True, 0, W,
                      lambda specs=specs: h.edge_series_device(S, 0, W, *specs)))
    cases.append((f"b_keys100_x{W}_p99", [(Q, 0.99)], False, 0, W,
                  lambda: h.edge_series_keys_device(keys, 0, W, (Q, 0.99))))
    cases.append(("c_rows_x_tier1_p99", [(Q, 0.99)], True, 1, tier_depth,
                  lambda: h.edge_series_device(S, 1, tier_depth, (Q, 0.99))))
    for name, specs, source, tier, k, f in cases:
        pv, pp, rows, P, pts, info = f()
        present = int(h.d2h(pp, rows * P, np.uint8).sum()) if rows * P else 0
        ms = timed(torch, stream, h, {name: f}, a.reps)[name]
        u = rows if source else len(np.unique(keys.view(np.uint64).reshape(-1, 2), axis=0))
        b = series_bytes(rows, u, info["rows_in"], P, present, specs, source)
        c = {"case": name, "rows": rows, "points": P, "entry_rows": info["rows_in"], "present_slots": present,
             "call_ms": ms, "kernels_ms": kernel_times(torch, h, [f], 5), "bytes": b,
             "share_of_peak": round(b / (ms["median"] * 1e-3) / (PEAK_TBS * 1e12), 4)}
        result["cases"].append(c)
        print(json.dumps(c), flush=True)

    # the host alternative, once: W window rollups of growing size, each copied to the host
    h.sync()
    t0 = time.perf_counter()
    moved = 0
    for j in range(1, W + 1):
        rows, _ = h.rollup(j)
        moved += rows.nbytes
    host = {"case": "host_differencing_rollups", "ms": round((time.perf_counter() - t0) * 1e3, 1),
            "bytes_copied": moved}
    result["cases"].append(host)
    print(json.dumps(host), flush=True)
    h.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
