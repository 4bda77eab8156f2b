#!/usr/bin/env python
"""What does a span rollup cost on the bench.py config-2 topology? Window history of depth 64, tiers (60, 60): a
tier-1 entry is 60 windows, a tier-2 entry 60 tier-1 entries.

Streams windows as bench.py does (Topo(10_000), 100M device-resident events per step, a different window of the
stream each step) into one handle until tier 1 retains `depth` entries and its open block holds `open` windows,
then prints one JSON line:
  - alz_window_rollup_span_device for N = 60, 900 and 3600 in both modes, device-event time of the whole call (which
    includes the host's two waits: the plan's read of the open blocks, and the count of distinct rows), with the
    pieces it took;
  - alz_window_rollup_tier_device of tier 1 for k = 1, 15 and 60 (the same windows, without the open block);
  - in a separate pass under torch.profiler, the device-time split of the N = 900 span;
  - the card (nvidia-smi --query-gpu=name,power.limit,clocks.max.sm, read only).
Usage (GPU box): python scripts/span_prof.py [--reps R] [--trace-dir DIR]
"""
import argparse
import collections
import json
import os
import statistics
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from alaz_b200 import abi, capi  # noqa: E402
from flush_prof import GPU_CATS, SEED, card, short_name  # noqa: E402


def summary(xs):
    return {"median": round(statistics.median(xs), 4), "min": round(min(xs), 4), "max": round(max(xs), 4),
            "n": len(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--services", type=int, default=10_000)
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--windows", type=int, default=4)
    ap.add_argument("--factor", type=int, default=60)
    ap.add_argument("--depth", type=int, default=60, help="tier-1 entries retained")
    ap.add_argument("--history", type=int, default=64, help="depth of the window history")
    ap.add_argument("--open", type=int, default=30, help="windows in tier 1's open block when measured")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--trace-dir", default=None)
    a = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    if not torch.cuda.is_available():
        raise SystemExit("span_prof.py: no CUDA device")
    topo = capi.Topo(a.services, seed=SEED)
    max_pairs = max(1 << 20, int(1.6 * topo.n_edges) + (1 << 19))   # as bench.py sizes a single rank
    max_edges = max(1 << 20, int(2.3 * topo.n_edges))
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    h = capi.Handle(max_endpoints=4 * a.services, max_pairs=max_pairs, max_edges=max_edges, max_batch=1 << 22)
    h.set_stream(stream.cuda_stream)
    h.load_tables(topo.pod_ip, topo.svc_ip)
    wins = []
    for k in range(a.windows):
        d = h.dev_alloc(a.events * 32)
        topo.fill_device(h, k * a.events, a.events, d)
        wins.append(d)
    h.sync()
    step = [0]

    def flush_once():
        h.submit_device(wins[step[0] % a.windows], a.events)
        step[0] += 1
        return h.flush_device()[1]

    edges = [flush_once() for _ in range(4)]                         # warm-up, nothing retained
    block_rows = max(edges) + max(edges) // 4
    tiers = [(a.factor, a.depth, a.depth * block_rows, block_rows), (a.factor, 2, 2 * block_rows, block_rows)]
    h.window_history(a.history, a.history * block_rows)
    h.window_history_tiers(tiers)
    for _ in range(a.depth * a.factor + a.open):
        flush_once()
    h.sync()

    def timed(call):
        dev_ms, last = [], None
        for rep in range(a.reps + 2):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            last = call()
            e1.record(stream)
            e1.synchronize()
            if rep >= 2:                                               # the first calls size the scratch
                dev_ms.append(e0.elapsed_time(e1))
        return dev_ms, last

    spans = []
    for N in (60, 900, 3600):
        for mode, name in ((abi.SPAN_AT_MOST, "at_most"), (abi.SPAN_AT_LEAST, "at_least")):
            dev_ms, (_, u, info) = timed(lambda: h.rollup_span_device(N, mode))
            spans.append({"N": N, "mode": name, "windows": info["windows"], "rows_in": info["rows_in"], "U": u,
                          "entries": info["entries"], "open_blocks": info["open_blocks"],
                          "device_ms": summary(dev_ms)})
    tier_rollups = []
    for k in (1, 15, a.depth):
        dev_ms, (_, u, info) = timed(lambda: h.rollup_tier_device(1, k))
        tier_rollups.append({"tier": 1, "k": k, "windows": info["windows"], "rows_in": info["rows_in"], "U": u,
                             "device_ms": summary(dev_ms)})

    # ---- the split of one span under torch.profiler (tracing slows the host: the times above are without it)
    n_prof = 3
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n_prof):
            h.rollup_span_device(900, abi.SPAN_AT_LEAST)
        torch.cuda.synchronize()
    tdir = a.trace_dir or tempfile.mkdtemp(prefix="span_prof_")
    os.makedirs(tdir, exist_ok=True)
    path = os.path.join(tdir, "span_prof.pt.trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        trace = json.load(f)
    per = collections.defaultdict(float)
    for e in trace.get("traceEvents", []):
        if e.get("ph") == "X" and e.get("cat") in GPU_CATS:
            per[short_name(e)] += e["dur"]
    split_us = {k: round(v / n_prof, 2) for k, v in sorted(per.items(), key=lambda kv: -kv[1])}

    out = {
        "card": card(),
        "edges_per_window": edges,
        "history_depth": a.history,
        "tiers": tiers,
        "windows": h.stats()["windows"],
        "tier1_state": h.tier_state(1),
        "spans": spans,
        "tier_rollups": tier_rollups,
        "span_900_at_least_split_us": split_us,
        "trace": path,
    }
    print(json.dumps(out))
    h.close()


if __name__ == "__main__":
    main()
