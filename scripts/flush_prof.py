#!/usr/bin/env python
"""Where does the window flush of the bench.py config-2 step spend its device time?

Runs the flagship workload (Topo(10_000), 100M events per step, rotating resident windows, the handle sizes of
bench.py) under torch.profiler with CUDA activities and prints one JSON line:
  - mean device time per step of every kernel, memset and copy, by stable short name;
  - the idle gaps on the GPU between the end of the ingest kernel and the end of the last flush activity;
  - the live pair rows before the flush and the edges it emits;
  - the card (nvidia-smi --query-gpu=name,power.limit,clocks.max.sm, read only).
Tracing slows the host: take step times from bench.py, not from here. Usage (GPU box):
  python scripts/flush_prof.py [--steps K] [--trace-dir DIR]
"""
import argparse
import collections
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from alaz_b200 import capi  # noqa: E402

SEED = 0xA1A20001
GPU_CATS = ("kernel", "gpu_memset", "gpu_memcpy")


def short_name(ev):
    name = ev["name"]
    if ev["cat"] != "kernel":
        return name.split(" (")[0]
    name = re.sub(r"^void ", "", name)
    base = name.split("<")[0].split("(")[0]
    return base.replace("alz::", "").replace("(anonymous namespace)::", "")


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--services", type=int, default=10_000)
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--windows", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--trace-dir", default=None, help="keep the chrome trace there (default: a temporary directory)")
    a = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    if not torch.cuda.is_available():
        raise SystemExit("flush_prof.py: no CUDA device")
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
    # warm-up steps also count the rows (the stats call synchronises, so the profiled steps do without it)
    pair_rows, edges = [], []
    for k in range(a.warmup):
        h.submit_device(wins[k % a.windows], a.events)
        pair_rows.append(h.stats()["pairs_live"])
        edges.append(h.flush_device()[1])
    h.sync()
    torch.cuda.synchronize()

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(a.steps):   # as bench.py times a step: submit and flush back to back
            h.submit_device(wins[(a.warmup + k) % a.windows], a.events)
            h.flush_device()
        torch.cuda.synchronize()

    tdir = a.trace_dir or tempfile.mkdtemp(prefix="flush_prof_")
    os.makedirs(tdir, exist_ok=True)
    path = os.path.join(tdir, "flush_prof_trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        trace = json.load(f)
    evs = sorted((e for e in trace.get("traceEvents", []) if e.get("ph") == "X" and e.get("cat") in GPU_CATS),
                 key=lambda e: e["ts"])
    # one step = the ingest kernel and every GPU activity after it up to the next ingest kernel
    starts = [i for i, e in enumerate(evs) if "ingest_pairs" in e["name"]]
    if len(starts) != a.steps:
        raise SystemExit(f"flush_prof.py: found {len(starts)} ingest launches in the trace, expected {a.steps}")
    per = collections.defaultdict(float)
    calls = collections.defaultdict(int)
    gaps, spans = [], []
    for s, i0 in enumerate(starts):
        i1 = starts[s + 1] if s + 1 < len(starts) else len(evs)
        step = evs[i0:i1]
        for e in step[1:]:
            per[short_name(e)] += e["dur"]
            calls[short_name(e)] += 1
        end = step[0]["ts"] + step[0]["dur"]
        gap = 0.0
        for e in step[1:]:
            gap += max(0.0, e["ts"] - end)
            end = max(end, e["ts"] + e["dur"])
        gaps.append(gap)
        spans.append(end - (step[0]["ts"] + step[0]["dur"]))
    busy = sum(per.values()) / a.steps
    out = {
        "card": card(),
        "steps": a.steps,
        "pair_rows_live": pair_rows,
        "edges": edges,
        "flush_us_per_step": {k: round(v / a.steps, 2) for k, v in sorted(per.items(), key=lambda kv: -kv[1])},
        "launches_per_step": {k: v // a.steps for k, v in calls.items()},
        "flush_busy_us": round(busy, 2),
        "flush_idle_gaps_us": round(sum(gaps) / a.steps, 2),
        "flush_span_us": round(sum(spans) / a.steps, 2),
        "trace": path,
    }
    print(json.dumps(out))
    h.close()


if __name__ == "__main__":
    main()
