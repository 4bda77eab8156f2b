#!/usr/bin/env python
"""What does a rollup of retained windows cost on the bench.py config-2 topology, and what does retaining them add
to a flush?

Streams windows as bench.py does (Topo(10_000), 100M device-resident events per step, a different window of the
stream each step) into a handle with a history of depth 64, then prints one JSON line:
  - alz_window_rollup_device for k in {1, 2, 8, 60}: device-event time and host time per call over --reps calls,
    source rows N, output rows U, the bytes the algorithm needs (296 B x (N + U) of rows; the radix sort's
    12 B x N read and written once per 8-bit pass over the 64-bit key) and the rate the row bytes give;
  - the flush with the history on and off, alternated in blocks: the difference is the append;
  - in a separate pass under torch.profiler, the device time of every kernel and copy of a k = 60 rollup;
  - the card (nvidia-smi --query-gpu=name,power.limit,clocks.max.sm, read only).
Usage (GPU box): python scripts/rollup_prof.py [--reps R] [--trace-dir DIR]
"""
import argparse
import collections
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from alaz_b200 import capi  # noqa: E402
from flush_prof import GPU_CATS, SEED, card, short_name  # noqa: E402

ROW = 296
SORT_PASSES = 8          # 64-bit keys, 8 bits per pass
SORT_ITEM = 12           # key + arena row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--services", type=int, default=10_000)
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--windows", type=int, default=4)
    ap.add_argument("--depth", type=int, default=64)
    ap.add_argument("--ks", default="1,2,8,60")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--blocks", type=int, default=4, help="on/off blocks of the flush comparison")
    ap.add_argument("--trace-dir", default=None)
    a = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    if not torch.cuda.is_available():
        raise SystemExit("rollup_prof.py: no CUDA device")
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
        """one step as bench.py runs it; returns the device-event time of the flush alone, ms"""
        h.submit_device(wins[step[0] % a.windows], a.events)
        step[0] += 1
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        n = h.flush_device()[1]
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1), n

    edges = [flush_once()[1] for _ in range(4)]                      # warm-up, history off
    arena_rows = a.depth * (max(edges) + max(edges) // 8)

    # ---- the append: flush with the history on and off, alternated
    on, off = [], []
    for _ in range(a.blocks):
        h.window_history(a.depth, arena_rows)
        flush_once()
        on += [flush_once()[0] for _ in range(4)]
        h.window_history(0, 0)
        flush_once()
        off += [flush_once()[0] for _ in range(4)]

    # ---- rollups
    h.window_history(a.depth, arena_rows)
    for _ in range(a.depth):
        flush_once()
    h.sync()
    rollups = []
    for k in (int(x) for x in a.ks.split(",")):
        dev_ms, host_ms = [], []
        for rep in range(a.reps + 2):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record(stream)
            _, u, info = h.rollup_device(k)
            e1.record(stream)
            e1.synchronize()
            t1 = time.perf_counter()
            if rep >= 2:                                               # the first calls size the scratch
                dev_ms.append(e0.elapsed_time(e1))
                host_ms.append((t1 - t0) * 1e3)
        n = info["rows_in"]
        row_bytes = ROW * (n + u)
        med = statistics.median(dev_ms)
        rollups.append({
            "k": k, "windows": info["windows"], "N": n, "U": u,
            "device_ms_median": round(med, 4), "device_ms_min": round(min(dev_ms), 4),
            "device_ms_max": round(max(dev_ms), 4), "host_ms_median": round(statistics.median(host_ms), 4),
            "row_bytes": row_bytes, "sort_bytes": 2 * SORT_ITEM * n * SORT_PASSES,
            "row_GBps_at_median": round(row_bytes / (med * 1e-3) / 1e9, 1),
        })

    # ---- per-kernel split of a k = 60 rollup, traced (tracing slows the host: times above are without it)
    kp = max(int(x) for x in a.ks.split(","))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            h.rollup_device(kp)
        torch.cuda.synchronize()
    tdir = a.trace_dir or tempfile.mkdtemp(prefix="rollup_prof_")
    os.makedirs(tdir, exist_ok=True)
    path = os.path.join(tdir, "rollup_prof.pt.trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        trace = json.load(f)
    per = collections.defaultdict(float)
    for e in trace.get("traceEvents", []):
        if e.get("ph") == "X" and e.get("cat") in GPU_CATS:
            per[short_name(e)] += e["dur"]

    out = {
        "card": card(),
        "edges_per_window": edges,
        "depth": a.depth, "arena_rows": arena_rows,
        "flush_ms_history_on": {"median": round(statistics.median(on), 4), "min": round(min(on), 4),
                                "max": round(max(on), 4), "n": len(on)},
        "flush_ms_history_off": {"median": round(statistics.median(off), 4), "min": round(min(off), 4),
                                 "max": round(max(off), 4), "n": len(off)},
        "rollups": rollups,
        "rollup_k%d_us_per_call" % kp: {k: round(v / 3, 2) for k, v in sorted(per.items(), key=lambda kv: -kv[1])},
        "trace": path,
    }
    print(json.dumps(out))
    h.close()


if __name__ == "__main__":
    main()
