#!/usr/bin/env python
"""What do tiers cost on the bench.py config-2 topology? Tiers (60, 60): a tier-1 entry is 60 windows, a tier-2
entry 60 tier-1 entries.

Streams windows as bench.py does (Topo(10_000), 100M device-resident events per step, a different window of the
stream each step) into one handle, then prints one JSON line:
  - the flush with tiers on and off, alternated in blocks on the same handle (each on-block configures the tiers
    afresh and runs one whole tier-1 block: 59 flushes that close no block, one that closes it), device-event time;
  - in a separate pass under torch.profiler, the device time of the merge (tier_match_kernel, the scan,
    tier_merge_kernel) per flush that closes no block, and the rate the bytes it must move give: 296 B x (block rows
    read + window rows read + block rows written) + 8 B keys of each, with the block at the size it closes at;
  - alz_window_rollup_tier_device of tier 1 for k = 1 and 60, once 60 tier-1 entries are retained;
  - the card (nvidia-smi --query-gpu=name,power.limit,clocks.max.sm, read only).
Usage (GPU box): python scripts/tier_prof.py [--blocks B] [--reps R] [--trace-dir DIR]
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
from alaz_b200 import capi  # noqa: E402
from flush_prof import GPU_CATS, SEED, card, short_name  # noqa: E402

ROW = 296
MERGE_KERNELS = ("tier_match_kernel", "tier_merge_kernel", "DeviceScan")


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
    ap.add_argument("--blocks", type=int, default=4, help="on/off blocks of the flush comparison")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--trace-dir", default=None)
    a = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    if not torch.cuda.is_available():
        raise SystemExit("tier_prof.py: no CUDA device")
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
        """one step as bench.py runs it; returns the device-event time of the flush alone, ms, and its rows"""
        h.submit_device(wins[step[0] % a.windows], a.events)
        step[0] += 1
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        n = h.flush_device()[1]
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1), n

    edges = [flush_once()[1] for _ in range(4)]                      # warm-up, tiers off
    block_rows = max(edges) + max(edges) // 4
    tiers = [(a.factor, a.depth, a.depth * block_rows, block_rows), (a.factor, 2, 2 * block_rows, block_rows)]

    # ---- flush with tiers on (closing / not closing a block) and off, alternated on one handle
    on_open, on_close, off = [], [], []
    for _ in range(a.blocks):
        h.window_history_tiers(tiers)
        for i in range(a.factor):
            ms, _ = flush_once()
            (on_close if i == a.factor - 1 else on_open).append(ms)
        h.window_history_tiers([])
        off += [flush_once()[0] for _ in range(16)]

    # ---- fill tier 1: depth entries of factor windows each
    h.window_history_tiers(tiers)
    for _ in range(a.depth * a.factor):
        flush_once()
    h.sync()
    st1 = h.tier_state(1)

    # ---- the merge of one window into the open tier-1 block, traced (tracing slows the host: times above are
    # without it). The open block has just been emptied; run into it so that it holds most of its rows.
    for _ in range(a.factor // 2):
        flush_once()
    n_prof = min(8, a.factor // 2 - 2)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n_prof):
            flush_once()
        torch.cuda.synchronize()
    tdir = a.trace_dir or tempfile.mkdtemp(prefix="tier_prof_")
    os.makedirs(tdir, exist_ok=True)
    path = os.path.join(tdir, "tier_prof.pt.trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        trace = json.load(f)
    per = collections.defaultdict(float)
    for e in trace.get("traceEvents", []):
        if e.get("ph") == "X" and e.get("cat") in GPU_CATS:
            per[short_name(e)] += e["dur"]
    merge_us = {k: round(v / n_prof, 2) for k, v in per.items() if any(m in k for m in MERGE_KERNELS)}

    # ---- tier rollups
    rollups = []
    for k in (1, a.depth):
        dev_ms = []
        for rep in range(a.reps + 2):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            _, u, info = h.rollup_tier_device(1, k)
            e1.record(stream)
            e1.synchronize()
            if rep >= 2:                                               # the first calls size the scratch
                dev_ms.append(e0.elapsed_time(e1))
        rollups.append({"tier": 1, "k": k, "windows": info["windows"], "N": info["rows_in"], "U": u,
                        "device_ms": summary(dev_ms)})
    u1 = rollups[0]["U"]                                               # rows of one closed tier-1 block
    w = statistics.median(edges)
    merge_bytes = ROW * (u1 + w + u1) + 8 * (u1 + w + u1)
    merge_total_us = sum(merge_us.values())

    out = {
        "card": card(),
        "edges_per_window": edges,
        "tiers": tiers,
        "tier1_state": st1,
        "flush_ms_tiers_off": summary(off),
        "flush_ms_tiers_on_no_close": summary(on_open),
        "flush_ms_tiers_on_close": summary(on_close),
        "merge_us_per_flush": merge_us,
        "merge_us_total": round(merge_total_us, 2),
        "merge_bytes_at_closed_block_size": int(merge_bytes),
        "merge_GBps": round(merge_bytes / (merge_total_us * 1e-6) / 1e9, 1) if merge_total_us else None,
        "rollups": rollups,
        "trace": path,
    }
    print(json.dumps(out))
    h.close()


if __name__ == "__main__":
    main()
