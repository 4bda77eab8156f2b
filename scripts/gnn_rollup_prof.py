#!/usr/bin/env python
"""What does the GNN pass over a rollup cost on the bench.py config-2 topology? The set-up of scripts/span_prof.py:
window history of depth 64, tiers (60, 60), so a tier-1 entry is 60 windows (a minute of one-second windows) and 60
of them are an hour.

Streams windows as bench.py does (Topo(10_000), 100M device-resident events per step, a different window of the
stream each step) into one handle until tier 1 retains `depth` entries and its open block holds `open` windows,
then times, with device events around the whole call, each of:
  - alz_gnn_score_device on the last flushed window;
  - alz_gnn_score_rollup_device after a window rollup of k = 1 and 60;
  - after a tier-1 rollup of 1, 15 and 60 entries;
  - after a 900-window span (ALZ_SPAN_AT_LEAST).
Every shape is scored twice before it is timed (the first pass over a rollup above max_edges grows the GNN state).
The rollup itself is not timed. Prints one JSON line with the rows, the nodes and the card
(nvidia-smi --query-gpu=name,power.limit,clocks.max.sm, read only).
Usage (GPU box): python scripts/gnn_rollup_prof.py [--reps R]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from alaz_b200 import abi, capi  # noqa: E402
from flush_prof import SEED, card  # noqa: E402


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
    a = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("gnn_rollup_prof.py: no CUDA device")
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

    def node_count():
        n = C.c_size_t(0)
        rc = h.L.alz_gnn_nodes(h.h, None, None, 0, C.byref(n))
        assert rc in (abi.OK, abi.E_CAPACITY), rc
        return n.value

    def timed(score):
        for _ in range(2):                                             # warm-up: the first pass may grow the state
            score()
        h.sync()
        dev_ms, n = [], 0
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            _, n = score()
            e1.record(stream)
            e1.synchronize()
            dev_ms.append(e0.elapsed_time(e1))
        return {"rows": n, "nodes": node_count(), "device_ms": summary(dev_ms)}

    def score_window():
        p, n = C.c_void_p(), C.c_size_t(0)
        h._ck(h.L.alz_gnn_score_device(h.h, C.byref(p), C.byref(n)), "alz_gnn_score_device")
        return p.value, n.value

    results = [dict({"call": "alz_gnn_score_device", "what": "last window"}, **timed(score_window))]
    shapes = [("window", 1, lambda: h.rollup_device(1)), ("window", 60, lambda: h.rollup_device(60)),
              ("tier1", 1, lambda: h.rollup_tier_device(1, 1)), ("tier1", 15, lambda: h.rollup_tier_device(1, 15)),
              ("tier1", a.depth, lambda: h.rollup_tier_device(1, a.depth)),
              ("span_at_least", 900, lambda: h.rollup_span_device(900, abi.SPAN_AT_LEAST))]
    for name, k, rollup in shapes:
        _, n_rows, info = rollup()
        kind = {"window": abi.ROLLUP_WINDOWS, "tier1": abi.ROLLUP_TIER}.get(name, abi.ROLLUP_SPAN)
        r = timed(lambda: h.gnn_score_rollup_device(kind))
        assert r["rows"] == n_rows
        r.update({"call": "alz_gnn_score_rollup_device", "what": f"{name} {k}", "windows": info["windows"]})
        results.append(r)

    out = {
        "card": card(),
        "edges_per_window": edges,
        "max_edges": max_edges,
        "history_depth": a.history,
        "tiers": tiers,
        "windows": h.stats()["windows"],
        "gnn": results,
    }
    print(json.dumps(out))
    h.close()


if __name__ == "__main__":
    main()
