#!/usr/bin/env python
"""What does the top-row selection (docs/SPEC.md §16) add to the GNN pass? Two sources on one handle each:
  - the last flushed window of the bench.py config-2 topology (Topo(10_000), 100M device-resident events);
  - a window rollup of several 100M-event windows of the config-5 topology (Topo(1_000_000)), millions of rows.
For each, alz_gnn_score*_device and alz_gnn_top*_device for k = 10, 1000 and 100000 (min_score 0: every row
eligible) are called alternately, with device events around the whole call: median and min-max over --reps calls,
after two warm-up calls of each. The selection's cost is the top call minus the score call. A separate
torch.profiler pass per source gives the kernels of one score call and one top call (k = 1000).

Algorithmic bytes of the selection: 5 reads of the n scores (3 digit passes, the tie count, the emit) = 20 n B, the
candidates (m x 12 B written, sorted by CUB), and the gather (m x (296 + 4 + 4) B read and written).
Prints one JSON line with the card (nvidia-smi --query-gpu=name,power.limit,clocks.max.sm, read only).
Usage (GPU box): python scripts/gnn_top_prof.py [--reps R] [--big-windows W]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from alaz_b200 import abi, capi  # noqa: E402
from flush_prof import SEED, card  # noqa: E402

KS = (10, 1000, 100_000)


def summary(xs):
    return {"median": round(statistics.median(xs), 4), "min": round(min(xs), 4), "max": round(max(xs), 4),
            "n": len(xs)}


def handle_for(torch, stream, services, events, windows, edge_cap=None):
    """edge_cap: at most that many rows per window, so that the GNN state (1,792 B per row of max_edges, DESIGN §4)
    fits next to the history"""
    topo = capi.Topo(services, seed=SEED)
    max_pairs = max(1 << 20, int(1.6 * topo.n_edges) + (1 << 19))   # as bench.py sizes a single rank
    max_edges = max(1 << 20, int(2.3 * topo.n_edges))
    if edge_cap:
        max_edges = min(max_edges, edge_cap)
    h = capi.Handle(max_endpoints=4 * services, max_pairs=max_pairs, max_edges=max_edges, max_batch=1 << 22)
    h.set_stream(stream.cuda_stream)
    h.load_tables(topo.pod_ip, topo.svc_ip)
    bufs = []
    for k in range(windows):
        d = h.dev_alloc(events * 32)
        topo.fill_device(h, k * events, events, d)
        bufs.append(d)
    h.sync()
    return h, bufs, max_edges


def measure(torch, stream, h, score, top, reps):
    """score() / top(k) -> rows; alternated, device events around each call."""
    calls = [("score", score)] + [(f"top_k{k}", (lambda k=k: top(k))) for k in KS]
    for _ in range(2):
        for _, f in calls:
            f()
    h.sync()
    ms = {name: [] for name, _ in calls}
    for _ in range(reps):
        for name, f in calls:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            f()
            e1.record(stream)
            e1.synchronize()
            ms[name].append(e0.elapsed_time(e1))
    out = {name: summary(v) for name, v in ms.items()}
    base = statistics.median(ms["score"])
    for k in KS:
        out[f"top_k{k}"]["selection_ms"] = round(statistics.median(ms[f"top_k{k}"]) - base, 4)
    return out


def kernels(torch, h, score, top, out_dir, tag):
    """torch.profiler over 5 score calls, then 5 top calls (k = 1000): mean device us per call by kernel name."""
    from torch.profiler import ProfilerActivity, profile
    res = {}
    for name, f in (("score", score), ("top_k1000", lambda: top(1000))):
        f()
        h.sync()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                f()
            h.sync()
        per = {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            if t > 0 and not ev.key.startswith(("Memcpy", "Memset", "cuda")):
                per[ev.key[:90]] = round(t / 5, 2)
        res[name] = dict(sorted(per.items(), key=lambda kv: -kv[1]))
        prof.export_chrome_trace(os.path.join(out_dir, f"gnn_top_{tag}_{name}.pt.trace.json"))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--big-services", type=int, default=1_000_000)
    ap.add_argument("--big-events", type=int, default=100_000_000)
    ap.add_argument("--big-windows", type=int, default=4)
    ap.add_argument("--big-max-edges", type=int, default=1 << 23)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "gnn_top_prof"), help="profiler traces")
    a = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("gnn_top_prof.py: no CUDA device")
    os.makedirs(a.out, exist_ok=True)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    result = {"card": card(), "sources": []}

    def score_window(h):
        p, n = C.c_void_p(), C.c_size_t(0)
        h._ck(h.L.alz_gnn_score_device(h.h, C.byref(p), C.byref(n)), "alz_gnn_score_device")
        return n.value

    # config-2 window
    h, bufs, max_edges = handle_for(torch, stream, 10_000, 100_000_000, 1)
    h.submit_device(bufs[0], 100_000_000)
    n_rows = h.flush_device()[1]
    score = lambda: score_window(h)  # noqa: E731
    top = lambda k: h.gnn_top_device(k, 0.0)[3]  # noqa: E731
    r = {"source": "config-2 last window", "rows": n_rows, "max_edges": max_edges,
         "calls_ms": measure(torch, stream, h, score, top, a.reps), "kernels_us": kernels(torch, h, score, top, a.out, "c2")}
    result["sources"].append(r)
    print(json.dumps(r), flush=True)                                   # each source as soon as it is measured
    h.close()

    # config-5 topology: a window rollup of several windows
    h, bufs, max_edges = handle_for(torch, stream, a.big_services, a.big_events, a.big_windows, a.big_max_edges)
    h.submit_device(bufs[0], a.big_events)
    first = h.flush_device()[1]                                        # sizes the history; not retained
    h.window_history(a.big_windows, a.big_windows * (first + first // 2))
    per_window = []
    for d in bufs:
        h.submit_device(d, a.big_events)
        per_window.append(h.flush_device()[1])
    _, n_rows, info = h.rollup_device(a.big_windows)
    score = lambda: h.gnn_score_rollup_device(abi.ROLLUP_WINDOWS)[1]  # noqa: E731
    top = lambda k: h.gnn_top_rollup_device(abi.ROLLUP_WINDOWS, k, 0.0)[3]  # noqa: E731
    r = {"source": f"config-5 topology, window rollup of {info['windows']} windows of {a.big_events} events",
         "rows": n_rows, "rows_per_window": per_window, "max_edges": max_edges,
         "calls_ms": measure(torch, stream, h, score, top, a.reps), "kernels_us": kernels(torch, h, score, top, a.out, "c5")}
    result["sources"].append(r)
    h.close()
    for s in result["sources"]:
        n = s["rows"]
        s["selection_bytes"] = {f"k{k}": 20 * n + min(k, n) * (12 * 2 + 296 * 2 + 8) for k in KS}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
