#!/usr/bin/env python
"""What do the edge metrics and the top edges by a metric (docs/SPEC.md §17) cost, and what do they save? Two sources:
  - the last flushed window of the bench.py config-2 topology (Topo(10_000), 100M device-resident events);
  - a window rollup of several 100M-event windows of the config-5 topology (Topo(1_000_000)), millions of rows.
Calls, alternated, device events around each whole call, median and min-max over --reps after two warm-ups:
  - alz_edge_metrics*_device with {p50, p99, 5xx rate};
  - alz_edge_top*_device by p99 and by 5xx count at k = 10, 1000 and 100000 (min_value 0: every row eligible);
  - the host alternative on the window: copy every row to the host and rank by p99 in numpy (host clock);
  - on the rollup, the copy of its rows alone.
--gnn-tree DIR adds the GNN top call (alz_gnn_top_device, k = 1000) on the config-2 window, measured in child
processes that alternate this tree's build and the built tree DIR (e.g. a checkout of the parent commit), three
times each; each child loads its own tree's alaz_b200 package and library.

Algorithmic bytes: the metrics pass reads 256 B of histogram per row (quantiles) or 24 B (sums only) and writes
8 B per value; the selection reads the 8-byte values 8 times (6 digit passes, the count, the emit).
Prints one JSON line per source and a last one with everything, with the card (nvidia-smi name, power limit).
Usage (GPU box): python scripts/edge_top_prof.py [--reps R] [--big-windows W] [--gnn-tree DIR] [--skip-sources]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.environ.get("EDGE_TOP_PROF_TREE", ROOT))   # --gnn-child: the other build's own package
from alaz_b200 import abi  # noqa: E402
from flush_prof import card  # noqa: E402
from gnn_top_prof import handle_for, summary  # noqa: E402

KS = (10, 1000, 100_000)


def timed(torch, stream, h, calls, reps):
    """calls: name -> f(); alternated, device events around each call."""
    for _ in range(2):
        for f in calls.values():
            f()
    h.sync()
    ms = {name: [] for name in calls}
    for _ in range(reps):
        for name, f in calls.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            f()
            e1.record(stream)
            e1.synchronize()
            ms[name].append(e0.elapsed_time(e1))
    return {name: summary(v) for name, v in ms.items()}


def host_alternative(h, dev_rows, n, reps):
    """copy the rows to the host and rank by p99 in numpy: ms per call (host clock)."""
    import metric_ref as mr
    import numpy as np
    Q = abi.METRIC_QUANTILE
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        rows = h.d2h(dev_rows, n, abi.EDGE_OUT)
        v = mr.values(rows, (Q, 0.99))
        sel = np.argpartition(-v, 1000)[:1000]
        sel[np.lexsort((sel, -v[sel]))]
        out.append((time.perf_counter() - t0) * 1e3)
    return summary(out)


def copy_only(h, dev_rows, n, reps):
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        h.d2h(dev_rows, n, abi.EDGE_OUT)
        out.append((time.perf_counter() - t0) * 1e3)
    return summary(out)


def gnn_child(reps):
    """child: the GNN top call (k = 1000) on the config-2 window, with the package and library of the tree that
    EDGE_TOP_PROF_TREE names (this tree without it)."""
    import torch
    from alaz_b200 import capi  # noqa: F401
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    h, bufs, _ = handle_for(torch, stream, 10_000, 100_000_000, 1)
    h.submit_device(bufs[0], 100_000_000)
    n = h.flush_device()[1]
    r = timed(torch, stream, h, {"gnn_top_k1000": lambda: h.gnn_top_device(1000, 0.0)}, reps)
    print(json.dumps({"rows": n, **r}))
    h.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--big-services", type=int, default=1_000_000)
    ap.add_argument("--big-events", type=int, default=100_000_000)
    ap.add_argument("--big-windows", type=int, default=4)
    ap.add_argument("--big-max-edges", type=int, default=1 << 23)
    ap.add_argument("--gnn-tree", default=None, help="another built tree to time alz_gnn_top_device against")
    ap.add_argument("--skip-sources", action="store_true", help="only the GNN top comparison")
    ap.add_argument("--gnn-child", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.gnn_child:
        return gnn_child(a.reps)

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("edge_top_prof.py: no CUDA device")
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    result = {"card": card(), "sources": []}

    if not a.skip_sources:
        sources(torch, stream, a, result)
    if a.gnn_tree:
        runs = []
        for _ in range(3):
            for tag, tree in (("this", None), ("other", os.path.abspath(a.gnn_tree))):
                env = dict(os.environ)
                env.pop("ALZ_LIB_PATH", None)
                env.pop("EDGE_TOP_PROF_TREE", None)
                if tree:
                    env["EDGE_TOP_PROF_TREE"] = tree
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--gnn-child", "--reps", str(a.reps)],
                                   env=env, capture_output=True, text=True, check=True)
                runs.append({"tree": tag, **json.loads(p.stdout.strip().splitlines()[-1])})
        result["gnn_top_alternated"] = runs
    print(json.dumps(result))


def sources(torch, stream, a, result):
    Q = abi.METRIC_QUANTILE
    TRIO = ((Q, 0.5), (Q, 0.99), abi.METRIC_ERR_RATE)

    def calls(h, metrics, top):
        c = {"metrics_p50_p99_rate": lambda: metrics(*TRIO)}
        for name, spec in (("p99", (Q, 0.99)), ("err5xx", abi.METRIC_ERR5XX)):
            for k in KS:
                c[f"top_{name}_k{k}"] = (lambda spec=spec, k=k: top(spec, k))
        return c

    # config-2 window
    h, bufs, _ = handle_for(torch, stream, 10_000, 100_000_000, 1)
    h.submit_device(bufs[0], 100_000_000)
    dev_rows, n_rows = h.flush_device()
    r = {"source": "config-2 last window", "rows": n_rows,
         "calls_ms": timed(torch, stream, h, calls(h, h.edge_metrics_device,
                                                   lambda s, k: h.edge_top_device(s, k, 0.0)), a.reps),
         "host_copy_and_numpy_p99_top1000_ms": host_alternative(h, dev_rows, n_rows, 5)}
    result["sources"].append(r)
    print(json.dumps(r), flush=True)
    h.close()

    # config-5 topology: a window rollup of several windows
    h, bufs, _ = handle_for(torch, stream, a.big_services, a.big_events, a.big_windows, a.big_max_edges)
    h.submit_device(bufs[0], a.big_events)
    first = h.flush_device()[1]                                        # sizes the history; not retained
    h.window_history(a.big_windows, a.big_windows * (first + first // 2))
    for d in bufs:
        h.submit_device(d, a.big_events)
        h.flush_device()
    dev_rows, n_rows, info = h.rollup_device(a.big_windows)
    W = abi.ROLLUP_WINDOWS
    r = {"source": f"config-5 topology, window rollup of {info['windows']} windows of {a.big_events} events",
         "rows": n_rows,
         "calls_ms": timed(torch, stream, h, calls(h, lambda *s: h.edge_metrics_rollup_device(W, *s),
                                                   lambda s, k: h.edge_top_rollup_device(W, s, k, 0.0)), a.reps),
         "host_copy_rows_ms": copy_only(h, dev_rows, n_rows, 3)}
    result["sources"].append(r)
    print(json.dumps(r), flush=True)
    h.close()

    for src in result["sources"]:
        n = src["rows"]
        src["bytes"] = {"metrics_p50_p99_rate": n * (256 + 24 + 24), "top_select": 8 * 8 * n}


if __name__ == "__main__":
    main()
