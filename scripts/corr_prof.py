#!/usr/bin/env python
"""What does a correlation (docs/SPEC.md §29) cost? At bench.py config-2 sizes (Topo(10_000), --events device-resident
events per window, --buffers distinct event buffers taken in turn): the window history keeps 60 windows and a tier of
factor 5 keeps 12 entries. The source is a span rollup of the last 60 windows, and the target is the series of the
source's first row, edge or node (or of a synthetic group series), over the 60 history points. Timed, as device calls,
for max_lag 0, 8 and 32 and the metrics p99 and count:
  edge   the top 100 edges (alz_edge_correlations_top_device) next to the §19 series call of the same metric
  node   the top 100 nodes on side IN next to the §22 node series call
  group  the top 100 group nodes on side IN, pods mapped into 500 groups, next to the §26 group node series call
and, for the edges, once, the host alternative: the series copied to the host (alz_edge_series) and the correlations
and top computed in numpy (tests/corr_ref.py).

Per call: device events around the whole call, median and min-max over --reps after two warm-ups, calls alternated.
Per kernel: device time from torch.profiler over the same calls, summed per kernel name and divided by the calls.
corr_kernel reads 8 + 1 B per slot once when a row fits one 64-point tile (P <= 64), else once per tile, lag and
pass; it writes 48 B per row (+ 8 B for a top call). corr_gbs is the bytes it must read over its time.
Prints one JSON line per case and a last one with everything, with the card (name, power limit, SM clock now and max).
Usage (GPU box): python scripts/corr_prof.py [--reps R] [--events N] [--buffers B]
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
from alaz_b200 import abi, capi  # noqa: E402
from edge_changes_prof import kernel_times  # noqa: E402
from edge_series_prof import card  # noqa: E402
from edge_top_prof import timed  # noqa: E402
from gnn_top_prof import handle_for  # noqa: E402

Q = abi.METRIC_QUANTILE
TOP = 100


def host_alternative(h, source, k, spec, corr, target, reps=3):
    """alz_edge_series copied to the host, then the correlations and the top in numpy: ms per call (host clock)"""
    import numpy as np
    import corr_ref as cr
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        v, p, _, _ = h.edge_series(source, 0, k, spec)
        rec = cr.records(None, v[:, :, 0], p, target.values, target.present, direction=corr.direction,
                         absent=corr.absent, max_lag=corr.max_lag, min_points=corr.min_points)
        cr.top(rec, TOP)
        out.append((time.perf_counter() - t0) * 1e3)
    return round(sorted(out)[len(out) // 2], 1)


def target_of(h, pv, pp, P, last):
    """the target: series row 0 of a series device call (values, presence), aligned to the ring"""
    import numpy as np
    return capi.Handle.Target(h.d2h(pv, P, np.float64), h.d2h(pp, P, np.uint8), last)


def corr_kernel_ms(kernels):
    return round(sum(v for k_, v in kernels.items() if "corr_kernel" in k_), 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--buffers", type=int, default=4)
    ap.add_argument("--windows", type=int, default=60)
    ap.add_argument("--factor", type=int, default=5)
    ap.add_argument("--host", type=int, default=1, help="1: time the host alternative once per edge case")
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("corr_prof.py: no CUDA device")
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
    nodes = h.node_rows(S)
    pods = nodes["value"][nodes["type"] == abi.NODE_POD]
    h.group_set([(abi.NODE_POD, int(v)) for v in pods], (pods % 500).astype(np.uint32))
    series = {"edge": lambda spec: h.edge_series_device(S, 0, W, spec),
              "node": lambda spec: h._series_device("alz_node_series_device", (S, abi.SIDE_IN), (0, W), (spec,)),
              "group_node": lambda spec: h._series_device("alz_group_node_series_device", (S, abi.SIDE_IN), (0, W),
                                                          (spec,))}
    for level in ("edge", "node", "group_node"):
        for mname, spec in (("p99", (Q, 0.99)), ("count", abi.METRIC_COUNT)):
            pv, pp, rows, P, pts, _ = series[level](spec)
            target = target_of(h, pv, pp, P, pts[-1]["window_last"])
            for max_lag in (0, 8, 32):
                corr = capi.Handle.corr(abi.CORR_ABS, abi.CORR_ABSENT_SKIP, max_lag, 3)
                name = f"{level}_top{TOP}_{mname}_lag{max_lag}_x{W}"

                def f(level=level, spec=spec, corr=corr, target=target):
                    return h.correlations_top_device(level, S, 0, W, spec, corr, target, TOP, side=abi.SIDE_IN)

                def g(level=level, spec=spec):
                    return series[level](spec)
                info = f()[-1]
                ms = timed(torch, stream, h, {name: f, "series": g}, a.reps)
                kern = kernel_times(torch, h, [f], 5)
                kms = corr_kernel_ms(kern)
                read = info["rows"] * info["points"] * 9 * (1 if info["points"] <= 64 else 2 * (max_lag + 1))
                c = {"case": name, "rows": info["rows"], "points": info["points"], "valid": info["valid"],
                     "above": info["above"], "call_ms": ms[name], "series_call_ms": ms["series"],
                     "corr_kernel_ms": kms, "corr_bytes": read,
                     "corr_gbs": round(read / (kms * 1e6), 1) if kms else None,
                     "kernels_ms": kern, "series_kernels_ms": kernel_times(torch, h, [g], 5)}
                if level == "edge" and a.host:
                    c["host_alternative_ms"] = host_alternative(h, S, W, spec, corr, target)
                result["cases"].append(c)
                print(json.dumps(c), flush=True)
    result["card_after"] = card()
    h.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
