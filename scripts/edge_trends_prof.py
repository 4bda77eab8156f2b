#!/usr/bin/env python
"""What does an edge trend (docs/SPEC.md §20) cost? At bench.py config-2 sizes (Topo(10_000), --events device-resident
events per window, --buffers distinct event buffers taken in turn): the window history keeps 60 windows and a tier of
factor 5 keeps 12 entries. The source is a span rollup of the last 60 windows. Timed, as device calls:
  (a) the top 100 rows by p99 ZSCORE (the last 5 points against the 55 before) over the 60 history points
  (b) the top 100 rows by count SLOPE, FALLING, absent points as 0, over the 60 history points
  (c) every row's p99 SLOPE over the 60 history points (the full list)
  (d) the top 100 rows by p99 ZSCORE (the last point against the 11 before) over the tier's 12 points
each next to the §19 series call of the same metric over the same points, and once, for scale, the host alternative:
the series copied to the host (alz_edge_series) and the same trend and top computed in numpy (tests/trend_ref.py).

Per call: device events around the whole call, median and min-max over --reps after two warm-ups, calls alternated.
Per kernel: device time from torch.profiler over the same calls, summed per kernel name and divided by the calls.
The trend pass reads 8 + 1 B per slot (a row's P values and presence bytes, twice for SLOPE and ZSCORE, the second
pass mostly from cache) and 16 B of each source row, and writes 48 B per row (+ 8 B for a top call).
Prints one JSON line per case and a last one with everything, with the card (name, power limit, SM clock now and max).
Usage (GPU box): python scripts/edge_trends_prof.py [--reps R] [--events N] [--buffers B]
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


def host_alternative(h, source, tier, k, spec, t, top, reps=3):
    """alz_edge_series copied to the host, then the trend and the top in numpy: ms per call (host clock)"""
    import numpy as np
    import trend_ref as tr
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        v, p, _, _ = h.edge_series(source, tier, k, spec)
        rec = tr.trends(v[:, :, 0], p, stat=t.stat, direction=t.direction, absent=t.absent, recent=t.recent,
                        min_points=t.min_points)
        if top:
            vals = np.where(rec["valid"] == 1, rec["trend"], -np.inf)
            np.argsort(-vals, kind="stable")[:top]
        out.append((time.perf_counter() - t0) * 1e3)
    return round(sorted(out)[len(out) // 2], 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--buffers", type=int, default=4)
    ap.add_argument("--windows", type=int, default=60)
    ap.add_argument("--factor", type=int, default=5)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("edge_trends_prof.py: no CUDA device")
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
    T = capi.Handle.trend
    p99 = (Q, 0.99)
    cases = [
        (f"a_top{TOP}_p99_zscore_x{W}", 0, W, p99, T(abi.TREND_ZSCORE, recent=5), TOP),
        (f"b_top{TOP}_count_slope_falling_zero_x{W}", 0, W, abi.METRIC_COUNT,
         T(abi.TREND_SLOPE, abi.TREND_FALLING, abi.TREND_ABSENT_ZERO, recent=1), TOP),
        (f"c_all_p99_slope_x{W}", 0, W, p99, T(abi.TREND_SLOPE, recent=1), 0),
        (f"d_top{TOP}_p99_zscore_tier1_x{tier_depth}", 1, tier_depth, p99, T(abi.TREND_ZSCORE, recent=1), TOP),
    ]
    for name, tier, k, spec, t, top in cases:
        if top:
            def f(tier=tier, k=k, spec=spec, t=t, top=top):
                return h.edge_trends_top_device(S, tier, k, spec, t, top)
        else:
            def f(tier=tier, k=k, spec=spec, t=t):
                return h.edge_trends_device(S, tier, k, spec, t)

        def g(tier=tier, k=k, spec=spec):
            return h.edge_series_device(S, tier, k, spec)
        info = f()[-1]
        ms = timed(torch, stream, h, {name: f, "series": g}, a.reps)
        c = {"case": name, "rows": info["edges"], "points": info["points"], "valid": info["valid"],
             "above": info["above"], "call_ms": ms[name], "series_call_ms": ms["series"],
             "kernels_ms": kernel_times(torch, h, [f], 5), "series_kernels_ms": kernel_times(torch, h, [g], 5),
             "host_alternative_ms": host_alternative(h, S, tier, k, spec, t, top)}
        result["cases"].append(c)
        print(json.dumps(c), flush=True)
    h.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
