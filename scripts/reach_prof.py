#!/usr/bin/env python
"""What do the reach calls (docs/SPEC.md §27) cost? At bench.py config-2 sizes (Topo(10_000), --events
device-resident events per window, --buffers distinct event buffers taken in turn): the window history keeps --windows
windows. Two sources: the last window, and a span rollup of all of them. Three forms: the node form, and the group
form under group_prof.py's two maps (owners, namespaces).
Timed, as device calls (alz_reach_device / alz_group_reach_device), for every combination of:
  direction  DOWN, UP
  seeds      1 and 100 (the pods, or the groups, with the most rows on the direction's tail side first)
  max_hops   3, 64
  filter     none, ERR5XX >= 1
Per call: device events around the whole call, median and min-max over --reps after two warm-ups, calls alternated;
with levels, nodes and rows listed. Once per source and form, for scale, the host route: the traversed rows copied to
the host and searched there (tests/reach_ref.py, DOWN, 1 seed, max_hops 64, no filter).
Prints one JSON line per case and a last one with everything, with the card (name, power limit, SM clock now and max).
Usage (GPU box): python scripts/reach_prof.py [--reps R] [--events N] [--buffers B] [--windows W]
"""
import argparse
import ctypes as C
import itertools
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from alaz_b200 import abi  # noqa: E402
from edge_series_prof import card  # noqa: E402
from edge_top_prof import timed  # noqa: E402
from gnn_top_prof import handle_for  # noqa: E402
from group_prof import maps  # noqa: E402

W, S = abi.SOURCE_WINDOW, abi.ROLLUP_SPAN
DOWN, UP = abi.REACH_DOWN, abi.REACH_UP


def busiest(rows, direction, k, group_only):
    """NODE_ENDS of the k nodes with the most rows on the direction's tail side (from for DOWN, to for UP)"""
    t, v = ("from_type", "from") if direction == DOWN else ("to_type", "to")
    keys = (rows[t].astype(np.uint64) << np.uint64(32)) | rows[v].astype(np.uint64)
    if group_only:
        keys = keys[(keys >> np.uint64(32)) == abi.NODE_GROUP]
    elif direction == DOWN:
        keys = keys[(keys >> np.uint64(32)) == abi.NODE_POD]
    u, c = np.unique(keys, return_counts=True)
    top = u[np.argsort(-c, kind="stable")[:k]]
    e = np.zeros(len(top), dtype=abi.NODE_ENDS)
    e["type"], e["value"] = top >> np.uint64(32), top & np.uint64(0xFFFFFFFF)
    return e


def host_route(h, p, n, seeds, reps=3):
    """ms per call (host clock): the traversed rows copied to the host and searched"""
    import reach_ref
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        rows = h.d2h(p, n, abi.EDGE_OUT)
        reach_ref.reach(rows, seeds, DOWN, 64)
        out.append((time.perf_counter() - t0) * 1e3)
    return round(sorted(out)[len(out) // 2], 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--buffers", type=int, default=4)
    ap.add_argument("--windows", type=int, default=60)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("reach_prof.py: no CUDA device")
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    result = {"card": card(), "cases": []}
    print(json.dumps({"card": result["card"]}), flush=True)

    h, bufs, _ = handle_for(torch, stream, 10_000, a.events, a.buffers)
    h.submit_device(bufs[0], a.events)
    first = h.flush_device()[1]                                       # sizes the history
    h.window_history(a.windows, a.windows * (first + first // 2))
    for w in range(a.windows):
        h.submit_device(bufs[w % len(bufs)], a.events)
        h.flush_device()
    ps, ns, info_s = h.rollup_span_device(a.windows)
    span_rows = h.d2h(ps, ns, abi.EDGE_OUT)
    result["source"] = {"span_rows": ns, "span_windows": info_s["windows"]}
    forms = [("node", None)] + [(name, (ends, groups)) for name, ends, groups in maps(span_rows)]
    for (src_name, src), (form, mp) in itertools.product((("window", W), ("span", S)), forms):
        group = mp is not None
        h.group_set(*(mp if group else ([], [])))
        if group:
            p, n, _ = h.group_edges_device(src)
        elif src == S:
            p, n = ps, ns
        else:   # the last window's rows, fetched and put back on the device for the host route's copy
            fetched, m = np.zeros(h.max_edges, dtype=abi.EDGE_OUT), C.c_size_t(0)
            h._ck(h.L.alz_window_fetch(h.h, fetched.ctypes.data_as(C.c_void_p), len(fetched), C.byref(m)),
                  "alz_window_fetch")
            fetched = fetched[: m.value]
            p, n = h.dev_alloc(max(fetched.nbytes, 1)), len(fetched)
            h.h2d(p, fetched)
        traversed = h.d2h(p, n, abi.EDGE_OUT)
        fn = h.group_reach_device if group else h.reach_device
        calls, meta = {}, {}
        for d, k, hops, filt in itertools.product((DOWN, UP), (1, 100), (3, 64), ("none", "err5xx>=1")):
            seeds = busiest(traversed, d, k, group)
            spec, mv = (None, 0.0) if filt == "none" else (abi.METRIC_ERR5XX, 1.0)
            name = f"{'down' if d == DOWN else 'up'}/{k}/{hops}/{filt}"
            calls[name] = (lambda fn=fn, s=seeds, d=d, hops=hops, spec=spec, mv=mv:
                           fn(src, s, d, hops, spec, mv))
            r = calls[name]()
            meta[name] = {"levels": r[5]["levels"], "nodes": r[1], "rows": r[4], "cut": r[5]["cut"],
                          "traversable": r[5]["traversable"], "seeds_found": r[5]["seeds_found"]}
        ms = timed(torch, stream, h, calls, a.reps)
        host_ms = host_route(h, p, n, busiest(traversed, DOWN, 1, group))
        if not group and src == W:
            h.dev_free(p)
        for name in calls:
            case = {"source": src_name, "form": form, "traversed_rows": n, "case": name, "call_ms": ms[name],
                    **meta[name]}
            result["cases"].append(case)
            print(json.dumps(case), flush=True)
        hr = {"source": src_name, "form": form, "traversed_rows": n, "host_route_ms": host_ms}
        result["cases"].append(hr)
        print(json.dumps(hr), flush=True)
    h.group_set([], [])
    result["card_after"] = card()
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
