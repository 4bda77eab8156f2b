#!/usr/bin/env python
"""Flush time of a window whose edges are mostly one hub: one pod calling M distinct outbound addresses (an egress or
NAT pod; outbound edges are keyed by raw IPv4), next to a few thousand ordinary edges. Prints one JSON line with the
median and range of the flush's host time (the flush ends in a device synchronise) over the timed windows, and the
card. Usage (GPU box): python scripts/flush_hub_prof.py [--hub 1048576] [--windows 5]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from alaz_b200 import abi, capi  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hub", type=int, default=1 << 20)
    ap.add_argument("--windows", type=int, default=5)
    a = ap.parse_args()
    pod_net, svc_net, out_net = 0x0A000001, 0xAC000001, 0x08000000
    rng = np.random.default_rng(1)
    h = capi.Handle(max_endpoints=4096, max_pairs=a.hub + (1 << 18), max_edges=a.hub + (1 << 18))
    h.upsert_batch(abi.TABLE_POD, np.arange(pod_net, pod_net + 1000, dtype=np.uint32), np.arange(1000, dtype=np.uint32))
    h.upsert_batch(abi.TABLE_SVC, np.arange(svc_net, svc_net + 100, dtype=np.uint32), np.arange(100, dtype=np.uint32))
    h.commit()
    n_other = 100_000
    recs = np.zeros(a.hub + n_other, dtype=abi.L7_REC)
    recs["saddr"][: a.hub] = pod_net
    recs["daddr"][: a.hub] = out_net + rng.permutation(1 << 24)[: a.hub]
    recs["saddr"][a.hub:] = pod_net + rng.integers(1, 1000, n_other)
    recs["daddr"][a.hub:] = svc_net + rng.integers(0, 100, n_other)
    recs["protocol"], recs["method_flags"], recs["status"] = abi.PROTO_HTTP, 1, 200
    recs["duration_ns"] = rng.integers(1000, 1 << 30, len(recs))
    times, n = [], 0
    for w in range(a.windows + 1):
        h.submit(recs)
        h.sync()
        t0 = time.perf_counter()
        _, n = h.flush_device()
        h.sync()
        if w:   # the first window warms up
            times.append((time.perf_counter() - t0) * 1e3)
    h.close()
    print(json.dumps({"hub": a.hub, "edges": n, "flush_ms_median": statistics.median(times),
                      "flush_ms_min": min(times), "flush_ms_max": max(times), "card": card()}))


if __name__ == "__main__":
    main()
