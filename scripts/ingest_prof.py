#!/usr/bin/env python
"""Where does a warp of the ingest kernel spend its cycles in a REAL run (warm caches, no profiler)?
Runs the profiling build (alaz_b200/build.py --prof -> libalazgpu_prof.so) on config 2 and prints the
per-section cycle shares, and the per-CTA timeline of every timed launch: when each CTA started, left its main loop
and ended (%globaltimer), on which SM, against the launch's CUDA-event time. Usage (GPU box):
  ALZ_LIB_PATH=alaz_b200/lib/libalazgpu_prof.so python scripts/ingest_prof.py [--max-pairs N] [--steps K] [--out F]
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from alaz_b200 import abi, capi  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--services", type=int, default=10_000)
ap.add_argument("--events", type=int, default=100_000_000)
ap.add_argument("--max-pairs", type=int, default=1 << 20)
ap.add_argument("--steps", type=int, default=6)
ap.add_argument("--windows", type=int, default=3)
ap.add_argument("--out", default=None, help="also write the JSON result here")
a = ap.parse_args()

import numpy as np  # noqa: E402
import torch  # noqa: E402
L = capi.load()
stream = torch.cuda.Stream()   # the handle runs on this stream, so the CUDA events below time its launches
torch.cuda.set_stream(stream)
L.alz_debug_ingest_prof.argtypes = [C.c_void_p]
L.alz_debug_ingest_timeline.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
topo = capi.Topo(a.services, seed=0xA1A20001)
h = capi.Handle(max_endpoints=4 * a.services, max_pairs=a.max_pairs)
h.set_stream(stream.cuda_stream)
h.load_tables(topo.pod_ip, topo.svc_ip)
wins = []
for k in range(a.windows):
    d = h.dev_alloc(a.events * 32)
    topo.fill_device(h, k * a.events, a.events, d)
    wins.append(d)
h.sync()
buf = (C.c_ulonglong * 12)()
for k in range(3):
    h.submit_device(wins[k % a.windows], a.events); h.flush_device()
h.sync()
rc = L.alz_debug_ingest_prof(buf)
if rc != 0:
    raise SystemExit("not a profiling build: set ALZ_LIB_PATH=alaz_b200/lib/libalazgpu_prof.so")
dims = (C.c_uint * 3)()
n_tl = C.c_uint(0)
L.alz_debug_ingest_timeline(None, C.byref(n_tl), dims)
tl = np.zeros(tuple(dims), dtype=np.uint64)
L.alz_debug_ingest_timeline(tl.ctypes.data, C.byref(n_tl), dims)   # starts the timeline over
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
ms = 0.0
ev_ms = []
for k in range(a.steps):
    torch.cuda.synchronize()
    e0.record(stream)
    h.submit_device(wins[(3 + k) % a.windows], a.events)
    e1.record(stream)
    h.flush_device()
    torch.cuda.synchronize()
    ev_ms.append(e0.elapsed_time(e1))
    ms += ev_ms[-1]
L.alz_debug_ingest_prof(buf)
L.alz_debug_ingest_timeline(tl.ctypes.data, C.byref(n_tl), dims)
v = [int(x) for x in buf]
tot = max(1, v[0])
names = ["loop total", "wait for the TMA stage", "wait for the probes (cp.async)", "cold tier incl. its waits + slow",
         "slow batches", "hot tier (record loads .. queue pushes)", "iterations", "cold batches"]
out = {"ingest_ms_with_instrumentation": ms / a.steps, "max_pairs": a.max_pairs,
       "cycles_per_iteration": v[0] / max(1, v[6]),
       "shares": {names[i]: round(v[i] / tot, 4) for i in (1, 2, 3, 4, 5)},
       "cold_batches_per_iteration": v[7] / max(1, v[6])}
ctas = max(1, v[11])
warps_per_cta = 16
out["phases_cycles_per_cta"] = {"prologue (smem init, hot list preload)": v[8] / ctas,
                                "main loop until the slowest warp is done": v[9] / ctas,
                                "mean warp's main loop (16 warps assumed)": v[0] / ctas / warps_per_cta,
                                "drain of the private rows": v[10] / ctas}
out["phases_ms_at_1965MHz"] = {k: round(c / 1.965e6, 4) for k, c in out["phases_cycles_per_cta"].items()}


def spread_us(t, t0):
    d = (t.astype(np.int64) - int(t0)) / 1e3
    return {"min": round(float(d.min()), 2), "median": round(float(np.median(d)), 2), "max": round(float(d.max()), 2)}


# one flush per step does not launch the ingest kernel, so timed launch k is timeline entry k
launches, by_sm = [], {}
for k in range(min(int(n_tl.value), a.steps, tl.shape[0])):
    e = tl[k]
    e = e[e[:, 0] != 0]                                     # CTAs of this launch
    t0 = e[:, 0].min()
    end = e[:, 2].astype(np.int64)
    med_end = float(np.median(end))
    sm_mhz = (e[:, 5] - e[:, 4]).astype(np.float64) / np.maximum(1, (e[:, 2] - e[:, 0]).astype(np.float64)) * 1e3
    launches.append({
        "ctas": int(len(e)), "event_ms": round(ev_ms[k], 4),
        "span_ms": round((int(end.max()) - int(t0)) / 1e6, 4),       # first CTA start .. last CTA end
        "start_us": spread_us(e[:, 0], t0), "loop_end_us": spread_us(e[:, 1], t0), "end_us": spread_us(e[:, 2], t0),
        "latest_end_after_median_us": round((int(end.max()) - med_end) / 1e3, 2),
        "chunks_per_cta": {"min": int(e[:, 6].min()), "max": int(e[:, 6].max())},
        "sm_clock_mhz": round(float(np.median(sm_mhz)), 0)})
    for sm, t in zip(e[:, 3].tolist(), ((end - med_end) / 1e3).tolist()):
        by_sm.setdefault(int(sm), []).append(t)
sm_ids = sorted(by_sm)
mean_end = np.array([np.mean(by_sm[i]) for i in sm_ids])
# does an SM end late in every launch (a placement effect) or at random? correlation of consecutive launches
per_launch = [np.array([by_sm[i][k] for i in sm_ids if len(by_sm[i]) > k]) for k in range(len(launches))]
corr = [float(np.corrcoef(per_launch[k], per_launch[k + 1])[0, 1]) for k in range(len(per_launch) - 1)
        if len(per_launch[k]) == len(per_launch[k + 1]) and len(per_launch[k]) > 1]
order = np.argsort(mean_end)
out["timeline"] = {
    "launches": launches,
    "event_minus_span_us": round(float(np.median([(l["event_ms"] - l["span_ms"]) * 1e3 for l in launches])), 2)
    if launches else None,
    "end_after_median_by_sm_us": {str(i): round(float(v), 1) for i, v in zip(sm_ids, mean_end)},
    "slowest_sms": [int(sm_ids[i]) for i in order[::-1][:12]],
    "fastest_sms": [int(sm_ids[i]) for i in order[:12]],
    "sm_end_corr_between_launches": round(float(np.mean(corr)), 3) if corr else None}
try:
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as ex:  # noqa: BLE001
    q = f"nvidia-smi unavailable: {ex}"
out["card"] = q
out["device"] = torch.cuda.get_device_name(0)
print(json.dumps(out))
if a.out:
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)
