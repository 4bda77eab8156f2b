"""Cost of the window clock in the multi-rank merge: 8 ranks on one GPU through the loopback collective
(tests/loopback_nccl.cu, child tests/loopback_clock.py), about 190k rows per rank per window (config-2-sized), with
the clock on and off alternated in one call. Prints one JSON line: merge_us_last (alz_stats) of every timed window
per arm, and the card's name and power limit.

Loopback times are not NVLink times: the loopback all-gather is device-to-device copies on one GPU.

    python scripts/merge_clock_cost.py [--rounds 3] [--windows 4] [--rows 190000]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

from alaz_b200 import abi  # noqa: E402
from gnn_graphs import POD_NET, SVC_NET  # noqa: E402
from loopback_ranks import owner_rank  # noqa: E402
from test_gpu_loopback_ranks import build_shim  # noqa: E402

R = 8
W = 1_000_000_000
CFG = dict(max_endpoints=1 << 14, max_pairs=1 << 19, max_edges=1 << 21, max_batch=1 << 18)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def window_recs(rank, rows, j, rng):
    """`rows` distinct edges of rank r's own pods, one record each, all in epoch 10 + j"""
    pods = POD_NET + np.arange(4096)
    mine = pods[owner_rank(pods, R) == rank]
    x = np.zeros(rows, dtype=abi.L7_REC)
    x["saddr"] = mine[np.arange(rows) % len(mine)]
    x["daddr"] = (12 << 24) + np.arange(rows) // len(mine) + (j << 16)
    x["protocol"], x["method_flags"], x["status"] = abi.PROTO_HTTP, 1, 200
    x["duration_ns"] = rng.integers(1, 1 << 30, rows, dtype=np.uint64)
    x["write_time_ns"] = (10 + j) * W + rng.integers(0, W, rows, dtype=np.uint64)
    return x


def run_arm(shim, tmp, clocked, windows, rows):
    rng = np.random.default_rng(1)
    tabs = np.concatenate([np.stack([np.full(4096, abi.TABLE_POD), POD_NET + np.arange(4096), np.arange(4096)], 1),
                           np.array([[abi.TABLE_SVC, SVC_NET, 7]])]).astype(np.int64)
    arrays, ops = {"tables": tabs}, [{"op": "join"}]
    if clocked:
        ops += [{"op": "clock", "r": r, "args": [0, 0, W]} for r in range(R)]
    for j in range(windows + 1):            # the first window is warm-up
        for r in range(R):
            arrays[f"w{j}_{r}"] = window_recs(r, rows, j, rng)
            ops.append({"op": "submit", "r": r, "key": f"w{j}_{r}"})
        ops.append({"op": "flush", "how": "device"})
    spec = {"nranks": R, "cfg": CFG, "ops": ops}
    sp, ip, op = (os.path.join(tmp, x) for x in ("spec.json", "in.npz", "out.npz"))
    with open(sp, "w") as f:
        json.dump(spec, f)
    np.savez(ip, **arrays)
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = os.path.dirname(shim) + os.pathsep + env.get("LD_LIBRARY_PATH", "")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "loopback_clock.py"), sp, ip, op], cwd=ROOT,
                       env=env, capture_output=True, text=True, timeout=1200)
    if p.returncode != 0:
        raise RuntimeError(p.stdout[-2000:] + p.stderr[-2000:])
    meta = json.loads(str(np.load(op)["meta"]))
    if meta["errors"]:
        raise RuntimeError(meta["errors"])
    flushes = [i for i, o in enumerate(ops) if o["op"] == "flush"][1:]
    us, n_out = [], set()
    for i in flushes:
        for r in range(R):
            d = meta["ranks"][str(r)][i]
            if d["rc"] != abi.OK:
                raise RuntimeError(f"flush {i} rank {r}: {d['rc']}")
            n_out.add(d["n_out"])
            us.append(d["stats"]["merge_us_last"])
    return us, sorted(n_out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--windows", type=int, default=4)
    ap.add_argument("--rows", type=int, default=190_000)
    a = ap.parse_args()
    res = {"card": card(), "ranks": R, "rows_per_rank": a.rows, "note": "loopback on one GPU, not NVLink",
           "clock_on_us": [], "clock_off_us": []}
    with tempfile.TemporaryDirectory() as tmp:
        shim = build_shim(tmp)
        for _ in range(a.rounds):
            for clocked in (True, False):
                d = os.path.join(tmp, f"arm{int(clocked)}")
                os.makedirs(d, exist_ok=True)
                us, n_out = run_arm(shim, d, clocked, a.windows, a.rows)
                res["clock_on_us" if clocked else "clock_off_us"] += us
                res["merged_rows"] = n_out
    for k in ("clock_on_us", "clock_off_us"):
        res[k.replace("_us", "_median_us")] = float(np.median(res[k]))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
