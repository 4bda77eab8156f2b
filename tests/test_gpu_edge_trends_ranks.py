"""GPU: edge trends on several ranks, on one GPU through the loopback collective (tests/loopback_trends_ranks.py).
After a merge every rank holds the merged rows, so every rank retains the same history: every rank returns the same
trends, with no collective of its own, and they equal tests/trend_ref.py over the entries that tests/rollup_model.py
and tests/tier_model.py retain from the merged windows."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import trend_ref as tr
from alaz_b200 import abi
from loopback_trends_ranks import SPEC
from rollup_model import RollupModel
from test_gpu_loopback_ranks import HERE, ROOT, SMALL, shim, spread_groups  # noqa: F401  (shim is a fixture)
from tier_model import TierModel, rows_of


@pytest.mark.gpu
def test_three_ranks_return_identical_trends(shim, tmp_path):  # noqa: F811
    R, J, rng = 3, 7, np.random.default_rng(57)
    tabs, groups, _ = spread_groups(rng, 600)
    own = np.arange(len(groups)) % R
    per_rank = []
    for j in range(J):
        part = [g for i, g in enumerate(groups) if i % 5 != j % 5]
        w = [np.concatenate([g for i, g in enumerate(groups) if i % 5 != j % 5 and own[i] == r]) for r in range(R)]
        if j % 3 == 1:                                                            # keys on every rank
            w = [np.concatenate([x, np.concatenate(part[:50])]) for x in w]
        per_rank.append(w)
    history, tiers = [4, 1 << 14], [[2, 3, 1 << 14, 1 << 12]]
    rings = [[0, 6], [0, 2], [1, 3]]
    trends = [[abi.TREND_ZSCORE, abi.TREND_RISING, abi.TREND_ABSENT_SKIP, 1, 0],
              [abi.TREND_SLOPE, abi.TREND_FALLING, abi.TREND_ABSENT_ZERO, 1, 2],
              [abi.TREND_RATIO, abi.TREND_RISING, abi.TREND_ABSENT_ZERO, 1, 0]]
    spec = {"nranks": R, "cfg": SMALL, "history": history, "tiers": tiers, "windows": J, "rings": rings,
            "trends": trends, "top": 40}
    arrays = {"tab0": np.asarray(tabs, np.int64).reshape(-1, 3)}
    for j, w in enumerate(per_rank):
        for r in range(R):
            arrays[f"w{j}_r{r}"] = np.ascontiguousarray(w[r], dtype=abi.L7_REC)
    sp, ip, op = (str(tmp_path / x) for x in ("spec.json", "in.npz", "out.npz"))
    with open(sp, "w") as f:
        json.dump(spec, f)
    np.savez(ip, **arrays)
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = os.path.dirname(shim) + os.pathsep + env.get("LD_LIBRARY_PATH", "")
    env["LOOPBACK_NCCL_TIMEOUT_S"] = "60"
    p = subprocess.run([sys.executable, os.path.join(HERE, "loopback_trends_ranks.py"), sp, ip, op], cwd=ROOT,
                       env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    z = np.load(op)
    meta = json.loads(str(z["meta"]))
    assert not meta["errors"], meta["errors"]
    assert meta["maps"] == [shim], meta["maps"]
    rm, tm = RollupModel(), TierModel()
    rm.history(*history)
    tm.configure(tiers)
    valid = 0
    for j in range(J):
        names = [f"{x}{c}_{t}_{{}}_{{}}" for c in range(len(rings)) for t in range(len(trends))
                 for x in ("rec", "pts", "top", "trow", "tser", "tpre")]
        for r in range(1, R):
            for x in names + ["win_{}_{}"]:
                assert z[x.format(j, r)].tobytes() == z[x.format(j, 0)].tobytes(), (x, j, r)
        win = z[f"win_{j}_0"]
        rm.append(win, j + 1)
        tm.window(win, j + 1)
        for c, (tier, k) in enumerate(rings):
            ring = rm.entries if tier == 0 else tm.tiers[tier - 1].ring.entries
            ents = [rows_of(e["rows"]) for e in ring]
            for t, (stat, direction, absent, recent, min_points) in enumerate(trends):
                rec, y, p = tr.expect(ents, win, SPEC, k, stat=stat, direction=direction, absent=absent,
                                      recent=recent, min_points=min_points)
                assert z[f"rec{c}_{t}_{j}_0"].tobytes() == rec.tobytes(), (j, c, t)
                idx, _ = tr.top(rec, 40)
                assert z[f"top{c}_{t}_{j}_0"].tobytes() == rec[idx].tobytes(), (j, c, t)
                assert z[f"trow{c}_{t}_{j}_0"].tobytes() == win[idx].tobytes(), (j, c, t)
                assert z[f"tser{c}_{t}_{j}_0"].tobytes() == y[idx].tobytes(), (j, c, t)
                assert z[f"tpre{c}_{t}_{j}_0"].tobytes() == p[idx].tobytes(), (j, c, t)
                pts = json.loads(str(z[f"pts{c}_{t}_{j}_0"]))
                assert [x["window_last"] for x in pts] == [e["window"] for e in ring[max(len(ring) - k, 0):]], (j, c)
                valid += int(rec["valid"].sum())
    assert valid > 0
