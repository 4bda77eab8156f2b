"""GPU: correlations on several ranks, on one GPU through the loopback collective (tests/loopback_corr_ranks.py). After
a merge every rank holds the merged rows and the same map, so every rank retains the same history: every rank returns
the same correlations of every level, with no collective of its own, and the edge level equals tests/corr_ref.py over
the entries that tests/rollup_model.py and tests/tier_model.py retain from the merged windows."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import corr_ref as cr
import series_ref as sr
from alaz_b200 import abi
from change_ref import row_keys
from loopback_corr_ranks import CALLS, SPEC
from rollup_model import RollupModel
from test_gpu_loopback_ranks import HERE, ROOT, SMALL, shim, spread_groups  # noqa: F401  (shim is a fixture)
from tier_model import TierModel, rows_of


@pytest.mark.gpu
def test_three_ranks_return_identical_correlations(shim, tmp_path):  # noqa: F811
    R, J, rng = 3, 6, np.random.default_rng(58)
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
    rings = [[0, 4], [1, 3]]
    corrs = [[abi.CORR_POSITIVE, abi.CORR_ABSENT_SKIP, 1, 3], [abi.CORR_ABS, abi.CORR_ABSENT_ZERO, 2, 3]]
    spec = {"nranks": R, "cfg": SMALL, "history": history, "tiers": tiers, "windows": J, "rings": rings,
            "corrs": corrs, "top": 40, "groups": 7}
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
    p = subprocess.run([sys.executable, os.path.join(HERE, "loopback_corr_ranks.py"), sp, ip, op], cwd=ROOT,
                       env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    z = np.load(op)
    meta = json.loads(str(z["meta"]))
    assert not meta["errors"], meta["errors"]
    assert meta["maps"] == [shim], meta["maps"]
    rm, tm = RollupModel(), TierModel()
    rm.history(*history)
    tm.configure(tiers)
    valid, listed = 0, 0
    for j in range(J):
        for r in range(1, R):
            assert z[f"win_{j}_{r}"].tobytes() == z[f"win_{j}_0"].tobytes(), (j, r)
            for c in range(len(rings)):
                for g in range(2):
                    assert str(z[f"tgt{c}_{g}_{j}_{r}"]) == str(z[f"tgt{c}_{g}_{j}_0"]), (j, r, c, g)
                    for s in range(len(corrs)):
                        for level, side in CALLS:
                            for x in ("rec", "top", "trow", "tser", "tpre"):
                                key = f"{c}_{g}_{s}_{level}_{side}_{j}"
                                assert z[f"{x}{key}_{r}"].tobytes() == z[f"{x}{key}_0"].tobytes(), (x, key, r)
                                listed += len(z[f"{x}{key}_0"]) if x == "top" else 0
        win = z[f"win_{j}_0"]
        rm.append(win, j + 1)
        tm.window(win, j + 1)
        for c, (tier, k) in enumerate(rings):
            ring = rm.entries if tier == 0 else tm.tiers[tier - 1].ring.entries
            ents = [rows_of(e["rows"]) for e in ring]
            v, p = sr.series(ents, row_keys(win), [SPEC], k)
            y, pp = v[:, :, 0], p
            for g in range(2):
                tv, tp, last = json.loads(str(z[f"tgt{c}_{g}_{j}_0"]))
                assert last == (ring[-1]["window"] if ring else 0), (j, c)
                for s, (direction, absent, max_lag, min_points) in enumerate(corrs):
                    rec = cr.records(win, y, pp, np.array(tv), np.array(tp, np.uint8), direction=direction,
                                     absent=absent, max_lag=max_lag, min_points=min_points)
                    key = f"{c}_{g}_{s}_edge_{abi.SIDE_IN}_{j}_0"
                    assert z["rec" + key].tobytes() == rec.tobytes(), (j, c, g, s)
                    idx, _ = cr.top(rec, 40)
                    assert z["top" + key].tobytes() == rec[idx].tobytes(), (j, c, g, s)
                    assert z["trow" + key].tobytes() == win[idx].tobytes(), (j, c, g, s)
                    assert z["tser" + key].tobytes() == y[idx].tobytes(), (j, c, g, s)
                    valid += int(rec["valid"].sum())
    assert valid > 0 and listed > 0
