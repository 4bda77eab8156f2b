"""GPU: edge series on several ranks, on one GPU through the loopback collective (tests/loopback_series_ranks.py).
After a merge every rank holds the merged rows, so every rank retains the same history: every rank returns the same
series, with no collective of its own, and they equal tests/series_ref.py over the entries that
tests/rollup_model.py and tests/tier_model.py retain from the merged windows."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import series_ref as sr
from alaz_b200 import abi
from change_ref import row_keys
from loopback_series_ranks import SPECS, UNKNOWN
from rollup_model import RollupModel
from test_gpu_loopback_ranks import HERE, ROOT, SMALL, shim, spread_groups  # noqa: F401  (shim is a fixture)
from tier_model import TierModel, rows_of


@pytest.mark.gpu
def test_three_ranks_return_identical_series(shim, tmp_path):  # noqa: F811
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
    spec = {"nranks": R, "cfg": SMALL, "history": history, "tiers": tiers, "windows": J, "rings": rings}
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
    p = subprocess.run([sys.executable, os.path.join(HERE, "loopback_series_ranks.py"), sp, ip, op], cwd=ROOT,
                       env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    z = np.load(op)
    meta = json.loads(str(z["meta"]))
    assert not meta["errors"], meta["errors"]
    assert meta["maps"] == [shim], meta["maps"]
    rm, tm = RollupModel(), TierModel()
    rm.history(*history)
    tm.configure(tiers)
    points = 0
    for j in range(J):
        names = [f"{x}{c}_{{}}_{{}}" for c in range(len(rings)) for x in ("val", "pre", "pts", "kval", "kpre")]
        for r in range(1, R):
            for x in names + ["win_{}_{}"]:
                assert z[x.format(j, r)].tobytes() == z[x.format(j, 0)].tobytes(), (x, j, r)
        win = z[f"win_{j}_0"]
        rm.append(win, j + 1)
        tm.window(win, j + 1)
        ekeys = row_keys(win)
        kkeys = np.concatenate([ekeys[::-1], np.array([sr.pack_ends(*UNKNOWN)], dtype=np.uint64)])
        for c, (tier, k) in enumerate(rings):
            ring = rm.entries if tier == 0 else tm.tiers[tier - 1].ring.entries
            ents = [rows_of(e["rows"]) for e in ring]
            v, p_ = sr.series(ents, ekeys, SPECS, k)
            assert z[f"val{c}_{j}_0"].tobytes() == v.tobytes() and z[f"pre{c}_{j}_0"].tobytes() == p_.tobytes(), (j, c)
            v, p_ = sr.series(ents, kkeys, SPECS, k)
            assert z[f"kval{c}_{j}_0"].tobytes() == v.tobytes() and z[f"kpre{c}_{j}_0"].tobytes() == p_.tobytes(), (j, c)
            pts = json.loads(str(z[f"pts{c}_{j}_0"]))
            assert [x["window_last"] for x in pts] == [e["window"] for e in ring[max(len(ring) - k, 0):]], (j, c)
            points += p_.sum()
    assert points > 0
