"""GPU: tiered history on several ranks, on one GPU through the loopback collective (tests/loopback_tier_ranks.py).
After a merge every rank holds the merged rows, so every rank builds the same tiers with no collective of their own."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from alaz_b200 import abi
from test_gpu_loopback_ranks import HERE, ROOT, SMALL, shim, spread_groups  # noqa: F401  (shim is a fixture)
from tier_model import TierModel


@pytest.mark.gpu
def test_three_ranks_build_the_same_tiers(shim, tmp_path):  # noqa: F811
    R, J, K, rng = 3, 8, 3, np.random.default_rng(23)
    tabs, groups, _ = spread_groups(rng, 600)
    own = np.arange(len(groups)) % R
    per_rank = []
    for j in range(J):
        part = [g for i, g in enumerate(groups) if i % 4 != j % 4]                # the windows' edge sets differ
        w = [np.concatenate([g for i, g in enumerate(groups) if i % 4 != j % 4 and own[i] == r]) for r in range(R)]
        if j % 3 == 1:                                                            # keys on every rank: the general path
            w = [np.concatenate([x, np.concatenate(part[:50])]) for x in w]
        per_rank.append(w)
    tiers = [[2, 3, 1 << 14, 1 << 12], [2, 2, 1 << 14, 1 << 12]]
    spec = {"nranks": R, "cfg": SMALL, "tiers": tiers, "windows": J, "k": K}
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
    p = subprocess.run([sys.executable, os.path.join(HERE, "loopback_tier_ranks.py"), sp, ip, op], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    z = np.load(op)
    meta = json.loads(str(z["meta"]))
    assert not meta["errors"], meta["errors"]
    assert meta["maps"] == [shim], meta["maps"]
    rank = lambda r: meta["ranks"][str(r)]
    m = TierModel()
    m.configure(tiers)
    for j in range(J):
        for r in range(R):
            assert rank(r)[j]["rc"] == abi.OK
            assert z[f"rows_{j}_{r}"].tobytes() == z[f"rows_{j}_0"].tobytes()
        m.window(z[f"rows_{j}_0"], rank(0)[j]["windows"])
        for t in (1, 2):
            exp, info = m.rollup(t, K)
            for r in range(R):
                assert rank(r)[j]["info"][str(t)] == info, (r, j, t, rank(r)[j]["info"][str(t)], info)
                assert rank(r)[j]["state"][str(t)] == m.state(t), (r, j, t)
                assert z[f"tier_{j}_{r}_{t}"].tobytes() == exp.tobytes(), (r, j, t)
    assert m.state(1)["entries"] == 3 and m.state(2)["entries"] == 2
