"""GPU: top anomalous rows on several ranks, on one GPU through the loopback collective (tests/loopback_gnn_top_ranks.py).
After a merge every rank holds the merged rows, so every rank's window and rollup rows are the same, and so are their
top lists, with no collective of the selection's own."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import top_ref
from alaz_b200 import abi
from test_gpu_loopback_ranks import HERE, ROOT, SMALL, shim, spread_groups  # noqa: F401  (shim is a fixture)


@pytest.mark.gpu
def test_three_ranks_return_identical_top_lists(shim, tmp_path):  # noqa: F811
    R, J, rng = 3, 6, np.random.default_rng(43)
    tabs, groups, _ = spread_groups(rng, 600)
    own = np.arange(len(groups)) % R
    per_rank = []
    for j in range(J):
        part = [g for i, g in enumerate(groups) if i % 4 != j % 4]
        w = [np.concatenate([g for i, g in enumerate(groups) if i % 4 != j % 4 and own[i] == r]) for r in range(R)]
        if j % 3 == 1:                                                            # keys on every rank
            w = [np.concatenate([x, np.concatenate(part[:50])]) for x in w]
        per_rank.append(w)
    rollups = [["window", 1], ["window", 3], ["tier", 1, 2], ["span", 5, abi.SPAN_AT_LEAST]]
    k, ms = 40, 0.3
    spec = {"nranks": R, "cfg": SMALL, "history": [3, 1 << 14], "tiers": [[2, 3, 1 << 14, 1 << 12]], "windows": J,
            "rollups": rollups, "k": k, "min_score": ms}
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
    p = subprocess.run([sys.executable, os.path.join(HERE, "loopback_gnn_top_ranks.py"), sp, ip, op], cwd=ROOT,
                       env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    z = np.load(op)
    meta = json.loads(str(z["meta"]))
    assert not meta["errors"], meta["errors"]
    assert meta["maps"] == [shim], meta["maps"]
    nonempty = 0
    for j in range(J):
        for s in range(1 + len(rollups)):
            for r in range(1, R):
                for x in ("top_{}_{}_{}_rows", "top_{}_{}_{}_scores", "top_{}_{}_{}_index", "info_{}_{}_{}"):
                    assert z[x.format(j, r, s)].tobytes() == z[x.format(j, 0, s)].tobytes(), (x, j, r, s)
            rows, scores = z[f"rows_{j}_0_{s}"], z[f"scores_{j}_0_{s}"]
            idx, above = top_ref.top(scores, k, ms)
            assert z[f"top_{j}_0_{s}_index"].tolist() == idx.tolist(), (j, s)
            assert z[f"top_{j}_0_{s}_rows"].tobytes() == rows[idx].tobytes(), (j, s)
            assert z[f"top_{j}_0_{s}_scores"].tobytes() == scores[idx].tobytes(), (j, s)
            assert z[f"info_{j}_0_{s}"].tolist() == [len(rows), above], (j, s)
            nonempty += len(idx) > 0
    assert nonempty >= J * (1 + len(rollups)) - 2                                 # tier 1 has no entry before window 2
