"""GPU: edge metrics and top edges on several ranks, on one GPU through the loopback collective
(tests/loopback_edge_top_ranks.py). After a merge every rank holds the merged rows, so every rank's window and rollup
rows are the same, and so are their metrics and top lists, with no collective of their own."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import metric_ref as mr
from alaz_b200 import abi
from loopback_edge_top_ranks import METRICS, TOPS
from test_gpu_loopback_ranks import HERE, ROOT, SMALL, shim, spread_groups  # noqa: F401  (shim is a fixture)


@pytest.mark.gpu
def test_three_ranks_return_identical_metrics_and_top_edges(shim, tmp_path):  # noqa: F811
    R, J, rng = 3, 6, np.random.default_rng(47)
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
    k, ms = 40, 0.0
    spec = {"nranks": R, "cfg": SMALL, "history": [3, 1 << 14], "tiers": [[2, 3, 1 << 14, 1 << 12]], "windows": J,
            "rollups": rollups, "k": k, "min_value": ms}
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
    p = subprocess.run([sys.executable, os.path.join(HERE, "loopback_edge_top_ranks.py"), sp, ip, op], cwd=ROOT,
                       env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    z = np.load(op)
    meta = json.loads(str(z["meta"]))
    assert not meta["errors"], meta["errors"]
    assert meta["maps"] == [shim], meta["maps"]
    nonempty = 0
    for j in range(J):
        for s in range(1 + len(rollups)):
            names = [f"values_{{}}_{{}}_{s}"] + [f"{x}{t}_{{}}_{{}}_{s}{y}" for t in range(len(TOPS))
                                                for x, y in (("top", "_rows"), ("top", "_values"), ("top", "_index"),
                                                             ("info", ""))]
            for r in range(1, R):
                for x in names:
                    assert z[x.format(j, r)].tobytes() == z[x.format(j, 0)].tobytes(), (x, j, r, s)
            rows = z[f"rows_{j}_0_{s}"]
            assert z[f"values_{j}_0_{s}"].tobytes() == mr.matrix(rows, METRICS).tobytes(), (j, s)
            for t, spec_t in enumerate(TOPS):
                v = mr.values(rows, spec_t)
                idx, above = mr.top(v, k, ms)
                assert z[f"top{t}_{j}_0_{s}_index"].tolist() == idx.tolist(), (j, s, t)
                assert z[f"top{t}_{j}_0_{s}_rows"].tobytes() == rows[idx].tobytes(), (j, s, t)
                assert z[f"top{t}_{j}_0_{s}_values"].tobytes() == v[idx].tobytes(), (j, s, t)
                assert z[f"info{t}_{j}_0_{s}"].tolist() == [len(rows), above], (j, s, t)
            nonempty += len(rows) > 0
    assert nonempty >= J * (1 + len(rollups)) - 2                                 # tier 1 has no entry before window 2
