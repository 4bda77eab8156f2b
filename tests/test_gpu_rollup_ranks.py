"""GPU: rolling windows on several ranks, on one GPU through the loopback collective (tests/loopback_rollup_ranks.py).
After a merge every rank holds the merged rows, so every rank's history, and every rank's rollup, is the same."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import loopback_ranks as lr
from alaz_b200 import abi
from rollup_model import RollupModel
from test_gpu_loopback_ranks import HERE, ROOT, SMALL, shim, spread_groups  # noqa: F401  (shim is a fixture)


def run_rollup_ranks(shim_lib, tmp_path, R, per_rank, tables, history, rollups):
    """per_rank[j][r]: records rank r submits in window j; rollups[j]: k of the rollup after window j's flush."""
    spec = {"nranks": R, "cfg": SMALL, "history": history, "rollups": rollups}
    arrays = {"tab0": np.asarray(tables, np.int64).reshape(-1, 3)}
    for j, w in enumerate(per_rank):
        for r in range(R):
            arrays[f"w{j}_r{r}"] = np.ascontiguousarray(w[r], dtype=abi.L7_REC)
    sp, ip, op = (str(tmp_path / x) for x in ("spec.json", "in.npz", "out.npz"))
    with open(sp, "w") as f:
        json.dump(spec, f)
    np.savez(ip, **arrays)
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = os.path.dirname(shim_lib) + os.pathsep + env.get("LD_LIBRARY_PATH", "")
    env["LOOPBACK_NCCL_TIMEOUT_S"] = "60"
    p = subprocess.run([sys.executable, os.path.join(HERE, "loopback_rollup_ranks.py"), sp, ip, op], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    z = np.load(op)
    meta = json.loads(str(z["meta"]))
    assert not meta["errors"], meta["errors"]
    assert meta["maps"] == [shim_lib], meta["maps"]     # the loopback library is the only libnccl of the process
    return z, meta


@pytest.mark.gpu
def test_three_ranks_disjoint_owners_and_one_general_window(shim, tmp_path):  # noqa: F811
    R, rng = 3, np.random.default_rng(21)
    tabs, groups, _ = spread_groups(rng, 600)
    own = np.arange(len(groups)) % R
    per_rank = []
    for j in range(4):
        part = [g for i, g in enumerate(groups) if i % 4 != j]                    # the windows' edge sets differ
        w = [np.concatenate([g for i, g in enumerate(groups) if i % 4 != j and own[i] == r]) for r in range(R)]
        if j == 1:                                                                # keys on every rank: the general path
            w = [np.concatenate([x, np.concatenate(part[:50])]) for x in w]
        per_rank.append(w)
    depth, ks = 3, [1, 2, 3, 4]
    z, meta = run_rollup_ranks(shim, tmp_path, R, per_rank, tabs, [depth, 1 << 14], ks)
    rank = lambda r: meta["ranks"][str(r)]
    m = RollupModel()
    m.history(depth, 1 << 14)
    for j, k in enumerate(ks):
        ops = [op for op, _ in rank(0)[j]["log"]]
        assert (lr.OP_ALLREDUCE in ops) == (j == 1), ops
        for r in range(R):
            assert rank(r)[j]["rc"] == abi.OK
            assert z[f"rows_{j}_{r}"].tobytes() == z[f"rows_{j}_0"].tobytes()
        m.append(z[f"rows_{j}_0"], rank(0)[j]["windows"])
        exp, info = m.rollup(k)
        assert info["windows"] == min(k, depth, j + 1)
        for r in range(R):
            assert rank(r)[j]["info"] == info, (r, j, rank(r)[j]["info"], info)
            assert z[f"rollup_{j}_{r}"].tobytes() == exp.tobytes(), (r, j)
        assert int(exp["count"].sum()) == sum(int(z[f"rows_{i}_0"]["count"].sum())
                                              for i in range(j + 1)[-info["windows"]:])
