"""GPU: span rollups on several ranks, on one GPU through the loopback collective (tests/loopback_span_ranks.py).
After a merge every rank holds the merged rows, so every rank makes the same plan and returns the same rows with no
collective of its own."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from alaz_b200 import abi
from span_model import AT_LEAST, AT_MOST, SpanModel
from test_gpu_loopback_ranks import HERE, ROOT, SMALL, shim, spread_groups  # noqa: F401  (shim is a fixture)


@pytest.mark.gpu
def test_three_ranks_return_the_same_spans(shim, tmp_path):  # noqa: F811
    R, J, rng = 3, 9, np.random.default_rng(29)
    tabs, groups, _ = spread_groups(rng, 600)
    own = np.arange(len(groups)) % R
    per_rank = []
    for j in range(J):
        part = [g for i, g in enumerate(groups) if i % 4 != j % 4]                # the windows' edge sets differ
        w = [np.concatenate([g for i, g in enumerate(groups) if i % 4 != j % 4 and own[i] == r]) for r in range(R)]
        if j % 3 == 1:                                                            # keys on every rank: the general path
            w = [np.concatenate([x, np.concatenate(part[:50])]) for x in w]
        per_rank.append(w)
    history = [2, 1 << 14]
    tiers = [[2, 3, 1 << 14, 1 << 12], [2, 2, 1 << 14, 1 << 12]]
    spans = [[1, AT_MOST], [3, AT_MOST], [3, AT_LEAST], [5, AT_LEAST], [100, AT_LEAST]]
    spec = {"nranks": R, "cfg": SMALL, "history": history, "tiers": tiers, "windows": J, "spans": spans}
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
    p = subprocess.run([sys.executable, os.path.join(HERE, "loopback_span_ranks.py"), sp, ip, op], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    z = np.load(op)
    meta = json.loads(str(z["meta"]))
    assert not meta["errors"], meta["errors"]
    assert meta["maps"] == [shim], meta["maps"]
    rank = lambda r: meta["ranks"][str(r)]
    m = SpanModel()
    m.history(*history)
    m.configure(tiers)
    for j in range(J):
        for r in range(R):
            assert rank(r)[j]["rc"] == abi.OK
            assert z[f"rows_{j}_{r}"].tobytes() == z[f"rows_{j}_0"].tobytes()
        m.window(z[f"rows_{j}_0"], rank(0)[j]["windows"])
        for s, (N, mode) in enumerate(spans):
            exp, info = m.span(N, mode)
            for r in range(R):
                assert rank(r)[j]["info"][str(s)] == info, (r, j, s, rank(r)[j]["info"][str(s)], info)
                assert z[f"span_{j}_{r}_{s}"].tobytes() == exp.tobytes(), (r, j, s)
    assert m.span(100, AT_LEAST)[1]["windows"] == J
