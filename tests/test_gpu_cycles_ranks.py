"""GPU: cycles on several ranks, on one GPU through the loopback collective (tests/loopback_cycles_ranks.py). Every
rank holds the same merged rows and sets the same map, so every rank returns the same records, row positions, rows and
info with no collective of its own, and they equal tests/cycle_ref.py over the merged rows."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import group_ref as gr
import cycle_ref as cr
from alaz_b200 import abi
from loopback_cycles_ranks import FILTERS, INFO
from test_gpu_loopback_ranks import HERE, ROOT, SMALL, shim, spread_groups  # noqa: F401  (shim is a fixture)


@pytest.mark.gpu
def test_three_ranks_return_identical_cycles(shim, tmp_path):  # noqa: F811
    R, J, K, rng = 3, 4, 3, np.random.default_rng(64)
    tabs, groups, _ = spread_groups(rng, 600)
    own = np.arange(len(groups)) % R
    per_rank = []
    for j in range(J):
        w = [np.concatenate([g for i, g in enumerate(groups) if i % 4 != j % 4 and own[i] == r]) for r in range(R)]
        per_rank.append(w)
    spec = {"nranks": R, "cfg": SMALL, "history": [4, 1 << 14], "windows": J, "rollup": K}
    arrays = {"tab0": np.asarray(tabs, np.int64).reshape(-1, 3)}
    # pods three per group; services unmapped
    pods = np.arange(600)
    arrays["map_types"] = np.full(len(pods), abi.NODE_POD, np.uint8)
    arrays["map_values"] = pods.astype(np.uint32)
    arrays["map_groups"] = (pods // 3).astype(np.uint32)
    gmap = gr.make_map(list(zip(arrays["map_types"].tolist(), arrays["map_values"].tolist())), arrays["map_groups"])
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
    p = subprocess.run([sys.executable, os.path.join(HERE, "loopback_cycles_ranks.py"), sp, ip, op], cwd=ROOT,
                       env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    z = np.load(op)
    meta = json.loads(str(z["meta"]))
    assert not meta["errors"], meta["errors"]
    assert meta["maps"] == [shim], meta["maps"]
    cases = range(len(FILTERS))
    names = ["win_{}_{}", "roll_{}_{}"] + [f"{f}{x}{s}{c}_{{}}_{{}}" for f in ("n", "g") for x in
                                           ("rec", "idx", "rows", "info") for s in (0, 1) for c in cases]
    listed = 0
    for j in range(J):
        for r in range(1, R):
            for x in names:
                assert z[x.format(j, r)].tobytes() == z[x.format(j, 0)].tobytes(), (x, j, r)
        for s, rows in enumerate((z[f"win_{j}_0"], z[f"roll_{j}_0"])):
            assert len(rows) > 0
            for c, (m, mv, ms) in enumerate(FILTERS):
                kw = dict(spec=m, min_value=mv, min_size=ms)
                for f, exp in (("n", cr.cycles(rows, **kw)), ("g", cr.group_cycles(rows, gmap, **kw))):
                    what = (f, j, s, c)
                    assert z[f"{f}rec{s}{c}_{j}_0"].tobytes() == exp[0].tobytes(), what
                    assert z[f"{f}idx{s}{c}_{j}_0"].tobytes() == exp[1].tobytes(), what
                    assert z[f"{f}rows{s}{c}_{j}_0"].tobytes() == exp[2].tobytes(), what
                    assert z[f"{f}info{s}{c}_{j}_0"].tolist() == [exp[3][k] for k in INFO], what
                    listed += len(exp[0])
    assert listed > 0
