"""GPU: reach on several ranks, on one GPU through the loopback collective (tests/loopback_reach_ranks.py). Every rank
holds the same merged rows and sets the same map, so every rank returns the same records, row positions, rows and
info with no collective of its own, and they equal tests/reach_ref.py over the merged rows."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import group_ref as gr
import reach_ref as rr
from alaz_b200 import abi
from loopback_reach_ranks import DIRS, INFO
from test_gpu_loopback_ranks import HERE, ROOT, SMALL, shim, spread_groups  # noqa: F401  (shim is a fixture)


@pytest.mark.gpu
def test_three_ranks_return_identical_reach(shim, tmp_path):  # noqa: F811
    R, J, K, HOPS, rng = 3, 4, 3, 3, np.random.default_rng(63)
    tabs, groups, _ = spread_groups(rng, 600)
    own = np.arange(len(groups)) % R
    per_rank = []
    for j in range(J):
        w = [np.concatenate([g for i, g in enumerate(groups) if i % 4 != j % 4 and own[i] == r]) for r in range(R)]
        per_rank.append(w)
    spec = {"nranks": R, "cfg": SMALL, "history": [4, 1 << 14], "windows": J, "rollup": K, "max_hops": HOPS}
    arrays = {"tab0": np.asarray(tabs, np.int64).reshape(-1, 3)}
    # pods three per group; services unmapped
    pods = np.arange(600)
    arrays["map_types"] = np.full(len(pods), abi.NODE_POD, np.uint8)
    arrays["map_values"] = pods.astype(np.uint32)
    arrays["map_groups"] = (pods // 3).astype(np.uint32)
    gmap = gr.make_map(list(zip(arrays["map_types"].tolist(), arrays["map_values"].tolist())), arrays["map_groups"])
    # pods, the service every pod calls, and ids no row holds
    arrays["seed_types"] = np.array([abi.NODE_POD] * 4 + [abi.NODE_SVC, abi.NODE_SVC], np.uint8)
    arrays["seed_values"] = np.array([0, 5, 5, 599, 7, 8], np.uint32)
    arrays["gseed_types"] = np.array([abi.NODE_GROUP, abi.NODE_GROUP, abi.NODE_SVC], np.uint8)
    arrays["gseed_values"] = np.array([1, 150, 7], np.uint32)
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
    p = subprocess.run([sys.executable, os.path.join(HERE, "loopback_reach_ranks.py"), sp, ip, op], cwd=ROOT,
                       env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    z = np.load(op)
    meta = json.loads(str(z["meta"]))
    assert not meta["errors"], meta["errors"]
    assert meta["maps"] == [shim], meta["maps"]
    seeds = list(zip(arrays["seed_types"].tolist(), arrays["seed_values"].tolist()))
    gseeds = list(zip(arrays["gseed_types"].tolist(), arrays["gseed_values"].tolist()))
    names = ["win_{}_{}", "roll_{}_{}"] + [f"{f}{x}{s}{d}_{{}}_{{}}" for f in ("n", "g") for x in
                                           ("rec", "idx", "rows", "info") for s in (0, 1) for d in DIRS]
    listed = 0
    for j in range(J):
        for r in range(1, R):
            for x in names:
                assert z[x.format(j, r)].tobytes() == z[x.format(j, 0)].tobytes(), (x, j, r)
        for s, rows in enumerate((z[f"win_{j}_0"], z[f"roll_{j}_0"])):
            assert len(rows) > 0
            for d in DIRS:
                for f, exp in (("n", rr.reach(rows, seeds, d, HOPS)),
                               ("g", rr.group_reach(rows, gseeds, gmap, direction=d, max_hops=HOPS))):
                    what = (f, j, s, d)
                    assert z[f"{f}rec{s}{d}_{j}_0"].tobytes() == exp[0].tobytes(), what
                    assert z[f"{f}idx{s}{d}_{j}_0"].tobytes() == exp[1].tobytes(), what
                    assert z[f"{f}rows{s}{d}_{j}_0"].tobytes() == exp[2].tobytes(), what
                    assert z[f"{f}info{s}{d}_{j}_0"].tolist() == [exp[3][k] for k in INFO], what
                    listed += len(exp[0])
    assert listed > 0
