"""GPU: group changes against a pinned baseline on several ranks, on one GPU through the loopback collective
(tests/loopback_group_changes_ranks.py). After a merge every rank holds the merged rows and sets the same map, so every
rank pins the same baseline, groups the same rows and compares the same sources: every rank returns the same group
edge and group node lists and top changes, with no collective of their own, and they equal tests/group_change_ref.py
over the merged rows."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import group_change_ref as gcr
import group_ref as gr
from alaz_b200 import abi
from loopback_group_changes_ranks import CASES, INFO
from test_gpu_loopback_ranks import HERE, ROOT, SMALL, shim, spread_groups  # noqa: F401  (shim is a fixture)


@pytest.mark.gpu
@pytest.mark.parametrize("pin", [["window"], ["span", 3, abi.SPAN_AT_MOST]])
def test_three_ranks_return_identical_group_changes(shim, tmp_path, pin):  # noqa: F811
    R, J, P, rng = 3, 7, 3, np.random.default_rng(58)
    tabs, groups, _ = spread_groups(rng, 600)
    own = np.arange(len(groups)) % R
    per_rank = []
    for j in range(J):
        part = [g for i, g in enumerate(groups) if i % 5 != j % 5]
        w = [np.concatenate([g for i, g in enumerate(groups) if i % 5 != j % 5 and own[i] == r]) for r in range(R)]
        if j % 3 == 1:                                                            # keys on every rank
            w = [np.concatenate([x, np.concatenate(part[:50])]) for x in w]
        per_rank.append(w)
    rollups = [["window", 2], ["tier", 1, 1], ["span", 4, abi.SPAN_AT_LEAST]]
    k, mc = 25, 0.0
    spec = {"nranks": R, "cfg": SMALL, "history": [4, 1 << 14], "tiers": [[2, 3, 1 << 14, 1 << 12]], "windows": J,
            "pin_after": P, "pin": pin, "rollups": rollups, "k": k, "min_change": mc}
    arrays = {"tab0": np.asarray(tabs, np.int64).reshape(-1, 3)}
    # pods three per group, services each its own group; outbound ends unmapped
    pods, svcs = np.arange(1 << 12), np.arange(1 << 8)
    arrays["map_types"] = np.r_[np.full(len(pods), abi.NODE_POD), np.full(len(svcs), abi.NODE_SVC)].astype(np.uint8)
    arrays["map_values"] = np.r_[pods, svcs].astype(np.uint32)
    arrays["map_groups"] = np.r_[pods // 3, (1 << 20) + svcs].astype(np.uint32)
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
    p = subprocess.run([sys.executable, os.path.join(HERE, "loopback_group_changes_ranks.py"), sp, ip, op], cwd=ROOT,
                       env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    z = np.load(op)
    meta = json.loads(str(z["meta"]))
    assert not meta["errors"], meta["errors"]
    assert meta["maps"] == [shim], meta["maps"]
    for r in range(1, R):
        assert z[f"base_{r}"].tobytes() == z["base_0"].tobytes()
    base, bw = z["base_0"], int(z["basew_0"][0])
    assert len(base) > 0
    listed = 0
    for j in range(P + 1, J):
        for s in range(1 + len(rollups)):
            names = [f"{x}{c}_{{}}_{{}}_{s}" for c in range(len(CASES)) for x in ("list", "top", "info", "tinfo")]
            for r in range(1, R):
                for x in names + [f"rows_{{}}_{{}}_{s}"]:
                    assert z[x.format(j, r)].tobytes() == z[x.format(j, 0)].tobytes(), (x, j, r, s)
            rows, w = z[f"rows_{j}_0_{s}"], int(z[f"win_{j}_0_{s}"][0])
            for c, (side, metric, mode, presence) in enumerate(CASES):
                if side is None:
                    lst, info = gcr.edge_changes(rows, base, gmap, metric, mode, presence, w, bw)
                else:
                    lst, info = gcr.node_changes(rows, base, gmap, side, metric, mode, presence, w, bw)
                assert z[f"list{c}_{j}_0_{s}"].tobytes() == lst.tobytes(), (j, s, c)
                assert z[f"info{c}_{j}_0_{s}"].tolist() == [info[x] for x in INFO], (j, s, c)
                top, tinfo = gcr.top(lst, info, k, mc)
                assert z[f"top{c}_{j}_0_{s}"].tobytes() == top.tobytes(), (j, s, c)
                assert z[f"tinfo{c}_{j}_0_{s}"].tolist() == [tinfo[x] for x in INFO], (j, s, c)
                listed += len(lst)
    assert listed > 0
