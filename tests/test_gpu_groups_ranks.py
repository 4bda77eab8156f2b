"""GPU: groups on several ranks, on one GPU through the loopback collective (tests/loopback_groups_ranks.py). After a
merge every rank holds the merged rows and every rank sets the same map, so every rank returns the same group edges,
group nodes, values and top results of the window and of a window rollup, with no collective of its own, and they equal
tests/group_ref.py over the merged rows."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import group_ref as gr
import node_ref as nr
from alaz_b200 import abi
from loopback_groups_ranks import SPECS
from test_gpu_loopback_ranks import HERE, ROOT, SMALL, shim, spread_groups  # noqa: F401  (shim is a fixture)


@pytest.mark.gpu
def test_three_ranks_return_identical_groups(shim, tmp_path):  # noqa: F811
    R, J, K, TOP, rng = 3, 5, 3, 40, np.random.default_rng(59)
    tabs, groups, _ = spread_groups(rng, 600)
    own = np.arange(len(groups)) % R
    per_rank = []
    for j in range(J):
        part = [g for i, g in enumerate(groups) if i % 5 != j % 5]
        w = [np.concatenate([g for i, g in enumerate(groups) if i % 5 != j % 5 and own[i] == r]) for r in range(R)]
        if j % 3 == 1:                                                            # keys on every rank
            w = [np.concatenate([x, np.concatenate(part[:50])]) for x in w]
        per_rank.append(w)
    spec = {"nranks": R, "cfg": SMALL, "history": [4, 1 << 14], "windows": J, "rollup": K, "top": TOP}
    tab = np.asarray(tabs, np.int64).reshape(-1, 3)
    ids = np.unique(tab[:, [0, 2]], axis=0)                                       # (table, id): pod 0, service 1
    mnodes = np.zeros(len(ids), dtype=abi.NODE_ENDS)
    mnodes["type"], mnodes["value"] = ids[:, 0], ids[:, 1]
    mgroups = np.where(ids[:, 0] == abi.TABLE_POD, ids[:, 1] // 3, 1000 + ids[:, 1] % 5).astype(np.uint32)
    gmap = gr.make_map(mnodes, mgroups)
    arrays = {"tab0": tab, "map_nodes": mnodes, "map_groups": mgroups}
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
    p = subprocess.run([sys.executable, os.path.join(HERE, "loopback_groups_ranks.py"), sp, ip, op], cwd=ROOT,
                       env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    z = np.load(op)
    meta = json.loads(str(z["meta"]))
    assert not meta["errors"], meta["errors"]
    assert meta["maps"] == [shim], meta["maps"]
    names = ["win_{}_{}", "roll_{}_{}"] + [f"{x}{s}_{{}}_{{}}" for s in (0, 1)
                                           for x in ("edges", "einfo", "emet", "etop", "eidx", "nodes")] + \
        [f"{x}{s}{side}_{{}}_{{}}" for s in (0, 1) for side in (0, 1) for x in ("val", "top", "tval", "tidx")]
    for j in range(J):
        for r in range(1, R):
            for x in names:
                assert z[x.format(j, r)].tobytes() == z[x.format(j, 0)].tobytes(), (x, j, r)
        for s, rows in enumerate((z[f"win_{j}_0"], z[f"roll_{j}_0"])):
            edges, info = gr.group(rows, gmap)
            assert len(edges) > 0 and z[f"edges{s}_{j}_0"].tobytes() == edges.tobytes(), (j, s)
            assert list(z[f"einfo{s}_{j}_0"]) == [info[k] for k in sorted(info)], (j, s)
            assert info["mapped_ends"] > 0
            assert z[f"emet{s}_{j}_0"].tobytes() == gr.edge_matrix(edges, SPECS).tobytes(), (j, s)
            idx, _ = gr.edge_top(edges, SPECS[0], TOP, -np.inf)
            assert z[f"eidx{s}_{j}_0"].tobytes() == idx.tobytes() and z[f"etop{s}_{j}_0"].tobytes() == \
                edges[idx].tobytes(), (j, s)
            exp = nr.group(edges)
            assert z[f"nodes{s}_{j}_0"].tobytes() == exp.tobytes(), (j, s)
            for side in (abi.SIDE_IN, abi.SIDE_OUT):
                assert z[f"val{s}{side}_{j}_0"].tobytes() == nr.matrix(exp, side, SPECS).tobytes(), (j, s, side)
                idx, _ = nr.top(exp, side, SPECS[side], TOP, -np.inf)
                assert z[f"tidx{s}{side}_{j}_0"].tobytes() == idx.tobytes(), (j, s, side)
                assert z[f"top{s}{side}_{j}_0"].tobytes() == exp[idx].tobytes(), (j, s, side)
                assert z[f"tval{s}{side}_{j}_0"].tobytes() == nr.values(exp, side, SPECS[side])[idx].tobytes()
