"""GPU: group series and group trends on several ranks, on one GPU through the loopback collective
(tests/loopback_group_series_ranks.py). Every rank holds the same merged history and sets the same map, so every rank
returns the same group edge and group node series, records, rows and top series with no collective of its own, and
they equal tests/group_series_ref.py over the merged windows."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import group_ref as gr
import group_series_ref as gsr
import node_ref as nr
from alaz_b200 import abi
from loopback_group_series_ranks import SPECS, TREND
from test_gpu_loopback_ranks import HERE, ROOT, SMALL, shim, spread_groups  # noqa: F401  (shim is a fixture)


@pytest.mark.gpu
def test_three_ranks_return_identical_group_series(shim, tmp_path):  # noqa: F811
    R, J, K, TOP, DEPTH, rng = 3, 5, 3, 30, 4, np.random.default_rng(62)
    tabs, groups, _ = spread_groups(rng, 600)
    own = np.arange(len(groups)) % R
    per_rank = []
    for j in range(J):
        part = [g for i, g in enumerate(groups) if i % 5 != j % 5]
        w = [np.concatenate([g for i, g in enumerate(groups) if i % 5 != j % 5 and own[i] == r]) for r in range(R)]
        if j % 3 == 1:                                                            # keys on every rank
            w = [np.concatenate([x, np.concatenate(part[:50])]) for x in w]
        per_rank.append(w)
    spec = {"nranks": R, "cfg": SMALL, "history": [DEPTH, 1 << 14], "windows": J, "rollup": K, "top": TOP}
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
    p = subprocess.run([sys.executable, os.path.join(HERE, "loopback_group_series_ranks.py"), sp, ip, op], cwd=ROOT,
                       env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    z = np.load(op)
    meta = json.loads(str(z["meta"]))
    assert not meta["errors"], meta["errors"]
    assert meta["maps"] == [shim], meta["maps"]
    names = ["win_{}_{}", "roll_{}_{}"] + [f"{x}{s}_{{}}_{{}}" for s in (0, 1) for x in ("eser", "epres")] + \
        [f"{x}{s}{d}_{{}}_{{}}" for s in (0, 1) for d in (0, 1) for x in ("ser", "pres")]
    tops = [f"{x}{y}_{{}}_{{}}" for x in ("e", "n") for y in ("trec", "trows", "tser", "tpres")]
    grouped = 0
    for j in range(J):
        for r in range(1, R):
            for x in names + (tops if j >= 1 else []):
                assert z[x.format(j, r)].tobytes() == z[x.format(j, 0)].tobytes(), (x, j, r)
        entries = [z[f"win_{i}_0"] for i in range(max(0, j + 1 - DEPTH), j + 1)]
        for s, rows in enumerate((z[f"win_{j}_0"], z[f"roll_{j}_0"])):
            ge = gsr.source_edges(rows, gmap)
            keys = nr.keys(ge)
            assert len(keys) > 0
            grouped += int((ge["from_type"] == abi.NODE_GROUP).sum())
            v, pr = gsr.edge_series(entries, *gsr.row_ends(ge), SPECS, gmap, DEPTH)
            assert z[f"epres{s}_{j}_0"].tobytes() == pr.tobytes(), (j, s)
            assert z[f"eser{s}_{j}_0"].tobytes() == v.tobytes(), (j, s)
            for d in (abi.SIDE_IN, abi.SIDE_OUT):
                v, pr = gsr.node_series(entries, keys, d, SPECS, gmap, DEPTH)
                assert z[f"pres{s}{d}_{j}_0"].tobytes() == pr.tobytes(), (j, s, d)
                assert z[f"ser{s}{d}_{j}_0"].tobytes() == v.tobytes(), (j, s, d)
        if j >= 1:
            rows = z[f"roll_{j}_0"]
            for x, (rec, y, pr), srows in (
                    ("e", gsr.edge_expect(entries, rows, abi.METRIC_COUNT, DEPTH, gmap, **TREND),
                     gsr.source_edges(rows, gmap)),
                    ("n", gsr.node_expect(entries, rows, abi.SIDE_IN, abi.METRIC_COUNT, DEPTH, gmap, **TREND),
                     gsr.source_nodes(rows, gmap))):
                idx, _ = gsr.top(rec, TOP)
                assert z[f"{x}trec_{j}_0"].tobytes() == rec[idx].tobytes(), (x, j)
                assert z[f"{x}trows_{j}_0"].tobytes() == srows[idx].tobytes(), (x, j)
                assert z[f"{x}tser_{j}_0"].tobytes() == y[idx].tobytes(), (x, j)
                assert z[f"{x}tpres_{j}_0"].tobytes() == pr[idx].tobytes(), (x, j)
    assert grouped > 0
