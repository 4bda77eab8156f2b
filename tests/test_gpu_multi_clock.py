"""GPU, >= 2 devices: time-cut windows on several ranks (docs/SPEC.md §8 "Several ranks") over the real NCCL, one
handle per GPU: every rank opening in one epoch, and openings staggered by one epoch, against the model of
tests/window_ranks_model.py. Skipped with fewer GPUs than ranks, like tests/test_gpu_multi.py."""
import ctypes as C
import threading

import numpy as np
import pytest

from alaz_b200 import abi, capi
from helpers import edges_equal, explain_diff
from test_gpu_loopback_clock import FK, FU, SMALL, TABLES, W, Case

pytestmark = pytest.mark.gpu


def _ngpu():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.parametrize("stagger", [0, 1])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_clocked_ranks_on_several_gpus(world, stagger):
    if _ngpu() < world:
        pytest.skip(f"needs {world} GPUs")
    E0 = 10**6 + 9
    c = Case(world, seed=world + stagger)
    c.clock_all()
    per_rank = [[] for _ in range(world)]
    for r in range(world):
        per_rank[r].append(c.recs(r, [E0 + (stagger if r % 2 else 0)] * 200 + [E0 + 1] * 100 + [E0 - 1] * 10))
        c.submit(r, per_rank[r][-1])
    exp = [c.flush() for _ in range(3)]
    L = capi.load()
    idbuf = (C.c_uint8 * abi.COMM_ID_BYTES)()
    assert L.alz_comm_unique_id(idbuf) == 0
    out, errs = [None] * world, []
    bar = threading.Barrier(world, timeout=120)   # allocation and collective phases fenced apart (test_gpu_multi.py)

    def run(rank):
        try:
            h = capi.Handle(device=rank, **SMALL)
            h._ck(L.alz_comm_init(h.h, world, rank, idbuf), "alz_comm_init")
            h.upsert_batch(abi.TABLE_POD, TABLES[TABLES[:, 0] == abi.TABLE_POD, 1], TABLES[TABLES[:, 0] == abi.TABLE_POD, 2])
            h.upsert_batch(abi.TABLE_SVC, TABLES[TABLES[:, 0] == abi.TABLE_SVC, 1], TABLES[TABLES[:, 0] == abi.TABLE_SVC, 2])
            h.commit()
            h.window_clock(FK, FU, W)
            for x in per_rank[rank]:
                h.submit(x)
            h.sync()
            bar.wait()
            res = []
            for _ in range(3):
                res.append((h.flush(), h.window_epoch(), h.stats()))
            out[rank] = res
            bar.wait()
            h.close()
        except Exception as e:   # noqa: BLE001
            errs.append((rank, repr(e)))
            bar.abort()

    th = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for x in th:
        x.start()
    for x in th:
        x.join(timeout=300)
    assert not errs, errs
    for j, (st, rows) in enumerate(exp):
        assert st == abi.OK
        for r in range(world):
            got, epoch, stats = out[r][j]
            assert got.tobytes() == out[0][j][0].tobytes()
            assert edges_equal(got, rows), f"window {j} rank {r}: " + explain_diff(got, rows)
            assert epoch == c.snap[c.flush_indices()[j]][1][r]
            want = c.snap[c.flush_indices()[j]][0][r]
            for k in ("late_events", "deferred_events", "rows_emitted", "capacity_events", "windows"):
                assert stats[k] == want[k], (j, r, k, stats[k], want[k])
