"""The multi-rank window merge (alaz_b200/csrc/alz_comm.cu) on ONE GPU: 2 to 64 ranks of one process talk through a
loopback collective (tests/loopback_nccl.cu) that takes the place of libnccl.so.2 in a child process
(tests/loopback_ranks.py). Every rank's rows are compared with the single-rank oracle on all the ranks' records, and
with every other rank's byte for byte; the statuses, the stats sums across ranks and each rank's collective log are
checked too. CPU tests at the end build the loopback library and pin the numpy restatements the cases are made with.
"""
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import loopback_ranks as lr
import oracle_lib as ol
from alaz_b200 import abi
from gnn_graphs import POD_NET, SVC_NET
from helpers import edges_equal, explain_diff
from test_gpu_flush import oracle_edges, records

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CAN_WORDS = 3 + 64                     # u64 words per row of the general path's all-reduce
SMALL = dict(max_endpoints=1 << 14, max_pairs=1 << 15, max_edges=1 << 14, max_batch=1 << 16)
NCCL_EXPORTS = ["ncclGetUniqueId", "ncclCommInitRank", "ncclCommDestroy", "ncclAllGather", "ncclAllReduce",
                "ncclGetErrorString"]


def build_shim(out_dir):
    nvcc = shutil.which("nvcc") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    lib = os.path.join(str(out_dir), "libnccl.so.2")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
           "-Xlinker", "-soname=libnccl.so.2", os.path.join(HERE, "loopback_nccl.cu"), "-o", lib]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return lib


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    """The loopback libnccl.so.2, built into a temporary directory."""
    return build_shim(tmp_path_factory.mktemp("loopback_nccl"))


class Run:
    def __init__(self, npz, R):
        self.z, self.R = npz, R
        self.meta = json.loads(str(npz["meta"]))

    def rank(self, r):
        return self.meta["ranks"][str(r)]

    def rows(self, j, r):
        return self.z[f"rows_{j}_{r}"]

    def solo(self, j):
        return self.meta["solo"][j], self.z[f"rows_{j}_solo"]

    def stat_sum(self, j, name):
        return sum(self.rank(r)[j]["stats"][name] for r in range(self.R))

    def stat_delta(self, j, name):
        """a cumulative counter's growth over window j, summed over the ranks"""
        return self.stat_sum(j, name) - (self.stat_sum(j - 1, name) if j else 0)


def run_ranks(shim, tmp_path, R, per_rank, tables, cfg=SMALL, windows=None, cfg_rank=None, fault=None,
              solo=False, commits=None, timeout=600, init_only=False):
    """per_rank[j][r]: records rank r submits in window j. tables: (table, ip, id) rows."""
    spec = {"nranks": R, "cfg": cfg, "cfg_rank": cfg_rank or {}, "tables": 1,
            "windows": windows or [{} for _ in per_rank], "fault": fault, "solo": solo, "init_only": init_only}
    arrays = {"tab0": np.asarray(tables, np.int64).reshape(-1, 3)}
    for j, w in enumerate(per_rank):
        for r in range(R):
            arrays[f"w{j}_r{r}"] = np.ascontiguousarray(w[r], dtype=abi.L7_REC)
    for j, c in (commits or {}).items():
        arrays[f"commit{j}"] = np.asarray(c, np.int64).reshape(-1, 3)
    sp, ip, op = (str(tmp_path / x) for x in ("spec.json", "in.npz", "out.npz"))
    with open(sp, "w") as f:
        json.dump(spec, f)
    np.savez(ip, **arrays)
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = os.path.dirname(shim) + os.pathsep + env.get("LD_LIBRARY_PATH", "")
    env["LOOPBACK_NCCL_TIMEOUT_S"] = "5" if init_only else "60"
    p = subprocess.run([sys.executable, os.path.join(HERE, "loopback_ranks.py"), sp, ip, op], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=timeout)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    run = Run(np.load(op), R)
    assert not run.meta["errors"], run.meta["errors"]
    if not init_only:
        # the loopback library is the only libnccl of the process
        assert run.meta["maps"] == [shim], run.meta["maps"]
    return run


def table_rows(tab, ips, ids):
    return np.stack([np.full(len(ips), tab, np.int64), np.asarray(ips, np.int64), np.asarray(ids, np.int64)], 1)


def tables_of(rows):
    """table rows -> the (table, ips, ids) list oracle_edges takes"""
    rows = np.asarray(rows, np.int64).reshape(-1, 3)
    return [(tab, rows[rows[:, 0] == tab, 1], rows[rows[:, 0] == tab, 2]) for tab in (abi.TABLE_POD, abi.TABLE_SVC)]


def keys_of(rows):
    return np.array([lr.row_key_of(x) for x in rows], dtype=np.uint64)


def expect_log(R, counts_per_window):
    """Each window's collectives on the default path with no key on two ranks, from the ranks' local row counts:
    a count gather before the first window only, then a block gather of (cap + 1) rows per rank, sent again
    larger when the largest count exceeds cap. Returns (logs, collective_bytes_last per window)."""
    cap, logs, nbytes = 0, [], []
    for counts in counts_per_window:
        mx, log = max(counts), []
        if cap == 0:
            log.append([lr.OP_ALLGATHER, 4 * R])
            cap = lr.block_rows_for(mx)
        if mx > cap:
            log.append([lr.OP_ALLGATHER, (cap + 1) * R * lr.ROW_BYTES])
            cap = lr.block_rows_for(mx)
        log.append([lr.OP_ALLGATHER, (cap + 1) * R * lr.ROW_BYTES])
        cap = lr.block_rows_for(mx)
        logs.append(log)
        nbytes.append(sum(b for _, b in log if b >= 1025 * R * lr.ROW_BYTES))   # the block gathers
    return logs, nbytes


def check_window(run, j, exp, rc=abi.OK, events=None, since_start=False):
    """Every rank: status rc, the same bytes, equal to the oracle's edges in canonical order; stats sums over the
    window (since_start: over every window so far, when earlier windows were kept)."""
    rows0 = run.rows(j, 0)
    for r in range(run.R):
        d = run.rank(r)[j]
        assert d["rc"] == rc, (r, d["rc"])
        assert d["n_out"] == len(rows0)
        assert run.rows(j, r).tobytes() == rows0.tobytes(), f"rank {r} differs from rank 0"
    assert edges_equal(rows0, exp), explain_diff(rows0, exp)
    k = keys_of(rows0)
    assert np.all(k[1:] > k[:-1]), "rows not in canonical (ascending packed key) order"
    if events is not None:
        assert run.stat_sum(j, "events_in") == events
    if rc == abi.OK:
        grew = run.stat_sum if since_start else run.stat_delta
        assert grew(j, "rows_emitted") == int(exp["count"].sum())
        assert grew(j, "capacity_events") == 0
    return rows0


def cumulative_events(per_rank, j):
    return sum(len(per_rank[i][r]) for i in range(j + 1) for r in range(len(per_rank[i])))


# ---- streams ------------------------------------------------------------------------------------------------
def topo_case(R, n_events, seed, n_windows=2):
    """Topo stream with every protocol plus Host-keyed rows, each window routed by alz_owner_rank."""
    t = ol.Topo(600, seed=seed, mix=abi.MIX_ALL)
    tabs = np.concatenate([table_rows(abi.TABLE_POD, t.pod_ip, np.arange(len(t.pod_ip))),
                           table_rows(abi.TABLE_SVC, t.svc_ip, np.arange(len(t.svc_ip)))])
    rng = np.random.default_rng(seed)
    per_rank, exps, counts = [], [], []

    def expect(ev, hosts):
        o = ol.Oracle()
        o.load_tables(t.pod_ip, t.svc_ip)
        o.process(ev, 4)
        e = np.concatenate([o.edges(), oracle_edges(tables_of(tabs), hosts, range(1, 40))])
        o.close()
        return e

    for j in range(n_windows):
        ev = t.events(j * n_events, n_events)
        nh = n_events // 20
        hosts = records(t.pod_ip[rng.integers(0, len(t.pod_ip), nh)], rng.integers(1, 40, nh), rng,
                        host=np.ones(nh, bool))
        exps.append(expect(ev, hosts))
        own_e, own_h = lr.owner_rank(ev["saddr"], R), lr.owner_rank(hosts["saddr"], R)
        per_rank.append([np.concatenate([ev[own_e == r], hosts[own_h == r]]) for r in range(R)])
        counts.append([len(expect(ev[own_e == r], hosts[own_h == r])) for r in range(R)])   # each rank's own rows
    t.close()
    return tabs, per_rank, exps, counts


@pytest.mark.gpu
@pytest.mark.parametrize("R", [2, 3, 8, 9, 17, 64])
def test_topo_disjoint_owners(shim, tmp_path, R):
    """Records routed by alz_owner_rank: every rank returns the single-rank oracle's rows, the same bytes on every
    rank; a second window of the same topology starts from zero; the collectives are one count gather before the
    first window and one block gather per window, sized from the largest rank."""
    n = 20_000 if R == 64 else 60_000
    tabs, per_rank, exps, counts = topo_case(R, n, seed=100 + R)
    run = run_ranks(shim, tmp_path, R, per_rank, tabs, solo=True)
    logs, nbytes = expect_log(R, counts)
    for j in range(len(per_rank)):
        rows = check_window(run, j, exps[j], events=cumulative_events(per_rank, j))
        for r in range(R):
            assert run.rank(r)[j]["log"] == logs[j], (j, r)
            assert run.rank(r)[j]["stats"]["collective_bytes_last"] == nbytes[j]
        d, solo = run.solo(j)
        assert d["rc"] == abi.OK and solo.tobytes() == rows.tobytes()


def edge_groups(rng):
    """Record groups, one edge each, at the ends of the packed key space: pod ids 0 and 2^29 - 1, outbound
    addresses 0.0.0.1 and 255.255.255.255, service rows and their reversed (AMQP DELIVER) twins, reversed outbound
    rows, Host-keyed rows (type 3) and pod <-> pod rows from both sides (one canonical edge)."""
    LO, HI = 0, (1 << 29) - 1
    pods = {LO: POD_NET + 1, HI: POD_NET + 2, 5: POD_NET + 3, 6: POD_NET + 4}
    svcs = {0: SVC_NET + 1, 9: SVC_NET + 2}
    tabs = np.concatenate([table_rows(abi.TABLE_POD, list(pods.values()), list(pods.keys())),
                           table_rows(abi.TABLE_SVC, list(svcs.values()), list(svcs.keys()))])
    groups = []
    for pid, pip in pods.items():
        for other in (1, 0xFFFFFFFF, abi.ip("8.8.8.8")):
            groups.append(records(np.full(3, pip), np.full(3, other), rng))                     # pod -> outbound
            groups.append(records(np.full(2, pip), np.full(2, other), rng, reversed_=np.ones(2, bool)))  # rev
        for sip in svcs.values():
            groups.append(records(np.full(4, pip), np.full(4, sip), rng))
            groups.append(records(np.full(2, pip), np.full(2, sip), rng, reversed_=np.ones(2, bool)))
        for host in (1, 0xFFFFFFFF):
            groups.append(records(np.full(3, pip), np.full(3, host), rng, host=np.ones(3, bool)))
    ids = list(pods.items())
    for a in range(len(ids)):
        for b in range(a + 1, len(ids)):
            fw = records(np.full(2, ids[a][1]), np.full(2, ids[b][1]), rng)
            bw = records(np.full(2, ids[b][1]), np.full(2, ids[a][1]), rng, reversed_=np.ones(2, bool))
            groups.append(np.concatenate([fw, bw]))
    return tabs, groups, [1, 0xFFFFFFFF]


def spread_groups(rng, n):
    """n pods, one service each: edge i has a key that grows with i."""
    tabs = np.concatenate([table_rows(abi.TABLE_POD, POD_NET + np.arange(n), np.arange(n)),
                           table_rows(abi.TABLE_SVC, [SVC_NET], [7])])
    return tabs, [records(np.full(1 + i % 3, POD_NET + i), np.full(1 + i % 3, SVC_NET), rng) for i in range(n)], []


LAYOUTS = ["rank_order", "reverse_order", "interleaved", "extreme_interleaved", "extreme_reverse", "some_empty",
           "one_rank", "all_empty"]


@pytest.mark.gpu
@pytest.mark.parametrize("R", [5, 9])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_constructed_layouts(shim, tmp_path, R, layout):
    """Edges placed on chosen ranks: key ranges in rank order and in reverse, key i on rank i mod R, the extreme
    keys interleaved and reversed, ranks with no rows, every row on one rank, every rank empty. Nine ranks make the
    eight lanes of a row's binary searches take a second pass; five need the third shuffle step."""
    rng = np.random.default_rng(R * 100 + LAYOUTS.index(layout))
    if layout.startswith("extreme"):
        tabs, groups, host_ids = edge_groups(rng)
        keys = [lr.row_key_of(e[0]) for e in (oracle_edges(tables_of(tabs), g, [1, 0xFFFFFFFF]) for g in groups)]
        order = np.argsort(np.array(keys, np.uint64))
        rank_of = np.empty(len(groups), int)
        rank_of[order] = np.arange(len(groups)) % R if layout == "extreme_interleaved" else \
            (R - 1 - np.arange(len(groups)) * R // len(groups))
    else:
        tabs, groups, host_ids = spread_groups(rng, 3000)
        i = np.arange(len(groups))
        rank_of = {"rank_order": i * R // len(i), "reverse_order": R - 1 - i * R // len(i), "interleaved": i % R,
                   "some_empty": np.where(i % 2 == 0, 1, R - 2), "one_rank": np.full(len(i), R // 2),
                   "all_empty": np.zeros(len(i), int)}[layout]
        if layout == "all_empty":
            groups = []
            rank_of = rank_of[:0]
    w = [np.concatenate([g for g, q in zip(groups, rank_of) if q == r] or [np.zeros(0, abi.L7_REC)])
         for r in range(R)]
    allrecs = np.concatenate(w)
    exp = oracle_edges(tables_of(tabs), allrecs, host_ids) if len(allrecs) else np.zeros(0, abi.EDGE_OUT)
    run = run_ranks(shim, tmp_path, R, [w, w], tabs, windows=[{}, {"flush": "device"}])
    rows = check_window(run, 0, exp, events=len(allrecs))
    for r in range(R):   # the device flush of the same records: the same bytes
        assert run.rank(r)[1]["rc"] == abi.OK
        assert run.rows(1, r).tobytes() == rows.tobytes()


def outbound_fan(pod_id, pod_ip, n, base, rng):
    """n edges pod -> n distinct outbound addresses, one record each"""
    return records(np.full(n, pod_ip), base + np.arange(n), rng)


@pytest.mark.gpu
def test_block_sizing(shim, tmp_path):
    """The block of the all-gather: the first window sizes it from the largest rank's count (a count gather, then
    one block gather); a window whose largest rank has exactly cap rows needs one gather; cap + 1 rows two, the
    second larger (the receive buffer grows); a smaller window a smaller block. collective_bytes_last is the sum
    over the attempts of (cap + 1) * R * 296."""
    R, rng = 4, np.random.default_rng(7)
    tabs = table_rows(abi.TABLE_POD, POD_NET + np.arange(R), np.arange(R))
    c0 = lr.block_rows_for(1000)
    c1 = lr.block_rows_for(c0)
    biggest = [1000, c0, c1 + 1, 100, 5]
    per_rank, counts = [], []
    for j, mx in enumerate(biggest):
        cnt = [mx, mx // 3, 0, 17][j % R:] + [mx, mx // 3, 0, 17][:j % R]
        per_rank.append([outbound_fan(r, POD_NET + r, cnt[r], abi.ip("11.0.0.0") + j * (1 << 20), rng)
                         for r in range(R)])
        counts.append(cnt)
    cfg = dict(SMALL, max_edges=1 << 15, max_pairs=1 << 15)
    run = run_ranks(shim, tmp_path, R, per_rank, tabs, cfg=cfg)
    logs, nbytes = expect_log(R, counts)
    assert [len(x) for x in logs] == [2, 1, 2, 1, 1]
    for j in range(len(biggest)):
        exp = oracle_edges(tables_of(tabs), np.concatenate(per_rank[j]))
        check_window(run, j, exp)
        for r in range(R):
            assert run.rank(r)[j]["log"] == logs[j], (j, r, run.rank(r)[j]["log"], logs[j])
            assert run.rank(r)[j]["stats"]["collective_bytes_last"] == nbytes[j]


GENERAL = ["first_n_to_all", "one_key_all_ranks", "two_ranks", "lat_wrap"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", GENERAL)
def test_general_path(shim, tmp_path, case):
    """Keys on several ranks take the sort + unique + all-reduce path: the first N records sent to every rank; one
    key on all ranks; keys on exactly two ranks; latency sums that wrap mod 2^64 across ranks. The ranks hold
    unequal counts, so the gathered key lists carry padding keys. Windows alternate disjoint and overlapping on
    the same edges, so nothing may carry over from one to the next."""
    R, rng = 6, np.random.default_rng(GENERAL.index(case))
    tabs, groups, _ = spread_groups(rng, 1500)
    own = np.arange(len(groups)) % R
    own[: len(groups) // 3] = 0          # unequal counts
    base = [np.concatenate([g for g, q in zip(groups, own) if q == r]) for r in range(R)]
    per_rank = []
    for j in range(4):
        w = [b.copy() for b in base]
        if j % 2 == 1:
            if case == "first_n_to_all":
                extra = np.concatenate(groups[:200])
                w = [np.concatenate([x, extra]) for x in w]
            elif case == "one_key_all_ranks":
                one = records(np.full(R * 3, POD_NET + 11), np.full(R * 3, SVC_NET), rng)
                w = [np.concatenate([x, one[3 * r: 3 * r + 3]]) for r, x in enumerate(w)]
            elif case == "two_ranks":
                for r in range(R):
                    w[(r + 1) % R] = np.concatenate([w[(r + 1) % R], groups[r * 7 + 100]])
            else:
                big = records(np.full(2 * R, POD_NET + 20), np.full(2 * R, SVC_NET), rng)
                big["duration_ns"] = np.uint64(1 << 63) + rng.integers(0, 1 << 40, 2 * R).astype(np.uint64)
                w = [np.concatenate([x, big[2 * r: 2 * r + 2]]) for r, x in enumerate(w)]
        per_rank.append(w)
    run = run_ranks(shim, tmp_path, R, per_rank, tabs)
    for j in range(4):
        exp = oracle_edges(tables_of(tabs), np.concatenate(per_rank[j]))
        if case == "lat_wrap" and j % 2:
            allr = np.concatenate(per_rank[j])
            tot = sum(int(x) for x in allr["duration_ns"][allr["saddr"] == POD_NET + 20])
            assert tot >= 1 << 64 and int(exp["lat_sum_ns"][exp["from"] == 20][0]) == tot % (1 << 64)
        check_window(run, j, exp, events=cumulative_events(per_rank, j))
        ops = [op for op, _ in run.rank(0)[j]["log"]]
        assert (lr.OP_ALLREDUCE in ops) == (j % 2 == 1), ops
        if j % 2:
            n_can = len(exp)
            blocks = sum(b for op, b in run.rank(0)[j]["log"] if op == lr.OP_ALLGATHER and b % (R * lr.ROW_BYTES) == 0
                         and b >= 1025 * R * lr.ROW_BYTES)
            assert run.rank(0)[j]["log"][-1] == [lr.OP_ALLREDUCE, n_can * CAN_WORDS * 8]
            assert run.rank(0)[j]["stats"]["collective_bytes_last"] == blocks + n_can * CAN_WORDS * 8


# ---- capacity and failures ----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_local_loss_is_every_ranks_capacity(shim, tmp_path):
    """Rank 1's pair table overflows: every rank returns ALZ_E_CAPACITY with the same rows, the other ranks' edges
    are exact, the ranks' rows_emitted add up to the rows returned, and the next window is exact and ALZ_OK."""
    R, rng = 4, np.random.default_rng(3)
    n_pods = 400
    tabs = np.concatenate([table_rows(abi.TABLE_POD, POD_NET + np.arange(n_pods), np.arange(n_pods)),
                           table_rows(abi.TABLE_SVC, [SVC_NET], [7])])
    w0 = [records(np.full(5, POD_NET + r), np.full(5, SVC_NET), rng) for r in range(R)]
    # rank 1: 6000 distinct socket pairs from its own pods in a 1024-row pair table
    w0[1] = records(POD_NET + 100 + np.arange(6000) % 300, abi.ip("12.0.0.0") + np.arange(6000), rng)
    w1 = [records(np.full(3, POD_NET + r), np.full(3, SVC_NET), rng) for r in range(R)]
    run = run_ranks(shim, tmp_path, R, [w0, w1], tabs, cfg_rank={"1": {"max_pairs": 1024}})
    rows = run.rows(0, 0)
    assert run.rank(1)[0]["stats"]["capacity_events"] > 0
    for r in range(R):
        assert run.rank(r)[0]["rc"] == abi.E_CAPACITY, (r, run.rank(r)[0]["rc"])
        assert run.rows(0, r).tobytes() == rows.tobytes()
    others = oracle_edges(tables_of(tabs), np.concatenate([w0[r] for r in range(R) if r != 1]))
    mine = rows[rows["from"] < 100]
    assert edges_equal(mine, others), explain_diff(mine, others)
    assert run.stat_sum(0, "rows_emitted") == int(rows["count"].sum())
    check_window(run, 1, oracle_edges(tables_of(tabs), np.concatenate(w1)))
    assert run.stat_delta(1, "capacity_events") == 0


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["host", "device"])
def test_merged_graph_over_max_edges(shim, tmp_path, path):
    """Every rank under max_edges, the union over it: every rank returns ALZ_E_CAPACITY with the first max_edges
    rows of the canonical order, consumes its window and counts the events of its own rows past the cut as lost;
    the next window is exact."""
    R, rng, me = 3, np.random.default_rng(4), 4096
    tabs = table_rows(abi.TABLE_POD, POD_NET + np.arange(R), np.arange(R))
    w0 = [outbound_fan(r, POD_NET + r, 2000, abi.ip("13.0.0.0") + (r % 2) * 3000, rng) for r in range(R)]
    w0 = [np.concatenate([x, x[: 500 * (r + 1)]]) for r, x in enumerate(w0)]   # counts 1 and 2 per edge
    w1 = [outbound_fan(r, POD_NET + r, 10, abi.ip("14.0.0.0"), rng) for r in range(R)]
    cfg = dict(SMALL, max_edges=me, max_pairs=1 << 14)
    run = run_ranks(shim, tmp_path, R, [w0, w1], tabs, cfg=cfg,
                    windows=[{"flush": path}, {"flush": path}])
    exp = lr.canonical(oracle_edges(tables_of(tabs), np.concatenate(w0)))
    assert len(exp) == 6000
    rows = run.rows(0, 0)
    for r in range(R):
        d = run.rank(r)[0]
        assert d["rc"] == abi.E_CAPACITY and d["n_out"] == me, (r, d)
        assert run.rows(0, r).tobytes() == rows.tobytes()
    assert edges_equal(rows, exp[:me]), explain_diff(rows, exp[:me])
    assert keys_of(rows).tolist() == keys_of(exp[:me]).tolist()
    assert run.stat_sum(0, "rows_emitted") == int(rows["count"].sum())
    assert run.stat_sum(0, "capacity_events") == int(exp["count"][me:].sum())
    check_window(run, 1, oracle_edges(tables_of(tabs), np.concatenate(w1)), events=cumulative_events([w0, w1], 1))
    assert run.stat_sum(1, "capacity_events") == int(exp["count"][me:].sum())


@pytest.mark.gpu
def test_general_path_gather_bound(shim, tmp_path):
    """Keys on several ranks whose gathered lists (R x the largest count) pass max_edges although their union fits:
    every rank consumes its window, returns ALZ_E_CAPACITY and no rows, and counts every event lost; the next
    window is exact."""
    R, rng, me = 3, np.random.default_rng(5), 4096
    tabs = table_rows(abi.TABLE_POD, POD_NET + np.arange(R), np.arange(R))
    same = outbound_fan(0, POD_NET, 1500, abi.ip("15.0.0.0"), rng)
    w0 = [same.copy() for _ in range(R)]
    w1 = [outbound_fan(r, POD_NET + r, 20, abi.ip("16.0.0.0"), rng) for r in range(R)]
    cfg = dict(SMALL, max_edges=me, max_pairs=1 << 14)
    run = run_ranks(shim, tmp_path, R, [w0, w1], tabs, cfg=cfg, windows=[{}, {"flush": "device"}])
    for r in range(R):
        d = run.rank(r)[0]
        assert d["rc"] == abi.E_CAPACITY and d["n_out"] == 0, (r, d)
    assert run.stat_sum(0, "capacity_events") == R * len(same)
    assert run.stat_sum(0, "rows_emitted") == 0
    check_window(run, 1, oracle_edges(tables_of(tabs), np.concatenate(w1)))


@pytest.mark.gpu
def test_caller_buffer_too_small(shim, tmp_path):
    """A host buffer one row short: ALZ_E_CAPACITY with *n_out the merged count, alz_window_fetch returns the rows,
    and the next flush is exact."""
    R, rng = 5, np.random.default_rng(6)
    tabs, groups, _ = spread_groups(rng, 700)
    w0 = [np.concatenate(groups[r::R]) for r in range(R)]
    w1 = [np.concatenate(groups[r:300:R]) for r in range(R)]
    run = run_ranks(shim, tmp_path, R, [w0, w1], tabs, windows=[{"cap": 699, "fetch": True}, {}])
    exp = oracle_edges(tables_of(tabs), np.concatenate(w0))
    f0 = run.z["fetch_0_0"]
    for r in range(R):
        d = run.rank(r)[0]
        assert d["rc"] == abi.E_CAPACITY and d["n_out"] == 700 and d["fetch_rc"] == abi.OK, (r, d)
        assert run.z[f"fetch_0_{r}"].tobytes() == f0.tobytes()
    assert edges_equal(f0, exp), explain_diff(f0, exp)
    check_window(run, 1, oracle_edges(tables_of(tabs), np.concatenate(w1)))


@pytest.mark.gpu
def test_failed_peer_keeps_the_window(shim, tmp_path):
    """A peer whose local preparation failed (its block header carries ALZ_E_CUDA): every rank returns that status
    and no rows and keeps its window; the next flush returns both windows' events."""
    R, rng = 5, np.random.default_rng(8)
    tabs, groups, _ = spread_groups(rng, 500)
    w0 = [np.concatenate(groups[r::R]) for r in range(R)]
    w1 = [np.concatenate(groups[r:250:R]) for r in range(R)]
    run = run_ranks(shim, tmp_path, R, [w0, w1], tabs, fault=[2, 1, abi.E_CUDA],
                    windows=[{}, {"flush": "device"}])
    for r in range(R):
        d = run.rank(r)[0]
        assert d["rc"] == abi.E_CUDA and d["n_out"] == 0, (r, d)
        assert len(run.rows(0, r)) == 0
    both = np.concatenate(w0 + w1)
    rows = check_window(run, 1, oracle_edges(tables_of(tabs), both), events=len(both), since_start=True)
    assert len(rows) == 500


# ---- plans and neighbours ---------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("flags", [0, abi.CFG_EAGER_JOIN, abi.CFG_NO_SMEM_CACHE])
def test_plans_commit_and_gnn(shim, tmp_path, flags):
    """Each ingest plan, a table commit in the middle of a window on every rank (a pod that only the second half's
    records come from), then a window whose GNN scores are byte-identical on every rank and equal to those of a
    single-rank handle on all the records."""
    R, rng = 5, np.random.default_rng(9 + flags)
    tabs, groups, _ = spread_groups(rng, 400)
    late_ip, late_id = POD_NET + 5000, 4242
    w0 = [np.concatenate(groups[r::R]) for r in range(R)]
    for r in range(R):   # the late pod's records at the end: in each rank's second half
        late = records(np.full(4, late_ip), abi.ip("17.0.0.0") + r + np.arange(4) * R, rng)
        w0[r] = np.concatenate([w0[r], late])
        assert len(w0[r]) // 2 <= len(w0[r]) - 4
    w1 = [np.concatenate(groups[r::R] + [records(np.full(2, late_ip), np.full(2, SVC_NET), rng)])
          for r in range(R)]
    commit = table_rows(abi.TABLE_POD, [late_ip], [late_id])
    cfg = dict(SMALL, flags=flags)
    run = run_ranks(shim, tmp_path, R, [w0, w1], tabs, cfg=cfg, windows=[{"commit": True}, {"gnn": True}],
                    commits={0: commit}, solo=True)
    all_tabs = np.concatenate([tabs, commit])
    exp0 = oracle_edges(tables_of(all_tabs), np.concatenate(w0))
    check_window(run, 0, exp0)
    exp1 = oracle_edges(tables_of(all_tabs), np.concatenate(w1))
    rows = check_window(run, 1, exp1)
    g0 = run.z["gnn_1_0"]
    assert len(g0) == len(rows)
    for r in range(R):
        assert run.rank(r)[1]["gnn_rc"] == abi.OK
        assert run.z[f"gnn_1_{r}"].tobytes() == g0.tobytes()
    d, solo = run.solo(1)
    assert solo.tobytes() == rows.tobytes()
    assert run.z["gnn_1_solo"].tobytes() == g0.tobytes()


# ---- alz_comm_init ------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_comm_init_arguments(shim, tmp_path):
    """nranks over 64: ALZ_E_UNSUPPORTED before NCCL is even loaded; a rank out of range or no ranks:
    ALZ_E_INVAL; a second init on a handle: ALZ_E_STATE."""
    run = run_ranks(shim, tmp_path, 1, [], [], init_only=True)
    m = run.meta
    assert m["loaded_before"] == []
    assert m["rc_65"] == abi.E_UNSUPPORTED and m["rc_100"] == abi.E_UNSUPPORTED
    assert m["rc_rank_high"] == abi.E_INVAL and m["rc_rank_neg"] == abi.E_INVAL and m["rc_zero"] == abi.E_INVAL
    assert m["rc_one"] == abi.OK and m["rc_again"] == abi.E_STATE
    assert m["maps"] == [shim]


@pytest.mark.gpu
def test_one_rank_communicator_is_a_single_rank(shim, tmp_path):
    """nranks = 1: the same bytes as a handle without a communicator, and no collective."""
    tabs, per_rank, exps, _ = topo_case(1, 30_000, seed=55)
    run = run_ranks(shim, tmp_path, 1, per_rank, tabs, solo=True)
    for j in range(2):
        rows = check_window(run, j, exps[j])
        assert run.rank(0)[j]["log"] == []
        assert run.solo(j)[1].tobytes() == rows.tobytes()


# ---- CPU ------------------------------------------------------------------------------------------------------
def test_shim_builds_with_the_nccl_symbols(tmp_path):
    """The loopback library compiles for sm_90a, is named libnccl.so.2 and exports what the product resolves."""
    lib = build_shim(tmp_path)
    nm = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True, check=True).stdout
    syms = {ln.split()[-1] for ln in nm.splitlines() if ln.strip()}
    assert set(NCCL_EXPORTS) <= syms
    assert {"loopback_log_count", "loopback_log_entry", "loopback_log_clear", "loopback_fault_block_status"} <= syms
    dyn = subprocess.run(["readelf", "-d", lib], capture_output=True, text=True, check=True).stdout
    assert "Library soname: [libnccl.so.2]" in dyn
    with open(os.path.join(ROOT, "alaz_b200", "csrc", "alz_comm.cu")) as f:
        src = f.read()
    assert all(f'"{s}"' in src for s in NCCL_EXPORTS)      # the names load_nccl_once resolves


def test_owner_rank_restatement():
    from alaz_b200 import capi
    L = capi.load()
    rng = np.random.default_rng(1)
    s = np.concatenate([rng.integers(0, 1 << 32, 3000, dtype=np.uint64), [0, 1, 0xFFFFFFFF, 0xA1A2B200]])
    for R in (1, 2, 3, 8, 9, 17, 64, 65):
        got = lr.owner_rank(s, R)
        assert got.tolist() == [L.alz_owner_rank(int(x), R) for x in s], R
        assert got.max() < R


def test_block_rows_for_restatement():
    """DESIGN §6: a block is the largest count plus 25 % head room, rounded up to 1024 rows, never under 1024."""
    assert lr.block_rows_for(0) == 1024
    assert lr.block_rows_for(1) == 2048
    assert lr.block_rows_for(1000) == 3072          # 1000 + 250 + 1024 = 2274
    assert lr.block_rows_for(3072) == 5120          # 3072 + 768 + 1024 = 4864
    assert lr.block_rows_for(5121) == 8192          # 5121 + 1280 + 1024 = 7425
    for m in (0, 1, 5, 1023, 4096, 1 << 20):
        b = lr.block_rows_for(m)
        assert b % 1024 == 0 and b >= m + m // 4 + 1024 > b - 1024


def test_row_key_restatement():
    """The canonical order: pod-first rows by (other type, pod id, other); rows into a pod after every pod-first
    row (the rev bit); pod <-> pod rows always pod-first from the smaller side of make_edge_key."""
    e = np.zeros(4, dtype=abi.EDGE_OUT)
    e[0]["from_type"], e[0]["from"], e[0]["to_type"], e[0]["to"] = abi.NODE_POD, (1 << 29) - 1, abi.NODE_SVC, 0
    e[1]["from_type"], e[1]["from"], e[1]["to_type"], e[1]["to"] = abi.NODE_SVC, 0, abi.NODE_POD, 0
    e[2]["from_type"], e[2]["from"], e[2]["to_type"], e[2]["to"] = abi.NODE_POD, 0, abi.NODE_OUTBOUND_HOST, 0xFFFFFFFF
    e[3]["from_type"], e[3]["from"], e[3]["to_type"], e[3]["to"] = abi.NODE_POD, 3, abi.NODE_POD, 2
    k = [lr.row_key_of(x) for x in e]
    assert k[1] >> 63 == 1 and k[0] >> 63 == 0
    assert k[0] == (abi.NODE_SVC << 61) | (((1 << 29) - 1) << 32)
    assert k[2] == (abi.NODE_OUTBOUND_HOST << 61) | 0xFFFFFFFF
    assert k[3] == (3 << 32) | 2
    assert lr.make_edge_key(2, abi.NODE_POD, 3, True) == (3 << 32) | 2
    assert [int(x["from"]) for x in lr.canonical(e)] == [3, (1 << 29) - 1, 0, 0]
