"""Time-cut windows on several ranks (docs/SPEC.md §8 "Several ranks") on ONE GPU: 2 to 64 ranks of one process talk
through the loopback collective (tests/loopback_nccl.cu) in a child process (tests/loopback_clock.py). Every
operation is replayed on the model of tests/window_ranks_model.py; after every operation every rank's stats and
alz_window_epoch are compared with it, and every flush's rows with it and with every other rank's, byte for byte."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import loopback_ranks as lr
from alaz_b200 import abi
from gnn_graphs import POD_NET, SVC_NET
from helpers import edges_equal, explain_diff
from test_gpu_loopback_ranks import build_shim
from window_ranks_model import M64, STATE_ERR, RanksModel

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SMALL = dict(max_endpoints=1 << 14, max_pairs=1 << 15, max_edges=1 << 14, max_batch=1 << 14)
N_PODS, N_SVCS = 1024, 8
TABLES = np.concatenate([
    np.stack([np.full(N_PODS, abi.TABLE_POD), POD_NET + np.arange(N_PODS), np.arange(N_PODS)], 1),
    np.stack([np.full(N_SVCS, abi.TABLE_SVC), SVC_NET + np.arange(N_SVCS), 100 + np.arange(N_SVCS)], 1)]).astype(np.int64)
W = 1_000_000
FK, FU = 12345, 12345 + 10**6 * W + 77          # offset 10^12 + 77: epoch 10^6 starts at kernel time W - 77
STATS = ("events_in", "late_events", "deferred_events", "capacity_events", "not_request", "windows")


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return build_shim(tmp_path_factory.mktemp("loopback_nccl"))


def wt_of(e, k=0, fk=FK, fu=FU, w=W):
    """kernel write time of the k-th ns of epoch e (mod 2^64)"""
    return (e * w - (fu - fk) + k) % M64


class Case:
    """Operations on R ranks, recorded for the child and replayed on the model as they are added."""

    def __init__(self, R, cfg=SMALL, seed=0, join=True):
        self.R, self.cfg = R, dict(cfg)
        self.rng = np.random.default_rng(seed)
        self.ops, self.arrays = [], {"tables": TABLES}
        me = cfg.get("max_edges") or cfg["max_pairs"]
        self.m = RanksModel(R, 2 * cfg["max_batch"], max_edges=me)
        for r in range(R):
            for tab, ip, id_ in TABLES:
                self.m.upsert(r, int(tab), int(ip), int(id_))
            self.m.commit(r)
        self.snap = []                    # per op: (model stats, epochs, expected flush or None)
        own = lr.owner_rank(POD_NET + np.arange(N_PODS), R)
        self.pods_of = [POD_NET + np.flatnonzero(own == r) for r in range(R)]
        if join:
            self.join()

    def _done(self, op, flush=None):
        self.ops.append(op)
        self.snap.append(([self.m.stats(r) for r in range(self.R)], [self.m.epoch(r) for r in range(self.R)], flush))

    # ---- records
    def recs(self, r, epochs, n_per=1, src=None, w=W, fk=FK, fu=FU):
        """n_per records per entry of epochs from rank r's own pods to a service or an outbound address"""
        e = np.repeat(np.asarray(epochs, dtype=object), n_per)
        n = len(e)
        x = np.zeros(n, dtype=abi.L7_REC)
        x["saddr"] = src if src is not None else self.rng.choice(self.pods_of[r][:64], n)
        x["daddr"] = np.where(self.rng.random(n) < 0.7, SVC_NET + self.rng.integers(0, N_SVCS, n),
                              abi.ip("9.0.0.0") + self.rng.integers(0, 50, n))
        x["sport"], x["dport"] = 40000, 80
        x["protocol"] = self.rng.choice([abi.PROTO_HTTP, abi.PROTO_HTTP2, abi.PROTO_REDIS, abi.PROTO_POSTGRES], n)
        x["method_flags"] = 1
        x["status"] = self.rng.choice([200, 500, 503], n)
        x["duration_ns"] = self.rng.integers(1, 1 << 34, n, dtype=np.uint64)
        x["write_time_ns"] = [wt_of(int(ep), int(k), fk, fu, w) for ep, k in zip(e, self.rng.integers(0, w, n))]
        return x

    # ---- operations
    def clock(self, r, fk=FK, fu=FU, w=W, model=True):
        if model:
            self.m.clock(r, fk, fu, w)
        self._done({"op": "clock", "r": r, "args": [fk, fu, w]})

    def clock_all(self, **kw):
        for r in range(self.R):
            self.clock(r, **kw)

    def submit(self, r, recs, how="host"):
        key = f"a{len(self.arrays)}"
        self.arrays[key] = np.ascontiguousarray(recs, dtype=abi.L7_REC)
        self.m.submit(r, recs)
        self._done({"op": "submit", "r": r, "key": key, "how": how})

    def commit(self, r, rows):
        key = f"a{len(self.arrays)}"
        self.arrays[key] = np.asarray(rows, np.int64).reshape(-1, 3)
        for tab, ip, id_ in self.arrays[key]:
            self.m.upsert(r, int(tab), int(ip), int(id_))
        self.m.commit(r)
        self._done({"op": "commit", "r": r, "key": key})

    def fold(self, r):
        self._done({"op": "fold", "r": r})

    def join(self):
        self._done({"op": "join"})

    def solo_flush(self, r):
        rows = self.m.solo_flush(r)
        self._done({"op": "flush", "r": r}, (abi.OK, rows))

    def flush(self, how="host", cap=None, fetch=False):
        st, rows = self.m.flush()
        self._done({"op": "flush", "how": how, "cap": cap, "fetch": fetch}, (st, rows))
        return st, rows

    # ---- run and compare
    def run(self, shim, tmp_path, solo=False, check=True, timeout=600):
        spec = {"nranks": self.R, "cfg": self.cfg, "ops": self.ops, "solo": solo}
        sp, ip, op = (str(tmp_path / x) for x in ("spec.json", "in.npz", "out.npz"))
        with open(sp, "w") as f:
            json.dump(spec, f)
        np.savez(ip, **self.arrays)
        env = dict(os.environ)
        env["LD_LIBRARY_PATH"] = os.path.dirname(shim) + os.pathsep + env.get("LD_LIBRARY_PATH", "")
        env["LOOPBACK_NCCL_TIMEOUT_S"] = "60"
        p = subprocess.run([sys.executable, os.path.join(HERE, "loopback_clock.py"), sp, ip, op], cwd=ROOT, env=env,
                           capture_output=True, text=True, timeout=timeout)
        assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
        self.z = np.load(op)
        self.meta = json.loads(str(self.z["meta"]))
        assert not self.meta["errors"], self.meta["errors"]
        assert self.meta["maps"] == [shim], self.meta["maps"]
        if check:
            self.check()
        return self

    def at(self, i, r):
        return self.meta["ranks"][str(r)][i]

    def rows(self, i, r):
        return self.z[f"rows_{i}_{r}"]

    def check(self):
        for i, (op, (stats, epochs, exp)) in enumerate(zip(self.ops, self.snap)):
            for r in range(self.R):
                d = self.at(i, r)
                got, want = d["stats"], stats[r]
                for k in STATS:
                    assert got[k] == want[k], (i, op, r, k, got[k], want[k])
                assert got["rows_emitted"] + got["src_unresolved"] == want["rows_emitted"] + want["src_unresolved"], \
                    (i, op, r, got, want)
                if op["op"] in ("flush", "fold"):
                    assert got["rows_emitted"] == want["rows_emitted"], (i, op, r, got, want)
                rc, e = d["epoch"]
                assert (rc, e) == ((abi.E_STATE, None) if epochs[r] is None else (abi.OK, epochs[r])), (i, op, r, d)
                if op["op"] == "clock" and op["r"] == r:
                    assert d["rc"] == abi.OK
            if op["op"] != "flush":
                continue
            st, rows = exp
            ranks = [op["r"]] if "r" in op else range(self.R)
            want_rc = abi.E_STATE if st == STATE_ERR else st
            if op.get("cap") is not None and len(rows) > op["cap"]:
                want_rc = abi.E_CAPACITY
            r0 = ranks[0]
            for r in ranks:
                d = self.at(i, r)
                assert d["rc"] == want_rc, (i, r, d["rc"], want_rc)
                if op.get("fetch"):
                    assert d["fetch_rc"] == abi.OK and d["n_out"] == len(rows)
                    got = self.z[f"fetch_{i}_{r}"]
                else:
                    got = self.rows(i, r)
                assert got.tobytes() == (self.z[f"fetch_{i}_{r0}"] if op.get("fetch") else self.rows(i, r0)).tobytes()
                assert edges_equal(got, rows), f"op {i} rank {r}: " + explain_diff(got, rows)
                k = np.array([lr.row_key_of(x) for x in got], dtype=np.uint64)
                assert np.all(k[1:] > k[:-1]), "rows not in canonical order"

    def flush_indices(self):
        return [i for i, op in enumerate(self.ops) if op["op"] == "flush" and "r" not in op]


# ---- every rank opens in the same epoch ----------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("R", [2, 3, 8, 17, 64])
def test_same_epoch_equals_a_solo_handle(shim, tmp_path, R):
    """Every rank's first record in epoch E0; then records of E0 - 1 (late), E0 .. E0 + 2: four flushes, each the
    merged rows of one epoch, equal to one handle fed every rank's records under the same clock."""
    c, E0 = Case(R, seed=R), 10**6 + 5
    c.clock_all()
    n = 40 if R < 64 else 10
    for r in range(R):
        c.submit(r, c.recs(r, [E0], 1))
    for r in range(R):
        c.submit(r, c.recs(r, [E0 - 1, E0, E0 + 1, E0 + 2], n))
    for _ in range(4):
        c.flush()
    c.run(shim, tmp_path, solo=True)
    for j, i in enumerate(c.flush_indices()):
        assert c.meta["solo"][j]["rc"] == abi.OK
        assert c.z[f"rows_{i}_solo"].tobytes() == c.rows(i, 0).tobytes(), j


# ---- staggered openings --------------------------------------------------------------------------------------
AHEAD = {"rank0": lambda R: [0], "last": lambda R: [R - 1], "several": lambda R: [1, 2, R - 1]}


@pytest.mark.gpu
@pytest.mark.parametrize("how", ["host", "device"])
@pytest.mark.parametrize("ahead", list(AHEAD))
@pytest.mark.parametrize("shift", [1, 3])
def test_staggered_openings(shim, tmp_path, shift, ahead, how):
    """Ranks in `ahead` open `shift` epochs after the others: they keep their windows through `shift` flushes, take
    records of earlier epochs as late meanwhile, and then merge with the rest; host and device flushes."""
    R, E0 = 5, 10**6 + 100
    c = Case(R, seed=shift * 10 + len(ahead))
    c.clock_all()
    late = set(AHEAD[ahead](R))
    for r in range(R):
        c.submit(r, c.recs(r, [E0 + (shift if r in late else 0)] * 20 + [E0 + shift + 1] * 5))
    for k in range(shift + 2):
        for r in range(R):
            if r in late:
                c.submit(r, c.recs(r, [E0 + k], 3))            # late on an ahead rank until the ranks agree
            else:
                c.submit(r, c.recs(r, [E0 + k, E0 + k + 1], 4))
        c.flush(how=how)
    c.run(shim, tmp_path)


@pytest.mark.gpu
def test_rank_without_records_for_three_windows(shim, tmp_path):
    """Rank 2 gets no records for three windows: the first flush opens it at E + 1 and it follows from there; its
    first records are then of its open epoch, a later one (set aside) and an earlier one (late)."""
    R, E0 = 4, 10**6 + 7
    c = Case(R, seed=3)
    c.clock_all()
    for k in range(3):
        for r in (0, 1, 3):
            c.submit(r, c.recs(r, [E0 + k], 10))
        c.flush()
    c.submit(2, c.recs(2, [E0 + 3, E0 + 5, E0 + 1], 4))
    for r in (0, 1, 3):
        c.submit(r, c.recs(r, [E0 + 3], 2))
    for _ in range(3):
        c.flush()
    c.run(shim, tmp_path)


@pytest.mark.gpu
def test_set_aside_records_across_rolls_and_a_commit(shim, tmp_path):
    """Ranks 0 and 3 hold records of the next four epochs across several rolls; rank 1 opens two epochs ahead and
    takes late records; a table commit in the middle of a window on every rank (a pod only the second half comes
    from, on ranks holding set-aside records), then the windows drain."""
    R, E0 = 4, 10**6 + 40
    c = Case(R, seed=4)
    c.clock_all()
    for r in range(R):
        c.submit(r, c.recs(r, [E0 + (2 if r == 1 else 0)], 5))
    for r in (0, 3):
        c.submit(r, c.recs(r, [E0 + 1, E0 + 2, E0 + 3, E0 + 4], 30))
    c.submit(1, c.recs(1, [E0, E0 + 1], 6))
    c.flush()
    newcomer = POD_NET + 50_000
    for r in range(R):
        c.submit(r, c.recs(r, [E0 + 1, E0 + 3], 4))
    for r in range(R):
        c.commit(r, [[abi.TABLE_POD, newcomer, 9999]])
    for r in range(R):
        c.submit(r, c.recs(r, [E0 + 1, E0 + 2], 3, src=np.full(6, newcomer)))
    for _ in range(5):
        c.flush()
    c.run(shim, tmp_path)


@pytest.mark.gpu
def test_general_path_with_staggered_openings(shim, tmp_path):
    """One source's records routed to two ranks (keys on several ranks: the sort + all-reduce path) while rank 2 is
    ahead: it contributes no rows and keeps its window until E reaches it."""
    R, E0 = 4, 10**6 + 60
    c = Case(R, seed=6)
    c.clock_all()
    shared = POD_NET + 7
    for r in range(R):
        e = E0 + (1 if r == 2 else 0)
        c.submit(r, np.concatenate([c.recs(r, [e], 8), c.recs(r, [e], 3, src=np.full(3, shared))]))
    for _ in range(3):
        for r in range(R):
            c.submit(r, c.recs(r, [E0 + 1], 2, src=np.full(2, shared)))
        c.flush()
    c.run(shim, tmp_path)


# ---- clock mismatch ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("field", ["len", "off", "off_on_one_rank"])
def test_clock_mismatch_keeps_every_window(shim, tmp_path, field):
    """Rank 1's clock differs (another length; another offset; no clock): ALZ_E_STATE on every rank, every window
    and epoch kept; after rank 1 folds and sets the common clock, the window flushes. The same offset from other
    first times is the same clock."""
    R, E0 = 3, 10**6 + 3
    c = Case(R, seed=7)
    for r in (0, 2):
        c.clock(r)
    if field == "len":
        c.clock(1, w=2 * W)
    elif field == "off":
        c.clock(1, fu=FU + 1)
    for r in (0, 2):
        c.submit(r, c.recs(r, [E0], 6))
    if field != "off_on_one_rank":
        w = 2 * W if field == "len" else W
        fu = FU + (1 if field == "off" else 0)
        c.submit(1, c.recs(1, [(E0 * W) // w], 6, w=w, fu=fu))
    c.flush()
    c.flush(how="device")
    if field != "off_on_one_rank":
        c.fold(1)
    c.clock(1, fk=FK + 1000, fu=FU + 1000)         # the same offset
    c.flush()
    c.flush()
    c.run(shim, tmp_path)


# ---- capacity ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_ahead_rank_loss_is_reported_with_its_window(shim, tmp_path):
    """Rank 1 opens one epoch ahead and overflows its set-aside buffer: the flush at E is ALZ_OK, the flush that
    merges rank 1's window is ALZ_E_CAPACITY on every rank."""
    R, E0 = 3, 10**6 + 11
    cfg = dict(SMALL, max_batch=1 << 10)            # set-aside buffer: 2048 records
    c = Case(R, cfg=cfg, seed=8)
    c.clock_all()
    c.submit(0, c.recs(0, [E0], 4))
    c.submit(2, c.recs(2, [E0], 4))
    c.submit(1, c.recs(1, [E0 + 1], 4))
    big = c.recs(1, [E0 + 3], 1, src=np.full(1, c.pods_of[1][0]))
    c.submit(1, np.repeat(big, 3000))               # identical records: which ones overflow does not matter
    for _ in range(4):
        c.flush()
    c.run(shim, tmp_path)
    sts = [c.snap[i][2][0] for i in c.flush_indices()]
    assert sts == [abi.OK, abi.E_CAPACITY, abi.OK, abi.OK], sts


@pytest.mark.gpu
@pytest.mark.parametrize("how", ["host", "device"])
def test_merged_graph_over_max_edges(shim, tmp_path, how):
    """The union of the at-E ranks' rows passes max_edges (an ahead rank's rows do not count): cut in canonical
    order, the owners count their rows past the cut as lost."""
    R, E0, me = 3, 10**6 + 13, 512
    cfg = dict(SMALL, max_edges=me, max_pairs=1 << 13)
    c = Case(R, cfg=cfg, seed=9)
    c.clock_all()
    for r in range(R):
        x = c.recs(r, [E0 + (1 if r == 2 else 0)], 300)
        x["daddr"] = abi.ip("11.0.0.0") + r * 1000 + np.arange(300)
        c.submit(r, x)
    c.flush(how=how)
    c.flush(how=how)
    c.run(shim, tmp_path)


@pytest.mark.gpu
def test_caller_buffer_too_small_then_fetch(shim, tmp_path):
    R, E0 = 4, 10**6 + 17
    c = Case(R, seed=10)
    c.clock_all()
    for r in range(R):
        c.submit(r, c.recs(r, [E0 + (1 if r == 3 else 0)], 40))
    st, rows = c.flush(cap=1, fetch=True)
    assert len(rows) > 1
    c.flush(cap=1, fetch=True)
    c.flush()
    c.run(shim, tmp_path)


# ---- the end of the clock ------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_write_times_near_2_64_and_the_past_state(shim, tmp_path):
    """window_ns 2^62 + 1, offset 0: epochs 0..3, the last ending past 2^64. Rank 0 reaches the past state alone
    before the ranks join; at the first merge rank 1 is at epoch 2 and rank 2 has no epoch: E = 2, rank 0 keeps
    its window (every record late), rank 2 opens epoch 3. Then E = 3, and after it every rank is past."""
    R, w = 3, (1 << 62) + 1
    c = Case(R, seed=11, join=False)
    clk = dict(fk=0, fu=0, w=w)
    c.clock_all(**clk)
    c.submit(0, c.recs(0, [3], 5, **clk))
    c.solo_flush(0)
    c.submit(0, c.recs(0, [0, 3], 3, **clk))
    c.join()
    c.submit(1, c.recs(1, [2, 3], 4, **clk))
    c.flush()
    c.submit(2, c.recs(2, [3, 1], 2, **clk))
    c.submit(1, _at(c, 1, M64 - 1))
    c.flush()
    c.submit(2, _at(c, 2, M64 - 1))
    c.flush()
    c.flush()
    c.run(shim, tmp_path)


def _at(c, r, wt):
    x = c.recs(r, [0], 1, fk=0, fu=0, w=1)
    x["write_time_ns"] = wt
    return x


# ---- collectives ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_clocked_flush_issues_the_clockless_collectives(shim, tmp_path):
    """Every rank in one epoch: each flush's collective log (operations and byte counts) and collective_bytes_last
    are those of the same records on ranks without a clock."""
    R, E0 = 6, 10**6 + 21
    c = Case(R, seed=12)
    c.clock_all()
    for j in range(3):
        for r in range(R):
            c.submit(r, c.recs(r, [E0 + j], 30 + 20 * r))
        c.flush()
    (tmp_path / "clocked").mkdir()
    c.run(shim, tmp_path / "clocked")
    bare = Case(R)
    bare.arrays = c.arrays
    bare.ops = [op for op in c.ops if op["op"] != "clock"]
    (tmp_path / "bare").mkdir()
    bare.run(shim, tmp_path / "bare", check=False)

    def logs(case):
        return [[(case.at(i, r)["log"], case.at(i, r)["stats"]["collective_bytes_last"]) for r in range(R)]
                for i in case.flush_indices()]
    assert logs(c) == logs(bare)
    assert all(len(x[0][0]) >= 1 for x in logs(c))
    for i in bare.flush_indices():   # and the rows: every window holds one epoch, flushed as it came
        assert bare.rows(i, 0).tobytes() == c.rows(i + R, 0).tobytes()


# ---- CPU -----------------------------------------------------------------------------------------------------
def test_cases_replay_on_the_model():
    """The model side of two cases, without a GPU: the staggered opening keeps the ahead rank's window."""
    c = Case(3, seed=1)
    c.clock_all()
    c.submit(0, c.recs(0, [10**6 + 1], 3))
    c.submit(1, c.recs(1, [10**6 + 2], 3))
    st, rows = c.flush()
    assert st == abi.OK and int(rows["count"].sum()) == c.m.stats(0)["rows_emitted"] > 0
    assert c.snap[-1][1] == [10**6 + 2, 10**6 + 2, 10**6 + 2]
    assert c.m.stats(1)["rows_emitted"] + c.m.stats(1)["not_request"] + c.m.stats(1)["src_unresolved"] == 3
