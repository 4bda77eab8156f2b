"""Sequential model of time-cut windows on several ranks (docs/SPEC.md §8 "Several ranks"): one WindowModel per rank
(tests/window_model.py) plus the agreement rule of the merge.

At a flush, E is the smallest open epoch of the ranks that have one, the past state after every epoch. A rank at E
flushes its window as one handle does; a rank ahead of E keeps everything; a rank without an epoch opens E + 1
(with the rows it held from before its clock, as its own first record would have). No rank with an epoch: no rows,
no change. The ranks' clocks must agree (length and offset, or off on every rank), otherwise the flush fails and
nothing changes. The merged rows are the at-E ranks' rows summed per edge, in the canonical order, cut at
`max_edges`; the owner of a row past the cut counts its events lost.
"""
import numpy as np

from alaz_b200 import abi
from window_model import WindowModel

M64 = 1 << 64
STATE_ERR = "state"


def row_key(row):
    """Packed edge key of an output row (the canonical order of merged rows is ascending key)."""
    ft, f, tt, t = int(row["from_type"]), int(row["from"]), int(row["to_type"]), int(row["to"])
    if ft == abi.NODE_POD:
        return (tt << 61) | ((f & 0x1FFFFFFF) << 32) | t
    return (1 << 63) | (ft << 61) | ((t & 0x1FFFFFFF) << 32) | f


def sum_rows(parts):
    """Rows of several ranks summed per edge (integer sums: counts and sums mod 2^64, cells mod 2^32), in
    canonical order. Returns (rows, owners): owners[i] = the ranks that had row i."""
    acc, own = {}, {}
    for r, rows in parts:
        for x in rows:
            k = row_key(x)
            if k in acc:
                a = acc[k]
                a["count"] += x["count"]
                a["err5xx"] += x["err5xx"]
                with np.errstate(over="ignore"):
                    a["lat_sum_ns"] = np.uint64(a["lat_sum_ns"]) + np.uint64(x["lat_sum_ns"])
                    a["hist"] = a["hist"] + x["hist"]
                own[k].append((r, int(x["count"])))
            else:
                acc[k] = x.copy()
                own[k] = [(r, int(x["count"]))]
    keys = sorted(acc)
    out = np.zeros(len(keys), dtype=abi.EDGE_OUT)
    for i, k in enumerate(keys):
        out[i] = acc[k]
    return out, [own[k] for k in keys]


class RanksModel:
    def __init__(self, R, defer_cap, max_edges=None):
        self.R, self.max_edges = R, max_edges
        # one WindowModel per rank; its clock counts only once the rank has set one (clk[r] not None)
        self.ranks = [WindowModel(0, 0, 1, defer_cap) for _ in range(R)]
        self.clk = [None] * R            # (window_ns, offset mod 2^64) per rank
        self.reported = [0] * R          # set-aside overflow already reported by a flush
        self.windows = [0] * R           # successful flushes per rank

    # ---- per rank
    def clock(self, r, first_kernel, first_user, window_ns):
        self.ranks[r].clock(first_kernel, first_user, window_ns)
        self.clk[r] = (int(window_ns), (int(first_user) - int(first_kernel)) % M64)

    def submit(self, r, recs):
        assert self.clk[r] is not None, "the model has no clockless windows"
        self.ranks[r].submit(recs)

    def upsert(self, r, table, ip, id_):
        self.ranks[r].upsert(table, ip, id_)

    def commit(self, r):
        self.ranks[r].commit()

    def key(self, r):
        """The rank's open epoch for the agreement; M64 for the past state; None without one."""
        m = self.ranks[r]
        if m.epoch_open is None:
            return None
        return M64 if m.epoch_open > (M64 - 1) // m.W else m.epoch_open

    def epoch(self, r):
        """alz_window_epoch: None until the rank has an epoch."""
        m = self.ranks[r]
        return None if self.clk[r] is None or m.epoch_open is None else m.epoch_open % M64

    def stats(self, r):
        s = self.ranks[r].stats()
        s["windows"] = self.windows[r]
        return s

    def solo_flush(self, r):
        """a flush of rank r alone, before it joins the other ranks"""
        self.windows[r] += 1
        return self.ranks[r].flush()

    # ---- collective
    def flush(self):
        """(status, rows) as every rank gets them: status abi.OK, abi.E_CAPACITY or STATE_ERR."""
        if len(set(self.clk)) != 1 or self.clk[0] is None:
            return STATE_ERR, np.zeros(0, dtype=abi.EDGE_OUT)
        self.windows = [w + 1 for w in self.windows]
        keys = [self.key(r) for r in range(self.R)]
        open_ = [k for k in keys if k is not None]
        if not open_:
            return abi.OK, np.zeros(0, dtype=abi.EDGE_OUT)
        E = min(open_)
        at_e = [r for r in range(self.R) if keys[r] == E]
        e_counter = self.ranks[at_e[0]].epoch_open    # an unopened rank copies the clock of the first rank at E
        lost = any(self.ranks[r].lost > self.reported[r] for r in at_e)
        parts = []
        for r, k in enumerate(keys):
            m = self.ranks[r]
            if k == E:
                self.reported[r] = m.lost
                parts.append((r, m.flush()))
            elif k is None:
                m.epoch_open = e_counter + 1
                if m.carry is not None:
                    m.inst[m.epoch_open] = m.carry
                    m.carry = None
        rows, owners = sum_rows(parts)
        status = abi.E_CAPACITY if lost else abi.OK
        if self.max_edges is not None and len(rows) > self.max_edges:
            for own in owners[self.max_edges:]:
                for r, c in own:
                    self.ranks[r].lost += c
                    self.reported[r] += c
                    self.ranks[r].closed["rows_emitted"] -= c
            rows = rows[: self.max_edges]
            status = abi.E_CAPACITY
        return status, rows
