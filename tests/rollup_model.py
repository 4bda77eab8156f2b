"""Sequential model of the rolling windows (docs/SPEC.md §12): the history as a list of {packed key -> row} dicts with
the arena's placement and eviction rule, and the sum of the last k of them with the wrap widths of an edge row."""
import numpy as np

from alaz_b200 import abi

M64 = (1 << 64) - 1


def packed_key(row):
    """The packed edge key of docs/SPEC.md §3, from the fields of an alz_edge_out row."""
    ft, tt, f, t = int(row["from_type"]), int(row["to_type"]), int(row["from"]), int(row["to"])
    if ft == abi.NODE_POD:
        return (tt << 61) | ((f & 0x1FFFFFFF) << 32) | t
    return (1 << 63) | (ft << 61) | ((t & 0x1FFFFFFF) << 32) | f


def add_rows(a, b):
    """a + b of two alz_edge_out rows of one key: u64 sums modulo 2^64, histogram cells modulo 2^32."""
    out = a.copy()
    for f in ("count", "err5xx", "lat_sum_ns"):
        out[f] = (int(a[f]) + int(b[f])) & M64
    out["hist"] = (a["hist"].astype(np.uint64) + b["hist"].astype(np.uint64)).astype(np.uint32)
    return out


class RollupModel:
    def __init__(self):
        self.depth, self.arena_rows = 0, 0
        self.entries = []   # oldest first: dicts first_row, n, rows {key: row}, window, epoch (None: not clocked)

    def history(self, depth, arena_rows):
        if (depth, arena_rows) == (self.depth, self.arena_rows):
            return
        self.depth, self.arena_rows, self.entries = depth, arena_rows, []

    def append(self, rows, window, epoch=None):
        """A flush consumed its window: `rows` is what it returned, `window` alz_stats.windows after it, `epoch` the
        epoch it closed under a window clock."""
        if self.depth == 0:
            return
        n = len(rows)
        if n > self.arena_rows:
            self.entries = []
            return
        while True:
            while len(self.entries) >= self.depth:
                self.entries.pop(0)
            at = self.entries[-1]["first_row"] + self.entries[-1]["n"] if self.entries else 0
            if at + n > self.arena_rows:
                at = 0
            if not any(at < e["first_row"] + e["n"] and e["first_row"] < at + n for e in self.entries):
                break
            self.entries.pop(0)
        self.entries.append(dict(first_row=at, n=n, rows={packed_key(r): r.copy() for r in rows}, window=window,
                                 epoch=epoch))

    def rollup(self, k):
        """(rows in ascending key order, alz_rollup_info as a dict)"""
        assert self.depth and k > 0
        take = self.entries[-k:]
        acc = {}
        for e in take:
            for key, r in e["rows"].items():
                acc[key] = add_rows(acc[key], r) if key in acc else r.copy()
        rows = np.zeros(len(acc), dtype=abi.EDGE_OUT)
        for i, key in enumerate(sorted(acc)):
            rows[i] = acc[key]
        clocked = bool(take) and all(e["epoch"] is not None for e in take)
        info = dict(windows=len(take), clocked=int(clocked),
                    window_first=take[0]["window"] if take else 0, window_last=take[-1]["window"] if take else 0,
                    epoch_first=take[0]["epoch"] if clocked else 0, epoch_last=take[-1]["epoch"] if clocked else 0,
                    rows_in=sum(e["n"] for e in take))
        return rows, info
