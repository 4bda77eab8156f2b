"""Sequential model of time-cut windows (docs/SPEC.md §8) on top of the C oracle.

The model keeps one oracle per epoch that has received records. Every instance follows the same table log, and a new
instance replays the log before it takes records, so each record is resolved by the tables in force when it was
submitted (the arrival-tables rule). A flush returns the open epoch's edges and opens the next epoch.

Which records overflow the device's set-aside buffer is not deterministic: past `defer_cap` the model keeps the first
records of a submit and drops the rest, which matches the device only when the dropped records are interchangeable
(tests that overflow use identical records).
"""
import numpy as np

import oracle_lib as ol
from alaz_b200 import abi


def epoch(first_kernel, first_user, window_ns, wt):
    """user_ns / window_ns with user_ns = first_user - (first_kernel - wt), all mod 2^64 (SPEC §8); vectorised."""
    wt = np.asarray(wt, dtype=np.uint64)
    with np.errstate(over="ignore"):
        user = np.uint64(first_user) - (np.uint64(first_kernel) - wt)
    return user // np.uint64(window_ns)


class WindowModel:
    STAT_KEYS = ("events_in", "late_events", "deferred_events", "capacity_events", "not_request", "src_unresolved",
                 "rows_emitted")

    def __init__(self, first_kernel, first_user, window_ns, defer_cap):
        self.cap = int(defer_cap)
        self.log = []             # committed table operations, in order
        self.staged = []          # upserts / erases since the last commit
        self.inst = {}            # epoch -> ol.Oracle of the records of that epoch
        self.held = {}            # epoch > epoch_open -> records set aside for it
        self.events_in = self.late = self.lost = 0
        self.closed = dict(not_request=0, src_unresolved=0, rows_emitted=0)   # epochs already flushed
        self.epoch_open = None
        self.carry = None
        self.clock(first_kernel, first_user, window_ns)

    # ---- tables: staged until commit, as on the device
    def upsert(self, table, ip, id_):
        self.staged.append(("u", table, int(ip), int(id_)))

    def erase(self, table, ip):
        self.staged.append(("e", table, int(ip), 0))

    def commit(self):
        for op in self.staged:
            for o in self.inst.values():
                self._apply(o, op)
        self.log += self.staged
        self.staged = []

    @staticmethod
    def _apply(o, op):
        if op[0] == "u":
            o.upsert(op[1], op[2], op[3])
        else:
            o.erase(op[1], op[2])

    def _instance(self, e):
        if e not in self.inst:
            o = ol.Oracle()
            for op in self.log:
                self._apply(o, op)
            self.inst[e] = o
        return self.inst[e]

    # ---- clock
    def clock(self, first_kernel, first_user, window_ns):
        """alz_window_clock: only with nothing set aside. The open window's records stay and go out with the window the
        next record opens."""
        assert self.n_held == 0
        self.fk, self.fu, self.W = int(first_kernel), int(first_user), int(window_ns)
        if self.epoch_open is not None:
            self.carry = self.inst.pop(self.epoch_open, None)
        self.epoch_open = None

    def epochs(self, wt):
        return epoch(self.fk, self.fu, self.W, wt)

    @property
    def n_held(self):
        return sum(self.held.values())

    # ---- records
    def submit(self, recs):
        recs = np.ascontiguousarray(recs, dtype=abi.L7_REC)
        if len(recs) == 0:
            return
        self.events_in += len(recs)
        e = np.array(self.epochs(recs["write_time_ns"]).tolist(), dtype=object)   # epoch_open may pass 2^64 - 1
        if self.epoch_open is None:
            self.epoch_open = int(e[0])
            if self.carry is not None:
                self.inst[self.epoch_open] = self.carry
                self.carry = None
        now = e <= self.epoch_open
        self.late += int(np.count_nonzero(e < self.epoch_open))
        if now.any():
            self._instance(self.epoch_open).process(recs[now])
        fut = np.flatnonzero(~now)
        room = max(0, self.cap - self.n_held)
        self.lost += max(0, len(fut) - room)
        fut = fut[:room]
        for k in sorted(set(e[fut].tolist())):
            sel = fut[e[fut] == k]
            self._instance(k).process(recs[sel])
            self.held[k] = self.held.get(k, 0) + len(sel)

    def flush(self):
        """The open window's edges; epoch_open advances by one (nothing happens before the first record)."""
        if self.epoch_open is None:
            return np.zeros(0, dtype=abi.EDGE_OUT)
        o = self.inst.pop(self.epoch_open, None)
        out = np.zeros(0, dtype=abi.EDGE_OUT)
        if o is not None:
            out = o.edges()
            st = o.stats()
            for k in self.closed:
                self.closed[k] += st[k]
            o.close()
        self.epoch_open += 1
        self.held.pop(self.epoch_open, None)
        return out

    def stats(self):
        """Counters as alz_get_stats gives them once every pending pair is folded. A set-aside record enters
        not_request and src_unresolved when its window opens; until then it is in deferred_events."""
        s = dict(self.closed)
        for o in (self.inst.get(self.epoch_open), self.carry):
            if o is not None:
                st = o.stats()
                for k in s:
                    s[k] += st[k]
        s.update(events_in=self.events_in, late_events=self.late, deferred_events=self.n_held,
                 capacity_events=self.lost)
        return s
