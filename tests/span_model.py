"""Sequential model of span rollups (docs/SPEC.md §14), built on tests/tier_model.py and tests/rollup_model.py: the
retained pieces (window-history entries, closed tier entries, usable open blocks), the planner that picks the span and
its pieces, and the expected rows, which are the direct sum of the flushed windows the span covers, not a sum of
pieces."""
import numpy as np

from alaz_b200 import abi
from rollup_model import RollupModel, add_rows, packed_key
from tier_model import TierModel, rows_of

AT_MOST, AT_LEAST = abi.SPAN_AT_MOST, abi.SPAN_AT_LEAST


class _Tiers(TierModel):
    """TierModel that also records the newest window of each open block: that of the flush that fed its last input."""

    def _input(self, t, acc_in, window_first, window_last, windows, epoch_first, epoch_last, poisoned):
        self.tiers[t].window_last = window_last
        super()._input(t, acc_in, window_first, window_last, windows, epoch_first, epoch_last, poisoned)


def units_of(m0, mt):
    """Every retained piece of a window history (RollupModel) and tiers (TierModel) as dicts: level (0 = the window
    history, t = tier t), open, window_first, window_last, n (rows), epoch_first / epoch_last (None: not clocked)."""
    units = []
    for e in m0.entries if m0.depth else []:
        units.append(dict(level=0, open=False, window_first=e["window"], window_last=e["window"], n=e["n"],
                          epoch_first=e["epoch"], epoch_last=e["epoch"]))
    for i, t in enumerate(mt.tiers):
        for e in t.ring.entries:
            units.append(dict(level=i + 1, open=False, window_first=e["window_first"], window_last=e["window"],
                              n=e["n"], epoch_first=e["epoch_first"], epoch_last=e["epoch_last"]))
        if t.inputs and not t.poisoned and not t.overflow:
            ef, el = (t.epoch_first, t.epoch_last) if t.clocked else (None, None)
            units.append(dict(level=i + 1, open=True, window_first=t.window_first, window_last=t.window_last,
                              n=len(t.acc), epoch_first=ef, epoch_last=el))
    return units


def cost(plan, units):
    """the order of docs/SPEC.md §14: fewer source rows, fewer pieces, then piece by piece from the oldest the
    coarser piece (a higher level sorts first)"""
    return (sum(units[i]["n"] for i in plan), len(plan), [-units[i]["level"] for i in plan])


def coverable(units, W):
    """{m: the best plan (unit indices, oldest first)} for every m that disjoint units cover exactly as (W - m, W]"""
    best = {W: []}   # p -> the best plan of (p, W]
    for i in sorted(range(len(units)), key=lambda i: -units[i]["window_last"]):
        u = units[i]
        if u["window_last"] not in best:
            continue
        cand = [i] + best[u["window_last"]]
        p = u["window_first"] - 1
        if p not in best or cost(cand, units) < cost(best[p], units):
            best[p] = cand
    return {W - p: plan for p, plan in best.items() if W - p < 1 << 32}


def choose(ms, N, mode):
    """the span a mode picks among the coverable ones (0 always is)"""
    ms = set(ms) | {0}
    if mode == AT_MOST:
        return max(m for m in ms if m <= N)
    above = [m for m in ms if m >= N]
    return min(above) if above else max(ms)


class SpanModel:
    """The window history, the tiers and every consumed window, driven by the rows each flush returned."""

    def __init__(self):
        self.m0, self.mt = RollupModel(), _Tiers()
        self.wins = {}   # alz_stats.windows -> rows of that consumed window

    def history(self, depth, arena_rows):
        self.m0.history(depth, arena_rows)

    def configure(self, tiers):
        self.mt.configure(tiers)

    def window(self, rows, window, epoch=None):
        self.m0.append(rows, window, epoch)
        self.mt.window(rows, window, epoch)
        self.wins[window] = rows

    def units(self):
        return units_of(self.m0, self.mt)

    def plan(self, N, mode):
        """(m, the units, the plan as unit indices oldest first)"""
        W = max(self.wins, default=0)
        units = self.units()
        cov = coverable(units, W)
        m = choose(cov, N, mode)
        return m, units, cov.get(m, [])

    def span(self, N, mode=AT_MOST):
        """(rows in ascending key order, alz_span_info as a dict) of alz_window_rollup_span(N, mode)"""
        assert N > 0 and mode in (AT_MOST, AT_LEAST)
        m, units, plan = self.plan(N, mode)
        W = max(self.wins, default=0)
        acc = {}
        for w in range(W - m + 1, W + 1):
            for r in self.wins[w]:
                k = packed_key(r)
                acc[k] = add_rows(acc[k], r) if k in acc else r.copy()
        rows = rows_of(acc) if acc else np.zeros(0, dtype=abi.EDGE_OUT)
        entries, open_blocks = [0] * (1 + abi.MAX_TIERS), 0
        for i in plan:
            if units[i]["open"]:
                open_blocks |= 1 << units[i]["level"]
            else:
                entries[units[i]["level"]] += 1
        take = [units[i] for i in plan]
        clocked = bool(take) and all(u["epoch_first"] is not None and u["epoch_last"] is not None for u in take)
        info = dict(windows=m, clocked=int(clocked), window_first=take[0]["window_first"] if take else 0,
                    window_last=take[-1]["window_last"] if take else 0,
                    epoch_first=take[0]["epoch_first"] if clocked else 0,
                    epoch_last=take[-1]["epoch_last"] if clocked else 0, rows_in=sum(u["n"] for u in take),
                    entries=entries, open_blocks=open_blocks)
        return rows, info
