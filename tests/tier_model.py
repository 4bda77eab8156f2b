"""Sequential model of the tiered history (docs/SPEC.md §13), built on tests/rollup_model.py: each tier's retained
entries follow the §12 ring rule (a RollupModel per tier), each tier's open block is a {packed key -> row} dict fed
by the consumed windows (tier 1) or the closed blocks of the tier below."""
import numpy as np

from alaz_b200 import abi
from rollup_model import RollupModel, add_rows, packed_key


def rows_of(acc):
    """A {packed key -> row} dict as an alz_edge_out array in ascending key order."""
    rows = np.zeros(len(acc), dtype=abi.EDGE_OUT)
    for i, key in enumerate(sorted(acc)):
        rows[i] = acc[key]
    return rows


class _Tier:
    def __init__(self, factor, depth, arena_rows, block_rows):
        self.factor, self.block_rows = factor, block_rows
        self.ring = RollupModel()
        self.ring.history(depth, arena_rows)
        self.dropped = 0
        self.reset()

    def reset(self):
        self.acc, self.inputs, self.poisoned, self.overflow = {}, 0, False, False
        self.window_first = self.epoch_first = self.epoch_last = None
        self.windows, self.clocked = 0, True


class TierModel:
    def __init__(self):
        self.cfg, self.tiers = (), []

    def configure(self, tiers):
        """tiers: a list of (factor, depth, arena_rows, block_rows), tier 1 first."""
        tiers = tuple(tuple(int(x) for x in t) for t in tiers)
        if tiers == self.cfg:
            return
        self.cfg, self.tiers = tiers, [_Tier(*t) for t in tiers]

    def window(self, rows, window, epoch=None):
        """A flush consumed its window: `rows` what it returned, `window` alz_stats.windows after it, `epoch` the
        epoch it closed under a window clock (None: not clocked)."""
        if self.tiers:
            self._input(0, {packed_key(r): r.copy() for r in rows}, window, window, 1, epoch, epoch, False)

    def _input(self, t, acc_in, window_first, window_last, windows, epoch_first, epoch_last, poisoned):
        tier = self.tiers[t]
        if tier.inputs == 0:
            tier.window_first, tier.epoch_first = window_first, epoch_first
        tier.epoch_last = epoch_last
        tier.clocked &= epoch_first is not None and epoch_last is not None
        tier.windows += windows
        tier.poisoned |= poisoned
        if not tier.poisoned:
            for key, r in acc_in.items():
                tier.acc[key] = add_rows(tier.acc[key], r) if key in tier.acc else r.copy()
            tier.overflow |= len(tier.acc) > tier.block_rows
        tier.inputs += 1
        if tier.inputs < tier.factor:
            return
        # the block closes
        drop = tier.poisoned or tier.overflow or len(tier.acc) > tier.ring.arena_rows
        ef, el = (tier.epoch_first, tier.epoch_last) if tier.clocked else (None, None)
        if drop:
            tier.ring.entries = []
            tier.dropped += 1
        else:
            tier.ring.append(rows_of(tier.acc), window_last)
            tier.ring.entries[-1].update(window_first=tier.window_first, windows=tier.windows, epoch_first=ef,
                                         epoch_last=el)
        acc, wf, windows = tier.acc, tier.window_first, tier.windows
        tier.reset()
        if t + 1 < len(self.tiers):
            self._input(t + 1, {} if drop else acc, wf, window_last, windows, ef, el, drop)

    def rollup(self, tier, k):
        """(rows in ascending key order, alz_rollup_info as a dict) of the last k entries of tier 1..n"""
        assert k > 0
        ring = self.tiers[tier - 1].ring
        rows, _ = ring.rollup(k)
        take = ring.entries[-k:]
        clocked = bool(take) and all(e["epoch_first"] is not None for e in take)
        info = dict(windows=sum(e["windows"] for e in take), clocked=int(clocked),
                    window_first=take[0]["window_first"] if take else 0, window_last=take[-1]["window"] if take else 0,
                    epoch_first=take[0]["epoch_first"] if clocked else 0,
                    epoch_last=take[-1]["epoch_last"] if clocked else 0, rows_in=sum(e["n"] for e in take))
        return rows, info

    def state(self, tier):
        t = self.tiers[tier - 1]
        per_input = int(np.prod([f for f, _, _, _ in self.cfg[: tier - 1]], dtype=np.int64)) if tier > 1 else 1
        return dict(entries=len(t.ring.entries), open_windows=t.inputs * per_input, dropped=t.dropped)
