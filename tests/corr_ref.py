"""The correlations of docs/SPEC.md §29 in numpy float64: the reference the GPU tests of alz_*_correlations* compare
against, bit for bit.

A candidate's series (x, px) over P points is what tests/series_ref.py (or node_series_ref.py, group_series_ref.py)
gives for it with one metric; the target (y, py) is the caller's. The loops run over the lag and the point index j with
the rows vectorised, so every SPEC operation is one float64 rounding in the SPEC's order: sums start at +0.0 and add in
ascending j, the means come first, then Sxx, Syy and Sxy about them, and numpy neither fuses nor reorders elementwise
operations."""
import numpy as np

import metric_ref as mr
from alaz_b200 import abi

INVALID = np.uint64(0xFFFFFFFFFFFFFFFF)   # an invalid row's selection value: a negative NaN, key 0


def correlations(x, px, y, py=None, direction=abi.CORR_POSITIVE, absent=abi.CORR_ABSENT_SKIP, max_lag=0,
                 min_points=3, clamp=True):
    """dict of per-row arrays: valid (uint8), lag (uint8), used (uint32), r, score, r0, for candidates x [n, P] float64
    with presence px [n, P] and a target y [P] with presence py [P] (None: every point present). clamp=False leaves r
    unclamped (for tests that need r past 1; not the SPEC)."""
    x = np.asarray(x, dtype=np.float64)
    px = np.asarray(px, dtype=np.uint8) != 0
    n, P = x.shape
    y = np.asarray(y, dtype=np.float64).reshape(P)
    py = np.ones(P, bool) if py is None else np.asarray(py, dtype=np.uint8).reshape(P) != 0
    x = np.where(px, x, 0.0)                  # an absent point is +0.0
    y = np.where(py, y, 0.0)
    zero = absent == abi.CORR_ABSENT_ZERO
    valid = np.zeros(n, bool)
    lag = np.zeros(n, np.uint8)
    used = np.zeros(n, np.int64)
    r_best = np.zeros(n)
    s_best = np.zeros(n)
    used0 = np.zeros(n, np.int64)
    r0 = np.zeros(n)
    for L in range(int(max_lag) + 1):
        sx, sy, u = np.zeros(n), np.zeros(n), np.zeros(n, np.int64)
        for j in range(L, P):
            a = j - L
            use = np.ones(n, bool) if zero else px[:, a] & py[j]
            sx = np.where(use, sx + x[:, a], sx)
            sy = np.where(use, sy + y[j], sy)
            u = u + use
        with np.errstate(divide="ignore", invalid="ignore"):
            mx = np.where(u > 0, sx / np.maximum(u, 1), 0.0)
            my = np.where(u > 0, sy / np.maximum(u, 1), 0.0)
        sxx, syy, sxy = np.zeros(n), np.zeros(n), np.zeros(n)
        for j in range(L, P):
            a = j - L
            use = np.ones(n, bool) if zero else px[:, a] & py[j]
            dx = x[:, a] - mx
            dy = y[j] - my
            sxx = np.where(use, sxx + dx * dx, sxx)
            syy = np.where(use, syy + dy * dy, syy)
            sxy = np.where(use, sxy + dx * dy, sxy)
        den = np.sqrt(sxx) * np.sqrt(syy)
        defined = (u >= int(min_points)) & (den > 0)
        with np.errstate(divide="ignore", invalid="ignore"):
            r = np.where(defined, sxy / np.where(defined, den, 1.0), 0.0)
        if clamp:
            r = np.minimum(np.maximum(r, -1.0), 1.0)
        if direction == abi.CORR_POSITIVE:
            score = r
        elif direction == abi.CORR_NEGATIVE:
            score = 0.0 - r
        elif direction == abi.CORR_ABS:
            score = np.abs(r)
        else:
            raise ValueError(direction)
        better = defined & (~valid | (score > s_best))
        lag = np.where(better, L, lag).astype(np.uint8)
        used = np.where(better, u, used)
        r_best = np.where(better, r, r_best)
        s_best = np.where(better, score, s_best)
        valid = valid | defined
        if L == 0:
            used0 = u
            r0 = np.where(defined, r, 0.0)
    return dict(valid=valid.astype(np.uint8), lag=lag, used=np.where(valid, used, used0).astype(np.uint32),
                r=r_best, score=s_best, r0=r0)


def records(heads, x, px, y, py=None, node=False, **corr):
    """EDGE_CORR (node: NODE_CORR) records of every candidate: heads are EDGE_OUT / EDGE_ENDS-like rows (from_type,
    to_type, from, to) or, for nodes, uint64 node keys (type << 32) | value; None gives zero heads."""
    c = correlations(x, px, y, py, **corr)
    n = len(c["valid"])
    out = np.zeros(n, dtype=abi.NODE_CORR if node else abi.EDGE_CORR)
    if heads is not None:
        if node:
            keys = np.asarray(heads, dtype=np.uint64)
            out["type"] = (keys >> np.uint64(32)).astype(np.uint8)
            out["value"] = (keys & np.uint64(0xFFFFFFFF)).astype(np.uint32)
        else:
            for f in ("from_type", "to_type", "from", "to"):
                out[f] = heads[f]
    out["index"] = np.arange(n, dtype=np.uint32)
    for f in ("valid", "lag", "used", "r", "score", "r0"):
        out[f] = c[f]
    return out


def select_values(rec):
    """The selection value of each record: its score when valid, else all ones."""
    return np.where(rec["valid"] == 1, np.ascontiguousarray(rec["score"]).view(np.uint64), INVALID).view(np.float64)


def top(rec, k, min_score=-np.inf):
    """(indices uint32 in rank order, above) of the records: §17 order over the selection values."""
    return mr.top(select_values(rec), k, min_score)
