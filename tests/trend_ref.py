"""The edge trends of docs/SPEC.md §20 in numpy float64: the reference the GPU tests of alz_edge_trends* compare
against, bit for bit.

A row's series (y, p) over P points is what tests/series_ref.py gives for it with one metric. The loops run over the
point index j with the rows vectorised, so every SPEC operation is one float64 rounding, in the SPEC's order: sums
start at +0.0 and add in ascending j, a mean is its sum divided by the count, and numpy neither fuses nor reorders
elementwise operations."""
import numpy as np

import metric_ref as mr
import series_ref as sr
from alaz_b200 import abi
from change_ref import row_keys

INF = np.inf
INVALID = np.uint64(0xFFFFFFFFFFFFFFFF)   # an invalid row's selection value: a negative NaN, key 0


def _ratio(num, den):
    """num / den, or +inf when den = 0 and num > 0, or 1.0 when both are 0 (the §18 RATIO rule)"""
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(den > 0, num / np.where(den > 0, den, 1.0), np.where(num > 0, INF, 1.0))


def trends(y, p, stat, direction=abi.TREND_RISING, absent=abi.TREND_ABSENT_SKIP, recent=1, min_points=0):
    """dict of per-row arrays: trend, valid (uint8), used (uint32), recent, before, for y [n, P] float64 and
    p [n, P] uint8."""
    y = np.asarray(y, dtype=np.float64)
    p = np.asarray(p, dtype=np.uint8)
    n, P = y.shape
    use = np.ones((n, P), bool) if absent == abi.TREND_ABSENT_ZERO else p.astype(bool)
    y = np.where(p == 1, y, 0.0)         # an absent point's value is +0.0 (the series gives it so)
    lo = max(P - int(recent), 0)         # B = U ∩ [0, lo), R = U ∩ [lo, P)
    su, sb, sr_ = np.zeros(n), np.zeros(n), np.zeros(n)
    nu, nb, nr = (np.zeros(n, np.int64) for _ in range(3))
    sj = np.zeros(n, np.int64)
    for j in range(P):
        u = use[:, j]
        su = np.where(u, su + y[:, j], su)
        sj = sj + np.where(u, j, 0)
        nu = nu + u
        if j < lo:
            sb = np.where(u, sb + y[:, j], sb)
            nb = nb + u
        else:
            sr_ = np.where(u, sr_ + y[:, j], sr_)
            nr = nr + u
    before = np.where(nb > 0, sb / np.maximum(nb, 1), 0.0)
    rec = np.where(nr > 0, sr_ / np.maximum(nr, 1), 0.0)
    falling = direction == abi.TREND_FALLING
    with np.errstate(divide="ignore", invalid="ignore"):
        if stat == abi.TREND_SLOPE:
            ok = nu >= 2
            xm = sj.astype(np.float64) / np.maximum(nu, 1)
            ym = su / np.maximum(nu, 1)
            sxy, sxx = np.zeros(n), np.zeros(n)
            for j in range(P):
                u = use[:, j]
                dx = float(j) - xm
                sxy = np.where(u, sxy + dx * (y[:, j] - ym), sxy)
                sxx = np.where(u, sxx + dx * dx, sxx)
            t = np.where(ok, sxy / np.where(ok, sxx, 1.0), 0.0)
            if falling:
                t = 0.0 - t
        elif stat in (abi.TREND_SHIFT, abi.TREND_RATIO):
            ok = (nr >= 1) & (nb >= 1)
            if stat == abi.TREND_SHIFT:
                t = before - rec if falling else rec - before
            else:
                t = _ratio(before, rec) if falling else _ratio(rec, before)
        elif stat == abi.TREND_ZSCORE:
            ok = (nr >= 1) & (nb >= 2)
            ss = np.zeros(n)
            for j in range(lo):
                u = use[:, j]
                d = y[:, j] - before
                ss = np.where(u, ss + d * d, ss)
            sd = np.sqrt(ss / np.maximum(nb, 1))
            d = before - rec if falling else rec - before
            t = np.where(sd > 0, d / np.where(sd > 0, sd, 1.0), np.where(d > 0, INF, np.where(d < 0, -INF, 0.0)))
        else:
            raise ValueError(stat)
    ok = ok & (nu >= int(min_points))
    t = np.where(ok, t, 0.0)
    return dict(trend=t, valid=ok.astype(np.uint8), used=nu.astype(np.uint32), recent=rec, before=before)


def records(rows, y, p, **spec):
    """EDGE_TREND records of every source row (EDGE_OUT rows, series y [n, P] and p [n, P])."""
    t = trends(y, p, **spec)
    out = np.zeros(len(rows), dtype=abi.EDGE_TREND)
    for f in ("from_type", "to_type", "from", "to"):
        out[f] = rows[f]
    out["index"] = np.arange(len(rows), dtype=np.uint32)
    for f in ("valid", "used", "trend", "recent", "before"):
        out[f] = t[f]
    return out


def select_values(rec):
    """The selection value of each record: its trend when valid, else all ones."""
    return np.where(rec["valid"] == 1, np.ascontiguousarray(rec["trend"]).view(np.uint64), INVALID).view(np.float64)


def top(rec, k, min_trend=-INF):
    """(indices uint32 in rank order, above) of the records: §17 order over the selection values."""
    return mr.top(select_values(rec), k, min_trend)


def expect(entries, rows, spec, k, **trend):
    """(records, y [n, P], p [n, P]) of the source rows `rows` over the last min(k, len(entries)) entries (EDGE_OUT
    row arrays, oldest first), by one metric."""
    v, p = sr.series(entries, row_keys(rows), [spec], k)
    y = v[:, :, 0]
    return records(rows, y, p, **trend), y, p
