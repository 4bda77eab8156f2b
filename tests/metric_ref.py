"""The edge metrics and the top edges of docs/SPEC.md §17 in numpy float64: the reference the GPU tests of
alz_edge_metrics*, alz_edge_top* and the debug hooks compare against, bit for bit.

A metric is a METRIC_* kind, or a (METRIC_QUANTILE, q) pair. Each row's value is a float64; the quantile is SPEC §5
(gnn_ref.quantiles_vec, which tests/test_metric_ref.py pins against alz_edge_quantiles and the oracle). Each value's
bits u map to a 64-bit key: u ^ 2^63 when the sign bit is clear, ~u when it is set (IEEE total order). Rows rank by
key descending, then by index ascending; a row is eligible when key(value) >= key(min_value)."""
import numpy as np

import gnn_ref
from alaz_b200 import abi

SIGN = np.uint64(1 << 63)


def values(rows, spec):
    """float64 values of one metric for every row of an EDGE_OUT array."""
    kind, q = (spec if isinstance(spec, tuple) else (spec, 0.0))
    count = rows["count"].astype(np.float64)
    nz = rows["count"] != 0
    safe = np.where(nz, count, 1.0)
    if kind == abi.METRIC_COUNT:
        return count
    if kind == abi.METRIC_ERR5XX:
        return rows["err5xx"].astype(np.float64)
    if kind == abi.METRIC_ERR_RATE:
        return np.where(nz, rows["err5xx"].astype(np.float64) / safe, 0.0)
    if kind == abi.METRIC_MEAN_NS:
        return np.where(nz, rows["lat_sum_ns"].astype(np.float64) / safe, 0.0)
    if kind == abi.METRIC_QUANTILE:
        if len(rows) == 0:
            return np.zeros(0)
        return gnn_ref.quantiles_vec(rows["hist"], float(q))
    raise ValueError(kind)


def matrix(rows, specs):
    """values[i, j]: metric j of row i."""
    out = np.zeros((len(rows), len(specs)))
    for j, s in enumerate(specs):
        out[:, j] = values(rows, s)
    return out


def order_key(v):
    """uint64 keys of float64 values (an array or a scalar)."""
    u = np.atleast_1d(np.asarray(v, dtype=np.float64)).view(np.uint64)
    return np.where(u & SIGN, ~u, u ^ SIGN).astype(np.uint64)


def top(v, k, min_value):
    """(indices uint32 in rank order, above): lexsort on (index, -key), eligible rows only, cut at k."""
    key = order_key(v)
    kmin = order_key(min_value)[0]
    elig = np.flatnonzero(key >= kmin)
    # -key as a uint64 that sorts ascending where key sorts descending: ~key
    order = elig[np.lexsort((elig, ~key[elig]))]
    return order[: int(k)].astype(np.uint32), len(elig)
