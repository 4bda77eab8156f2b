"""The node series and node trends of docs/SPEC.md §22 in numpy: the reference the GPU tests of alz_node_series* and
alz_node_trends* compare against, bit for bit.

A node series is a set of nodes (node keys (type << 32) | value, one per series row, duplicates allowed), a side and
the last P = min(k, retained) entries of a ring, oldest first, each given as its EDGE_OUT rows. Point j of node i is
present when entry j has a row on the side of the node; its values are then the §17 values of the side's §21 sums over
entry j's rows (node_ref.group of the entry alone), else present 0 and +0.0 for every metric. A node trend is the §20
statistic (trend_ref.trends) of a node's series of one metric."""
import numpy as np

import node_ref as nr
import trend_ref as tr
from alaz_b200 import abi

M29 = 1 << 29


def pack(t, v):
    """The node key of a caller's node, or None for a malformed one: a type above NODE_OUTBOUND_HOST, or a pod or
    service value >= 2^29."""
    t, v = int(t), int(v)
    if t > abi.NODE_OUTBOUND_HOST or (t in (abi.NODE_POD, abi.NODE_SVC) and v >= M29):
        return None
    return (t << 32) | v


def ends_keys(ends):
    """uint64 keys of a NODE_ENDS (or NODE_OUT) array; ValueError when one is malformed."""
    out = np.zeros(len(ends), dtype=np.uint64)
    for i, e in enumerate(ends):
        k = pack(e["type"], e["value"])
        if k is None:
            raise ValueError(f"malformed key {i}")
        out[i] = k
    return out


def node_keys(nodes):
    """uint64 keys of NODE_OUT rows"""
    return (nodes["type"].astype(np.uint64) << np.uint64(32)) | nodes["value"].astype(np.uint64)


def series(entries, keys, side, specs, k=None):
    """(values [n, P, nm] float64, present [n, P] uint8) of side `side` of the nodes `keys` (uint64) over the last
    min(k, len(entries)) entries (k None: all)."""
    take = entries if k is None else entries[max(len(entries) - int(k), 0):]
    keys = np.asarray(keys, dtype=np.uint64)
    n, P, nm = len(keys), len(take), len(specs)
    values = np.zeros((n, P, nm))
    present = np.zeros((n, P), dtype=np.uint8)
    edges = "in_edges" if side == abi.SIDE_IN else "out_edges"
    for j, rows in enumerate(take):
        if len(rows) == 0 or n == 0:
            continue
        g = nr.group(rows)
        gk = node_keys(g)
        pos = np.minimum(np.searchsorted(gk, keys), len(gk) - 1)
        hit = (gk[pos] == keys) & (g[edges][pos] > 0)   # a node seen only on the other side is absent on this one
        vals = nr.matrix(g, side, specs)
        values[hit, j, :] = vals[pos[hit]]
        present[hit, j] = 1
    return values, present


def records(keys, y, p, **trend):
    """NODE_TREND records of the nodes `keys` (in node order) over series y [n, P] and p [n, P]."""
    keys = np.asarray(keys, dtype=np.uint64)
    t = tr.trends(y, p, **trend)
    out = np.zeros(len(keys), dtype=abi.NODE_TREND)
    out["type"] = (keys >> np.uint64(32)).astype(np.uint8)
    out["value"] = (keys & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    out["index"] = np.arange(len(keys), dtype=np.uint32)
    for f in ("valid", "used", "trend", "recent", "before"):
        out[f] = t[f]
    return out


def expect(entries, rows, side, spec, k, **trend):
    """(records, y [n, P], p [n, P]) of the nodes of the source rows `rows` over the last min(k, len(entries)) entries,
    by one metric of one side."""
    keys = nr.keys(rows)
    v, p = series(entries, keys, side, [spec], k)
    y = v[:, :, 0]
    return records(keys, y, p, **trend), y, p


def top(rec, k, min_trend=-np.inf):
    """(node indices uint32 in rank order, above): the §17 order over the records' selection values."""
    return tr.top(rec, k, min_trend)
