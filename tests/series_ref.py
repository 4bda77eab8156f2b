"""The edge series of docs/SPEC.md §19 in numpy float64: the reference the GPU tests of alz_edge_series* compare
against, bit for bit.

A series is a set of edges (packed keys, §3, one per series row, duplicates allowed) and the last P = min(k, retained)
entries of a ring, oldest first, each given as its EDGE_OUT rows in ascending key order. Point j of edge i is the row
entry j holds with the edge's key: present 1 and the §17 values of that row (metric_ref.values), or present 0 and
+0.0 for every metric."""
import numpy as np

import metric_ref as mr
from alaz_b200 import abi
from change_ref import row_keys

M29 = 1 << 29


def pack_ends(ft, f, tt, t):
    """The packed key of a caller's edge (alz_device.cuh pack_edge_ends), or None for ends no flush emits: a type
    above NODE_OUTBOUND_HOST, no pod end, or a pod or service id >= 2^29."""
    ft, f, tt, t = int(ft), int(f), int(tt), int(t)
    if ft > abi.NODE_OUTBOUND_HOST or tt > abi.NODE_OUTBOUND_HOST:
        return None
    for ty, v in ((ft, f), (tt, t)):
        if ty in (abi.NODE_POD, abi.NODE_SVC) and v >= M29:
            return None
    if ft == abi.NODE_POD:
        return (tt << 61) | (f << 32) | t
    if tt == abi.NODE_POD:
        return (1 << 63) | (ft << 61) | (t << 32) | f
    return None


def ends_keys(ends):
    """uint64 keys of an EDGE_ENDS (or EDGE_OUT) array; ValueError when one is malformed."""
    out = np.zeros(len(ends), dtype=np.uint64)
    for i, e in enumerate(ends):
        k = pack_ends(e["from_type"], e["from"], e["to_type"], e["to"])
        if k is None:
            raise ValueError(f"malformed key {i}")
        out[i] = k
    return out


def series(entries, keys, specs, k=None):
    """(values [n, P, nm] float64, present [n, P] uint8) of the edges `keys` (uint64) over the last min(k, len(entries))
    entries (k None: all)."""
    take = entries if k is None else entries[max(len(entries) - int(k), 0):]
    keys = np.asarray(keys, dtype=np.uint64)
    n, P, nm = len(keys), len(take), len(specs)
    values = np.zeros((n, P, nm))
    present = np.zeros((n, P), dtype=np.uint8)
    for j, rows in enumerate(take):
        if len(rows) == 0 or n == 0:
            continue
        rk = row_keys(rows)
        assert np.all(rk[1:] > rk[:-1]), "an entry's rows are strictly ascending"
        pos = np.minimum(np.searchsorted(rk, keys), len(rk) - 1)
        hit = rk[pos] == keys
        vals = mr.matrix(rows, specs)
        values[hit, j, :] = vals[pos[hit]]
        present[hit, j] = 1
    return values, present
