"""The group series and group trends of docs/SPEC.md §26 in numpy: the reference the GPU tests of alz_group_*_series*
and alz_group_*_trends* compare against, bit for bit.

One map groups every entry and the source (group_ref.group). A group-edge series row is a (from key, to key) pair of
node keys; point j is present when entry j, grouped alone, holds that group edge, and its values are then the §17
values of that group-edge row (metric_ref). A group-node series row is a node key; point j is the §22 point of the
node over entry j grouped alone (node_series_ref.series over the grouped entries). Trends are trend_ref's statistic
over those series; records carry the group-edge row's ends or the group node's key."""
import numpy as np

import group_ref as gr
import metric_ref as mr
import node_ref as nr
import node_series_ref as nsr
import series_ref as sr
import trend_ref as tr
from alaz_b200 import abi

M29 = 1 << 29


def pack_node(t, v):
    """The node key of a caller's §26 node, or None for a malformed one: §22's rules, or (NODE_GROUP, g < 2^29)."""
    t, v = int(t), int(v)
    if t == abi.NODE_GROUP:
        return (t << 32) | v if v < M29 else None
    return nsr.pack(t, v)


def pack_edge(ft, f, tt, t):
    """The (from key, to key) of a caller's §26 group edge, or None: §19's rules when neither end is a group, else two
    valid node keys."""
    if int(ft) != abi.NODE_GROUP and int(tt) != abi.NODE_GROUP:
        if sr.pack_ends(ft, f, tt, t) is None:
            return None
        return (int(ft) << 32) | int(f), (int(tt) << 32) | int(t)
    kf, kt = pack_node(ft, f), pack_node(tt, t)
    return None if kf is None or kt is None else (kf, kt)


def node_ends_keys(ends):
    """uint64 keys of a NODE_ENDS array; ValueError when one is malformed."""
    out = np.zeros(len(ends), dtype=np.uint64)
    for i, e in enumerate(ends):
        k = pack_node(e["type"], e["value"])
        if k is None:
            raise ValueError(f"malformed key {i}")
        out[i] = k
    return out


def edge_ends_keys(ends):
    """(from keys, to keys) uint64 of an EDGE_ENDS (or EDGE_OUT) array; ValueError when one is malformed."""
    kf = np.zeros(len(ends), dtype=np.uint64)
    kt = np.zeros(len(ends), dtype=np.uint64)
    for i, e in enumerate(ends):
        k = pack_edge(e["from_type"], e["from"], e["to_type"], e["to"])
        if k is None:
            raise ValueError(f"malformed key {i}")
        kf[i], kt[i] = k
    return kf, kt


def row_ends(rows):
    """(from keys, to keys) of EDGE_OUT rows"""
    return gr.node_keys(rows["from_type"], rows["from"]), gr.node_keys(rows["to_type"], rows["to"])


def _take(entries, k):
    return entries if k is None else entries[max(len(entries) - int(k), 0):]


def edge_series(entries, kf, kt, specs, gmap=gr.EMPTY, k=None):
    """(values [n, P, nm], present [n, P]) of the group edges (kf[i], kt[i]) over the last min(k, len(entries))
    entries, each grouped by gmap alone."""
    take = _take(entries, k)
    kf, kt = np.asarray(kf, dtype=np.uint64), np.asarray(kt, dtype=np.uint64)
    n, P, nm = len(kf), len(take), len(specs)
    values = np.zeros((n, P, nm))
    present = np.zeros((n, P), dtype=np.uint8)
    for j, rows in enumerate(take):
        g = gr.group(rows, gmap)[0]
        if len(g) == 0 or n == 0:
            continue
        gf, gt = row_ends(g)
        idx = {(int(a), int(b)): i for i, (a, b) in enumerate(zip(gf, gt))}
        vals = mr.matrix(g, specs)
        for i in range(n):
            u = idx.get((int(kf[i]), int(kt[i])))
            if u is not None:
                values[i, j, :] = vals[u]
                present[i, j] = 1
    return values, present


def node_series(entries, keys, side, specs, gmap=gr.EMPTY, k=None):
    """(values [n, P, nm], present [n, P]) of side `side` of the nodes `keys` over the last min(k, len(entries))
    entries, each grouped by gmap alone."""
    grouped = [gr.group(rows, gmap)[0] for rows in _take(entries, k)]
    return nsr.series(grouped, keys, side, specs)


def source_edges(rows, gmap=gr.EMPTY):
    """the source's group-edge rows: the series rows of a by-source group edge call"""
    return gr.group(rows, gmap)[0]


def source_nodes(rows, gmap=gr.EMPTY):
    """the source's group nodes (NODE_OUT): the series rows of a by-source group node call"""
    return gr.nodes(rows, gmap)


def edge_expect(entries, rows, spec, k, gmap=gr.EMPTY, **trend):
    """(records, y [n, P], p [n, P]) of the group edges of the source rows `rows`, by one metric."""
    g = source_edges(rows, gmap)
    v, p = edge_series(entries, *row_ends(g), [spec], gmap, k)
    y = v[:, :, 0]
    return tr.records(g, y, p, **trend), y, p


def node_expect(entries, rows, side, spec, k, gmap=gr.EMPTY, **trend):
    """(records, y [n, P], p [n, P]) of the group nodes of the source rows `rows`, by one metric of one side."""
    keys = nr.keys(source_edges(rows, gmap))
    v, p = node_series(entries, keys, side, [spec], gmap, k)
    y = v[:, :, 0]
    return nsr.records(keys, y, p, **trend), y, p


def top(rec, k, min_trend=-np.inf):
    """(indices uint32 in rank order, above)"""
    return tr.top(rec, k, min_trend)
