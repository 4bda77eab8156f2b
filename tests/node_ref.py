"""The node rows, node metrics and top nodes of docs/SPEC.md §21 in numpy: the reference the GPU tests of
alz_node_rows*, alz_node_metrics*, alz_node_top* and alz_debug_node_rows compare against, byte for byte.

A node is an edge end (type, value), keyed (type << 32) | value; nodes are listed in ascending key. Side IN of a node
sums the rows whose to end is the node, side OUT the rows whose from end is (a row with both ends on one node counts on
both). count, err5xx and lat_sum_ns are u64 sums mod 2^64, the cells u32 sums mod 2^32. A node metric is the §17 value
(tests/metric_ref.py) of an EDGE_OUT row that carries one side's sums; the top nodes rank as metric_ref.top ranks rows."""
import numpy as np

import metric_ref
from alaz_b200 import abi

SIDES = {abi.SIDE_IN: "in", abi.SIDE_OUT: "out"}
FIELDS = ("count", "err5xx", "lat_sum_ns")


def end_keys(rows, side):
    """uint64 node keys of every row's to end (SIDE_IN) or from end (SIDE_OUT)"""
    t, v = ("to_type", "to") if side == abi.SIDE_IN else ("from_type", "from")
    return (rows[t].astype(np.uint64) << np.uint64(32)) | rows[v].astype(np.uint64)


def keys(rows):
    """the ascending node keys of an EDGE_OUT array"""
    rows = np.asarray(rows, dtype=abi.EDGE_OUT)
    return np.unique(np.concatenate([end_keys(rows, abi.SIDE_IN), end_keys(rows, abi.SIDE_OUT)]))


def group(rows):
    """the NODE_OUT rows of an EDGE_OUT array, in node order"""
    rows = np.asarray(rows, dtype=abi.EDGE_OUT)
    uniq = keys(rows)
    out = np.zeros(len(uniq), dtype=abi.NODE_OUT)
    out["type"] = (uniq >> np.uint64(32)).astype(np.uint8)
    out["value"] = (uniq & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    for side, name in SIDES.items():
        ids = np.searchsorted(uniq, end_keys(rows, side))
        order = np.argsort(ids, kind="stable")
        ids, r = ids[order], rows[order]
        if len(ids) == 0:
            continue
        starts = np.flatnonzero(np.r_[True, ids[1:] != ids[:-1]])
        nid = ids[starts]
        out[f"{name}_edges"][nid] = np.diff(np.r_[starts, len(ids)])
        sums = out[name]
        for f in FIELDS:
            sums[f][nid] = np.add.reduceat(r[f].astype(np.uint64), starts)   # uint64 adds wrap mod 2^64
        sums["hist"][nid] = np.add.reduceat(r["hist"], starts, axis=0, dtype=np.uint32)   # uint32 adds wrap mod 2^32
    return out


def side_rows(nodes, side):
    """EDGE_OUT rows that carry one side's sums of each node (the ends are left 0)"""
    out = np.zeros(len(nodes), dtype=abi.EDGE_OUT)
    s = nodes[SIDES[side]]
    for f in FIELDS + ("hist",):
        out[f] = s[f]
    return out


def values(nodes, side, spec):
    """float64 values of one metric of one side for every node"""
    return metric_ref.values(side_rows(nodes, side), spec)


def matrix(nodes, side, specs):
    """values[i, j]: metric j of node i's side"""
    return metric_ref.matrix(side_rows(nodes, side), specs)


def top(nodes, side, spec, k, min_value):
    """(node indices uint32 in rank order, above)"""
    return metric_ref.top(values(nodes, side, spec), k, min_value)
