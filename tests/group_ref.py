"""The group edges, group nodes, their metrics and top of docs/SPEC.md §24 in numpy: the reference the GPU tests of
alz_group_* and alz_debug_group_edges compare against, byte for byte.

A map sends node keys (type << 32) | value to groups; a mapped end becomes the node (NODE_GROUP, g), an unmapped one
stays as it is. Rows equal in both mapped ends are summed (count, err5xx, lat_sum_ns u64 mod 2^64, cells u32 mod
2^32) and listed in ascending (node key of from, node key of to). Group nodes are tests/node_ref.py over those rows,
metrics tests/metric_ref.py, top metric_ref.top."""
import numpy as np

import metric_ref
import node_ref
from alaz_b200 import abi

FIELDS = ("count", "err5xx", "lat_sum_ns")
U32 = np.uint64(32)


def node_keys(types, values):
    return (np.asarray(types).astype(np.uint64) << U32) | np.asarray(values).astype(np.uint64)


def make_map(nodes, groups):
    """(sorted node keys, their groups) of a map given as (type, value) pairs or a NODE_ENDS array and group ids"""
    if isinstance(nodes, np.ndarray) and nodes.dtype.names:
        keys = node_keys(nodes["type"], nodes["value"])
    else:
        keys = np.array([(int(t) << 32) | int(v) for t, v in nodes], dtype=np.uint64)
    groups = np.asarray(groups, dtype=np.uint64)
    order = np.argsort(keys, kind="stable")
    keys, groups = keys[order], groups[order]
    assert len(np.unique(keys)) == len(keys), "a node twice in one map"
    return keys, groups


EMPTY = (np.zeros(0, dtype=np.uint64), np.zeros(0, dtype=np.uint64))


def map_keys(keys, gmap):
    """(mapped keys, held) of node keys under a map"""
    mk, mg = gmap
    if len(mk) == 0:
        return keys.copy(), np.zeros(len(keys), dtype=bool)
    pos = np.minimum(np.searchsorted(mk, keys), len(mk) - 1)
    held = mk[pos] == keys
    out = keys.copy()
    out[held] = (np.uint64(abi.NODE_GROUP) << U32) | mg[pos[held]]
    return out, held


def group(rows, gmap=EMPTY):
    """(EDGE_OUT group-edge rows, info dict) of an EDGE_OUT array under a map"""
    rows = np.asarray(rows, dtype=abi.EDGE_OUT)
    kf, hf = map_keys(node_keys(rows["from_type"], rows["from"]), gmap)
    kt, ht = map_keys(node_keys(rows["to_type"], rows["to"]), gmap)
    info = dict(source_rows=len(rows), mapped_ends=int(hf.sum() + ht.sum()), edges=0, internal=int((kf == kt).sum()))
    if len(rows) == 0:
        return np.zeros(0, dtype=abi.EDGE_OUT), info
    order = np.lexsort((kt, kf))
    kf, kt, r = kf[order], kt[order], rows[order]
    starts = np.flatnonzero(np.r_[True, (kf[1:] != kf[:-1]) | (kt[1:] != kt[:-1])])
    out = np.zeros(len(starts), dtype=abi.EDGE_OUT)
    out["from_type"] = (kf[starts] >> U32).astype(np.uint8)
    out["from"] = (kf[starts] & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    out["to_type"] = (kt[starts] >> U32).astype(np.uint8)
    out["to"] = (kt[starts] & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    for f in FIELDS:
        out[f] = np.add.reduceat(r[f].astype(np.uint64), starts)   # uint64 adds wrap mod 2^64
    out["hist"] = np.add.reduceat(r["hist"], starts, axis=0, dtype=np.uint32)   # uint32 adds wrap mod 2^32
    info["edges"] = len(out)
    return out, info


def nodes(rows, gmap=EMPTY):
    """the NODE_OUT rows of the group-edge rows"""
    return node_ref.group(group(rows, gmap)[0])


def edge_matrix(edges, specs):
    return metric_ref.matrix(edges, specs)


def edge_top(edges, spec, k, min_value):
    """(row indices uint32 in rank order, above)"""
    return metric_ref.top(metric_ref.values(edges, spec), k, min_value)
