"""The group changes of docs/SPEC.md §25 in numpy: the reference the GPU tests of alz_group_edge_changes*,
alz_group_node_changes* and alz_debug_group_edge_changes_rows compare against, byte for byte.

Both sides are grouped by one map (tests/group_ref.py). Group edge changes are tests/change_ref.py's rules over the two
group-edge lists, matched by the pair (node key of from, node key of to) rather than the §3 packed key, in that
ascending order: a pair of ends needs 70 bits, so no 64-bit key stands in for it. Group node changes are
tests/node_change_ref.py over the two group-node lists. The top calls rank as metric_ref.top over the list's changes."""
import numpy as np

import change_ref
import group_ref
import metric_ref
import node_change_ref
from alaz_b200 import abi

ABSENT = abi.ABSENT


def ends_keys(rows):
    """(node keys of the from ends, node keys of the to ends) of EDGE_OUT rows"""
    return (group_ref.node_keys(rows["from_type"], rows["from"]), group_ref.node_keys(rows["to_type"], rows["to"]))


def edge_changes_of(ga, gb, spec, mode, presence, src_windows=1, base_windows=1):
    """(EDGE_CHANGE records, info dict with above = 0) of two group-edge lists, each strictly ascending in (from key,
    to key)."""
    fa, ta = ends_keys(ga)
    fb, tb = ends_keys(gb)
    for f, t in ((fa, ta), (fb, tb)):
        assert np.all((f[1:] > f[:-1]) | ((f[1:] == f[:-1]) & (t[1:] > t[:-1]))), "each side must be strictly ascending"
    na, nb = len(ga), len(gb)
    f, t = np.concatenate([fa, fb]), np.concatenate([ta, tb])
    order = np.lexsort((t, f))
    fs, ts = f[order], t[order]
    start = np.r_[True, (fs[1:] != fs[:-1]) | (ts[1:] != ts[:-1])] if len(fs) else np.zeros(0, bool)
    rank = np.empty(len(f), np.int64)
    rank[order] = np.cumsum(start) - 1
    nu = int(start.sum())
    pa, pb = np.full(nu, -1, np.int64), np.full(nu, -1, np.int64)
    pa[rank[:na]] = np.arange(na)
    pb[rank[na:]] = np.arange(nb)
    in_a, in_b = pa >= 0, pb >= 0
    both = int((in_a & in_b).sum())
    pres = np.where(in_a & in_b, abi.PRESENT_BOTH, np.where(in_a, abi.PRESENT_NEW, abi.PRESENT_GONE)).astype(np.uint8)
    keep = (pres & np.uint8(presence)) != 0
    pa, pb, in_a, in_b, pres = pa[keep], pb[keep], in_a[keep], in_b[keep], pres[keep]
    va = change_ref.side_values(ga, spec, src_windows)
    vb = change_ref.side_values(gb, spec, base_windows)
    out = np.zeros(len(pres), dtype=abi.EDGE_CHANGE)
    out["presence"] = pres
    out["index"] = np.where(in_a, pa, ABSENT)
    out["base_index"] = np.where(in_b, pb, ABSENT)
    for fld in ("from_type", "to_type", "from", "to"):
        out[fld] = np.where(in_a, ga[fld][np.maximum(pa, 0)] if na else 0, gb[fld][np.maximum(pb, 0)] if nb else 0)
    out["value"] = np.where(in_a, va[np.maximum(pa, 0)] if na else 0.0, 0.0)
    out["base_value"] = np.where(in_b, vb[np.maximum(pb, 0)] if nb else 0.0, 0.0)
    out["change"] = change_ref.change_of(mode, out["value"], out["base_value"])
    info = dict(source_rows=na, base_rows=nb, both=both, added=na - both, gone=nb - both, listed=len(out), above=0,
                source_windows=int(src_windows), base_windows=int(base_windows))
    return out, info


def edge_changes(src, base, gmap, spec, mode, presence, src_windows=1, base_windows=1):
    """The group edge changes of two EDGE_OUT arrays (any order) under one map: (records, info dict)."""
    return edge_changes_of(group_ref.group(src, gmap)[0], group_ref.group(base, gmap)[0], spec, mode, presence,
                           src_windows, base_windows)


def node_changes(src, base, gmap, side, spec, mode, presence, src_windows=1, base_windows=1):
    """The group node changes of side `side` of two EDGE_OUT arrays (any order) under one map: (records, info)."""
    return node_change_ref.changes_of_nodes(group_ref.nodes(src, gmap), group_ref.nodes(base, gmap), side, spec, mode,
                                            presence, src_windows, base_windows)


def top(lst, info, k, min_change):
    """(the first min(k, above) records of a change list by change in rank order, info dict with above set)."""
    idx, above = metric_ref.top(lst["change"], k, min_change)
    return lst[idx], dict(info, above=above)
