"""The node changes of docs/SPEC.md §23 in numpy: the reference the GPU tests of alz_node_changes*,
alz_node_changes_top* and alz_debug_node_changes_rows compare against, byte for byte.

Each side's node list is the §21 node list of its rows (node_ref.group). A node is a member of a list on side `side`
when it has a row there (in_edges > 0 for IN, out_edges > 0 for OUT). The list is the union of the two lists' members,
matched by node key (type << 32) | value, in ascending key order, and filtered by a presence mask. index / base_index
are positions in the full node lists. Each side's value is the §17 value of one metric on the node's side sums,
divided by the side's windows for COUNT and ERR5XX (change_ref.side_values); a side where the node is absent gives
+0.0. The change and the top follow §18 (change_ref.change_of, metric_ref.top)."""
import numpy as np

import change_ref
import metric_ref
import node_ref
from alaz_b200 import abi

ABSENT = abi.ABSENT


def node_keys(nodes):
    return (nodes["type"].astype(np.uint64) << np.uint64(32)) | nodes["value"].astype(np.uint64)


def members(nodes, side):
    """bool per node: it has a row on `side`"""
    return nodes[f"{node_ref.SIDES[side]}_edges"] > 0


def changes_of_nodes(na, nb, side, spec, mode, presence, src_windows=1, base_windows=1):
    """(NODE_CHANGE records, info dict with above = 0) of two NODE_OUT lists, each in ascending node key order."""
    ka, kb = node_keys(na), node_keys(nb)
    assert np.all(ka[1:] > ka[:-1]) and np.all(kb[1:] > kb[:-1])
    ia_m, ib_m = np.flatnonzero(members(na, side)), np.flatnonzero(members(nb, side))
    ka_m, kb_m = ka[ia_m], kb[ib_m]
    va = change_ref.side_values(node_ref.side_rows(na, side), spec, src_windows)
    vb = change_ref.side_values(node_ref.side_rows(nb, side), spec, base_windows)
    keys = np.union1d(ka_m, kb_m)
    pa, pb = np.searchsorted(ka_m, keys), np.searchsorted(kb_m, keys)
    in_a = pa < len(ka_m)
    in_a[in_a] = ka_m[pa[in_a]] == keys[in_a]
    in_b = pb < len(kb_m)
    in_b[in_b] = kb_m[pb[in_b]] == keys[in_b]
    pres = np.where(in_a & in_b, abi.PRESENT_BOTH, np.where(in_a, abi.PRESENT_NEW, abi.PRESENT_GONE)).astype(np.uint8)
    keep = (pres & np.uint8(presence)) != 0
    keys, pa, pb, in_a, in_b, pres = keys[keep], pa[keep], pb[keep], in_a[keep], in_b[keep], pres[keep]
    index = np.full(len(keys), ABSENT, np.uint32)
    index[in_a] = ia_m[pa[in_a]]
    base_index = np.full(len(keys), ABSENT, np.uint32)
    base_index[in_b] = ib_m[pb[in_b]]
    out = np.zeros(len(keys), dtype=abi.NODE_CHANGE)
    out["type"] = (keys >> np.uint64(32)).astype(np.uint8)
    out["node"] = (keys & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    out["presence"] = pres
    out["index"] = index
    out["base_index"] = base_index
    value = np.zeros(len(keys))
    value[in_a] = va[index[in_a]]
    base = np.zeros(len(keys))
    base[in_b] = vb[base_index[in_b]]
    out["value"] = value
    out["base_value"] = base
    out["change"] = change_ref.change_of(mode, value, base)
    both = int(np.isin(ka_m, kb_m).sum())
    info = dict(source_rows=len(ka_m), base_rows=len(kb_m), both=both, added=len(ka_m) - both,
                gone=len(kb_m) - both, listed=len(out), above=0, source_windows=int(src_windows),
                base_windows=int(base_windows))
    return out, info


def changes(src, base, side, spec, mode, presence, src_windows=1, base_windows=1):
    """(NODE_CHANGE records of the filtered union in ascending node key order, info dict with above = 0). src and base
    are EDGE_OUT arrays in any order."""
    return changes_of_nodes(node_ref.group(src), node_ref.group(base), side, spec, mode, presence, src_windows,
                            base_windows)


def top(src, base, side, spec, mode, presence, k, min_change, src_windows=1, base_windows=1):
    """(the first min(k, above) records by change in rank order, info dict with above set)."""
    lst, info = changes(src, base, side, spec, mode, presence, src_windows, base_windows)
    idx, above = metric_ref.top(lst["change"], k, min_change)
    return lst[idx], dict(info, above=above)
