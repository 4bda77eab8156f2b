"""Reach (docs/SPEC.md §27) in plain Python: the reference the GPU tests of alz_reach*, alz_group_reach* and
alz_debug_reach_rows compare against, byte for byte.

A level-by-level breadth-first search with sets, independent of the device algorithm. The node list is
tests/node_ref.py's (ascending node key); the group form runs over tests/group_ref.py's group-edge rows. A row is
traversable with no metric, or when metric_ref.order_key of its value is at least that of min_value. DOWN follows
a row from its from end to its to end, UP the other way, ANY both. A node's parent is the smallest node index among
the previous level's nodes with a traversable row to it, its row the smallest such row from that parent."""
import numpy as np

import group_ref
import metric_ref
import node_ref
from alaz_b200 import abi

NONE = abi.REACH_NONE


def seed_keys(seeds):
    """uint64 node keys of (type, value) pairs or a NODE_ENDS / NODE_OUT / REACH_NODE array"""
    if isinstance(seeds, np.ndarray) and seeds.dtype.names:
        return group_ref.node_keys(seeds["type"], seeds["value"])
    return np.array([(int(t) << 32) | int(v) for t, v in seeds], dtype=np.uint64)


def orientations(direction):
    """the (tail, head) orientations a direction follows: 'f' from -> to, 't' to -> from"""
    return {abi.REACH_DOWN: ("f",), abi.REACH_UP: ("t",), abi.REACH_ANY: ("f", "t")}[direction]


def reach(rows, seeds, direction=abi.REACH_DOWN, max_hops=abi.REACH_MAX_HOPS, spec=None, min_value=0.0):
    """(REACH_NODE records, row_index uint32, EDGE_OUT rows, info dict) of a search over an EDGE_OUT array"""
    rows = np.asarray(rows, dtype=abi.EDGE_OUT)
    n = len(rows)
    keys = node_ref.keys(rows)
    kf = group_ref.node_keys(rows["from_type"], rows["from"])
    kt = group_ref.node_keys(rows["to_type"], rows["to"])
    fi = np.searchsorted(keys, kf).tolist()
    ti = np.searchsorted(keys, kt).tolist()
    if spec is None or n == 0:
        trav = [True] * n
    else:
        vk = metric_ref.order_key(metric_ref.values(rows, spec))
        trav = (vk >= metric_ref.order_key(np.array([min_value]))[0]).tolist()
    ori = orientations(direction)
    out = {}   # tail index -> [(head index, row)]
    for r in range(n):
        if not trav[r]:
            continue
        for o in ori:
            u, v = (fi[r], ti[r]) if o == "f" else (ti[r], fi[r])
            out.setdefault(u, []).append((v, r))
    key_set = {int(k): i for i, k in enumerate(keys.tolist())}
    found = {key_set[int(k)] for k in seed_keys(seeds).tolist() if int(k) in key_set}
    hops = {v: 0 for v in found}
    via = {}   # node -> (parent index, row)
    frontier = set(found)
    level = 0
    while frontier and level < max_hops:
        nxt = {}
        for u in frontier:
            for v, r in out.get(u, ()):
                if v in hops:
                    continue
                if v not in nxt or (u, r) < nxt[v]:
                    nxt[v] = (u, r)
        for v, pr in nxt.items():
            hops[v] = level + 1
            via[v] = pr
        frontier = set(nxt)
        if frontier:
            level += 1
    listed = sorted(hops, key=lambda v: (hops[v], v))
    position = {v: j for j, v in enumerate(listed)}
    rec = np.zeros(len(listed), dtype=abi.REACH_NODE)
    for j, v in enumerate(listed):
        k = int(keys[v])
        p, r = via.get(v, (None, NONE))
        rec[j] = (k >> 32, (0, 0, 0), k & 0xFFFFFFFF, hops[v], v, NONE if p is None else position[p], r)
    inf = max_hops + 1
    h = lambda v: hops.get(v, inf)
    row_index, cut = [], 0
    for r in range(n):
        if not trav[r]:
            continue
        ends = [(fi[r], ti[r]) if o == "f" else (ti[r], fi[r]) for o in ori]
        if any(h(u) < max_hops for u, _ in ends):
            row_index.append(r)
        if any(h(u) == max_hops and v not in hops for u, v in ends):
            cut += 1
    row_index = np.array(row_index, dtype=np.uint32)
    info = dict(rows=n, traversable=int(sum(trav)), seeds_found=len(found), nodes=len(listed),
                levels=max(hops.values()) if hops else 0, cut=cut)
    return rec, row_index, rows[row_index], info


def group_reach(rows, seeds, gmap=group_ref.EMPTY, **kw):
    """reach over the group-edge rows of an EDGE_OUT array under a map"""
    return reach(group_ref.group(rows, gmap)[0], seeds, **kw)


def path(rec, j):
    """[(record position, row)] from the seed to record j, following parent and row"""
    out = []
    while rec["parent"][j] != NONE:
        out.append((j, int(rec["row"][j])))
        j = int(rec["parent"][j])
    out.append((j, NONE))
    return out[::-1]
