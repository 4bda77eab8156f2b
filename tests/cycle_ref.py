"""Cycles (docs/SPEC.md §28) in plain Python: the reference the GPU tests of alz_cycles*, alz_group_cycles* and
alz_debug_cycles_rows compare against, byte for byte.

An iterative Tarjan over the traversable rows (from end -> to end; self rows left out), independent of the device
algorithm, then the longest paths over the condensation in topological order, both ways. The node list is
tests/node_ref.py's (ascending node key); the group form runs over tests/group_ref.py's group-edge rows. A row is
traversable with no metric, or when metric_ref.order_key of its value is at least that of min_value, as in
tests/reach_ref.py."""
import numpy as np

import group_ref
import metric_ref
import node_ref
from alaz_b200 import abi


def tarjan(n, adj):
    """the strongly connected components of nodes 0 .. n - 1 with successor lists adj: comp[v], a label per component"""
    index, low, comp = [-1] * n, [0] * n, [-1] * n
    on, stack, counter, label = [False] * n, [], 0, 0
    for root in range(n):
        if index[root] >= 0:
            continue
        work = [(root, 0)]
        index[root] = low[root] = counter
        counter += 1
        stack.append(root)
        on[root] = True
        while work:
            v, i = work[-1]
            if i < len(adj[v]):
                work[-1] = (v, i + 1)
                w = adj[v][i]
                if index[w] < 0:
                    index[w] = low[w] = counter
                    counter += 1
                    stack.append(w)
                    on[w] = True
                    work.append((w, 0))
                elif on[w]:
                    low[v] = min(low[v], index[w])
                continue
            work.pop()
            if work:
                u = work[-1][0]
                low[u] = min(low[u], low[v])
            if low[v] == index[v]:
                while True:
                    w = stack.pop()
                    on[w] = False
                    comp[w] = label
                    if w == v:
                        break
                label += 1
    return comp


def longest(nc, crow):
    """per component of a DAG with nc components and rows crow [(a, b)]: the most rows on a path ending at it"""
    succ, indeg = [[] for _ in range(nc)], [0] * nc
    for a, b in crow:
        succ[a].append(b)
        indeg[b] += 1
    order = [c for c in range(nc) if indeg[c] == 0]
    depth = [0] * nc
    for c in order:   # grows while it is read: a topological order
        for b in succ[c]:
            depth[b] = max(depth[b], depth[c] + 1)
            indeg[b] -= 1
            if indeg[b] == 0:
                order.append(b)
    assert len(order) == nc
    return depth


def traversable(rows, spec, min_value):
    if spec is None or len(rows) == 0:
        return np.ones(len(rows), dtype=bool)
    vk = metric_ref.order_key(metric_ref.values(rows, spec))
    return vk >= metric_ref.order_key(np.array([min_value]))[0]


def cycles(rows, spec=None, min_value=0.0, min_size=1):
    """(CYCLE_NODE records, row_index uint32, EDGE_OUT rows, info dict) of the components of an EDGE_OUT array"""
    rows = np.asarray(rows, dtype=abi.EDGE_OUT)
    n = len(rows)
    keys = node_ref.keys(rows)
    N = len(keys)
    fi = np.searchsorted(keys, group_ref.node_keys(rows["from_type"], rows["from"])).tolist()
    ti = np.searchsorted(keys, group_ref.node_keys(rows["to_type"], rows["to"])).tolist()
    trav = traversable(rows, spec, min_value).tolist()
    adj = [[] for _ in range(N)]
    for r in range(n):
        if trav[r] and fi[r] != ti[r]:
            adj[fi[r]].append(ti[r])
    label = tarjan(N, adj)
    # number the components by their smallest node index
    number, num = {}, [0] * N
    for v in range(N):
        if label[v] not in number:
            number[label[v]] = len(number)
        num[v] = number[label[v]]
    C = len(number)
    size = [0] * C
    for v in range(N):
        size[num[v]] += 1
    crow = [(num[fi[r]], num[ti[r]]) for r in range(n) if trav[r] and num[fi[r]] != num[ti[r]]]
    depth = longest(C, crow)
    height = longest(C, [(b, a) for a, b in crow])
    listed = sorted((v for v in range(N) if size[num[v]] >= min_size), key=lambda v: (num[v], v))
    rec = np.zeros(len(listed), dtype=abi.CYCLE_NODE)
    for j, v in enumerate(listed):
        k, c = int(keys[v]), num[v]
        rec[j] = (k >> 32, (0, 0, 0), k & 0xFFFFFFFF, v, c, size[c], depth[c], height[c])
    inside = [r for r in range(n) if trav[r] and fi[r] != ti[r] and num[fi[r]] == num[ti[r]]]
    row_index = np.array(sorted((r for r in inside if size[num[fi[r]]] >= min_size), key=lambda r: (num[fi[r]], r)),
                         dtype=np.uint32)
    cyclic = [c for c in range(C) if size[c] >= 2]
    info = dict(rows=n, traversable=int(sum(trav)), self_rows=sum(1 for r in range(n) if trav[r] and fi[r] == ti[r]),
                nodes=N, components=C, cyclic=len(cyclic), cyclic_nodes=sum(size[c] for c in cyclic),
                largest=max(size) if C else 0, cycle_rows=len(inside), depth=max(depth) if C else 0)
    return rec, row_index, rows[row_index], info


def group_cycles(rows, gmap=group_ref.EMPTY, **kw):
    """cycles over the group-edge rows of an EDGE_OUT array under a map"""
    return cycles(group_ref.group(rows, gmap)[0], **kw)
