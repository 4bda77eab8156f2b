"""Service graphs built edge by edge for the GNN tests. TEST INFRASTRUCTURE ONLY.

A graph is a list of edges between nodes `(kind, value)`; every edge carries its events as `(duration_ns, status)`
pairs. `Built(graph)` turns it into pod and service tables and `alz_l7_rec` records that produce exactly those edges
through the public ingest path (docs/SPEC.md §1, §9):

  pod -> pod, pod -> svc, pod -> outbound   plain HTTP from the source pod's address
  pod -> host-keyed outbound (kind 3)       HTTP with ALZ_PROTO_F_HOSTKEY, the node's id in daddr
  svc -> pod, outbound -> pod, and pod -> pod with rev=True
                                            AMQP DELIVER from the destination pod's address (reversed on ingest)

Every edge has a pod at one end, as every ingested row has. The GNN numbers its nodes in ascending
`(kind, value)` order, so a test that wants a degree at a node index picks the node's value accordingly (all-pod
graphs: pod id = node index).
"""
import ctypes as C

import numpy as np

import oracle_lib as ol
from alaz_b200 import abi, capi
from helpers import edges_equal, explain_diff

POD, SVC, OUT, HOST = abi.NODE_POD, abi.NODE_SVC, abi.NODE_OUTBOUND, abi.NODE_OUTBOUND_HOST
POD_NET, SVC_NET = 0x0A000001, 0xAC000001        # 10.0.0.1.., 172.0.0.1.. in order of first use
HOST_DADDR = abi.ip("192.0.2.1")                 # what the oracle sees for a host-keyed row (not in any table)


class Graph:
    """Edges as arrays (vectorised for graphs of a million edges)."""

    def __init__(self, ft, fv, tt, tv, ev_edge, ev_dur, ev_status, rev=None):
        self.ft, self.fv = np.asarray(ft, np.uint8), np.asarray(fv, np.uint64)
        self.tt, self.tv = np.asarray(tt, np.uint8), np.asarray(tv, np.uint64)
        n = len(self.ft)
        self.rev = np.zeros(n, bool) if rev is None else np.asarray(rev, bool)
        self.ev_edge = np.asarray(ev_edge, np.int64)
        self.ev_dur = np.asarray(ev_dur, np.uint64)
        self.ev_status = np.asarray(ev_status, np.uint16)

    @classmethod
    def from_list(cls, edges):
        """[(from_node, to_node, [(duration_ns, status), ...]), ...] or with a 4th item rev (pod -> pod only)."""
        ft, fv, tt, tv, rev, ee, ed, es = [], [], [], [], [], [], [], []
        for i, e in enumerate(edges):
            (a, x), (b, y), evs = e[0], e[1], e[2]
            ft.append(a); fv.append(x); tt.append(b); tv.append(y)
            rev.append(bool(e[3]) if len(e) > 3 else False)
            for d, s in evs:
                ee.append(i); ed.append(d); es.append(s)
        return cls(ft, fv, tt, tv, ee, ed, es, rev)

    @classmethod
    def uniform(cls, ft, fv, tt, tv, dur=2_000_000, status=200, count=1, rev=None):
        """Every edge gets `count` identical events."""
        n = len(ft)
        ee = np.repeat(np.arange(n), count)
        return cls(ft, fv, tt, tv, ee, np.full(len(ee), dur, np.uint64), np.full(len(ee), status, np.uint16), rev)

    @property
    def n_edges(self):
        return len(self.ft)


class Built:
    """Tables and records of a graph: `recs` go to the device, `orc_recs` + `host_idx` + `names` to the oracle."""

    def __init__(self, g):
        ft, fv, tt, tv = g.ft, g.fv, g.tt, g.tv
        assert np.all((ft == POD) | (tt == POD)), "every ingested row has a pod at one end"
        assert not np.any(ft == HOST), "host-keyed rows are never reversed"
        assert not np.any(g.rev & ((ft != POD) | (tt != POD))), "rev is for pod -> pod edges"
        pods = np.unique(np.concatenate([fv[ft == POD], tv[tt == POD]]))
        svcs = np.unique(np.concatenate([fv[ft == SVC], tv[tt == SVC]]))
        outs = np.unique(np.concatenate([fv[ft == OUT], tv[tt == OUT]]))
        hosts = np.unique(tv[tt == HOST])
        assert pods.size == 0 or pods.max() < (1 << 29)
        assert svcs.size == 0 or svcs.max() < (1 << 29)
        self.pod_id, self.pod_ip = pods, (POD_NET + np.arange(len(pods))).astype(np.uint64)
        self.svc_id, self.svc_ip = svcs, (SVC_NET + np.arange(len(svcs))).astype(np.uint64)
        assert len(pods) < (1 << 24) and len(svcs) < (1 << 24)
        table_ips = np.concatenate([self.pod_ip, self.svc_ip, [HOST_DADDR]])
        assert not np.isin(outs, table_ips).any(), "an outbound address collides with a table address"
        self.host_ids = hosts
        self.names = ["h%d.example" % int(x) for x in hosts]

        def addr(kind, val):
            out = val.copy()
            for k, ids, ips in ((POD, pods, self.pod_ip), (SVC, svcs, self.svc_ip)):
                m = kind == k
                out[m] = ips[np.searchsorted(ids, val[m])]
            return out                                    # outbound: the address itself; host: the id
        fa, ta = addr(ft, fv), addr(tt, tv)
        # the record: forward rows go from the source pod; reversed rows (AMQP DELIVER) from the destination pod
        reverse = (ft != POD) | g.rev
        e = g.ev_edge
        n = len(e)
        recs = np.zeros(n, dtype=abi.L7_REC)
        recs["saddr"] = np.where(reverse, ta, fa)[e]
        recs["daddr"] = np.where(reverse, fa, ta)[e]
        recs["sport"] = 40000 + (np.arange(n) % 20000)
        recs["dport"] = 80
        recs["status"] = g.ev_status
        recs["protocol"] = np.where(reverse, abi.PROTO_AMQP, abi.PROTO_HTTP)[e]
        recs["method_flags"] = np.where(reverse, abi.AMQP_DELIVER, 1)[e]
        recs["duration_ns"] = g.ev_dur
        recs["write_time_ns"] = np.arange(n)
        host = (tt == HOST)[e]
        self.orc_recs = recs.copy()
        self.host_idx = np.zeros(n, np.uint32)
        if host.any():
            self.host_idx[host] = 1 + np.searchsorted(hosts, tv[e][host])
            self.orc_recs["daddr"][host] = HOST_DADDR
            recs["protocol"][host] |= abi.PROTO_F_HOSTKEY
        self.recs = recs
        self.n_edges = g.n_edges

    def oracle_edges(self):
        o = ol.Oracle()
        for ips, ids, tab in ((self.pod_ip, self.pod_id, abi.TABLE_POD), (self.svc_ip, self.svc_id, abi.TABLE_SVC)):
            for ip, i in zip(ips.tolist(), ids.tolist()):
                o.upsert(tab, ip, i)
        o.process_hosts(self.orc_recs, self.host_idx, self.names)
        e = o.edges()
        o.close()
        host = e["to_type"] == HOST                       # the oracle numbers host nodes by their index in names
        e["to"][host] = self.host_ids[e["to"][host]]
        return e


def handle_for(b):
    """A handle with room for the graph: every table entry, and twice its edges in pairs and edges."""
    pairs = 1 << max(8, int(np.ceil(np.log2(2 * max(b.n_edges, 1)))))
    return capi.Handle(max_endpoints=len(b.pod_ip) + len(b.svc_ip) + 16, max_pairs=pairs)


def load(h, b):
    h.upsert_batch(abi.TABLE_POD, b.pod_ip.astype(np.uint32), b.pod_id.astype(np.uint32))
    h.upsert_batch(abi.TABLE_SVC, b.svc_ip.astype(np.uint32), b.svc_id.astype(np.uint32))
    h.commit()


def ingest(h, b, order=None, check=True):
    """Submit the graph's records (in `order`, default as built) and flush. check: the flushed edges must equal
    the oracle's on the same records, so that what a test finds after this is in the GNN."""
    recs = b.recs if order is None else b.recs[order]
    step = 1 << 21
    for i in range(0, len(recs), step):
        h.submit(recs[i:i + step])
    got = h.flush()
    assert len(got) == b.n_edges, (len(got), b.n_edges)
    if check:
        exp = b.oracle_edges()
        assert edges_equal(got, exp), explain_diff(got, exp)
    return got


def gnn(h, n_edges):
    """alz_gnn_score + alz_gnn_nodes: (scores, node keys, h2)."""
    scores = np.zeros(n_edges, dtype=np.float32)
    n = C.c_size_t(0)
    h._ck(h.L.alz_gnn_score(h.h, scores.ctypes.data_as(C.c_void_p), len(scores), C.byref(n)), "alz_gnn_score")
    assert n.value == n_edges
    keys = np.zeros(2 * n_edges, dtype=np.uint64)
    h2 = np.zeros((2 * n_edges, 64), dtype=np.float32)
    nv = C.c_size_t(0)
    h._ck(h.L.alz_gnn_nodes(h.h, keys.ctypes.data_as(C.c_void_p), h2.ctypes.data_as(C.c_void_p), len(keys),
                            C.byref(nv)), "alz_gnn_nodes")
    return scores, keys[: nv.value], h2[: nv.value]


def gnn_device(h, n_edges):
    """alz_gnn_score_device, its scores copied back."""
    p, n = C.c_void_p(), C.c_size_t(0)
    h._ck(h.L.alz_gnn_score_device(h.h, C.byref(p), C.byref(n)), "alz_gnn_score_device")
    assert n.value == n_edges
    h.sync()
    return h.d2h(p.value, n_edges, np.float32)
