"""GPU: consecutive single-rank windows on one handle. A flush empties the dictionaries from the slots the window
claimed (or, when that log overflowed, the whole capacity) and sorts the edge keys by a counting sort on the key's
high word and a sort of each (rev, type, pod) segment. Every window is compared with the oracle and with a fresh
handle given the same tables and records, so a key left behind by an earlier window shows up as a difference, and
its rows are checked to be in strictly increasing key order."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as ol
from alaz_b200 import abi, capi
from gnn_graphs import POD_NET, SVC_NET
from helpers import edges_equal, explain_diff
from test_gpu_flush import oracle_edges, records

pytestmark = pytest.mark.gpu

OUT_NET = 0x08000000   # 8.0.0.0.. : in no table, outbound


def assert_key_order(rows):
    """The rows' packed edge keys (make_edge_key: rev | other type | pod id | other end) strictly increase."""
    ft, tt = rows["from_type"].astype(np.uint64), rows["to_type"].astype(np.uint64)
    f, t = rows["from"].astype(np.uint64), rows["to"].astype(np.uint64)
    pod_from = ft == abi.NODE_POD
    keys = np.where(pod_from, (tt << np.uint64(61)) | (f << np.uint64(32)) | t,
                    (np.uint64(1) << np.uint64(63)) | (ft << np.uint64(61)) | (t << np.uint64(32)) | f)
    assert np.all(keys[1:] > keys[:-1]), "rows out of key order"


class Windows:
    """One long-lived handle and its configuration; the table state is replayed on a fresh handle per window."""

    def __init__(self, **cfg):
        self.cfg = cfg
        self.h = capi.Handle(**cfg)
        self.tables = {}   # (table, ip) -> id

    def upsert(self, h, rows):
        for tab, ip, i in rows:
            h.upsert(tab, int(ip), int(i))
        h.commit()

    def put(self, rows):
        self.upsert(self.h, rows)
        for tab, ip, i in rows:
            self.tables[(tab, int(ip))] = int(i)

    def table_list(self):
        return [(tab, [ip], [i]) for (tab, ip), i in self.tables.items()]

    def flush(self, h):
        out = np.zeros(self.cfg.get("max_edges", self.cfg["max_pairs"]), dtype=abi.EDGE_OUT)
        n = C.c_size_t(0)
        rc = h.L.alz_window_flush(h.h, out.ctypes.data_as(C.c_void_p), len(out), C.byref(n))
        return rc, out[: n.value].copy()

    def window(self, parts, host_ids=(), exact=True):
        """parts: [(table rows to put before, records)]. Returns the long-lived handle's (status, rows) after checking
        them against the oracle and a fresh handle (exact) or only returning them (a window that loses events)."""
        start = dict(self.tables)
        fresh = capi.Handle(**self.cfg)
        self.upsert(fresh, [(tab, ip, i) for (tab, ip), i in start.items()])
        for put, recs in parts:
            if put:
                self.put(put)
                self.upsert(fresh, put)
            self.h.submit(recs)
            fresh.submit(recs)
        rc, got = self.flush(self.h)
        rc_f, got_f = self.flush(fresh)
        fresh.close()
        assert_key_order(got)
        if not exact:
            return rc, got
        assert rc == rc_f == abi.OK, (rc, rc_f)
        assert got.tobytes() == got_f.tobytes()
        recs = np.concatenate([r for _, r in parts]) if parts else np.zeros(0, dtype=abi.L7_REC)
        if len(parts) > 1 and any(p for p, _ in parts[1:]):
            exp = self.oracle_parts(start, parts)
        else:
            exp = oracle_edges(self.table_list(), recs, host_ids)
        assert edges_equal(got, exp), explain_diff(got, exp)
        return rc, got

    def oracle_parts(self, start, parts):
        o = ol.Oracle()
        for (tab, ip), i in start.items():
            o.upsert(tab, ip, i)
        for put, recs in parts:
            for tab, ip, i in put:
                o.upsert(tab, int(ip), int(i))
            o.process(recs)
        e = o.edges()
        o.close()
        return e

    def close(self):
        self.h.close()


def pods(first, n, id0):
    return [(abi.TABLE_POD, POD_NET + first + k, id0 + k) for k in range(n)]


def svcs(first, n, id0):
    return [(abi.TABLE_SVC, SVC_NET + first + k, id0 + k) for k in range(n)]


def mixed(rng, n_pods, n_svcs, n, pod_first=0, svc_first=0):
    """n records from pods [pod_first, +n_pods) to services, other pods and outbound addresses."""
    src = POD_NET + pod_first + rng.integers(0, n_pods, n)
    kind = rng.integers(0, 3, n)
    dst = np.where(kind == 0, SVC_NET + svc_first + rng.integers(0, n_svcs, n),
                   np.where(kind == 1, POD_NET + pod_first + rng.integers(0, n_pods, n), OUT_NET + rng.integers(0, 20, n)))
    return records(src.astype(np.uint64), dst.astype(np.uint64), rng)


def test_small_tables_window_sequence():
    """max_pairs 1024: a window that takes more pairs than that (events lost, the claimed-slot log overflows and the
    flush clears whole dictionaries), then windows with unresolvable sources, host-keyed and reversed-only pairs, a
    table commit in the middle, an empty window; each exact and equal to a fresh handle."""
    rng = np.random.default_rng(5)
    w = Windows(max_endpoints=4096, max_pairs=1 << 10)
    w.put(pods(0, 200, 0) + svcs(0, 50, 0))
    w.window([([], mixed(rng, 200, 50, 600))])
    # pair-table capacity: 4000 distinct outbound pairs against 1024 rows
    loss = records((POD_NET + rng.integers(0, 200, 4000)).astype(np.uint64), (OUT_NET + 10_000 + np.arange(4000)).astype(np.uint64), rng)
    rc, got = w.window([([], loss)], exact=False)
    assert rc == abi.E_CAPACITY and len(got) > 0
    # unresolvable sources, host-keyed pairs, pod <-> pod pairs seen only reversed
    unres = records((POD_NET + 5000 + rng.integers(0, 50, 500)).astype(np.uint64), (SVC_NET + rng.integers(0, 50, 500)).astype(np.uint64), rng)
    host = records((POD_NET + rng.integers(0, 200, 200)).astype(np.uint64), rng.integers(1, 30, 200).astype(np.uint64), rng,
                   host=np.ones(200, bool))
    rev = records((POD_NET + rng.integers(0, 100, 300)).astype(np.uint64), (POD_NET + 100 + rng.integers(0, 100, 300)).astype(np.uint64),
                  rng, reversed_=np.ones(300, bool))
    parts = np.concatenate([unres, host, rev, mixed(rng, 200, 50, 300)])
    w.window([([], parts[rng.permutation(len(parts))])], host_ids=range(1, 30))
    # a table commit in the middle of the window folds the first half into the edge table
    w.window([([], mixed(rng, 200, 50, 500)), (pods(200, 40, 200) + svcs(50, 10, 50), mixed(rng, 240, 60, 500))])
    w.window([])
    w.window([([], mixed(rng, 240, 60, 600))])
    w.close()


def test_hub_segments_window_sequence():
    """A pod with 70,000 outbound edges (18 sorted chunks, five merge passes), pods with 5,000 and 300 (one chunk),
    pod ids at and past max_endpoints (the shared last segment), reversed pod <-> pod rows; then an ordinary window
    and one with hubs that need four and two merge passes."""
    rng = np.random.default_rng(11)
    w = Windows(max_endpoints=1024, max_pairs=1 << 18)
    big_ids = [(abi.TABLE_POD, POD_NET + 900 + k, i) for k, i in enumerate([1023, 1024, 5000, (1 << 29) - 1])]
    w.put(pods(0, 100, 0) + svcs(0, 20, 0) + big_ids)
    hub = records(np.full(70_000, POD_NET + 7, np.uint64), (OUT_NET + rng.permutation(1 << 20)[:70_000]).astype(np.uint64), rng)
    mid = records(np.full(5000, POD_NET + 8, np.uint64), (OUT_NET + rng.permutation(1 << 16)[:5000]).astype(np.uint64), rng)
    small = records(np.full(300, POD_NET + 9, np.uint64), (OUT_NET + rng.permutation(4096)[:300]).astype(np.uint64), rng)
    big_src = POD_NET + 900 + rng.integers(0, 4, 3000)
    big = records(big_src.astype(np.uint64), (OUT_NET + rng.integers(0, 2000, 3000)).astype(np.uint64), rng)
    big_rev = records(big_src[:500].astype(np.uint64), (POD_NET + rng.integers(0, 100, 500)).astype(np.uint64), rng,
                      reversed_=np.ones(500, bool))
    recs = np.concatenate([hub, mid, small, big, big_rev, mixed(rng, 100, 20, 20_000)])
    _, got = w.window([([], recs[rng.permutation(len(recs))])])
    assert len(got) > 75_000
    w.window([([], mixed(rng, 100, 20, 20_000))])
    # 10 chunks (four merge passes) and 3 chunks (two passes, then copied along)
    other = records(np.full(9000, POD_NET + 10, np.uint64), (OUT_NET + rng.permutation(1 << 16)[:9000]).astype(np.uint64), rng)
    w.window([([], np.concatenate([hub[:40_000], other, mixed(rng, 100, 20, 5000)]))])
    w.close()
