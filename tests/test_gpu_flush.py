"""GPU: the single-rank window flush. The pair rows of a window are bucketed by the edge they resolve to and each
bucket is summed straight into its output row (emit_edges_kernel); a fold in the middle of the window (a table
commit) leaves sums in the edge accumulators, which the flush adds in. Every case is compared per edge, bit for bit,
against the oracle on the same records."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as ol
from alaz_b200 import abi, capi
from gnn_graphs import HOST, HOST_DADDR, POD_NET, SVC_NET
from helpers import edges_equal, explain_diff

pytestmark = pytest.mark.gpu

STATUSES = np.array([200, 201, 404, 500, 503, 599], np.uint16)


def records(saddr, daddr, rng, reversed_=None, host=None):
    """One record per (saddr, daddr) element: HTTP, or AMQP DELIVER where reversed_ (reversed on ingest), or
    Host-keyed HTTP where host (daddr is then the host id)."""
    n = len(saddr)
    rv = np.zeros(n, bool) if reversed_ is None else np.asarray(reversed_, bool)
    hk = np.zeros(n, bool) if host is None else np.asarray(host, bool)
    r = np.zeros(n, dtype=abi.L7_REC)
    r["saddr"], r["daddr"] = saddr, daddr
    r["sport"] = 40000 + (np.arange(n) % 20000)
    r["dport"] = 80
    r["status"] = np.where(rv, 0, STATUSES[rng.integers(0, len(STATUSES), n)])
    r["protocol"] = np.where(rv, abi.PROTO_AMQP, abi.PROTO_HTTP) | np.where(hk, abi.PROTO_F_HOSTKEY, 0)
    r["method_flags"] = np.where(rv, abi.AMQP_DELIVER, 1)
    r["duration_ns"] = np.where(rng.random(n) < 0.5, rng.integers(0, 1 << 20, n), rng.integers(0, 1 << 42, n))
    r["write_time_ns"] = np.arange(n)
    return r


def oracle_edges(tables, recs, host_ids=()):
    """The oracle on the same tables and records. Host-keyed rows reach it as they reach the reference: daddr the
    host's placeholder address, the header text in names (tests/gnn_graphs.py)."""
    host_ids = np.asarray(sorted(host_ids), np.uint64)
    orc = recs.copy()
    hk = (recs["protocol"] & abi.PROTO_F_HOSTKEY) != 0
    orc["protocol"] &= ~np.uint8(abi.PROTO_F_HOSTKEY)
    host_idx = np.zeros(len(recs), np.uint32)
    host_idx[hk] = 1 + np.searchsorted(host_ids, recs["daddr"][hk])
    orc["daddr"][hk] = HOST_DADDR
    o = ol.Oracle()
    for tab, ips, ids in tables:
        for ip, i in zip(np.asarray(ips).tolist(), np.asarray(ids).tolist()):
            o.upsert(tab, ip, i)
    o.process_hosts(orc, host_idx, ["h%d.example" % int(x) for x in host_ids])
    e = o.edges()
    o.close()
    m = e["to_type"] == HOST
    e["to"][m] = host_ids[e["to"][m]]
    return e


def flush_raw(h, cap):
    """alz_window_flush with the status instead of an exception: (status, rows, n_out)."""
    out = np.zeros(max(cap, 1), dtype=abi.EDGE_OUT)
    n = C.c_size_t(0)
    rc = h.L.alz_window_flush(h.h, out.ctypes.data_as(C.c_void_p), cap, C.byref(n))
    return rc, out[: min(n.value, cap)].copy(), n.value


def flush_device_raw(h):
    """alz_window_flush_device, the rows copied back: (status, rows)."""
    p, n = C.c_void_p(), C.c_size_t(0)
    rc = h.L.alz_window_flush_device(h.h, C.byref(p), C.byref(n))
    rows = h.d2h(p.value, n.value, abi.EDGE_OUT) if n.value else np.zeros(0, dtype=abi.EDGE_OUT)
    return rc, rows


def flush(h, path):
    if path == "host":
        return h.flush()
    rc, rows = flush_device_raw(h)
    assert rc == abi.OK, rc
    return rows


@pytest.mark.parametrize("k", [1, 2, 9, 10_000])
def test_edge_fed_by_k_pair_rows(k):
    """Four edges, three of them fed by k distinct pair rows each: pod -> service over k (pod address, service
    address) pairs of one pod id and one service id; pod -> pod over forward rows and the reversed rows of the other
    side; pod -> Host-keyed outbound from k addresses of one pod. Plus a one-row outbound edge."""
    rng = np.random.default_rng(k)
    m = {1: 1, 2: 2, 9: 3, 10_000: 100}[k]
    n = k // m
    P, S, A, B, H = 7, 3, 11, 12, 20
    p_ip = POD_NET + np.arange(m, dtype=np.uint64)
    s_ip = SVC_NET + np.arange(n, dtype=np.uint64)
    a_ip = POD_NET + 20_000 + np.arange(m, dtype=np.uint64)
    b_ip = POD_NET + 40_000 + np.arange(n, dtype=np.uint64)
    h_ip = POD_NET + 60_000 + np.arange(k, dtype=np.uint64)
    host_id, out_ip = 5, abi.ip("8.8.4.4")
    tables = [(abi.TABLE_POD, p_ip, np.full(m, P)), (abi.TABLE_SVC, s_ip, np.full(n, S)),
              (abi.TABLE_POD, a_ip, np.full(m, A)), (abi.TABLE_POD, b_ip, np.full(n, B)),
              (abi.TABLE_POD, h_ip, np.full(k, H))]
    gi, gj = (x.ravel() for x in np.meshgrid(np.arange(m), np.arange(n), indexing="ij"))
    ev = lambda x: np.repeat(x, 3)   # three events per pair row
    rev = (np.arange(k) % 2 == 1) if k > 1 else np.zeros(1, bool)   # pod <-> pod: every second row from B's side
    parts = [records(ev(p_ip[gi]), ev(s_ip[gj]), rng),
             records(ev(np.where(rev, b_ip[gj], a_ip[gi])), ev(np.where(rev, a_ip[gi], b_ip[gj])), rng,
                     reversed_=ev(rev)),
             records(ev(h_ip), np.full(3 * k, host_id, np.uint64), rng, host=np.ones(3 * k, bool)),
             records(np.full(4, p_ip[0]), np.full(4, out_ip), rng)]
    recs = np.concatenate(parts)
    recs = recs[rng.permutation(len(recs))]
    h = capi.Handle(max_endpoints=1 << 16, max_pairs=1 << 16)
    for tab, ips, ids in tables:
        h.upsert_batch(tab, ips.astype(np.uint32), ids.astype(np.uint32))
    h.commit()
    h.submit(recs)
    got = h.flush()
    exp = oracle_edges(tables, recs, [host_id])
    assert len(exp) == 4
    assert edges_equal(got, exp), explain_diff(got, exp)
    assert sorted(got["count"].tolist()) == sorted([3 * k, 3 * k, 3 * k, 4])
    h.close()


def topo_handle(t, **kw):
    h = capi.Handle(max_endpoints=4 * 4096, **kw)
    h.load_tables(t.pod_ip, t.svc_ip)
    o = ol.Oracle()
    o.load_tables(t.pod_ip, t.svc_ip)
    return h, o


def churn(h, o, t, rng, n=20):
    for k in rng.integers(0, len(t.pod_ip), n):
        h.erase(abi.TABLE_POD, int(t.pod_ip[k])); o.erase(abi.TABLE_POD, int(t.pod_ip[k]))
    for k in rng.integers(0, len(t.pod_ip), n):
        h.upsert(abi.TABLE_POD, int(t.pod_ip[k]), int(k) + 1); o.upsert(abi.TABLE_POD, int(t.pod_ip[k]), int(k) + 1)
    h.commit()


def check_stats(h, o):
    st, ost = h.stats(), o.stats()
    for key in ("events_in", "rows_emitted", "not_request", "src_unresolved"):
        assert st[key] == ost[key], (key, st[key], ost[key])


@pytest.mark.parametrize("path", ["host", "device"])
def test_table_commit_mid_window(path):
    """A commit folds the window so far into the edge accumulators; the flush adds the pair rows of the rest."""
    t = ol.Topo(1200, seed=31, mix=abi.MIX_ALL)
    h, o = topo_handle(t, max_pairs=1 << 16)
    rng = np.random.default_rng(31)
    ev = t.events(0, 600_000)
    cuts = [0, 150_000, 400_000, len(ev)]
    for c0, c1 in zip(cuts, cuts[1:]):
        if c0:
            churn(h, o, t, rng)
        h.submit(ev[c0:c1]); o.process(ev[c0:c1])
    got, exp = flush(h, path), o.edges()
    assert edges_equal(got, exp), explain_diff(got, exp)
    check_stats(h, o)
    # the next window starts from clean accumulators
    o.reset_window()
    ev2 = t.events(600_000, 200_000)
    h.submit(ev2); o.process(ev2)
    got, exp = flush(h, path), o.edges()
    assert edges_equal(got, exp), explain_diff(got, exp)
    h.close(); o.close()


@pytest.mark.parametrize("flags", [0, abi.CFG_NO_SMEM_CACHE])
def test_source_stops_being_a_pod(flags):
    """Rows of a source that leaves the pod table mid-window: those before the commit keep their edge, those after
    are unresolved. The pair key equal to the dictionaries' free marker (255.255.255.255 both ways) has a fixed row
    that is taken without the admission test, so its events reach the flush and are counted unresolved there."""
    rng = np.random.default_rng(3)
    x_ip, y_ip, s_ip = POD_NET, POD_NET + 1, SVC_NET
    tables = [(abi.TABLE_POD, [x_ip, y_ip], [1, 2]), (abi.TABLE_SVC, [s_ip], [9])]
    h = capi.Handle(max_endpoints=64, max_pairs=1024, flags=flags)
    o = ol.Oracle()
    for tab, ips, ids in tables:
        for ip, i in zip(ips, ids):
            h.upsert(tab, ip, i); o.upsert(tab, ip, i)
    h.commit()
    before = np.concatenate([records(np.full(50, x_ip), np.full(50, s_ip), rng),
                             records(np.full(30, y_ip), np.full(30, x_ip), rng)])
    h.submit(before); o.process(before)
    h.erase(abi.TABLE_POD, x_ip); o.erase(abi.TABLE_POD, x_ip)
    h.commit()
    after = np.concatenate([records(np.full(40, x_ip), np.full(40, s_ip), rng),
                            records(np.full(20, y_ip), np.full(20, x_ip), rng),
                            records(np.full(25, 0xFFFFFFFF), np.full(25, 0xFFFFFFFF), rng)])
    after = after[rng.permutation(len(after))]
    h.submit(after); o.process(after)
    got, exp = h.flush(), o.edges()
    assert edges_equal(got, exp), explain_diff(got, exp)
    check_stats(h, o)
    assert h.stats()["src_unresolved"] >= 65
    h.close(); o.close()


@pytest.mark.parametrize("path", ["host", "device"])
def test_window_over_max_edges(path):
    """More edges than max_edges: the flush returns ALZ_E_CAPACITY with max_edges rows, each exact; the events of
    the edges left out are counted lost; the next window is exact and holds nothing of this one."""
    t = ol.Topo(500, seed=8)
    ev = t.events(0, 300_000)
    h, o = topo_handle(t, max_pairs=1 << 15, max_edges=64)
    h.submit(ev); o.process(ev)
    if path == "host":
        rc, got, n = flush_raw(h, 64)
        assert n == 64
    else:
        rc, got = flush_device_raw(h)
    assert rc == abi.E_CAPACITY
    assert len(got) == 64
    exp = {(int(e["from_type"]), int(e["from"]), int(e["to_type"]), int(e["to"])): e.tobytes() for e in o.edges()}
    assert len(exp) > 64
    for e in got:
        assert exp[(int(e["from_type"]), int(e["from"]), int(e["to_type"]), int(e["to"]))] == e.tobytes()
    st = h.stats()
    assert st["capacity_events"] > 0
    assert int(got["count"].sum()) == st["rows_emitted"] == o.stats()["rows_emitted"] - st["capacity_events"]
    o.reset_window()
    small = ev[ev["saddr"] == ev["saddr"][0]][:2000]
    h.submit(small); o.process(small)
    got, exp = flush(h, path), o.edges()
    assert 0 < len(got) <= 64
    assert edges_equal(got, exp), explain_diff(got, exp)
    h.close(); o.close()


def test_too_small_buffer_keeps_the_window():
    """alz_window_flush into a buffer one row short returns ALZ_E_CAPACITY and the row count; the window stays, and
    the next flush returns it whole, including what a commit had folded before."""
    t = ol.Topo(800, seed=12, mix=abi.MIX_ALL)
    h, o = topo_handle(t, max_pairs=1 << 16)
    rng = np.random.default_rng(12)
    ev = t.events(0, 300_000)
    h.submit(ev[:100_000]); o.process(ev[:100_000])
    churn(h, o, t, rng)
    h.submit(ev[100_000:]); o.process(ev[100_000:])
    exp = o.edges()
    rc, _, n = flush_raw(h, len(exp) - 1)
    assert rc == abi.E_CAPACITY and n == len(exp)
    got = h.flush()
    assert edges_equal(got, exp), explain_diff(got, exp)
    check_stats(h, o)
    h.close(); o.close()


def test_consecutive_windows_leave_nothing_behind():
    """Three windows over disjoint events: each flush equals the oracle of its own events only."""
    t = ol.Topo(1500, seed=77, mix=abi.MIX_ALL)
    h, o = topo_handle(t, max_pairs=1 << 16)
    for w in range(3):
        ev = t.events(w * 500_000, 500_000)
        h.submit(ev); o.process(ev)
        got, exp = h.flush(), o.edges()
        assert edges_equal(got, exp), f"window {w}: " + explain_diff(got, exp)
        o.reset_window()
    check_stats(h, o)
    h.close(); o.close()


def test_host_and_device_flush_return_identical_bytes():
    """alz_window_flush and alz_window_flush_device on the same records give the same rows in the same order, byte
    for byte, for a plain window and for one with a commit in the middle."""
    t = ol.Topo(1000, seed=5, mix=abi.MIX_ALL)
    hs = [topo_handle(t, max_pairs=1 << 16)[0] for _ in range(2)]
    for w in range(2):
        ev = t.events(w * 400_000, 400_000)
        for h in hs:
            h.submit(ev[:200_000])
            if w == 1:
                h.upsert(abi.TABLE_POD, int(t.pod_ip[3]), 4242)
                h.commit()
            h.submit(ev[200_000:])
        a, b = hs[0].flush(), flush(hs[1], "device")
        assert len(a) > 0
        assert a.tobytes() == b.tobytes(), f"window {w}"
    for h in hs:
        h.close()
