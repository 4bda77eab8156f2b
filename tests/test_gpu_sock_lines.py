"""GPU: socket timelines (alz_sock.cu) on constructed lines against the C restatement (ol.SockMaps). Every lookup is
compared byte for byte, every alive export sorted, every joined window per edge, and after every sync the socket stats
against the bookkeeping model of tests/sock_lines.py, which says whether the index was rebuilt, a segment moved or the
pool was re-laid."""
import ctypes as C
import time

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings, strategies as st

import oracle_lib as ol
import sock_lines as sl
from alaz_b200 import abi
from helpers import edges_equal, explain_diff
from sock_lines import K, K2, K3, M64, MINUTE, Both, closed, opened, query, sock

pytestmark = pytest.mark.gpu

PODS = [abi.ip(f"10.0.0.{k}") for k in range(1, 9)]          # pod ids 1..8
SVCS = [abi.ip(f"172.16.0.{k}") for k in range(1, 4)]        # service ids 11..13
STRANGER = abi.ip("10.0.9.1")


def _get(b, key, ts, now):
    r = b.lookup(query(key[0], key[1], ts), now)[0]
    return sl.found_k(r["saddr"]) if r["found"] else None


def run_script(b, ops):
    out = []
    for op in ops:
        if op[0] in ("o", "c"):
            b.tcp(sl.script_rec(op))
        elif op[0] == "get":
            out.append(_get(b, *op[1:]))
        else:
            b.gc()
            out.append(b.o.records())
    return out


def lines_of(key, n, t0=1000, dt=1000, k0=0):
    """n values on one line: open, close, open, ... at t0, t0 + dt, ...; the j-th value's socket is k0 + j mod 20000."""
    j = np.arange(n)
    return sl.tcp_rec(key[0], key[1], t0 + j * dt, np.where(j % 2 == 0, 1, 5), saddr=sl.BASE + k0 + j % 20000,
                      daddr=sl.DST, sport=40000 + j % 20000, dport=80)


def grid(*ts):
    return sorted({max(0, min(M64, t + d)) for t in ts for d in (-1, 0, 1)})


# ---- 1. index probes ------------------------------------------------------------------------------------------------

def test_64_lines_with_one_home_slot_and_absent_keys_past_the_chain():
    mask = sl.index_cap_for(64) - 1
    keys = sl.keys_with_home(mask, 300, 70)
    b = Both()
    for i, k in enumerate(keys[:64]):
        b.tcp(np.concatenate([opened(*k, 100, **sock(i)), closed(*k, 200), opened(*k, 300, **sock(100 + i))]))
    got = b.sweep(keys, [50, 150, 250, 350], now=1)                  # the last six are absent: the probe crosses 64
    assert b.m.index_cap == mask + 1
    f = got.reshape(70, 4)
    assert [sl.found_k(s) for s in f["saddr"][:64, 1]] == list(range(64))
    assert [sl.found_k(s) for s in f["saddr"][:64, 3]] == list(range(100, 164))
    assert not f["found"][64:].any()
    b.close()


def test_chain_that_wraps_past_the_end_of_the_index():
    mask = sl.index_cap_for(6) - 1
    keys = sl.wrap_chain(mask, 5)                                     # homes mask-1 (x5) and 0: slots mask-1..3
    absent = sl.keys_with_home(mask, mask - 1, 8, pid=777)[5:] + sl.keys_with_home(mask, 0, 3, pid=778)[1:]
    b = Both()
    for i, k in enumerate(keys):
        b.tcp(opened(*k, 100, **sock(i)))
    got = b.sweep(keys + absent, [0, 100, 101], now=1)
    assert b.m.index_cap == mask + 1
    f = got.reshape(-1, 3)
    assert [sl.found_k(s) for s in f["saddr"][:6, 0]] == list(range(6)) and not f["found"][6:].any()
    b.close()


def test_keys_that_alias_in_the_hash_input():
    (a, a2), (_, a3) = sl.alias_pairs()
    b = Both()
    for i, k in enumerate((a, a2, a3)):
        b.tcp(opened(*k, 100, **sock(i)))
    b.tcp(closed(*a2, 200))
    got = b.sweep([a, a2, a3, (a[0] + (2 << 24), a[1])], [150, 100 + MINUTE + 1], now=1)
    assert [sl.found_k(s) if f else None for s, f in zip(got["saddr"], got["found"])] == [0, 0, 1, None, 2, 2,
                                                                                           None, None]
    b.close()


def test_lines_added_one_sync_at_a_time_across_two_rebuilds():
    """Lines 1..40 arrive one per sync: the index is rebuilt at 1, 9 and 33 lines (16, 64, 256 slots). Line 9 has 30000
    values, which do not fit the first pool: the second rebuild comes with a repool."""
    b = Both()
    keys = [(5000 + i, 3) for i in range(40)]
    cap = 0
    for i, k in enumerate(keys):
        b.tcp(lines_of(k, 30000 if i == 8 else 3, k0=i))
        b.sweep(keys[:i + 1] + [(9999, 9)], [500, 1500, 2500, 3500], now=1)
        cap = sl.index_cap_for(i + 1, cap)
        assert b.m.index_cap == cap
    assert b.m.rebuilds == 3 and b.m.rebuild_with_repool == 2
    assert b.h.sock_stats()["repools"] == 2
    b.close()


# ---- 2. segments and pool -------------------------------------------------------------------------------------------

def test_inserts_at_the_start_the_middle_and_the_end():
    b = Both()
    b.tcp(lines_of(K, 10))
    ts = grid(*range(0, 12000, 500), 5, 1450, 99999)
    b.sweep([K], ts, now=1)
    for t, k in ((5, 50), (1450, 51), (99999, 52)):
        b.tcp(opened(*K, t, **sock(k)))
        b.sweep([K], ts, now=1)
    b.tcp(np.concatenate([opened(*K, 3, **sock(60)), closed(*K, 1460), opened(*K, 10**6, **sock(61))]))
    b.sweep([K], ts + [10**6 + 1], now=1)
    b.close()


def test_4096_out_of_order_inserts_into_one_line():
    """One sync applies 4096 inserts at random positions of a line of 4096 values: one warp shifts the tail 4096 times."""
    rng = np.random.default_rng(1)
    b = Both()
    b.tcp(lines_of(K, 4096, t0=0, dt=1000))
    b.sweep([K], [5], now=1)
    ts = rng.integers(0, 4096 * 1000, 4096)
    b.tcp(sl.tcp_rec(K[0], K[1], ts, 1, saddr=sl.BASE + 5000 + np.arange(4096), daddr=sl.DST,
                     sport=45000 + np.arange(4096), dport=80))
    t0 = time.perf_counter()
    b.sweep([(9999, 9)], [1], now=1)                                  # the sync, and nothing else
    dt = time.perf_counter() - t0
    print(f"sync of 4096 out-of-order inserts into one line of 4096 values: {dt * 1e3:.1f} ms")
    b.lookup(query(K[0], K[1], rng.integers(0, 4096 * 1000 + 5000, 20000)), now=1)
    b.close()


def test_lines_that_cross_16_32_and_64_records_in_one_sync():
    b = Both()
    keys = [K, K2, K3]
    for k, n in zip(keys, (10, 20, 40)):
        b.tcp(lines_of(k, n, dt=100, k0=100 * k[0]))
    b.sweep(keys, [0], now=1)
    assert b.m.garbage == 0
    for k, n, add in zip(keys, (10, 20, 40), (7, 14, 30)):
        b.tcp(sl.tcp_rec(k[0], k[1], 1050 + 200 * np.arange(add), 1, saddr=sl.BASE + 50 + np.arange(add), daddr=sl.DST,
                         sport=41000 + np.arange(add), dport=80))
    b.sweep(keys, grid(*range(900, 10000, 50)), now=1)
    assert b.m.garbage == 16 + 32 + 64 and b.m.repools == 1
    b.close()


def test_pool_garbage_past_2_16_then_a_full_pool_re_lays():
    """66 lines of 1000 values (2048-record segments, a pool of 270336): 33 of them grow past 2048 in one sync and move,
    which fills the pool exactly and leaves 67584 records of garbage; one more move re-lays the pool."""
    b = Both()
    keys = [(7000 + i, 4) for i in range(66)]
    b.tcp(np.concatenate([lines_of(k, 1000, k0=i) for i, k in enumerate(keys)]))
    b.sweep(keys, [500], now=1)
    for k in keys[:33]:
        b.tcp(lines_of(k, 1100, t0=10**7))
    b.sweep(keys, [1500, 10**7 + 5], now=1)
    st_ = b.h.sock_stats()
    assert st_["pool_garbage"] == 33 * 2048 > 1 << 16 and st_["repools"] == 1
    b.tcp(lines_of(keys[40], 1100, t0=10**7))
    b.sweep(keys, [1500, 10**7 + 5, 10**7 + 10**6], now=1)
    st_ = b.h.sock_stats()
    assert st_["pool_garbage"] == 0 and st_["repools"] == 2 and b.m.garbage_repools == 0
    b.close()


def test_line_emptied_by_gc_grows_past_its_segment():
    b = Both()
    ops, exp = sl.BOUNDARY["emptied_and_regrown"]
    assert run_script(b, ops) == exp
    b.tcp(lines_of(K, 40, t0=10**6))
    b.sweep([K], grid(5, 50, *range(10**6, 10**6 + 41000, 1000)), now=1)
    assert b.m.garbage == 16
    b.close()


# ---- 3. LastMatch follows its record ---------------------------------------------------------------------------------

@pytest.mark.parametrize("d", [0, 1])
def test_last_match_follows_its_record_through_shifts_moves_and_a_repool(d):
    """o1000 is stamped T and o3000 T + 5 min + d. Then 15 opens are inserted before them (shifts, then a move), and a
    30000-value line forces a repool. The GC keeps the pair (o1000, c2000) iff d = 0."""
    T = 20 * MINUTE
    b = Both()
    b.tcp(np.concatenate([opened(*K, 1000, **sock(1)), closed(*K, 2000), opened(*K, 3000, **sock(2)),
                          closed(*K, 4000)]))
    assert _get(b, K, 1500, T) == 1
    assert _get(b, K, 3500, T + 5 * MINUTE + d) == 2
    for t in range(5, 0, -1):                                        # shifts: each at position 0
        b.tcp(opened(*K, t, **sock(10 + t)))
    b.sweep([(9999, 9)], [1], now=1)
    assert b.m.garbage == 0
    for t in range(15, 5, -1):                                       # position 5, and the line outgrows 16
        b.tcp(opened(*K, t, **sock(10 + t)))
    b.sweep([(9999, 9)], [1], now=1)
    assert b.m.garbage == 16
    b.tcp(lines_of(K2, 30000, k0=100))
    b.sweep([(9999, 9)], [1], now=1)
    assert b.h.sock_stats()["repools"] == 2
    b.gc()
    assert b.o.lines()[K] == 10 - 2 * d
    b.sweep([K], grid(0, 3, 8, 14, 15, 999, 1000, 1500, 2000, 3000, 4000, 5000), now=1)
    b.close()


# ---- 4 and 5. GetValue and DeleteUnused boundaries --------------------------------------------------------------------

@pytest.mark.parametrize("name", sorted(sl.BOUNDARY))
def test_boundary_lines(name):
    ops, expected = sl.BOUNDARY[name]
    b = Both()
    assert run_script(b, ops) == expected
    keys = sorted({op[1] for op in ops if op[0] != "gc"})
    ts = grid(*{op[2] for op in ops if op[0] != "gc"}, MINUTE, 10**6 + MINUTE)
    b.sweep(keys, ts, now=1)
    b.gc()
    b.sweep(keys, ts, now=2)
    b.close()


# ---- 6. alive export ----------------------------------------------------------------------------------------------------

def test_alive_export_tables_and_capacity():
    BOTH = PODS[7]
    b = Both()
    for k, ip in enumerate(PODS):
        b.upsert(abi.TABLE_POD, ip, k + 1)
    for k, ip in enumerate(SVCS):
        b.upsert(abi.TABLE_SVC, ip, k + 11)
    b.upsert(abi.TABLE_SVC, BOTH, 19)                                   # pod 8 is a service too
    b.commit()
    lines = [((1, 1), BOTH, PODS[1]),            # source both pod and service: a row from pod 8
             ((1, 2), PODS[0], BOTH),            # destination both: the service wins
             ((1, 3), PODS[2], abi.ip("8.8.8.8")),   # outbound
             ((1, 4), STRANGER, PODS[0]),        # source no pod (yet)
             ((1, 5), PODS[3], SVCS[0]),         # its pod is erased later
             ((1, 6), PODS[4], PODS[5])]
    for i, (k, s, dd) in enumerate(lines):
        b.tcp(opened(*k, 100, saddr=s, daddr=dd, sport=30000 + i, dport=80))
    b.tcp(opened(2, 1, 100, saddr=PODS[0], daddr=SVCS[1]))                # last value a close: no row
    b.tcp(closed(2, 1, 200))
    b.tcp(opened(2, 2, 10, saddr=PODS[1], daddr=SVCS[2]))               # emptied by the GC below
    b.tcp(closed(2, 2, 20))
    assert len(b.alive()) == 5
    b.lookup(query(2, 2, 25), now=10 * MINUTE)
    b.tcp(closed(2, 2, 30))
    b.gc()                                               # (2, 1) loses its last value, the close: it ends open again
    assert b.o.lines()[(2, 2)] == 0 and b.o.lines()[(2, 1)] == 1
    assert len(b.alive()) == 6
    b.erase(abi.TABLE_POD, PODS[3])
    b.commit()
    b.upsert(abi.TABLE_POD, STRANGER, 40)                               # staged only: the device uses committed tables
    assert len(b.alive()) == 5
    b.commit()
    rows = b.alive()
    assert len(rows) == 6
    assert {int(r["to_type"]) for r in rows} == {abi.NODE_POD, abi.NODE_SVC, abi.NODE_OUTBOUND}
    assert len(b.alive(cap=6)) == 6
    n = C.c_size_t(0)
    rc = b.h.L.alz_sock_alive(b.h.h, None, 0, C.byref(n))
    assert rc == abi.E_CAPACITY and n.value == 6
    b.close()


# ---- 7. join -----------------------------------------------------------------------------------------------------------

def l7(n, saddr=0, daddr=0, wt=1):
    r = np.zeros(n, dtype=abi.L7_REC)
    r["saddr"], r["daddr"] = saddr, daddr
    r["sport"], r["dport"], r["protocol"], r["method_flags"], r["status"] = 40000, 80, abi.PROTO_HTTP, 1, 200
    r["duration_ns"] = 1000 + np.arange(n)
    r["write_time_ns"] = wt
    return r


def _tables(b, o):
    for k, ip in enumerate(PODS):
        b.upsert(abi.TABLE_POD, ip, k + 1)
        o.upsert(abi.TABLE_POD, ip, k + 1)
    for k, ip in enumerate(SVCS):
        b.upsert(abi.TABLE_SVC, ip, k + 11)
        o.upsert(abi.TABLE_SVC, ip, k + 11)
    b.commit()


def _flush_equal(b, o):
    got, exp = b.h.flush(), o.edges()
    assert edges_equal(got, exp), explain_diff(got, exp)
    return got


def test_join_only_records_with_both_addresses_zero():
    b, o = Both(), ol.Oracle()
    _tables(b, o)
    b.tcp(opened(*K, 100, saddr=PODS[0], daddr=SVCS[0]))
    recs = np.concatenate([l7(3), l7(3, saddr=PODS[1]), l7(3, daddr=SVCS[1]), l7(3, saddr=PODS[2], daddr=PODS[3])])
    keys = query(K[0], K[1], [150] * len(recs))
    joined, n = b.join(recs, keys, now=5)
    assert n == 3
    o.process(joined)
    _flush_equal(b, o)
    b.close()


def test_join_before_any_tcp_event_passes_records_unchanged():
    b, o = Both(), ol.Oracle()
    _tables(b, o)
    recs = np.concatenate([l7(5), l7(5, saddr=PODS[0], daddr=SVCS[0])])
    joined, n = b.join(recs, query(K[0], K[1], [150] * len(recs)), now=5)
    assert n == 0 and joined.tobytes() == recs.tobytes() and b.h.sock_stats()["joined_events"] == 0
    o.process(recs)
    _flush_equal(b, o)
    b.close()


def test_join_in_max_batch_chunks_with_a_ragged_tail():
    rng = np.random.default_rng(3)
    b, o = Both(max_batch=1024), ol.Oracle()
    _tables(b, o)
    keys_ = [(300 + i, 5) for i in range(20)]
    for i, k in enumerate(keys_):
        b.tcp(np.concatenate([opened(*k, 100, saddr=PODS[i % 8], daddr=SVCS[i % 3], sport=30000 + i, dport=80),
                              closed(*k, 5000), opened(*k, 9000, saddr=PODS[(i + 1) % 8], daddr=PODS[i % 8])]))
    n = 3 * 1024 + 77
    recs = l7(n)
    recs["saddr"][::7] = PODS[0]
    recs["daddr"][::7] = SVCS[2]
    pick = rng.integers(0, 20, n)
    keys = query([keys_[p][0] for p in pick], [keys_[p][1] for p in pick], rng.integers(0, 12000, n))
    keys["pid"][::11] = 77                                               # no line
    joined, nj = b.join(recs, keys, now=5)
    assert 1000 < nj < n
    o.process(joined)
    _flush_equal(b, o)
    b.close()


@pytest.mark.parametrize("d", [0, 1])
def test_join_stamps_decide_a_later_gc(d):
    A = 10 * MINUTE
    b, o = Both(), ol.Oracle()
    _tables(b, o)
    for op in sl.BOUNDARY["five_minutes_equal"][0][:5]:
        b.tcp(sl.script_rec(op))
    b.join(l7(1), query(*K, 15), now=A)
    b.join(l7(1), query(*K, 35), now=A + 5 * MINUTE + d)
    b.gc()
    assert b.o.lines()[K] == (4 if d == 0 else 2)
    b.sweep([K], grid(5, 10, 15, 20, 30, 35, 40, 50, 60), now=1)
    b.close()


def test_join_under_a_window_clock():
    """Joined records of the open, a future and a late epoch, a table commit while joined records are held, and the roll:
    the window model takes the records as the restatement joined them."""
    from test_gpu_window_clock import Pair
    W = 1000
    p = Pair(0, 0, W)
    b = Both(handle=p.h)
    rng = np.random.default_rng(4)
    keys_ = [(400 + i, 6) for i in range(12)]
    for i, k in enumerate(keys_):
        b.tcp(np.concatenate([opened(*k, 0, saddr=PODS[i % 8], daddr=SVCS[i % 3], sport=30000 + i, dport=80),
                              closed(*k, 50 * W), opened(*k, 60 * W, saddr=PODS[(i + 3) % 8], daddr=PODS[i % 8])]))
    p.submit(l7(1, saddr=PODS[0], daddr=SVCS[0], wt=20 * W + 1))             # opens epoch 20

    def join(wts, now):
        n = len(wts)
        recs = l7(n, wt=np.asarray(wts, np.uint64))
        recs["saddr"][::5], recs["daddr"][::5] = PODS[2], SVCS[1]
        pick = rng.integers(0, 12, n)
        keys = query([keys_[j][0] for j in pick], [keys_[j][1] for j in pick], rng.integers(0, 80 * W, n))
        joined, nj = b.join(recs, keys, now)
        p.m.submit(joined)
        p.check()
        return nj
    wts = [20 * W + 5, 21 * W + 3, 19 * W + 999, 22 * W, 20 * W + 999]
    assert join([wts[i % 5] for i in range(3000)], now=7) > 1000
    assert p.h.stats()["deferred_events"] > 0
    p.erase(abi.TABLE_POD, PODS[2])                                            # commit while joined records are held
    p.upsert(abi.TABLE_POD, STRANGER, 51)
    p.commit()
    join([wts[(i + 2) % 5] for i in range(2000)], now=3)
    for k in range(4):
        p.flush(f"window {20 + k}")
    p.fold()
    p.close()
    b.o.close()
    b.tables.close()


# ---- 8. random operation sequences ----------------------------------------------------------------------------------

_ALIAS = sl.alias_pairs()
KEYS = [(1, 3), (1, 4), (2, 3), _ALIAS[0][0], _ALIAS[0][1], _ALIAS[1][1]] + sl.keys_with_home(15, 3, 3, pid=9)
TS = [0, 1, M64, M64 - 1, 20 * 10**9, 40 * 10**9, 60 * 10**9, 80 * 10**9, 100 * 10**9, 120 * 10**9]
NOWS = [0, 1, MINUTE, 4 * MINUTE, 6 * MINUTE, 11 * MINUTE, M64 - 5 * MINUTE, M64]
SOCKS = [dict(saddr=PODS[0], daddr=SVCS[0]), dict(saddr=PODS[1], daddr=SVCS[0]), dict(saddr=PODS[0], daddr=PODS[2]),
         dict(saddr=STRANGER, daddr=SVCS[1]), dict(saddr=PODS[3], daddr=SVCS[0], dport=443)]
_key = st.integers(0, len(KEYS) - 1)
_ts = st.integers(0, len(TS) - 1)
op_s = st.one_of(
    st.tuples(st.just("tcp"), st.lists(st.tuples(_key, _ts, st.sampled_from([1, 1, 5]), st.integers(0, len(SOCKS) - 1)),
                                       min_size=1, max_size=6)),
    st.tuples(st.just("sweep"), st.integers(0, len(NOWS) - 1)),
    st.tuples(st.just("get"), _key, _ts, st.integers(0, len(NOWS) - 1)),
    st.tuples(st.just("gc")),
    st.tuples(st.just("alive")),
    st.tuples(st.just("join"), st.lists(st.tuples(_key, _ts), min_size=1, max_size=5), st.integers(1, len(NOWS) - 1)),
)


@settings(max_examples=200, deadline=None, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(ops=st.lists(op_s, min_size=1, max_size=14))
def test_random_operation_sequences(ops):
    b = Both(max_endpoints=64, max_pairs=256)
    try:
        for k, ip in enumerate(PODS[:4]):
            b.upsert(abi.TABLE_POD, ip, k + 1)
        b.upsert(abi.TABLE_SVC, SVCS[0], 11)
        b.commit()
        for op in ops:
            if op[0] == "tcp":
                r = np.concatenate([sl.tcp_rec(*KEYS[ki], TS[ti], typ, **{**dict(sport=1000 + si, dport=80),
                                                                        **SOCKS[si]}) for ki, ti, typ, si in op[1]])
                b.tcp(r)
            elif op[0] == "sweep":
                b.sweep(KEYS, TS + [10 * 10**9, 70 * 10**9, 130 * 10**9], now=NOWS[op[1]])
            elif op[0] == "get":
                _get(b, KEYS[op[1]], TS[op[2]], NOWS[op[3]])
            elif op[0] == "gc":
                b.gc()
            elif op[0] == "alive":
                b.alive()
            else:
                n = len(op[1])
                b.join(l7(n), query([KEYS[k][0] for k, _ in op[1]], [KEYS[k][1] for k, _ in op[1]],
                                    [TS[t] for _, t in op[1]]), NOWS[op[2]])
        b.gc()
        b.sweep(KEYS, TS, now=1)
    finally:
        b.close()
