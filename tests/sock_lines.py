"""Constructed socket timelines for alaz_b200/csrc/alz_sock.cu. TEST INFRASTRUCTURE ONLY.

Plain numpy plus the oracle:
  - `hash64` (the fmix64 of alz_device.cuh) and `line_slot`, the home slot of a (pid, fd) in the line index, so that a
    test can build keys that share a home slot, chains that wrap past the end of the index, and keys that alias in the
    hash input;
  - `SyncModel`, the bookkeeping of `sync_lines`: when the index is rebuilt and to what size, where segments move, and
    when the record pool is re-laid. It predicts `alz_sock_stats` exactly, so a test can assert that a case reached
    the path it was built for;
  - `tcp_rec` / `query` record builders, and `Both`, which applies every operation to a `capi.Handle` and to the C
    restatement (`ol.SockMaps`, `ol.Oracle` for the alive export) and compares after each step.
"""
import numpy as np

import oracle_lib as ol
from alaz_b200 import abi

M64 = (1 << 64) - 1
MINUTE = 60 * 10**9
LOCALHOST = 0x7F000001
GOLDEN = 0x9E3779B97F4A7C15
POOL_MIN = 1 << 16


def hash64(x):
    """fmix64 (alz_device.cuh `hash64`), vectorised over uint64."""
    x = np.asarray(x, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = x ^ (x >> np.uint64(33))
        x = x * np.uint64(0xFF51AFD7ED558CCD)
        x = x ^ (x >> np.uint64(33))
        x = x * np.uint64(0xC4CEB9FE1A85EC53)
        x = x ^ (x >> np.uint64(33))
    return x


def line_key(pid, fd):
    """The hash input of a line: ((u64)pid << 40) ^ fd ^ golden. The shift drops pid bits 24..31."""
    pid = np.asarray(pid, dtype=np.uint64) & np.uint64(0xFFFFFFFF)
    with np.errstate(over="ignore"):
        return (pid << np.uint64(40)) ^ np.asarray(fd, dtype=np.uint64) ^ np.uint64(GOLDEN)


def line_slot(pid, fd, mask):
    return hash64(line_key(pid, fd)) & np.uint64(mask)


def pow2_at_least(x):
    p = 16
    while p < x:
        p <<= 1
    return p


def index_cap_for(n_lines, cap=0):
    """The index size after a sync with n_lines lines, from an index of `cap` slots."""
    return pow2_at_least(4 * n_lines + 1) if n_lines * 2 > cap else cap


def seg_cap_for(n):
    return max(8, pow2_at_least(n + n // 2))


# ---- key builders --------------------------------------------------------------------------------------------------

def keys_with_home(mask, slot, n, pid=4242, fd_from=3):
    """n (pid, fd) keys with one pid whose home slot is `slot`."""
    out, lo = [], fd_from
    while len(out) < n:
        fds = np.arange(lo, lo + (1 << 20), dtype=np.uint64)
        hit = fds[line_slot(pid, fds, mask) == np.uint64(slot)]
        out += [(pid, int(f)) for f in hit[: n - len(out)]]
        lo += 1 << 20
    return out


def wrap_chain(mask, n):
    """n keys whose home is slot mask - 1 (they fill mask - 1, mask, 0, 1, ...), then one key whose home is slot 0."""
    return keys_with_home(mask, mask - 1, n, pid=777) + keys_with_home(mask, 0, 1, pid=778)


def alias_pairs(pid=0x123, fd=0x45):
    """Pairs of distinct keys with one hash input: (pid, fd) ~ (pid + 2^24, fd) and (pid, fd) ~ (0, fd ^ pid << 40)."""
    return [((pid, fd), (pid + (1 << 24), fd)), ((pid, fd), (0, fd ^ (pid << 40)))]


# ---- records -------------------------------------------------------------------------------------------------------

def tcp_rec(pid, fd, ts, typ, saddr=0x0A000001, daddr=0x0A100001, sport=40000, dport=80):
    """One alz_tcp_rec per element; scalars broadcast. typ 1 = ESTABLISHED, 5 = CLOSED."""
    pid, fd, ts, typ, saddr, daddr, sport, dport = np.broadcast_arrays(
        *[np.asarray(a, dtype=object) for a in (pid, fd, ts, typ, saddr, daddr, sport, dport)])
    r = np.zeros(pid.size, dtype=abi.TCP_REC)
    for f, a in (("pid", pid), ("fd", fd), ("timestamp_ns", ts), ("type", typ), ("saddr", saddr), ("daddr", daddr),
                 ("sport", sport), ("dport", dport)):
        r[f] = [int(x) for x in a.ravel()]
    return r


def opened(pid, fd, ts, **kw):
    return tcp_rec(pid, fd, ts, 1, **kw)


def closed(pid, fd, ts):
    return tcp_rec(pid, fd, ts, 5)


def query(pid, fd, ts):
    pid, fd, ts = np.broadcast_arrays(*[np.asarray(a, dtype=object) for a in (pid, fd, ts)])
    q = np.zeros(pid.size, dtype=abi.SOCK_QUERY)
    q["pid"] = [int(x) for x in pid.ravel()]
    q["fd"] = [int(x) for x in fd.ravel()]
    q["timestamp_ns"] = [int(x) for x in ts.ravel()]
    return q


# ---- sync_lines bookkeeping ------------------------------------------------------------------------------------------

class SyncModel:
    """alz_sock.cu `sync_lines` without the records: per line its device length and segment capacity, the index size,
    and the pool counters. `sync(lens, forced)` takes every line's host length (ol.SockMaps.lines()) and the lines the
    GC re-sends whole."""

    def __init__(self):
        self.dev = {}                 # key -> [dev_len, seg_cap]
        self.index_cap = 0
        self.pool_cap = self.used = self.garbage = 0
        self.syncs = self.repools = self.rebuilds = self.ops = self.bytes = 0
        self.garbage_repools = self.rebuild_with_repool = self.max_garbage = 0

    def sync(self, lens, forced=()):
        forced = set(forced)
        for k in forced:
            self.dev[k][0] = 0
        dirty = [k for k, n in lens.items() if k not in self.dev or self.dev[k][0] != n or k in forced]
        if not dirty:
            return False
        for k in dirty:
            self.dev.setdefault(k, [0, 0])
        resend = len(lens) * 2 > self.index_cap
        if resend:
            self.index_cap = pow2_at_least(4 * len(lens) + 1)
            self.rebuilds += 1
        need = sum(seg_cap_for(lens[k]) for k in dirty if lens[k] > self.dev[k][1])
        full = self.used + need > self.pool_cap
        by_garbage = self.garbage > POOL_MIN and self.garbage * 2 > self.used
        ops = sum(lens[k] - self.dev[k][0] for k in dirty)
        if full or by_garbage:
            for k in lens:
                self.dev[k][1] = seg_cap_for(lens[k])
            total = sum(d[1] for d in self.dev.values())
            self.pool_cap, self.used, self.garbage = max(POOL_MIN, 2 * total), total, 0
            self.repools += 1
            self.garbage_repools += not full
            self.rebuild_with_repool += resend
            n_desc = len(lens)
        else:
            for k in dirty:
                if lens[k] > self.dev[k][1]:
                    self.garbage += self.dev[k][1]
                    self.dev[k][1] = seg_cap_for(lens[k])
                    self.used += self.dev[k][1]
            self.max_garbage = max(self.max_garbage, self.garbage)
            n_desc = len(dirty)
        for k in dirty:
            self.dev[k][0] = lens[k]
        self.syncs += 1
        self.ops += ops
        self.bytes += ((n_desc * 40 + 15) & ~15) + ops * 48 + (self.index_cap * 32 if resend else 0)
        return True

    def stats(self):
        return dict(lines=len(self.dev), pool_records=self.used, pool_garbage=self.garbage, syncs=self.syncs,
                    sync_ops=self.ops, sync_bytes=self.bytes, repools=self.repools)


# ---- both sides at once --------------------------------------------------------------------------------------------

def sort_alive(a):
    return np.sort(a, order=list(abi.ALIVE_CONN.names)[:-1]).tobytes()


class Both:
    """A handle, the C restatement and the sync model, driven together; every result is compared as it comes."""

    def __init__(self, handle=None, **kw):
        from alaz_b200 import capi
        self.h = handle if handle is not None else capi.Handle(max_endpoints=kw.pop("max_endpoints", 256),
                                                                max_pairs=kw.pop("max_pairs", 1 << 12), **kw)
        self.o = ol.SockMaps()
        self.m = SyncModel()
        self.tables = ol.Oracle()

    def close(self):
        self.h.close()
        self.o.close()
        self.tables.close()

    def _sync(self, forced=()):
        self.m.sync(self.o.lines(), forced)

    def tcp(self, recs):
        recs = np.ascontiguousarray(recs, dtype=abi.TCP_REC)
        self.h.submit_tcp(recs)
        self.o.process(recs)

    def lookup(self, q, now):
        q = np.ascontiguousarray(q, dtype=abi.SOCK_QUERY)
        got = self.h.sock_lookup(q, now_ns=now)
        exp = self.o.lookup(q, now_ns=now)
        self._sync()
        bad = np.flatnonzero(got != exp)
        assert got.tobytes() == exp.tobytes(), (now, q[bad[:8]], got[bad[:8]], exp[bad[:8]])
        self.check()
        return got

    def sweep(self, keys, tss, now):
        """Every key at every timestamp of tss, as one lookup."""
        pid = [k[0] for k in keys for _ in tss]
        fd = [k[1] for k in keys for _ in tss]
        return self.lookup(query(pid, fd, [t for _ in keys for t in tss]), now)

    def gc(self):
        self._sync()                                  # the GC syncs pending inserts before it reads the stamps
        forced = [k for k, n in self.o.lines().items() if n >= 2]
        self.h.sock_gc()
        self.o.gc()
        self._sync(forced)
        assert self.h.sock_stats()["pool_records"] == self.m.used
        self.check()

    def upsert(self, table, ip, id_):
        """Staged on the device until commit(); the restatement's tables follow only at the commit."""
        self.h.upsert(table, ip, id_)
        self._staged = getattr(self, "_staged", []) + [("u", table, ip, id_)]

    def erase(self, table, ip):
        self.h.erase(table, ip)
        self._staged = getattr(self, "_staged", []) + [("e", table, ip, 0)]

    def commit(self):
        self.h.commit()
        for op, table, ip, id_ in getattr(self, "_staged", []):
            if op == "u":
                self.tables.upsert(table, ip, id_)
            else:
                self.tables.erase(table, ip)
        self._staged = []

    def alive(self, cap=1 << 12):
        got = self.h.sock_alive(cap)
        exp = self.o.alive(self.tables, cap)
        self._sync()
        assert sort_alive(got) == sort_alive(exp), (got, exp)
        self.check()
        return got

    def join(self, recs, keys, now):
        """alz_submit_l7_join on the handle; returns the records as the restatement joined them (to feed an oracle)."""
        joined, n = self.o.join(recs, keys, now_ns=now)
        before = self.h.sock_stats()["joined_events"]
        self.h.submit_join(recs, keys, now_ns=now)
        self._sync()
        assert self.h.sock_stats()["joined_events"] - before == n
        self.check()
        return joined, n

    def check(self):
        got, exp = self.h.sock_stats(), self.m.stats()
        for k, v in exp.items():
            assert got[k] == v, (k, got[k], v, got, exp)


# ---- hand-derived boundary lines ---------------------------------------------------------------------------------
# A script is a list of operations on lines keyed (pid, fd):
#   ("o", key, ts, k)       an ESTABLISHED event of socket k: saddr BASE + k, daddr DST, sport 40000 + k, dport 80
#   ("o", key, ts, k, daddr, dport)
#   ("c", key, ts)          a CLOSED event
#   ("get", key, ts, now)   a lookup; expected: the k of the socket found, or None
#   ("gc",)                 one GC tick; expected: the records left in every line
# `expected` lists one value per get and gc, in order. Derived by hand from sock_num_line.go.

BASE, DST = 0x0A000000, 0x0A100001
K, K2, K3 = (100, 7), (101, 7), (102, 7)
TB = 10**6


def sock(k, daddr=DST, dport=80):
    return dict(saddr=BASE + k, daddr=daddr, sport=40000 + k, dport=dport)


def _d1(d):
    A = 10 * MINUTE
    return ([("o", K, 10, 1), ("c", K, 20), ("o", K, 30, 2), ("c", K, 40), ("o", K, 50, 3),
             ("get", K, 15, A), ("get", K, 35, A + 5 * MINUTE + d), ("gc",), ("get", K, 15, 1)],
            [1, 2, 4 if d == 0 else 2, 1 if d == 0 else 2])


def _near_wrap(x):
    keep = (x + 5 * MINUTE) % (1 << 64) >= x            # the sum does not wrap: the stamp's pair is kept
    return ([("o", K, 10, 1), ("c", K, 20), ("o", K, 30, 2), ("c", K, 40), ("o", K, 50, 3), ("o", K, 60, 4),
             ("get", K, 15, x), ("get", K, 35, 10**9), ("gc",), ("get", K, 15, 1)],
            [1, 2, 3 if keep else 1, 1 if keep else 4])


BOUNDARY = {
    # sort.Search lands on a record whose timestamp equals the query
    "equal_ts": ([("o", K, 100, 1), ("c", K, 200), ("o", K, 300, 3),
                  ("get", K, 100, 1), ("get", K, 200, 1), ("get", K, 300, 1), ("get", K, 301, 1), ("get", K, 99, 1)],
                 [1, 1, 3, 3, 1]),
    # AddValue inserts before equal timestamps: [close@100, s2@100, s1@100]
    "equal_values": ([("o", K, 100, 1), ("o", K, 100, 2), ("c", K, 100),
                      ("get", K, 99, 1), ("get", K, 100, 1), ("get", K, 101, 1)],
                     [None, None, 1]),
    "ts_0_and_max": ([("o", K, 0, 1), ("c", K, M64), ("get", K, 0, 1), ("get", K, M64, 1), ("get", K, 5, 1),
                      ("o", K, M64, 2), ("get", K, M64, 1), ("get", K, M64 - 1, 1),
                      ("o", K2, M64 - 10, 4), ("c", K2, M64 - 5), ("get", K2, M64 - 1, 1), ("get", K2, 0, 1)],
                     [1, 1, 1, 1, 1, 4, 4]),
    # after a last close: the open before it within one minute (exclusive)
    "one_minute": ([("o", K, TB, 1), ("c", K, TB + 1000), ("get", K, TB + MINUTE - 1, 1), ("get", K, TB + MINUTE, 1),
                    ("get", K, TB + 1000, 1)],
                   [1, None, 1]),
    # closed gap: the nearer open; on a tie the later one
    "closed_gap_tie": ([("o", K, 100, 1), ("c", K, 150), ("o", K, 300, 3),
                        ("get", K, 200, 1), ("get", K, 199, 1), ("get", K, 201, 1), ("get", K, 150, 1)],
                       [3, 1, 3, 1]),
    # a closed gap between sockets to different destinations finds nothing; other fields may differ
    "closed_gap_dest": ([("o", K, 100, 1), ("c", K, 150), ("o", K, 300, 3, DST + 1, 80),
                         ("o", K2, 100, 1), ("c", K2, 150), ("o", K2, 300, 3, DST, 443),
                         ("o", K3, 100, 1), ("c", K3, 150), ("o", K3, 300, 3),
                         ("get", K, 200, 1), ("get", K2, 200, 1), ("get", K3, 200, 1), ("get", K3, 199, 1)],
                        [None, None, 3, 1]),
    # a close older than the line's first open becomes its first value
    "first_is_close": ([("o", K, 200, 1), ("c", K, 100),
                        ("get", K, 50, 1), ("get", K, 100, 1), ("get", K, 150, 1), ("get", K, 200, 1),
                        ("get", K, 250, 1)],
                       [None, None, None, None, 1]),
    # the dedupe looks at the last value only, even when the new open is earlier in time
    "dedupe_earlier": ([("o", K, 300, 1), ("o", K, 100, 2), ("o", K, 50, 1),
                        ("get", K, 40, 1), ("get", K, 60, 1), ("get", K, 200, 1), ("get", K, 400, 1),
                        ("o", K2, 300, 5), ("c", K2, 400), ("o", K2, 100, 5),
                        ("get", K2, 50, 1), ("get", K2, 350, 1), ("get", K2, 450, 1)],
                       [2, 2, 2, 1, 5, 5, 5]),
    "five_minutes_equal": _d1(0),
    "five_minutes_plus_1ns": _d1(1),
    # a stamp of 0 means "never matched": a lookup at now = 0 after a stamp takes the pair out of the maximum
    "stamp_reset_to_0": ([("o", K, 10, 1), ("c", K, 20), ("o", K, 30, 2), ("c", K, 40), ("o", K, 50, 3),
                          ("get", K, 15, 9 * MINUTE), ("get", K, 35, MINUTE), ("get", K, 15, 0), ("gc",),
                          ("get", K, 35, 1)],
                         [1, 2, 1, 4, 2]),
    # LastMatch is the last call's now, not the largest: (10,20) goes with its 1-minute stamp
    "stamp_goes_back": ([("o", K, 10, 1), ("c", K, 20), ("o", K, 30, 2), ("c", K, 40), ("o", K, 50, 3), ("c", K, 60),
                         ("o", K, 70, 4),
                         ("get", K, 15, 9 * MINUTE), ("get", K, 15, MINUTE), ("get", K, 55, 7 * MINUTE), ("gc",),
                         ("get", K, 15, 1), ("get", K, 65, 1)],
                        [1, 1, 3, 2, 3, 3]),
    # DeleteUnused's first loop on lines that end open-open, open-close and close-open (nothing matched)
    "gc_endings": ([("o", K, 10, 1), ("c", K, 20), ("o", K, 30, 2), ("o", K, 40, 3),
                    ("o", K2, 10, 1), ("c", K2, 20), ("o", K2, 30, 2), ("c", K2, 40),
                    ("o", K3, 10, 1), ("c", K3, 20), ("c", K3, 30), ("o", K3, 40, 4), ("gc",),
                    ("get", K, 35, 1), ("get", K2, 35, 1), ("get", K3, 45, 1), ("get", K3, 25, 1)],
                   [9, 3, 2, None, None]),
    "stamp_at_max": _near_wrap(M64),
    "stamp_5min_below_2_64_minus_1": _near_wrap((1 << 64) - 5 * MINUTE - 1),
    "stamp_5min_below_2_64": _near_wrap((1 << 64) - 5 * MINUTE),
    "stamp_5min_below_2_64_plus_1": _near_wrap((1 << 64) - 5 * MINUTE + 1),
    # a close stamped as the last value takes its line's only pair with it: the line is empty, then grows again
    "emptied_and_regrown": ([("o", K, 10, 1), ("c", K, 20), ("get", K, 25, 10 * MINUTE), ("c", K, 30), ("gc",),
                             ("get", K, 25, 1), ("o", K, 40, 2), ("get", K, 50, 1), ("get", K, 5, 1)],
                            [1, 0, None, 2, 2]),
}


def script_rec(op):
    """The alz_tcp_rec of an "o" or "c" operation."""
    if op[0] == "o":
        s = sock(op[3], *op[4:])
        return opened(op[1][0], op[1][1], op[2], **s)
    return closed(op[1][0], op[1][1], op[2])


def found_k(saddr):
    return int(saddr) - BASE
