"""Constructed endpoint-table layouts and pod-address filter cases for alaz_b200/csrc/alz_api.cu and the device code
that reads them. TEST INFRASTRUCTURE ONLY.

Plain numpy plus the oracle:
  - `hash32` (alz_device.cuh) and its inverse `unhash32`: hash32 is a bijection, so a test chooses the hash of an
    address (its home slot, its two filter bits) and inverts it to get the address;
  - `ep_cap`, `home` and `filter_bits`, as `alz_create`, `ep_mirror_put` and `bloom_update` derive them;
  - constructors of addresses with a chosen home slot, with chosen filter bits, and of non-pod addresses that pass the
    filter of a given pod set (false positives);
  - `MirrorModel`, the host mirror of the table (linear probing, backward-shift deletion, applied at commit in the
    order the changes were made) with the filter counters of `FilterModel`, so that a test can assert that a case has
    the layout it claims;
  - `Both`, which applies upserts and erases to a `capi.Handle` at once and to an `ol.Oracle` only at `commit()`, and
    compares every flushed window per edge and the stats;
  - `probe_window`, the records that read every address of a universe through every device reader of the table.
"""
import numpy as np

import oracle_lib as ol
from alaz_b200 import abi

M32 = (1 << 32) - 1
C1, C2 = 0x85EBCA6B, 0xC2B2AE35
C1_INV, C2_INV = pow(C1, -1, 1 << 32), pow(C2, -1, 1 << 32)
BLOOM_BITS = 1 << 17                   # ALZ_BLOOM_WORDS * 32
BLOOM_MASK = BLOOM_BITS - 1
ID_MAX = (1 << 29) - 1
HOST_DADDR = abi.ip("192.0.2.1")       # what the oracle sees for a Host-keyed record (kept out of every table)
HOSTS = ["h%d.example" % k for k in range(4)]   # Host-keyed records carry ids 0..3; the oracle numbers hosts by index
SPECIAL = (0, M32, HOST_DADDR)


def _mul(x, c):
    return (x * np.uint64(c)) & np.uint64(M32)


def hash32(x):
    """alz_device.cuh `hash32`, vectorised (uint32 in, uint32 out)."""
    x = np.asarray(x, dtype=np.uint64) & np.uint64(M32)
    x ^= x >> np.uint64(16)
    x = _mul(x, C1)
    x ^= x >> np.uint64(13)
    x = _mul(x, C2)
    x ^= x >> np.uint64(16)
    return x.astype(np.uint32)


def unhash32(h):
    """The inverse of hash32: x ^= x >> 16 is its own inverse, the multiplies are undone by the modular inverses, and
    x ^= x >> 13 by x ^ x >> 13 ^ x >> 26."""
    x = np.asarray(h, dtype=np.uint64) & np.uint64(M32)
    x ^= x >> np.uint64(16)
    x = _mul(x, C2_INV)
    x = x ^ (x >> np.uint64(13)) ^ (x >> np.uint64(26))
    x = _mul(x, C1_INV)
    x ^= x >> np.uint64(16)
    return x.astype(np.uint32)


def ep_cap(max_endpoints):
    """Slots of the table: next_pow2(2 * max_endpoints), clamped at 2^31 (alz_api.cu)."""
    p = 1
    while p < 2 * max_endpoints:
        p <<= 1
    return min(p, 1 << 31)


def home(ip, cap):
    return hash32(ip) & np.uint32(cap - 1)


def filter_bits(ip):
    """(b1, b2) of `bloom_update` and `maybe_pod`: h & 0x1FFFF and (h >> 15) & 0x1FFFF."""
    h = hash32(ip)
    return h & np.uint32(BLOOM_MASK), (h >> np.uint32(15)) & np.uint32(BLOOM_MASK)


# ---- constructors ------------------------------------------------------------------------------------------------------

def _from_hashes(hs, n, avoid):
    """The first n addresses of the hash values hs that are not special and not in `avoid`."""
    avoid = set(int(a) for a in avoid) | set(SPECIAL)
    out = []
    for a in unhash32(np.asarray(hs, dtype=np.uint64)).tolist():
        if a not in avoid:
            avoid.add(a)
            out.append(a)
            if len(out) == n:
                return out
    raise ValueError("not enough addresses")


def with_home(cap, slot, n, seed=0, avoid=()):
    """n distinct addresses whose home slot is `slot` in a table of `cap` slots; the hash bits above the slot are
    drawn from `seed`, so that their filter bits differ."""
    shift = cap.bit_length() - 1
    free = np.random.default_rng(seed).permutation(1 << min(32 - shift, 20))[: 4 * n + 16].astype(np.uint64)
    return _from_hashes((free << np.uint64(shift)) | np.uint64(slot), n, avoid)


def with_b1(b1, n, seed=0, avoid=()):
    """n addresses whose filter bit b1 is `b1` (hash bits 17..31 drawn from `seed`). In a table of at most 2^17
    slots they all share one home slot, b1 & (cap - 1)."""
    free = np.random.default_rng(seed).permutation(1 << 15)[: 2 * n + 16].astype(np.uint64)
    return _from_hashes((free << np.uint64(17)) | np.uint64(b1), n, avoid)


def with_b2(b2, n, seed=0, avoid=()):
    """n addresses whose filter bit b2 is `b2` (hash bits 0..14 drawn from `seed`: their home slots differ)."""
    free = np.random.default_rng(seed).permutation(1 << 15)[: 2 * n + 16].astype(np.uint64)
    return _from_hashes((np.uint64(b2) << np.uint64(15)) | free, n, avoid)


def with_bits(b1, b2):
    """The one address with filter bits (b1, b2); they overlap in two hash bits, so b1 >> 15 must equal b2 & 3."""
    assert b1 >> 15 == b2 & 3, (b1, b2)
    return int(unhash32((b2 >> 2) << 17 | b1))


def equal_bits(n, seed=0, avoid=()):
    """n addresses whose two filter bits are one bit (b1 == b2)."""
    b = np.random.default_rng(seed).permutation(1 << 15)[: 2 * n + 16].astype(np.uint64)
    b = (b << np.uint64(2)) | ((b >> np.uint64(13)) & np.uint64(3))   # bits 0..1 = bits 15..16
    return _from_hashes(((b >> np.uint64(2)) << np.uint64(17)) | b, n, avoid)


def false_positives(pods, n, avoid=()):
    """n addresses outside `pods` and `avoid` whose two filter bits are both set by `pods`: the filter lets them
    through although none of them is a pod."""
    bits = sorted({int(b) for ab in filter_bits(np.asarray(pods, np.uint32)) for b in ab})
    by_low = {}
    for b in bits:
        by_low.setdefault(b & 3, []).append(b)
    hs = [(y >> 2) << 17 | x for x in bits for y in by_low.get(x >> 15, [])]
    return _from_hashes(hs, n, set(int(p) for p in pods) | set(int(a) for a in avoid))


def wrapped_chain(cap, seed=1):
    """12 addresses homed at cap - 4 and one homed at each of 0..3, and an insertion order that lays them out as
        low[0]: 0 | low[3]: 3 | chain[0..3]: cap-4..cap-1 | chain[4], chain[5]: 1, 2 | chain[6..8]: 4..6 |
        low[2]: 7 | chain[9..11]: 8..10 | low[1]: 11
    A delete before the wrap moves chain entries back across the end, while low[0] and low[3], at their homes, stay:
    low[0] only by the wrapped branch of the backward-shift rule (free slot cap - 1, entry at 0)."""
    chain = with_home(cap, cap - 4, 12, seed=seed)
    low = [with_home(cap, s, 1, seed=seed * 16 + s, avoid=chain)[0] for s in range(4)]
    order = [low[0], low[3]] + chain[:9] + [low[2]] + chain[9:] + [low[1]]
    return chain, low, order


def merged_chains(cap, h, n, seed=2):
    """n addresses homed at h and n at h + 1, interleaved: a[0], b[0], a[1], b[1], ... fill h, h + 1, h + 2, ..."""
    a = with_home(cap, h, n, seed=seed)
    b = with_home(cap, (h + 1) & (cap - 1), n, seed=seed + 1, avoid=a)
    return a, b, [x for pair in zip(a, b) for x in pair]


def random_addrs(n, seed=0, avoid=()):
    rng = np.random.default_rng(seed)
    return _from_hashes(rng.integers(1, M32, 2 * n + 16, dtype=np.uint64), n, avoid)


# ---- models ------------------------------------------------------------------------------------------------------------

class FilterModel:
    """The host's per-bit u8 counters: an add counts up to 255 and stays there, a delete counts down unless the counter
    is saturated, so that the filter only ever errs towards "maybe a pod"."""

    def __init__(self):
        self.cnt = np.zeros(BLOOM_BITS, np.int32)

    def update(self, ip, delta):
        for b in filter_bits(ip):
            c = self.cnt[int(b)]
            if delta > 0:
                self.cnt[int(b)] = min(c + 1, 255)
            elif c not in (0, 255):
                self.cnt[int(b)] = c - 1

    def bitmap(self):
        return self.cnt > 0


class MirrorModel:
    """The host side of the table (alz_api.cu): per address its pod and service, capacity checked at upsert, changes
    queued in order and applied to the open-addressed mirror at commit (linear probing; deletion by backward shift, no
    tombstones). `bits` is the filter as the device had it at the last commit."""

    def __init__(self, max_endpoints):
        self.max_endpoints = max_endpoints
        self.cap = ep_cap(max_endpoints)
        self.mask = self.cap - 1
        self.host = {}                                   # ip -> [pod or None, svc or None]
        self.dirty = []
        self.ip = np.zeros(self.cap, np.int64)
        self.occ = np.zeros(self.cap, bool)
        self.val = [None] * self.cap
        self.filter = FilterModel()
        self.bits = self.filter.bitmap()

    # ---- the API: what upsert / erase / commit do on the host
    def upsert(self, table, ip, id_):
        """abi.OK, abi.E_INVAL or abi.E_CAPACITY, with the effects of alz_table_upsert."""
        if id_ > ID_MAX:
            return abi.E_INVAL
        e = self.host.get(ip)
        if e is None:
            if len(self.host) >= self.max_endpoints:
                return abi.E_CAPACITY
            e = self.host[ip] = [None, None]
        if table == abi.TABLE_POD and e[0] is None:
            self.filter.update(ip, +1)
        e[0 if table == abi.TABLE_POD else 1] = id_
        self.dirty.append(ip)
        return abi.OK

    def erase(self, table, ip):
        e = self.host.get(ip)
        if e is None:
            return
        k = 0 if table == abi.TABLE_POD else 1
        if k == 0 and e[0] is not None:
            self.filter.update(ip, -1)
        e[k] = None
        if e == [None, None]:
            del self.host[ip]
        self.dirty.append(ip)

    def commit(self):
        for ip in self.dirty:
            if ip in self.host:
                self._put(ip, tuple(self.host[ip]))
            else:
                self._del(ip)
        self.dirty = []
        self.bits = self.filter.bitmap()

    # ---- the mirror
    def home(self, ip):
        return int(home(ip, self.cap))

    def _put(self, ip, v):
        s = self.home(ip)
        while self.occ[s] and self.ip[s] != ip:
            s = (s + 1) & self.mask
        self.occ[s], self.ip[s], self.val[s] = True, ip, v

    def _del(self, ip):
        i = self.home(ip)
        while self.occ[i] and self.ip[i] != ip:
            i = (i + 1) & self.mask
        if not self.occ[i]:
            return
        j = i
        while True:
            j = (j + 1) & self.mask
            if not self.occ[j]:
                break
            k = self.home(int(self.ip[j]))
            stays = (i < k <= j) if i <= j else (i < k or k <= j)
            if stays:
                continue
            self.ip[i], self.val[i] = self.ip[j], self.val[j]
            i = j
        self.occ[i], self.ip[i], self.val[i] = False, 0, None

    def slot_of(self, ip):
        """The slot that holds ip, or None."""
        s = self.home(ip)
        while self.occ[s]:
            if self.ip[s] == ip:
                return s
            s = (s + 1) & self.mask
        return None

    def probes(self, ip):
        """Slots a lookup of ip reads (ep_lookup): up to the one that holds it or the first free slot."""
        s, n = self.home(ip), 1
        while self.occ[s] and self.ip[s] != ip:
            s, n = (s + 1) & self.mask, n + 1
        return n

    def committed(self):
        """{ip: (pod, svc)} of the mirror."""
        return {int(self.ip[s]): self.val[s] for s in np.flatnonzero(self.occ)}

    def maybe_pod(self, ip):
        return all(self.bits[int(b)] for b in filter_bits(ip))

    def check(self):
        """Every key is reachable from its home without crossing a free slot, slots and keys agree in number, and the
        mirror holds what the host map held at the last commit."""
        occ = np.flatnonzero(self.occ)
        assert len(set(self.ip[occ].tolist())) == len(occ)
        for s in occ:
            h = self.home(int(self.ip[s]))
            t = h
            while t != s:
                assert self.occ[t], (int(self.ip[s]), h, int(s), t)
                t = (t + 1) & self.mask


# ---- records -----------------------------------------------------------------------------------------------------------

def records(saddr, daddr, dur, proto=abi.PROTO_HTTP, method=1, status=200, wt=1):
    saddr, daddr, dur, proto, method, status, wt = np.broadcast_arrays(
        *[np.asarray(a, dtype=np.uint64) for a in (saddr, daddr, dur, proto, method, status, wt)])
    r = np.zeros(saddr.size, dtype=abi.L7_REC)
    r["saddr"], r["daddr"] = saddr.ravel(), daddr.ravel()
    r["sport"], r["dport"] = 40000 + np.arange(saddr.size) % 20000, 80
    r["status"], r["protocol"], r["method_flags"] = status.ravel(), proto.ravel(), method.ravel()
    r["duration_ns"], r["write_time_ns"] = dur.ravel(), wt.ravel()
    return r


def probe_window(universe, pod0, svc0, wt=1):
    """For every address A of the universe (index i): A -> svc0 and pod0 -> A as plain HTTP (5xx on odd i), as AMQP
    DELIVER (reversed), and A -> host (i % 4) as a Host-keyed HTTP record. A -> ... reads A as a source (a pod row, or
    a drop); pod0 -> A reads it as a destination (service, pod or outbound). Every address has its own latencies, so
    two addresses that resolve to each other's rows show up."""
    u = np.asarray(universe, dtype=np.uint64)
    i = np.arange(len(u), dtype=np.uint64)
    d = np.uint64(1000) + i * np.uint64(7919)
    st = np.where(i % 2 == 1, 503, 200)
    H, A, D = abi.PROTO_HTTP, abi.PROTO_AMQP, abi.AMQP_DELIVER
    parts = [records(u, svc0, d, H, 1, st, wt), records(pod0, u, d + np.uint64(3), H, 1, st, wt),
             records(u, svc0, d << np.uint64(3), A, D, 200, wt), records(pod0, u, d << np.uint64(5), A, D, 200, wt),
             records(u, i % np.uint64(4), d << np.uint64(7), H | abi.PROTO_F_HOSTKEY, 1, st, wt)]
    return np.concatenate(parts)


def oracle_view(recs):
    """The records as the oracle takes them: a Host-keyed record's daddr becomes HOST_DADDR and its id a Host header."""
    recs = np.ascontiguousarray(recs, dtype=abi.L7_REC).copy()
    hk = (recs["protocol"] & abi.PROTO_F_HOSTKEY) != 0
    idx = np.zeros(len(recs), np.uint32)
    idx[hk] = 1 + recs["daddr"][hk]
    recs["daddr"][hk] = HOST_DADDR
    recs["protocol"][hk] &= ~np.uint8(abi.PROTO_F_HOSTKEY)
    return recs, idx


STAT_KEYS = ("events_in", "rows_emitted", "not_request", "src_unresolved", "capacity_events")


class Both:
    """A handle and the oracle driven together: upserts and erases reach the handle (and the mirror model) at once and
    the oracle only at commit(), so both resolve every record by the tables committed when it was submitted. `fmt16`
    submits packed 16-B records."""

    def __init__(self, max_endpoints, max_pairs=1 << 10, flags=0, fmt16=False, model=True, handle=None):
        from alaz_b200 import capi
        self.h = handle or capi.Handle(max_endpoints=max_endpoints, max_pairs=max_pairs, flags=flags)
        self.o = ol.Oracle()
        self.m = MirrorModel(max_endpoints) if model else None
        self.fmt16 = fmt16
        self.staged = []
        self.windows = 0

    def close(self):
        self.h.close()
        self.o.close()

    def upsert(self, table, ip, id_, expect=abi.OK):
        rc = self.h.L.alz_table_upsert(self.h.h, table, int(ip), int(id_))
        if self.m is not None:
            assert self.m.upsert(table, int(ip), int(id_)) == rc
        assert rc == expect, (rc, expect)
        if rc == abi.OK:
            self.staged.append(("u", table, int(ip), int(id_)))
        return rc

    def upsert_batch(self, table, ips, ids):
        """alz_table_upsert_batch; the model and the oracle take the prefix the handle applied."""
        ips, ids = np.asarray(ips, np.uint32), np.asarray(ids, np.uint32)
        rc = self.h.L.alz_table_upsert_batch(self.h.h, table, ips.ctypes.data, ids.ctypes.data, len(ips))
        exp = abi.OK
        for ip, i in zip(ips.tolist(), ids.tolist()):
            exp = self.m.upsert(table, ip, i) if self.m is not None else (abi.E_INVAL if i > ID_MAX else abi.OK)
            if exp != abi.OK:
                break
            self.staged.append(("u", table, ip, i))
        assert rc == exp, (rc, exp)
        return rc

    def erase(self, table, ip):
        self.h.erase(table, ip)
        if self.m is not None:
            self.m.erase(table, int(ip))
        self.staged.append(("e", table, int(ip), 0))

    def commit(self):
        self.h.commit()
        if self.m is not None:
            self.m.commit()
            self.m.check()
        for op, table, ip, id_ in self.staged:
            if op == "u":
                self.o.upsert(table, ip, id_)
            else:
                self.o.erase(table, ip)
        self.staged = []

    def submit(self, recs):
        from alaz_b200 import capi
        recs = np.ascontiguousarray(recs, dtype=abi.L7_REC)
        if self.fmt16:
            self.h.submit_packed(*capi.pack_l7(recs))
        else:
            self.h.submit(recs)
        self.oracle_submit(recs)

    def submit_device(self, recs):
        """One device submit of all the records (packed first under fmt16; no duration needs the overflow array)."""
        from alaz_b200 import capi
        recs = np.ascontiguousarray(recs, dtype=abi.L7_REC)
        d = self.h.dev_alloc(max(1, len(recs)) * 32)
        if self.fmt16:
            r16, ovf = capi.pack_l7(recs)
            assert len(ovf) == 0
            self.h.h2d(d, r16)
            self.h.submit_packed_device(d, len(recs))
        else:
            self.h.h2d(d, recs)
            self.h.submit_device(d, len(recs))
        self.h.sync()
        self.h.dev_free(d)
        self.oracle_submit(recs)

    def oracle_submit(self, recs):
        r, idx = oracle_view(recs)
        self.o.process_hosts(r, idx, HOSTS)

    def flush(self, what=""):
        from helpers import edges_equal, explain_diff
        got = self.h.flush()
        exp = self.o.edges()
        self.o.reset_window()
        self.windows += 1
        assert edges_equal(got, exp), f"{what} window {self.windows}: " + explain_diff(got, exp)
        gs, es = self.h.stats(), self.o.stats()
        es["capacity_events"] = 0
        for k in STAT_KEYS:
            assert gs[k] == es[k], (what, k, gs[k], es[k])
        return got

    def probe(self, universe, pod0, svc0, what=""):
        """One window of probe_window records over the universe, flushed and compared."""
        self.submit(probe_window(universe, pod0, svc0))
        return self.flush(what)
