"""GPU: the endpoint table and the pod-address filter on constructed layouts (tests/ep_tables.py). Every case ends in
windows of `probe_window` records, each compared per edge, bit for bit, with the oracle, and the stats with the
oracle's. The table cases run on the default plan (32-B and packed records), on ALZ_CFG_EAGER_JOIN and on
ALZ_CFG_NO_SMEM_CACHE; the filter is read by the default plan only."""
import time

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings, strategies as st

import ep_tables as et
import sock_lines as sl
from alaz_b200 import abi
from ep_tables import ID_MAX, Both
from helpers import edges_equal, explain_diff

pytestmark = pytest.mark.gpu

POD, SVC = abi.TABLE_POD, abi.TABLE_SVC
PLANS = {"v8": (0, False), "v8_packed": (0, True), "eager": (abi.CFG_EAGER_JOIN, False),
         "v1": (abi.CFG_NO_SMEM_CACHE, False)}
FILTER_PLANS = ["v8", "v8_packed"]


def both(plan, max_endpoints, **kw):
    flags, fmt16 = PLANS[plan]
    return Both(max_endpoints, flags=flags, fmt16=fmt16, **kw)


def ends(cap, avoid=()):
    """A pod and a service homed away from the slots the layouts use (around 0 and cap - 4..cap - 1)."""
    p = et.with_home(cap, cap // 2 - 7, 1, seed=91, avoid=avoid)[0]
    s = et.with_home(cap, cap // 2 - 5, 1, seed=92, avoid=list(avoid) + [p])[0]
    return p, s


def load(b, ips, first_id=0, svc_every=2):
    """ips as pods, every svc_every-th also as a service (ids first_id + k and first_id + k + 1000)."""
    for k, ip in enumerate(ips):
        b.upsert(POD, ip, first_id + k)
        if k % svc_every == svc_every - 1:
            b.upsert(SVC, ip, first_id + k + 1000)


# ---- 1. full table, one home -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("plan", list(PLANS))
def test_full_table_with_one_home(plan):
    """64 endpoints (128 slots) all homed at slot 120: the chain runs 120..127, 0..55 and an absent address homed there
    walks all 64 entries. A new address is refused; an update and an erase plus an add in one commit are not."""
    b = both(plan, 64)
    cap = b.m.cap
    addrs = et.with_home(cap, 120, 70, seed=5)
    members, extra = addrs[:64], addrs[64:]
    b.upsert(POD, members[0], 0)
    b.upsert(SVC, members[1], 1)
    load(b, members[2:], first_id=2, svc_every=3)
    b.commit()
    assert b.m.slot_of(members[63]) == 55 and b.m.probes(extra[0]) == 65
    pod0, svc0 = members[0], members[1]
    uni = members + extra + [0, et.M32]
    b.probe(uni, pod0, svc0, "full")
    b.upsert(POD, extra[0], 99, expect=abi.E_CAPACITY)
    b.upsert(SVC, extra[0], 99, expect=abi.E_CAPACITY)
    b.upsert(POD, members[40], ID_MAX)                      # update of a present address
    b.upsert(SVC, members[41], 7)
    b.commit()
    b.probe(uni, pod0, svc0, "updates")
    b.erase(POD, members[20])
    b.erase(SVC, members[20])
    b.upsert(POD, extra[1], 77)
    b.commit()
    assert b.m.slot_of(extra[1]) is not None and b.m.slot_of(members[20]) is None
    b.probe(uni, pod0, svc0, "erase + add")
    b.close()


# ---- 2. chain across the end -------------------------------------------------------------------------------------------

def wrapped_setup(b):
    cap = b.m.cap
    chain, low, order = et.wrapped_chain(cap)
    pod0, svc0 = ends(cap, order)
    b.upsert(POD, pod0, 500)
    b.upsert(SVC, svc0, 501)
    load(b, order)
    b.commit()
    absent = [et.with_home(cap, s, 2, seed=40 + s, avoid=order)[1] for s in (cap - 4, cap - 1, 0, 1, 2, 3)]
    return chain, low, order, pod0, svc0, order + absent + [0, et.M32]


@pytest.mark.parametrize("plan", list(PLANS))
def test_chain_across_the_end(plan):
    """Deletes of the head, of an entry before the wrap (entries after the wrap move back across the end, low[3]
    stays at its home) and of an entry after the wrap, each in its own commit, then all of them in one."""
    b = both(plan, 32)
    chain, low, order, pod0, svc0, uni = wrapped_setup(b)
    cap = b.m.cap
    assert b.m.slot_of(chain[4]) == 1 and b.m.slot_of(low[0]) == 0 and b.m.slot_of(low[3]) == 3
    b.probe(uni, pod0, svc0, "loaded")
    # the head: the free slot reaches cap - 1 with low[0] at slot 0, which stays (the wrapped branch of the rule)
    for ip, check in ((chain[0], lambda: b.m.slot_of(chain[1]) == cap - 4 and b.m.slot_of(low[0]) == 0),
                      (chain[2], lambda: b.m.slot_of(chain[5]) == cap - 1 and b.m.slot_of(low[3]) == 3),
                      (low[0], lambda: b.m.slot_of(low[3]) == 3)):
        b.erase(POD, ip)
        b.erase(SVC, ip)
        b.commit()
        assert check()
        b.probe(uni, pod0, svc0, f"erase {ip:#x}")
    for ip in order:
        b.erase(POD, ip)
        b.erase(SVC, ip)
    b.commit()
    assert b.m.occ.sum() == 2
    b.probe(uni, pod0, svc0, "all erased")
    b.close()


# ---- 3. merged chains --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("plan", list(PLANS))
def test_merged_chains(plan):
    b = both(plan, 32)
    cap = b.m.cap
    a, c, order = et.merged_chains(cap, 40, 6)
    pod0, svc0 = ends(cap, order)
    b.upsert(POD, pod0, 500)
    b.upsert(SVC, svc0, 501)
    load(b, order)
    b.commit()
    uni = order + et.with_home(cap, 40, 8, seed=2)[6:] + et.with_home(cap, 41, 8, seed=3, avoid=a)[6:] + [0]
    b.probe(uni, pod0, svc0, "merged")
    b.erase(POD, a[0])
    b.erase(SVC, a[0])
    b.commit()
    assert b.m.slot_of(c[0]) == 41 and b.m.slot_of(a[1]) == 40          # c[0]'s home is past the free slot
    b.probe(uni, pod0, svc0, "erase a[0]")
    b.erase(POD, c[1])
    b.commit()
    b.probe(uni, pod0, svc0, "erase c[1]")
    b.upsert(POD, a[0], 600)
    b.upsert(POD, c[1], 601)
    b.commit()
    b.probe(uni, pod0, svc0, "re-added")
    b.close()


# ---- 4. long chain -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("plan", list(PLANS))
def test_long_chain_of_4096(plan):
    """4096 addresses on one home of a 2^14-slot table; ep_lookup has no probe bound, and an absent address homed there
    walks the whole chain (on the eager plan once per event)."""
    b = both(plan, 1 << 13, model=False, max_pairs=1 << 16)
    cap = et.ep_cap(1 << 13)
    addrs = et.with_home(cap, 100, 4096 + 64, seed=8)
    members, absent = addrs[:4096], addrs[4096:]
    b.upsert_batch(POD, members, np.arange(4096))
    b.upsert_batch(SVC, members[1::2], np.arange(1, 4096, 2) + 10000)
    b.commit()
    uni = members + absent + [0, et.M32]
    t0 = time.perf_counter()
    b.probe(uni, members[4095], members[4093], "long chain")
    dt = time.perf_counter() - t0
    print(f"long chain, {plan}: window of {5 * len(uni)} records over a 4096-entry chain: {dt * 1e3:.1f} ms")
    b.erase(POD, members[0])                                  # the head: all 4095 successors move back one slot
    b.commit()
    b.probe(uni, members[4095], members[4093], "head erased")
    b.close()


# ---- 5. identity cases -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("plan", list(PLANS))
def test_pod_and_service_on_one_address(plan):
    b = both(plan, 16)
    cap = b.m.cap
    x, y, pod0, svc0 = et.random_addrs(4, seed=11)
    b.upsert(POD, pod0, 1)
    b.upsert(SVC, svc0, 2)
    b.upsert(SVC, x, 10)                                      # x: service first, then pod
    b.upsert(POD, y, 20)                                      # y: pod first, then service
    b.commit()
    b.upsert(POD, x, 11)
    b.upsert(SVC, y, 21)
    b.commit()
    uni = [x, y, pod0, svc0] + et.with_home(cap, int(et.home(x, cap)), 2, seed=3, avoid=[x, y, pod0, svc0])
    b.probe(uni, pod0, svc0, "both kinds")
    for table, ip in ((SVC, x), (POD, y), (POD, x), (SVC, y)):
        b.erase(table, ip)
        b.commit()
        b.probe(uni, pod0, svc0, f"erase {table} {ip:#x}")
    b.close()


@pytest.mark.parametrize("plan", list(PLANS))
def test_ids_reuse_and_staging(plan):
    """In-place updates to ids 0 and 2^29 - 1, a pod address taken by a new pod id, an address upserted and erased in
    one commit, a pod at 0.0.0.0, an id of 2^29 refused, and staged changes invisible to a submit made before the
    commit."""
    b = both(plan, 16)
    p, q, s, n, z, pod0, svc0 = et.random_addrs(7, seed=12)
    b.upsert(POD, pod0, 1)
    b.upsert(SVC, svc0, 2)
    b.upsert(POD, p, 0)
    b.upsert(SVC, s, ID_MAX)
    b.upsert(POD, 0, 5)
    b.upsert(POD, q, 6)
    b.upsert(POD, p, ID_MAX + 1, expect=abi.E_INVAL)
    b.commit()
    uni = [p, q, s, n, z, pod0, svc0, 0, et.M32]
    b.probe(uni, pod0, svc0, "ids")
    b.upsert(POD, p, ID_MAX)
    b.upsert(SVC, s, 0)
    b.commit()
    b.probe(uni, pod0, svc0, "in-place")
    b.erase(POD, q)                                           # same address, new pod
    b.upsert(POD, q, 66)
    b.upsert(POD, n, 70)                                      # here and gone in one commit
    b.erase(POD, n)
    b.commit()
    assert b.m.slot_of(n) is None
    b.probe(uni, pod0, svc0, "reuse")
    b.upsert(POD, z, 80)                                      # staged: the submit below does not see it
    b.erase(POD, 0)
    b.submit(et.probe_window(uni, pod0, svc0))
    b.commit()
    b.submit(et.probe_window(uni, pod0, svc0))
    b.flush("staged then committed")
    b.close()


def test_upsert_batch_applies_the_prefix_before_the_first_failure():
    b = Both(8)
    ips = et.random_addrs(12, seed=13)
    ids = np.arange(12, dtype=np.uint64)
    ids[3] = ID_MAX + 1
    assert b.upsert_batch(POD, ips, ids) == abi.E_INVAL
    b.commit()
    assert sorted(b.m.committed()) == sorted(ips[:3])
    assert b.upsert_batch(POD, ips[3:], np.arange(3, 12)) == abi.E_CAPACITY      # 8 endpoints: 5 more fit
    b.commit()
    assert sorted(b.m.committed()) == sorted(ips[:8])
    b.probe(ips, ips[0], ips[1], "batch prefix")
    b.close()


# ---- 6. churn at load 0.5 ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("plan", list(PLANS))
def test_churn_at_load_one_half(plan):
    """2^20 endpoints in a 2^21-slot table, loaded with one batch (the first patch, 2^20 slots, grows the patch buffer);
    then commits of 10^3 and 10^5 changes, each followed by a window."""
    n = 1 << 20
    b = both(plan, n, model=False, max_pairs=1 << 16)
    rng = np.random.default_rng(14)
    ips = np.array(et.random_addrs(n + 60_000, seed=14), np.uint32)
    live, spare = ips[:n], list(ips[n:])
    b.upsert_batch(POD, live[: n // 2], np.arange(n // 2))
    b.upsert_batch(SVC, live[n // 2:], np.arange(n // 2))
    b.commit()
    pod0, svc0 = int(live[0]), int(live[-1])
    absent = spare[-2000:]
    b.probe([int(x) for x in rng.choice(live, 3000)] + absent, pod0, svc0, "loaded")
    live = list(live[1:-1])
    for k in (1000, 100_000):
        idx = rng.permutation(len(live))
        gone, upd = [live[i] for i in idx[: k // 4]], [live[i] for i in idx[k // 4: k // 2]]
        new = [spare.pop() for _ in range(k // 2 - k // 4)]
        for ip in gone:
            b.erase(POD, ip)
            b.erase(SVC, ip)
        for j, ip in enumerate(upd):
            b.upsert(POD if j % 2 else SVC, ip, (7 * j) % ID_MAX)
        for j, ip in enumerate(new):
            b.upsert(SVC if j % 3 else POD, ip, j)
        b.commit()
        sample = gone[:1000] + upd[:1000] + new[:1000] + [live[i] for i in idx[k // 2: k // 2 + 1000]] + absent
        b.probe([int(x) for x in sample], pod0, svc0, f"{k} changes")
        gone_set = set(gone)
        live = [x for x in live if x not in gone_set] + new
    b.close()


# ---- 7.-9. the filter --------------------------------------------------------------------------------------------------

def shared_bit_pairs():
    """(kept, erased) pod pairs: same b1, same b2, b1 of one = b2 of the other, a pod with b1 == b2 and one sharing it."""
    pairs = [tuple(et.with_b1(0x0F0F3, 2, seed=1)), tuple(et.with_b2(0x1A0A1, 2, seed=2))]
    a = et.random_addrs(1, seed=3)[0]
    pairs.append((a, et.with_b2(int(et.filter_bits(a)[0]), 1, seed=4, avoid=[a])[0]))
    e = et.equal_bits(1, seed=5)[0]
    pairs.append((et.with_b1(int(et.filter_bits(e)[0]), 1, seed=6, avoid=[e])[0], e))
    pairs.append((e, pairs[-1][0]))
    return pairs


@pytest.mark.parametrize("plan", FILTER_PLANS)
def test_pods_that_share_filter_bits(plan):
    pairs = shared_bit_pairs()
    b = both(plan, 64)
    pod0, svc0 = et.random_addrs(2, seed=7, avoid=[x for p in pairs for x in p])
    b.upsert(POD, pod0, 1)
    b.upsert(SVC, svc0, 2)
    b.commit()
    for k, (keep, gone) in enumerate(pairs):
        for ip, i in ((keep, 10 * k), (gone, 10 * k + 1)):
            if b.m.host.get(ip, [None])[0] is None:
                b.upsert(POD, ip, i)
        b.commit()
        uni = [keep, gone, pod0]
        b.probe(uni, pod0, svc0, f"pair {k}")
        b.erase(POD, gone)
        b.commit()
        assert b.m.maybe_pod(keep)
        b.probe(uni, pod0, svc0, f"pair {k}, one erased")
        b.upsert(POD, gone, 10 * k + 2)
        b.commit()
        b.probe(uni, pod0, svc0, f"pair {k}, re-added")
    b.close()


@pytest.mark.parametrize("plan", FILTER_PLANS)
def test_saturated_filter_bit(plan):
    """300 pods set one bit (its counter stays at 255): erasing 299 leaves the last one resolving; after all are erased
    a new pod that shares only that bit resolves."""
    pods = et.with_b2(0x0BEEF, 302, seed=9)
    pods, newcomer, never = pods[:300], pods[300], pods[301]
    b = both(plan, 512)
    pod0, svc0 = et.random_addrs(2, seed=10, avoid=pods + [newcomer, never])
    b.upsert(POD, pod0, 1)
    b.upsert(SVC, svc0, 2)
    b.upsert_batch(POD, pods, np.arange(300) + 100)
    b.commit()
    assert b.m.filter.cnt[0x0BEEF] == 255
    uni = pods[:8] + pods[-8:] + [newcomer, never, pod0]
    b.probe(uni, pod0, svc0, "300 pods")
    for ip in pods[:299]:
        b.erase(POD, ip)
    b.commit()
    b.probe(uni, pod0, svc0, "299 erased")
    b.erase(POD, pods[299])
    b.upsert(POD, newcomer, 5)
    b.commit()
    assert b.m.filter.cnt[0x0BEEF] == 255 and b.m.maybe_pod(newcomer)
    b.probe(uni, pod0, svc0, "all erased, newcomer")
    b.close()


def fp_records(src, dst, rng, n):
    """n records from src to dst (cycled), forward, reversed and Host-keyed."""
    i = np.arange(n)
    s = np.asarray(src, np.uint32)[i % len(src)]
    d = np.asarray(dst, np.uint32)[(i // len(src)) % len(dst)]
    kind = rng.integers(0, 3, n)
    r = et.records(s, d, rng.integers(1, 1 << 30, n, dtype=np.uint64), status=rng.choice([200, 503], n))
    r["protocol"][kind == 1], r["method_flags"][kind == 1] = abi.PROTO_AMQP, abi.AMQP_DELIVER
    r["protocol"][kind == 2] |= abi.PROTO_F_HOSTKEY
    r["daddr"][kind == 2] = i[kind == 2] % 4
    return r


@pytest.mark.parametrize("plan", FILTER_PLANS)
def test_false_positives_at_volume(plan):
    """Sources that pass the filter and are no pods (two of them services) reach the dictionary's pod check and are
    counted unresolved, exactly: 2^20 events of a few such pairs in one device submit, then every event a new pair,
    then one such source becomes a pod by a commit in the middle of a window and leaves again."""
    rng = np.random.default_rng(15)
    pods = et.random_addrs(200, seed=16)
    fp = et.false_positives(pods, 8)
    b = both(plan, 512, max_pairs=1 << 12)
    load(b, pods, svc_every=5)
    b.upsert(SVC, fp[0], 900)
    b.upsert(SVC, fp[1], 901)
    b.commit()
    assert all(b.m.maybe_pod(a) for a in fp) and not any(b.m.host.get(a, [None])[0] is not None for a in fp)
    few = fp_records(fp[:4], pods[:3], rng, 1 << 20)
    few = np.concatenate([few, fp_records(pods[:5], fp[:2] + pods[5:7], rng, 5000)])
    b.submit_device(few)
    st0 = b.h.stats()
    b.flush("a few pairs, 2^20 events")
    assert b.o.stats()["src_unresolved"] >= 1 << 20 and st0["capacity_events"] == 0
    new = fp_records(fp, et.random_addrs(1 << 13, seed=17, avoid=pods + fp), rng, 1 << 16)
    b.submit(new)
    b.flush("every event a new pair")
    mover = fp[2]
    b.submit(fp_records([mover, pods[0]], pods[:4], rng, 4000))
    b.upsert(POD, mover, 777)
    b.commit()
    b.submit(fp_records([mover, pods[0]], pods[:4], rng, 4000))
    b.erase(POD, mover)
    b.commit()
    b.submit(fp_records([mover, pods[0]], pods[:4], rng, 4000))
    b.flush("a source joins and leaves mid-window")
    b.probe(fp + pods[:4], pods[0], pods[4], "probe")
    b.close()


# ---- 10. window clock --------------------------------------------------------------------------------------------------

def test_held_records_keep_their_resolution_across_a_chain_shift():
    """Records held for the next window have chain members at both ends; a commit erases some members, gives others
    new ids and shifts the rest of the chain. The held records are resolved before the patch."""
    from test_gpu_window_clock import Pair, recs_at
    W = 1000
    p = Pair(0, 0, W)
    cap = et.ep_cap(256)                                      # the Pair's handle has 256 endpoints
    chain = et.with_home(cap, cap - 3, 10, seed=18) + et.with_home(cap, 0, 4, seed=19)
    for k, ip in enumerate(chain):
        p.upsert(POD, ip, 300 + k)
        if k % 3 == 0:
            p.upsert(SVC, ip, 400 + k)
    p.commit()
    rng = np.random.default_rng(20)
    src = np.array(chain * 30, np.uint32)
    dst = np.array(chain[::-1] * 30, np.uint32)
    p.submit(recs_at([3 * W + 1] * 20 + [4 * W + 5] * (len(src) - 20), rng, src=src, dst=dst))
    for ip in chain[:3]:
        p.erase(POD, ip)                                      # the head of the chain: the rest shift back
    for k, ip in enumerate(chain[5:9]):
        p.upsert(POD, ip, 700 + k)
    p.erase(SVC, chain[9])
    p.upsert(SVC, chain[4], 999)
    p.commit()
    p.submit(recs_at([4 * W + 6] * 200, rng, src=src[:200], dst=dst[:200]))
    p.flush("window 3")
    p.fold()
    p.flush("window 4")
    p.close()


# ---- 11./12. alive export and joins ------------------------------------------------------------------------------------

def _lines_over(b, ips, pod0):
    """One open line per address as the source, and one from pod0 to it."""
    for k, ip in enumerate(ips):
        b.tcp(sl.opened(9, 2 * k, 100, saddr=ip, daddr=pod0, sport=30000 + k, dport=80))
        b.tcp(sl.opened(9, 2 * k + 1, 100, saddr=pod0, daddr=ip, sport=31000 + k, dport=81))


def test_alive_export_over_wrapped_and_merged_chains():
    b = sl.Both(max_endpoints=32)
    cap = et.ep_cap(32)
    chain, low, order = et.wrapped_chain(cap)
    a, c, merged = et.merged_chains(cap, 40, 4, seed=30)
    pod0, _ = ends(cap, order + merged)
    absent = [et.with_home(cap, s, 2, seed=40 + s, avoid=order)[1] for s in (cap - 4, 0, 3)] + \
        [et.with_home(cap, 40, 6, seed=30)[5]]
    b.upsert(POD, pod0, 1)
    for k, ip in enumerate(order + merged):
        b.upsert(POD if k % 3 else SVC, ip, 10 + k)
    b.commit()
    _lines_over(b, order + merged + absent, pod0)
    b.alive()
    for group in ([chain[0]], [chain[2]], [low[0]], [a[0]], [c[1]], order + merged):
        for ip in group:
            b.erase(POD, ip)
            b.erase(SVC, ip)
        b.commit()
        b.alive()
    b.close()


def test_joined_records_resolve_through_the_chain():
    b = sl.Both(max_endpoints=32)
    cap = et.ep_cap(32)
    chain, low, order = et.wrapped_chain(cap)
    pod0, svc0 = ends(cap, order)
    b.upsert(POD, pod0, 1)
    b.upsert(SVC, svc0, 2)
    for k, ip in enumerate(order):
        b.upsert(POD if k % 2 else SVC, ip, 10 + k)
    b.commit()
    keys = [(9, k) for k in range(len(order))]
    for (pid, fd), ip in zip(keys, order):
        b.tcp(sl.opened(pid, fd, 100, saddr=ip, daddr=order[(fd + 5) % len(order)], sport=30000 + fd, dport=80))
    n = 4 * len(keys)
    recs = et.records(0, 0, 1000 + np.arange(n) * 77, status=np.where(np.arange(n) % 3 == 0, 503, 200))
    q = sl.query([k[0] for k in keys] * 4, [k[1] for k in keys] * 4, [150] * n)
    joined, nj = b.join(recs, q, now=5)
    assert nj == n
    b.tables.process(joined)
    b.erase(POD, chain[1])                                    # chain[1] leaves: the chain shifts back across the end
    b.erase(SVC, chain[1])
    b.upsert(POD, chain[5], 60)
    b.commit()
    joined, nj = b.join(recs, q, now=6)
    b.tables.process(joined)
    got, exp = b.h.flush(), b.tables.edges()
    assert edges_equal(got, exp), explain_diff(got, exp)
    b.close()


# ---- 13. random sequences ----------------------------------------------------------------------------------------------

U48 = None


def _universe():
    global U48
    if U48 is None:
        U48 = [a for s in (61, 62, 63) for a in et.with_home(64, s, 16, seed=s)]
    return U48


_op = st.one_of(
    st.tuples(st.just("u"), st.integers(0, 1), st.integers(0, 47), st.sampled_from([0, 1, 5, ID_MAX])),
    st.tuples(st.just("e"), st.integers(0, 1), st.integers(0, 47)),
    st.tuples(st.just("c")),
    st.tuples(st.just("s"), st.lists(st.integers(0, 47), min_size=1, max_size=12), st.integers(0, 47)),
    st.tuples(st.just("f")),
)


@settings(max_examples=25, deadline=None, suppress_health_check=[HealthCheck.too_slow])
@given(st.lists(_op, min_size=1, max_size=40))
def test_random_operation_sequences(ops):
    """Upserts (refused past 32 endpoints), erases, commits, submits and flushes on 48 addresses homed at slots 61..63
    of a 64-slot table: chains that merge and wrap. Device and oracle are compared at every flush."""
    U = _universe()
    b = Both(32)
    for op in ops:
        if op[0] == "u":
            full = U[op[2]] not in b.m.host and len(b.m.host) >= 32
            b.upsert(op[1], U[op[2]], op[3], expect=abi.E_CAPACITY if full else abi.OK)
        elif op[0] == "e":
            b.erase(op[1], U[op[2]])
        elif op[0] == "c":
            b.commit()
        elif op[0] == "s":
            b.submit(et.probe_window([U[i] for i in op[1]], U[op[2]], U[(op[2] + 1) % 48]))
        else:
            b.flush("random")
    b.commit()
    b.submit(et.probe_window(U + [0], U[0], U[1]))
    b.flush("last")
    b.close()
