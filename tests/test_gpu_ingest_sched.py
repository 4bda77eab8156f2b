"""GPU: the ingest kernel's chunk schedule (alaz_b200/csrc/alz_ingest.cu, ChunkSched; host model in sched_model.py).

The first 5/8 of a launch's rounds of 64-record chunks keep the static map (chunk r * stride + w to warp w); the
rest are claimed from a per-handle cursor that is zeroed before every launch. In every stream here each chunk has
its own socket pair and latency sum (`numbered`), so a chunk taken twice or never changes some edge's count or
latency sum. Every case is compared per edge, bit for bit, with the oracle, on the three instantiations of the
kernel: 32-B records, 32-B records under a window clock (every record in the open window), 16-B packed records."""
import numpy as np
import pytest

import ingest_streams as ist
import sched_model as sm
from alaz_b200 import abi, capi
from helpers import edges_equal, explain_diff

pytestmark = pytest.mark.gpu

VARIANTS = ["rec32", "rec32_clock", "rec16"]
WIN_NS = 1 << 40
POD = [abi.ip("10.0.0.%d" % i) for i in range(1, 40)]
SVC = abi.ip("172.16.0.1")
TABLES = [(abi.TABLE_POD, POD, list(range(1, len(POD) + 1))), (abi.TABLE_SVC, [SVC], [7])]


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def handle(variant, max_pairs=1 << 16):
    h = capi.Handle(max_endpoints=256, max_pairs=max_pairs)
    if variant == "rec32_clock":
        h.window_clock(0, 0, WIN_NS)
    for tab, ips, ids in TABLES:
        h.upsert_batch(tab, np.asarray(ips, np.uint32), np.asarray(ids, np.uint32))
    h.commit()
    return h


def numbered(n, first=0):
    """n records; chunk j (records 64j .. 64j + 63 of the stream, counted from `first`) is pair
    (POD[j % 37], POD[(j // 37) % 39]) with durations 4096 j + 1000 + position: a chunk read twice or never shows
    in the count and the latency sum of its edge, whichever chunk it collides with."""
    i = first + np.arange(n, dtype=np.int64)
    j = i // sm.CHUNK
    pods = np.asarray(POD, np.uint64)
    r = ist.records(pods[j % 37], pods[(j // 37) % 39], (4096 * j + 1000 + i % sm.CHUNK).astype(np.uint64))
    r["write_time_ns"] = i % 1000
    return r


def to_device(h, variant, parts):
    """Concatenation of `parts` (32-B record arrays) in device memory, packed for rec16; returns (ptr, n)."""
    recs = np.concatenate(parts) if len(parts) > 1 else parts[0]
    if variant == "rec16":
        recs, ovf = capi.pack_l7(recs)
        assert len(ovf) == 0
    p = h.dev_alloc(max(1, recs.nbytes))
    step = 1 << 22
    for k in range(0, len(recs), step):
        h.h2d(p + k * recs.itemsize, recs[k:k + step])
    return p, len(recs)


def submit(h, variant, p, n):
    if variant == "rec16":
        h.submit_packed_device(p, n)
    else:
        h.submit_device(p, n)


def check(h, exp, est):
    got = h.flush()
    assert edges_equal(got, exp), explain_diff(got, exp)
    st = h.stats()
    for k in ist.STAT_KEYS:
        assert st[k] == est[k], (k, st[k], est[k])
    assert st["capacity_events"] == 0


def run_one(variant, n):
    h = handle(variant)
    recs = numbered(n)
    p, m = to_device(h, variant, [recs])
    submit(h, variant, p, m)
    h.sync()
    h.dev_free(p)
    check(h, *ist.oracle_run(TABLES, recs))
    h.close()


def sizes():
    """Record counts as functions of the SM count: ragged sizes, one round +- 1 record and +- 1 chunk, the last
    static and the first claimed chunk (a 3-round launch claims its third round), a partial last chunk among the
    claimed ones, and a grid with more warps than chunks."""
    C = sm.CHUNK
    rnd = lambda s: s * sm.WARPS * C   # noqa: E731
    return {
        "n1": lambda s: 1, "n63": lambda s: 63, "n64": lambda s: 64, "n65": lambda s: 65,
        "more_warps_than_chunks": lambda s: 5 * C + 1,
        "round-1": lambda s: rnd(s) - 1, "round": lambda s: rnd(s), "round+1": lambda s: rnd(s) + 1,
        "round+1chunk": lambda s: rnd(s) + C,
        "2rounds_all_static": lambda s: 2 * rnd(s),
        "first_claimed_chunk": lambda s: 2 * rnd(s) + C, "first_claimed_partial": lambda s: 2 * rnd(s) + 1,
        "second_claimed_chunk": lambda s: 2 * rnd(s) + 2 * C, "3rounds": lambda s: 3 * rnd(s),
        "claimed_partial_last": lambda s: 11 * rnd(s) - 5 * C - 17,
    }


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("case", list(sizes()))
def test_every_chunk_once(variant, case):
    sms = sm_count()
    n = sizes()[case](sms)
    st, d0 = sm.split(n, sms)
    if case.startswith(("first_claimed", "second_claimed", "claimed_partial")):
        assert sm.n_chunks(n) > d0                    # the case reaches the claimed part
    if case == "claimed_partial_last":
        assert n % sm.CHUNK and sm.n_chunks(n) - 1 >= d0
    run_one(variant, n)


@pytest.mark.parametrize("variant", VARIANTS)
def test_back_to_back_launches(variant):
    """Two launches without a flush between them, both with claimed chunks: the second one's claims start over
    at its own first claimed chunk (the cursor is zeroed before each launch)."""
    sms = sm_count()
    rnd = sms * sm.WARPS * sm.CHUNK
    a, b = numbered(11 * rnd - 3 * sm.CHUNK - 5), numbered(3 * rnd + 7, first=20 * rnd)
    h = handle(variant)
    pa, na = to_device(h, variant, [a])
    pb, nb = to_device(h, variant, [b])
    submit(h, variant, pa, na)
    submit(h, variant, pb, nb)
    h.sync()
    h.dev_free(pa)
    h.dev_free(pb)
    check(h, *ist.oracle_run(TABLES, np.concatenate([a, b])))
    h.close()


@pytest.mark.parametrize("variant", ["rec32", "rec16"])
def test_two_handles_two_streams(variant):
    """Two handles (each on its own stream) submit at once; each has its own cursor, so neither takes the
    other's claims. Both launches are issued before either is waited for."""
    sms = sm_count()
    rnd = sms * sm.WARPS * sm.CHUNK
    streams = [numbered(9 * rnd + 33), numbered(6 * rnd - 100, first=40 * rnd)]
    hs = [handle(variant) for _ in streams]
    ptrs = [to_device(h, variant, [r]) for h, r in zip(hs, streams)]
    for h in hs:
        h.sync()
    for k in range(3):                               # three launches each, interleaved on the two streams
        for h, (p, m) in zip(hs, ptrs):
            submit(h, variant, p, m)
    for h, (p, m), r in zip(hs, ptrs, streams):
        h.sync()
        h.dev_free(p)
        exp, est = ist.scaled_oracle(TABLES, r, 3)
        check(h, exp, est)
        h.close()


def merged_oracle(parts):
    """(edges, stats) of the concatenation of tile(pattern, reps) for (pattern, reps) in parts."""
    exp, est = ist.scaled_oracle(TABLES, *parts[0])
    for pat, reps in parts[1:]:
        e, s = ist.scaled_oracle(TABLES, pat, reps)
        at = {ist._key(x): i for i, x in enumerate(exp)}
        new = []
        for x in e:
            i = at.get(ist._key(x))
            if i is None:
                new.append(x)
                continue
            for f in ("count", "err5xx", "lat_sum_ns"):
                exp[f][i] = (int(exp[f][i]) + int(x[f])) & ist.M64
            exp["hist"][i] = ((exp["hist"][i].astype(np.uint64) + x["hist"]) & np.uint64(ist.M32)).astype(np.uint32)
        if new:
            exp = np.concatenate([exp, np.array(new, dtype=abi.EDGE_OUT)])
        est = {k: est[k] + s[k] for k in est}
    return exp, est


@pytest.mark.parametrize("variant", VARIANTS)
def test_spill_in_claimed_part(variant):
    """The 16-bit cell spill, reached only through claimed chunks. 200 rounds: the 125 static ones hold 16 other
    pairs (POD[1..16] -> SVC), the 75 claimed ones only the pair POD[0] -> SVC, 40 events per chunk in bucket 46 and
    24 in bucket 47 (as test_gpu_ingest.two_cell_pattern). That is 75 x 16 x 132 chunks on an H100, 6.3M events in
    bucket 46: more than 132 x 0x7FFF, so at least one CTA spills that cell whatever the claims, and every CTA does
    when they are near even (48,000 events each). The pair is new in this window: each CTA admits a private row for
    it at its first cold event, with most of its rows still free."""
    sms = sm_count()
    rnd = sms * sm.WARPS * sm.CHUNK
    rounds = 200
    st, d0 = sm.split(rounds * rnd, sms)
    assert (st, d0) == (125, 125 * sms * sm.WARPS)
    p = np.arange(64)
    other = ist.records(np.asarray(POD[1:17], np.uint64)[p % 16], SVC, (5000 + 17 * p).astype(np.uint64))
    d = np.where(p < 40, (1 << 31) + 12345 + 1000 * p, (1 << 32) - 1 - 1000 * p)
    assert [ist.latency_bucket(x) for x in d] == [46] * 40 + [47] * 24
    spill = ist.records(POD[0], SVC, d.astype(np.uint64), status=np.where(np.isin(p, [3, 11, 43, 60]), 503, 200))
    n_other, n_spill = d0, rounds * sms * sm.WARPS - d0           # chunks
    assert n_spill * 40 > sms * (ist.CELL_SPILL - 1)
    for r in (other, spill):
        r["write_time_ns"] = np.arange(64) % 1000
    h = handle(variant)
    other_p = capi.pack_l7(other)[0] if variant == "rec16" else other
    spill_p = capi.pack_l7(spill)[0] if variant == "rec16" else spill
    b = other_p.itemsize
    ptr = h.dev_alloc((n_other + n_spill) * 64 * b)
    group = 1 << 16
    for base, tile, count in ((0, other_p, n_other), (n_other, spill_p, n_spill)):
        block = np.tile(tile, group)
        for k in range(0, count, group):
            h.h2d(ptr + (base + k) * 64 * b, block[: min(group, count - k) * 64])
    submit(h, variant, ptr, (n_other + n_spill) * 64)
    h.sync()
    h.dev_free(ptr)
    check(h, *merged_oracle([(other, n_other), (spill, n_spill)]))
    h.close()
