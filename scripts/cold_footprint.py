#!/usr/bin/env python
"""How much of the L2 the ingest kernel's cold tier touches in one window of the bench stream (CPU only).

Replays the kernel's tier rules on the synthetic stream of `bench.py` (seed 0xA1A20001): the hot list is built from
window 0 as hot_emit_kernel builds it (the kPreload rows with the most events, each with the 16-bucket window that held
most of them), then every event of window 1 is put in its tier. For the events that stay cold it counts the distinct
128-byte lines of the pair dictionaries (home slots) and of the pair rows (512-B rows, a line per 16 buckets), for two
layouts:
  old  separate forward and reversed dictionaries (2·max_pairs and max_pairs/2 slots), only forward pairs in the hot list
  new  one slot per socket pair for both directions, forward and reversed pairs in the hot list
Per-CTA details (first-come rows, tier-S replicas, 16-bit spills) are left out. About three minutes at full size:
  python scripts/cold_footprint.py [--services 10000] [--events 100000000]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import oracle_lib as ol  # noqa: E402
from alaz_b200 import abi  # noqa: E402
from ingest_streams import latency_bucket, next_pow2, pair_hash  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--services", type=int, default=10_000)
ap.add_argument("--events", type=int, default=100_000_000)
ap.add_argument("--max-pairs", type=int, default=1 << 20)   # bench.py's at config 2
ap.add_argument("--preload", type=int, default=1008)        # Layout<16, 8>::kPreload
a = ap.parse_args()
N, CH = a.events, min(a.events, 10_000_000)
LINE = 128
t = ol.Topo(a.services, seed=0xA1A20001)
pods = np.sort(np.asarray(t.pod_ip, np.uint32))
B64 = np.array([latency_bucket(1 << k) for k in range(64)])


def buckets(d):
    """latency_bucket per duration: from the octave and the bit below it."""
    d = d.astype(np.uint64)
    o = np.zeros(len(d), np.int64)
    for s in (32, 16, 8, 4, 2, 1):
        m = (d >> np.uint64(o + s)) != 0
        o = np.where(m, o + s, o)
    sub = (d >> np.maximum(o - 1, 0).astype(np.uint64)) & np.uint64(1)
    b = 2 * (o - 8) + sub.astype(np.int64)
    return np.where(d < 256, 0, np.where(o >= 40, abi.NB - 1, b))


def classify(first, n):
    """key, kind (0 forward, 1 reversed), bucket of the events that build a row from a pod source (Host-keyed rows
    do not occur in this stream)."""
    ev = t.events(first, n)
    p, mf = ev["protocol"].astype(np.int64), ev["method_flags"].astype(np.int64)
    m = mf & abi.MF_METHOD_MASK
    row = np.isin(p, [abi.PROTO_HTTP, abi.PROTO_AMQP, abi.PROTO_REDIS]) | (
        np.isin(p, [abi.PROTO_POSTGRES, abi.PROTO_MYSQL, abi.PROTO_MONGO]) & ((mf & abi.MF_PAYLOAD_REJECT) == 0))
    rev = ((p == abi.PROTO_AMQP) & (m == abi.AMQP_DELIVER)) | ((p == abi.PROTO_REDIS) & (m == abi.REDIS_PUSHED_EVENT))
    keep = row & np.isin(ev["saddr"], pods)
    key = (ev["daddr"].astype(np.uint64) << np.uint64(32)) | ev["saddr"].astype(np.uint64)
    return key[keep], rev[keep].astype(np.int64), buckets(ev["duration_ns"][keep]), int(len(ev))


assert [int(x) for x in buckets(np.array([1 << k for k in range(64)], np.uint64))] == B64.tolist()

# window 0: events and best 16-bucket window (base a multiple of 4, <= 48) of every (pair, kind)
ks, kd, bs = [], [], []
for f in range(0, N, CH):
    k, d, b, _ = classify(f, CH)
    ks.append(k); kd.append(d); bs.append(b)
k0, d0, b0 = np.concatenate(ks), np.concatenate(kd), np.concatenate(bs)
ids, inv = np.unique(np.stack([k0, d0.astype(np.uint64)], axis=1), axis=0, return_inverse=True)
inv = inv.reshape(-1)
cnt = np.bincount(inv)
h = np.zeros((len(ids), 64), np.int64)
np.add.at(h, (inv, b0), 1)
cs = np.cumsum(np.pad(h, ((0, 0), (1, 0))), axis=1)
base = np.stack([cs[:, 4 * j + 16] - cs[:, 4 * j] for j in range(13)], axis=1).argmax(axis=1) * 4
del h, cs, k0, d0, b0, inv
fwd = np.nonzero(ids[:, 1] == 0)[0]
hot = {"old": fwd[np.argsort(-cnt[fwd], kind="stable")[: a.preload]],
       "new": np.argsort(-cnt, kind="stable")[: a.preload]}

# window 1: tier of every event under each layout
fcap = next_pow2(2 * a.max_pairs)
masks = {"old": (fcap - 1, max(1024, fcap >> 2) - 1), "new": (fcap - 1, fcap - 1)}
res = {}
for lay in ("old", "new"):
    hk, hb = ids[hot[lay]], base[hot[lay]]
    per_kind = []
    for kind in (0, 1):                                         # hot (key, window base) of each kind, sorted by key
        s = hk[:, 1] == kind
        o = np.argsort(hk[s, 0])
        per_kind.append((hk[s, 0][o], hb[s][o]))
    tot = dict(events=0, hot=0, cold_fwd=0, cold_rev=0)
    dict_lines, row_lines = set(), {0: set(), 1: set()}
    for f in range(N, 2 * N, CH):
        k, d, b, n = classify(f, CH)
        tot["events"] += n
        hit = np.zeros(len(k), bool)
        for kind, (hkk, hbb) in enumerate(per_kind):
            if len(hkk) == 0:
                continue
            pos = np.minimum(np.searchsorted(hkk, k), len(hkk) - 1)
            hit |= (d == kind) & (hkk[pos] == k) & (b >= hbb[pos]) & (b < hbb[pos] + 16)
        tot["hot"] += int(hit.sum())
        c = ~hit
        tot["cold_fwd"] += int((c & (d == 0)).sum()); tot["cold_rev"] += int((c & (d == 1)).sum())
        kc, dc, bc = k[c], d[c], b[c]
        slot = pair_hash(kc).astype(np.int64) & np.where(dc == 1, masks[lay][1], masks[lay][0])
        table = dc if lay == "old" else np.zeros_like(dc)       # old: the two kinds live in different tables
        dict_lines.update(np.unique(table * (1 << 40) + slot // (LINE // 16)).tolist())
        for kind in (0, 1):
            s = dc == kind
            u = np.unique(np.stack([kc[s], (bc[s] // 16).astype(np.uint64)], axis=1), axis=0)
            row_lines[kind].update(map(tuple, u.tolist()))
    res[lay] = (tot, len(dict_lines), len(row_lines[0]), len(row_lines[1]))

for lay, (tot, nd, nf, nr) in res.items():
    e = tot["events"]
    print(f"{lay}: hot {tot['hot'] / e:.4f}, cold forward {tot['cold_fwd'] / e:.4f}, cold reversed "
          f"{tot['cold_rev'] / e:.4f} of {e} events")
    print(f"  distinct 128-B lines: dictionary {nd} ({nd * LINE / 1e6:.1f} MB), forward rows {nf} "
          f"({nf * LINE / 1e6:.1f} MB), reversed rows {nr} ({nr * LINE / 1e6:.1f} MB), "
          f"total {(nd + nf + nr) * LINE / 1e6:.1f} MB")
