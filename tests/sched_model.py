"""Host model of the ingest kernel's chunk schedule (alaz_b200/csrc/alz_ingest.cu, ChunkSched).

A chunk is 64 consecutive records. In the first rounds, warp w of the grid takes chunk r * stride + w in round r
(stride = warps in the grid). The chunks after the static rounds are claimed: claimed chunk d0 + j belongs to warp
slot j mod WARPS (the warp's index in its CTA), and slot p's chunks are handed out CLAIM at a time from cursor p,
which is zero at the start of the launch. Lane 0 claims CLAIM chunks before its first chunk is needed; each warp
asks for its next chunk once per loop iteration, two iterations before it reads it."""
import random

CHUNK = 64
WARPS = 16
DYN_EIGHTHS = 3   # the last 3/8 of the rounds are claimed
CLAIM = 2         # chunks per claim


def n_chunks(n):
    return (n + CHUNK - 1) // CHUNK


def split(n, sms):
    """(static rounds, first claimed chunk) of a launch of n records on `sms` CTAs."""
    stride = sms * WARPS
    rounds = (n_chunks(n) + stride - 1) // stride
    st = rounds - rounds * DYN_EIGHTHS // 8
    return st, st * stride


class Warp:
    """One warp's ChunkSched, step for step (every lane holds the same state; `claim` is lane 0's register)."""

    def __init__(self, n, sms, g, cursors):
        self.cursor = cursors[g % WARPS]      # [value]: this warp slot's cursor
        self.stride = sms * WARPS
        self.st_left, d0 = split(n, sms)
        self.dyn0 = d0 + g % WARPS
        self.st_next = g
        self.blk = self.blk_left = 0
        self.claim = None
        self.claims = 0
        if self.st_left <= CLAIM:
            self.claim_ahead()

    def claim_ahead(self):
        self.claim = self.cursor[0]           # atomicAdd(cursor, CLAIM)
        self.cursor[0] += CLAIM
        self.claims += 1

    def next(self):
        if self.st_left:
            c = self.st_next
            self.st_next += self.stride
            self.st_left -= 1
            if self.st_left == CLAIM:
                self.claim_ahead()
            return c
        if self.blk_left == 0:
            assert self.claim is not None, "a claim is read before it was made"
            self.blk = self.dyn0 + self.claim * WARPS
            self.blk_left = CLAIM
            self.claim_ahead()
        self.blk_left -= 1
        c = self.blk
        self.blk += WARPS
        return c


def run(n, sms, rng=None, speed=None):
    """Runs every warp of a launch to its end, one loop iteration of a random warp at a time (a warp of CTA b is
    picked with weight speed[b]). Returns, per warp, the chunks it read in order."""
    rng = rng or random.Random(0)
    nc = n_chunks(n)
    cursors = [[0] for _ in range(WARPS)]
    warps = [Warp(n, sms, g, cursors) for g in range(sms * WARPS)]
    pipe = []                                 # per warp: [chunk of this iteration, of the next one]
    for w in warps:                           # prologue: the first two chunks are requested
        pipe.append([w.next(), w.next()])
    taken = [[] for _ in warps]
    live = [g for g in range(len(warps)) if pipe[g][0] < nc]
    weights = [speed[g // WARPS] if speed else 1.0 for g in range(len(warps))]
    while live:
        k = rng.choices(range(len(live)), [weights[g] for g in live])[0] if speed else rng.randrange(len(live))
        g = live[k]
        c, c_ahead = pipe[g]
        taken[g].append(c)
        c_req = warps[g].next()               # requested two iterations ahead
        pipe[g] = [c_ahead, c_req]
        if c_ahead >= nc:                     # the loop ends: every chunk it still holds lies beyond the array
            assert c_req >= nc and (warps[g].claim is None or warps[g].dyn0 + warps[g].claim * WARPS >= nc)
            live[k] = live[-1]
            live.pop()
    return taken


def check(n, sms, rng=None, speed=None):
    """Every chunk of the launch is read by exactly one warp, each warp's chunks in increasing order."""
    taken = run(n, sms, rng, speed)
    got = sorted(c for t in taken for c in t)
    assert got == list(range(n_chunks(n))), (n, sms)
    for t in taken:
        assert t == sorted(t) and len(set(t)) == len(t)
    return taken
