"""A stream whose histogram cells wrap modulo 2^32 when W = 16 of its windows are summed (docs/SPEC.md §3), and the
closed form of any sum of m of its windows. TEST INFRASTRUCTURE ONLY.

One window is TILES copies of a tile of 8,200 records. The tile holds four edges:
  - A, pod -> service over HTTP, every record 503: HOT records in bucket 50 (the low cell of the pair (50, 51) of
    lane 6 of an edge row), one in bucket 51 and one in bucket 10; durations of 2^33 and more (packed records carry
    them in the overflow array), so lat_sum_ns passes 2^64 too;
  - B, a reversed pod <-> pod row (AMQP deliver): HOT records in bucket 8 (the first cell of lane 1), one each in
    the neighbours 7 and 9;
  - C, pod -> outbound address, and D, Host-keyed: one record each, never near a wrap.
HOT * TILES * W = 4097 * 2^20 = 2^32 + 2^20: cells 50 and 8 wrap to 2^20 in a sum of 16 windows and to nothing in
one of 15. Each of their neighbours holds 2^20 then, so a carry out of the wrapped cell into its neighbour shows.
Row A's quantile total after the wrap is the sum of its cells, 3 * 2^20, far below its count 2^32 + 3 * 2^20
(SPEC §5): its p50 is 2^33 + 2^31, in the middle of bucket 50, where a total taken from count would give 2^40.
"""
import numpy as np

import ingest_streams as ist
from alaz_b200 import abi

M32, M64 = ist.M32, ist.M64
W = 16                           # windows whose sum wraps
TILES = 1 << 16                  # tiles per window
BUF_TILES = 1 << 13              # tiles in one device buffer: a window is SUBMITS submits of it (1.07 GB)
SUBMITS = TILES // BUF_TILES
HOT = 4097

POD = [abi.ip("10.0.0.%d" % i) for i in range(1, 5)]
SVC = abi.ip("172.16.0.1")
OUT = abi.ip("203.0.113.9")
HOST_ID = 77
TABLES = [(abi.TABLE_POD, POD, [1, 2, 3, 4]), (abi.TABLE_SVC, [SVC], [7])]

# bucket -> duration, and the records of each bucket per tile
A_DUR = {50: (1 << 33) + 12345, 51: (3 << 32) + 12345, 10: 8192 + 100}
A_PER_TILE = {50: HOT, 51: 1, 10: 1}
B_DUR = {8: 5000, 7: 3500, 9: 7000}
B_PER_TILE = {8: HOT, 7: 1, 9: 1}


def tile():
    """The 8,200 records of one tile (32-B records)."""
    for dur in (A_DUR, B_DUR):
        assert all(ist.latency_bucket(d) == b for b, d in dur.items())
    a = np.concatenate([np.full(A_PER_TILE[b], A_DUR[b], np.uint64) for b in (50, 51, 10)])
    b = np.concatenate([np.full(B_PER_TILE[k], B_DUR[k], np.uint64) for k in (8, 7, 9)])
    return np.concatenate([
        ist.records(POD[0], SVC, a, status=503),
        ist.records(POD[0], POD[1], b, protocol=abi.PROTO_AMQP, method=abi.AMQP_DELIVER),
        ist.records(POD[2], OUT, 1_000_000),
        ist.records(POD[3], HOST_ID, 2_000_000, protocol=abi.PROTO_HTTP | abi.PROTO_F_HOSTKEY)])


def window_edges():
    """(edges, stats) the oracle gives for one window: the tile times TILES."""
    return ist.scaled_oracle(TABLES, tile(), TILES)


def row_a(rows):
    (i,) = np.flatnonzero(rows["to_type"] == abi.NODE_SVC)
    return rows[i]


def row_b(rows):
    (i,) = np.flatnonzero((rows["from_type"] == abi.NODE_POD) & (rows["to_type"] == abi.NODE_POD))
    return rows[i]


def closed_form(m, tiles=TILES):
    """{"A": (count, err5xx, lat_sum_ns, {bucket: cell}), "B": ...} of the sum of m windows: u64 sums mod 2^64, cells
    mod 2^32, every other cell 0."""
    n = m * tiles
    out = {}
    for name, dur, per, err in (("A", A_DUR, A_PER_TILE, True), ("B", B_DUR, B_PER_TILE, False)):
        count = sum(per.values()) * n
        lat = sum(per[b] * dur[b] for b in per) * n
        out[name] = (count & M64, count & M64 if err else 0, lat & M64, {b: per[b] * n & M32 for b in per})
    return out


def check_closed_form(rows, m, tiles=TILES):
    """Rows A and B of a sum of m windows equal the closed form, field by field and cell by cell."""
    cf = closed_form(m, tiles)
    for name, r in (("A", row_a(rows)), ("B", row_b(rows))):
        count, err, lat, cells = cf[name]
        assert (int(r["count"]), int(r["err5xx"]), int(r["lat_sum_ns"])) == (count, err, lat), (m, name)
        hist = np.zeros(abi.NB, np.uint32)
        for b, c in cells.items():
            hist[b] = c
        assert np.array_equal(r["hist"], hist), (m, name, {b: int(r["hist"][b]) for b in cells})
