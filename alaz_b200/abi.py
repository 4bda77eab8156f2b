"""Python mirror of include/alazgpu.h: record layouts and constants.

Pure data definitions (numpy dtypes + ctypes structs); no compute. The sizes
are asserted against the C header in tests/test_abi.py.
"""
import ctypes as C
import os

import numpy as np

ABI_VERSION = int(os.environ.get("ALZ_ABI_VERSION", "2"))   # override only to drive an older build for A/B timing
NB = 64
BPF_L7_EVENT_SIZE = 1096
COMM_ID_BYTES = 128

# status codes
OK, E_INVAL, E_NOMEM, E_CUDA, E_NODEVICE, E_CAPACITY, E_STATE, E_NCCL, E_UNSUPPORTED = (
    0, -1, -2, -3, -4, -5, -6, -7, -8)

# ebpf/l7_req/l7.go:19-29
PROTO_UNKNOWN, PROTO_HTTP, PROTO_AMQP, PROTO_POSTGRES, PROTO_HTTP2 = 0, 1, 2, 3, 4
PROTO_REDIS, PROTO_KAFKA, PROTO_MYSQL, PROTO_MONGO = 5, 6, 7, 8
AMQP_PUBLISH, AMQP_DELIVER = 1, 2
REDIS_COMMAND, REDIS_PUSHED_EVENT, REDIS_PING = 1, 2, 3
MF_METHOD_MASK, MF_PAYLOAD_REJECT, MF_TLS = 0x3F, 0x40, 0x80
NODE_POD, NODE_SVC, NODE_OUTBOUND, NODE_OUTBOUND_HOST = 0, 1, 2, 3
NODE_GROUP = 4                                                      # a caller-defined group (§24)
PROTO_F_HOSTKEY = 0x40
TABLE_POD, TABLE_SVC = 0, 1
CFG_EAGER_JOIN = 0x1
CFG_NO_SMEM_CACHE = 0x2
MIX_SURVEY, MIX_ALL = 0, 1

L7_REC = np.dtype([
    ("saddr", "<u4"), ("daddr", "<u4"), ("sport", "<u2"), ("dport", "<u2"),
    ("status", "<u2"), ("protocol", "u1"), ("method_flags", "u1"),
    ("duration_ns", "<u8"), ("write_time_ns", "<u8"),
])
assert L7_REC.itemsize == 32

L7_REC16 = np.dtype([
    ("saddr", "<u4"), ("daddr", "<u4"), ("status", "<u2"), ("protocol", "u1"), ("method_flags", "u1"),
    ("duration_ns", "<u4"),
])
assert L7_REC16.itemsize == 16
REC16_DUR_OVERFLOW = 0x80

TCP_REC = np.dtype([
    ("fd", "<u8"), ("timestamp_ns", "<u8"), ("pid", "<u4"), ("saddr", "<u4"),
    ("daddr", "<u4"), ("sport", "<u2"), ("dport", "<u2"), ("type", "<u4"), ("_pad", "<u4"),
])
assert TCP_REC.itemsize == 40

# struct tcp_event as the perf ring carries it (ebpf/c/struct.h:2-12), 64 B with tail padding
BPF_TCP_EVENT = np.dtype({"names": ["fd", "timestamp", "type", "pid", "sport", "dport", "saddr", "daddr"],
                          "formats": ["<u8", "<u8", "<u4", "<u4", "<u2", "<u2", ("u1", (16,)), ("u1", (16,))],
                          "offsets": [0, 8, 16, 20, 24, 26, 28, 44], "itemsize": 64})
SOCK_QUERY = np.dtype([("fd", "<u8"), ("timestamp_ns", "<u8"), ("pid", "<u4"), ("_pad", "<u4")])
assert SOCK_QUERY.itemsize == 24
SOCK_RESULT = np.dtype([("found", "<u4"), ("saddr", "<u4"), ("daddr", "<u4"),
                        ("sport", "<u2"), ("dport", "<u2")])
assert SOCK_RESULT.itemsize == 16
ALIVE_CONN = np.dtype([("from_ip", "<u4"), ("from_id", "<u4"), ("to_ip", "<u4"), ("to_id", "<u4"),
                       ("from_port", "<u2"), ("to_port", "<u2"), ("to_type", "u1"), ("_pad", "u1", (3,))])
assert ALIVE_CONN.itemsize == 24

EDGE_OUT = np.dtype([
    ("from_type", "u1"), ("to_type", "u1"), ("_pad", "u1", (6,)),
    ("from", "<u4"), ("to", "<u4"),
    ("count", "<u8"), ("err5xx", "<u8"), ("lat_sum_ns", "<u8"),
    ("hist", "<u4", (NB,)),
])
assert EDGE_OUT.itemsize == 296


class Config(C.Structure):
    _fields_ = [
        ("abi_version", C.c_uint32), ("device", C.c_int32),
        ("max_endpoints", C.c_uint32), ("max_pairs", C.c_uint32),
        ("max_edges", C.c_uint32), ("max_batch", C.c_uint32),
        ("flags", C.c_uint32), ("_reserved", C.c_uint32 * 9),
    ]


class Stats(C.Structure):
    _fields_ = [
        ("events_in", C.c_uint64), ("rows_emitted", C.c_uint64),
        ("not_request", C.c_uint64), ("src_unresolved", C.c_uint64),
        ("pairs_live", C.c_uint64), ("edges_live", C.c_uint64),
        ("tcp_events_in", C.c_uint64), ("tcp_localhost_dropped", C.c_uint64),
        ("capacity_events", C.c_uint64), ("windows", C.c_uint64),
        ("kernel_launches", C.c_uint64), ("collective_bytes_last", C.c_uint64),
        ("flush_local_us_last", C.c_uint64), ("merge_us_last", C.c_uint64),
        ("late_events", C.c_uint64), ("deferred_events", C.c_uint64),
    ]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_ if not n.startswith("_")}


class RollupInfo(C.Structure):
    """alz_rollup_info."""
    _fields_ = [
        ("windows", C.c_uint32), ("clocked", C.c_uint32),
        ("window_first", C.c_uint64), ("window_last", C.c_uint64),
        ("epoch_first", C.c_uint64), ("epoch_last", C.c_uint64), ("rows_in", C.c_uint64),
    ]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


MAX_TIERS = 4


class HistoryTier(C.Structure):
    """alz_history_tier."""
    _fields_ = [("factor", C.c_uint32), ("depth", C.c_uint32), ("arena_rows", C.c_uint64), ("block_rows", C.c_uint64)]


class TierState(C.Structure):
    """alz_tier_state."""
    _fields_ = [("entries", C.c_uint32), ("open_windows", C.c_uint32), ("dropped", C.c_uint64)]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


SPAN_AT_MOST, SPAN_AT_LEAST = 0, 1
ROLLUP_WINDOWS, ROLLUP_TIER, ROLLUP_SPAN = 0, 1, 2   # alz_gnn_score_rollup kinds


class TopInfo(C.Structure):
    """alz_top_info."""
    _fields_ = [("scored", C.c_uint64), ("above", C.c_uint64)]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


METRIC_COUNT, METRIC_ERR5XX, METRIC_ERR_RATE, METRIC_MEAN_NS, METRIC_QUANTILE = 0, 1, 2, 3, 4   # alz_metric kinds
MAX_METRICS = 8


class Metric(C.Structure):
    """alz_metric: kind METRIC_*, q for METRIC_QUANTILE."""
    _fields_ = [("kind", C.c_uint32), ("_pad", C.c_uint32), ("q", C.c_double)]


def metrics(*specs):
    """A ctypes array of alz_metric from kinds or (kind, q) pairs, e.g. metrics((METRIC_QUANTILE, 0.99), METRIC_COUNT)."""
    ms = [Metric(s[0], 0, float(s[1])) if isinstance(s, tuple) else Metric(int(s), 0, 0.0) for s in specs]
    return (Metric * max(len(ms), 1))(*ms)


SOURCE_WINDOW = 0xFFFFFFFF                                    # alz_baseline_pin / alz_edge_changes* sources
CHANGE_DELTA, CHANGE_DROP, CHANGE_RATIO = 0, 1, 2             # change modes
PRESENT_BOTH, PRESENT_NEW, PRESENT_GONE = 0x1, 0x2, 0x4       # presence bits and filter masks
PRESENT_ALL = PRESENT_BOTH | PRESENT_NEW | PRESENT_GONE
ABSENT = 0xFFFFFFFF                                           # index / base_index of the side a row is absent from

EDGE_CHANGE = np.dtype([
    ("from_type", "u1"), ("to_type", "u1"), ("presence", "u1"), ("_pad", "u1", (5,)),
    ("from", "<u4"), ("to", "<u4"), ("index", "<u4"), ("base_index", "<u4"),
    ("value", "<f8"), ("base_value", "<f8"), ("change", "<f8"),
])
assert EDGE_CHANGE.itemsize == 48


class ChangeInfo(C.Structure):
    """alz_change_info."""
    _fields_ = [(n, C.c_uint64) for n in ("source_rows", "base_rows", "both", "added", "gone", "listed", "above")] + \
        [("source_windows", C.c_uint32), ("base_windows", C.c_uint32)]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


EDGE_ENDS = np.dtype([("from_type", "u1"), ("to_type", "u1"), ("_pad", "u1", (6,)), ("from", "<u4"), ("to", "<u4")])
assert EDGE_ENDS.itemsize == 16


class EdgeEnds(C.Structure):
    """alz_edge_ends: the head of alz_edge_out, the key of an edge series row (_pad is ignored)."""
    _fields_ = [("from_type", C.c_uint8), ("to_type", C.c_uint8), ("_pad", C.c_uint8 * 6), ("from_", C.c_uint32),
                ("to", C.c_uint32)]


class SeriesInfo(C.Structure):
    """alz_series_info."""
    _fields_ = [("edges", C.c_uint64), ("rows_in", C.c_uint64), ("points", C.c_uint32), ("tier", C.c_uint32)]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


TREND_SLOPE, TREND_SHIFT, TREND_RATIO, TREND_ZSCORE = 0, 1, 2, 3   # alz_trend stats
TREND_RISING, TREND_FALLING = 0, 1                                  # directions
TREND_ABSENT_SKIP, TREND_ABSENT_ZERO = 0, 1                         # absent modes

EDGE_TREND = np.dtype([
    ("from_type", "u1"), ("to_type", "u1"), ("valid", "u1"), ("_pad", "u1", (5,)),
    ("from", "<u4"), ("to", "<u4"), ("index", "<u4"), ("used", "<u4"),
    ("trend", "<f8"), ("recent", "<f8"), ("before", "<f8"),
])
assert EDGE_TREND.itemsize == 48


class Trend(C.Structure):
    """alz_trend: stat TREND_*, direction TREND_RISING / TREND_FALLING, absent TREND_ABSENT_*, the last `recent`
    points are recent, a valid row uses at least min_points points."""
    _fields_ = [(n, C.c_uint32) for n in ("stat", "direction", "absent", "recent", "min_points", "_pad")]


class TrendInfo(C.Structure):
    """alz_trend_info."""
    _fields_ = [(n, C.c_uint64) for n in ("edges", "rows_in", "valid", "above")] + \
        [("points", C.c_uint32), ("tier", C.c_uint32)]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


SIDE_IN, SIDE_OUT = 0, 1                                            # alz_node_metrics* / alz_node_top* sides

NODE_SUMS = np.dtype([("count", "<u8"), ("err5xx", "<u8"), ("lat_sum_ns", "<u8"), ("hist", "<u4", (NB,))])
assert NODE_SUMS.itemsize == 280
NODE_OUT = np.dtype([
    ("type", "u1"), ("_pad", "u1", (3,)), ("value", "<u4"), ("in_edges", "<u4"), ("out_edges", "<u4"),
    ("in", NODE_SUMS), ("out", NODE_SUMS),
])
assert NODE_OUT.itemsize == 576

NODE_ENDS = np.dtype([("type", "u1"), ("_pad", "u1", (3,)), ("value", "<u4")])   # the head of NODE_OUT
assert NODE_ENDS.itemsize == 8 and NODE_ENDS.fields["value"][1] == NODE_OUT.fields["value"][1]
NODE_TREND = np.dtype([
    ("type", "u1"), ("_pad0", "u1"), ("valid", "u1"), ("_pad1", "u1", (5,)),
    ("value", "<u4"), ("_pad2", "<u4"), ("index", "<u4"), ("used", "<u4"),
    ("trend", "<f8"), ("recent", "<f8"), ("before", "<f8"),
])
assert NODE_TREND.itemsize == 48
assert all(NODE_TREND.fields[f][1] == EDGE_TREND.fields[f][1]
           for f in ("valid", "index", "used", "trend", "recent", "before"))   # laid out as EDGE_TREND from valid on
NODE_CHANGE = np.dtype([
    ("type", "u1"), ("_pad0", "u1"), ("presence", "u1"), ("_pad1", "u1", (5,)),
    ("node", "<u4"), ("_pad2", "<u4"), ("index", "<u4"), ("base_index", "<u4"),
    ("value", "<f8"), ("base_value", "<f8"), ("change", "<f8"),
])
assert NODE_CHANGE.itemsize == 48
assert all(NODE_CHANGE.fields[f][1] == EDGE_CHANGE.fields[f][1]
           for f in ("presence", "index", "base_index", "value", "base_value", "change"))   # EDGE_CHANGE's offsets


class GroupInfo(C.Structure):
    """alz_group_info."""
    _fields_ = [(n, C.c_uint64) for n in ("source_rows", "mapped_ends", "edges", "internal")]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


GROUP_INFO = GroupInfo

REACH_DOWN, REACH_UP, REACH_ANY = 0, 1, 2                           # alz_reach* directions (§27)
REACH_MAX_HOPS = 64
REACH_NONE = 0xFFFFFFFF                                             # parent / row of a seed
REACH_NODE = np.dtype([
    ("type", "u1"), ("_pad", "u1", (3,)), ("value", "<u4"), ("hops", "<u4"), ("index", "<u4"), ("parent", "<u4"),
    ("row", "<u4"),
])
assert REACH_NODE.itemsize == 24 and REACH_NODE.fields["value"][1] == NODE_ENDS.fields["value"][1]


class ReachInfo(C.Structure):
    """alz_reach_info."""
    _fields_ = [(n, C.c_uint64) for n in ("rows", "traversable", "seeds_found", "nodes", "levels", "cut")]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


CYCLE_NODE = np.dtype([                                             # alz_cycle_node (§28)
    ("type", "u1"), ("_pad", "u1", (3,)), ("value", "<u4"), ("index", "<u4"), ("component", "<u4"), ("size", "<u4"),
    ("depth", "<u4"), ("height", "<u4"),
])
assert CYCLE_NODE.itemsize == 28 and CYCLE_NODE.fields["value"][1] == NODE_ENDS.fields["value"][1]


class CycleInfo(C.Structure):
    """alz_cycle_info."""
    _fields_ = [(n, C.c_uint64) for n in ("rows", "traversable", "self_rows", "nodes", "components", "cyclic",
                                          "cyclic_nodes", "largest", "cycle_rows", "depth")]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


CORR_POSITIVE, CORR_NEGATIVE, CORR_ABS = 0, 1, 2                     # alz_corr directions (§29)
CORR_ABSENT_SKIP, CORR_ABSENT_ZERO = 0, 1                           # absent modes
CORR_MAX_LAG = 32

EDGE_CORR = np.dtype([                                              # alz_edge_corr
    ("from_type", "u1"), ("to_type", "u1"), ("valid", "u1"), ("lag", "u1"), ("_pad", "u1", (4,)),
    ("from", "<u4"), ("to", "<u4"), ("index", "<u4"), ("used", "<u4"),
    ("r", "<f8"), ("score", "<f8"), ("r0", "<f8"),
])
assert EDGE_CORR.itemsize == 48
NODE_CORR = np.dtype([                                              # alz_node_corr
    ("type", "u1"), ("_pad0", "u1"), ("valid", "u1"), ("lag", "u1"), ("_pad1", "u1", (4,)),
    ("value", "<u4"), ("_pad2", "<u4"), ("index", "<u4"), ("used", "<u4"),
    ("r", "<f8"), ("score", "<f8"), ("r0", "<f8"),
])
assert NODE_CORR.itemsize == 48
assert all(NODE_CORR.fields[f][1] == EDGE_CORR.fields[f][1]
           for f in ("valid", "lag", "index", "used", "r", "score", "r0"))   # laid out as EDGE_CORR from valid on


class Corr(C.Structure):
    """alz_corr: direction CORR_*, absent CORR_ABSENT_*, lags 0 .. max_lag, a defined lag uses >= min_points pairs."""
    _fields_ = [(n, C.c_uint32) for n in ("direction", "absent", "max_lag", "min_points")]


class CorrTarget(C.Structure):
    """alz_corr_target: n values (and presence bytes, or NULL) in host memory, the window_last of the newest point."""
    _fields_ = [("values", C.c_void_p), ("present", C.c_void_p), ("n", C.c_size_t), ("window_last", C.c_uint64)]


class CorrInfo(C.Structure):
    """alz_corr_info."""
    _fields_ = [(n, C.c_uint64) for n in ("rows", "rows_in", "valid", "above")] + \
        [(n, C.c_uint32) for n in ("points", "tier", "target_used", "_pad")]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_ if n != "_pad"}


class SpanInfo(C.Structure):
    """alz_span_info."""
    _fields_ = [("r", RollupInfo), ("entries", C.c_uint32 * (1 + MAX_TIERS)), ("open_blocks", C.c_uint32),
                ("_reserved", C.c_uint32 * 2)]

    def as_dict(self):
        """alz_rollup_info's fields, `entries` as a list per tier (0 = window history), `open_blocks` as a bit mask"""
        return dict(self.r.as_dict(), entries=[int(x) for x in self.entries], open_blocks=int(self.open_blocks))


class SockStats(C.Structure):
    """alz_sock_stats_t."""
    _fields_ = [(n, C.c_uint64) for n in ("lines", "pool_records", "pool_garbage", "syncs", "sync_ops", "sync_bytes",
                                          "repools", "joined_events")]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


class SynthView(C.Structure):
    """alz_synth_view (alaz_b200/synth/alz_synth.h)."""
    _fields_ = [
        ("seed", C.c_uint64), ("t0_ns", C.c_uint64), ("dt_ns", C.c_uint32),
        ("mix", C.c_uint32), ("n_edges", C.c_uint32), ("n_unknown", C.c_uint32),
        ("unknown_base", C.c_uint32), ("_pad", C.c_uint32),
        ("edge_saddr", C.c_void_p), ("edge_daddr", C.c_void_p), ("edge_flags", C.c_void_p),
        ("alias_thresh", C.c_void_p), ("alias_idx", C.c_void_p), ("lat_q", C.c_void_p),
    ]


class SynthTopo(C.Structure):
    """alz_synth_topo (alaz_b200/synth/alz_synth.h)."""
    _fields_ = [
        ("n_services", C.c_uint32), ("n_pods", C.c_uint32),
        ("n_edges", C.c_uint32), ("n_outbound", C.c_uint32),
        ("pod_ip", C.POINTER(C.c_uint32)), ("svc_ip", C.POINTER(C.c_uint32)),
        ("out_ip", C.POINTER(C.c_uint32)),
        ("edge_saddr", C.POINTER(C.c_uint32)), ("edge_daddr", C.POINTER(C.c_uint32)),
        ("edge_flags", C.POINTER(C.c_uint8)),
        ("alias_thresh", C.POINTER(C.c_uint32)), ("alias_idx", C.POINTER(C.c_uint32)),
        ("lat_q", C.POINTER(C.c_uint64)),
        ("view", SynthView),
    ]


def ip(s: str) -> int:
    """Dotted quad -> the u32 the reference feeds IntToIPv4 (first octet in MSB)."""
    a, b, c, d = (int(x) for x in s.split("."))
    return (a << 24) | (b << 16) | (c << 8) | d
