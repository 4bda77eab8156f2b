"""ctypes binding of libalazgpu.so (include/alazgpu.h). Thin: every method is
one C call. Fails loudly when the library or a CUDA device is missing — there
is no Python or CPU fallback for any of it."""
import ctypes as C
import os

import numpy as np

from . import abi, build as _build


class AlzError(RuntimeError):
    def __init__(self, status, what, detail=""):
        self.status = status
        super().__init__(f"{what}: status {status} {detail}".strip())


_lib = None

# every symbol include/alazgpu.h declares (tests/test_abi.py checks the header against this)
EXPORTS = [
    "alz_create", "alz_destroy", "alz_strerror", "alz_last_cuda_error", "alz_set_stream", "alz_sync",
    "alz_table_upsert", "alz_table_upsert_batch", "alz_table_erase", "alz_table_commit", "alz_submit_l7", "alz_submit_l7_device",
    "alz_submit_l7_packed", "alz_submit_l7_packed_device", "alz_pack_l7",
    "alz_submit_l7_raw", "alz_window_flush", "alz_window_flush_device", "alz_window_fetch", "alz_get_stats",
    "alz_window_clock", "alz_window_epoch", "alz_window_history", "alz_window_rollup", "alz_window_rollup_device",
    "alz_window_history_tiers", "alz_window_rollup_tier", "alz_window_rollup_tier_device", "alz_window_tier_state",
    "alz_window_rollup_span", "alz_window_rollup_span_device", "alz_gnn_score",
    "alz_gnn_score_device", "alz_gnn_score_rollup", "alz_gnn_score_rollup_device", "alz_gnn_top", "alz_gnn_top_device",
    "alz_gnn_top_rollup", "alz_gnn_top_rollup_device", "alz_edge_metrics", "alz_edge_metrics_device",
    "alz_edge_metrics_rollup", "alz_edge_metrics_rollup_device", "alz_edge_top", "alz_edge_top_device",
    "alz_edge_top_rollup", "alz_edge_top_rollup_device", "alz_baseline_pin", "alz_baseline_clear", "alz_edge_changes",
    "alz_edge_changes_device", "alz_edge_changes_top", "alz_edge_changes_top_device", "alz_edge_series",
    "alz_edge_series_device", "alz_edge_series_keys", "alz_edge_series_keys_device", "alz_edge_trends",
    "alz_edge_trends_device", "alz_edge_trends_top", "alz_edge_trends_top_device", "alz_node_rows",
    "alz_node_rows_device", "alz_node_metrics", "alz_node_metrics_device", "alz_node_top", "alz_node_top_device",
    "alz_node_series", "alz_node_series_device", "alz_node_series_keys", "alz_node_series_keys_device",
    "alz_node_trends", "alz_node_trends_device", "alz_node_trends_top", "alz_node_trends_top_device",
    "alz_node_changes", "alz_node_changes_device", "alz_node_changes_top", "alz_node_changes_top_device",
    "alz_group_set", "alz_group_edges", "alz_group_edges_device", "alz_group_edge_metrics",
    "alz_group_edge_metrics_device", "alz_group_edge_top", "alz_group_edge_top_device", "alz_group_nodes",
    "alz_group_nodes_device", "alz_group_node_metrics", "alz_group_node_metrics_device", "alz_group_node_top",
    "alz_group_node_top_device", "alz_group_edge_changes", "alz_group_edge_changes_device",
    "alz_group_edge_changes_top", "alz_group_edge_changes_top_device", "alz_group_node_changes",
    "alz_group_node_changes_device", "alz_group_node_changes_top", "alz_group_node_changes_top_device",
    "alz_group_edge_series", "alz_group_edge_series_device", "alz_group_edge_series_keys",
    "alz_group_edge_series_keys_device", "alz_group_node_series", "alz_group_node_series_device",
    "alz_group_node_series_keys", "alz_group_node_series_keys_device", "alz_group_edge_trends",
    "alz_group_edge_trends_device", "alz_group_edge_trends_top", "alz_group_edge_trends_top_device",
    "alz_group_node_trends", "alz_group_node_trends_device", "alz_group_node_trends_top",
    "alz_group_node_trends_top_device", "alz_reach", "alz_reach_device", "alz_group_reach", "alz_group_reach_device",
    "alz_cycles", "alz_cycles_device", "alz_group_cycles", "alz_group_cycles_device",
    "alz_edge_correlations", "alz_edge_correlations_device", "alz_edge_correlations_top",
    "alz_edge_correlations_top_device", "alz_node_correlations", "alz_node_correlations_device",
    "alz_node_correlations_top", "alz_node_correlations_top_device", "alz_group_edge_correlations",
    "alz_group_edge_correlations_device", "alz_group_edge_correlations_top", "alz_group_edge_correlations_top_device",
    "alz_group_node_correlations", "alz_group_node_correlations_device", "alz_group_node_correlations_top",
    "alz_group_node_correlations_top_device",
    "alz_edge_quantiles", "alz_submit_tcp", "alz_submit_tcp_raw", "alz_sock_lookup", "alz_sock_lookup_at",
    "alz_submit_l7_join", "alz_sock_gc", "alz_sock_alive", "alz_sock_stats", "alz_comm_unique_id", "alz_comm_init",
    "alz_owner_rank",
]


def load(rebuild=False):
    """dlopen alaz_b200/lib/libalazgpu.so (building it first when it is missing and nvcc exists)."""
    global _lib
    if _lib is not None and not rebuild:
        return _lib
    path = os.environ.get("ALZ_LIB_PATH") or _build.LIB   # ALZ_LIB_PATH: A/B runs of two builds on one box
    if rebuild or not os.path.exists(path):
        path = _build.build(force=rebuild)
    L = C.CDLL(path, mode=C.RTLD_GLOBAL)
    vp, u32, u64, sz, i = C.c_void_p, C.c_uint32, C.c_uint64, C.c_size_t, C.c_int
    pp = C.POINTER(vp)
    sig = {
        "alz_create": ([C.POINTER(abi.Config), pp], i),
        "alz_destroy": ([vp], i),
        "alz_strerror": ([i], C.c_char_p),
        "alz_last_cuda_error": ([vp], C.c_char_p),
        "alz_set_stream": ([vp, vp], i),
        "alz_sync": ([vp], i),
        "alz_table_upsert": ([vp, i, u32, u32], i),
        "alz_table_erase": ([vp, i, u32], i),
        "alz_table_upsert_batch": ([vp, i, vp, vp, sz], i),
        "alz_table_commit": ([vp], i),
        "alz_submit_l7": ([vp, vp, sz], i),
        "alz_submit_l7_device": ([vp, vp, sz], i),
        "alz_submit_l7_raw": ([vp, vp, sz], i),
        "alz_submit_l7_packed": ([vp, vp, sz, vp, sz], i),
        "alz_submit_l7_packed_device": ([vp, vp, sz, vp], i),
        "alz_pack_l7": ([vp, sz, vp, vp, sz], C.c_long),
        "alz_window_fetch": ([vp, vp, sz, C.POINTER(sz)], i),
        "alz_window_clock": ([vp, u64, u64, u64], i),
        "alz_window_epoch": ([vp, C.POINTER(u64)], i),
        "alz_window_history": ([vp, u32, u64], i),
        "alz_window_rollup": ([vp, u32, vp, sz, C.POINTER(sz), C.POINTER(abi.RollupInfo)], i),
        "alz_window_rollup_device": ([vp, u32, pp, C.POINTER(sz), C.POINTER(abi.RollupInfo)], i),
        "alz_window_history_tiers": ([vp, C.POINTER(abi.HistoryTier), u32], i),
        "alz_window_rollup_tier": ([vp, u32, u32, vp, sz, C.POINTER(sz), C.POINTER(abi.RollupInfo)], i),
        "alz_window_rollup_tier_device": ([vp, u32, u32, pp, C.POINTER(sz), C.POINTER(abi.RollupInfo)], i),
        "alz_window_tier_state": ([vp, u32, C.POINTER(abi.TierState)], i),
        "alz_window_rollup_span": ([vp, u64, u32, vp, sz, C.POINTER(sz), C.POINTER(abi.SpanInfo)], i),
        "alz_window_rollup_span_device": ([vp, u64, u32, pp, C.POINTER(sz), C.POINTER(abi.SpanInfo)], i),
        "alz_pinned_alloc_local": ([vp, sz, pp], i),
        "alz_window_flush": ([vp, vp, sz, C.POINTER(sz)], i),
        "alz_window_flush_device": ([vp, pp, C.POINTER(sz)], i),
        "alz_get_stats": ([vp, C.POINTER(abi.Stats)], i),
        "alz_gnn_score": ([vp, vp, sz, C.POINTER(sz)], i),
        "alz_gnn_score_device": ([vp, pp, C.POINTER(sz)], i),
        "alz_gnn_score_rollup": ([vp, u32, vp, sz, C.POINTER(sz)], i),
        "alz_gnn_score_rollup_device": ([vp, u32, pp, C.POINTER(sz)], i),
        "alz_gnn_top": ([vp, u32, C.c_float, vp, vp, vp, sz, C.POINTER(sz), C.POINTER(abi.TopInfo)], i),
        "alz_gnn_top_device": ([vp, u32, C.c_float, pp, pp, pp, C.POINTER(sz), C.POINTER(abi.TopInfo)], i),
        "alz_gnn_top_rollup": ([vp, u32, u32, C.c_float, vp, vp, vp, sz, C.POINTER(sz), C.POINTER(abi.TopInfo)], i),
        "alz_gnn_top_rollup_device": ([vp, u32, u32, C.c_float, pp, pp, pp, C.POINTER(sz), C.POINTER(abi.TopInfo)], i),
        "alz_gnn_nodes": ([vp, vp, vp, sz, C.POINTER(sz)], i),
        "alz_debug_top_scores": ([vp, vp, sz, u32, C.c_float, vp, sz, C.POINTER(sz), C.POINTER(u64)], i),
        "alz_edge_metrics": ([vp, vp, u32, vp, sz, C.POINTER(sz)], i),
        "alz_edge_metrics_device": ([vp, vp, u32, pp, C.POINTER(sz)], i),
        "alz_edge_metrics_rollup": ([vp, u32, vp, u32, vp, sz, C.POINTER(sz)], i),
        "alz_edge_metrics_rollup_device": ([vp, u32, vp, u32, pp, C.POINTER(sz)], i),
        "alz_edge_top": ([vp, vp, u32, C.c_double, vp, vp, vp, sz, C.POINTER(sz), C.POINTER(abi.TopInfo)], i),
        "alz_edge_top_device": ([vp, vp, u32, C.c_double, pp, pp, pp, C.POINTER(sz), C.POINTER(abi.TopInfo)], i),
        "alz_edge_top_rollup": ([vp, u32, vp, u32, C.c_double, vp, vp, vp, sz, C.POINTER(sz), C.POINTER(abi.TopInfo)],
                                i),
        "alz_edge_top_rollup_device": ([vp, u32, vp, u32, C.c_double, pp, pp, pp, C.POINTER(sz),
                                        C.POINTER(abi.TopInfo)], i),
        "alz_debug_edge_metrics_rows": ([vp, vp, sz, vp, u32, vp, sz, C.POINTER(sz)], i),
        "alz_debug_top_keys64": ([vp, vp, sz, u32, C.c_double, vp, sz, C.POINTER(sz), C.POINTER(u64)], i),
        "alz_baseline_pin": ([vp, u32, C.POINTER(abi.RollupInfo)], i),
        "alz_baseline_clear": ([vp], i),
        "alz_edge_changes": ([vp, u32, vp, u32, u32, vp, sz, C.POINTER(sz), C.POINTER(abi.ChangeInfo)], i),
        "alz_edge_changes_device": ([vp, u32, vp, u32, u32, pp, C.POINTER(sz), C.POINTER(abi.ChangeInfo)], i),
        "alz_edge_changes_top": ([vp, u32, vp, u32, u32, u32, C.c_double, vp, sz, C.POINTER(sz),
                                  C.POINTER(abi.ChangeInfo)], i),
        "alz_edge_changes_top_device": ([vp, u32, vp, u32, u32, u32, C.c_double, pp, C.POINTER(sz),
                                         C.POINTER(abi.ChangeInfo)], i),
        "alz_debug_edge_changes_rows": ([vp, vp, sz, u32, vp, sz, u32, vp, u32, u32, vp, sz, C.POINTER(sz),
                                         C.POINTER(abi.ChangeInfo)], i),
        "alz_edge_series": ([vp, u32, u32, u32, vp, u32, vp, vp, sz, C.POINTER(sz), C.POINTER(u32), vp,
                             C.POINTER(abi.SeriesInfo)], i),
        "alz_edge_series_device": ([vp, u32, u32, u32, vp, u32, pp, pp, C.POINTER(sz), C.POINTER(u32), vp,
                                    C.POINTER(abi.SeriesInfo)], i),
        "alz_edge_series_keys": ([vp, vp, sz, u32, u32, vp, u32, vp, vp, sz, C.POINTER(sz), C.POINTER(u32), vp,
                                  C.POINTER(abi.SeriesInfo)], i),
        "alz_edge_series_keys_device": ([vp, vp, sz, u32, u32, vp, u32, pp, pp, C.POINTER(sz), C.POINTER(u32), vp,
                                         C.POINTER(abi.SeriesInfo)], i),
        "alz_edge_trends": ([vp, u32, u32, u32, vp, C.POINTER(abi.Trend), vp, sz, C.POINTER(sz), C.POINTER(u32), vp,
                             C.POINTER(abi.TrendInfo)], i),
        "alz_edge_trends_device": ([vp, u32, u32, u32, vp, C.POINTER(abi.Trend), pp, C.POINTER(sz), C.POINTER(u32),
                                    vp, C.POINTER(abi.TrendInfo)], i),
        "alz_edge_trends_top": ([vp, u32, u32, u32, vp, C.POINTER(abi.Trend), u32, C.c_double, vp, vp, vp, vp, sz,
                                 C.POINTER(sz), C.POINTER(u32), vp, C.POINTER(abi.TrendInfo)], i),
        "alz_edge_trends_top_device": ([vp, u32, u32, u32, vp, C.POINTER(abi.Trend), u32, C.c_double, pp, pp, pp, pp,
                                        C.POINTER(sz), C.POINTER(u32), vp, C.POINTER(abi.TrendInfo)], i),
        "alz_node_rows": ([vp, u32, vp, sz, C.POINTER(sz)], i),
        "alz_node_rows_device": ([vp, u32, pp, C.POINTER(sz)], i),
        "alz_node_metrics": ([vp, u32, u32, vp, u32, vp, sz, C.POINTER(sz)], i),
        "alz_node_metrics_device": ([vp, u32, u32, vp, u32, pp, C.POINTER(sz)], i),
        "alz_node_top": ([vp, u32, u32, vp, u32, C.c_double, vp, vp, vp, sz, C.POINTER(sz), C.POINTER(abi.TopInfo)], i),
        "alz_node_top_device": ([vp, u32, u32, vp, u32, C.c_double, pp, pp, pp, C.POINTER(sz),
                                 C.POINTER(abi.TopInfo)], i),
        "alz_debug_node_rows": ([vp, vp, sz, vp, sz, C.POINTER(sz)], i),
        "alz_node_series": ([vp, u32, u32, u32, u32, vp, u32, vp, vp, sz, C.POINTER(sz), C.POINTER(u32), vp,
                             C.POINTER(abi.SeriesInfo)], i),
        "alz_node_series_device": ([vp, u32, u32, u32, u32, vp, u32, pp, pp, C.POINTER(sz), C.POINTER(u32), vp,
                                    C.POINTER(abi.SeriesInfo)], i),
        "alz_node_series_keys": ([vp, vp, sz, u32, u32, u32, vp, u32, vp, vp, sz, C.POINTER(sz), C.POINTER(u32), vp,
                                  C.POINTER(abi.SeriesInfo)], i),
        "alz_node_series_keys_device": ([vp, vp, sz, u32, u32, u32, vp, u32, pp, pp, C.POINTER(sz), C.POINTER(u32),
                                         vp, C.POINTER(abi.SeriesInfo)], i),
        "alz_node_trends": ([vp, u32, u32, u32, u32, vp, C.POINTER(abi.Trend), vp, sz, C.POINTER(sz), C.POINTER(u32),
                             vp, C.POINTER(abi.TrendInfo)], i),
        "alz_node_trends_device": ([vp, u32, u32, u32, u32, vp, C.POINTER(abi.Trend), pp, C.POINTER(sz),
                                    C.POINTER(u32), vp, C.POINTER(abi.TrendInfo)], i),
        "alz_node_trends_top": ([vp, u32, u32, u32, u32, vp, C.POINTER(abi.Trend), u32, C.c_double, vp, vp, vp, vp,
                                 sz, C.POINTER(sz), C.POINTER(u32), vp, C.POINTER(abi.TrendInfo)], i),
        "alz_node_trends_top_device": ([vp, u32, u32, u32, u32, vp, C.POINTER(abi.Trend), u32, C.c_double, pp, pp,
                                        pp, pp, C.POINTER(sz), C.POINTER(u32), vp, C.POINTER(abi.TrendInfo)], i),
        "alz_node_changes": ([vp, u32, u32, vp, u32, u32, vp, sz, C.POINTER(sz), C.POINTER(abi.ChangeInfo)], i),
        "alz_node_changes_device": ([vp, u32, u32, vp, u32, u32, pp, C.POINTER(sz), C.POINTER(abi.ChangeInfo)], i),
        "alz_node_changes_top": ([vp, u32, u32, vp, u32, u32, u32, C.c_double, vp, sz, C.POINTER(sz),
                                  C.POINTER(abi.ChangeInfo)], i),
        "alz_node_changes_top_device": ([vp, u32, u32, vp, u32, u32, u32, C.c_double, pp, C.POINTER(sz),
                                         C.POINTER(abi.ChangeInfo)], i),
        "alz_debug_node_changes_rows": ([vp, vp, sz, u32, vp, sz, u32, u32, vp, u32, u32, vp, sz, C.POINTER(sz),
                                         C.POINTER(abi.ChangeInfo)], i),
        "alz_group_set": ([vp, vp, vp, sz], i),
        "alz_group_edges": ([vp, u32, vp, sz, C.POINTER(sz), C.POINTER(abi.GroupInfo)], i),
        "alz_group_edges_device": ([vp, u32, pp, C.POINTER(sz), C.POINTER(abi.GroupInfo)], i),
        "alz_group_edge_metrics": ([vp, u32, vp, u32, vp, sz, C.POINTER(sz)], i),
        "alz_group_edge_metrics_device": ([vp, u32, vp, u32, pp, C.POINTER(sz)], i),
        "alz_group_edge_top": ([vp, u32, vp, u32, C.c_double, vp, vp, vp, sz, C.POINTER(sz), C.POINTER(abi.TopInfo)],
                               i),
        "alz_group_edge_top_device": ([vp, u32, vp, u32, C.c_double, pp, pp, pp, C.POINTER(sz),
                                       C.POINTER(abi.TopInfo)], i),
        "alz_group_nodes": ([vp, u32, vp, sz, C.POINTER(sz)], i),
        "alz_group_nodes_device": ([vp, u32, pp, C.POINTER(sz)], i),
        "alz_group_node_metrics": ([vp, u32, u32, vp, u32, vp, sz, C.POINTER(sz)], i),
        "alz_group_node_metrics_device": ([vp, u32, u32, vp, u32, pp, C.POINTER(sz)], i),
        "alz_group_node_top": ([vp, u32, u32, vp, u32, C.c_double, vp, vp, vp, sz, C.POINTER(sz),
                                C.POINTER(abi.TopInfo)], i),
        "alz_group_node_top_device": ([vp, u32, u32, vp, u32, C.c_double, pp, pp, pp, C.POINTER(sz),
                                       C.POINTER(abi.TopInfo)], i),
        "alz_debug_group_edges": ([vp, vp, sz, vp, sz, C.POINTER(sz), C.POINTER(abi.GroupInfo)], i),
        "alz_reach": ([vp, u32, vp, sz, u32, u32, vp, C.c_double, vp, sz, C.POINTER(sz), vp, vp, sz, C.POINTER(sz),
                       C.POINTER(abi.ReachInfo)], i),
        "alz_reach_device": ([vp, u32, vp, sz, u32, u32, vp, C.c_double, pp, C.POINTER(sz), pp, pp, C.POINTER(sz),
                              C.POINTER(abi.ReachInfo)], i),
        "alz_group_reach": ([vp, u32, vp, sz, u32, u32, vp, C.c_double, vp, sz, C.POINTER(sz), vp, vp, sz,
                             C.POINTER(sz), C.POINTER(abi.ReachInfo)], i),
        "alz_group_reach_device": ([vp, u32, vp, sz, u32, u32, vp, C.c_double, pp, C.POINTER(sz), pp, pp,
                                    C.POINTER(sz), C.POINTER(abi.ReachInfo)], i),
        "alz_debug_reach_rows": ([vp, vp, sz, vp, sz, u32, u32, vp, C.c_double, vp, sz, C.POINTER(sz), vp, vp, sz,
                                  C.POINTER(sz), C.POINTER(abi.ReachInfo)], i),
        "alz_cycles": ([vp, u32, vp, C.c_double, u32, vp, sz, C.POINTER(sz), vp, vp, sz, C.POINTER(sz),
                        C.POINTER(abi.CycleInfo)], i),
        "alz_cycles_device": ([vp, u32, vp, C.c_double, u32, pp, C.POINTER(sz), pp, pp, C.POINTER(sz),
                               C.POINTER(abi.CycleInfo)], i),
        "alz_group_cycles": ([vp, u32, vp, C.c_double, u32, vp, sz, C.POINTER(sz), vp, vp, sz, C.POINTER(sz),
                              C.POINTER(abi.CycleInfo)], i),
        "alz_group_cycles_device": ([vp, u32, vp, C.c_double, u32, pp, C.POINTER(sz), pp, pp, C.POINTER(sz),
                                     C.POINTER(abi.CycleInfo)], i),
        "alz_debug_cycles_rows": ([vp, vp, sz, vp, C.c_double, u32, vp, sz, C.POINTER(sz), vp, vp, sz, C.POINTER(sz),
                                   C.POINTER(abi.CycleInfo)], i),
        "alz_group_edge_changes": ([vp, u32, vp, u32, u32, vp, sz, C.POINTER(sz), C.POINTER(abi.ChangeInfo)], i),
        "alz_group_edge_changes_device": ([vp, u32, vp, u32, u32, pp, C.POINTER(sz), C.POINTER(abi.ChangeInfo)], i),
        "alz_group_edge_changes_top": ([vp, u32, vp, u32, u32, u32, C.c_double, vp, sz, C.POINTER(sz),
                                        C.POINTER(abi.ChangeInfo)], i),
        "alz_group_edge_changes_top_device": ([vp, u32, vp, u32, u32, u32, C.c_double, pp, C.POINTER(sz),
                                               C.POINTER(abi.ChangeInfo)], i),
        "alz_group_node_changes": ([vp, u32, u32, vp, u32, u32, vp, sz, C.POINTER(sz), C.POINTER(abi.ChangeInfo)],
                                   i),
        "alz_group_node_changes_device": ([vp, u32, u32, vp, u32, u32, pp, C.POINTER(sz), C.POINTER(abi.ChangeInfo)],
                                          i),
        "alz_group_node_changes_top": ([vp, u32, u32, vp, u32, u32, u32, C.c_double, vp, sz, C.POINTER(sz),
                                        C.POINTER(abi.ChangeInfo)], i),
        "alz_group_node_changes_top_device": ([vp, u32, u32, vp, u32, u32, u32, C.c_double, pp, C.POINTER(sz),
                                               C.POINTER(abi.ChangeInfo)], i),
        "alz_debug_group_edge_changes_rows": ([vp, vp, sz, u32, vp, sz, u32, vp, u32, u32, vp, sz, C.POINTER(sz),
                                               C.POINTER(abi.ChangeInfo)], i),
        "alz_group_edge_series": ([vp, u32, u32, u32, vp, u32, vp, vp, sz, C.POINTER(sz), C.POINTER(u32), vp,
                                   C.POINTER(abi.SeriesInfo)], i),
        "alz_group_edge_series_device": ([vp, u32, u32, u32, vp, u32, pp, pp, C.POINTER(sz), C.POINTER(u32), vp,
                                          C.POINTER(abi.SeriesInfo)], i),
        "alz_group_edge_series_keys": ([vp, vp, sz, u32, u32, vp, u32, vp, vp, sz, C.POINTER(sz), C.POINTER(u32), vp,
                                        C.POINTER(abi.SeriesInfo)], i),
        "alz_group_edge_series_keys_device": ([vp, vp, sz, u32, u32, vp, u32, pp, pp, C.POINTER(sz), C.POINTER(u32),
                                               vp, C.POINTER(abi.SeriesInfo)], i),
        "alz_group_node_series": ([vp, u32, u32, u32, u32, vp, u32, vp, vp, sz, C.POINTER(sz), C.POINTER(u32), vp,
                                   C.POINTER(abi.SeriesInfo)], i),
        "alz_group_node_series_device": ([vp, u32, u32, u32, u32, vp, u32, pp, pp, C.POINTER(sz), C.POINTER(u32), vp,
                                          C.POINTER(abi.SeriesInfo)], i),
        "alz_group_node_series_keys": ([vp, vp, sz, u32, u32, u32, vp, u32, vp, vp, sz, C.POINTER(sz), C.POINTER(u32),
                                        vp, C.POINTER(abi.SeriesInfo)], i),
        "alz_group_node_series_keys_device": ([vp, vp, sz, u32, u32, u32, vp, u32, pp, pp, C.POINTER(sz),
                                               C.POINTER(u32), vp, C.POINTER(abi.SeriesInfo)], i),
        "alz_group_edge_trends": ([vp, u32, u32, u32, vp, C.POINTER(abi.Trend), vp, sz, C.POINTER(sz), C.POINTER(u32),
                                   vp, C.POINTER(abi.TrendInfo)], i),
        "alz_group_edge_trends_device": ([vp, u32, u32, u32, vp, C.POINTER(abi.Trend), pp, C.POINTER(sz),
                                          C.POINTER(u32), vp, C.POINTER(abi.TrendInfo)], i),
        "alz_group_edge_trends_top": ([vp, u32, u32, u32, vp, C.POINTER(abi.Trend), u32, C.c_double, vp, vp, vp, vp,
                                       sz, C.POINTER(sz), C.POINTER(u32), vp, C.POINTER(abi.TrendInfo)], i),
        "alz_group_edge_trends_top_device": ([vp, u32, u32, u32, vp, C.POINTER(abi.Trend), u32, C.c_double, pp, pp,
                                              pp, pp, C.POINTER(sz), C.POINTER(u32), vp, C.POINTER(abi.TrendInfo)], i),
        "alz_group_node_trends": ([vp, u32, u32, u32, u32, vp, C.POINTER(abi.Trend), vp, sz, C.POINTER(sz),
                                   C.POINTER(u32), vp, C.POINTER(abi.TrendInfo)], i),
        "alz_group_node_trends_device": ([vp, u32, u32, u32, u32, vp, C.POINTER(abi.Trend), pp, C.POINTER(sz),
                                          C.POINTER(u32), vp, C.POINTER(abi.TrendInfo)], i),
        "alz_group_node_trends_top": ([vp, u32, u32, u32, u32, vp, C.POINTER(abi.Trend), u32, C.c_double, vp, vp, vp,
                                       vp, sz, C.POINTER(sz), C.POINTER(u32), vp, C.POINTER(abi.TrendInfo)], i),
        "alz_group_node_trends_top_device": ([vp, u32, u32, u32, u32, vp, C.POINTER(abi.Trend), u32, C.c_double, pp,
                                              pp, pp, pp, C.POINTER(sz), C.POINTER(u32), vp,
                                              C.POINTER(abi.TrendInfo)], i),
        "alz_edge_correlations": ([vp, u32, u32, u32, vp, C.POINTER(abi.Corr), C.POINTER(abi.CorrTarget), vp, sz, C.POINTER(sz), C.POINTER(u32), vp,
            C.POINTER(abi.CorrInfo)], i),
        "alz_edge_correlations_device": ([vp, u32, u32, u32, vp, C.POINTER(abi.Corr), C.POINTER(abi.CorrTarget), pp, C.POINTER(sz), C.POINTER(u32),
            vp, C.POINTER(abi.CorrInfo)], i),
        "alz_edge_correlations_top": ([vp, u32, u32, u32, vp, C.POINTER(abi.Corr), C.POINTER(abi.CorrTarget), u32, C.c_double, vp, vp, vp, vp, sz,
            C.POINTER(sz), C.POINTER(u32), vp, C.POINTER(abi.CorrInfo)], i),
        "alz_edge_correlations_top_device": ([vp, u32, u32, u32, vp, C.POINTER(abi.Corr), C.POINTER(abi.CorrTarget), u32, C.c_double, pp, pp, pp,
            pp, C.POINTER(sz), C.POINTER(u32), vp, C.POINTER(abi.CorrInfo)], i),
        "alz_node_correlations": ([vp, u32, u32, u32, u32, vp, C.POINTER(abi.Corr), C.POINTER(abi.CorrTarget), vp, sz, C.POINTER(sz), C.POINTER(u32), vp,
            C.POINTER(abi.CorrInfo)], i),
        "alz_node_correlations_device": ([vp, u32, u32, u32, u32, vp, C.POINTER(abi.Corr), C.POINTER(abi.CorrTarget), pp, C.POINTER(sz), C.POINTER(u32),
            vp, C.POINTER(abi.CorrInfo)], i),
        "alz_node_correlations_top": ([vp, u32, u32, u32, u32, vp, C.POINTER(abi.Corr), C.POINTER(abi.CorrTarget), u32, C.c_double, vp, vp, vp, vp, sz,
            C.POINTER(sz), C.POINTER(u32), vp, C.POINTER(abi.CorrInfo)], i),
        "alz_node_correlations_top_device": ([vp, u32, u32, u32, u32, vp, C.POINTER(abi.Corr), C.POINTER(abi.CorrTarget), u32, C.c_double, pp, pp, pp,
            pp, C.POINTER(sz), C.POINTER(u32), vp, C.POINTER(abi.CorrInfo)], i),
        "alz_group_edge_correlations": ([vp, u32, u32, u32, vp, C.POINTER(abi.Corr), C.POINTER(abi.CorrTarget), vp, sz, C.POINTER(sz), C.POINTER(u32), vp,
            C.POINTER(abi.CorrInfo)], i),
        "alz_group_edge_correlations_device": ([vp, u32, u32, u32, vp, C.POINTER(abi.Corr), C.POINTER(abi.CorrTarget), pp, C.POINTER(sz), C.POINTER(u32),
            vp, C.POINTER(abi.CorrInfo)], i),
        "alz_group_edge_correlations_top": ([vp, u32, u32, u32, vp, C.POINTER(abi.Corr), C.POINTER(abi.CorrTarget), u32, C.c_double, vp, vp, vp, vp, sz,
            C.POINTER(sz), C.POINTER(u32), vp, C.POINTER(abi.CorrInfo)], i),
        "alz_group_edge_correlations_top_device": ([vp, u32, u32, u32, vp, C.POINTER(abi.Corr), C.POINTER(abi.CorrTarget), u32, C.c_double, pp, pp, pp,
            pp, C.POINTER(sz), C.POINTER(u32), vp, C.POINTER(abi.CorrInfo)], i),
        "alz_group_node_correlations": ([vp, u32, u32, u32, u32, vp, C.POINTER(abi.Corr), C.POINTER(abi.CorrTarget), vp, sz, C.POINTER(sz), C.POINTER(u32), vp,
            C.POINTER(abi.CorrInfo)], i),
        "alz_group_node_correlations_device": ([vp, u32, u32, u32, u32, vp, C.POINTER(abi.Corr), C.POINTER(abi.CorrTarget), pp, C.POINTER(sz), C.POINTER(u32),
            vp, C.POINTER(abi.CorrInfo)], i),
        "alz_group_node_correlations_top": ([vp, u32, u32, u32, u32, vp, C.POINTER(abi.Corr), C.POINTER(abi.CorrTarget), u32, C.c_double, vp, vp, vp, vp, sz,
            C.POINTER(sz), C.POINTER(u32), vp, C.POINTER(abi.CorrInfo)], i),
        "alz_group_node_correlations_top_device": ([vp, u32, u32, u32, u32, vp, C.POINTER(abi.Corr), C.POINTER(abi.CorrTarget), u32, C.c_double, pp, pp, pp,
            pp, C.POINTER(sz), C.POINTER(u32), vp, C.POINTER(abi.CorrInfo)], i),
        "alz_debug_corr_series": ([vp, vp, vp, sz, u32, C.POINTER(abi.CorrTarget), C.POINTER(abi.Corr), u32,
                                   C.c_double, vp, vp, sz, C.POINTER(sz), C.POINTER(u64), C.POINTER(u64)], i),
        "alz_edge_quantiles": ([vp, vp, sz, vp], i),
        "alz_submit_tcp": ([vp, vp, sz], i),
        "alz_sock_lookup": ([vp, vp, sz, vp], i),
        "alz_sock_lookup_at": ([vp, vp, sz, vp, u64], i),
        "alz_submit_tcp_raw": ([vp, vp, sz], i),
        "alz_submit_l7_join": ([vp, vp, vp, sz, u64], i),
        "alz_sock_gc": ([vp], i),
        "alz_sock_alive": ([vp, vp, sz, C.POINTER(sz)], i),
        "alz_sock_stats": ([vp, C.POINTER(abi.SockStats)], i),
        "alz_comm_unique_id": ([vp], i),
        "alz_comm_init": ([vp, i, i, vp], i),
        "alz_owner_rank": ([u32, u32], u32),
        "alz_pinned_alloc": ([sz, pp], i),
        "alz_pinned_free": ([vp], i),
        "alz_dev_alloc": ([vp, sz, pp], i),
        "alz_dev_free": ([vp, vp], i),
        "alz_memcpy_h2d": ([vp, vp, vp, sz], i),
        "alz_memcpy_d2h": ([vp, vp, vp, sz], i),
        "alz_fold": ([vp], i),
        "alz_synth_topo_create": ([u32, u64, u32], C.POINTER(abi.SynthTopo)),
        "alz_synth_topo_destroy": ([C.POINTER(abi.SynthTopo)], None),
        "alz_synth_fill": ([C.POINTER(abi.SynthTopo), u64, u64, vp], None),
        "alz_synth_dev_create": ([vp, C.POINTER(abi.SynthTopo), pp], i),
        "alz_synth_dev_fill": ([vp, vp, u64, u64, vp], i),
        "alz_synth_dev_fill_owned": ([vp, vp, u64, u32, u32, vp, u64, C.POINTER(u64), C.POINTER(u64)], i),
        "alz_synth_dev_destroy": ([vp, vp], i),
    }
    if abi.ABI_VERSION < 2:    # A/B timing against a round-1 build (ALZ_LIB_PATH + ALZ_ABI_VERSION=1)
        for k in ("alz_submit_l7_packed", "alz_submit_l7_packed_device", "alz_pack_l7", "alz_window_fetch",
                  "alz_pinned_alloc_local", "alz_table_upsert_batch", "alz_window_clock", "alz_window_epoch",
                  "alz_sock_lookup_at", "alz_submit_l7_join", "alz_sock_gc", "alz_sock_alive", "alz_sock_stats",
                  "alz_submit_tcp_raw", "alz_window_history", "alz_window_rollup", "alz_window_rollup_device",
                  "alz_window_history_tiers", "alz_window_rollup_tier", "alz_window_rollup_tier_device",
                  "alz_window_tier_state", "alz_window_rollup_span", "alz_window_rollup_span_device",
                  "alz_gnn_score_rollup", "alz_gnn_score_rollup_device", "alz_gnn_top", "alz_gnn_top_device",
                  "alz_gnn_top_rollup", "alz_gnn_top_rollup_device", "alz_debug_top_scores", "alz_edge_metrics",
                  "alz_edge_metrics_device", "alz_edge_metrics_rollup", "alz_edge_metrics_rollup_device",
                  "alz_edge_top", "alz_edge_top_device", "alz_edge_top_rollup", "alz_edge_top_rollup_device",
                  "alz_debug_edge_metrics_rows", "alz_debug_top_keys64", "alz_baseline_pin", "alz_baseline_clear",
                  "alz_edge_changes", "alz_edge_changes_device", "alz_edge_changes_top", "alz_edge_changes_top_device",
                  "alz_debug_edge_changes_rows", "alz_edge_series", "alz_edge_series_device", "alz_edge_series_keys",
                  "alz_edge_series_keys_device", "alz_edge_trends", "alz_edge_trends_device", "alz_edge_trends_top",
                  "alz_edge_trends_top_device", "alz_node_rows", "alz_node_rows_device", "alz_node_metrics",
                  "alz_node_metrics_device", "alz_node_top", "alz_node_top_device", "alz_debug_node_rows",
                  "alz_node_series", "alz_node_series_device", "alz_node_series_keys", "alz_node_series_keys_device",
                  "alz_node_trends", "alz_node_trends_device", "alz_node_trends_top", "alz_node_trends_top_device",
                  "alz_node_changes", "alz_node_changes_device", "alz_node_changes_top",
                  "alz_node_changes_top_device", "alz_debug_node_changes_rows", "alz_group_set", "alz_group_edges",
                  "alz_group_edges_device", "alz_group_edge_metrics", "alz_group_edge_metrics_device",
                  "alz_group_edge_top", "alz_group_edge_top_device", "alz_group_nodes", "alz_group_nodes_device",
                  "alz_group_node_metrics", "alz_group_node_metrics_device", "alz_group_node_top",
                  "alz_group_node_top_device", "alz_debug_group_edges", "alz_group_edge_changes",
                  "alz_group_edge_changes_device", "alz_group_edge_changes_top", "alz_group_edge_changes_top_device",
                  "alz_group_node_changes", "alz_group_node_changes_device", "alz_group_node_changes_top",
                  "alz_group_node_changes_top_device", "alz_debug_group_edge_changes_rows",
                  "alz_group_edge_series", "alz_group_edge_series_device", "alz_group_edge_series_keys",
                  "alz_group_edge_series_keys_device", "alz_group_node_series", "alz_group_node_series_device",
                  "alz_group_node_series_keys", "alz_group_node_series_keys_device", "alz_group_edge_trends",
                  "alz_group_edge_trends_device", "alz_group_edge_trends_top", "alz_group_edge_trends_top_device",
                  "alz_group_node_trends", "alz_group_node_trends_device", "alz_group_node_trends_top",
                  "alz_group_node_trends_top_device", "alz_reach", "alz_reach_device", "alz_group_reach",
                  "alz_group_reach_device", "alz_debug_reach_rows", "alz_cycles", "alz_cycles_device",
                  "alz_group_cycles", "alz_group_cycles_device", "alz_debug_cycles_rows", "alz_edge_correlations",
                  "alz_edge_correlations_device", "alz_edge_correlations_top", "alz_edge_correlations_top_device",
                  "alz_node_correlations", "alz_node_correlations_device", "alz_node_correlations_top",
                  "alz_node_correlations_top_device", "alz_group_edge_correlations",
                  "alz_group_edge_correlations_device", "alz_group_edge_correlations_top",
                  "alz_group_edge_correlations_top_device", "alz_group_node_correlations",
                  "alz_group_node_correlations_device", "alz_group_node_correlations_top",
                  "alz_group_node_correlations_top_device", "alz_debug_corr_series"):
            sig.pop(k)
    for name, (args, res) in sig.items():
        f = getattr(L, name)   # AttributeError = header/library mismatch: loud
        f.argtypes, f.restype = args, res
    _lib = L
    return L


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


class PinnedBuffer:
    """Library-owned pinned host memory exposed as a numpy array."""

    def __init__(self, n, dtype, handle=None):
        """handle: allocate on the NUMA node next to that handle's GPU (alz_pinned_alloc_local)."""
        self.L = load()
        self.dtype = np.dtype(dtype)
        self.nbytes = int(n) * self.dtype.itemsize
        p = C.c_void_p()
        if handle is not None and abi.ABI_VERSION >= 2:
            rc = self.L.alz_pinned_alloc_local(handle.h, max(self.nbytes, 1), C.byref(p))
        else:
            rc = self.L.alz_pinned_alloc(max(self.nbytes, 1), C.byref(p))
        if rc != 0:
            raise AlzError(rc, "alz_pinned_alloc")
        self.ptr = p.value
        buf = (C.c_char * max(self.nbytes, 1)).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=self.dtype, count=int(n))

    def free(self):
        if self.ptr:
            self.array = None
            self.L.alz_pinned_free(self.ptr)
            self.ptr = None


class Handle:
    """One GPU's aggregator instance (alz_handle)."""

    def __init__(self, device=0, max_endpoints=1 << 16, max_pairs=1 << 20, max_edges=0,
                 max_batch=1 << 22, flags=0):
        self.L = load()
        cfg = abi.Config(abi_version=abi.ABI_VERSION, device=device, max_endpoints=max_endpoints,
                         max_pairs=max_pairs, max_edges=max_edges, max_batch=max_batch, flags=flags)
        h = C.c_void_p()
        rc = self.L.alz_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise AlzError(rc, "alz_create", self.L.alz_strerror(rc).decode())
        self.h = h
        self.max_edges = max_edges or max_pairs

    def _ck(self, rc, what, allow=()):
        if rc != 0 and rc not in allow:
            raise AlzError(rc, what, self.L.alz_strerror(rc).decode() + " | " +
                           self.L.alz_last_cuda_error(self.h).decode())
        return rc

    def close(self):
        if getattr(self, "h", None):
            self.L.alz_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- tables
    def upsert(self, table, ip, id_):
        self._ck(self.L.alz_table_upsert(self.h, table, int(ip), int(id_)), "alz_table_upsert")

    def erase(self, table, ip):
        self._ck(self.L.alz_table_erase(self.h, table, int(ip)), "alz_table_erase")

    def commit(self):
        self._ck(self.L.alz_table_commit(self.h), "alz_table_commit")

    def upsert_batch(self, table, ips, ids):
        ips = np.ascontiguousarray(ips, dtype=np.uint32)
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        assert len(ips) == len(ids)
        self._ck(self.L.alz_table_upsert_batch(self.h, table, _ptr(ips), _ptr(ids), len(ips)), "alz_table_upsert_batch")

    def load_tables(self, pod_ip, svc_ip):
        if abi.ABI_VERSION < 2:
            for k, v in enumerate(pod_ip):
                self.upsert(abi.TABLE_POD, int(v), k)
            for k, v in enumerate(svc_ip):
                self.upsert(abi.TABLE_SVC, int(v), k)
        else:
            self.upsert_batch(abi.TABLE_POD, pod_ip, np.arange(len(pod_ip)))
            self.upsert_batch(abi.TABLE_SVC, svc_ip, np.arange(len(svc_ip)))
        self.commit()

    # ---- ingest
    def submit(self, recs):
        recs = np.ascontiguousarray(recs, dtype=abi.L7_REC)
        self._ck(self.L.alz_submit_l7(self.h, _ptr(recs), len(recs)), "alz_submit_l7")

    def submit_ptr(self, host_ptr, n):
        self._ck(self.L.alz_submit_l7(self.h, C.c_void_p(host_ptr), n), "alz_submit_l7")

    def submit_device(self, dev_ptr, n):
        self._ck(self.L.alz_submit_l7_device(self.h, C.c_void_p(dev_ptr), n), "alz_submit_l7_device")

    def submit_packed(self, recs16, overflow=None):
        recs16 = np.ascontiguousarray(recs16, dtype=abi.L7_REC16)
        ovf = np.ascontiguousarray(overflow if overflow is not None else np.zeros(0, np.uint64), dtype=np.uint64)
        self._ck(self.L.alz_submit_l7_packed(self.h, _ptr(recs16), len(recs16), _ptr(ovf) if len(ovf) else None,
                                             len(ovf)), "alz_submit_l7_packed")

    def submit_packed_ptr(self, host_ptr, n, ovf_ptr=None, n_ovf=0):
        self._ck(self.L.alz_submit_l7_packed(self.h, C.c_void_p(host_ptr), n, C.c_void_p(ovf_ptr) if ovf_ptr else None,
                                             n_ovf), "alz_submit_l7_packed")

    def submit_packed_device(self, dev_ptr, n, dev_ovf=None):
        """alz_submit_l7_packed_device: n 16-B records already in device memory; dev_ovf the device array of overflow
        durations their indices point into (None: no record has ALZ_REC16_DUR_OVERFLOW)."""
        self._ck(self.L.alz_submit_l7_packed_device(self.h, C.c_void_p(dev_ptr), n,
                                                    C.c_void_p(dev_ovf) if dev_ovf else None),
                 "alz_submit_l7_packed_device")

    def submit_raw(self, raw):
        raw = np.ascontiguousarray(raw, dtype=np.uint8)
        n = raw.size // abi.BPF_L7_EVENT_SIZE
        self._ck(self.L.alz_submit_l7_raw(self.h, _ptr(raw), n), "alz_submit_l7_raw")

    def submit_raw_ptr(self, host_ptr, n):
        self._ck(self.L.alz_submit_l7_raw(self.h, C.c_void_p(host_ptr), n), "alz_submit_l7_raw")

    # ---- results
    def flush(self, cap=None):
        cap = self.max_edges if cap is None else cap
        out = np.zeros(cap, dtype=abi.EDGE_OUT)
        n = C.c_size_t(0)
        self._ck(self.L.alz_window_flush(self.h, _ptr(out), cap, C.byref(n)), "alz_window_flush")
        return out[: n.value].copy()

    def flush_device(self):
        p = C.c_void_p()
        n = C.c_size_t(0)
        self._ck(self.L.alz_window_flush_device(self.h, C.byref(p), C.byref(n)), "alz_window_flush_device")
        return p.value, n.value

    def stats(self):
        st = abi.Stats()
        self._ck(self.L.alz_get_stats(self.h, C.byref(st)), "alz_get_stats")
        return st.as_dict()

    # ---- tcp_state sink + socket timelines (alz_sock.cu) ----
    def submit_tcp(self, recs):
        recs = np.ascontiguousarray(recs, dtype=abi.TCP_REC)
        self._ck(self.L.alz_submit_tcp(self.h, _ptr(recs), len(recs)), "alz_submit_tcp")

    def sock_lookup(self, q, now_ns=None):
        q = np.ascontiguousarray(q, dtype=abi.SOCK_QUERY)
        out = np.zeros(len(q), dtype=abi.SOCK_RESULT)
        if now_ns is None:
            self._ck(self.L.alz_sock_lookup(self.h, _ptr(q), len(q), _ptr(out)), "alz_sock_lookup")
        else:
            self._ck(self.L.alz_sock_lookup_at(self.h, _ptr(q), len(q), _ptr(out), int(now_ns)), "alz_sock_lookup_at")
        return out

    def submit_join(self, recs, keys, now_ns=0):
        recs = np.ascontiguousarray(recs, dtype=abi.L7_REC)
        keys = np.ascontiguousarray(keys, dtype=abi.SOCK_QUERY)
        assert len(recs) == len(keys)
        self._ck(self.L.alz_submit_l7_join(self.h, _ptr(recs), _ptr(keys), len(recs), int(now_ns)), "alz_submit_l7_join")

    def sock_gc(self):
        self._ck(self.L.alz_sock_gc(self.h), "alz_sock_gc")

    def sock_alive(self, cap=1 << 20):
        out = np.zeros(cap, dtype=abi.ALIVE_CONN)
        n = C.c_size_t(0)
        self._ck(self.L.alz_sock_alive(self.h, _ptr(out), cap, C.byref(n)), "alz_sock_alive")
        return out[: n.value]

    def sock_stats(self):
        st = abi.SockStats()
        self._ck(self.L.alz_sock_stats(self.h, C.byref(st)), "alz_sock_stats")
        return st.as_dict()

    def window_clock(self, first_kernel_ns, first_user_ns, window_ns):
        self._ck(self.L.alz_window_clock(self.h, int(first_kernel_ns), int(first_user_ns), int(window_ns)),
                 "alz_window_clock")

    def window_epoch(self):
        e = C.c_uint64(0)
        self._ck(self.L.alz_window_epoch(self.h, C.byref(e)), "alz_window_epoch")
        return e.value

    # ---- rolling windows (alz_rollup.cu)
    def window_history(self, depth, arena_rows):
        self._ck(self.L.alz_window_history(self.h, int(depth), int(arena_rows)), "alz_window_history")

    def _rollup(self, fn, args, info, cap):
        """fn(h, *args, out, cap, &n, &info): (rows, info dict). cap=None sizes the buffer from a first call with
        cap 0."""
        f, n = getattr(self.L, fn), C.c_size_t(0)
        if cap is None:
            if self._ck(f(self.h, *args, None, 0, C.byref(n), C.byref(info)), fn, allow=(abi.E_CAPACITY,)) == 0:
                return np.zeros(0, dtype=abi.EDGE_OUT), info.as_dict()
            cap = n.value
        out = np.zeros(cap, dtype=abi.EDGE_OUT)
        self._ck(f(self.h, *args, _ptr(out), cap, C.byref(n), C.byref(info)), fn)
        return out[: n.value].copy(), info.as_dict()

    def _rollup_device(self, fn, args, info):
        """fn(h, *args, &dev_rows, &n, &info): (device pointer, rows, info dict)."""
        p, n = C.c_void_p(), C.c_size_t(0)
        self._ck(getattr(self.L, fn)(self.h, *args, C.byref(p), C.byref(n), C.byref(info)), fn)
        return p.value, n.value, info.as_dict()

    def rollup(self, k, cap=None):
        """alz_window_rollup: (rows, info dict). cap=None sizes the buffer from a first call with cap 0."""
        return self._rollup("alz_window_rollup", (int(k),), abi.RollupInfo(), cap)

    def rollup_device(self, k):
        """alz_window_rollup_device: (device pointer, rows, info dict)."""
        return self._rollup_device("alz_window_rollup_device", (int(k),), abi.RollupInfo())

    # ---- tiered history (alz_rollup.cu, docs/SPEC.md §13)
    def window_history_tiers(self, tiers):
        """tiers: a list of (factor, depth, arena_rows, block_rows), tier 1 first; [] turns the tiers off."""
        arr = (abi.HistoryTier * max(len(tiers), 1))(*[abi.HistoryTier(*map(int, t)) for t in tiers])
        self._ck(self.L.alz_window_history_tiers(self.h, arr, len(tiers)), "alz_window_history_tiers")

    def rollup_tier(self, tier, k, cap=None):
        """alz_window_rollup_tier: (rows, info dict). cap=None sizes the buffer from a first call with cap 0."""
        return self._rollup("alz_window_rollup_tier", (int(tier), int(k)), abi.RollupInfo(), cap)

    def rollup_tier_device(self, tier, k):
        """alz_window_rollup_tier_device: (device pointer, rows, info dict)."""
        return self._rollup_device("alz_window_rollup_tier_device", (int(tier), int(k)), abi.RollupInfo())

    def tier_state(self, tier):
        st = abi.TierState()
        self._ck(self.L.alz_window_tier_state(self.h, int(tier), C.byref(st)), "alz_window_tier_state")
        return st.as_dict()

    # ---- span rollups (alz_rollup.cu, docs/SPEC.md §14)
    def rollup_span(self, windows, mode=abi.SPAN_AT_MOST, cap=None):
        """alz_window_rollup_span: (rows, info dict). cap=None sizes the buffer from a first call with cap 0."""
        return self._rollup("alz_window_rollup_span", (int(windows), int(mode)), abi.SpanInfo(), cap)

    def rollup_span_device(self, windows, mode=abi.SPAN_AT_MOST):
        """alz_window_rollup_span_device: (device pointer, rows, info dict)."""
        return self._rollup_device("alz_window_rollup_span_device", (int(windows), int(mode)), abi.SpanInfo())

    # ---- GNN anomaly pass over a rollup (alz_gnn.cu, docs/SPEC.md §15)
    def gnn_score_rollup(self, kind, cap=None):
        """alz_gnn_score_rollup: the scores of the rows the last rollup of `kind` (abi.ROLLUP_*) returned, one per
        row. cap=None sizes the buffer from a first call with cap 0."""
        n = C.c_size_t(0)
        if cap is None:
            if self._ck(self.L.alz_gnn_score_rollup(self.h, int(kind), None, 0, C.byref(n)), "alz_gnn_score_rollup",
                        allow=(abi.E_CAPACITY,)) == 0:
                return np.zeros(0, dtype=np.float32)
            cap = n.value
        out = np.zeros(cap, dtype=np.float32)
        self._ck(self.L.alz_gnn_score_rollup(self.h, int(kind), _ptr(out), cap, C.byref(n)), "alz_gnn_score_rollup")
        return out[: n.value].copy()

    def gnn_score_rollup_device(self, kind):
        """alz_gnn_score_rollup_device: (device pointer, scores)."""
        p, n = C.c_void_p(), C.c_size_t(0)
        self._ck(self.L.alz_gnn_score_rollup_device(self.h, int(kind), C.byref(p), C.byref(n)),
                 "alz_gnn_score_rollup_device")
        return p.value, n.value

    # ---- top anomalous rows (alz_gnn.cu, docs/SPEC.md §16)
    def _top(self, fn, args, k, min_score):
        """fn(h, *args, k, min_score, rows, scores, index, cap, &n, &info): (rows, scores, index, info dict). The first
        call offers room for min(k, 65536) results; when more came out, the call is repeated with room for all."""
        f, n, info = getattr(self.L, fn), C.c_size_t(0), abi.TopInfo()
        cap = min(int(k), 1 << 16)
        while True:
            rows = np.zeros(cap, dtype=abi.EDGE_OUT)
            scores = np.zeros(cap, dtype=np.float32)
            index = np.zeros(cap, dtype=np.uint32)
            rc = self._ck(f(self.h, *args, int(k), float(min_score), _ptr(rows), _ptr(scores), _ptr(index), cap,
                            C.byref(n), C.byref(info)), fn, allow=(abi.E_CAPACITY,))
            if rc == 0:
                m = n.value
                return rows[:m].copy(), scores[:m].copy(), index[:m].copy(), info.as_dict()
            cap = n.value

    def _top_device(self, fn, args, k, min_score):
        """fn(h, *args, k, min_score, &rows, &scores, &index, &n, &info): (rows, scores, index device pointers, results,
        info dict)."""
        pr, ps, pi, n, info = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_size_t(0), abi.TopInfo()
        self._ck(getattr(self.L, fn)(self.h, *args, int(k), float(min_score), C.byref(pr), C.byref(ps), C.byref(pi),
                                     C.byref(n), C.byref(info)), fn)
        return pr.value, ps.value, pi.value, n.value, info.as_dict()

    def gnn_top(self, k, min_score=0.0):
        """alz_gnn_top over the last flushed window: (rows, scores, index, info dict), rank order."""
        return self._top("alz_gnn_top", (), k, min_score)

    def gnn_top_device(self, k, min_score=0.0):
        """alz_gnn_top_device: (rows, scores, index device pointers, results, info dict)."""
        return self._top_device("alz_gnn_top_device", (), k, min_score)

    def gnn_top_rollup(self, kind, k, min_score=0.0):
        """alz_gnn_top_rollup over the rows the last rollup of `kind` (abi.ROLLUP_*) returned: (rows, scores, index,
        info dict), rank order."""
        return self._top("alz_gnn_top_rollup", (int(kind),), k, min_score)

    def gnn_top_rollup_device(self, kind, k, min_score=0.0):
        """alz_gnn_top_rollup_device: (rows, scores, index device pointers, results, info dict)."""
        return self._top_device("alz_gnn_top_rollup_device", (int(kind),), k, min_score)

    # ---- edge metrics and the top edges by a metric (alz_metrics.cu, docs/SPEC.md §17)
    def _edge_metrics(self, fn, args, specs):
        """fn(h, *args, m, nm, values, cap, &n): values [rows x nm] float64; the first call with cap 0 sizes it."""
        m, nm = abi.metrics(*specs), len(specs)
        f, n = getattr(self.L, fn), C.c_size_t(0)
        if self._ck(f(self.h, *args, m, nm, None, 0, C.byref(n)), fn, allow=(abi.E_CAPACITY,)) == 0:
            return np.zeros((0, nm))
        out = np.zeros((n.value, nm))
        self._ck(f(self.h, *args, m, nm, _ptr(out), n.value, C.byref(n)), fn)
        return out

    def _edge_metrics_device(self, fn, args, specs):
        """fn(h, *args, m, nm, &values, &n): (device pointer, rows)."""
        p, n = C.c_void_p(), C.c_size_t(0)
        self._ck(getattr(self.L, fn)(self.h, *args, abi.metrics(*specs), len(specs), C.byref(p), C.byref(n)), fn)
        return p.value, n.value

    def edge_metrics(self, *specs):
        """alz_edge_metrics over the last flushed window: values [rows x len(specs)]; a spec is a METRIC_* kind or a
        (kind, q) pair."""
        return self._edge_metrics("alz_edge_metrics", (), specs)

    def edge_metrics_device(self, *specs):
        """alz_edge_metrics_device: (device pointer, rows)."""
        return self._edge_metrics_device("alz_edge_metrics_device", (), specs)

    def edge_metrics_rollup(self, kind, *specs):
        """alz_edge_metrics_rollup over the rows the last rollup of `kind` (abi.ROLLUP_*) returned."""
        return self._edge_metrics("alz_edge_metrics_rollup", (int(kind),), specs)

    def edge_metrics_rollup_device(self, kind, *specs):
        """alz_edge_metrics_rollup_device: (device pointer, rows)."""
        return self._edge_metrics_device("alz_edge_metrics_rollup_device", (int(kind),), specs)

    def _edge_top(self, fn, args, spec, k, min_value):
        """fn(h, *args, m, k, min_value, rows, values, index, cap, &n, &info): (rows, values, index, info dict). The
        first call offers room for min(k, 65536) results; when more came out, the call is repeated with room for all."""
        f, n, info, m = getattr(self.L, fn), C.c_size_t(0), abi.TopInfo(), abi.metrics(spec)
        cap = min(int(k), 1 << 16)
        while True:
            rows = np.zeros(cap, dtype=abi.EDGE_OUT)
            values = np.zeros(cap, dtype=np.float64)
            index = np.zeros(cap, dtype=np.uint32)
            rc = self._ck(f(self.h, *args, m, int(k), float(min_value), _ptr(rows), _ptr(values), _ptr(index), cap,
                            C.byref(n), C.byref(info)), fn, allow=(abi.E_CAPACITY,))
            if rc == 0:
                r = n.value
                return rows[:r].copy(), values[:r].copy(), index[:r].copy(), info.as_dict()
            cap = n.value

    def _edge_top_device(self, fn, args, spec, k, min_value):
        """fn(h, *args, m, k, min_value, &rows, &values, &index, &n, &info): (rows, values, index device pointers,
        results, info dict)."""
        pr, pv, pi, n, info = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_size_t(0), abi.TopInfo()
        self._ck(getattr(self.L, fn)(self.h, *args, abi.metrics(spec), int(k), float(min_value), C.byref(pr),
                                     C.byref(pv), C.byref(pi), C.byref(n), C.byref(info)), fn)
        return pr.value, pv.value, pi.value, n.value, info.as_dict()

    def edge_top(self, spec, k, min_value=0.0):
        """alz_edge_top over the last flushed window by one metric (a METRIC_* kind or a (kind, q) pair): (rows,
        values, index, info dict), rank order."""
        return self._edge_top("alz_edge_top", (), spec, k, min_value)

    def edge_top_device(self, spec, k, min_value=0.0):
        """alz_edge_top_device: (rows, values, index device pointers, results, info dict)."""
        return self._edge_top_device("alz_edge_top_device", (), spec, k, min_value)

    def edge_top_rollup(self, kind, spec, k, min_value=0.0):
        """alz_edge_top_rollup over the rows the last rollup of `kind` (abi.ROLLUP_*) returned."""
        return self._edge_top("alz_edge_top_rollup", (int(kind),), spec, k, min_value)

    def edge_top_rollup_device(self, kind, spec, k, min_value=0.0):
        """alz_edge_top_rollup_device: (rows, values, index device pointers, results, info dict)."""
        return self._edge_top_device("alz_edge_top_rollup_device", (int(kind),), spec, k, min_value)

    # ---- edge changes against a pinned baseline (alz_changes.cu, docs/SPEC.md §18)
    def baseline_pin(self, source=abi.SOURCE_WINDOW):
        """alz_baseline_pin: the rows of `source` (abi.SOURCE_WINDOW or abi.ROLLUP_*) become the baseline; its info
        dict."""
        info = abi.RollupInfo()
        self._ck(self.L.alz_baseline_pin(self.h, int(source), C.byref(info)), "alz_baseline_pin")
        return info.as_dict()

    def baseline_clear(self):
        self._ck(self.L.alz_baseline_clear(self.h), "alz_baseline_clear")

    def _changes(self, fn, args, dtype=abi.EDGE_CHANGE):
        """fn(h, *args, out, cap, &n, &info): (alz_edge_change or alz_node_change records, info dict); a first call with
        cap 0 sizes the buffer (ALZ_E_CAPACITY when there are records)."""
        f, n, info = getattr(self.L, fn), C.c_size_t(0), abi.ChangeInfo()
        cap = 0
        while True:
            out = np.zeros(cap, dtype=dtype)
            rc = self._ck(f(self.h, *args, _ptr(out) if cap else None, cap, C.byref(n), C.byref(info)), fn,
                          allow=(abi.E_CAPACITY,))
            if rc == 0:
                return out[: n.value].copy(), info.as_dict()
            if n.value <= cap:   # a capacity error that no buffer cures: the union is too large
                raise AlzError(rc, fn)
            cap = n.value

    def edge_changes(self, spec, mode=abi.CHANGE_DELTA, presence=abi.PRESENT_ALL, source=abi.SOURCE_WINDOW):
        """alz_edge_changes of `source` against the pinned baseline by one metric (a METRIC_* kind or a (kind, q)
        pair): (records in ascending key order, info dict)."""
        return self._changes("alz_edge_changes", (int(source), abi.metrics(spec), int(mode), int(presence)))

    def edge_changes_device(self, spec, mode=abi.CHANGE_DELTA, presence=abi.PRESENT_ALL, source=abi.SOURCE_WINDOW):
        """alz_edge_changes_device: (device pointer, records, info dict)."""
        p, n, info = C.c_void_p(), C.c_size_t(0), abi.ChangeInfo()
        self._ck(self.L.alz_edge_changes_device(self.h, int(source), abi.metrics(spec), int(mode), int(presence),
                                                C.byref(p), C.byref(n), C.byref(info)), "alz_edge_changes_device")
        return p.value, n.value, info.as_dict()

    def edge_changes_top(self, spec, k, min_change=0.0, mode=abi.CHANGE_DELTA, presence=abi.PRESENT_ALL,
                         source=abi.SOURCE_WINDOW):
        """alz_edge_changes_top: (the first min(k, above) records by change, rank order; info dict)."""
        return self._changes("alz_edge_changes_top", (int(source), abi.metrics(spec), int(mode), int(presence),
                                                      int(k), float(min_change)))

    def edge_changes_top_device(self, spec, k, min_change=0.0, mode=abi.CHANGE_DELTA, presence=abi.PRESENT_ALL,
                                source=abi.SOURCE_WINDOW):
        """alz_edge_changes_top_device: (device pointer, records, info dict)."""
        p, n, info = C.c_void_p(), C.c_size_t(0), abi.ChangeInfo()
        self._ck(self.L.alz_edge_changes_top_device(self.h, int(source), abi.metrics(spec), int(mode), int(presence),
                                                    int(k), float(min_change), C.byref(p), C.byref(n),
                                                    C.byref(info)), "alz_edge_changes_top_device")
        return p.value, n.value, info.as_dict()

    def debug_edge_changes_rows(self, src, base, spec, mode=abi.CHANGE_DELTA, presence=abi.PRESENT_ALL,
                                src_windows=1, base_windows=1):
        """alz_debug_edge_changes_rows over two host row arrays (copied to the device, each in strictly ascending
        key order): (records, info dict)."""
        src = np.ascontiguousarray(src, dtype=abi.EDGE_OUT)
        base = np.ascontiguousarray(base, dtype=abi.EDGE_OUT)
        ps = self.dev_alloc(max(src.nbytes, 1))
        pb = self.dev_alloc(max(base.nbytes, 1))
        try:
            if len(src):
                self.h2d(ps, src)
            if len(base):
                self.h2d(pb, base)
            return self._changes("alz_debug_edge_changes_rows",
                                 (C.c_void_p(ps), len(src), int(src_windows), C.c_void_p(pb), len(base),
                                  int(base_windows), abi.metrics(spec), int(mode), int(presence)))
        finally:
            self.dev_free(ps)
            self.dev_free(pb)

    # ---- edge series (alz_series.cu, docs/SPEC.md §19)
    @staticmethod
    def edge_ends(edges):
        """An EDGE_ENDS array from an EDGE_ENDS or EDGE_OUT array (its key fields), or (from_type, from, to_type, to)
        tuples."""
        if isinstance(edges, np.ndarray) and edges.dtype.names:
            out = np.zeros(len(edges), dtype=abi.EDGE_ENDS)
            for f in ("from_type", "to_type", "from", "to"):
                out[f] = edges[f]
            return out
        out = np.zeros(len(edges), dtype=abi.EDGE_ENDS)
        for i, (ft, f, tt, t) in enumerate(edges):
            out[i] = (ft, tt, (0,) * 6, f, t)
        return out

    def _series(self, fn, head, tail, specs):
        """fn(h, *head, *tail, m, nm, values, present, cap, &n, &P, points, &info): (values [n, P, nm] float64,
        present [n, P] uint8, points as a list of alz_rollup_info dicts, info dict). A first call with cap 0 and no
        points gives n and P."""
        m, nm = abi.metrics(*specs), len(specs)
        f, n, p, info = getattr(self.L, fn), C.c_size_t(0), C.c_uint32(0), abi.SeriesInfo()
        self._ck(f(self.h, *head, *tail, m, nm, None, None, 0, C.byref(n), C.byref(p), None, C.byref(info)), fn,
                 allow=(abi.E_CAPACITY,))
        rows, P = n.value, p.value
        values = np.zeros((rows, P, nm))
        present = np.zeros((rows, P), dtype=np.uint8)
        points = (abi.RollupInfo * max(P, 1))()
        self._ck(f(self.h, *head, *tail, m, nm, _ptr(values), _ptr(present), rows, C.byref(n), C.byref(p), points,
                   C.byref(info)), fn)
        return values, present, [points[j].as_dict() for j in range(P)], info.as_dict()

    def _series_device(self, fn, head, tail, specs):
        """fn(h, *head, *tail, m, nm, &values, &present, &n, &P, points, &info): (values and present device pointers,
        n, P, points, info dict). points has room for k entries."""
        pv, pp_, n, p, info = C.c_void_p(), C.c_void_p(), C.c_size_t(0), C.c_uint32(0), abi.SeriesInfo()
        k = int(tail[-1])
        points = (abi.RollupInfo * max(min(k, 1 << 16), 1))()
        self._ck(getattr(self.L, fn)(self.h, *head, *tail, abi.metrics(*specs), len(specs), C.byref(pv), C.byref(pp_),
                                     C.byref(n), C.byref(p), points if k <= (1 << 16) else None, C.byref(info)), fn)
        pts = [points[j].as_dict() for j in range(p.value)] if k <= (1 << 16) else None
        return pv.value, pp_.value, n.value, p.value, pts, info.as_dict()

    def edge_series(self, source, tier, k, *specs):
        """alz_edge_series: every row of `source` (abi.SOURCE_WINDOW or abi.ROLLUP_*) over the last k entries of
        `tier` (0: the window history): (values [rows, P, nm], present [rows, P], points, info dict)."""
        return self._series("alz_edge_series", (int(source),), (int(tier), int(k)), specs)

    def edge_series_device(self, source, tier, k, *specs):
        """alz_edge_series_device: (values and present device pointers, rows, P, points, info dict)."""
        return self._series_device("alz_edge_series_device", (int(source),), (int(tier), int(k)), specs)

    def edge_series_keys(self, edges, tier, k, *specs):
        """alz_edge_series_keys: the caller's edges (see edge_ends), in their order, over the last k entries of
        `tier`: (values [n, P, nm], present [n, P], points, info dict)."""
        keys = np.ascontiguousarray(self.edge_ends(edges))
        return self._series("alz_edge_series_keys", (_ptr(keys), len(keys)), (int(tier), int(k)), specs)

    def edge_series_keys_device(self, edges, tier, k, *specs):
        """alz_edge_series_keys_device: (values and present device pointers, n, P, points, info dict)."""
        keys = np.ascontiguousarray(self.edge_ends(edges))
        return self._series_device("alz_edge_series_keys_device", (_ptr(keys), len(keys)), (int(tier), int(k)), specs)

    # ---- edge trends (alz_trends.cu, docs/SPEC.md §20)
    @staticmethod
    def trend(stat=abi.TREND_SLOPE, direction=abi.TREND_RISING, absent=abi.TREND_ABSENT_SKIP, recent=1, min_points=0):
        """An alz_trend."""
        return abi.Trend(int(stat), int(direction), int(absent), int(recent), int(min_points), 0)

    def _trends(self, fn, head, k, spec, trend, dtype):
        """fn(h, *head, k, m, &trend, out, cap, &n, &P, points, &info): (records in source order, points, info dict).
        A first call with cap 0 gives the records."""
        f, n, p, info, m = getattr(self.L, fn), C.c_size_t(0), C.c_uint32(0), abi.TrendInfo(), abi.metrics(spec)
        self._ck(f(self.h, *head, int(k), m, C.byref(trend), None, 0, C.byref(n), C.byref(p), None, C.byref(info)), fn,
                 allow=(abi.E_CAPACITY,))
        out = np.zeros(n.value, dtype=dtype)
        points = (abi.RollupInfo * max(int(k), 1))()
        self._ck(f(self.h, *head, int(k), m, C.byref(trend), _ptr(out), len(out), C.byref(n), C.byref(p), points,
                   C.byref(info)), fn)
        return out, [points[j].as_dict() for j in range(p.value)], info.as_dict()

    def _trends_device(self, fn, head, k, spec, trend):
        d, n, p, info = C.c_void_p(), C.c_size_t(0), C.c_uint32(0), abi.TrendInfo()
        points = (abi.RollupInfo * max(int(k), 1))()
        self._ck(getattr(self.L, fn)(self.h, *head, int(k), abi.metrics(spec), C.byref(trend), C.byref(d), C.byref(n),
                                     C.byref(p), points, C.byref(info)), fn)
        return d.value, n.value, p.value, [points[j].as_dict() for j in range(p.value)], info.as_dict()

    def _trends_top(self, fn, head, k, spec, trend, top, min_trend, rec_dtype, row_dtype):
        """fn(h, *head, k, m, &trend, top, min_trend, out, rows, series, present, cap, &n, &P, points, &info). The
        first call offers room for min(top, 4096) results; when more came out, it is repeated with room for all."""
        f, n, p, info, m = getattr(self.L, fn), C.c_size_t(0), C.c_uint32(0), abi.TrendInfo(), abi.metrics(spec)
        cap = min(int(top), 1 << 12)
        points = (abi.RollupInfo * max(int(k), 1))()
        while True:
            out = np.zeros(cap, dtype=rec_dtype)
            rows = np.zeros(cap, dtype=row_dtype)
            series = np.zeros(cap * int(k))
            present = np.zeros(cap * int(k), dtype=np.uint8)
            rc = self._ck(f(self.h, *head, int(k), m, C.byref(trend), int(top), float(min_trend), _ptr(out),
                            _ptr(rows), _ptr(series), _ptr(present), cap, C.byref(n), C.byref(p), points,
                            C.byref(info)), fn, allow=(abi.E_CAPACITY,))
            if rc == 0:
                break
            if n.value <= cap:   # a capacity error that no buffer cures: too many slots
                raise AlzError(rc, fn)
            cap = n.value
        r, P = n.value, p.value
        return (out[:r].copy(), rows[:r].copy(), series[: r * P].reshape(r, P).copy(),
                present[: r * P].reshape(r, P).copy(), [points[j].as_dict() for j in range(P)], info.as_dict())

    def _trends_top_device(self, fn, head, k, spec, trend, top, min_trend):
        pr, pw, ps, pp_ = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
        n, p, info = C.c_size_t(0), C.c_uint32(0), abi.TrendInfo()
        points = (abi.RollupInfo * max(int(k), 1))()
        self._ck(getattr(self.L, fn)(self.h, *head, int(k), abi.metrics(spec), C.byref(trend), int(top),
                                     float(min_trend), C.byref(pr), C.byref(pw), C.byref(ps), C.byref(pp_), C.byref(n),
                                     C.byref(p), points, C.byref(info)), fn)
        return (pr.value, pw.value, ps.value, pp_.value, n.value, p.value, [points[j].as_dict() for j in range(p.value)],
                info.as_dict())

    def edge_trends(self, source, tier, k, spec, trend):
        """alz_edge_trends: every row of `source` (abi.SOURCE_WINDOW or abi.ROLLUP_*) over the last k entries of
        `tier` by one metric (a METRIC_* kind or a (kind, q) pair) and an abi.Trend: (EDGE_TREND records in source
        order, points as a list of alz_rollup_info dicts, info dict). A first call with cap 0 gives the rows."""
        return self._trends("alz_edge_trends", (int(source), int(tier)), k, spec, trend, abi.EDGE_TREND)

    def edge_trends_device(self, source, tier, k, spec, trend):
        """alz_edge_trends_device: (device pointer to the records, rows, P, points, info dict)."""
        return self._trends_device("alz_edge_trends_device", (int(source), int(tier)), k, spec, trend)

    def edge_trends_top(self, source, tier, k, spec, trend, top, min_trend=-np.inf):
        """alz_edge_trends_top: the first min(top, above) valid rows by trend, rank order: (records, source rows,
        series [m, P] float64, present [m, P] uint8, points, info dict). The first call offers room for min(top, 4096) results; when more came out, it is repeated with room for all."""
        return self._trends_top("alz_edge_trends_top", (int(source), int(tier)), k, spec, trend, top, min_trend,
                                abi.EDGE_TREND, abi.EDGE_OUT)

    def edge_trends_top_device(self, source, tier, k, spec, trend, top, min_trend=-np.inf):
        """alz_edge_trends_top_device: (records, rows, series and present device pointers, results, P, points, info
        dict)."""
        return self._trends_top_device("alz_edge_trends_top_device", (int(source), int(tier)), k, spec, trend, top,
                                       min_trend)

    # ---- node metrics (alz_nodes.cu, docs/SPEC.md §21)
    def _node_rows(self, fn, args):
        """fn(h, *args, out, cap, &n): NODE_OUT rows in node order; a first call with cap 0 gives the nodes."""
        f, n = getattr(self.L, fn), C.c_size_t(0)
        if self._ck(f(self.h, *args, None, 0, C.byref(n)), fn, allow=(abi.E_CAPACITY,)) == 0:
            return np.zeros(0, dtype=abi.NODE_OUT)
        out = np.zeros(n.value, dtype=abi.NODE_OUT)
        self._ck(f(self.h, *args, _ptr(out), n.value, C.byref(n)), fn)
        return out

    def node_rows(self, source=abi.SOURCE_WINDOW):
        """alz_node_rows: every node of `source` (abi.SOURCE_WINDOW or abi.ROLLUP_*) as NODE_OUT rows, node order."""
        return self._node_rows("alz_node_rows", (int(source),))

    def node_rows_device(self, source=abi.SOURCE_WINDOW):
        """alz_node_rows_device: (device pointer, nodes)."""
        p, n = C.c_void_p(), C.c_size_t(0)
        self._ck(self.L.alz_node_rows_device(self.h, int(source), C.byref(p), C.byref(n)), "alz_node_rows_device")
        return p.value, n.value

    def node_metrics(self, source, side, *specs):
        """alz_node_metrics: values [nodes x len(specs)] of side abi.SIDE_IN / SIDE_OUT; a spec is a METRIC_* kind or
        a (kind, q) pair."""
        return self._edge_metrics("alz_node_metrics", (int(source), int(side)), specs)

    def node_metrics_device(self, source, side, *specs):
        """alz_node_metrics_device: (device pointer, nodes)."""
        return self._edge_metrics_device("alz_node_metrics_device", (int(source), int(side)), specs)

    def node_top(self, source, side, spec, k, min_value=0.0):
        """alz_node_top: the first min(k, above) nodes by one metric of one side: (NODE_OUT rows, values, node
        indices, info dict), rank order. The first call offers room for min(k, 65536) results; when more came out,
        it is repeated with room for all."""
        f, n, info, m = self.L.alz_node_top, C.c_size_t(0), abi.TopInfo(), abi.metrics(spec)
        cap = min(int(k), 1 << 16)
        while True:
            nodes = np.zeros(cap, dtype=abi.NODE_OUT)
            values = np.zeros(cap, dtype=np.float64)
            index = np.zeros(cap, dtype=np.uint32)
            rc = self._ck(f(self.h, int(source), int(side), m, int(k), float(min_value), _ptr(nodes), _ptr(values),
                            _ptr(index), cap, C.byref(n), C.byref(info)), "alz_node_top", allow=(abi.E_CAPACITY,))
            if rc == 0:
                r = n.value
                return nodes[:r].copy(), values[:r].copy(), index[:r].copy(), info.as_dict()
            cap = n.value

    def node_top_device(self, source, side, spec, k, min_value=0.0):
        """alz_node_top_device: (nodes, values, index device pointers, results, info dict)."""
        pn, pv, pi, n, info = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_size_t(0), abi.TopInfo()
        self._ck(self.L.alz_node_top_device(self.h, int(source), int(side), abi.metrics(spec), int(k),
                                            float(min_value), C.byref(pn), C.byref(pv), C.byref(pi), C.byref(n),
                                            C.byref(info)), "alz_node_top_device")
        return pn.value, pv.value, pi.value, n.value, info.as_dict()

    def debug_node_rows(self, rows):
        """alz_debug_node_rows over a host EDGE_OUT array (copied to the device): NODE_OUT rows in node order."""
        rows = np.ascontiguousarray(rows, dtype=abi.EDGE_OUT)
        p = self.dev_alloc(max(rows.nbytes, 1))
        try:
            if len(rows):
                self.h2d(p, rows)
            return self._node_rows("alz_debug_node_rows", (C.c_void_p(p), len(rows)))
        finally:
            self.dev_free(p)

    # ---- groups (alz_groups.cu, docs/SPEC.md §24)
    def group_set(self, nodes, groups):
        """alz_group_set: node nodes[i] (see node_ends) is a member of group groups[i]; empty lists clear the map."""
        keys = np.ascontiguousarray(self.node_ends(nodes))
        g = np.ascontiguousarray(groups, dtype=np.uint32)
        if len(keys) != len(g):
            raise ValueError("one group per node")
        self._ck(self.L.alz_group_set(self.h, _ptr(keys), _ptr(g), len(keys)), "alz_group_set")

    def _group_edges(self, fn, args):
        """fn(h, *args, out, cap, &n, &info): (EDGE_OUT group-edge rows, info dict); a first call with cap 0 sizes it."""
        f, n, info = getattr(self.L, fn), C.c_size_t(0), abi.GroupInfo()
        if self._ck(f(self.h, *args, None, 0, C.byref(n), C.byref(info)), fn, allow=(abi.E_CAPACITY,)) == 0:
            return np.zeros(0, dtype=abi.EDGE_OUT), info.as_dict()
        out = np.zeros(n.value, dtype=abi.EDGE_OUT)
        self._ck(f(self.h, *args, _ptr(out), n.value, C.byref(n), C.byref(info)), fn)
        return out, info.as_dict()

    def group_edges(self, source=abi.SOURCE_WINDOW):
        """alz_group_edges: the group-edge rows of `source` (abi.SOURCE_WINDOW or abi.ROLLUP_*) as EDGE_OUT rows in
        (from key, to key) order, and the info dict."""
        return self._group_edges("alz_group_edges", (int(source),))

    def group_edges_device(self, source=abi.SOURCE_WINDOW):
        """alz_group_edges_device: (device pointer, rows, info dict)."""
        p, n, info = C.c_void_p(), C.c_size_t(0), abi.GroupInfo()
        self._ck(self.L.alz_group_edges_device(self.h, int(source), C.byref(p), C.byref(n), C.byref(info)),
                 "alz_group_edges_device")
        return p.value, n.value, info.as_dict()

    def group_edge_metrics(self, source, *specs):
        """alz_group_edge_metrics: values [group-edge rows x len(specs)]."""
        return self._edge_metrics("alz_group_edge_metrics", (int(source),), specs)

    def group_edge_metrics_device(self, source, *specs):
        """alz_group_edge_metrics_device: (device pointer, rows)."""
        return self._edge_metrics_device("alz_group_edge_metrics_device", (int(source),), specs)

    def group_edge_top(self, source, spec, k, min_value=0.0):
        """alz_group_edge_top: (group-edge rows, values, row indices, info dict), rank order."""
        return self._edge_top("alz_group_edge_top", (int(source),), spec, k, min_value)

    def group_edge_top_device(self, source, spec, k, min_value=0.0):
        """alz_group_edge_top_device: (rows, values, index device pointers, results, info dict)."""
        return self._edge_top_device("alz_group_edge_top_device", (int(source),), spec, k, min_value)

    def group_nodes(self, source=abi.SOURCE_WINDOW):
        """alz_group_nodes: the §21 NODE_OUT rows of the group-edge rows of `source`, node order."""
        return self._node_rows("alz_group_nodes", (int(source),))

    def group_nodes_device(self, source=abi.SOURCE_WINDOW):
        """alz_group_nodes_device: (device pointer, nodes)."""
        p, n = C.c_void_p(), C.c_size_t(0)
        self._ck(self.L.alz_group_nodes_device(self.h, int(source), C.byref(p), C.byref(n)), "alz_group_nodes_device")
        return p.value, n.value

    def group_node_metrics(self, source, side, *specs):
        """alz_group_node_metrics: values [group nodes x len(specs)] of side abi.SIDE_IN / SIDE_OUT."""
        return self._edge_metrics("alz_group_node_metrics", (int(source), int(side)), specs)

    def group_node_metrics_device(self, source, side, *specs):
        """alz_group_node_metrics_device: (device pointer, nodes)."""
        return self._edge_metrics_device("alz_group_node_metrics_device", (int(source), int(side)), specs)

    def group_node_top(self, source, side, spec, k, min_value=0.0):
        """alz_group_node_top: (NODE_OUT rows, values, node indices, info dict), rank order."""
        f, n, info, m = self.L.alz_group_node_top, C.c_size_t(0), abi.TopInfo(), abi.metrics(spec)
        cap = min(int(k), 1 << 16)
        while True:
            nodes = np.zeros(cap, dtype=abi.NODE_OUT)
            values = np.zeros(cap, dtype=np.float64)
            index = np.zeros(cap, dtype=np.uint32)
            rc = self._ck(f(self.h, int(source), int(side), m, int(k), float(min_value), _ptr(nodes), _ptr(values),
                            _ptr(index), cap, C.byref(n), C.byref(info)), "alz_group_node_top",
                          allow=(abi.E_CAPACITY,))
            if rc == 0:
                r = n.value
                return nodes[:r].copy(), values[:r].copy(), index[:r].copy(), info.as_dict()
            cap = n.value

    def group_node_top_device(self, source, side, spec, k, min_value=0.0):
        """alz_group_node_top_device: (nodes, values, index device pointers, results, info dict)."""
        pn, pv, pi, n, info = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_size_t(0), abi.TopInfo()
        self._ck(self.L.alz_group_node_top_device(self.h, int(source), int(side), abi.metrics(spec), int(k),
                                                  float(min_value), C.byref(pn), C.byref(pv), C.byref(pi), C.byref(n),
                                                  C.byref(info)), "alz_group_node_top_device")
        return pn.value, pv.value, pi.value, n.value, info.as_dict()

    def debug_group_edges(self, rows):
        """alz_debug_group_edges over a host EDGE_OUT array (copied to the device) with the handle's map: (group-edge
        rows, info dict)."""
        rows = np.ascontiguousarray(rows, dtype=abi.EDGE_OUT)
        p = self.dev_alloc(max(rows.nbytes, 1))
        try:
            if len(rows):
                self.h2d(p, rows)
            return self._group_edges("alz_debug_group_edges", (C.c_void_p(p), len(rows)))
        finally:
            self.dev_free(p)

    # ---- node series and trends (alz_node_series.cu, alz_trends.cu, docs/SPEC.md §22)
    @staticmethod
    def node_ends(nodes):
        """A NODE_ENDS array from a NODE_ENDS or NODE_OUT array (its type and value), or (type, value) tuples."""
        out = np.zeros(len(nodes), dtype=abi.NODE_ENDS)
        if isinstance(nodes, np.ndarray) and nodes.dtype.names:
            out["type"], out["value"] = nodes["type"], nodes["value"]
            return out
        for i, (t, v) in enumerate(nodes):
            out[i] = (t, (0,) * 3, v)
        return out

    def node_series(self, source, side, tier, k, *specs):
        """alz_node_series: every node of `source` (abi.SOURCE_WINDOW or abi.ROLLUP_*), side abi.SIDE_IN / SIDE_OUT,
        over the last k entries of `tier` (0: the window history): (values [nodes, P, nm], present [nodes, P], points,
        info dict)."""
        return self._series("alz_node_series", (int(source), int(side)), (int(tier), int(k)), specs)

    def node_series_device(self, source, side, tier, k, *specs):
        """alz_node_series_device: (values and present device pointers, nodes, P, points, info dict)."""
        return self._series_device("alz_node_series_device", (int(source), int(side)), (int(tier), int(k)), specs)

    def node_series_keys(self, nodes, side, tier, k, *specs):
        """alz_node_series_keys: the caller's nodes (see node_ends), in their order: (values [n, P, nm], present
        [n, P], points, info dict)."""
        keys = np.ascontiguousarray(self.node_ends(nodes))
        return self._series("alz_node_series_keys", (_ptr(keys), len(keys), int(side)), (int(tier), int(k)), specs)

    def node_series_keys_device(self, nodes, side, tier, k, *specs):
        """alz_node_series_keys_device: (values and present device pointers, n, P, points, info dict)."""
        keys = np.ascontiguousarray(self.node_ends(nodes))
        return self._series_device("alz_node_series_keys_device", (_ptr(keys), len(keys), int(side)),
                                   (int(tier), int(k)), specs)

    def node_trends(self, source, side, tier, k, spec, trend):
        """alz_node_trends: every node of `source`, side `side`, over the last k entries of `tier` by one metric and an
        abi.Trend: (NODE_TREND records in node order, points, info dict)."""
        return self._trends("alz_node_trends", (int(source), int(side), int(tier)), k, spec, trend, abi.NODE_TREND)

    def node_trends_device(self, source, side, tier, k, spec, trend):
        """alz_node_trends_device: (device pointer to the records, nodes, P, points, info dict)."""
        return self._trends_device("alz_node_trends_device", (int(source), int(side), int(tier)), k, spec, trend)

    def node_trends_top(self, source, side, tier, k, spec, trend, top, min_trend=-np.inf):
        """alz_node_trends_top: the first min(top, above) valid nodes by trend, rank order: (records, NODE_OUT rows,
        series [m, P] float64, present [m, P] uint8, points, info dict)."""
        return self._trends_top("alz_node_trends_top", (int(source), int(side), int(tier)), k, spec, trend, top,
                                min_trend, abi.NODE_TREND, abi.NODE_OUT)

    def node_trends_top_device(self, source, side, tier, k, spec, trend, top, min_trend=-np.inf):
        """alz_node_trends_top_device: (records, node rows, series and present device pointers, results, P, points,
        info dict)."""
        return self._trends_top_device("alz_node_trends_top_device", (int(source), int(side), int(tier)), k, spec,
                                       trend, top, min_trend)

    # ---- node changes against the pinned baseline (alz_changes.cu, docs/SPEC.md §23)
    def node_changes(self, side, spec, mode=abi.CHANGE_DELTA, presence=abi.PRESENT_ALL, source=abi.SOURCE_WINDOW):
        """alz_node_changes of side `side` (abi.SIDE_*) of the nodes of `source` against the pinned baseline by one
        metric: (NODE_CHANGE records in ascending node key order, info dict)."""
        return self._changes("alz_node_changes", (int(source), int(side), abi.metrics(spec), int(mode), int(presence)),
                             abi.NODE_CHANGE)

    def node_changes_device(self, side, spec, mode=abi.CHANGE_DELTA, presence=abi.PRESENT_ALL,
                            source=abi.SOURCE_WINDOW):
        """alz_node_changes_device: (device pointer, records, info dict)."""
        p, n, info = C.c_void_p(), C.c_size_t(0), abi.ChangeInfo()
        self._ck(self.L.alz_node_changes_device(self.h, int(source), int(side), abi.metrics(spec), int(mode),
                                                int(presence), C.byref(p), C.byref(n), C.byref(info)),
                 "alz_node_changes_device")
        return p.value, n.value, info.as_dict()

    def node_changes_top(self, side, spec, k, min_change=0.0, mode=abi.CHANGE_DELTA, presence=abi.PRESENT_ALL,
                         source=abi.SOURCE_WINDOW):
        """alz_node_changes_top: (the first min(k, above) NODE_CHANGE records by change, rank order; info dict)."""
        return self._changes("alz_node_changes_top", (int(source), int(side), abi.metrics(spec), int(mode),
                                                      int(presence), int(k), float(min_change)), abi.NODE_CHANGE)

    def node_changes_top_device(self, side, spec, k, min_change=0.0, mode=abi.CHANGE_DELTA, presence=abi.PRESENT_ALL,
                                source=abi.SOURCE_WINDOW):
        """alz_node_changes_top_device: (device pointer, records, info dict)."""
        p, n, info = C.c_void_p(), C.c_size_t(0), abi.ChangeInfo()
        self._ck(self.L.alz_node_changes_top_device(self.h, int(source), int(side), abi.metrics(spec), int(mode),
                                                    int(presence), int(k), float(min_change), C.byref(p), C.byref(n),
                                                    C.byref(info)), "alz_node_changes_top_device")
        return p.value, n.value, info.as_dict()

    def debug_node_changes_rows(self, src, base, side, spec, mode=abi.CHANGE_DELTA, presence=abi.PRESENT_ALL,
                                src_windows=1, base_windows=1):
        """alz_debug_node_changes_rows over two host row arrays (copied to the device, any order, repeats allowed):
        (NODE_CHANGE records, info dict)."""
        src = np.ascontiguousarray(src, dtype=abi.EDGE_OUT)
        base = np.ascontiguousarray(base, dtype=abi.EDGE_OUT)
        ps = self.dev_alloc(max(src.nbytes, 1))
        pb = self.dev_alloc(max(base.nbytes, 1))
        try:
            if len(src):
                self.h2d(ps, src)
            if len(base):
                self.h2d(pb, base)
            return self._changes("alz_debug_node_changes_rows",
                                 (C.c_void_p(ps), len(src), int(src_windows), C.c_void_p(pb), len(base),
                                  int(base_windows), int(side), abi.metrics(spec), int(mode), int(presence)),
                                 abi.NODE_CHANGE)
        finally:
            self.dev_free(ps)
            self.dev_free(pb)

    # ---- group changes against the pinned baseline (alz_changes.cu, docs/SPEC.md §25)
    def group_edge_changes(self, spec, mode=abi.CHANGE_DELTA, presence=abi.PRESENT_ALL, source=abi.SOURCE_WINDOW):
        """alz_group_edge_changes of the group edges of `source` against the pinned baseline's, both grouped by the
        current map, by one metric: (EDGE_CHANGE records in ascending (from key, to key) order, info dict)."""
        return self._changes("alz_group_edge_changes", (int(source), abi.metrics(spec), int(mode), int(presence)))

    def group_edge_changes_device(self, spec, mode=abi.CHANGE_DELTA, presence=abi.PRESENT_ALL,
                                  source=abi.SOURCE_WINDOW):
        """alz_group_edge_changes_device: (device pointer, records, info dict)."""
        p, n, info = C.c_void_p(), C.c_size_t(0), abi.ChangeInfo()
        self._ck(self.L.alz_group_edge_changes_device(self.h, int(source), abi.metrics(spec), int(mode), int(presence),
                                                      C.byref(p), C.byref(n), C.byref(info)),
                 "alz_group_edge_changes_device")
        return p.value, n.value, info.as_dict()

    def group_edge_changes_top(self, spec, k, min_change=0.0, mode=abi.CHANGE_DELTA, presence=abi.PRESENT_ALL,
                               source=abi.SOURCE_WINDOW):
        """alz_group_edge_changes_top: (the first min(k, above) EDGE_CHANGE records by change, rank order; info
        dict)."""
        return self._changes("alz_group_edge_changes_top", (int(source), abi.metrics(spec), int(mode), int(presence),
                                                            int(k), float(min_change)))

    def group_edge_changes_top_device(self, spec, k, min_change=0.0, mode=abi.CHANGE_DELTA, presence=abi.PRESENT_ALL,
                                      source=abi.SOURCE_WINDOW):
        """alz_group_edge_changes_top_device: (device pointer, records, info dict)."""
        p, n, info = C.c_void_p(), C.c_size_t(0), abi.ChangeInfo()
        self._ck(self.L.alz_group_edge_changes_top_device(self.h, int(source), abi.metrics(spec), int(mode),
                                                          int(presence), int(k), float(min_change), C.byref(p),
                                                          C.byref(n), C.byref(info)),
                 "alz_group_edge_changes_top_device")
        return p.value, n.value, info.as_dict()

    def group_node_changes(self, side, spec, mode=abi.CHANGE_DELTA, presence=abi.PRESENT_ALL,
                           source=abi.SOURCE_WINDOW):
        """alz_group_node_changes of side `side` (abi.SIDE_*) of the group nodes of `source` against the pinned
        baseline's by one metric: (NODE_CHANGE records in ascending node key order, info dict)."""
        return self._changes("alz_group_node_changes", (int(source), int(side), abi.metrics(spec), int(mode),
                                                        int(presence)), abi.NODE_CHANGE)

    def group_node_changes_device(self, side, spec, mode=abi.CHANGE_DELTA, presence=abi.PRESENT_ALL,
                                  source=abi.SOURCE_WINDOW):
        """alz_group_node_changes_device: (device pointer, records, info dict)."""
        p, n, info = C.c_void_p(), C.c_size_t(0), abi.ChangeInfo()
        self._ck(self.L.alz_group_node_changes_device(self.h, int(source), int(side), abi.metrics(spec), int(mode),
                                                      int(presence), C.byref(p), C.byref(n), C.byref(info)),
                 "alz_group_node_changes_device")
        return p.value, n.value, info.as_dict()

    def group_node_changes_top(self, side, spec, k, min_change=0.0, mode=abi.CHANGE_DELTA, presence=abi.PRESENT_ALL,
                               source=abi.SOURCE_WINDOW):
        """alz_group_node_changes_top: (the first min(k, above) NODE_CHANGE records by change, rank order; info
        dict)."""
        return self._changes("alz_group_node_changes_top", (int(source), int(side), abi.metrics(spec), int(mode),
                                                            int(presence), int(k), float(min_change)),
                             abi.NODE_CHANGE)

    def group_node_changes_top_device(self, side, spec, k, min_change=0.0, mode=abi.CHANGE_DELTA,
                                      presence=abi.PRESENT_ALL, source=abi.SOURCE_WINDOW):
        """alz_group_node_changes_top_device: (device pointer, records, info dict)."""
        p, n, info = C.c_void_p(), C.c_size_t(0), abi.ChangeInfo()
        self._ck(self.L.alz_group_node_changes_top_device(self.h, int(source), int(side), abi.metrics(spec),
                                                          int(mode), int(presence), int(k), float(min_change),
                                                          C.byref(p), C.byref(n), C.byref(info)),
                 "alz_group_node_changes_top_device")
        return p.value, n.value, info.as_dict()

    def debug_group_edge_changes_rows(self, src, base, spec, mode=abi.CHANGE_DELTA, presence=abi.PRESENT_ALL,
                                      src_windows=1, base_windows=1):
        """alz_debug_group_edge_changes_rows over two host row arrays (copied to the device, any order, repeats
        allowed) with the handle's map: (EDGE_CHANGE records, info dict)."""
        src = np.ascontiguousarray(src, dtype=abi.EDGE_OUT)
        base = np.ascontiguousarray(base, dtype=abi.EDGE_OUT)
        ps = self.dev_alloc(max(src.nbytes, 1))
        pb = self.dev_alloc(max(base.nbytes, 1))
        try:
            if len(src):
                self.h2d(ps, src)
            if len(base):
                self.h2d(pb, base)
            return self._changes("alz_debug_group_edge_changes_rows",
                                 (C.c_void_p(ps), len(src), int(src_windows), C.c_void_p(pb), len(base),
                                  int(base_windows), abi.metrics(spec), int(mode), int(presence)))
        finally:
            self.dev_free(ps)
            self.dev_free(pb)

    # ---- group series and trends (alz_group_series.cu, alz_trends.cu, docs/SPEC.md §26)
    def group_edge_series(self, source, tier, k, *specs):
        """alz_group_edge_series: every group edge of `source` (alz_group_edges order) over the last k entries of
        `tier`, each entry grouped by the map in force: (values [rows, P, nm], present [rows, P], points, info)."""
        return self._series("alz_group_edge_series", (int(source),), (int(tier), int(k)), specs)

    def group_edge_series_device(self, source, tier, k, *specs):
        """alz_group_edge_series_device: (values and present device pointers, rows, P, points, info dict)."""
        return self._series_device("alz_group_edge_series_device", (int(source),), (int(tier), int(k)), specs)

    def group_edge_series_keys(self, edges, tier, k, *specs):
        """alz_group_edge_series_keys: the caller's group edges (see edge_ends; a type may be abi.NODE_GROUP), in
        their order: (values [n, P, nm], present [n, P], points, info dict)."""
        keys = np.ascontiguousarray(self.edge_ends(edges))
        return self._series("alz_group_edge_series_keys", (_ptr(keys), len(keys)), (int(tier), int(k)), specs)

    def group_edge_series_keys_device(self, edges, tier, k, *specs):
        """alz_group_edge_series_keys_device: (values and present device pointers, n, P, points, info dict)."""
        keys = np.ascontiguousarray(self.edge_ends(edges))
        return self._series_device("alz_group_edge_series_keys_device", (_ptr(keys), len(keys)), (int(tier), int(k)),
                                   specs)

    def group_node_series(self, source, side, tier, k, *specs):
        """alz_group_node_series: every group node of `source` (alz_group_nodes order), side `side`: (values
        [nodes, P, nm], present [nodes, P], points, info dict)."""
        return self._series("alz_group_node_series", (int(source), int(side)), (int(tier), int(k)), specs)

    def group_node_series_device(self, source, side, tier, k, *specs):
        """alz_group_node_series_device: (values and present device pointers, nodes, P, points, info dict)."""
        return self._series_device("alz_group_node_series_device", (int(source), int(side)), (int(tier), int(k)),
                                   specs)

    def group_node_series_keys(self, nodes, side, tier, k, *specs):
        """alz_group_node_series_keys: the caller's nodes (see node_ends; a type may be abi.NODE_GROUP), in their
        order: (values [n, P, nm], present [n, P], points, info dict)."""
        keys = np.ascontiguousarray(self.node_ends(nodes))
        return self._series("alz_group_node_series_keys", (_ptr(keys), len(keys), int(side)), (int(tier), int(k)),
                            specs)

    def group_node_series_keys_device(self, nodes, side, tier, k, *specs):
        """alz_group_node_series_keys_device: (values and present device pointers, n, P, points, info dict)."""
        keys = np.ascontiguousarray(self.node_ends(nodes))
        return self._series_device("alz_group_node_series_keys_device", (_ptr(keys), len(keys), int(side)),
                                   (int(tier), int(k)), specs)

    def group_edge_trends(self, source, tier, k, spec, trend):
        """alz_group_edge_trends: every group edge of `source` by one metric and an abi.Trend: (EDGE_TREND records in
        alz_group_edges order, points, info dict)."""
        return self._trends("alz_group_edge_trends", (int(source), int(tier)), k, spec, trend, abi.EDGE_TREND)

    def group_edge_trends_device(self, source, tier, k, spec, trend):
        """alz_group_edge_trends_device: (device pointer to the records, rows, P, points, info dict)."""
        return self._trends_device("alz_group_edge_trends_device", (int(source), int(tier)), k, spec, trend)

    def group_edge_trends_top(self, source, tier, k, spec, trend, top, min_trend=-np.inf):
        """alz_group_edge_trends_top: the first min(top, above) valid group edges by trend, rank order: (records,
        EDGE_OUT group-edge rows, series [m, P], present [m, P], points, info dict)."""
        return self._trends_top("alz_group_edge_trends_top", (int(source), int(tier)), k, spec, trend, top, min_trend,
                                abi.EDGE_TREND, abi.EDGE_OUT)

    def group_edge_trends_top_device(self, source, tier, k, spec, trend, top, min_trend=-np.inf):
        """alz_group_edge_trends_top_device: (records, rows, series and present device pointers, results, P, points,
        info dict)."""
        return self._trends_top_device("alz_group_edge_trends_top_device", (int(source), int(tier)), k, spec, trend,
                                       top, min_trend)

    def group_node_trends(self, source, side, tier, k, spec, trend):
        """alz_group_node_trends: every group node of `source`, side `side`, by one metric and an abi.Trend:
        (NODE_TREND records in alz_group_nodes order, points, info dict)."""
        return self._trends("alz_group_node_trends", (int(source), int(side), int(tier)), k, spec, trend,
                            abi.NODE_TREND)

    def group_node_trends_device(self, source, side, tier, k, spec, trend):
        """alz_group_node_trends_device: (device pointer to the records, nodes, P, points, info dict)."""
        return self._trends_device("alz_group_node_trends_device", (int(source), int(side), int(tier)), k, spec,
                                   trend)

    def group_node_trends_top(self, source, side, tier, k, spec, trend, top, min_trend=-np.inf):
        """alz_group_node_trends_top: the first min(top, above) valid group nodes by trend, rank order: (records,
        NODE_OUT rows, series [m, P], present [m, P], points, info dict)."""
        return self._trends_top("alz_group_node_trends_top", (int(source), int(side), int(tier)), k, spec, trend, top,
                                min_trend, abi.NODE_TREND, abi.NODE_OUT)

    def group_node_trends_top_device(self, source, side, tier, k, spec, trend, top, min_trend=-np.inf):
        """alz_group_node_trends_top_device: (records, node rows, series and present device pointers, results, P,
        points, info dict)."""
        return self._trends_top_device("alz_group_node_trends_top_device", (int(source), int(side), int(tier)), k,
                                       spec, trend, top, min_trend)

    # ---- reach (alz_reach.cu, docs/SPEC.md §27)
    def _reach(self, fn, head, seeds, direction, max_hops, spec, min_value):
        """fn(h, *head, seeds, n_seeds, dir, max_hops, m, min_value, nodes, node_cap, &n_nodes, row_index, rows,
        row_cap, &n_rows, &info): (REACH_NODE records, row_index, EDGE_OUT rows, info dict); a first call without
        arrays sizes them."""
        f, nn, nr, info = getattr(self.L, fn), C.c_size_t(0), C.c_size_t(0), abi.ReachInfo()
        keys = np.ascontiguousarray(self.node_ends(seeds))
        m = abi.metrics(spec) if spec is not None else None
        args = (self.h, *head, _ptr(keys), len(keys), int(direction), int(max_hops), m, float(min_value))
        self._ck(f(*args, None, 0, C.byref(nn), None, None, 0, C.byref(nr), C.byref(info)), fn)
        nodes = np.zeros(nn.value, dtype=abi.REACH_NODE)
        index = np.zeros(nr.value, dtype=np.uint32)
        rows = np.zeros(nr.value, dtype=abi.EDGE_OUT)
        self._ck(f(*args, _ptr(nodes), len(nodes), C.byref(nn), _ptr(index), _ptr(rows), len(rows), C.byref(nr),
                   C.byref(info)), fn)
        return nodes, index, rows, info.as_dict()

    def _reach_device(self, fn, source, seeds, direction, max_hops, spec, min_value):
        pn, pi, pr, nn, nr, info = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_size_t(0), C.c_size_t(0), \
            abi.ReachInfo()
        keys = np.ascontiguousarray(self.node_ends(seeds))
        m = abi.metrics(spec) if spec is not None else None
        self._ck(getattr(self.L, fn)(self.h, int(source), _ptr(keys), len(keys), int(direction), int(max_hops), m,
                                     float(min_value), C.byref(pn), C.byref(nn), C.byref(pi), C.byref(pr),
                                     C.byref(nr), C.byref(info)), fn)
        return pn.value, nn.value, pi.value, pr.value, nr.value, info.as_dict()

    def reach(self, source, seeds, direction=abi.REACH_DOWN, max_hops=abi.REACH_MAX_HOPS, spec=None, min_value=0.0):
        """alz_reach: the nodes of `source` within max_hops rows of the seeds (see node_ends) in abi.REACH_DOWN / UP /
        ANY, following only rows whose metric `spec` is at least min_value when spec is given: (REACH_NODE records,
        row positions, EDGE_OUT rows, info dict)."""
        return self._reach("alz_reach", (int(source),), seeds, direction, max_hops, spec, min_value)

    def reach_device(self, source, seeds, direction=abi.REACH_DOWN, max_hops=abi.REACH_MAX_HOPS, spec=None,
                     min_value=0.0):
        """alz_reach_device: (records pointer, nodes, row_index pointer, rows pointer, rows, info dict)."""
        return self._reach_device("alz_reach_device", source, seeds, direction, max_hops, spec, min_value)

    def group_reach(self, source, seeds, direction=abi.REACH_DOWN, max_hops=abi.REACH_MAX_HOPS, spec=None,
                    min_value=0.0):
        """alz_group_reach: reach over the group-edge rows of `source` under the handle's map; seeds may be
        (abi.NODE_GROUP, g)."""
        return self._reach("alz_group_reach", (int(source),), seeds, direction, max_hops, spec, min_value)

    def group_reach_device(self, source, seeds, direction=abi.REACH_DOWN, max_hops=abi.REACH_MAX_HOPS, spec=None,
                           min_value=0.0):
        """alz_group_reach_device: (records pointer, nodes, row_index pointer, rows pointer, rows, info dict)."""
        return self._reach_device("alz_group_reach_device", source, seeds, direction, max_hops, spec, min_value)

    def debug_reach_rows(self, rows, seeds, direction=abi.REACH_DOWN, max_hops=abi.REACH_MAX_HOPS, spec=None,
                         min_value=0.0):
        """alz_debug_reach_rows over a host EDGE_OUT array (copied to the device): as reach."""
        rows = np.ascontiguousarray(rows, dtype=abi.EDGE_OUT)
        p = self.dev_alloc(max(rows.nbytes, 1))
        try:
            if len(rows):
                self.h2d(p, rows)
            return self._reach("alz_debug_reach_rows", (C.c_void_p(p), len(rows)), seeds, direction, max_hops, spec,
                               min_value)
        finally:
            self.dev_free(p)

    # ---- cycles (alz_cycles.cu, docs/SPEC.md §28)
    def _cycles(self, fn, head, spec, min_value, min_size):
        """fn(h, *head, m, min_value, min_size, nodes, node_cap, &n_nodes, row_index, rows, row_cap, &n_rows, &info):
        (CYCLE_NODE records, row_index, EDGE_OUT rows, info dict); a first call without arrays sizes them."""
        f, nn, nr, info = getattr(self.L, fn), C.c_size_t(0), C.c_size_t(0), abi.CycleInfo()
        m = abi.metrics(spec) if spec is not None else None
        args = (self.h, *head, m, float(min_value), int(min_size))
        self._ck(f(*args, None, 0, C.byref(nn), None, None, 0, C.byref(nr), C.byref(info)), fn)
        nodes = np.zeros(nn.value, dtype=abi.CYCLE_NODE)
        index = np.zeros(nr.value, dtype=np.uint32)
        rows = np.zeros(nr.value, dtype=abi.EDGE_OUT)
        self._ck(f(*args, _ptr(nodes), len(nodes), C.byref(nn), _ptr(index), _ptr(rows), len(rows), C.byref(nr),
                   C.byref(info)), fn)
        return nodes, index, rows, info.as_dict()

    def _cycles_device(self, fn, source, spec, min_value, min_size):
        pn, pi, pr, nn, nr, info = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_size_t(0), C.c_size_t(0), \
            abi.CycleInfo()
        m = abi.metrics(spec) if spec is not None else None
        self._ck(getattr(self.L, fn)(self.h, int(source), m, float(min_value), int(min_size), C.byref(pn), C.byref(nn),
                                     C.byref(pi), C.byref(pr), C.byref(nr), C.byref(info)), fn)
        return pn.value, nn.value, pi.value, pr.value, nr.value, info.as_dict()

    def cycles(self, source, spec=None, min_value=0.0, min_size=1):
        """alz_cycles: the strongly connected components of `source`'s nodes, following only rows whose metric `spec`
        is at least min_value when spec is given, listing the nodes of components of at least min_size nodes:
        (CYCLE_NODE records, row positions, EDGE_OUT rows, info dict)."""
        return self._cycles("alz_cycles", (int(source),), spec, min_value, min_size)

    def cycles_device(self, source, spec=None, min_value=0.0, min_size=1):
        """alz_cycles_device: (records pointer, nodes, row_index pointer, rows pointer, rows, info dict)."""
        return self._cycles_device("alz_cycles_device", source, spec, min_value, min_size)

    def group_cycles(self, source, spec=None, min_value=0.0, min_size=1):
        """alz_group_cycles: cycles over the group-edge rows of `source` under the handle's map."""
        return self._cycles("alz_group_cycles", (int(source),), spec, min_value, min_size)

    def group_cycles_device(self, source, spec=None, min_value=0.0, min_size=1):
        """alz_group_cycles_device: (records pointer, nodes, row_index pointer, rows pointer, rows, info dict)."""
        return self._cycles_device("alz_group_cycles_device", source, spec, min_value, min_size)

    def debug_cycles_rows(self, rows, spec=None, min_value=0.0, min_size=1):
        """alz_debug_cycles_rows over a host EDGE_OUT array (copied to the device): as cycles."""
        rows = np.ascontiguousarray(rows, dtype=abi.EDGE_OUT)
        p = self.dev_alloc(max(rows.nbytes, 1))
        try:
            if len(rows):
                self.h2d(p, rows)
            return self._cycles("alz_debug_cycles_rows", (C.c_void_p(p), len(rows)), spec, min_value, min_size)
        finally:
            self.dev_free(p)

    # ---- correlations (alz_corr.cu, docs/SPEC.md §29)
    @staticmethod
    def corr(direction=abi.CORR_POSITIVE, absent=abi.CORR_ABSENT_SKIP, max_lag=0, min_points=3):
        """An alz_corr."""
        return abi.Corr(int(direction), int(absent), int(max_lag), int(min_points))

    class Target:
        """An alz_corr_target over host arrays it keeps alive: values (float64), present (uint8, or None: every point
        present), window_last; n = len(values) unless given."""

        def __init__(self, values, present=None, window_last=0, n=None):
            self.values = np.ascontiguousarray(values, dtype=np.float64)
            self.present = None if present is None else np.ascontiguousarray(present, dtype=np.uint8)
            self.s = abi.CorrTarget(_ptr(self.values) if len(self.values) else None,
                                    None if self.present is None else _ptr(self.present),
                                    len(self.values) if n is None else int(n), int(window_last))

    @staticmethod
    def _target_of(target):
        return target if isinstance(target, Handle.Target) else Handle.Target(*target)

    def _corrs(self, fn, head, k, spec, corr, target, dtype):
        """fn(h, *head, k, m, &corr, &target, out, cap, &n, &P, points, &info): (records in source order, points, info
        dict). A first call with cap 0 gives the records."""
        f, n, p, info, m = getattr(self.L, fn), C.c_size_t(0), C.c_uint32(0), abi.CorrInfo(), abi.metrics(spec)
        t = self._target_of(target)
        self._ck(f(self.h, *head, int(k), m, C.byref(corr), C.byref(t.s), None, 0, C.byref(n), C.byref(p), None,
                   C.byref(info)), fn, allow=(abi.E_CAPACITY,))
        out = np.zeros(n.value, dtype=dtype)
        points = (abi.RollupInfo * max(int(k), 1))()
        self._ck(f(self.h, *head, int(k), m, C.byref(corr), C.byref(t.s), _ptr(out), len(out), C.byref(n), C.byref(p),
                   points, C.byref(info)), fn)
        return out, [points[j].as_dict() for j in range(p.value)], info.as_dict()

    def _corrs_device(self, fn, head, k, spec, corr, target):
        d, n, p, info = C.c_void_p(), C.c_size_t(0), C.c_uint32(0), abi.CorrInfo()
        t = self._target_of(target)
        points = (abi.RollupInfo * max(int(k), 1))()
        self._ck(getattr(self.L, fn)(self.h, *head, int(k), abi.metrics(spec), C.byref(corr), C.byref(t.s), C.byref(d),
                                     C.byref(n), C.byref(p), points, C.byref(info)), fn)
        return d.value, n.value, p.value, [points[j].as_dict() for j in range(p.value)], info.as_dict()

    def _corrs_top(self, fn, head, k, spec, corr, target, top, min_score, rec_dtype, row_dtype):
        """fn(h, *head, k, m, &corr, &target, top, min_score, out, rows, series, present, cap, &n, &P, points, &info).
        The first call offers room for min(top, 4096) results; when more came out, it is repeated with room for all."""
        f, n, p, info, m = getattr(self.L, fn), C.c_size_t(0), C.c_uint32(0), abi.CorrInfo(), abi.metrics(spec)
        t = self._target_of(target)
        cap = min(int(top), 1 << 12)
        points = (abi.RollupInfo * max(int(k), 1))()
        while True:
            out = np.zeros(cap, dtype=rec_dtype)
            rows = np.zeros(cap, dtype=row_dtype)
            series = np.zeros(cap * int(k))
            present = np.zeros(cap * int(k), dtype=np.uint8)
            rc = self._ck(f(self.h, *head, int(k), m, C.byref(corr), C.byref(t.s), int(top), float(min_score),
                            _ptr(out), _ptr(rows), _ptr(series), _ptr(present), cap, C.byref(n), C.byref(p), points,
                            C.byref(info)), fn, allow=(abi.E_CAPACITY,))
            if rc == 0:
                break
            if n.value <= cap:   # a capacity error that no buffer cures: too many slots
                raise AlzError(rc, fn)
            cap = n.value
        r, P = n.value, p.value
        return (out[:r].copy(), rows[:r].copy(), series[: r * P].reshape(r, P).copy(),
                present[: r * P].reshape(r, P).copy(), [points[j].as_dict() for j in range(P)], info.as_dict())

    def _corrs_top_device(self, fn, head, k, spec, corr, target, top, min_score):
        pr, pw, ps, pp_ = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
        n, p, info = C.c_size_t(0), C.c_uint32(0), abi.CorrInfo()
        t = self._target_of(target)
        points = (abi.RollupInfo * max(int(k), 1))()
        self._ck(getattr(self.L, fn)(self.h, *head, int(k), abi.metrics(spec), C.byref(corr), C.byref(t.s), int(top),
                                     float(min_score), C.byref(pr), C.byref(pw), C.byref(ps), C.byref(pp_), C.byref(n),
                                     C.byref(p), points, C.byref(info)), fn)
        return (pr.value, pw.value, ps.value, pp_.value, n.value, p.value, [points[j].as_dict() for j in range(p.value)],
                info.as_dict())

    _CORR_LEVELS = {"edge": (False, abi.EDGE_CORR, abi.EDGE_OUT), "node": (True, abi.NODE_CORR, abi.NODE_OUT),
                    "group_edge": (False, abi.EDGE_CORR, abi.EDGE_OUT),
                    "group_node": (True, abi.NODE_CORR, abi.NODE_OUT)}

    def _corr_head(self, level, source, side, tier):
        return (int(source), int(side), int(tier)) if self._CORR_LEVELS[level][0] else (int(source), int(tier))

    def correlations(self, level, source, tier, k, spec, corr, target, side=abi.SIDE_IN):
        """alz_{level}_correlations (level "edge", "node", "group_edge" or "group_node"): every candidate of `source`
        against `target` (an Alz.Target or a (values, present, window_last) tuple) by one metric and an abi.Corr:
        (EDGE_CORR / NODE_CORR records in source order, points, info dict). side: node levels only."""
        return self._corrs(f"alz_{level}_correlations", self._corr_head(level, source, side, tier), k, spec, corr,
                           target, self._CORR_LEVELS[level][1])

    def correlations_device(self, level, source, tier, k, spec, corr, target, side=abi.SIDE_IN):
        """alz_{level}_correlations_device: (device pointer to the records, rows, P, points, info dict)."""
        return self._corrs_device(f"alz_{level}_correlations_device", self._corr_head(level, source, side, tier), k,
                                  spec, corr, target)

    def correlations_top(self, level, source, tier, k, spec, corr, target, top, min_score=-np.inf, side=abi.SIDE_IN):
        """alz_{level}_correlations_top: the first min(top, above) valid candidates by score, rank order: (records,
        EDGE_OUT or NODE_OUT rows, series [m, P], present [m, P], points, info dict)."""
        _, rec, row = self._CORR_LEVELS[level]
        return self._corrs_top(f"alz_{level}_correlations_top", self._corr_head(level, source, side, tier), k, spec,
                               corr, target, top, min_score, rec, row)

    def correlations_top_device(self, level, source, tier, k, spec, corr, target, top, min_score=-np.inf,
                                side=abi.SIDE_IN):
        """alz_{level}_correlations_top_device: (records, rows, series and present device pointers, results, P, points,
        info dict)."""
        return self._corrs_top_device(f"alz_{level}_correlations_top_device", self._corr_head(level, source, side, tier),
                                      k, spec, corr, target, top, min_score)

    def debug_corr_series(self, values, present, target, corr, top=0, min_score=-np.inf, offset=0):
        """alz_debug_corr_series over host series values [n, P] float64 and present [n, P] uint8 (copied to the
        device, `offset` elements past the start of their allocations): (EDGE_CORR records, top indices (top > 0) or
        None, valid, above)."""
        values = np.ascontiguousarray(values, dtype=np.float64)
        present = np.ascontiguousarray(present, dtype=np.uint8)
        n, P = values.shape
        t = self._target_of(target)
        pv, pp_ = self.dev_alloc(max(values.nbytes, 16) + 16), self.dev_alloc(max(present.nbytes, 16) + 16)
        dv, dp = pv + 8 * int(offset), pp_ + int(offset)
        try:
            if values.size:
                self.h2d(dv, values)
                self.h2d(dp, present)
            cap = n if not top else min(int(top), n)
            out = np.zeros(cap, dtype=abi.EDGE_CORR)
            idx = np.zeros(cap, dtype=np.uint32)
            m, valid, above = C.c_size_t(0), C.c_uint64(0), C.c_uint64(0)
            self._ck(self.L.alz_debug_corr_series(self.h, C.c_void_p(dv), C.c_void_p(dp), n, P, C.byref(t.s),
                                                  C.byref(corr), int(top), float(min_score), _ptr(out), _ptr(idx), cap,
                                                  C.byref(m), C.byref(valid), C.byref(above)),
                     "alz_debug_corr_series")
            r = m.value
            return out[:r].copy(), (idx[:r].copy() if top else None), valid.value, above.value
        finally:
            self.dev_free(pv)
            self.dev_free(pp_)

    def fold(self):
        self._ck(self.L.alz_fold(self.h), "alz_fold")

    def sync(self):
        self._ck(self.L.alz_sync(self.h), "alz_sync")

    def set_stream(self, cuda_stream):
        self._ck(self.L.alz_set_stream(self.h, C.c_void_p(cuda_stream)), "alz_set_stream")

    # ---- device helpers (bench/test support)
    def dev_alloc(self, nbytes):
        p = C.c_void_p()
        self._ck(self.L.alz_dev_alloc(self.h, nbytes, C.byref(p)), "alz_dev_alloc")
        return p.value

    def dev_free(self, p):
        self._ck(self.L.alz_dev_free(self.h, C.c_void_p(p)), "alz_dev_free")

    def h2d(self, dev_ptr, arr):
        arr = np.ascontiguousarray(arr)
        self._ck(self.L.alz_memcpy_h2d(self.h, C.c_void_p(dev_ptr), _ptr(arr), arr.nbytes), "alz_memcpy_h2d")

    def d2h(self, dev_ptr, n, dtype):
        out = np.zeros(n, dtype=dtype)
        self._ck(self.L.alz_memcpy_d2h(self.h, _ptr(out), C.c_void_p(dev_ptr), out.nbytes), "alz_memcpy_d2h")
        return out


def pack_l7(recs):
    """alz_pack_l7: 32-B records -> (16-B records, overflow durations)."""
    L = load()
    recs = np.ascontiguousarray(recs, dtype=abi.L7_REC)
    out = np.zeros(len(recs), dtype=abi.L7_REC16)
    cap = max(16, len(recs) // 64)
    while True:
        ovf = np.zeros(cap, dtype=np.uint64)
        k = L.alz_pack_l7(_ptr(recs), len(recs), _ptr(out), _ptr(ovf), cap)
        if k >= 0:
            return out, ovf[:k].copy()
        if cap >= len(recs):
            raise AlzError(abi.E_INVAL, "alz_pack_l7")
        cap = len(recs)


class Topo:
    """Synthetic cluster + stream tables via libalazgpu's own copy of the generator."""

    def __init__(self, n_services, seed=0xA1A20000, mix=abi.MIX_SURVEY):
        self.L = load()
        self.p = self.L.alz_synth_topo_create(n_services, seed, mix)
        if not self.p:
            raise MemoryError("alz_synth_topo_create")
        t = self.p.contents
        self.n_services, self.n_pods, self.n_edges = t.n_services, t.n_pods, t.n_edges
        self.pod_ip = np.ctypeslib.as_array(t.pod_ip, (t.n_pods,)).copy()
        self.svc_ip = np.ctypeslib.as_array(t.svc_ip, (t.n_services,)).copy()
        self.dev = None
        self._handle = None

    def events(self, first, n):
        out = np.zeros(n, dtype=abi.L7_REC)
        self.L.alz_synth_fill(self.p, int(first), int(n), _ptr(out))
        return out

    def to_device(self, handle):
        d = C.c_void_p()
        handle._ck(self.L.alz_synth_dev_create(handle.h, self.p, C.byref(d)), "alz_synth_dev_create")
        self.dev, self._handle = d, handle
        return d

    def fill_device(self, handle, first, n, dev_ptr):
        if self.dev is None:
            self.to_device(handle)
        handle._ck(self.L.alz_synth_dev_fill(handle.h, self.dev, int(first), int(n), C.c_void_p(dev_ptr)),
                   "alz_synth_dev_fill")

    def close(self):
        if self.dev is not None and self._handle is not None and getattr(self._handle, "h", None):
            self.L.alz_synth_dev_destroy(self._handle.h, self.dev)
        self.dev = None
        if self.p:
            self.L.alz_synth_topo_destroy(self.p)
            self.p = None
