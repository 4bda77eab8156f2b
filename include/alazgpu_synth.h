/*
 * alazgpu_synth.h — bench/test support exported by libalazgpu next to the
 * product ABI: device-memory helpers and the device-side synthetic l7_req
 * stream (alaz_b200/synth/alz_synth.h). Not part of the drop-in boundary.
 */
#ifndef ALAZGPU_SYNTH_H
#define ALAZGPU_SYNTH_H
#include "alazgpu.h"
#include "../alaz_b200/synth/alz_synth.h"
#ifdef __cplusplus
extern "C" {
#endif

/* pinned host buffers: alz_submit_l7 / alz_submit_l7_raw from such a buffer skip
 * the staging memcpy (the Go side can fill them directly: C memory, cgo-legal) */
int alz_pinned_alloc(size_t bytes, void** out);
/* same, on the NUMA node next to the handle's GPU (8 ranks feeding 8 GPUs: staging on the remote socket
 * halves the reachable H2D rate) */
int alz_pinned_alloc_local(alz_handle* h, size_t bytes, void** out);
int alz_pinned_free(void* p);

int alz_dev_alloc(alz_handle* h, size_t bytes, void** out);
int alz_dev_free(alz_handle* h, void* p);
int alz_memcpy_h2d(alz_handle* h, void* dst, const void* src, size_t bytes);
int alz_memcpy_d2h(alz_handle* h, void* dst, const void* src, size_t bytes);
/* fold pending socket pairs into the edge accumulators now (flush does it anyway) */
int alz_fold(alz_handle* h);

/* test/debug: node keys ((kind << 32) | value, ascending) and layer-2 embeddings [n x 64] of the last GNN pass */
int alz_gnn_nodes(alz_handle* h, uint64_t* node_keys, float* h2, size_t cap, size_t* n_out);
/* test/debug: the selection of alz_gnn_top (docs/SPEC.md §16) over n scores in device memory: *n_out results, their
 * indices into index (or NULL; cap too small: ALZ_E_CAPACITY, nothing written), *above the eligible scores (or
 * NULL). Uses the GNN state's scratch, grown when smaller to the rows the selection needs, about min(k, n) (then
 * alz_gnn_nodes reports no nodes).
 * n > 2^30 - 1: ALZ_E_CAPACITY; k = 0 or a NaN min_score: ALZ_E_INVAL. */
int alz_debug_top_scores(alz_handle* h, const float* dev_scores, size_t n, uint32_t k, float min_score,
                         uint32_t* index, size_t cap, size_t* n_out, uint64_t* above);
/* test/debug: the metric kernel of alz_edge_metrics (docs/SPEC.md §17) over n rows in device memory, which may hold
 * histograms the ingest path cannot make (cells of 2^32 - 1, count = 0 with a non-empty histogram); the rules of
 * alz_edge_metrics otherwise */
int alz_debug_edge_metrics_rows(alz_handle* h, const alz_edge_out* dev_rows, size_t n, const alz_metric* m,
                                uint32_t nm, double* values, size_t cap, size_t* n_out);
/* test/debug: the selection of alz_edge_top over n float64 values in device memory: *n_out results, their indices
 * into index (or NULL; cap too small: ALZ_E_CAPACITY, nothing written), *above the eligible values (or NULL).
 * n > 2^30 - 1: ALZ_E_CAPACITY; k = 0 or a NaN min_value: ALZ_E_INVAL. */
int alz_debug_top_keys64(alz_handle* h, const double* dev_values, size_t n, uint32_t k, double min_value,
                         uint32_t* index, size_t cap, size_t* n_out, uint64_t* above);
/* test/debug: the join of alz_edge_changes (docs/SPEC.md §18) over two caller row lists in device memory, each in
 * strictly ascending packed-key order and covering src_windows / base_windows (>= 1) windows; the pinned baseline
 * is not used or touched. The rules of alz_edge_changes otherwise. */
int alz_debug_edge_changes_rows(alz_handle* h, const alz_edge_out* dev_src, size_t n_src, uint32_t src_windows,
                                const alz_edge_out* dev_base, size_t n_base, uint32_t base_windows,
                                const alz_metric* m, uint32_t mode, uint32_t presence, alz_edge_change* out,
                                size_t cap, size_t* n_out, alz_change_info* info);
/* test/debug: the group-by of alz_node_rows (docs/SPEC.md §21) over n caller rows in device memory, which may hold
 * layouts ingest cannot make (one node on 2^20 rows, cells of 2^32 - 1, any row order, repeated edges); the rules of
 * alz_node_rows otherwise. Uses the node calls' buffers. */
int alz_debug_node_rows(alz_handle* h, const alz_edge_out* dev_rows, size_t n, alz_node_out* out, size_t cap,
                        size_t* n_out);
/* test/debug: alz_node_changes (docs/SPEC.md §23) between the §21 node lists of two caller row lists in device memory,
 * each in any order with repeats allowed and covering src_windows / base_windows (>= 1) windows; the pinned baseline
 * and its cached node rows are not used. More than 2^29 - 1 rows in a list: ALZ_E_CAPACITY. The rules of
 * alz_node_changes otherwise. Uses the node change calls' buffers. */
int alz_debug_node_changes_rows(alz_handle* h, const alz_edge_out* dev_src, size_t n_src, uint32_t src_windows,
                                const alz_edge_out* dev_base, size_t n_base, uint32_t base_windows, uint32_t side,
                                const alz_metric* m, uint32_t mode, uint32_t presence, alz_node_change* out,
                                size_t cap, size_t* n_out, alz_change_info* info);
/* test/debug: the group edges of alz_group_edges (docs/SPEC.md §24) of n caller rows in device memory with the
 * handle's group map, which may hold layouts ingest cannot make (any row order, repeated edges, one group edge on 2^20
 * rows, cells of 2^32 - 1); the rules of alz_group_edges otherwise. Uses the group calls' buffers. */
int alz_debug_group_edges(alz_handle* h, const alz_edge_out* dev_rows, size_t n, alz_edge_out* out, size_t cap,
                          size_t* n_out, alz_group_info* info);
/* test/debug: alz_group_edge_changes (docs/SPEC.md §25) between the group edges of two caller row lists in device
 * memory under the handle's map, each in any order with repeats allowed and covering src_windows / base_windows (>= 1)
 * windows, which may hold layouts ingest cannot make (ends whose node keys collide when packed into 64 bits, one group
 * edge on 2^20 rows, cells of 2^32 - 1); the pinned baseline and its cached groups are neither used nor touched. More
 * than 2^29 - 1 rows in a list: ALZ_E_CAPACITY. The rules of alz_group_edge_changes otherwise. Uses the group change
 * calls' buffers. */
int alz_debug_group_edge_changes_rows(alz_handle* h, const alz_edge_out* dev_src, size_t n_src, uint32_t src_windows,
                                      const alz_edge_out* dev_base, size_t n_base, uint32_t base_windows,
                                      const alz_metric* m, uint32_t mode, uint32_t presence, alz_edge_change* out,
                                      size_t cap, size_t* n_out, alz_change_info* info);
/* test/debug: alz_reach (docs/SPEC.md §27) over n caller rows in device memory, which may hold layouts ingest cannot
 * make (any row order, any type byte, long chains, one node on 2^20 rows); the traversed rows are the caller's rows and
 * the node list their §21 node list. More than 2^29 - 1 rows: ALZ_E_CAPACITY. The rules of alz_reach otherwise. Uses
 * the reach calls' buffers. */
int alz_debug_reach_rows(alz_handle* h, const alz_edge_out* dev_rows, size_t n, const alz_node_ends* seeds,
                         size_t n_seeds, uint32_t dir, uint32_t max_hops, const alz_metric* m, double min_value,
                         alz_reach_node* nodes, size_t node_cap, size_t* n_nodes, uint32_t* row_index,
                         alz_edge_out* rows, size_t row_cap, size_t* n_rows, alz_reach_info* info);
/* test/debug: alz_cycles (docs/SPEC.md §28) over n caller rows in device memory, which may hold layouts ingest cannot
 * make (any row order, any type byte, repeated ends, long chains and rings, one node on 2^20 rows); the traversed rows
 * are the caller's rows and the node list their §21 node list. More than 2^29 - 1 rows: ALZ_E_CAPACITY. The rules of
 * alz_cycles otherwise. Uses the cycles calls' buffers. */
int alz_debug_cycles_rows(alz_handle* h, const alz_edge_out* dev_rows, size_t n, const alz_metric* m, double min_value,
                          uint32_t min_size, alz_cycle_node* nodes, size_t node_cap, size_t* n_nodes,
                          uint32_t* row_index, alz_edge_out* rows, size_t row_cap, size_t* n_rows,
                          alz_cycle_info* info);
/* test/debug: the §29 statistic and selection over n caller series of P points in device memory (values[i * P + j],
 * present[i * P + j], which may hold layouts no series call makes: any P, rows past 2^20, values at absent points). The
 * values must be finite with |v| <= 2^64, as every §17 metric is. target->n must be P; its window_last is not read.
 * Records carry a zero head (`valid` and `lag` set). top = 0: every row's record in row order into out[n]; top > 0:
 * the first min(top, above) in rank order into out, their rows into top_index. More than 2^30 - 1 rows or slots:
 * ALZ_E_CAPACITY. *n_out, *valid and *above (each may be NULL but n_out) as alz_corr_info gives them. Uses the edge
 * correlation calls' buffers. */
int alz_debug_corr_series(alz_handle* h, const double* dev_values, const uint8_t* dev_present, size_t n, uint32_t P,
                          const alz_corr_target* target, const alz_corr* corr, uint32_t top, double min_score,
                          alz_edge_corr* out, uint32_t* top_index, size_t cap, size_t* n_out, uint64_t* valid,
                          uint64_t* above);

typedef struct alz_synth_dev alz_synth_dev;
int alz_synth_dev_create(alz_handle* h, const alz_synth_topo* topo, alz_synth_dev** out);
int alz_synth_dev_fill(alz_handle* h, alz_synth_dev* d, uint64_t first, uint64_t n, alz_l7_rec* dev_out);
int alz_synth_dev_fill_owned(alz_handle* h, alz_synth_dev* d, uint64_t first, uint32_t nranks, uint32_t rank,
                             alz_l7_rec* dev_out, uint64_t want, uint64_t* n_written, uint64_t* n_scanned);
int alz_synth_dev_destroy(alz_handle* h, alz_synth_dev* d);

#ifdef __cplusplus
}
#endif
#endif
