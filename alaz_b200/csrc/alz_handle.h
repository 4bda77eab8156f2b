// alz_handle.h — the handle behind the C ABI: everything one GPU owns.
#pragma once
#include <cstdint>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>
#include <cuda_runtime.h>

#include "../../include/alazgpu.h"
#include "../../include/alazgpu_synth.h"
#include "alz_kernels.cuh"

struct HostEp {
  uint32_t state = 0;  // kEpPod | kEpSvc
  uint32_t pod = 0, svc = 0;
};

// return ALZ_E_CUDA from a function of the handle `h` when a CUDA call fails, the call and its error in h->last_err
#define CK(expr)                                                                       \
  do {                                                                                 \
    cudaError_t _e = (expr);                                                           \
    if (_e != cudaSuccess) {                                                           \
      h->last_err = std::string(#expr) + ": " + cudaGetErrorString(_e);                \
      return ALZ_E_CUDA;                                                               \
    }                                                                                  \
  } while (0)

struct alz_gnn_state;   // alz_gnn.cu
struct alz_sock_state;  // alz_sock.cu
struct alz_comm_state;  // alz_comm.cu
struct alz_rollup_state;  // alz_rollup.cu
struct alz_tier_set;      // alz_rollup.cu
struct alz_span_state;    // alz_rollup.cu
struct alz_metrics_state; // alz_metrics.cu
struct alz_changes_state; // alz_changes.cu
struct alz_series_state;  // alz_series.cu
struct alz_trend_state;   // alz_trends.cu
struct alz_node_state;    // alz_nodes.cu
struct alz_node_series_state;   // alz_node_series.cu
struct alz_group_state;         // alz_groups.cu
struct alz_group_series_state;  // alz_group_series.cu
struct alz_reach_state;         // alz_reach.cu
struct alz_cycle_state;         // alz_cycles.cu

// One host->device staging slot: pinned host buffer + device buffer. A submitting thread owns the slot
// (mu) from the copy into the pinned buffer until its H2D and kernel are enqueued.
struct StageSlot {
  std::mutex mu;
  void* h = nullptr;
  void* d = nullptr;
  void* d_aux = nullptr;                  // raw path: compacted 32-B records
  cudaEvent_t copied = nullptr;           // H2D out of h done -> h may be rewritten
  cudaEvent_t consumed = nullptr;         // kernel that read d (and d_aux) done -> d may be rewritten
};
constexpr int kStageSlots = 4;
constexpr int kRawSlots = 2;

struct alz_handle {
  alz_config cfg{};
  int device = 0, sms = 0;
  cudaStream_t own_stream = nullptr, stream = nullptr, copy_stream = nullptr;
  cudaEvent_t ev_tmp = nullptr, ev_count = nullptr;
  std::string last_err;

  // Serialises everything that enqueues on `stream` or touches the bookkeeping below. Submitting threads
  // take it only around their enqueue; flush / commit / stats hold it for the whole call.
  std::mutex mu;
  std::mutex turn_mu;                     // staging slot hand-out
  uint64_t stage_turn = 0, raw_turn = 0;
  StageSlot stage[kStageSlots];
  StageSlot raw[kRawSlots];
  size_t raw_chunk = 0;                   // samples per raw slot

  // join build side: host mirror of the ClusterInfo maps and of the device's open-addressed table;
  // a commit patches only the slots that changed (alz_table_commit)
  std::unordered_map<uint32_t, HostEp> ep_host;
  std::vector<uint32_t> ep_dirty_ips;
  std::vector<alz::EpEntry> ep_tab;       // host mirror, ep_cap entries
  std::vector<uint8_t> ep_touched;        // per slot: changed since the last upload
  std::vector<uint32_t> ep_touched_list;
  alz::EpEntry* d_ep = nullptr;
  uint32_t ep_cap = 0;
  std::vector<uint8_t> bloom_cnt;         // per filter bit: how many pod addresses set it (saturating at 255)
  bool bloom_dirty = false;
  uint32_t* d_bloom = nullptr;            // ALZ_BLOOM_WORDS words
  uint32_t* h_bloom = nullptr;            // pinned staging
  void* h_patch = nullptr;                // pinned: (slot, entry) records of one commit
  void* d_patch = nullptr;
  size_t patch_cap = 0;
  cudaEvent_t ev_patch = nullptr;

  // accumulators
  alz::PairTable pairs{};                 // not with ALZ_CFG_EAGER_JOIN
  alz::EdgeTable edges{};
  alz::Counters* d_ctr = nullptr;
  alz::Counters* h_ctr = nullptr;  // pinned
  alz::HotState* d_hot = nullptr;
  uint32_t* d_cursor = nullptr;           // the ingest's claim cursors (zeroed before each launch)

  // flush scratch
  uint64_t* d_keys[2] = {nullptr, nullptr};
  uint32_t* d_rows[2] = {nullptr, nullptr};
  void* d_sort_tmp = nullptr;
  size_t sort_tmp_bytes = 0;
  alz_edge_out* d_out = nullptr;
  alz::EdgeSortScratch es{};              // the edge-key sort (alz_sort.cu): keys/rows are d_keys[0] / d_rows[0]
  uint32_t n_live = 0, last_n_edges = 0;
  alz::FlushBuckets bk{};                 // single-rank flush: pair rows by edge row (not with ALZ_CFG_EAGER_JOIN)
  bool bucketed = false;                  // prepare_flush bucketed the pair rows; finish_flush emits them
  bool edges_dirty = false;               // a fold since the last flush left sums in the edge accumulators
  uint64_t lost_reported = 0;             // capacity_events already reported by an earlier flush

  // time-cut windows (alz_window_clock)
  bool win_on = false;
  uint64_t win_off = 0, win_len = 0;      // first_user - first_kernel (mod 2^64), window length
  uint64_t* d_win = nullptr;              // device WinClock {lo, len, ready, off, epoch} (alz_ingest.cu)
  alz_l7_rec* d_defer[2] = {nullptr, nullptr};   // records of later windows (ping-pong)
  uint32_t defer_cap = 0;
  int defer_cur = 0;
  uint64_t deferred_last = 0;

  uint64_t events_in = 0, pending_since_fold = 0, windows = 0;
  uint64_t launches = 0;                  // own kernels launched (stats)
  cudaEvent_t ev_t[3] = {nullptr, nullptr, nullptr};   // flush start / local part done / merge done (timing events)
  bool ev_t_valid = false;
  uint64_t collective_bytes_last = 0;
  uint64_t tcp_events_in = 0, tcp_localhost_dropped = 0;

  int comm_nranks = 1, comm_rank = 0;
  alz_comm_state* comm = nullptr;
  uint64_t merge_lost_events = 0;         // events of this rank's rows that a merge left out (merged graph > max_edges)
  alz_gnn_state* gnn = nullptr;
  alz_sock_state* sock = nullptr;
  alz_rollup_state* roll = nullptr;       // rolling windows (alz_window_history); null = off
  alz_tier_set* tiers = nullptr;          // tiered history (alz_window_history_tiers); null = off
  alz_span_state* span = nullptr;         // span rollup scratch (alz_window_rollup_span); null until the first one
  alz_metrics_state* metrics = nullptr;   // edge metric buffers (alz_edge_metrics*, alz_edge_top*); null until the first
  alz_changes_state* changes = nullptr;   // the pinned baseline and the change list's buffers; null until the first
  alz_series_state* series = nullptr;     // the edge series' buffers (alz_edge_series*); null until the first
  alz_trend_state* trends = nullptr;      // the edge trends' buffers (alz_edge_trends*); null until the first
  alz_node_state* nodes = nullptr;        // the node calls' buffers (alz_node_*); null until the first
  alz_node_series_state* node_series = nullptr;   // the node series' buffers (alz_node_series*); null until the first
  alz_trend_state* node_trends = nullptr;         // the node trends' buffers (alz_node_trends*); null until the first
  alz_group_state* groups = nullptr;      // the group map and the group calls' buffers (alz_group_*); null until the
                                          // first
  alz_group_series_state* group_series = nullptr;     // the group series' buffers (alz_group_*_series*); null until
                                                      // the first
  alz_trend_state* group_trends = nullptr;            // the group trends' buffers (alz_group_*_trends*); null until
                                                      // the first
  alz_reach_state* reach = nullptr;                   // the reach calls' buffers (alz_reach*, alz_group_reach*); null
                                                      // until the first
  alz_cycle_state* cycles = nullptr;                  // the cycles calls' buffers (alz_cycles*, alz_group_cycles*);
                                                      // null until the first
  alz_trend_state* corr = nullptr;                    // the edge correlations' buffers (alz_edge_correlations*,
                                                      // alz_debug_corr_series); null until the first
  alz_trend_state* node_corr = nullptr;               // the node correlations' buffers (alz_node_correlations*)
  alz_trend_state* group_corr = nullptr;              // the group correlations' buffers (alz_group_*_correlations*)
};

int alz_internal_fold(alz_handle* h);
// device records -> the ingest kernel of the current mode; caller holds h->mu and has set the device
int alz_internal_ingest(alz_handle* h, const alz_l7_rec* d_recs, size_t n);
// multi-GPU merge of the prepared (sorted) live edges of a handle with comm_nranks > 1. local_rc: this rank's
// own status so far (every rank enters the collectives even when its local preparation failed, and all ranks
// return the same failure). *lost: in, this rank lost events in this window; out, some rank did or the merged
// graph was cut at max_edges (the same answer on every rank). ALZ_OK: the window is consumed, h->last_n_edges
// merged rows are in h->d_out; any other status: the window is kept. *roll (with ALZ_OK): the flush closes this
// rank's time-cut window; false: the rank is ahead of the ranks' merged epoch, or no rank has one, and keeps it.
int alz_internal_merge_ranks(alz_handle* h, int local_rc, bool* lost, bool* roll);
// device WinClock of the epoch E the last merge closed (ready 0 when no rank had an epoch); valid after a merge
const uint64_t* alz_internal_merged_clock(alz_handle* h);
// Rolling windows: the window a flush has just consumed (h->last_n_edges rows in h->d_out, h->windows counted) becomes
// the newest entry of the history. d_clk: the device WinClock of the epoch it closed, read in stream order, so before
// the flush's roll advances it; null without a window clock. Nothing happens with the history off. Caller holds h->mu.
// With tiers configured the window is also the next input of tier 1 (docs/SPEC.md §13).
int alz_internal_history_append(alz_handle* h, const uint64_t* d_clk);
// The rows the last rollup of `kind` (ALZ_ROLLUP_*) returned with ALZ_OK, on the device: *rows, *n, and what that
// call reported into *info when not null (docs/SPEC.md §15). ALZ_E_INVAL for an unknown kind; ALZ_E_STATE when there
// are none. Caller holds h->mu.
int alz_internal_rollup_rows(alz_handle* h, uint32_t kind, const alz_edge_out** rows, size_t* n,
                             alz_rollup_info* info = nullptr);
// What a k = 1 window rollup reports for the last flushed window (docs/SPEC.md §18): windows 1, its rows, its
// alz_stats.windows, and its clock when the window history holds it as its newest entry (one wait); not clocked
// otherwise. Caller holds h->mu and has set the device.
int alz_internal_window_info(alz_handle* h, alz_rollup_info* info);
// The last min(k, retained) closed entries of one ring, oldest first, read only: the window history (tier 0) or tier
// t >= 1. Each is a run of rows [first_row, first_row + n) of the ring's arena.
struct alz_ring_view {
  const alz_edge_out* arena = nullptr;
  std::vector<uint64_t> first_row, n;
};
// *v for tier `tier` and k >= 1; enqueues the copy of the ring's clocks to the host, which alz_internal_ring_points
// reads once the stream has passed it. ALZ_E_STATE: tier 0 without the window history, t >= 1 without tiers;
// ALZ_E_INVAL: a tier above the configured ones. Caller holds h->mu and has set the device.
int alz_internal_ring_view(alz_handle* h, uint32_t tier, uint32_t k, alz_ring_view* v);
// points[j] = what a rollup of view entry j alone reports, for the view the last alz_internal_ring_view call gave
// (same tier and k, no call on the handle in between), after a wait on the stream. Caller holds h->mu.
void alz_internal_ring_points(alz_handle* h, uint32_t tier, uint32_t k, alz_rollup_info* points);
// The alz_rollup_info.window_last of the newest closed entry of one ring (0 when it holds none), from the host's
// records: no wait. The ring exists (an alz_internal_ring_view call for it succeeded). Caller holds h->mu.
uint64_t alz_internal_ring_last(alz_handle* h, uint32_t tier);
void alz_internal_free_rollup(alz_handle* h);
void alz_internal_free_tiers(alz_handle* h);
void alz_internal_free_span(alz_handle* h);
void alz_internal_free_comm(alz_handle* h);
void alz_internal_free_gnn(alz_handle* h);
void alz_internal_free_metrics(alz_handle* h);
void alz_internal_free_changes(alz_handle* h);
void alz_internal_free_series(alz_handle* h);
void alz_internal_free_trends(alz_handle* h);
void alz_internal_free_nodes(alz_handle* h);
void alz_internal_free_node_series(alz_handle* h);
void alz_internal_free_node_trends(alz_handle* h);
void alz_internal_free_groups(alz_handle* h);
void alz_internal_free_group_series(alz_handle* h);
void alz_internal_free_group_trends(alz_handle* h);
void alz_internal_free_reach(alz_handle* h);
void alz_internal_free_cycles(alz_handle* h);
void alz_internal_free_corr(alz_handle* h);
void alz_internal_free_sock(alz_handle* h);
