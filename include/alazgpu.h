/*
 * alazgpu.h — C ABI of libalazgpu: the H100-native replacement for the
 * service-map aggregation hot path of getanteon/alaz (reference @ 828b997f).
 *
 * The reference has no FFI boundary for this path; the seam this library sits
 * behind is the aggregator's channel-in / DataStore-out pair:
 *   in : *l7_req.L7Event              ebpf/l7_req/l7.go:396-421 (from bpfL7Event, l7.go:345-369)
 *        *tcp_state.TcpConnectEvent   ebpf/tcp_state/tcp.go:75-84 (from BpfTcpEvent, tcp.go:63-72)
 *        k8s.K8sResourceMessage       k8s/informer.go:236-240 -> processPod/processSvc
 *                                     aggregator/persist.go:55-71, 114-130
 *   out: datastore.DataStore.PersistRequest  datastore/datastore.go:13
 *                                     (one row per request; this library instead
 *                                     returns the rows grouped by (From,To))
 *
 * Rules: plain C, flat PODs, no pointer is retained past the call that
 * received it (cgo rule), every entry point returns 0 on success or a negative
 * alz_status. No exceptions cross the boundary. One handle drives one GPU.
 * INTEGRATION.md shows the cgo binding a maintainer would add.
 */
#ifndef ALAZGPU_H
#define ALAZGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ALZ_ABI_VERSION 2

/* ---- status codes -------------------------------------------------------- */
typedef enum alz_status {
  ALZ_OK = 0,
  ALZ_E_INVAL = -1,      /* bad argument */
  ALZ_E_NOMEM = -2,      /* host or device allocation failed */
  ALZ_E_CUDA = -3,       /* CUDA runtime error (alz_last_cuda_error) */
  ALZ_E_NODEVICE = -4,   /* no CUDA device: there is NO CPU fallback */
  ALZ_E_CAPACITY = -5,   /* pair/edge dictionary or output buffer too small */
  ALZ_E_STATE = -6,      /* call not valid in this state (e.g. no comm) */
  ALZ_E_NCCL = -7,       /* NCCL error or libnccl.so.2 not loadable */
  ALZ_E_UNSUPPORTED = -8
} alz_status;

/* ---- wire enums: values equal the eBPF side (ebpf/l7_req/l7.go:19-29) ----- */
enum {
  ALZ_PROTO_UNKNOWN = 0, ALZ_PROTO_HTTP = 1, ALZ_PROTO_AMQP = 2,
  ALZ_PROTO_POSTGRES = 3, ALZ_PROTO_HTTP2 = 4, ALZ_PROTO_REDIS = 5,
  ALZ_PROTO_KAFKA = 6, ALZ_PROTO_MYSQL = 7, ALZ_PROTO_MONGO = 8
};
/* method enums that change routing (l7.go:91-95, 120-125) */
enum { ALZ_AMQP_PUBLISH = 1, ALZ_AMQP_DELIVER = 2 };
enum { ALZ_REDIS_COMMAND = 1, ALZ_REDIS_PUSHED_EVENT = 2, ALZ_REDIS_PING = 3 };

/* method_flags byte of alz_l7_rec */
#define ALZ_MF_METHOD_MASK 0x3Fu
#define ALZ_MF_PAYLOAD_REJECT 0x40u /* host-side payload parser says the reference
                                       would drop the row: Postgres/MySQL text query
                                       without SQL keyword (aggregator/data.go:1440-1443,
                                       1495-1497), Mongo parse failure (:1252-1255) */
#define ALZ_MF_TLS 0x80u

/* protocol byte of alz_l7_rec: bit 6 says "daddr holds a host id, not an address". The caller sets it for an
 * HTTP event whose payload carried a Host header AND whose daddr is neither a service nor a pod in the
 * tables as committed so far — the case in which setFromToV2 keys the destination by the header
 * (aggregator/data.go:851-854). The caller owns both the payload parser and the interner of header strings
 * (strings never cross this ABI), and it owns the tables it upserts here, so it can decide this exactly
 * as the reference does; the device keeps such events in their own key space. */
#define ALZ_PROTO_F_HOSTKEY 0x40u

/* node kinds of an edge end (aggregator/data.go POD/SVC/OUTBOUND) */
enum { ALZ_NODE_POD = 0, ALZ_NODE_SVC = 1, ALZ_NODE_OUTBOUND = 2,
       ALZ_NODE_OUTBOUND_HOST = 3 /* outbound destination keyed by the HTTP Host header (aggregator/data.go:851-854);
                                     value = the caller's dense id of the header string */,
       ALZ_NODE_GROUP = 4 /* a caller-defined group of nodes (docs/SPEC.md §24), value = the caller's dense id of the
                             group; only the group calls produce it, never a flush */ };
/* tables of the join's build side (aggregator/cluster.go:15-16) */
enum { ALZ_TABLE_POD = 0, ALZ_TABLE_SVC = 1 };

#define ALZ_NB 64 /* latency histogram buckets, see docs/SPEC.md §4 */

/* ---- records -------------------------------------------------------------- */

/* Compact L7 record, 32 B. Lossless w.r.t. struct l7_event (ebpf/c/l7.c:19-47)
 * for everything resolve/emit/reduce reads; pid/fd/payload stay host-side.
 * saddr/daddr are host-order u32 with the first octet in the MSB, exactly the
 * integer the reference feeds to IntToIPv4 (aggregator/data.go:1751-1767). */
typedef struct alz_l7_rec {
  uint32_t saddr;
  uint32_t daddr;
  uint16_t sport;
  uint16_t dport;
  uint16_t status;       /* l7_event.status saturated to 65535 */
  uint8_t protocol;      /* ALZ_PROTO_* */
  uint8_t method_flags;  /* method | ALZ_MF_* */
  uint64_t duration_ns;  /* l7_event.duration (l7.c:788) */
  uint64_t write_time_ns;
} alz_l7_rec;

/* Packed L7 record, 16 B: the fields of alz_l7_rec that resolve/emit/reduce read, for callers whose
 * events cross PCIe (half the bytes per event on the wire). Lossless: a duration >= 2^32 ns is stored
 * in the overflow array handed to the same submit call, the record carries its index there and bit 7
 * of `protocol` is set. No ports and no write time: windows of packed records are cut by the caller. */
typedef struct alz_l7_rec16 {
  uint32_t saddr;
  uint32_t daddr;
  uint16_t status;
  uint8_t protocol;      /* ALZ_PROTO_* | ALZ_REC16_DUR_OVERFLOW */
  uint8_t method_flags;  /* method | ALZ_MF_* */
  uint32_t duration_ns;  /* or index into the overflow array */
} alz_l7_rec16;
#define ALZ_REC16_DUR_OVERFLOW 0x80u

/* tcp_state record, 40 B, from struct tcp_event (ebpf/c/struct.h:2-12).
 * type: 1=ESTABLISHED 5=CLOSED (ebpf/tcp_state/tcp.go:19-25); addresses as in
 * alz_l7_rec (first octet in MSB). */
typedef struct alz_tcp_rec {
  uint64_t fd;
  uint64_t timestamp_ns;
  uint32_t pid;
  uint32_t saddr;
  uint32_t daddr;
  uint16_t sport;
  uint16_t dport;
  uint32_t type;
  uint32_t _pad;
} alz_tcp_rec;

/* query / result of the temporal socket join (SocketLine.GetValue,
 * aggregator/sock_num_line.go:82-158) */
typedef struct alz_sock_query {
  uint64_t fd;
  uint64_t timestamp_ns;
  uint32_t pid;
  uint32_t _pad;
} alz_sock_query;

typedef struct alz_sock_result {
  uint32_t found; /* 1 = SockInfo returned, 0 = the reference returns an error */
  uint32_t saddr;
  uint32_t daddr;
  uint16_t sport;
  uint16_t dport;
} alz_sock_result;

/* One edge of the service graph for one window. Rows the reference would have
 * handed to PersistRequest (datastore/backend.go:819-847), grouped by
 * (FromType,FromUID,ToType,ToUID). from/to are the caller's dense ids for pod
 * and service ends and the raw IPv4 for outbound ends (aggregator/data.go:862). */
typedef struct alz_edge_out {
  uint8_t from_type; /* ALZ_NODE_* */
  uint8_t to_type;
  uint8_t _pad[6];
  uint32_t from;
  uint32_t to;
  uint64_t count;
  uint64_t err5xx;
  uint64_t lat_sum_ns;
  uint32_t hist[ALZ_NB];
} alz_edge_out;

typedef struct alz_config {
  uint32_t abi_version;     /* ALZ_ABI_VERSION */
  int32_t device;           /* CUDA device ordinal */
  uint32_t max_endpoints;   /* pods + services the tables must hold */
  uint32_t max_pairs;       /* distinct (saddr,daddr) pairs per window */
  uint32_t max_edges;       /* distinct edges per window */
  uint32_t max_batch;       /* largest n of one alz_submit_l7 (host staging) */
  uint32_t flags;           /* ALZ_CFG_* */
  uint32_t _reserved[9];
} alz_config;

#define ALZ_CFG_EAGER_JOIN 0x1u /* resolve every event through the tables before
                                   reducing (the textbook plan) instead of
                                   reducing per socket pair and joining the
                                   distinct pairs (default); same results */

#define ALZ_CFG_NO_SMEM_CACHE 0x2u /* ingest without the per-CTA shared-memory cache of
                                      hot socket pairs (profiling comparison only) */

typedef struct alz_stats {
  uint64_t events_in;        /* records submitted */
  uint64_t rows_emitted;     /* rows the reference would have persisted */
  uint64_t not_request;      /* protocol switch emits no request row
                                (HTTP2/KAFKA/UNKNOWN, payload reject) */
  uint64_t src_unresolved;   /* setFromToV2 error: saddr is not a pod
                                (aggregator/data.go:829-832) */
  uint64_t pairs_live;
  uint64_t edges_live;
  uint64_t tcp_events_in;
  uint64_t tcp_localhost_dropped; /* aggregator/data.go:409, 455 */
  uint64_t capacity_events;  /* events lost to an exhausted pair/edge table (cumulative) */
  uint64_t windows;          /* windows flushed */
  uint64_t kernel_launches;  /* kernels of this library launched so far (CUB passes, memsets, copies not counted) */
  uint64_t collective_bytes_last; /* bytes this rank contributed to / received from the last window's collective */
  uint64_t flush_local_us_last;   /* device time of the last flush up to the cross-rank merge */
  uint64_t merge_us_last;         /* device time of the last cross-rank merge (0 on one rank) */
  uint64_t late_events;           /* time-cut windows: records older than the open window (cumulative) */
  uint64_t deferred_events;       /* time-cut windows: records waiting on the device for their window */
} alz_stats;

typedef struct alz_handle alz_handle;

/* ---- lifecycle -------------------------------------------------------------- */
int alz_create(const alz_config* cfg, alz_handle** out);
int alz_destroy(alz_handle* h);
const char* alz_strerror(int status);
const char* alz_last_cuda_error(alz_handle* h);
/* Run all device work of this handle on `cuda_stream` (a cudaStream_t; 0 =
 * the library's own stream). Lets a host time the work with its own events. */
int alz_set_stream(alz_handle* h, void* cuda_stream);
int alz_sync(alz_handle* h);

/* ---- join build side: replaces ClusterInfo map writes ------------------------
 * (aggregator/persist.go:55-71 PodIPToPodUid, :114-130 ServiceIPToServiceUid).
 * UID strings stay with the caller, who interns them to dense ids < 2^29.
 * Single writer. Changes become visible to submits after alz_table_commit,
 * which first folds everything already submitted through the old tables, so
 * each event is resolved by the tables in force when it was submitted. */
int alz_table_upsert(alz_handle* h, int table, uint32_t ipv4, uint32_t id);
int alz_table_erase(alz_handle* h, int table, uint32_t ipv4);
/* n upserts in one call (informer resync / initial list: k8s/informer.go hands the whole cluster at start).
 * Not atomic: the upserts are applied in order and the call stops at the first that fails, returning
 * ALZ_E_INVAL (ids[i] >= 2^29) or ALZ_E_CAPACITY (a new address with max_endpoints already in the table).
 * The upserts before it stay staged and take effect at the next alz_table_commit; the rest are not applied. */
int alz_table_upsert_batch(alz_handle* h, int table, const uint32_t* ipv4, const uint32_t* ids, size_t n);
int alz_table_commit(alz_handle* h);

/* ---- event ingest: replaces processL7 .. PersistRequest --------------------
 * (aggregator/data.go:1364-1383 dispatch, :1081-1362 row build,
 *  :827-870 setFromToV2). The alz_submit_* calls may be made from many OS threads at once, like the
 * reference's 4*NumCPU processL7 workers (aggregator/data.go:230-232): callers copy into separate
 * pinned staging slots in parallel and only the enqueue is serialised. A flush or table commit is
 * ordered after every submit that returned before it was called. */
int alz_submit_l7(alz_handle* h, const alz_l7_rec* host_recs, size_t n);
/* same, records already resident in this GPU's HBM */
int alz_submit_l7_device(alz_handle* h, const alz_l7_rec* dev_recs, size_t n);
/* same, 16-B packed records (host memory); dur_overflow[n_overflow] holds the durations the records
 * index (may be NULL when n_overflow == 0) */
int alz_submit_l7_packed(alz_handle* h, const alz_l7_rec16* host_recs, size_t n,
                         const uint64_t* dur_overflow, size_t n_overflow);
int alz_submit_l7_packed_device(alz_handle* h, const alz_l7_rec16* dev_recs, size_t n,
                                const uint64_t* dev_dur_overflow);
/* host-side packer: alz_l7_rec[n] -> alz_l7_rec16[n]; overflow durations appended to dur_overflow
 * (capacity cap_overflow). Returns the number of overflow entries written, or -1 if cap is too small. */
long alz_pack_l7(const alz_l7_rec* recs, size_t n, alz_l7_rec16* out, uint64_t* dur_overflow, size_t cap_overflow);
/* n raw perf samples exactly as perf.Reader yields them: 1096-B
 * struct l7_event (ebpf/l7_req/l7.go:345-369, :704); payload ignored. */
int alz_submit_l7_raw(alz_handle* h, const void* host_bpf_l7_events, size_t n);
#define ALZ_BPF_L7_EVENT_SIZE 1096

/* ---- window result: the grouped rows ----------------------------------------
 * Folds pending pairs, (multi-GPU: merges all ranks, one all-reduce on the
 * accumulators), writes the live edges in ascending packed-key order
 * (docs/SPEC.md §3; the same order on every rank) and resets the window. n_out is always set to the number of live edges; if
 * cap is too small returns ALZ_E_CAPACITY and keeps the window. */
int alz_window_flush(alz_handle* h, alz_edge_out* out, size_t cap, size_t* n_out);
/* as above but leaves the result on the device for alz_gnn_score / peers;
 * *dev_edges stays valid until the next flush on this handle */
int alz_window_flush_device(alz_handle* h, const alz_edge_out** dev_edges, size_t* n_out);
/* the rows of the last flushed window once more. On a multi-rank handle the merge consumes the window on
 * every rank, so a flush whose `cap` was too small cannot keep it: it returns ALZ_E_CAPACITY with *n_out set
 * and the merged rows stay fetchable here until the next flush. */
int alz_window_fetch(alz_handle* h, alz_edge_out* out, size_t cap, size_t* n_out);
int alz_get_stats(alz_handle* h, alz_stats* out);

/* ---- time-cut windows (SURVEY §8 row R13, docs/SPEC.md §8) ---------------------
 * By default a window is whatever was submitted between two flushes. After alz_window_clock the records' own
 * write_time decides: epoch(t) = convertKernelTimeToUserspaceTime(t) / window_ns with
 * convertKernelTimeToUserspaceTime(t) = first_user_ns - (first_kernel_ns - t) (aggregator/data.go:1740-1743;
 * l7_req.FirstKernelTime / FirstUserspaceTime). The open window is the epoch of the first record submitted
 * afterwards. A record of a later epoch is kept on the device and submitted again by the flush that opens its
 * window; a record of an earlier epoch is late: it is reduced into the open window and counted
 * (alz_stats.late_events). Each alz_window_flush* closes the open epoch and opens the next one. Only 32-byte
 * records carry a write time: packed submits return ALZ_E_STATE while the clock is set. window_ns = 0 turns
 * the clock off again.
 * Several ranks (alz_comm_init): every rank must set the same clock, the same window_ns and the same offset
 * first_user_ns - first_kernel_ns; otherwise the next flush returns ALZ_E_STATE on every rank and every rank
 * keeps its window. Each rank opens at its own first record; a flush merges epoch E, the smallest open epoch of
 * the ranks (the past state after every epoch). A rank at E is flushed and advances; a rank ahead of E keeps its
 * window, its set-aside records and any loss it recorded until E reaches it; a rank with no epoch yet opens E + 1.
 * After one merge at E the ranks agree and advance together (docs/SPEC.md §8 "Several ranks"). */
int alz_window_clock(alz_handle* h, uint64_t first_kernel_ns, uint64_t first_user_ns, uint64_t window_ns);
/* epoch of the open window; ALZ_E_STATE until the first record has been submitted */
int alz_window_epoch(alz_handle* h, uint64_t* epoch);

/* ---- rolling windows (docs/SPEC.md §12) -------------------------------------------
 * Keep the rows of the last `depth` flushed windows on the device, in an arena of `arena_rows` alz_edge_out
 * rows (296 B each). depth = 0 turns the history off and frees it. A call with other values than the current
 * ones drops what is retained; a call with the current values changes nothing. Off by default.
 * Every flush that consumes its window appends that window's rows (what alz_window_fetch would return), also a
 * window of 0 rows and one returned with ALZ_E_CAPACITY; a flush that keeps its window appends nothing. Appending
 * evicts the oldest windows until at most `depth` remain and the rows fit; a window with more rows than the
 * arena clears the history and is not retained. arena_rows >= 2^31 (or 0 with depth > 0): ALZ_E_INVAL; no
 * memory: ALZ_E_NOMEM and the history is off. */
int alz_window_history(alz_handle* h, uint32_t depth, uint64_t arena_rows);

typedef struct alz_rollup_info {
  uint32_t windows;        /* windows summed: min(k, retained) */
  uint32_t clocked;        /* 1: every summed window was cut by alz_window_clock and the epochs below are set */
  uint64_t window_first;   /* alz_stats.windows as it was after the oldest / newest summed window's flush */
  uint64_t window_last;
  uint64_t epoch_first;    /* the epochs those flushes closed (several ranks: the merged epoch E) */
  uint64_t epoch_last;
  uint64_t rows_in;        /* rows read: the sum of the summed windows' row counts */
} alz_rollup_info;

/* The last k retained windows added up per edge: count, err5xx, lat_sum_ns mod 2^64, hist cells mod 2^32, in
 * ascending packed-key order: what one window holding those windows' events would have returned. Rows are
 * matched by (from_type, from, to_type, to), that is by the CALLER'S ids: a pod or service id that was given
 * to another UID inside the retained span merges the two nodes into one. The number of rows is not bounded by
 * max_edges. Reads only: the open window, the last flushed window (alz_window_fetch, alz_gnn_score) and the
 * history are unchanged. *n_out = rows of the sum; cap too small: ALZ_E_CAPACITY, nothing written, call again.
 * ALZ_E_STATE without a history; ALZ_E_INVAL for k = 0. info may be NULL. */
int alz_window_rollup(alz_handle* h, uint32_t k, alz_edge_out* out, size_t cap, size_t* n_out, alz_rollup_info* info);
/* same, rows left on the device; valid until the next rollup or alz_window_history on this handle */
int alz_window_rollup_device(alz_handle* h, uint32_t k, const alz_edge_out** dev_rows, size_t* n_out,
                             alz_rollup_info* info);

/* ---- tiered history (docs/SPEC.md §13) ---------------------------------------------
 * Tier 1 sums `factor` consecutive consumed windows into one entry, tier t + 1 sums `factor` consecutive entries of
 * tier t, so a few retained entries span minutes, hours or days. The windows that enter tier 1 are exactly those
 * that enter the window history (§12), whether or not that is on. Block boundaries are counted from the configuring
 * call and never move. A block with more distinct rows than block_rows, or more rows than its arena, is not
 * retained: it clears its tier, and the blocks of the tiers above that would contain it are dropped when they close
 * (each drop counted in alz_tier_state.dropped). The open block of each tier lives on the device; a flush that closes
 * no block adds no host synchronisation. */
#define ALZ_MAX_TIERS 4
typedef struct alz_history_tier {
  uint32_t factor;         /* entries of the tier below that one entry of this tier sums (>= 2) */
  uint32_t depth;          /* entries retained (>= 1) */
  uint64_t arena_rows;     /* rows of the ring the retained entries live in (1 .. 2^31 - 1), as in §12 */
  uint64_t block_rows;     /* distinct rows the open block can hold (1 .. 2^31 - 1) */
} alz_history_tier;

/* Configure tiers 1..n (n <= ALZ_MAX_TIERS; n = 0 frees them). The current values change nothing; other values drop
 * every retained entry and open block. Bad values, among them tiers whose retained entries would cover 2^32
 * flushed windows or more (factor_1 x ... x factor_t x depth_t): ALZ_E_INVAL; no memory: ALZ_E_NOMEM and the tiers
 * are off.
 * alz_window_history never touches the tiers and this call never touches the window history. Off by default. */
int alz_window_history_tiers(alz_handle* h, const alz_history_tier* tiers, uint32_t n);

/* The last k closed entries of tier `tier` added up per edge, as alz_window_rollup does (tier 0 is
 * alz_window_rollup). The open blocks are never included; the call reads only. info->windows counts flushed windows
 * covered, window_* / epoch_* refer to the oldest and newest of them, rows_in counts entry rows read.
 * ALZ_E_STATE without tiers; ALZ_E_INVAL for k = 0 or a tier above the configured ones. */
int alz_window_rollup_tier(alz_handle* h, uint32_t tier, uint32_t k, alz_edge_out* out, size_t cap, size_t* n_out,
                           alz_rollup_info* info);
/* same, rows left on the device; valid until the next tier rollup or alz_window_history_tiers on this handle */
int alz_window_rollup_tier_device(alz_handle* h, uint32_t tier, uint32_t k, const alz_edge_out** dev_rows,
                                  size_t* n_out, alz_rollup_info* info);

typedef struct alz_tier_state {
  uint32_t entries;        /* entries retained */
  uint32_t open_windows;   /* flushed windows in the open block */
  uint64_t dropped;        /* blocks not retained since the configuring call */
} alz_tier_state;
/* tier 1..n: ALZ_E_INVAL otherwise; ALZ_E_STATE without tiers */
int alz_window_tier_state(alz_handle* h, uint32_t tier, alz_tier_state* st);

/* ---- span rollups (docs/SPEC.md §14) -----------------------------------------------
 * The last N consumed windows up to now, added up from whatever is retained: window-history entries, closed tier
 * entries and the open blocks of the tiers (a tier's open block counts when it has an input, is not poisoned by a
 * dropped block below and has not overflowed). Of the spans m that disjoint retained pieces cover exactly (the last
 * m windows), ALZ_SPAN_AT_MOST takes the largest m <= N (0: an empty result), ALZ_SPAN_AT_LEAST the smallest m >= N,
 * or the largest m there is when none reaches N; info->r.windows == N means the answer is exact. Of the pieces that
 * cover m, the fewest source rows are read (ties: fewer pieces, then the coarser piece, oldest first). Rows as
 * alz_window_rollup returns them, not bounded by max_edges. Reads only: nothing retained, no open block and no
 * earlier rollup's device rows change. ALZ_E_INVAL for N = 0 or an unknown mode; ALZ_E_STATE with neither the
 * window history nor the tiers on; ALZ_E_CAPACITY with nothing written for more than 2^31 - 1 source rows, or
 * (host call) for cap below *n_out. info may be NULL. */
#define ALZ_SPAN_AT_MOST  0u
#define ALZ_SPAN_AT_LEAST 1u
typedef struct alz_span_info {
  alz_rollup_info r;                     /* windows covered, window_ / epoch_ first / last, clocked, rows_in */
  uint32_t entries[1 + ALZ_MAX_TIERS];   /* closed entries used per tier (0 = window history) */
  uint32_t open_blocks;                  /* bit t: tier t's open block was used */
  uint32_t _reserved[2];
} alz_span_info;
int alz_window_rollup_span(alz_handle* h, uint64_t windows, uint32_t mode, alz_edge_out* out, size_t cap,
                           size_t* n_out, alz_span_info* info);
/* same, rows left on the device; valid until the next span rollup on this handle */
int alz_window_rollup_span_device(alz_handle* h, uint64_t windows, uint32_t mode, const alz_edge_out** dev_rows,
                                  size_t* n_out, alz_span_info* info);

/* ---- GNN anomaly pass over the last flushed window (docs/SPEC.md §6) -------- */
int alz_gnn_score(alz_handle* h, float* edge_scores, size_t cap, size_t* n_out);
/* same, scores left on the device (valid until the next call on this handle) */
int alz_gnn_score_device(alz_handle* h, const float** dev_scores, size_t* n_out);
/* quantiles from the histogram, the same float64 interpolation the scores use */
int alz_edge_quantiles(const alz_edge_out* e, const double* qs, size_t nq, double* out_ns);

/* ---- GNN anomaly pass over a rollup (docs/SPEC.md §15) ---------------------------
 * The pass of §6 over the rows that the last rollup call of a kind returned with ALZ_OK: nodes are the distinct edge
 * ends of those rows, and scores[i] belongs to row i of the rollup (ascending packed-key order). The result is a
 * function of the rows and their order alone, so a rollup of one window scores bit for bit as alz_gnn_score scored
 * that window after its flush. The rows stay scorable until the next call of that kind; window rollups' rows also
 * go with an alz_window_history call with other values, tier rollups' with an alz_window_history_tiers call with
 * other values (span rows survive both). A call of that kind that does not return ALZ_OK (ALZ_E_CAPACITY of a host
 * call, k = 0, ...) leaves nothing to score: ALZ_E_STATE, as before any such call. ALZ_E_INVAL for an unknown kind.
 * A 0-row rollup scores to *n_out = 0. *n_out is always set; cap too small: ALZ_E_CAPACITY, nothing written. Reads
 * only: the rollup's rows, every retained entry, the open blocks and the window are unchanged. A rollup above
 * max_edges rows grows the GNN state (it never shrinks); no memory: ALZ_E_NOMEM. Scores and alz_gnn_nodes refer to
 * the last GNN pass on the handle, window or rollup; device scores stay valid until the next GNN call. Several
 * ranks hold the same rollup rows, so they get the same scores with no collective. */
#define ALZ_ROLLUP_WINDOWS 0u   /* alz_window_rollup*, and alz_window_rollup_tier* with tier 0 */
#define ALZ_ROLLUP_TIER    1u   /* alz_window_rollup_tier* with tier >= 1 */
#define ALZ_ROLLUP_SPAN    2u   /* alz_window_rollup_span* */
int alz_gnn_score_rollup(alz_handle* h, uint32_t kind, float* scores, size_t cap, size_t* n_out);
/* same, scores left on the device (valid until the next GNN call on this handle) */
int alz_gnn_score_rollup_device(alz_handle* h, uint32_t kind, const float** dev_scores, size_t* n_out);

/* ---- top anomalous rows (docs/SPEC.md §16) ----------------------------------------
 * The pass of §6 / §15, then only its best rows: the first min(k, above) rows in rank order, where each score maps to
 * the key u ^ 0x80000000 (sign bit clear) or ~u (set) of its bits u (IEEE total order), rows rank by key descending,
 * then by row index ascending, and a row is eligible when key(score) >= key(min_score). Result j: the row
 * (byte for byte as in the window or rollup), its score (bit for bit what alz_gnn_score* returns for it) and its row
 * index. rows, scores, index and info may each be NULL. *n_out is always set; cap too small: ALZ_E_CAPACITY, nothing
 * written. k = 0, a NaN min_score or an unknown kind: ALZ_E_INVAL; no rollup rows to score: ALZ_E_STATE, as in §15; a
 * 0-row source: *n_out = 0. More than 2^30 - 1 rows: ALZ_E_CAPACITY; no memory: ALZ_E_NOMEM. Reads only, as §15;
 * alz_gnn_nodes then refers to this pass. The pass always runs. The result is a function of the rows and their order
 * alone: every rank gets the same result with no collective. Device results stay valid until the next GNN call. */
typedef struct alz_top_info {
  uint64_t scored;   /* rows the pass scored */
  uint64_t above;    /* of those, rows whose score is >= min_score (before the cut at k) */
} alz_top_info;
/* over the last flushed window, the rows alz_gnn_score scores */
int alz_gnn_top(alz_handle* h, uint32_t k, float min_score, alz_edge_out* rows, float* scores, uint32_t* index,
                size_t cap, size_t* n_out, alz_top_info* info);
int alz_gnn_top_device(alz_handle* h, uint32_t k, float min_score, const alz_edge_out** dev_rows,
                       const float** dev_scores, const uint32_t** dev_index, size_t* n_out, alz_top_info* info);
/* over the rows the last rollup of `kind` (ALZ_ROLLUP_*) returned, the rows alz_gnn_score_rollup scores */
int alz_gnn_top_rollup(alz_handle* h, uint32_t kind, uint32_t k, float min_score, alz_edge_out* rows, float* scores,
                       uint32_t* index, size_t cap, size_t* n_out, alz_top_info* info);
int alz_gnn_top_rollup_device(alz_handle* h, uint32_t kind, uint32_t k, float min_score, const alz_edge_out** dev_rows,
                              const float** dev_scores, const uint32_t** dev_index, size_t* n_out, alz_top_info* info);

/* ---- edge metrics and the top edges by a metric (docs/SPEC.md §17) ------------------------------------------------
 * A metric's value for one row is a float64: COUNT (double)count; ERR5XX (double)err5xx; ERR_RATE err5xx / count;
 * MEAN_NS lat_sum_ns / count (the stored sum, mod 2^64); the last two are 0 for count = 0. QUANTILE: the SPEC §5
 * q-quantile of the row's histogram, bit for bit what alz_edge_quantiles(row, &q, 1, &v) returns. q must be in [0, 1]
 * for QUANTILE and is ignored otherwise. Every value is finite and >= +0.
 * Sources: the last flushed window (the rows alz_gnn_score scores), or the rows the last rollup of `kind`
 * (ALZ_ROLLUP_*) returned, with the availability rule of §15 (none: ALZ_E_STATE). *n_out is always set; a host call
 * whose cap (in rows) is below it returns ALZ_E_CAPACITY and writes nothing. k = 0, nm of 0 or more than
 * ALZ_MAX_METRICS, an unknown metric or rollup kind, a q outside [0, 1] or NaN, a NaN min_value or a null required
 * pointer: ALZ_E_INVAL. A 0-row source: *n_out = 0. More than 2^30 - 1 rows: ALZ_E_CAPACITY; no memory: ALZ_E_NOMEM.
 * Reads only: no GNN pass runs and the GNN's scores, top results and alz_gnn_nodes stay valid; the source rows stay
 * scorable. Device results stay valid until the next metric call on the handle. Every rank holds the same rows, so
 * every rank gets the same result with no collective. */
#define ALZ_METRIC_COUNT    0u
#define ALZ_METRIC_ERR5XX   1u
#define ALZ_METRIC_ERR_RATE 2u
#define ALZ_METRIC_MEAN_NS  3u
#define ALZ_METRIC_QUANTILE 4u
#define ALZ_MAX_METRICS     8u
typedef struct alz_metric {
  uint32_t kind;   /* ALZ_METRIC_* */
  uint32_t _pad;
  double q;        /* ALZ_METRIC_QUANTILE: the quantile, in [0, 1] */
} alz_metric;
/* values[i * nm + j]: metric j of row i of the last flushed window, in its row order; cap counts rows */
int alz_edge_metrics(alz_handle* h, const alz_metric* m, uint32_t nm, double* values, size_t cap, size_t* n_out);
int alz_edge_metrics_device(alz_handle* h, const alz_metric* m, uint32_t nm, const double** dev_values, size_t* n_out);
/* same, over the rows the last rollup of `kind` (ALZ_ROLLUP_*) returned */
int alz_edge_metrics_rollup(alz_handle* h, uint32_t kind, const alz_metric* m, uint32_t nm, double* values, size_t cap,
                            size_t* n_out);
int alz_edge_metrics_rollup_device(alz_handle* h, uint32_t kind, const alz_metric* m, uint32_t nm,
                                   const double** dev_values, size_t* n_out);
/* The first min(k, above) rows by one metric's value, ranked as alz_gnn_top ranks scores but on the 64-bit key of the
 * float64 value (u ^ 2^63 with the sign bit clear, ~u with it set), key descending, then row index ascending; a row is
 * eligible when key(value) >= key(min_value). Result j: the row (byte for byte), its value (bit for bit what
 * alz_edge_metrics* gives) and its row index; rows, values, index and info may each be NULL. info->scored = the
 * source's rows, info->above = the eligible ones. Counts above 2^53 rank by their float64 value. */
int alz_edge_top(alz_handle* h, const alz_metric* m, uint32_t k, double min_value, alz_edge_out* rows, double* values,
                 uint32_t* index, size_t cap, size_t* n_out, alz_top_info* info);
int alz_edge_top_device(alz_handle* h, const alz_metric* m, uint32_t k, double min_value, const alz_edge_out** dev_rows,
                        const double** dev_values, const uint32_t** dev_index, size_t* n_out, alz_top_info* info);
int alz_edge_top_rollup(alz_handle* h, uint32_t kind, const alz_metric* m, uint32_t k, double min_value,
                        alz_edge_out* rows, double* values, uint32_t* index, size_t cap, size_t* n_out,
                        alz_top_info* info);
int alz_edge_top_rollup_device(alz_handle* h, uint32_t kind, const alz_metric* m, uint32_t k, double min_value,
                               const alz_edge_out** dev_rows, const double** dev_values, const uint32_t** dev_index,
                               size_t* n_out, alz_top_info* info);

/* ---- edge changes against a pinned baseline (docs/SPEC.md §18) ----------------------------------------------------
 * A source is the last flushed window (ALZ_SOURCE_WINDOW) or the rows the last rollup of a kind (ALZ_ROLLUP_*)
 * returned, with the availability rule of §15 (none: ALZ_E_STATE). alz_baseline_pin copies the source's rows, their
 * packed keys and its alz_rollup_info into a baseline the handle owns (a window: windows = 1 and what a k = 1
 * alz_window_rollup reports for it; a rollup: what that rollup call reported). The baseline survives flushes,
 * rollups, alz_window_history* and every GNN or metric call; it goes with the next pin, alz_baseline_clear or
 * alz_destroy. An empty source pins an empty baseline. info may be NULL. A failed growth: ALZ_E_NOMEM, no baseline. */
#define ALZ_SOURCE_WINDOW 0xFFFFFFFFu   /* the last flushed window; the other sources are ALZ_ROLLUP_* */
int alz_baseline_pin(alz_handle* h, uint32_t source, alz_rollup_info* info);
int alz_baseline_clear(alz_handle* h);
/* The union of a source's rows and the baseline's, matched by packed key (§3), in ascending key order, keeping the
 * rows whose presence bit is in `presence`. value / base_value: the §17 value of metric m on the source / baseline row,
 * bit for bit what alz_edge_metrics* gives, divided by the side's windows for COUNT and ERR5XX (one rounding); 0 on a
 * side where the row is absent. change: from value and base_value by mode, one rounding. Unknown metric, mode or
 * source, presence 0 or above 7, or a null required pointer: ALZ_E_INVAL. No baseline, or no source rows: ALZ_E_STATE.
 * *n_out is always set; a host call whose cap (in records) is below it returns ALZ_E_CAPACITY and writes nothing. A
 * union of more than 2^30 - 1 rows: ALZ_E_CAPACITY; no memory: ALZ_E_NOMEM. info may be NULL. Reads only: the source,
 * the baseline, GNN state and metric results are unchanged. Device results stay valid until the next change call.
 * Every rank holds the same rows and pins the same baseline, so every rank gets the same result with no collective. */
#define ALZ_CHANGE_DELTA 0u   /* change = value - base_value */
#define ALZ_CHANGE_DROP  1u   /* change = base_value - value */
#define ALZ_CHANGE_RATIO 2u   /* base_value > 0: value / base_value; base_value = 0: +inf when value > 0, else 1.0 */
#define ALZ_PRESENT_BOTH 0x1u /* presence bits, and the filter mask: in both */
#define ALZ_PRESENT_NEW  0x2u /* in the source only */
#define ALZ_PRESENT_GONE 0x4u /* in the baseline only */
typedef struct alz_edge_change {   /* 48 B */
  uint8_t from_type;     /* ALZ_NODE_* */
  uint8_t to_type;
  uint8_t presence;      /* ALZ_PRESENT_* */
  uint8_t _pad[5];
  uint32_t from;
  uint32_t to;
  uint32_t index;        /* row index in the source, 0xFFFFFFFF when absent */
  uint32_t base_index;   /* row index in the baseline, 0xFFFFFFFF when absent */
  double value;
  double base_value;
  double change;
} alz_edge_change;
typedef struct alz_change_info {
  uint64_t source_rows, base_rows;    /* the two sides' rows */
  uint64_t both, added, gone;         /* the union by presence, before the filter */
  uint64_t listed;                    /* union rows that pass the presence filter */
  uint64_t above;                     /* top calls: listed rows with key(change) >= key(min_change); 0 otherwise */
  uint32_t source_windows, base_windows;
} alz_change_info;
/* every listed row, in ascending key order */
int alz_edge_changes(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode, uint32_t presence,
                     alz_edge_change* out, size_t cap, size_t* n_out, alz_change_info* info);
int alz_edge_changes_device(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode, uint32_t presence,
                            const alz_edge_change** dev_out, size_t* n_out, alz_change_info* info);
/* The first min(k, above) listed rows by change, ranked as alz_edge_top ranks values (64-bit key of the float64,
 * descending, then position in the list ascending); a row is eligible when key(change) >= key(min_change). k = 0 or a
 * NaN min_change: ALZ_E_INVAL. */
int alz_edge_changes_top(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode, uint32_t presence,
                         uint32_t k, double min_change, alz_edge_change* out, size_t cap, size_t* n_out,
                         alz_change_info* info);
int alz_edge_changes_top_device(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode, uint32_t presence,
                                uint32_t k, double min_change, const alz_edge_change** dev_out, size_t* n_out,
                                alz_change_info* info);

/* ---- edge series (docs/SPEC.md §19) --------------------------------------------------------------------------------
 * The §17 metric values of a set of edges in each of the last P = min(k, retained) closed entries of one ring, oldest
 * first: the window history (tier 0) or tier t >= 1. Series row i is row i of a source (ALZ_SOURCE_WINDOW or
 * ALZ_ROLLUP_*, with the availability rule of §15) or the caller's edge keys[i]. values[(i * P + j) * nm + m] is metric
 * m on the row entry j holds for edge i (matched by packed key, §3), bit for bit what alz_edge_metrics* gives for that
 * row; present[i * P + j] = 1 when the entry holds the edge, else 0 and every value +0.0. points[j] is what a rollup of
 * entry j alone reports; points needs room for P <= k entries. *n_out (series rows) and *n_points (P) are always set;
 * a host call whose cap (in series rows) is below *n_out returns ALZ_E_CAPACITY and writes nothing else. k = 0, a tier
 * above the configured ones, a bad metric list (§17), an unknown source, a malformed key or a null required pointer:
 * ALZ_E_INVAL. Tier 0 without the window history, t >= 1 without tiers, or no rows of a rollup source: ALZ_E_STATE.
 * More than 2^30 - 1 slots (rows x P): ALZ_E_CAPACITY; no memory: ALZ_E_NOMEM. No retained entry: P = 0, ALZ_OK.
 * present, points and info may be NULL. Reads only: the window, the retained entries, the open blocks, every rollup's
 * rows, the baseline, metric, top, change and GNN results are unchanged. Device results stay valid until the next
 * series call. Every rank holds the same history, so every rank gets the same result with no collective. */
typedef struct alz_edge_ends {   /* 16 B: the head of alz_edge_out; _pad is ignored */
  uint8_t from_type;   /* ALZ_NODE_* */
  uint8_t to_type;
  uint8_t _pad[6];
  uint32_t from;
  uint32_t to;
} alz_edge_ends;
typedef struct alz_series_info {
  uint64_t edges;      /* series rows: the source's rows or n_keys */
  uint64_t rows_in;    /* entry rows read: the sum of the P entries' rows */
  uint32_t points;     /* P */
  uint32_t tier;
} alz_series_info;
/* every row of a source; cap counts series rows */
int alz_edge_series(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m, uint32_t nm,
                    double* values, uint8_t* present, size_t cap, size_t* n_out, uint32_t* n_points,
                    alz_rollup_info* points, alz_series_info* info);
int alz_edge_series_device(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m, uint32_t nm,
                           const double** dev_values, const uint8_t** dev_present, size_t* n_out, uint32_t* n_points,
                           alz_rollup_info* points, alz_series_info* info);
/* the caller's edges, keys in host memory, in the caller's order; duplicates get identical rows. A key no flush can
 * produce (a node type above 3, neither end a pod, a pod or service id >= 2^29) is malformed. A pod <-> pod edge named
 * (A, B) is the row a flush emitted with from = A, to = B. */
int alz_edge_series_keys(alz_handle* h, const alz_edge_ends* keys, size_t n_keys, uint32_t tier, uint32_t k,
                         const alz_metric* m, uint32_t nm, double* values, uint8_t* present, size_t cap, size_t* n_out,
                         uint32_t* n_points, alz_rollup_info* points, alz_series_info* info);
int alz_edge_series_keys_device(alz_handle* h, const alz_edge_ends* keys, size_t n_keys, uint32_t tier, uint32_t k,
                                const alz_metric* m, uint32_t nm, const double** dev_values,
                                const uint8_t** dev_present, size_t* n_out, uint32_t* n_points,
                                alz_rollup_info* points, alz_series_info* info);

/* ---- edge trends (docs/SPEC.md §20) --------------------------------------------------------------------------------
 * One statistic per row of a source (ALZ_SOURCE_WINDOW or ALZ_ROLLUP_*, with the availability rule of §15) over that
 * row's §19 series of one metric in the last P = min(k, retained) closed entries of one ring (tier 0: the window
 * history; t >= 1: a tier), oldest first: the least-squares slope, or the recent points' mean against the earlier
 * points' mean as a shift, a ratio or a z-score (SPEC §20 gives every rounding). The top calls rank the valid rows as
 * alz_edge_top ranks values (64-bit key of the float64 trend, descending, then source row ascending; eligible when
 * key(trend) >= key(min_trend)) and return the first min(top, above) with their source rows and their series.
 * *n_out and *n_points (P) are always set; a host call whose cap is below *n_out returns ALZ_E_CAPACITY and writes
 * nothing else. k < 2, recent outside [1, k - 1], an unknown stat, direction or absent mode, a bad metric (§17), an
 * unknown source, top = 0, a NaN min_trend or a null required pointer: ALZ_E_INVAL. Tier 0 without the window history,
 * t >= 1 without tiers, or no rows of a rollup source: ALZ_E_STATE. More than 2^30 - 1 slots (rows x P):
 * ALZ_E_CAPACITY; no memory: ALZ_E_NOMEM. No retained entry: P = 0, every row invalid, ALZ_OK. points (room for k
 * entries) and info may be NULL. Reads only: the window, the retained entries, the open blocks, every rollup's rows,
 * the baseline, and the series, metric, top, change and GNN results are unchanged. Device results stay valid until the
 * next trend call. Every rank holds the same history, so every rank gets the same result with no collective. */
#define ALZ_TREND_SLOPE  0u   /* least-squares slope of y against the point index, in metric units per point */
#define ALZ_TREND_SHIFT  1u   /* recent - before */
#define ALZ_TREND_RATIO  2u   /* recent / before; before = 0: +inf when recent > 0, else 1.0 */
#define ALZ_TREND_ZSCORE 3u   /* (recent - before) / the population standard deviation of the earlier points */
#define ALZ_TREND_RISING  0u  /* the largest rises rank first */
#define ALZ_TREND_FALLING 1u  /* the largest falls rank first: -slope, before - recent, before / recent */
#define ALZ_TREND_ABSENT_SKIP 0u   /* a point where the entry does not hold the edge is left out */
#define ALZ_TREND_ABSENT_ZERO 1u   /* ... counts as +0.0 (no traffic) */
typedef struct alz_trend {   /* 24 B */
  uint32_t stat;         /* ALZ_TREND_SLOPE / SHIFT / RATIO / ZSCORE */
  uint32_t direction;    /* ALZ_TREND_RISING / FALLING */
  uint32_t absent;       /* ALZ_TREND_ABSENT_SKIP / ABSENT_ZERO */
  uint32_t recent;       /* r: the last r points are "recent"; 1 <= r <= k - 1 */
  uint32_t min_points;   /* a valid row uses at least this many points (0: no extra bound) */
  uint32_t _pad;
} alz_trend;
typedef struct alz_edge_trend {   /* 48 B; the head is laid out as alz_edge_ends / alz_edge_change */
  uint8_t from_type;     /* ALZ_NODE_* */
  uint8_t to_type;
  uint8_t valid;         /* 1: the statistic is defined for this row */
  uint8_t _pad[5];
  uint32_t from;
  uint32_t to;
  uint32_t index;        /* row index in the source */
  uint32_t used;         /* points used */
  double trend;          /* +0.0 when not valid */
  double recent;         /* mean of the used recent points */
  double before;         /* mean of the used earlier points */
} alz_edge_trend;
typedef struct alz_trend_info {
  uint64_t edges;        /* the source's rows */
  uint64_t rows_in;      /* entry rows read: the sum of the P entries' rows */
  uint64_t valid;        /* rows with a defined trend */
  uint64_t above;        /* top calls: eligible rows before the cut; 0 otherwise */
  uint32_t points;       /* P */
  uint32_t tier;
} alz_trend_info;
/* every source row, in source order; cap counts records */
int alz_edge_trends(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m, const alz_trend* t,
                    alz_edge_trend* out, size_t cap, size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                    alz_trend_info* info);
int alz_edge_trends_device(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                           const alz_trend* t, const alz_edge_trend** dev_out, size_t* n_out, uint32_t* n_points,
                           alz_rollup_info* points, alz_trend_info* info);
/* the first min(top, above) valid rows by trend, in rank order: their records, their source rows, and their series
 * (series[j * P + p], present[j * P + p], as alz_edge_series gives for the row with nm = 1). cap counts result rows;
 * series and present need room for cap x k elements. out, rows, series and present may each be NULL (dev_rows,
 * dev_series and dev_present too). */
int alz_edge_trends_top(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                        const alz_trend* t, uint32_t top, double min_trend, alz_edge_trend* out, alz_edge_out* rows,
                        double* series, uint8_t* present, size_t cap, size_t* n_out, uint32_t* n_points,
                        alz_rollup_info* points, alz_trend_info* info);
int alz_edge_trends_top_device(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                               const alz_trend* t, uint32_t top, double min_trend, const alz_edge_trend** dev_out,
                               const alz_edge_out** dev_rows, const double** dev_series, const uint8_t** dev_present,
                               size_t* n_out, uint32_t* n_points, alz_rollup_info* points, alz_trend_info* info);

/* ---- node metrics (docs/SPEC.md §21) -------------------------------------------------------------------------------
 * A node is an edge end (type, value) as in §2: pod 7 and service 7 are different nodes, and so are outbound v and
 * Host-keyed v. The nodes of a source (ALZ_SOURCE_WINDOW or ALZ_ROLLUP_*, with the availability rule of §15) are every
 * from end and every to end of its rows, in ascending node key (type << 32) | value, the key alz_gnn_nodes reports; a
 * node's index is its position in that list. Side IN of a node sums the rows whose to end is the node, side OUT the
 * rows whose from end is; a row whose two ends are one node counts on both. count, err5xx and lat_sum_ns are u64 sums
 * mod 2^64, hist[b] the u32 sum of the rows' cells mod 2^32 (§3); in_edges / out_edges count each side's rows. A node
 * metric is the §17 value of one side's sums, bit for bit what alz_edge_metrics* gives for an alz_edge_out that
 * carries them. Top nodes rank as alz_edge_top ranks rows: 64-bit key of the float64 value, descending, then node
 * index ascending; eligible when key(value) >= key(min_value); the first min(k, above) nodes.
 * *n_out is always set; a host call whose cap (in nodes) is below it returns ALZ_E_CAPACITY and writes nothing. An
 * unknown source, side or metric, nm of 0 or more than ALZ_MAX_METRICS, a q outside [0, 1] or NaN, k = 0, a NaN
 * min_value or a null required pointer: ALZ_E_INVAL. No rows of a rollup source: ALZ_E_STATE. A 0-row source: 0 nodes,
 * ALZ_OK. More than 2^29 - 1 source rows: ALZ_E_CAPACITY, before anything runs; no memory: ALZ_E_NOMEM.
 * Reads only: the window, the retained entries, the open blocks, every rollup's rows and the baseline are unchanged, and
 * so are the GNN, metric, top, change, series and trend results, device pointers included. Device results stay valid
 * until the next node call on the handle. Every rank holds the same rows, so every rank gets the same result with no
 * collective. */
#define ALZ_SIDE_IN  0u   /* the rows into the node: requests it served, messages delivered to it */
#define ALZ_SIDE_OUT 1u   /* the rows out of the node */
typedef struct alz_node_sums {   /* 280 B: laid out as the tail of alz_edge_out from count on */
  uint64_t count;
  uint64_t err5xx;
  uint64_t lat_sum_ns;
  uint32_t hist[ALZ_NB];
} alz_node_sums;
typedef struct alz_node_out {    /* 576 B */
  uint8_t type;          /* ALZ_NODE_* */
  uint8_t _pad[3];
  uint32_t value;
  uint32_t in_edges;     /* rows on the IN side */
  uint32_t out_edges;    /* rows on the OUT side */
  alz_node_sums in;      /* in.count sits at offset 16, as alz_edge_out.count does */
  alz_node_sums out;
} alz_node_out;
/* every node of a source, in node order; cap counts nodes */
int alz_node_rows(alz_handle* h, uint32_t source, alz_node_out* out, size_t cap, size_t* n_out);
int alz_node_rows_device(alz_handle* h, uint32_t source, const alz_node_out** dev_out, size_t* n_out);
/* values[i * nm + j]: metric j of node i's side `side` (ALZ_SIDE_*), in node order; cap counts nodes */
int alz_node_metrics(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t nm, double* values,
                     size_t cap, size_t* n_out);
int alz_node_metrics_device(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t nm,
                            const double** dev_values, size_t* n_out);
/* The first min(k, above) nodes by one metric of one side. Result j: the node's row, its value (bit for bit what
 * alz_node_metrics* gives) and its node index; nodes, values, index and info may each be NULL (dev_nodes, dev_values and
 * dev_index too). info->scored = the source's nodes, info->above = the eligible ones. */
int alz_node_top(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t k, double min_value,
                 alz_node_out* nodes, double* values, uint32_t* index, size_t cap, size_t* n_out, alz_top_info* info);
int alz_node_top_device(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t k,
                        double min_value, const alz_node_out** dev_nodes, const double** dev_values,
                        const uint32_t** dev_index, size_t* n_out, alz_top_info* info);

/* ---- node series and trends (docs/SPEC.md §22) ---------------------------------------------------------------------
 * The §17 metric values of one side (ALZ_SIDE_*) of a set of nodes in each of the last P = min(k, retained) closed
 * entries of one ring, oldest first: the window history (tier 0) or tier t >= 1. Series row i is node i of a source
 * (ALZ_SOURCE_WINDOW or ALZ_ROLLUP_*, with the availability rule of §15, in §21 node order) or the caller's keys[i].
 * Point j of node i is present when entry j holds a row on the side (IN: a row whose to end is the node, OUT: whose
 * from end is); values[(i * P + j) * nm + m] is then metric m of the side's §21 sums over entry j's rows, bit for bit
 * what alz_node_metrics* gives for the node over a source that held entry j alone. An absent point has present 0 and
 * every value +0.0. points[j] is what a rollup of entry j alone reports (room for P <= k entries). *n_out (series rows)
 * and *n_points (P) are always set; a host call whose cap (in series rows) is below *n_out returns ALZ_E_CAPACITY and
 * writes nothing else. k = 0, an unknown side or source, a tier above the configured ones, a bad metric list (§17), a
 * malformed key or a null required pointer: ALZ_E_INVAL. Tier 0 without the window history, t >= 1 without tiers, or
 * no rows of a rollup source: ALZ_E_STATE. A source of more than 2^29 - 1 rows (before anything runs) or more than
 * 2^30 - 1 slots (series rows x P, before the entries are read): ALZ_E_CAPACITY; no memory: ALZ_E_NOMEM. No retained
 * entry: P = 0, ALZ_OK. present, points and info (info->edges counts series rows, here nodes) may be NULL.
 * Reads only: the window, the retained entries, the open blocks, every rollup's rows, the baseline, and the node, edge
 * series, edge trend, metric, top, change and GNN results are unchanged. Device results stay valid until the next call
 * of the same family (node series, node trends). Every rank holds the same history, so every rank gets the same result
 * with no collective. */
typedef struct alz_node_ends {   /* 8 B: the head of alz_node_out; _pad is ignored */
  uint8_t type;                  /* ALZ_NODE_* */
  uint8_t _pad[3];
  uint32_t value;
} alz_node_ends;
/* every node of a source; cap counts series rows */
int alz_node_series(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k, const alz_metric* m,
                    uint32_t nm, double* values, uint8_t* present, size_t cap, size_t* n_out, uint32_t* n_points,
                    alz_rollup_info* points, alz_series_info* info);
int alz_node_series_device(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                           const alz_metric* m, uint32_t nm, const double** dev_values, const uint8_t** dev_present,
                           size_t* n_out, uint32_t* n_points, alz_rollup_info* points, alz_series_info* info);
/* the caller's nodes, keys in host memory, in the caller's order; duplicates get identical rows. A type above
 * ALZ_NODE_OUTBOUND_HOST or a pod or service value >= 2^29 is malformed; a node no entry holds is absent everywhere. */
int alz_node_series_keys(alz_handle* h, const alz_node_ends* keys, size_t n_keys, uint32_t side, uint32_t tier,
                         uint32_t k, const alz_metric* m, uint32_t nm, double* values, uint8_t* present, size_t cap,
                         size_t* n_out, uint32_t* n_points, alz_rollup_info* points, alz_series_info* info);
int alz_node_series_keys_device(alz_handle* h, const alz_node_ends* keys, size_t n_keys, uint32_t side, uint32_t tier,
                                uint32_t k, const alz_metric* m, uint32_t nm, const double** dev_values,
                                const uint8_t** dev_present, size_t* n_out, uint32_t* n_points,
                                alz_rollup_info* points, alz_series_info* info);
/* Node trends: the §20 statistic of each source node's series of one metric of one side, with §20's directions,
 * absent modes, validity rules and roundings; k < 2 and everything alz_edge_trends* refuses is refused the same way.
 * The records are one per source node, in node order; the top calls rank the valid nodes in the §17 order of the trend
 * (then node index ascending) and return the first min(top, above) with the source's alz_node_out rows (as
 * alz_node_rows gives them) and their P-point series (series[j * P + p], present[j * P + p]; room for cap x k each).
 * info->edges counts the source's nodes. */
typedef struct alz_node_trend {  /* 48 B; from `valid` on, laid out as alz_edge_trend */
  uint8_t type;                  /* ALZ_NODE_* */
  uint8_t _pad0;
  uint8_t valid;                 /* 1: the statistic is defined for this node */
  uint8_t _pad1[5];
  uint32_t value;
  uint32_t _pad2;
  uint32_t index;                /* node index in the source (§21 node order) */
  uint32_t used;                 /* points used */
  double trend;                  /* +0.0 when not valid */
  double recent;                 /* mean of the used recent points */
  double before;                 /* mean of the used earlier points */
} alz_node_trend;
int alz_node_trends(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k, const alz_metric* m,
                    const alz_trend* t, alz_node_trend* out, size_t cap, size_t* n_out, uint32_t* n_points,
                    alz_rollup_info* points, alz_trend_info* info);
int alz_node_trends_device(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                           const alz_metric* m, const alz_trend* t, const alz_node_trend** dev_out, size_t* n_out,
                           uint32_t* n_points, alz_rollup_info* points, alz_trend_info* info);
/* out, nodes, series and present may each be NULL (dev_nodes, dev_series and dev_present too) */
int alz_node_trends_top(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k, const alz_metric* m,
                        const alz_trend* t, uint32_t top, double min_trend, alz_node_trend* out, alz_node_out* nodes,
                        double* series, uint8_t* present, size_t cap, size_t* n_out, uint32_t* n_points,
                        alz_rollup_info* points, alz_trend_info* info);
int alz_node_trends_top_device(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                               const alz_metric* m, const alz_trend* t, uint32_t top, double min_trend,
                               const alz_node_trend** dev_out, const alz_node_out** dev_nodes,
                               const double** dev_series, const uint8_t** dev_present, size_t* n_out,
                               uint32_t* n_points, alz_rollup_info* points, alz_trend_info* info);

/* ---- node changes against a pinned baseline (docs/SPEC.md §23) ---------------------------------------------------
 * The §18 comparison for nodes. The source is ALZ_SOURCE_WINDOW or ALZ_ROLLUP_* (availability rule of §15), the
 * baseline the one alz_baseline_pin holds; each side's node list is the §21 node list of its rows. A node is a member
 * of a list on side `side` when it has a row there (IN: in_edges > 0, OUT: out_edges > 0). The list is the union of
 * the two lists' members, matched by node key (type << 32) | value, in ascending key order, keeping the nodes whose
 * presence bit is in `presence`: a node that served requests before and now only makes them is GONE on IN. index /
 * base_index: the node's position in the source's / baseline's full §21 node list (alz_node_rows order), 0xFFFFFFFF
 * where it is not a member. value / base_value: the §17 value of m on that node's side sums, bit for bit what
 * alz_node_metrics* gives, divided by the side's windows for COUNT and ERR5XX (one rounding); +0.0 where absent.
 * change and the top calls' ranking and eligibility: as alz_edge_changes* (§18). info->source_rows / base_rows count
 * each side's member nodes; both, added and gone are counted before the filter, listed after it. Unknown metric,
 * mode, side or source, presence 0 or above 7, k = 0, a NaN min_change or a null required pointer: ALZ_E_INVAL. No
 * baseline, or no rows of a rollup source: ALZ_E_STATE. A side of more than 2^29 - 1 rows (before anything runs) or a
 * union of more than 2^30 - 1 nodes: ALZ_E_CAPACITY; no memory: ALZ_E_NOMEM. *n_out is always set; a host call whose
 * cap (in records) is below it returns ALZ_E_CAPACITY and writes nothing. info may be NULL. Reads only: the window,
 * every ring, the open blocks, every rollup's rows and the baseline are unchanged, and so are the node, node series,
 * node trend, change, metric, top, series, trend and GNN results, device pointers included. The baseline's node rows
 * are grouped on the first node change call after a pin and kept for later calls. Device results stay valid until the
 * next node change call. Every rank holds the same rows and pins the same baseline, so every rank gets the same
 * result with no collective. */
typedef struct alz_node_change {   /* 48 B; presence, index, base_index, value, base_value and change at the offsets
                                      of alz_edge_change's */
  uint8_t type;          /* ALZ_NODE_* */
  uint8_t _pad0;         /* zero */
  uint8_t presence;      /* ALZ_PRESENT_* */
  uint8_t _pad1[5];      /* zero */
  uint32_t node;         /* the node's value: pod or service id, IPv4, Host id (offset 8, as alz_node_trend.value) */
  uint32_t _pad2;        /* zero */
  uint32_t index;        /* §21 node index in the source, 0xFFFFFFFF when absent there */
  uint32_t base_index;   /* §21 node index in the baseline's node list, 0xFFFFFFFF when absent there */
  double value;
  double base_value;
  double change;
} alz_node_change;
/* every listed node, in ascending node key order */
int alz_node_changes(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t mode,
                     uint32_t presence, alz_node_change* out, size_t cap, size_t* n_out, alz_change_info* info);
int alz_node_changes_device(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t mode,
                            uint32_t presence, const alz_node_change** dev_out, size_t* n_out, alz_change_info* info);
/* the first min(k, above) listed nodes by change, in rank order; info->above = the eligible ones */
int alz_node_changes_top(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t mode,
                         uint32_t presence, uint32_t k, double min_change, alz_node_change* out, size_t cap,
                         size_t* n_out, alz_change_info* info);
int alz_node_changes_top_device(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t mode,
                                uint32_t presence, uint32_t k, double min_change,
                                const alz_node_change** dev_out, size_t* n_out, alz_change_info* info);

/* ---- groups (docs/SPEC.md §24) --------------------------------------------------------------------------------------
 * The group map sends nodes to caller-defined groups (a deployment, a namespace): node nodes[i] is a member of group
 * groups[i], the node (ALZ_NODE_GROUP, groups[i]). Any of the four flushed node types may be mapped. alz_group_set
 * replaces the whole map; n = 0 clears it, and a handle starts with it empty. A malformed key (a type above
 * ALZ_NODE_OUTBOUND_HOST, a pod or service value >= 2^29), a group >= 2^29, one node twice in one call, or null arrays
 * with n > 0: ALZ_E_INVAL. More than 2^30 - 1 entries: ALZ_E_CAPACITY; no memory: ALZ_E_NOMEM. Every failure leaves
 * the previous map in force. The map lives on the device; it survives flushes, rollups, pins and every other call and
 * goes with the next alz_group_set or alz_destroy. On several ranks, every rank sets the same map: no collective runs.
 *
 * The group edges of a source (ALZ_SOURCE_WINDOW or ALZ_ROLLUP_*, with the availability rule of §15): each row's from
 * end and to end is replaced by its group when the map holds it and kept otherwise; rows equal in (from_type, from,
 * to_type, to) after that are summed by the §3 rule (count, err5xx, lat_sum_ns mod 2^64, hist cells mod 2^32). Rows
 * come out in ascending (node key of from, node key of to), node key (type << 32) | value: with an empty map, the
 * source's rows in that order. Each row keeps its orientation; a row whose two ends land in one group is an internal
 * row (g -> g) and is kept. Padding is zero. Group edge metrics and top: §17 over the group-edge rows, the index being
 * the group-edge row's position. Group nodes, their metrics and top: §21 over the group-edge rows, so a group's side IN
 * sums every row into any of its members, and a group node (type 4) is listed after every other node.
 * *n_out is always set; a host call whose cap is below it returns ALZ_E_CAPACITY and writes nothing. An unknown source
 * or side, a bad metric list (§17), k = 0, a NaN min_value or a null required pointer: ALZ_E_INVAL. No rows of a rollup
 * source: ALZ_E_STATE. More than 2^29 - 1 source rows: ALZ_E_CAPACITY, before anything runs; no memory: ALZ_E_NOMEM. A
 * 0-row source: 0 rows, ALZ_OK. info (may be NULL): the source's rows, the row ends the map held, the group-edge rows,
 * and the source rows whose two ends are one node after the mapping. Reads only: the window, every ring, the open
 * blocks, every rollup's rows, the baseline and every other family's results, device pointers included, are unchanged.
 * Device results stay valid until the next group call on the handle. Every rank holds the same rows and the same map,
 * so every rank gets the same result. */
typedef struct alz_group_info {
  uint64_t source_rows;   /* rows of the source */
  uint64_t mapped_ends;   /* row ends (two per row) the map held */
  uint64_t edges;         /* group-edge rows */
  uint64_t internal;      /* source rows whose from and to are one node after the mapping */
} alz_group_info;
int alz_group_set(alz_handle* h, const alz_node_ends* nodes, const uint32_t* groups, size_t n);
/* every group-edge row of a source, in (from key, to key) order; cap counts rows */
int alz_group_edges(alz_handle* h, uint32_t source, alz_edge_out* out, size_t cap, size_t* n_out, alz_group_info* info);
int alz_group_edges_device(alz_handle* h, uint32_t source, const alz_edge_out** dev_out, size_t* n_out,
                           alz_group_info* info);
/* values[i * nm + j]: metric j of group-edge row i; cap counts rows */
int alz_group_edge_metrics(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t nm, double* values, size_t cap,
                           size_t* n_out);
int alz_group_edge_metrics_device(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t nm,
                                  const double** dev_values, size_t* n_out);
/* the first min(k, above) group-edge rows by one metric, ranked as alz_edge_top; rows, values, index and info may each
 * be NULL. info->scored = the group-edge rows. */
int alz_group_edge_top(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t k, double min_value,
                       alz_edge_out* rows, double* values, uint32_t* index, size_t cap, size_t* n_out,
                       alz_top_info* info);
int alz_group_edge_top_device(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t k, double min_value,
                              const alz_edge_out** dev_rows, const double** dev_values, const uint32_t** dev_index,
                              size_t* n_out, alz_top_info* info);
/* the §21 node rows of the group-edge rows, in node order; cap counts nodes */
int alz_group_nodes(alz_handle* h, uint32_t source, alz_node_out* out, size_t cap, size_t* n_out);
int alz_group_nodes_device(alz_handle* h, uint32_t source, const alz_node_out** dev_out, size_t* n_out);
/* values[i * nm + j]: metric j of group node i's side `side` (ALZ_SIDE_*); cap counts nodes */
int alz_group_node_metrics(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t nm,
                           double* values, size_t cap, size_t* n_out);
int alz_group_node_metrics_device(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t nm,
                                  const double** dev_values, size_t* n_out);
/* the first min(k, above) group nodes by one metric of one side, ranked as alz_node_top; nodes, values, index and info
 * may each be NULL (dev_nodes, dev_values and dev_index too). info->scored = the group nodes. */
int alz_group_node_top(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t k,
                       double min_value, alz_node_out* nodes, double* values, uint32_t* index, size_t cap,
                       size_t* n_out, alz_top_info* info);
int alz_group_node_top_device(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t k,
                              double min_value, const alz_node_out** dev_nodes, const double** dev_values,
                              const uint32_t** dev_index, size_t* n_out, alz_top_info* info);

/* ---- group changes against a pinned baseline (docs/SPEC.md §25) -----------------------------------------------------
 * §18 and §23 over groups: a source (ALZ_SOURCE_WINDOW or ALZ_ROLLUP_*, availability rule of §15) against the baseline
 * alz_baseline_pin holds, both sides grouped by the map in force at the call (§24; an empty map is allowed). Each side's
 * group-edge rows are what alz_group_edges gives for a source holding that side's rows, and its group nodes what
 * alz_group_nodes gives. Rows and nodes a rollout replaces (pods) are NEW and GONE; the groups they belong to are
 * BOTH, with a quantile of the summed histograms on each side.
 *
 * Group edge changes: the union of the two group-edge lists, matched by (node key of from, node key of to), in that
 * ascending order (§24), filtered by presence; index / base_index: the row's position in each side's group-edge list.
 * Group node changes: §23 over the two group-node lists, with its side-membership rule; index / base_index: positions
 * in each side's full group-node list, and a group node (type 4) sorts after every other type. value, base_value,
 * change and the top calls' ranking and eligibility: as §18 (COUNT and ERR5XX per window, one rounding each).
 * info->source_rows / base_rows count group-edge rows (edge calls) or member group nodes (node calls). Unknown metric,
 * mode, side or source, presence 0 or above 7, k = 0, a NaN min_change or a null required pointer: ALZ_E_INVAL. No
 * baseline, or no rows of a rollup source: ALZ_E_STATE. A side of more than 2^29 - 1 rows (before anything runs) or a
 * union of more than 2^30 - 1 entries: ALZ_E_CAPACITY; no memory: ALZ_E_NOMEM. *n_out is always set; a host call whose
 * cap (in records) is below it returns ALZ_E_CAPACITY and writes nothing. info may be NULL.
 *
 * Reads only: the window, every ring, the open blocks, every rollup's rows, the baseline and the map are unchanged, and
 * so are every other family's results (groups, edge and node changes, node, metric, top, series, trend, GNN), device
 * pointers included. The baseline's group edges, and its group nodes once a node call needs them, are grouped on the
 * first call that needs them and kept until the next pin or the next alz_group_set that succeeds. Device results stay
 * valid until the next group change call. Every rank holds the same rows, map and baseline, so every rank gets the
 * same result with no collective. */
/* every listed group edge, in ascending (from key, to key) order */
int alz_group_edge_changes(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode, uint32_t presence,
                           alz_edge_change* out, size_t cap, size_t* n_out, alz_change_info* info);
int alz_group_edge_changes_device(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode,
                                  uint32_t presence, const alz_edge_change** dev_out, size_t* n_out,
                                  alz_change_info* info);
/* the first min(k, above) listed group edges by change, in rank order; info->above = the eligible ones */
int alz_group_edge_changes_top(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode, uint32_t presence,
                               uint32_t k, double min_change, alz_edge_change* out, size_t cap, size_t* n_out,
                               alz_change_info* info);
int alz_group_edge_changes_top_device(alz_handle* h, uint32_t source, const alz_metric* m, uint32_t mode,
                                      uint32_t presence, uint32_t k, double min_change,
                                      const alz_edge_change** dev_out, size_t* n_out, alz_change_info* info);
/* every listed group node of side `side` (ALZ_SIDE_*), in ascending node key order */
int alz_group_node_changes(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t mode,
                           uint32_t presence, alz_node_change* out, size_t cap, size_t* n_out, alz_change_info* info);
int alz_group_node_changes_device(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t mode,
                                  uint32_t presence, const alz_node_change** dev_out, size_t* n_out,
                                  alz_change_info* info);
/* the first min(k, above) listed group nodes by change, in rank order; info->above = the eligible ones */
int alz_group_node_changes_top(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m, uint32_t mode,
                               uint32_t presence, uint32_t k, double min_change, alz_node_change* out, size_t cap,
                               size_t* n_out, alz_change_info* info);
int alz_group_node_changes_top_device(alz_handle* h, uint32_t source, uint32_t side, const alz_metric* m,
                                      uint32_t mode, uint32_t presence, uint32_t k, double min_change,
                                      const alz_node_change** dev_out, size_t* n_out, alz_change_info* info);

/* ---- group series and trends (docs/SPEC.md §26) ---------------------------------------------------------------------
 * §19, §20 and §22 over groups: the map in force at the call (§24; an empty map is allowed) groups the source and every
 * entry the call reads. Series rows: the group-edge rows of alz_group_edges(source), or the group nodes of
 * alz_group_nodes(source) (type 4 last), in that order; or the caller's keys in the caller's order, duplicates giving
 * identical rows. Point j of a group edge is present when entry j holds a row that maps onto it, and its values are
 * then bit for bit what alz_group_edge_metrics* gives for a source holding entry j alone; point j of a group node is
 * present when entry j holds a row whose mapped end on the side is the node (§22's rule: a group seen only on the other
 * side is absent), with the values alz_group_node_metrics* gives for such a source. An absent point is +0.0 in every
 * value, present 0. With an empty map, the group node series are alz_node_series* byte for byte, and the group edge
 * series alz_edge_series* up to row order.
 * Keys: a node key is one §22 accepts or (ALZ_NODE_GROUP, g) with g < 2^29; a group-edge key with no group end follows
 * §19's rules, one with a group end needs two valid node keys. A key naming a node the map holds is absent at every
 * point. Malformed keys are ALZ_E_INVAL, checked before any size; §19's and §22's own key rules do not change.
 * Trends (by source only): §20's statistics, directions, absent modes, validity rules and roundings over those series.
 * Records are alz_edge_trend (the head is the group-edge row's ends: from_type / to_type may be 4) and alz_node_trend;
 * index is the position in alz_group_edges(source) / alz_group_nodes(source), and a top result's rows / nodes entry is
 * byte for byte what those calls give at that index.
 * Errors, outputs and waits as §19, §20 and §22, plus ALZ_E_CAPACITY for a source of more than 2^29 - 1 rows, checked
 * before anything runs; *n_out and *n_points are always set; no retained entry gives P = 0, ALZ_OK. Reads only: the
 * window, every ring, the open blocks, every rollup's rows, the baseline, the map, the group changes' baseline groups
 * and every other family's device results are unchanged. Device results stay valid until the next call of the same
 * family (group series, group trends). Each family's buffers grow to its largest call and are kept until alz_destroy:
 * a group edge series holds a 576-byte node row per present slot, several GB for 60 points of 200,000 group edges. Every rank holds the same history and map, so every rank gets the same result
 * with no collective. */
/* every group edge of a source; cap counts series rows */
int alz_group_edge_series(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m, uint32_t nm,
                          double* values, uint8_t* present, size_t cap, size_t* n_out, uint32_t* n_points,
                          alz_rollup_info* points, alz_series_info* info);
int alz_group_edge_series_device(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                                 uint32_t nm, const double** dev_values, const uint8_t** dev_present, size_t* n_out,
                                 uint32_t* n_points, alz_rollup_info* points, alz_series_info* info);
/* the caller's group edges (from_type / to_type may be ALZ_NODE_GROUP), keys in host memory */
int alz_group_edge_series_keys(alz_handle* h, const alz_edge_ends* keys, size_t n_keys, uint32_t tier, uint32_t k,
                               const alz_metric* m, uint32_t nm, double* values, uint8_t* present, size_t cap,
                               size_t* n_out, uint32_t* n_points, alz_rollup_info* points, alz_series_info* info);
int alz_group_edge_series_keys_device(alz_handle* h, const alz_edge_ends* keys, size_t n_keys, uint32_t tier,
                                      uint32_t k, const alz_metric* m, uint32_t nm, const double** dev_values,
                                      const uint8_t** dev_present, size_t* n_out, uint32_t* n_points,
                                      alz_rollup_info* points, alz_series_info* info);
/* every group node of a source, side `side` (ALZ_SIDE_*) */
int alz_group_node_series(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                          const alz_metric* m, uint32_t nm, double* values, uint8_t* present, size_t cap,
                          size_t* n_out, uint32_t* n_points, alz_rollup_info* points, alz_series_info* info);
int alz_group_node_series_device(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                 const alz_metric* m, uint32_t nm, const double** dev_values,
                                 const uint8_t** dev_present, size_t* n_out, uint32_t* n_points,
                                 alz_rollup_info* points, alz_series_info* info);
/* the caller's nodes (type may be ALZ_NODE_GROUP), keys in host memory */
int alz_group_node_series_keys(alz_handle* h, const alz_node_ends* keys, size_t n_keys, uint32_t side, uint32_t tier,
                               uint32_t k, const alz_metric* m, uint32_t nm, double* values, uint8_t* present,
                               size_t cap, size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                               alz_series_info* info);
int alz_group_node_series_keys_device(alz_handle* h, const alz_node_ends* keys, size_t n_keys, uint32_t side,
                                      uint32_t tier, uint32_t k, const alz_metric* m, uint32_t nm,
                                      const double** dev_values, const uint8_t** dev_present, size_t* n_out,
                                      uint32_t* n_points, alz_rollup_info* points, alz_series_info* info);
/* one record per group edge / group node of the source; the top calls as alz_edge_trends_top / alz_node_trends_top */
int alz_group_edge_trends(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                          const alz_trend* t, alz_edge_trend* out, size_t cap, size_t* n_out, uint32_t* n_points,
                          alz_rollup_info* points, alz_trend_info* info);
int alz_group_edge_trends_device(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                                 const alz_trend* t, const alz_edge_trend** dev_out, size_t* n_out,
                                 uint32_t* n_points, alz_rollup_info* points, alz_trend_info* info);
int alz_group_edge_trends_top(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                              const alz_trend* t, uint32_t top, double min_trend, alz_edge_trend* out,
                              alz_edge_out* rows, double* series, uint8_t* present, size_t cap, size_t* n_out,
                              uint32_t* n_points, alz_rollup_info* points, alz_trend_info* info);
int alz_group_edge_trends_top_device(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                                     const alz_trend* t, uint32_t top, double min_trend,
                                     const alz_edge_trend** dev_out, const alz_edge_out** dev_rows,
                                     const double** dev_series, const uint8_t** dev_present, size_t* n_out,
                                     uint32_t* n_points, alz_rollup_info* points, alz_trend_info* info);
int alz_group_node_trends(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                          const alz_metric* m, const alz_trend* t, alz_node_trend* out, size_t cap, size_t* n_out,
                          uint32_t* n_points, alz_rollup_info* points, alz_trend_info* info);
int alz_group_node_trends_device(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                 const alz_metric* m, const alz_trend* t, const alz_node_trend** dev_out,
                                 size_t* n_out, uint32_t* n_points, alz_rollup_info* points, alz_trend_info* info);
int alz_group_node_trends_top(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                              const alz_metric* m, const alz_trend* t, uint32_t top, double min_trend,
                              alz_node_trend* out, alz_node_out* nodes, double* series, uint8_t* present, size_t cap,
                              size_t* n_out, uint32_t* n_points, alz_rollup_info* points, alz_trend_info* info);
int alz_group_node_trends_top_device(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                     const alz_metric* m, const alz_trend* t, uint32_t top, double min_trend,
                                     const alz_node_trend** dev_out, const alz_node_out** dev_nodes,
                                     const double** dev_series, const uint8_t** dev_present, size_t* n_out,
                                     uint32_t* n_points, alz_rollup_info* points, alz_trend_info* info);

/* ---- reach (docs/SPEC.md §27) ---------------------------------------------------------------------------------------
 * A breadth-first search of a source's graph (ALZ_SOURCE_WINDOW or ALZ_ROLLUP_*, with the availability rule of §15)
 * from chosen seed nodes, up to max_hops (1 .. ALZ_REACH_MAX_HOPS) rows away. alz_reach* traverses the source's rows
 * and its nodes are alz_node_rows(source); alz_group_reach* traverses the source's group-edge rows under the map in
 * force at the call (§24; an empty map is allowed) and its nodes are alz_group_nodes(source). A node's index is its
 * position in that node list. ALZ_REACH_DOWN: a row leads from its from end to its to end (dependencies); ALZ_REACH_UP:
 * from its to end to its from end (callers); ALZ_REACH_ANY: both ways. With m NULL every row is traversable and
 * min_value is ignored; otherwise m is one §17 metric and a row is traversable when the IEEE total-order key of its
 * value (bit for bit alz_edge_metrics* / alz_group_edge_metrics*) is at least key(min_value): ERR5XX >= 1 follows failing
 * calls only. hops(v) is the fewest traversable rows on a path from a seed to v. A seed that is no node of the traversed
 * rows is skipped (info->seeds_found counts the distinct ones that are); duplicates are allowed.
 * Nodes: every node with hops <= max_hops, ordered by (hops, node key (type << 32) | value). A record's parent is the
 * position in this result of the node with the smallest index among the listed nodes at hops - 1 that have a
 * traversable row leading to it, and its row the smallest position among the traversable rows leading from that parent
 * to it (under ANY, either orientation counts); seeds have parent = row = 0xFFFFFFFF. The bytes do not depend on thread
 * order, and parent and row rebuild one shortest path with the row of every hop.
 * Rows: every traversable row whose tail (from for DOWN, to for UP, either end for ANY) has hops < max_hops, in
 * traversed-list order: row_index[j] its position there, rows[j] the row byte for byte (a source row, or a group-edge
 * row for the group form). Their heads are listed nodes.
 * Seeds: the node form takes §22's keys (a type above ALZ_NODE_OUTBOUND_HOST or a pod or service value >= 2^29 is
 * malformed), the group form §26's (also (ALZ_NODE_GROUP, g) with g < 2^29); malformed seeds are checked before any
 * size. An unknown source or dir, max_hops 0 or above 64, n_seeds 0, a null seeds, n_nodes or n_rows, a bad metric
 * (§17) or a NaN min_value with a metric: ALZ_E_INVAL. No rows of a rollup source: ALZ_E_STATE. More than 2^29 - 1
 * source rows (before anything runs) or more than 2^30 - 1 seeds: ALZ_E_CAPACITY; no memory: ALZ_E_NOMEM. No seed
 * found, or a 0-row source: 0 nodes, 0 rows, ALZ_OK. *n_nodes and *n_rows are always set. Host forms: nodes, row_index
 * and rows may each be NULL; node_cap is checked when nodes is not NULL and row_cap when row_index or rows is not; a
 * failed check returns ALZ_E_CAPACITY and writes none of the three. Device forms: dev_nodes, dev_row_index and dev_rows
 * may each be NULL; the results stay valid until the next reach call of either form. info may be NULL.
 * Waits: one for the node count (§21), one for the seeds found, one per level expanded (min(levels + 1, max_hops) of
 * them), one for the listed rows, and a host call one more for its copies; the group form adds §24's two. Reads only:
 * the window, every ring, the open blocks, every rollup's rows and info, the baseline and its caches, the map and every
 * other family's device results are unchanged; reach keeps its buffers in a state of its own, grown on demand and freed
 * in alz_destroy. Every rank holds the same rows and the same map, so every rank returns the same bytes with no
 * collective. */
#define ALZ_REACH_DOWN 0u   /* from end -> to end: what the seeds call */
#define ALZ_REACH_UP   1u   /* to end -> from end: who calls the seeds */
#define ALZ_REACH_ANY  2u   /* both ways */
#define ALZ_REACH_MAX_HOPS 64u
typedef struct alz_reach_node {   /* 24 B; the first 8 bytes are an alz_node_ends */
  uint8_t type;                   /* ALZ_NODE_* */
  uint8_t _pad[3];                /* zero */
  uint32_t value;
  uint32_t hops;
  uint32_t index;                 /* the node's position in the traversed rows' node list */
  uint32_t parent;                /* the predecessor's position in this result; 0xFFFFFFFF for a seed */
  uint32_t row;                   /* the traversed row used from the parent; 0xFFFFFFFF for a seed */
} alz_reach_node;
typedef struct alz_reach_info {
  uint64_t rows;          /* traversed rows */
  uint64_t traversable;   /* of which traversable */
  uint64_t seeds_found;   /* distinct seeds that are nodes */
  uint64_t nodes;         /* nodes listed */
  uint64_t levels;        /* the largest hops listed */
  uint64_t cut;           /* traversable rows from a node at hops = max_hops to a node not listed; 0: a larger
                             max_hops lists no more nodes */
} alz_reach_info;
int alz_reach(alz_handle* h, uint32_t source, const alz_node_ends* seeds, size_t n_seeds, uint32_t dir,
              uint32_t max_hops, const alz_metric* m, double min_value, alz_reach_node* nodes, size_t node_cap,
              size_t* n_nodes, uint32_t* row_index, alz_edge_out* rows, size_t row_cap, size_t* n_rows,
              alz_reach_info* info);
int alz_reach_device(alz_handle* h, uint32_t source, const alz_node_ends* seeds, size_t n_seeds, uint32_t dir,
                     uint32_t max_hops, const alz_metric* m, double min_value, const alz_reach_node** dev_nodes,
                     size_t* n_nodes, const uint32_t** dev_row_index, const alz_edge_out** dev_rows, size_t* n_rows,
                     alz_reach_info* info);
int alz_group_reach(alz_handle* h, uint32_t source, const alz_node_ends* seeds, size_t n_seeds, uint32_t dir,
                    uint32_t max_hops, const alz_metric* m, double min_value, alz_reach_node* nodes, size_t node_cap,
                    size_t* n_nodes, uint32_t* row_index, alz_edge_out* rows, size_t row_cap, size_t* n_rows,
                    alz_reach_info* info);
int alz_group_reach_device(alz_handle* h, uint32_t source, const alz_node_ends* seeds, size_t n_seeds, uint32_t dir,
                           uint32_t max_hops, const alz_metric* m, double min_value, const alz_reach_node** dev_nodes,
                           size_t* n_nodes, const uint32_t** dev_row_index, const alz_edge_out** dev_rows,
                           size_t* n_rows, alz_reach_info* info);

/* ---- cycles (docs/SPEC.md §28) --------------------------------------------------------------------------------------
 * The strongly connected components of a source's graph (ALZ_SOURCE_WINDOW or ALZ_ROLLUP_*, with the availability
 * rule of §15), with each component's depth and height. alz_cycles* traverses the source's rows and its nodes are
 * alz_node_rows(source); alz_group_cycles* traverses the source's group-edge rows under the map in force at the call
 * (§24; an empty map is allowed) and its nodes are alz_group_nodes(source). A node's index is its position in that node
 * list. With m NULL every row is traversable and min_value is ignored; otherwise m is one §17 metric and a row is
 * traversable when the IEEE total-order key of its value is at least key(min_value), as in §27.
 * A self row is a traversable row whose from end and to end are one node (in the group form every internal row g -> g):
 * it never makes a component cyclic, is never listed and is counted in info->self_rows.
 * Components: two nodes are in one component when each reaches the other along traversable rows (from end -> to end).
 * Every node is in exactly one, nodes without a traversable row included. Components are numbered from 0 in ascending
 * order of their smallest node index; one of 2 or more nodes is cyclic. A traversable row between two components is a
 * row of the condensation: depth(C) is the most condensation rows on a path that ends at C (0 without one into C),
 * height(C) the most on a path that starts at C. Every node carries its component's number, size, depth and height.
 * Nodes: the nodes of every component of at least min_size nodes (0 or 1: all; 2: the nodes on cycles), ordered by
 * (component, index). Rows: every traversable row that is not a self row and whose two ends lie in one listed cyclic
 * component, ordered by (component, row position): row_index[j] its position in the traversed list, rows[j] the row byte
 * for byte (a source row, or a group-edge row for the group form). The components are unique, so every byte of the
 * result follows from the rows whatever the order of the work.
 * An unknown source, a null n_nodes or n_rows, a bad metric (§17) or a NaN min_value with a metric: ALZ_E_INVAL. No rows
 * of a rollup source: ALZ_E_STATE. More than 2^29 - 1 source rows (before anything runs): ALZ_E_CAPACITY; no memory:
 * ALZ_E_NOMEM. A 0-row source: 0 nodes, 0 rows, ALZ_OK. *n_nodes and *n_rows are always set. Host forms: nodes,
 * row_index and rows may each be NULL; node_cap is checked when nodes is not NULL and row_cap when row_index or rows is
 * not; a failed check returns ALZ_E_CAPACITY and writes none of the three. Device forms: dev_nodes, dev_row_index and
 * dev_rows may each be NULL; the results stay valid until the next cycles call of either form. info may be NULL.
 * Waits: one for the node count (§21), one for the totals that size the results, and a host call one more for its
 * copies; the group form adds §24's two. The fixed-point phases run in cooperative launches with grid-wide barriers, so
 * the waits do not grow with their rounds. The rounds are data-dependent: about one per node on a chain or a ring, and
 * O(N^2) for N nodes in the worst case (each colouring iteration may take about N rounds and settle one component;
 * iterations alternate direction, which settles a chain of loops in two, but layouts that defeat both may exist). Reads only: the window, every ring, the open blocks, every rollup's rows and info, the
 * baseline and its caches, the map and every other family's device results are unchanged; cycles keeps its buffers in
 * a state of its own, grown on demand and freed in alz_destroy. Every rank holds the same rows and the same map, so
 * every rank returns the same bytes with no collective. */
typedef struct alz_cycle_node {   /* 28 B; the first 8 bytes are an alz_node_ends */
  uint8_t type;                   /* ALZ_NODE_* */
  uint8_t _pad[3];                /* zero */
  uint32_t value;
  uint32_t index;                 /* the node's position in the traversed rows' node list */
  uint32_t component;             /* its component's number */
  uint32_t size;                  /* the component's node count */
  uint32_t depth;                 /* the component's depth in the condensation */
  uint32_t height;                /* the component's height in the condensation */
} alz_cycle_node;
typedef struct alz_cycle_info {
  uint64_t rows;           /* traversed rows */
  uint64_t traversable;    /* of which traversable */
  uint64_t self_rows;      /* of which self rows */
  uint64_t nodes;          /* nodes of the traversed rows */
  uint64_t components;     /* components */
  uint64_t cyclic;         /* components of 2 or more nodes */
  uint64_t cyclic_nodes;   /* their nodes */
  uint64_t largest;        /* the node count of the largest component */
  uint64_t cycle_rows;     /* traversable rows that are not self rows inside cyclic components, whatever min_size */
  uint64_t depth;          /* the largest depth (= the largest height) */
} alz_cycle_info;
int alz_cycles(alz_handle* h, uint32_t source, const alz_metric* m, double min_value, uint32_t min_size,
               alz_cycle_node* nodes, size_t node_cap, size_t* n_nodes, uint32_t* row_index, alz_edge_out* rows,
               size_t row_cap, size_t* n_rows, alz_cycle_info* info);
int alz_cycles_device(alz_handle* h, uint32_t source, const alz_metric* m, double min_value, uint32_t min_size,
                      const alz_cycle_node** dev_nodes, size_t* n_nodes, const uint32_t** dev_row_index,
                      const alz_edge_out** dev_rows, size_t* n_rows, alz_cycle_info* info);
int alz_group_cycles(alz_handle* h, uint32_t source, const alz_metric* m, double min_value, uint32_t min_size,
                     alz_cycle_node* nodes, size_t node_cap, size_t* n_nodes, uint32_t* row_index, alz_edge_out* rows,
                     size_t row_cap, size_t* n_rows, alz_cycle_info* info);
int alz_group_cycles_device(alz_handle* h, uint32_t source, const alz_metric* m, double min_value, uint32_t min_size,
                            const alz_cycle_node** dev_nodes, size_t* n_nodes, const uint32_t** dev_row_index,
                            const alz_edge_out** dev_rows, size_t* n_rows, alz_cycle_info* info);

/* ---- correlations (docs/SPEC.md §29) -------------------------------------------------------------------------------
 * How closely each row's series of one metric followed a target series the caller supplies, at the best lag. The
 * candidates are the series rows of §20 (alz_edge_correlations*: a source's rows), §22 (alz_node_correlations*: its
 * nodes on one side) or §26 (alz_group_edge_correlations* / alz_group_node_correlations*: its group edges or group
 * nodes under the map in force at the call) over the last P = min(k, retained) closed entries of one ring, oldest
 * first. The target is aligned to the same ring and k: n = P points, and window_last the alz_rollup_info.window_last
 * of its newest point (a one-key alz_*_series_keys call at the same tier and k gives both). n != P, or P > 0 and a
 * window_last that is not the ring's newest entry's: ALZ_E_STATE (a flush came between). A present target value must be
 * finite with |v| <= 2^64; an absent one is read as +0.0 whatever it holds.
 * At lag L (0 .. max_lag) the candidate leads the target by L points: the pairs are (x[j - L], y[j]) for j in [L, P).
 * ALZ_CORR_ABSENT_SKIP uses the pairs where both points are present, ALZ_CORR_ABSENT_ZERO every pair with an absent
 * point as +0.0. With `used` the pairs used, the means, then Sxx, Syy and Sxy about them (sums from +0.0 in ascending
 * j, each operation one float64 rounding), r = Sxy / (sqrt(Sxx) * sqrt(Syy)) clamped to [-1, 1]. A lag is defined when
 * used >= min_points and the denominator is > 0; its score is r, 0.0 - r or |r| by direction. A row is valid when some
 * lag is defined; its best lag is the defined lag with the largest score, the smallest on ties. An invalid row's record
 * is all +0.0 but its head and `used`, which then counts the pairs of lag 0.
 * The full-list calls give one record per candidate in source order; the top calls rank the valid rows as §20 does
 * (64-bit key of the float64 score, descending, then row ascending; eligible when key(score) >= key(min_score)) and
 * return the first min(top, above) with their source rows or node rows and their series (series[j * P + p],
 * present[j * P + p]; room for cap x k each). k = 0, max_lag above ALZ_CORR_MAX_LAG or not below k, min_points below 3,
 * an unknown direction or absent mode, a null target, a null target->values with n > 0, a bad target value, and
 * everything the matching trend call refuses with ALZ_E_INVAL: ALZ_E_INVAL. The other errors, the waits, the
 * availability rule, "reads only" (every other family's device results, trends and series included, are unchanged)
 * and "every rank returns the same bytes with no collective" are §20's. Device results stay valid until the next
 * correlation call of the same level. */
#define ALZ_CORR_POSITIVE 0u   /* score r: the rows that rose and fell with the target rank first */
#define ALZ_CORR_NEGATIVE 1u   /* score -r: the rows that moved against it */
#define ALZ_CORR_ABS      2u   /* score |r|: either */
#define ALZ_CORR_ABSENT_SKIP 0u   /* a pair with an absent point is left out */
#define ALZ_CORR_ABSENT_ZERO 1u   /* an absent point counts as +0.0 */
#define ALZ_CORR_MAX_LAG 32u
typedef struct alz_corr {   /* 16 B */
  uint32_t direction;    /* ALZ_CORR_POSITIVE / NEGATIVE / ABS */
  uint32_t absent;       /* ALZ_CORR_ABSENT_SKIP / ABSENT_ZERO */
  uint32_t max_lag;      /* lags 0 .. max_lag; max_lag <= ALZ_CORR_MAX_LAG and max_lag < k */
  uint32_t min_points;   /* a defined lag uses at least this many pairs; >= 3 */
} alz_corr;
typedef struct alz_corr_target {   /* 32 B */
  const double* values;    /* host memory, n values */
  const uint8_t* present;  /* host memory, n bytes (nonzero: present), or NULL: every point present */
  size_t n;                /* P */
  uint64_t window_last;    /* alz_rollup_info.window_last of the newest point */
} alz_corr_target;
typedef struct alz_edge_corr {   /* 48 B; the head is laid out as alz_edge_trend's */
  uint8_t from_type;     /* ALZ_NODE_* */
  uint8_t to_type;
  uint8_t valid;         /* 1: some lag is defined */
  uint8_t lag;           /* the best lag */
  uint8_t _pad[4];
  uint32_t from;
  uint32_t to;
  uint32_t index;        /* row index in the source */
  uint32_t used;         /* pairs used at the best lag (invalid: at lag 0) */
  double r;              /* r at the best lag */
  double score;          /* its score */
  double r0;             /* r at lag 0, +0.0 when lag 0 is undefined */
} alz_edge_corr;
typedef struct alz_node_corr {   /* 48 B; from `valid` on, laid out as alz_edge_corr */
  uint8_t type;          /* ALZ_NODE_* */
  uint8_t _pad0;
  uint8_t valid;
  uint8_t lag;
  uint8_t _pad1[4];
  uint32_t value;
  uint32_t _pad2;
  uint32_t index;        /* node index in the source (§21 node order) */
  uint32_t used;
  double r;
  double score;
  double r0;
} alz_node_corr;
typedef struct alz_corr_info {
  uint64_t rows;          /* candidates: the source's rows, nodes, group edges or group nodes */
  uint64_t rows_in;       /* entry rows read: the sum of the P entries' rows */
  uint64_t valid;         /* valid candidates */
  uint64_t above;         /* top calls: eligible candidates before the cut; 0 otherwise */
  uint32_t points;        /* P */
  uint32_t tier;
  uint32_t target_used;   /* the target's present points */
  uint32_t _pad;
} alz_corr_info;
int alz_edge_correlations(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                          const alz_corr* corr, const alz_corr_target* target, alz_edge_corr* out, size_t cap,
                          size_t* n_out, uint32_t* n_points, alz_rollup_info* points, alz_corr_info* info);
int alz_edge_correlations_device(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                                 const alz_corr* corr, const alz_corr_target* target, const alz_edge_corr** dev_out,
                                 size_t* n_out, uint32_t* n_points, alz_rollup_info* points, alz_corr_info* info);
int alz_edge_correlations_top(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                              const alz_corr* corr, const alz_corr_target* target, uint32_t top, double min_score,
                              alz_edge_corr* out, alz_edge_out* rows, double* series, uint8_t* present, size_t cap,
                              size_t* n_out, uint32_t* n_points, alz_rollup_info* points, alz_corr_info* info);
int alz_edge_correlations_top_device(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                                     const alz_corr* corr, const alz_corr_target* target, uint32_t top,
                                     double min_score, const alz_edge_corr** dev_out, const alz_edge_out** dev_rows,
                                     const double** dev_series, const uint8_t** dev_present, size_t* n_out,
                                     uint32_t* n_points, alz_rollup_info* points, alz_corr_info* info);
int alz_node_correlations(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                          const alz_metric* m, const alz_corr* corr, const alz_corr_target* target,
                          alz_node_corr* out, size_t cap, size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                          alz_corr_info* info);
int alz_node_correlations_device(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                 const alz_metric* m, const alz_corr* corr, const alz_corr_target* target,
                                 const alz_node_corr** dev_out, size_t* n_out, uint32_t* n_points,
                                 alz_rollup_info* points, alz_corr_info* info);
int alz_node_correlations_top(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                              const alz_metric* m, const alz_corr* corr, const alz_corr_target* target, uint32_t top,
                              double min_score, alz_node_corr* out, alz_node_out* nodes, double* series,
                              uint8_t* present, size_t cap, size_t* n_out, uint32_t* n_points,
                              alz_rollup_info* points, alz_corr_info* info);
int alz_node_correlations_top_device(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                     const alz_metric* m, const alz_corr* corr, const alz_corr_target* target,
                                     uint32_t top, double min_score, const alz_node_corr** dev_out,
                                     const alz_node_out** dev_nodes, const double** dev_series,
                                     const uint8_t** dev_present, size_t* n_out, uint32_t* n_points,
                                     alz_rollup_info* points, alz_corr_info* info);
int alz_group_edge_correlations(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                                const alz_corr* corr, const alz_corr_target* target, alz_edge_corr* out, size_t cap,
                                size_t* n_out, uint32_t* n_points, alz_rollup_info* points, alz_corr_info* info);
int alz_group_edge_correlations_device(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                                       const alz_corr* corr, const alz_corr_target* target,
                                       const alz_edge_corr** dev_out, size_t* n_out, uint32_t* n_points,
                                       alz_rollup_info* points, alz_corr_info* info);
int alz_group_edge_correlations_top(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                                    const alz_corr* corr, const alz_corr_target* target, uint32_t top,
                                    double min_score, alz_edge_corr* out, alz_edge_out* rows, double* series,
                                    uint8_t* present, size_t cap, size_t* n_out, uint32_t* n_points,
                                    alz_rollup_info* points, alz_corr_info* info);
int alz_group_edge_correlations_top_device(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k,
                                           const alz_metric* m, const alz_corr* corr, const alz_corr_target* target,
                                           uint32_t top, double min_score, const alz_edge_corr** dev_out,
                                           const alz_edge_out** dev_rows, const double** dev_series,
                                           const uint8_t** dev_present, size_t* n_out, uint32_t* n_points,
                                           alz_rollup_info* points, alz_corr_info* info);
int alz_group_node_correlations(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                const alz_metric* m, const alz_corr* corr, const alz_corr_target* target,
                                alz_node_corr* out, size_t cap, size_t* n_out, uint32_t* n_points,
                                alz_rollup_info* points, alz_corr_info* info);
int alz_group_node_correlations_device(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                       const alz_metric* m, const alz_corr* corr, const alz_corr_target* target,
                                       const alz_node_corr** dev_out, size_t* n_out, uint32_t* n_points,
                                       alz_rollup_info* points, alz_corr_info* info);
int alz_group_node_correlations_top(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                    const alz_metric* m, const alz_corr* corr, const alz_corr_target* target,
                                    uint32_t top, double min_score, alz_node_corr* out, alz_node_out* nodes,
                                    double* series, uint8_t* present, size_t cap, size_t* n_out, uint32_t* n_points,
                                    alz_rollup_info* points, alz_corr_info* info);
int alz_group_node_correlations_top_device(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                           const alz_metric* m, const alz_corr* corr, const alz_corr_target* target,
                                           uint32_t top, double min_score, const alz_node_corr** dev_out,
                                           const alz_node_out** dev_nodes, const double** dev_series,
                                           const uint8_t** dev_present, size_t* n_out, uint32_t* n_points,
                                           alz_rollup_info* points, alz_corr_info* info);

/* ---- tcp_state sink + temporal socket join (SURVEY §8f.2) -------------------
 * alz_submit_tcp replaces processTcpConnect (aggregator/data.go:404-506) +
 * SocketLine.AddValue (sock_num_line.go:62-80); alz_sock_lookup replaces
 * SocketLine.GetValue (sock_num_line.go:82-158). */
int alz_submit_tcp(alz_handle* h, const alz_tcp_rec* host_recs, size_t n);
/* n raw perf samples of the tcp_connect_events ring exactly as perf.Reader yields
 * them: struct tcp_event (ebpf/c/struct.h:2-12; BpfTcpEvent, ebpf/tcp_state/
 * tcp.go:63-72), 64 bytes with its tail padding. The IPv4 sits in the first four
 * address bytes, first octet first (tcp.go:241-242). */
#define ALZ_BPF_TCP_EVENT_SIZE 64
int alz_submit_tcp_raw(alz_handle* h, const void* host_bpf_tcp_events, size_t n);
int alz_sock_lookup(alz_handle* h, const alz_sock_query* host_q, size_t n,
                    alz_sock_result* host_out);
/* the same with the caller's clock for the LastMatch stamps (the reference uses
 * time.Now(), sock_num_line.go:96, :156); alz_sock_lookup passes CLOCK_REALTIME */
int alz_sock_lookup_at(alz_handle* h, const alz_sock_query* host_q, size_t n,
                       alz_sock_result* host_out, uint64_t now_ns);
/* L7 events that may carry an empty 5-tuple (get_sock miss, ebpf/c/l7.c:313-314):
 * host_keys[i] = (Pid, Fd, WriteTimeNs) of host_recs[i]. Records with saddr == 0
 * and daddr == 0 take their addresses from the (pid, fd) timeline on the device
 * (findRelatedSocket, aggregator/data.go:1407-1429), then the whole batch is
 * ingested like alz_submit_l7. A miss leaves the zeros and the event is dropped
 * and counted as src_unresolved (0.0.0.0 is no pod, data.go:829-832).
 * now_ns: LastMatch stamp, 0 = CLOCK_REALTIME. */
int alz_submit_l7_join(alz_handle* h, const alz_l7_rec* host_recs,
                       const alz_sock_query* host_keys, size_t n, uint64_t now_ns);
/* One tick of clearSocketLines (aggregator/data.go:1681-1716): SocketLine.
 * DeleteUnused (sock_num_line.go:160-209) on every line. */
int alz_sock_gc(alz_handle* h);
/* sendOpenConnection (aggregator/data.go:1628-1679) for every line: one row per
 * line whose last value is an open socket with a pod at its source address.
 * Rows come in no particular order. *n_out = rows there are; ALZ_E_CAPACITY
 * (first `cap` rows written) when cap was too small. Resolves against the
 * tables as of the last alz_table_commit. */
typedef struct alz_alive_conn {
  uint32_t from_ip;
  uint32_t from_id;   /* pod id */
  uint32_t to_ip;
  uint32_t to_id;     /* pod / service id; the raw address for ALZ_NODE_OUTBOUND */
  uint16_t from_port;
  uint16_t to_port;
  uint8_t to_type;    /* ALZ_NODE_* */
  uint8_t _pad[3];
} alz_alive_conn;
int alz_sock_alive(alz_handle* h, alz_alive_conn* host_out, size_t cap, size_t* n_out);
typedef struct alz_sock_stats_t {
  uint64_t lines;          /* (pid, fd) timelines */
  uint64_t pool_records;   /* device pool: records allocated to segments */
  uint64_t pool_garbage;   /* ... of which in segments left behind by grown lines */
  uint64_t syncs;          /* host -> device syncs so far */
  uint64_t sync_ops;       /* inserts they carried */
  uint64_t sync_bytes;     /* bytes they copied */
  uint64_t repools;        /* times the pool was re-laid (full or half garbage) */
  uint64_t joined_events;  /* alz_submit_l7_join: empty 5-tuples filled */
} alz_sock_stats_t;
int alz_sock_stats(alz_handle* h, alz_sock_stats_t* st);

/* ---- multi-GPU: one rank per GPU, events pre-partitioned by alz_owner_rank ---- */
#define ALZ_COMM_ID_BYTES 128
int alz_comm_unique_id(void* out_id /* ALZ_COMM_ID_BYTES */);
/* nranks 1..64 (more: ALZ_E_UNSUPPORTED, before any NCCL call); a second init on a handle: ALZ_E_STATE.
 * Time-cut windows on several ranks need the same alz_window_clock on every rank (see there). */
int alz_comm_init(alz_handle* h, int nranks, int rank, const void* id);
/* rank that owns an event: hash of the source address only, so every event of
 * an edge lands on one rank before any resolve (From is the pod at saddr,
 * aggregator/data.go:834-835) */
uint32_t alz_owner_rank(uint32_t saddr, uint32_t nranks);

#ifdef __cplusplus
}
#endif
#endif /* ALAZGPU_H */
