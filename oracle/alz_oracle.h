/*
 * alz_oracle.h — CPU restatement of the reference aggregator's resolve/emit
 * path plus the group-by-edge the new build defines. TEST INFRASTRUCTURE ONLY:
 * nothing under alaz_b200/ may include, link or call this. Allowed users:
 * tests/, __graft_entry__.smoke(), bench.py's cpu_baseline / --impl reference.
 *
 * PARITY STATUS
 *   resolve / emit / reversal / per-edge grouping: PARITY UNPINNED. The
 *     reference (Go) cannot be built here (no Go toolchain, SURVEY.md §8c) and
 *     none of its tests assert this path; the pins are hand-derived vectors
 *     (tests/golden/resolve_branches.json), one per branch of setFromToV2.
 *   temporal socket join (SocketLine): pinned by the reference's own KATs
 *     (aggregator/sock_line_test.go:11-349, :443-473, :475-501).
 */
#ifndef ALZ_ORACLE_H
#define ALZ_ORACLE_H

#include <stddef.h>
#include <stdint.h>
#include "../include/alazgpu.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct orc orc;

orc* orc_create(void);
void orc_destroy(orc* o);

/* ClusterInfo writers, aggregator/persist.go:55-71 / :114-130. uid strings are
 * "pod-<id>" / "svc-<id>" (the interner is 1:1, so ids stand in for UIDs). */
void orc_table_upsert(orc* o, int table, uint32_t ipv4, uint32_t id);
void orc_table_erase(orc* o, int table, uint32_t ipv4);

/* processL7 -> handlers -> setFromToV2 -> PersistRequest -> group by edge.
 * nthreads <= 1: single thread. Otherwise events are split across threads
 * (like the reference's 4*NumCPU workers, data.go:230-232) with thread-local
 * groups merged at the end. */
void orc_process_l7(orc* o, const alz_l7_rec* recs, size_t n, int nthreads);

/* Same with the HTTP Host header of each event (SURVEY §8 f.4): host_idx[i] = 0 for "no Host header",
 * else 1 + index into names[]. An outbound destination is then keyed by the header instead of the raw
 * daddr (setFromToV2, aggregator/data.go:851-854). Edges to such a node come out with
 * to_type = ALZ_NODE_OUTBOUND_HOST and to = the index into names[] — unless the header text is itself a
 * dotted quad, which the reference cannot tell from a raw-daddr key (same ToUID string): those come out
 * as ALZ_NODE_OUTBOUND with that address. */
void orc_process_l7_hosts(orc* o, const alz_l7_rec* recs, size_t n, const uint32_t* host_idx,
                          const char* const* names, size_t n_names);
/* parseHttpPayload's hostHeader (aggregator/data.go:508-531) on a payload of n bytes; writes a
 * NUL-terminated string into out (cap bytes), "" when the reference finds none. Returns its length. */
size_t orc_parse_http_host(const char* payload, size_t n, char* out, size_t cap);
/* convertKernelTimeToUserspaceTime (aggregator/data.go:1740-1743) followed by the window key of
 * docs/SPEC.md §8: epoch = userspace_ns / window_ns */
uint64_t orc_epoch(uint64_t first_kernel_ns, uint64_t first_user_ns, uint64_t window_ns, uint64_t write_time_ns);

/* live edges sorted by (from_type,from,to_type,to); returns count (<= cap
 * written). */
size_t orc_edges(orc* o, alz_edge_out* out, size_t cap);
void orc_window_reset(orc* o);
void orc_stats(orc* o, alz_stats* st);

/* docs/SPEC.md §4: latency histogram bucket, restated with a loop */
uint32_t orc_bucket(uint64_t duration_ns);
/* docs/SPEC.md §5: quantile from histogram, float64 */
double orc_quantile(const uint32_t* hist, double q);

/* raw 1096-B struct l7_event -> compact record (ebpf/l7_req/l7.go:345-369) */
void orc_compact_raw(const void* raw, size_t n, alz_l7_rec* out);

/* ---- SocketLine restatement (aggregator/sock_num_line.go) ----------------- */
typedef struct orc_sockline orc_sockline;
typedef struct orc_sockinfo {
  uint32_t saddr, daddr;
  uint16_t sport, dport;
} orc_sockinfo;
orc_sockline* orc_sockline_create(void);
void orc_sockline_destroy(orc_sockline* l);
/* AddValue (:62-80); si == NULL records a close */
void orc_sockline_add(orc_sockline* l, uint64_t ts, const orc_sockinfo* si);
/* GetValue (:82-158); returns 1 and fills *out, or 0 where the reference errors */
int orc_sockline_get(orc_sockline* l, uint64_t ts, orc_sockinfo* out);
size_t orc_sockline_len(orc_sockline* l);
int orc_sockline_get_at(orc_sockline* l, uint64_t ts, uint64_t now, orc_sockinfo* out);
void orc_sockline_delete_unused(orc_sockline* l);

/* processTcpConnect (aggregator/data.go:404-506) over many (pid,fd) lines,
 * then findRelatedSocket-style lookups (data.go:1407-1429). */
typedef struct orc_sockmaps orc_sockmaps;
orc_sockmaps* orc_sockmaps_create(void);
void orc_sockmaps_destroy(orc_sockmaps* m);
void orc_sockmaps_process_tcp(orc_sockmaps* m, const alz_tcp_rec* recs, size_t n,
                              uint64_t* localhost_dropped);
void orc_sockmaps_lookup(orc_sockmaps* m, const alz_sock_query* q, size_t n,
                         alz_sock_result* out);
void orc_sockmaps_lookup_at(orc_sockmaps* m, const alz_sock_query* q, size_t n, uint64_t now, alz_sock_result* out);
void orc_sockmaps_gc(orc_sockmaps* m);
size_t orc_sockmaps_records(orc_sockmaps* m);
size_t orc_sockmaps_lines(orc_sockmaps* m, uint32_t* pid, uint64_t* fd, uint64_t* len, size_t cap);
void orc_sockmaps_join(orc_sockmaps* m, alz_l7_rec* recs, const alz_sock_query* keys, size_t n, uint64_t now,
                       uint64_t* joined);
size_t orc_sockmaps_alive(orc_sockmaps* m, const orc* o, alz_alive_conn* out, size_t cap);

/* ---- "fair" CPU arm (alz_fastcpu.c): same results, integer keys, flat tables, pinned threads ---- */
typedef struct orc_fast orc_fast;
orc_fast* orc_fast_create(uint32_t max_endpoints);
void orc_fast_destroy(orc_fast* f);
void orc_fast_table_upsert(orc_fast* f, int table, uint32_t ipv4, uint32_t id);
void orc_fast_process(orc_fast* f, const alz_l7_rec* recs, size_t n, int nthreads);
size_t orc_fast_edges(orc_fast* f, alz_edge_out* out, size_t cap);
void orc_fast_reset(orc_fast* f);
void orc_fast_stats(orc_fast* f, alz_stats* st);

#ifdef __cplusplus
}
#endif
#endif
