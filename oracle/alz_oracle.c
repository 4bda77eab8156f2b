/*
 * alz_oracle.c — CPU restatement of the reference's aggregation hot path.
 * TEST INFRASTRUCTURE ONLY (see alz_oracle.h for who may use it and for the
 * parity status: resolve/emit is PARITY UNPINNED, SocketLine is KAT-pinned).
 *
 * It deliberately keeps the reference's data structures: dotted-quad strings
 * built per event, string-keyed maps for the IP->UID tables, one heap row per
 * surviving event, string compares for protocol/method — so that timing it is
 * a fair stand-in for the Go path ("port", not the Go binary).
 */
#define _GNU_SOURCE
#include "alz_oracle.h"

#include <pthread.h>
#include <sched.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

/* ======================= string-keyed open hash map ======================= */
typedef struct smap_ent {
  char* key; /* NULL = empty, (char*)1 = tombstone */
  void* val;
} smap_ent;
typedef struct smap {
  smap_ent* e;
  size_t cap, len, used;
} smap;
#define TOMB ((char*)1)

static uint64_t str_hash(const char* s) { /* FNV-1a, like a runtime string hash */
  uint64_t h = 1469598103934665603ull;
  for (; *s; s++) { h ^= (unsigned char)*s; h *= 1099511628211ull; }
  return h;
}
static void smap_init(smap* m, size_t cap) {
  m->cap = cap; m->len = 0; m->used = 0;
  m->e = (smap_ent*)calloc(cap, sizeof(smap_ent));
}
static void smap_free(smap* m, int free_vals) {
  for (size_t i = 0; i < m->cap; i++)
    if (m->e[i].key && m->e[i].key != TOMB) { free(m->e[i].key); if (free_vals) free(m->e[i].val); }
  free(m->e); m->e = NULL;
}
static smap_ent* smap_find(const smap* m, const char* k) {
  size_t i = str_hash(k) & (m->cap - 1);
  for (;;) {
    smap_ent* e = &m->e[i];
    if (!e->key) return NULL;
    if (e->key != TOMB && strcmp(e->key, k) == 0) return e;
    i = (i + 1) & (m->cap - 1);
  }
}
static void smap_put(smap* m, const char* k, void* v, int free_old);
static void smap_grow(smap* m) {
  smap old = *m;
  smap_init(m, old.cap * 2);
  for (size_t i = 0; i < old.cap; i++)
    if (old.e[i].key && old.e[i].key != TOMB) {
      size_t j = str_hash(old.e[i].key) & (m->cap - 1);
      while (m->e[j].key) j = (j + 1) & (m->cap - 1);
      m->e[j] = old.e[i]; m->len++; m->used++;
    }
  free(old.e);
}
static void smap_put(smap* m, const char* k, void* v, int free_old) {
  smap_ent* f = smap_find(m, k);
  if (f) { if (free_old) free(f->val); f->val = v; return; }
  if ((m->used + 1) * 2 > m->cap) smap_grow(m);
  size_t i = str_hash(k) & (m->cap - 1);
  while (m->e[i].key && m->e[i].key != TOMB) i = (i + 1) & (m->cap - 1);
  if (!m->e[i].key) m->used++;
  m->e[i].key = strdup(k); m->e[i].val = v; m->len++;
}
static void smap_del(smap* m, const char* k, int free_val) {
  smap_ent* f = smap_find(m, k);
  if (!f) return;
  free(f->key); if (free_val) free(f->val);
  f->key = TOMB; f->val = NULL; m->len--;
}

/* ============================ the aggregator ============================= */
/* aggregator/data.go:42-44 */
static const char* POD = "pod";
static const char* SVC = "service";
static const char* OUTBOUND = "outbound";

#define NSHARD 64
typedef struct acc {
  uint64_t count, err5xx, lat_sum;
  uint32_t hist[ALZ_NB];
} acc;

struct orc {
  const char* const* host_names; /* id -> Host header text, for orc_edges (set by orc_process_l7_hosts) */
  size_t n_host_names;
  smap pod_ip_to_uid; /* ClusterInfo.PodIPToPodUid, cluster.go:15 */
  smap svc_ip_to_uid; /* ClusterInfo.ServiceIPToServiceUid, cluster.go:16 */
  smap groups[NSHARD]; /* "ftype|fuid|ttype|tuid" -> acc*, sharded by key hash so that the
                          multi-threaded merge can run one shard per thread */
  alz_stats st;
};

orc* orc_create(void) {
  orc* o = (orc*)calloc(1, sizeof(*o));
  smap_init(&o->pod_ip_to_uid, 1024);
  smap_init(&o->svc_ip_to_uid, 1024);
  for (int i = 0; i < NSHARD; i++) smap_init(&o->groups[i], 256);
  return o;
}
void orc_destroy(orc* o) {
  if (!o) return;
  smap_free(&o->pod_ip_to_uid, 1);
  smap_free(&o->svc_ip_to_uid, 1);
  for (int i = 0; i < NSHARD; i++) smap_free(&o->groups[i], 1);
  free(o);
}

/* IntToIPv4(x).String(): big-endian bytes, aggregator/data.go:1751-1767 */
static void ip_string(uint32_t ip, char* buf /* >=16 */) {
  snprintf(buf, 16, "%u.%u.%u.%u", (ip >> 24) & 255u, (ip >> 16) & 255u, (ip >> 8) & 255u,
           ip & 255u);
}

void orc_table_upsert(orc* o, int table, uint32_t ipv4, uint32_t id) {
  char ip[16], uid[24];
  ip_string(ipv4, ip);
  if (table == ALZ_TABLE_POD) { /* persist.go:55-65 ADD/UPDATE */
    snprintf(uid, sizeof uid, "pod-%u", id);
    smap_put(&o->pod_ip_to_uid, ip, strdup(uid), 1);
  } else { /* persist.go:114-124 */
    snprintf(uid, sizeof uid, "svc-%u", id);
    smap_put(&o->svc_ip_to_uid, ip, strdup(uid), 1);
  }
}
void orc_table_erase(orc* o, int table, uint32_t ipv4) {
  char ip[16];
  ip_string(ipv4, ip);
  smap_del(table == ALZ_TABLE_POD ? &o->pod_ip_to_uid : &o->svc_ip_to_uid, ip, 1); /* :66-70, :125-129 */
}

/* ebpf/l7_req/l7.go:48-71 */
static const char* protocol_string(uint8_t p) {
  switch (p) {
    case 1: return "HTTP";   case 2: return "AMQP";  case 3: return "POSTGRES";
    case 4: return "HTTP2";  case 5: return "REDIS"; case 6: return "KAFKA";
    case 7: return "MYSQL";  case 8: return "MONGO"; case 0: return "UNKNOWN";
    default: return "Unknown";
  }
}
/* ebpf/l7_req/l7.go:204-325 and the switch in Consume, :712-734 */
static const char* method_string(const char* proto, uint8_t m) {
  static const char* http[] = {"Unknown", "GET", "POST", "PUT", "PATCH", "DELETE",
                               "HEAD", "CONNECT", "OPTIONS", "TRACE"};
  if (!strcmp(proto, "HTTP")) return m <= 9 ? http[m] : "Unknown";
  if (!strcmp(proto, "AMQP")) return m == 1 ? "PUBLISH" : m == 2 ? "DELIVER" : "Unknown";
  if (!strcmp(proto, "POSTGRES"))
    return m == 1 ? "CLOSE_OR_TERMINATE" : m == 2 ? "SIMPLE_QUERY" : m == 3 ? "EXTENDED_QUERY" : "Unknown";
  if (!strcmp(proto, "HTTP2")) return m == 1 ? "CLIENT_FRAME" : m == 2 ? "SERVER_FRAME" : "Unknown";
  if (!strcmp(proto, "REDIS")) return m == 1 ? "COMMAND" : m == 2 ? "PUSHED_EVENT" : m == 3 ? "PING" : "Unknown";
  if (!strcmp(proto, "KAFKA")) return m == 1 ? "PRODUCE_REQUEST" : m == 2 ? "FETCH_RESPONSE" : "Unknown";
  if (!strcmp(proto, "MYSQL"))
    return m == 1 ? "TEXT_QUERY" : m == 2 ? "PREPARE_STMT" : m == 3 ? "EXEC_STMT" : m == 4 ? "STMT_CLOSE" : "Unknown";
  return "Unknown"; /* default branch, :731-733 (Mongo has no case) */
}

/* datastore.Request (datastore/dto.go:197-218), the fields the group-by reads */
typedef struct request {
  uint64_t latency;
  char from_ip[16], to_ip[16];
  const char* from_type; const char* to_type;
  char from_uid[72], to_uid[72]; /* UID, or a host name / dotted quad for outbound */
  uint16_t from_port, to_port;
  const char* protocol;
  uint32_t status_code;
  const char* method;
  int tls;
} request;

/* Request.ReverseDirection, datastore/dto.go:246-251 */
static void reverse_direction(request* r) {
  char t[72];
  memcpy(t, r->from_ip, 16); memcpy(r->from_ip, r->to_ip, 16); memcpy(r->to_ip, t, 16);
  uint16_t p = r->from_port; r->from_port = r->to_port; r->to_port = p;
  memcpy(t, r->from_uid, 72); memcpy(r->from_uid, r->to_uid, 72); memcpy(r->to_uid, t, 72);
  const char* ty = r->from_type; r->from_type = r->to_type; r->to_type = ty;
}

/* setFromToV2, aggregator/data.go:827-870. hostHeader is always "" for compact
 * records (no payload) and reverse DNS (getHostnameFromIP, :1386-1405) is
 * treated as failing, so the outbound key is the raw daddr string (:862). */
static int set_from_to_v2(const orc* o, request* r, const char* host_header) {
  smap_ent* pod = smap_find(&o->pod_ip_to_uid, r->from_ip); /* getPodWithIP :812-817 */
  if (!pod) return -1;                                        /* :829-832 */
  snprintf(r->from_uid, sizeof r->from_uid, "%s", (const char*)pod->val);
  r->from_type = POD;
  smap_ent* svc = smap_find(&o->svc_ip_to_uid, r->to_ip);   /* getSvcWithIP :819-825 */
  if (svc) {
    snprintf(r->to_uid, sizeof r->to_uid, "%s", (const char*)svc->val);
    r->to_type = SVC;
  } else {
    smap_ent* dpod = smap_find(&o->pod_ip_to_uid, r->to_ip); /* :845 */
    if (dpod) {
      snprintf(r->to_uid, sizeof r->to_uid, "%s", (const char*)dpod->val);
      r->to_type = POD;
    } else {
      if (host_header && host_header[0]) snprintf(r->to_uid, sizeof r->to_uid, "%s", host_header); /* :851-854 */
      else snprintf(r->to_uid, sizeof r->to_uid, "%s", r->to_ip); /* :862 (reverse DNS treated as failing) */
      r->to_type = OUTBOUND;
    }
  }
  return 0;
}

uint32_t orc_bucket(uint64_t d) {
  /* docs/SPEC.md §4: 2 sub-buckets per octave over [2^8, 2^40), clamped */
  if (d < 256) return 0;
  uint32_t o = 0;
  uint64_t t = d;
  while (t > 1) { t >>= 1; o++; } /* floor(log2 d) */
  if (o >= 40) return ALZ_NB - 1;
  uint32_t half = (uint32_t)((d >> (o - 1)) & 1u);
  return 2 * (o - 8) + half;
}

/* PersistRequest stand-in: fold the emitted row into its (From,To) group */
static void persist_request(smap* shards, const request* r, alz_stats* st) {
  char key[192];
  snprintf(key, sizeof key, "%s|%s|%s|%s", r->from_type, r->from_uid, r->to_type, r->to_uid);
  smap* groups = &shards[str_hash(key) % NSHARD];
  smap_ent* g = smap_find(groups, key);
  acc* a;
  if (g) a = (acc*)g->val;
  else { a = (acc*)calloc(1, sizeof(acc)); smap_put(groups, key, a, 0); }
  a->count++;
  if ((!strcmp(r->protocol, "HTTP") || !strcmp(r->protocol, "HTTPS")) &&
      r->status_code >= 500 && r->status_code < 600)
    a->err5xx++;
  a->lat_sum += r->latency;
  a->hist[orc_bucket(r->latency)]++;
  st->rows_emitted++;
}

/* processL7 (aggregator/data.go:1364-1383) for one compact record */
static void process_l7(const orc* o, const alz_l7_rec* d, smap* groups, alz_stats* st, const char* host_header) {
  st->events_in++;
  const char* protocol = protocol_string(d->protocol);
  const uint8_t m = d->method_flags & ALZ_MF_METHOD_MASK;
  const char* method = method_string(protocol, m);
  const int tls = (d->method_flags & ALZ_MF_TLS) != 0;
  const int payload_reject = (d->method_flags & ALZ_MF_PAYLOAD_REJECT) != 0;

  int is_http = !strcmp(protocol, "HTTP");
  int is_amqp = !strcmp(protocol, "AMQP");
  int is_redis = !strcmp(protocol, "REDIS");
  int is_sql = !strcmp(protocol, "POSTGRES") || !strcmp(protocol, "MYSQL") || !strcmp(protocol, "MONGO");
  if (!(is_http || is_amqp || is_redis || is_sql)) {
    /* HTTP2 -> processHttp2Event (stateful frame pairing, :1019-1033, out of
     * scope); KAFKA -> PersistKafkaEvent, not a request row (:1035-1078);
     * UNKNOWN / others -> no case */
    st->not_request++;
    return;
  }
  /* parsePostgresCommand / parseMySQLCommand / parseMongoEvent returned an
   * error: the handler returns before building the row (:1252-1255,
   * :1288-1292, :1328-1332) */
  if (is_sql && payload_reject) { st->not_request++; return; }

  request* r = (request*)calloc(1, sizeof(request)); /* reqDto := &datastore.Request{...} */
  r->latency = d->duration_ns;
  ip_string(d->saddr, r->from_ip); /* extractAddressPair :1760-1767 */
  ip_string(d->daddr, r->to_ip);
  r->from_port = d->sport; r->to_port = d->dport;
  r->protocol = protocol; r->tls = tls; r->status_code = d->status; r->method = method;

  /* only processHttpEvent parses a Host header out of the payload (:1213); the other handlers pass "" */
  if (set_from_to_v2(o, r, is_http ? host_header : NULL) != 0) { st->src_unresolved++; free(r); return; }

  /* :1110-1112 AMQP DELIVER, :1151-1153 REDIS PUSHED_EVENT */
  if (is_amqp && !strcmp(method, "DELIVER")) reverse_direction(r);
  if (is_redis && !strcmp(method, "PUSHED_EVENT")) reverse_direction(r);
  /* :1240-1242 */
  if (is_http && tls) r->protocol = "HTTPS";

  persist_request(groups, r, st);
  free(r);
}

typedef struct worker {
  orc* o;
  const alz_l7_rec* recs;
  size_t n;
  smap groups[NSHARD];
  alz_stats st;
  struct worker* all;
  int nworkers, id;
} worker;
/* one thread per logical CPU, pinned (best effort): unpinned runs of this arm varied 2.8x from box to box */
static void pin_worker(int id) {
  cpu_set_t set; CPU_ZERO(&set); CPU_SET(id % CPU_SETSIZE, &set);
  pthread_setaffinity_np(pthread_self(), sizeof set, &set);
}
static void* worker_main(void* p) {
  worker* w = (worker*)p;
  pin_worker(w->id);
  for (size_t i = 0; i < w->n; i++) process_l7(w->o, &w->recs[i], w->groups, &w->st, NULL);
  return NULL;
}
static void merge_acc(acc* dst, const acc* src);
/* phase 2: thread `id` folds shards id, id+T, ... of every worker into the shared result */
static void* merge_main(void* p) {
  worker* w = (worker*)p;
  pin_worker(w->id);
  for (int sh = w->id; sh < NSHARD; sh += w->nworkers) {
    smap* dst = &w->o->groups[sh];
    for (int t = 0; t < w->nworkers; t++) {
      smap* src = &w->all[t].groups[sh];
      for (size_t i = 0; i < src->cap; i++) {
        smap_ent* e = &src->e[i];
        if (!e->key || e->key == TOMB) continue;
        smap_ent* g = smap_find(dst, e->key);
        if (g) { merge_acc((acc*)g->val, (acc*)e->val); free(e->val); }
        else smap_put(dst, e->key, e->val, 0);
      }
    }
  }
  return NULL;
}
static void merge_acc(acc* dst, const acc* src) {
  dst->count += src->count; dst->err5xx += src->err5xx; dst->lat_sum += src->lat_sum;
  for (int b = 0; b < ALZ_NB; b++) dst->hist[b] += src->hist[b];
}

void orc_process_l7(orc* o, const alz_l7_rec* recs, size_t n, int nthreads) {
  if (nthreads <= 1) {
    for (size_t i = 0; i < n; i++) process_l7(o, &recs[i], o->groups, &o->st, NULL);
    return;
  }
  worker* w = (worker*)calloc((size_t)nthreads, sizeof(worker));
  pthread_t* th = (pthread_t*)calloc((size_t)nthreads, sizeof(pthread_t));
  size_t per = (n + (size_t)nthreads - 1) / (size_t)nthreads;
  for (int t = 0; t < nthreads; t++) {
    size_t b = per * (size_t)t, e = b + per; if (b > n) b = n; if (e > n) e = n;
    w[t].o = o; w[t].recs = recs + b; w[t].n = e - b; w[t].all = w; w[t].nworkers = nthreads; w[t].id = t;
    for (int i = 0; i < NSHARD; i++) smap_init(&w[t].groups[i], 64);
    pthread_create(&th[t], NULL, worker_main, &w[t]);
  }
  for (int t = 0; t < nthreads; t++) pthread_join(th[t], NULL);
  for (int t = 0; t < nthreads; t++) pthread_create(&th[t], NULL, merge_main, &w[t]);
  for (int t = 0; t < nthreads; t++) pthread_join(th[t], NULL);
  for (int t = 0; t < nthreads; t++) {
    for (int i = 0; i < NSHARD; i++) smap_free(&w[t].groups[i], 0);
    o->st.events_in += w[t].st.events_in; o->st.rows_emitted += w[t].st.rows_emitted;
    o->st.not_request += w[t].st.not_request; o->st.src_unresolved += w[t].st.src_unresolved;
  }
  free(w); free(th);
}

void orc_process_l7_hosts(orc* o, const alz_l7_rec* recs, size_t n, const uint32_t* host_idx,
                          const char* const* names, size_t n_names) {
  o->host_names = names; o->n_host_names = n_names;
  for (size_t i = 0; i < n; i++) {
    const char* hh = (host_idx && host_idx[i]) ? names[host_idx[i] - 1] : NULL;
    process_l7(o, &recs[i], o->groups, &o->st, hh);
  }
}

/* parseHttpPayload, aggregator/data.go:508-531, the hostHeader part: lines = Split(request, "\n"); for the
 * lines after the first, the first one that HasPrefix "Host:" AND splits (on single spaces) into >= 2 parts
 * gives parts[1] without a trailing "\r". A "Host:" line with fewer parts is skipped and the scan goes on. */
size_t orc_parse_http_host(const char* payload, size_t n, char* out, size_t cap) {
  if (cap) out[0] = 0;
  size_t i = 0;
  while (i < n && payload[i] != '\n') i++; /* lines[0] */
  while (i < n) {
    i++; /* past the '\n' */
    size_t b = i;
    while (i < n && payload[i] != '\n') i++;
    const char* line = payload + b; size_t len = i - b;
    if (len >= 5 && !memcmp(line, "Host:", 5)) {
      /* strings.Split(line, " "): parts[0] ends at the first space, parts[1] at the second (or the end) */
      size_t sp = 0;
      while (sp < len && line[sp] != ' ') sp++;
      if (sp < len) { /* at least two parts */
        size_t q = sp + 1, e = q;
        while (e < len && line[e] != ' ') e++;
        size_t hl = e - q;
        if (hl > 0 && line[q + hl - 1] == '\r') hl--; /* TrimSuffix(hostHeader, "\r") */
        if (hl >= cap) hl = cap ? cap - 1 : 0;
        if (cap) { memcpy(out, line + q, hl); out[hl] = 0; }
        return hl;
      }
    }
  }
  return 0;
}

uint64_t orc_epoch(uint64_t first_kernel_ns, uint64_t first_user_ns, uint64_t window_ns, uint64_t write_time_ns) {
  const uint64_t user = first_user_ns - (first_kernel_ns - write_time_ns); /* data.go:1740-1743, uint64 arithmetic */
  return window_ns ? user / window_ns : 0;
}

static int parse_node(const orc* o, const char* type, const char* uid, uint8_t* t, uint32_t* v) {
  if (!strcmp(type, "pod")) { *t = ALZ_NODE_POD; *v = (uint32_t)strtoul(uid + 4, NULL, 10); return 0; }
  if (!strcmp(type, "service")) { *t = ALZ_NODE_SVC; *v = (uint32_t)strtoul(uid + 4, NULL, 10); return 0; }
  unsigned a, b, c, d; char tail;
  if (sscanf(uid, "%u.%u.%u.%u%c", &a, &b, &c, &d, &tail) == 4 && a < 256 && b < 256 && c < 256 && d < 256) {
    *t = ALZ_NODE_OUTBOUND; *v = (a << 24) | (b << 16) | (c << 8) | d;
    return 0;
  }
  for (size_t i = 0; i < o->n_host_names; i++)
    if (!strcmp(o->host_names[i], uid)) { *t = ALZ_NODE_OUTBOUND_HOST; *v = (uint32_t)i; return 0; }
  return -1;
}
static int edge_cmp(const void* pa, const void* pb) {
  const alz_edge_out* a = (const alz_edge_out*)pa; const alz_edge_out* b = (const alz_edge_out*)pb;
  if (a->from_type != b->from_type) return a->from_type < b->from_type ? -1 : 1;
  if (a->from != b->from) return a->from < b->from ? -1 : 1;
  if (a->to_type != b->to_type) return a->to_type < b->to_type ? -1 : 1;
  if (a->to != b->to) return a->to < b->to ? -1 : 1;
  return 0;
}
size_t orc_edges(orc* o, alz_edge_out* out, size_t cap) {
  size_t n = 0;
  for (int sh = 0; sh < NSHARD; sh++)
  for (size_t i = 0; i < o->groups[sh].cap; i++) {
    smap_ent* e = &o->groups[sh].e[i];
    if (!e->key || e->key == TOMB) continue;
    if (n < cap) {
      char k[192]; snprintf(k, sizeof k, "%s", e->key);
      char* ft = strtok(k, "|"); char* fu = strtok(NULL, "|");
      char* tt = strtok(NULL, "|"); char* tu = strtok(NULL, "|");
      alz_edge_out* r = &out[n]; memset(r, 0, sizeof *r);
      parse_node(o, ft, fu, &r->from_type, &r->from);
      parse_node(o, tt, tu, &r->to_type, &r->to);
      const acc* a = (const acc*)e->val;
      r->count = a->count; r->err5xx = a->err5xx; r->lat_sum_ns = a->lat_sum;
      memcpy(r->hist, a->hist, sizeof r->hist);
    }
    n++;
  }
  qsort(out, n < cap ? n : cap, sizeof(alz_edge_out), edge_cmp);
  return n;
}
void orc_window_reset(orc* o) {
  for (int i = 0; i < NSHARD; i++) { smap_free(&o->groups[i], 1); smap_init(&o->groups[i], 256); }
}
void orc_stats(orc* o, alz_stats* st) {
  *st = o->st;
  st->edges_live = 0;
  for (int i = 0; i < NSHARD; i++) st->edges_live += o->groups[i].len;
}

/* docs/SPEC.md §5 */
static double bucket_lo(uint32_t b) {
  if (b == 0) return 0.0;
  double base = (double)(1ull << (8 + b / 2));
  return (b & 1u) ? base * 1.5 : base;
}
static double bucket_hi(uint32_t b) {
  if (b == ALZ_NB - 1) return (double)(1ull << 40);
  return bucket_lo(b + 1);
}
double orc_quantile(const uint32_t* hist, double q) {
  uint64_t total = 0;
  for (int b = 0; b < ALZ_NB; b++) total += hist[b];
  if (total == 0) return 0.0;
  double target = q * (double)total;
  double cum = 0.0;
  for (uint32_t b = 0; b < ALZ_NB; b++) {
    double c = (double)hist[b];
    if (c > 0.0 && cum + c >= target) {
      double f = (target - cum) / c;
      if (f < 0.0) f = 0.0;
      return bucket_lo(b) + f * (bucket_hi(b) - bucket_lo(b));
    }
    cum += c;
  }
  return bucket_hi(ALZ_NB - 1);
}

/* bpfL7Event field offsets, ebpf/l7_req/l7.go:345-369 (Go struct layout) */
void orc_compact_raw(const void* raw, size_t n, alz_l7_rec* out) {
  const uint8_t* p = (const uint8_t*)raw;
  for (size_t i = 0; i < n; i++, p += ALZ_BPF_L7_EVENT_SIZE) {
    uint64_t write_time, duration; uint32_t status, saddr, daddr; uint16_t sport, dport;
    memcpy(&write_time, p + 8, 8); memcpy(&status, p + 20, 4); memcpy(&duration, p + 24, 8);
    uint8_t protocol = p[32], method = p[33], is_tls = p[1066];
    memcpy(&saddr, p + 1076, 4); memcpy(&sport, p + 1080, 2);
    memcpy(&daddr, p + 1084, 4); memcpy(&dport, p + 1088, 2);
    alz_l7_rec* r = &out[i];
    r->saddr = saddr; r->daddr = daddr; r->sport = sport; r->dport = dport;
    r->status = status > 65535u ? 65535u : (uint16_t)status;
    r->protocol = protocol;
    r->method_flags = (uint8_t)((method & ALZ_MF_METHOD_MASK) | (is_tls ? ALZ_MF_TLS : 0));
    r->duration_ns = duration; r->write_time_ns = write_time;
  }
}

/* ===================== SocketLine (sock_num_line.go) ====================== */
typedef struct ts_sock {
  uint64_t ts;
  uint64_t last_match; /* TimestampedSocket.LastMatch, sock_num_line.go:26 */
  int open; /* SockInfo != nil */
  orc_sockinfo si;
} ts_sock;
struct orc_sockline {
  ts_sock* v;
  size_t len, cap;
};
orc_sockline* orc_sockline_create(void) { return (orc_sockline*)calloc(1, sizeof(orc_sockline)); }
void orc_sockline_destroy(orc_sockline* l) { if (l) { free(l->v); free(l); } }
size_t orc_sockline_len(orc_sockline* l) { return l->len; }

void orc_sockline_add(orc_sockline* l, uint64_t ts, const orc_sockinfo* si) {
  /* :70-78 — drop if equal to the LAST element's open socket */
  if (l->len > 0) {
    const ts_sock* last = &l->v[l->len - 1];
    if (last->open && si && last->si.saddr == si->saddr && last->si.sport == si->sport &&
        last->si.daddr == si->daddr && last->si.dport == si->dport)
      return;
  }
  /* insertIntoSortedSlice :311-322 — first index with Timestamp >= new */
  size_t lo = 0, hi = l->len;
  while (lo < hi) { size_t mid = (lo + hi) / 2; if (l->v[mid].ts >= ts) hi = mid; else lo = mid + 1; }
  if (l->len == l->cap) { l->cap = l->cap ? l->cap * 2 : 8; l->v = (ts_sock*)realloc(l->v, l->cap * sizeof(ts_sock)); }
  memmove(&l->v[lo + 1], &l->v[lo], (l->len - lo) * sizeof(ts_sock));
  l->v[lo].ts = ts; l->v[lo].open = si != NULL; l->v[lo].last_match = 0;
  if (si) l->v[lo].si = *si; else memset(&l->v[lo].si, 0, sizeof(orc_sockinfo));
  l->len++;
}

int orc_sockline_get(orc_sockline* l, uint64_t ts, orc_sockinfo* out) { return orc_sockline_get_at(l, ts, 1, out); }

/* GetValue with time.Now() = now (the LastMatch stamps of :96 and :156) */
int orc_sockline_get_at(orc_sockline* l, uint64_t ts, uint64_t now, orc_sockinfo* out) {
  if (l->len == 0) return 0; /* :86-88 */
  /* sort.Search: first index with !(Timestamp < ts), :90-92 */
  size_t lo = 0, hi = l->len;
  while (lo < hi) { size_t mid = (lo + hi) / 2; if (!(l->v[mid].ts < ts)) hi = mid; else lo = mid + 1; }
  size_t index = lo;
  const uint64_t one_minute = 60ull * 1000000000ull;
  if (index == l->len) { /* :94-105 */
    l->v[index - 1].last_match = now; /* :96 */
    if (!l->v[l->len - 1].open) {
      if (index >= 2 && l->v[index - 2].open && (ts - l->v[index - 2].ts) < one_minute) {
        *out = l->v[index - 2].si; return 1;
      }
      return 0;
    }
    *out = l->v[l->len - 1].si; return 1;
  }
  if (index == 0) { /* :107-119 */
    if (l->v[0].open) { *out = l->v[0].si; return 1; }
    return 0;
  }
  if (!l->v[index - 1].open) { /* :123-153 */
    const ts_sock* prev = index >= 2 ? &l->v[index - 2] : NULL;
    const ts_sock* after = index < l->len ? &l->v[index] : NULL;
    if (prev && prev->open && after && after->open && prev->si.daddr == after->si.daddr &&
        prev->si.dport == after->si.dport) {
      if (ts - prev->ts < after->ts - ts) *out = prev->si; else *out = after->si;
      return 1;
    }
    return 0;
  }
  l->v[index - 1].last_match = now; /* :156 */
  *out = l->v[index - 1].si; /* :155-157 */
  return 1;
}

/* SocketLine.DeleteUnused, sock_num_line.go:160-209, as written: the first loop runs while i < len-1, so the
 * last element is carried over only when the loop steps over it (two opens in a row at the end). */
void orc_sockline_delete_unused(orc_sockline* l) {
  if (l->len <= 1) return; /* :165-167 */
  ts_sock* res = (ts_sock*)malloc(l->len * sizeof(ts_sock));
  size_t n = 0, i = 0;
  while (i < l->len - 1) { /* :172-181 */
    if (l->v[i].open && l->v[i + 1].open) { res[n++] = l->v[i + 1]; i += 2; }
    else { res[n++] = l->v[i]; i++; }
  }
  uint64_t last_matched = 0; /* :184-190 */
  for (size_t k = n; k-- > 0;)
    if (res[k].last_match != 0 && res[k].last_match > last_matched) last_matched = res[k].last_match;
  const uint64_t assumed_interval = 5ull * 60ull * 1000000000ull; /* :193 */
  for (long k = (long)n - 1; k >= 1; k--) { /* :197-208 */
    if (!res[k].open && res[k - 1].open && res[k - 1].last_match + assumed_interval < last_matched) {
      memmove(&res[k - 1], &res[k + 1], (n - (size_t)k - 1) * sizeof(ts_sock));
      n -= 2;
      k--;
    }
  }
  const size_t res_cap = l->len;
  free(l->v);
  l->v = res; l->len = n; l->cap = res_cap;
}

/* SocketMaps[pid].M[fd] -> *SocketLine (cluster.go:20, socket.go:30-40) */
typedef struct sm_ent { uint64_t fd; uint32_t pid; int used; orc_sockline* line; } sm_ent;
struct orc_sockmaps { sm_ent* e; size_t cap, len; };
orc_sockmaps* orc_sockmaps_create(void) {
  orc_sockmaps* m = (orc_sockmaps*)calloc(1, sizeof(*m));
  m->cap = 1024; m->e = (sm_ent*)calloc(m->cap, sizeof(sm_ent));
  return m;
}
void orc_sockmaps_destroy(orc_sockmaps* m) {
  if (!m) return;
  for (size_t i = 0; i < m->cap; i++) if (m->e[i].used) orc_sockline_destroy(m->e[i].line);
  free(m->e); free(m);
}
static uint64_t pf_hash(uint32_t pid, uint64_t fd) {
  uint64_t x = ((uint64_t)pid << 40) ^ fd ^ 0x9E3779B97F4A7C15ull;
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33;
  return x;
}
static sm_ent* sm_find(orc_sockmaps* m, uint32_t pid, uint64_t fd, int create) {
  if (create && (m->len + 1) * 2 > m->cap) {
    sm_ent* old = m->e; size_t oc = m->cap;
    m->cap *= 2; m->e = (sm_ent*)calloc(m->cap, sizeof(sm_ent));
    for (size_t i = 0; i < oc; i++) if (old[i].used) {
      size_t j = pf_hash(old[i].pid, old[i].fd) & (m->cap - 1);
      while (m->e[j].used) j = (j + 1) & (m->cap - 1);
      m->e[j] = old[i];
    }
    free(old);
  }
  size_t i = pf_hash(pid, fd) & (m->cap - 1);
  while (m->e[i].used) {
    if (m->e[i].pid == pid && m->e[i].fd == fd) return &m->e[i];
    i = (i + 1) & (m->cap - 1);
  }
  if (!create) return NULL;
  m->e[i].used = 1; m->e[i].pid = pid; m->e[i].fd = fd; m->e[i].line = orc_sockline_create();
  m->len++;
  return &m->e[i];
}

void orc_sockmaps_process_tcp(orc_sockmaps* m, const alz_tcp_rec* recs, size_t n,
                              uint64_t* localhost_dropped) {
  for (size_t i = 0; i < n; i++) {
    const alz_tcp_rec* d = &recs[i];
    char s[16], t[16];
    ip_string(d->saddr, s); ip_string(d->daddr, t); /* tcp.go:241-242 */
    if (d->type == 1) { /* EVENT_TCP_ESTABLISHED, data.go:406-449 */
      if (!strcmp(s, "127.0.0.1") || !strcmp(t, "127.0.0.1")) { if (localhost_dropped) (*localhost_dropped)++; continue; }
      /* socket map / line missing => created, event requeued and then applied
       * (:417-437); without /proc bootstrap the new line starts empty */
      sm_ent* e = sm_find(m, d->pid, d->fd, 1);
      orc_sockinfo si = {d->saddr, d->daddr, d->sport, d->dport};
      orc_sockline_add(e->line, d->timestamp_ns, &si);
    } else if (d->type == 5) { /* EVENT_TCP_CLOSED, :450-503 */
      if (!strcmp(s, "127.0.0.1") || !strcmp(t, "127.0.0.1")) { if (localhost_dropped) (*localhost_dropped)++; continue; }
      sm_ent* e = sm_find(m, d->pid, d->fd, 0);
      if (!e) continue; /* :471-473: no line => ignore */
      orc_sockline_add(e->line, d->timestamp_ns, NULL);
    }
  }
}

void orc_sockmaps_lookup(orc_sockmaps* m, const alz_sock_query* q, size_t n, alz_sock_result* out) {
  orc_sockmaps_lookup_at(m, q, n, 1, out);
}
void orc_sockmaps_lookup_at(orc_sockmaps* m, const alz_sock_query* q, size_t n, uint64_t now, alz_sock_result* out) {
  for (size_t i = 0; i < n; i++) {
    memset(&out[i], 0, sizeof out[i]);
    sm_ent* e = sm_find(m, q[i].pid, q[i].fd, 0); /* findRelatedSocket data.go:1407-1429 */
    orc_sockinfo si;
    if (e && orc_sockline_get_at(e->line, q[i].timestamp_ns, now, &si)) {
      out[i].found = 1; out[i].saddr = si.saddr; out[i].daddr = si.daddr;
      out[i].sport = si.sport; out[i].dport = si.dport;
    }
  }
}

/* one tick of clearSocketLines, data.go:1681-1716 (without the alive-connection export) */
void orc_sockmaps_gc(orc_sockmaps* m) {
  for (size_t i = 0; i < m->cap; i++) if (m->e[i].used) orc_sockline_delete_unused(m->e[i].line);
}
size_t orc_sockmaps_records(orc_sockmaps* m) {
  size_t n = 0;
  for (size_t i = 0; i < m->cap; i++) if (m->e[i].used) n += m->e[i].line->len;
  return n;
}
/* every line's (pid, fd) and length, in table order; returns the number of lines (the first `cap` are written) */
size_t orc_sockmaps_lines(orc_sockmaps* m, uint32_t* pid, uint64_t* fd, uint64_t* len, size_t cap) {
  size_t n = 0;
  for (size_t i = 0; i < m->cap; i++) {
    if (!m->e[i].used) continue;
    if (n < cap) { pid[n] = m->e[i].pid; fd[n] = m->e[i].fd; len[n] = m->e[i].line->len; }
    n++;
  }
  return n;
}

/* L7 events with an empty 5-tuple take the socket of (pid, fd) at WriteTimeNs (findRelatedSocket,
 * data.go:1407-1429); a miss leaves the record as it is */
void orc_sockmaps_join(orc_sockmaps* m, alz_l7_rec* recs, const alz_sock_query* keys, size_t n, uint64_t now,
                       uint64_t* joined) {
  for (size_t i = 0; i < n; i++) {
    if (recs[i].saddr != 0 || recs[i].daddr != 0) continue;
    sm_ent* e = sm_find(m, keys[i].pid, keys[i].fd, 0);
    orc_sockinfo si;
    if (e && orc_sockline_get_at(e->line, keys[i].timestamp_ns, now, &si)) {
      recs[i].saddr = si.saddr; recs[i].daddr = si.daddr; recs[i].sport = si.sport; recs[i].dport = si.dport;
      if (joined) (*joined)++;
    }
  }
}

/* sendOpenConnection, data.go:1628-1679, for every line (clearSocketLines with SEND_ALIVE_TCP_CONNECTIONS) */
size_t orc_sockmaps_alive(orc_sockmaps* m, const orc* o, alz_alive_conn* out, size_t cap) {
  size_t n = 0;
  for (size_t i = 0; i < m->cap; i++) {
    if (!m->e[i].used) continue;
    const orc_sockline* l = m->e[i].line;
    if (l->len == 0) continue; /* :1632-1634 */
    const ts_sock* t = &l->v[l->len - 1];
    if (!t->open) continue; /* a close: ignored */
    char from[16], to[16];
    ip_string(t->si.saddr, from); ip_string(t->si.daddr, to);
    smap_ent* pod = smap_find(&o->pod_ip_to_uid, from); /* :1643-1647 */
    if (!pod) continue;
    alz_alive_conn c;
    memset(&c, 0, sizeof c);
    c.from_ip = t->si.saddr; c.from_port = t->si.sport; c.to_ip = t->si.daddr; c.to_port = t->si.dport;
    c.from_id = (uint32_t)strtoul((const char*)pod->val + 4, NULL, 10);
    smap_ent* svc = smap_find(&o->svc_ip_to_uid, to); /* :1662-1665 */
    if (svc) { c.to_type = ALZ_NODE_SVC; c.to_id = (uint32_t)strtoul((const char*)svc->val + 4, NULL, 10); }
    else {
      smap_ent* dpod = smap_find(&o->pod_ip_to_uid, to); /* :1667-1670 */
      if (dpod) { c.to_type = ALZ_NODE_POD; c.to_id = (uint32_t)strtoul((const char*)dpod->val + 4, NULL, 10); }
      else { c.to_type = ALZ_NODE_OUTBOUND; c.to_id = t->si.daddr; } /* :1671-1674 */
    }
    if (n < cap) out[n] = c;
    n++;
  }
  return n;
}
