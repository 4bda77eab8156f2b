// alaz_aggregator.cc — see alaz_aggregator.hpp. Plain C++ over the C ABI; no CUDA here.
#include "alaz_aggregator.hpp"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <cstdint>

#include "../../include/alazgpu_synth.h"   // alz_pinned_alloc / alz_pinned_free

namespace alaz {

namespace {
// reverse of L7ProtocolConversion.String(), ebpf/l7_req/l7.go:48-71
uint8_t ProtocolEnum(const std::string& p) {
  if (p == "HTTP") return ALZ_PROTO_HTTP;
  if (p == "AMQP") return ALZ_PROTO_AMQP;
  if (p == "POSTGRES") return ALZ_PROTO_POSTGRES;
  if (p == "HTTP2") return ALZ_PROTO_HTTP2;
  if (p == "REDIS") return ALZ_PROTO_REDIS;
  if (p == "KAFKA") return ALZ_PROTO_KAFKA;
  if (p == "MYSQL") return ALZ_PROTO_MYSQL;
  if (p == "MONGO") return ALZ_PROTO_MONGO;
  return ALZ_PROTO_UNKNOWN;
}
// reverse of the per-protocol method conversions, l7.go:204-325
uint8_t MethodEnum(uint8_t proto, const std::string& m) {
  static const char* http[] = {"", "GET", "POST", "PUT", "PATCH", "DELETE", "HEAD", "CONNECT", "OPTIONS", "TRACE"};
  switch (proto) {
    case ALZ_PROTO_HTTP:
      for (int i = 1; i <= 9; ++i) if (m == http[i]) return (uint8_t)i;
      return 0;
    case ALZ_PROTO_AMQP: return m == "PUBLISH" ? 1 : m == "DELIVER" ? 2 : 0;
    case ALZ_PROTO_POSTGRES: return m == "CLOSE_OR_TERMINATE" ? 1 : m == "SIMPLE_QUERY" ? 2 : m == "EXTENDED_QUERY" ? 3 : 0;
    case ALZ_PROTO_HTTP2: return m == "CLIENT_FRAME" ? 1 : m == "SERVER_FRAME" ? 2 : 0;
    case ALZ_PROTO_REDIS: return m == "COMMAND" ? 1 : m == "PUSHED_EVENT" ? 2 : m == "PING" ? 3 : 0;
    case ALZ_PROTO_KAFKA: return m == "PRODUCE_REQUEST" ? 1 : m == "FETCH_RESPONSE" ? 2 : 0;
    case ALZ_PROTO_MYSQL: return m == "TEXT_QUERY" ? 1 : m == "PREPARE_STMT" ? 2 : m == "EXEC_STMT" ? 3 : m == "STMT_CLOSE" ? 4 : 0;
    default: return 0;
  }
}
const char* NodeTypeName(uint8_t t) {   // aggregator/data.go:42-44 (a Host-header keyed destination is OUTBOUND too)
  return t == ALZ_NODE_POD ? "pod" : t == ALZ_NODE_SVC ? "service" : t == ALZ_NODE_GROUP ? "group" : "outbound";
}
}  // namespace

uint32_t Aggregator::ParseIPv4(const std::string& s, bool* ok) {
  unsigned a, b, c, d;
  char tail;
  const bool good = sscanf(s.c_str(), "%u.%u.%u.%u%c", &a, &b, &c, &d, &tail) == 4 && a < 256 && b < 256 && c < 256 && d < 256;
  if (ok) *ok = good;
  return good ? (a << 24) | (b << 16) | (c << 8) | d : 0u;
}
std::string Aggregator::FormatIPv4(uint32_t ip) {
  char buf[16];
  snprintf(buf, sizeof buf, "%u.%u.%u.%u", ip >> 24, (ip >> 16) & 255u, (ip >> 8) & 255u, ip & 255u);
  return buf;
}

// parseHttpPayload, aggregator/data.go:508-531, the hostHeader part: the request is split on "\n"; among the
// lines after the first, the first one that starts with "Host:" AND splits on single spaces into >= 2 parts
// yields parts[1] minus a trailing "\r". A "Host:" line with fewer parts is skipped and the scan goes on.
std::string Aggregator::ParseHttpHostHeader(const std::string& payload) {
  size_t i = payload.find('\n');
  while (i != std::string::npos) {
    const size_t b = i + 1;
    const size_t e = payload.find('\n', b);
    const size_t len = (e == std::string::npos ? payload.size() : e) - b;
    if (len >= 5 && payload.compare(b, 5, "Host:") == 0) {
      const size_t sp = payload.find(' ', b);
      if (sp != std::string::npos && sp < b + len) {            // at least two parts
        size_t q = sp + 1, end = payload.find(' ', q);
        if (end == std::string::npos || end > b + len) end = b + len;
        std::string host = payload.substr(q, end - q);
        if (!host.empty() && host.back() == '\r') host.pop_back();
        return host;
      }
    }
    i = e;
  }
  return std::string();
}

Aggregator::Aggregator(DataStore* ds, const AggregatorConfig& cfg) : ds_(ds), cfg_(cfg) {
  alz_config c;
  memset(&c, 0, sizeof c);
  c.abi_version = ALZ_ABI_VERSION;
  c.device = cfg.Device;
  c.max_endpoints = cfg.MaxEndpoints;
  c.max_pairs = cfg.MaxPairs;
  c.max_batch = (uint32_t)cfg.BatchSize;
  if (cfg_.BatchSize == 0) cfg_.BatchSize = 1;
  const int rc = alz_create(&c, &h_);
  if (rc != ALZ_OK) { err_ = alz_strerror(rc); h_ = nullptr; return; }
  void* p = nullptr;
  if (alz_pinned_alloc(cfg_.BatchSize * sizeof(alz_l7_rec), &p) != ALZ_OK) {
    err_ = "alz_pinned_alloc";   // no batch buffer: the aggregator is unusable, Ok() says so
    alz_destroy(h_);
    h_ = nullptr;
    return;
  }
  batch_ = static_cast<alz_l7_rec*>(p);
  out_.resize(cfg.MaxPairs);
}

Aggregator::~Aggregator() {
  if (batch_) alz_pinned_free(batch_);
  if (h_) alz_destroy(h_);
}

uint32_t Aggregator::Interner::Acquire(const std::string& uid) {
  auto it = ids.find(uid);
  if (it != ids.end()) return it->second;
  uint32_t id;
  if (!free_ids.empty()) {
    id = free_ids.back();
    free_ids.pop_back();
    names[id] = uid;
    reused_after[id] = std::max(reused_after[id], unmapped_in[id]);
  } else {
    id = (uint32_t)names.size();
    names.push_back(uid); refs.push_back(0); unmapped_in.push_back(0); reused_after.push_back(0);
  }
  ids.emplace(uid, id);
  changes += 1;
  return id;
}
void Aggregator::Interner::Map(uint32_t ip, uint32_t id, uint64_t open_window) {
  auto it = ip_to_id.find(ip);
  if (it != ip_to_id.end()) { if (it->second == id) return; Unmap(ip, open_window); }
  ip_to_id[ip] = id;
  refs[id]++;
}
void Aggregator::Interner::Unmap(uint32_t ip, uint64_t open_window) {
  auto it = ip_to_id.find(ip);
  if (it == ip_to_id.end()) return;
  const uint32_t id = it->second;
  ip_to_id.erase(it);
  // no IP resolves to the id any more: edges of the open window, and the retained entries and open blocks that
  // will cover it, may still carry it, so it is recycled later (a UID whose stale IP entry is still in the table
  // keeps its id, like the reference keeps the map entry: ADD/UPDATE never delete the old IP, persist.go:55-65)
  if (--refs[id] == 0) { unmapped_in[id] = open_window; pending_free.push_back(id); }
}
void Aggregator::Interner::EndWindow(uint64_t flushed, uint64_t hold, uint64_t pinned_from) {
  size_t keep = 0;
  for (uint32_t id : pending_free) {
    auto it = ids.find(names[id]);
    if (refs[id] != 0 || it == ids.end() || it->second != id) continue;   // mapped again, or freed already
    if (unmapped_in[id] + hold > flushed) { pending_free[keep++] = id; continue; }   // inside the retained span
    if (pinned_from && unmapped_in[id] >= pinned_from) { pending_free[keep++] = id; continue; }   // in the baseline
    ids.erase(it);
    free_ids.push_back(id);
    changes += 1;
  }
  pending_free.resize(keep);
  keep = 0;
  for (uint32_t id : held) {
    if (pinned_from && unmapped_in[id] >= pinned_from) held[keep++] = id;
    else { free_ids.push_back(id); changes += 1; }
  }
  held.resize(keep);
}
bool Aggregator::Interner::CanHold(uint64_t pinned_from) const {
  for (uint64_t r : reused_after)
    if (r >= pinned_from) return false;
  return true;
}
void Aggregator::Interner::Hold(uint64_t pinned_from) {
  size_t keep = 0;
  for (uint32_t id : free_ids) {
    if (unmapped_in[id] >= pinned_from) held.push_back(id);
    else free_ids[keep++] = id;
  }
  free_ids.resize(keep);
}

// processPod / processSvc: ADD and UPDATE write map[ip] = uid, DELETE removes (persist.go:55-71, 114-130)
void Aggregator::ProcessK8s(const K8sResourceMessage& m) {
  if (!h_) return;
  std::lock_guard<std::mutex> g(mu_);
  const bool pod = m.ResourceType == "Pod";
  if (!pod && m.ResourceType != "Service") return;   // other kinds are only relayed to the backend
  if (m.IP.empty()) return;                          // persist.go:37-40
  bool ok = false;
  const uint32_t ip = ParseIPv4(m.IP, &ok);
  if (!ok) return;                                   // e.g. ClusterIP "None"
  // events already batched were resolved by the reference with the tables as they were: submit first
  if (batch_n_) SubmitBatch();
  const int table = pod ? ALZ_TABLE_POD : ALZ_TABLE_SVC;
  Interner& in = pod ? pods_ : svcs_;
  if (m.EventType == "Add" || m.EventType == "Update") {
    const uint32_t id = in.Acquire(m.UID);
    const int rc = alz_table_upsert(h_, table, ip, id);
    if (rc != ALZ_OK) { err_ = std::string("alz_table_upsert: ") + alz_strerror(rc); return; }
    in.Map(ip, id, windows_ + 1);
  } else if (m.EventType == "Delete") {
    alz_table_erase(h_, table, ip);
    in.Unmap(ip, windows_ + 1);
  } else {
    return;
  }
  tables_dirty_ = true;
}

int Aggregator::SubmitBatch() {
  if (!h_) return ALZ_E_STATE;
  if (tables_dirty_) {
    const int rc = alz_table_commit(h_);
    if (rc != ALZ_OK) {   // events batched behind a failed commit are dropped, never left to pile up
      dropped_events_ += batch_n_;
      batch_n_ = 0;
      err_ = std::string("alz_table_commit: ") + alz_strerror(rc);
      return rc;
    }
    tables_dirty_ = false;
  }
  if (batch_n_ == 0) return ALZ_OK;
  const int rc = alz_submit_l7(h_, batch_, batch_n_);
  if (rc != ALZ_OK) { dropped_events_ += batch_n_; err_ = std::string("alz_submit_l7: ") + alz_strerror(rc); }
  batch_n_ = 0;   // the batch is gone either way: a failed submit must not let the buffer overrun
  return rc;
}

// the reader side of processL7: one compact record per event; the switch itself runs on the device
void Aggregator::ProcessL7(const L7Event& e) {
  if (!h_) return;
  std::lock_guard<std::mutex> g(mu_);
  if (tables_dirty_ || batch_n_ >= cfg_.BatchSize) SubmitBatch();   // table changes precede the events that follow them
  if (batch_n_ >= cfg_.BatchSize) return;                            // cannot happen (SubmitBatch empties the batch)
  alz_l7_rec& r = batch_[batch_n_++];
  r.saddr = e.Saddr; r.daddr = e.Daddr; r.sport = e.Sport; r.dport = e.Dport;
  r.status = e.Status > 65535u ? 65535u : (uint16_t)e.Status;
  r.protocol = ProtocolEnum(e.Protocol);
  r.method_flags = (uint8_t)((MethodEnum(r.protocol, e.Method) & ALZ_MF_METHOD_MASK) | (e.Tls ? ALZ_MF_TLS : 0) |
                             (e.PayloadRejected ? ALZ_MF_PAYLOAD_REJECT : 0));
  r.duration_ns = e.Duration;
  r.write_time_ns = e.WriteTimeNs;
  // setFromToV2's third-party branch (data.go:851-854): an HTTP destination that is neither service nor pod is
  // keyed by the request's Host header when there is one. The maps consulted are this adapter's mirror of the
  // tables it has upserted, in the same order as the events, so the decision is the reference's.
  if (r.protocol == ALZ_PROTO_HTTP && !e.Payload.empty() && !svcs_.ip_to_id.count(e.Daddr) && !pods_.ip_to_id.count(e.Daddr)) {
    const std::string host = ParseHttpHostHeader(e.Payload);
    if (!host.empty()) {
      bool is_ip = false;
      const uint32_t ip = ParseIPv4(host, &is_ip);
      if (is_ip) r.daddr = ip;   // a header that is itself a dotted quad is the same node as that raw daddr (same ToUID string)
      else {
        auto it = host_ids_.find(host);
        if (it == host_ids_.end()) { it = host_ids_.emplace(host, (uint32_t)host_names_.size()).first; host_names_.push_back(host); }
        r.daddr = it->second;
        r.protocol |= ALZ_PROTO_F_HOSTKEY;
      }
    }
  }
  if (batch_n_ >= cfg_.BatchSize) SubmitBatch();
}

void Aggregator::ProcessTcpConnect(const TcpConnectEvent& e) {
  if (!h_) return;
  alz_tcp_rec r;
  memset(&r, 0, sizeof r);
  r.fd = e.Fd; r.timestamp_ns = e.Timestamp; r.pid = e.Pid; r.sport = e.SPort; r.dport = e.DPort;
  r.saddr = ParseIPv4(e.SAddr, nullptr);
  r.daddr = ParseIPv4(e.DAddr, nullptr);
  // TcpStateConversion.String(), ebpf/tcp_state/tcp.go:27-60
  r.type = e.Type_ == "EVENT_TCP_ESTABLISHED" ? 1u : e.Type_ == "EVENT_TCP_CONNECT_FAILED" ? 2u
         : e.Type_ == "EVENT_TCP_LISTEN" ? 3u : e.Type_ == "EVENT_TCP_LISTEN_CLOSED" ? 4u
         : e.Type_ == "EVENT_TCP_CLOSED" ? 5u : 0u;
  alz_submit_tcp(h_, &r, 1);
}

int Aggregator::Flush(bool with_scores) {
  if (!h_) return ALZ_E_STATE;
  std::lock_guard<std::mutex> g(mu_);
  int rc = SubmitBatch();
  if (rc != ALZ_OK) return rc;
  size_t n = 0;
  rc = alz_window_flush(h_, out_.data(), out_.size(), &n);
  if (rc != ALZ_OK) return rc;
  if (with_scores && n) {
    scores_.resize(n);
    size_t ns = 0;
    rc = alz_gnn_score(h_, scores_.data(), n, &ns);
    if (rc != ALZ_OK) return rc;
  }
  std::vector<EdgeWindow> edges = ToEdges(out_.data(), n, with_scores ? scores_.data() : nullptr);
  windows_ += 1;
  pods_.EndWindow(windows_, hold_, pinned_from_);
  svcs_.EndWindow(windows_, hold_, pinned_from_);
  return ds_ ? ds_->PersistEdgeWindow(edges) : ALZ_OK;
}

std::string Aggregator::UidOf(uint8_t t, uint32_t v) const {
  if (t == ALZ_NODE_POD) return v < pods_.names.size() ? pods_.names[v] : std::string("?");
  if (t == ALZ_NODE_SVC) return v < svcs_.names.size() ? svcs_.names[v] : std::string("?");
  if (t == ALZ_NODE_OUTBOUND_HOST) return v < host_names_.size() ? host_names_[v] : std::string("?");   // data.go:852
  if (t == ALZ_NODE_GROUP) return v < group_names_.size() ? group_names_[v] : std::string("?");
  return FormatIPv4(v);   // outbound: the raw daddr string (data.go:862)
}

std::vector<EdgeWindow> Aggregator::ToEdges(const alz_edge_out* rows, size_t n, const float* scores) const {
  std::vector<EdgeWindow> edges(n);
  for (size_t i = 0; i < n; ++i) {
    const alz_edge_out& o = rows[i];
    EdgeWindow& w = edges[i];
    w.FromType = NodeTypeName(o.from_type); w.FromUID = UidOf(o.from_type, o.from);
    w.ToType = NodeTypeName(o.to_type);     w.ToUID = UidOf(o.to_type, o.to);
    w.Count = o.count; w.Err5xx = o.err5xx; w.LatSumNs = o.lat_sum_ns;
    memcpy(w.Hist, o.hist, sizeof w.Hist);
    if (scores) w.Score = scores[i];
  }
  return edges;
}

int Aggregator::Anomalies(uint32_t source, uint32_t k, float min_score, std::vector<EdgeWindow>* out,
                          alz_top_info* info) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  // into roll_ / scores_, grown once when the results do not fit (ALZ_E_CAPACITY with n = the results; nothing written)
  auto call = [&](size_t* n) {
    return source == kLastWindow
               ? alz_gnn_top(h_, k, min_score, roll_.data(), scores_.data(), nullptr, roll_.size(), n, info)
               : alz_gnn_top_rollup(h_, source, k, min_score, roll_.data(), scores_.data(), nullptr, roll_.size(), n,
                                    info);
  };
  size_t n = 0;
  scores_.resize(roll_.size());
  int rc = call(&n);
  if (rc == ALZ_E_CAPACITY && n > roll_.size()) {
    roll_.resize(n);
    scores_.resize(n);
    rc = call(&n);
  }
  if (rc != ALZ_OK) return rc;
  *out = ToEdges(roll_.data(), n, scores_.data());
  return ALZ_OK;
}

int Aggregator::EdgeMetrics(uint32_t source, const std::vector<alz_metric>& metrics, std::vector<double>* values) {
  if (!h_) return ALZ_E_STATE;
  if (!values) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  const uint32_t nm = (uint32_t)metrics.size();
  auto call = [&](double* v, size_t cap, size_t* n) {
    return source == kLastWindow ? alz_edge_metrics(h_, metrics.data(), nm, v, cap, n)
                                 : alz_edge_metrics_rollup(h_, source, metrics.data(), nm, v, cap, n);
  };
  size_t n = 0;
  int rc = call(nullptr, 0, &n);                 // the row count, then the values
  if (rc == ALZ_E_CAPACITY) {
    values->assign(n * nm, 0.0);
    rc = call(values->data(), n, &n);
  } else if (rc == ALZ_OK) {
    values->clear();
  }
  return rc;
}

int Aggregator::TopEdges(uint32_t source, const alz_metric& metric, uint32_t k, double min_value,
                         std::vector<EdgeWindow>* out, alz_top_info* info) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  // into roll_ / values_, grown once when the results do not fit (ALZ_E_CAPACITY with n = the results; nothing written)
  auto call = [&](size_t* n) {
    return source == kLastWindow
               ? alz_edge_top(h_, &metric, k, min_value, roll_.data(), values_.data(), nullptr, roll_.size(), n, info)
               : alz_edge_top_rollup(h_, source, &metric, k, min_value, roll_.data(), values_.data(), nullptr,
                                     roll_.size(), n, info);
  };
  size_t n = 0;
  values_.resize(roll_.size());
  int rc = call(&n);
  if (rc == ALZ_E_CAPACITY && n > roll_.size()) {
    roll_.resize(n);
    values_.resize(n);
    rc = call(&n);
  }
  if (rc != ALZ_OK) return rc;
  *out = ToEdges(roll_.data(), n, nullptr);
  for (size_t i = 0; i < n; ++i) (*out)[i].Value = values_[i];
  return ALZ_OK;
}

// An id unmapped while window u was open may be carried by windows u and later only (refs fell to 0 in u), so a
// baseline whose oldest window is w may carry exactly the ids unmapped in w or later, whether they are still pending,
// already free (taken back here) or already handed to another UID (the pin is refused).
int Aggregator::PinBaseline(uint32_t source, alz_rollup_info* info) {
  if (!h_) return ALZ_E_STATE;
  std::lock_guard<std::mutex> g(mu_);
  alz_rollup_info ri{};
  int rc = alz_baseline_pin(h_, source, &ri);
  if (rc != ALZ_OK) return rc;   // an earlier baseline, if any, is still pinned and its hold stays
  // alz_stats.windows counts the handle's flushes, which are this adapter's (Flush); an empty window history pins
  // window_first = 0, which holds every id freed from window 1 on
  const uint64_t from = std::max<uint64_t>(ri.window_first, 1);
  if (!pods_.CanHold(from) || !svcs_.CanHold(from)) {
    err_ = "PinBaseline: an id the source may carry has gone to another UID";
    rc = alz_baseline_clear(h_);
    pinned_from_ = 0;
    pods_.EndWindow(windows_, hold_, 0);
    svcs_.EndWindow(windows_, hold_, 0);
    return rc != ALZ_OK ? rc : ALZ_E_STATE;
  }
  if (info) *info = ri;
  pinned_from_ = from;
  pods_.EndWindow(windows_, hold_, pinned_from_);   // the previous baseline's hold goes now
  svcs_.EndWindow(windows_, hold_, pinned_from_);
  pods_.Hold(pinned_from_);                         // and ids already free that this one may carry come back
  svcs_.Hold(pinned_from_);
  return ALZ_OK;
}

int Aggregator::ClearBaseline() {
  if (!h_) return ALZ_E_STATE;
  std::lock_guard<std::mutex> g(mu_);
  const int rc = alz_baseline_clear(h_);
  if (rc != ALZ_OK) return rc;
  pinned_from_ = 0;
  pods_.EndWindow(windows_, hold_, 0);
  svcs_.EndWindow(windows_, hold_, 0);
  return ALZ_OK;
}

template <class Rec, class Call>
int Aggregator::RunChanges(std::vector<Rec>* recs, size_t* n, Call call) {
  int rc = call(recs->data(), recs->size(), n);
  if (rc == ALZ_E_CAPACITY && *n > recs->size()) {
    recs->resize(*n);
    rc = call(recs->data(), recs->size(), n);
  }
  return rc;
}

int Aggregator::Changes(uint32_t source, const alz_metric& metric, uint32_t mode, uint32_t presence, uint32_t k,
                        double min_change, std::vector<EdgeChange>* out, alz_change_info* info) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  size_t n = 0;
  const int rc = RunChanges(&changes_, &n, [&](alz_edge_change* recs, size_t cap, size_t* n_out) {
    return k == 0 ? alz_edge_changes(h_, source, &metric, mode, presence, recs, cap, n_out, info)
                  : alz_edge_changes_top(h_, source, &metric, mode, presence, k, min_change, recs, cap, n_out, info);
  });
  if (rc != ALZ_OK) return rc;
  *out = ToChanges(changes_.data(), n);
  return ALZ_OK;
}

std::vector<EdgeChange> Aggregator::ToChanges(const alz_edge_change* recs, size_t n) const {
  std::vector<EdgeChange> out(n);
  for (size_t i = 0; i < n; ++i) {
    const alz_edge_change& c = recs[i];
    alz_edge_out row{};
    row.from_type = c.from_type; row.to_type = c.to_type; row.from = c.from; row.to = c.to;
    const EdgeWindow w = ToEdges(&row, 1, nullptr)[0];
    EdgeChange& e = out[i];
    e.FromType = w.FromType; e.FromUID = w.FromUID; e.ToType = w.ToType; e.ToUID = w.ToUID;
    e.Presence = c.presence; e.Value = c.value; e.BaseValue = c.base_value; e.Change = c.change;
  }
  return out;
}

bool Aggregator::EndOf(const std::string& type, const std::string& uid, uint8_t* t, uint32_t* v) const {
  if (type == "pod" || type == "service") {
    const Interner& in = type == "pod" ? pods_ : svcs_;
    const auto it = in.ids.find(uid);
    if (it == in.ids.end()) return false;
    *t = type == "pod" ? ALZ_NODE_POD : ALZ_NODE_SVC;
    *v = it->second;
    return true;
  }
  if (type != "outbound") return false;
  bool ok = false;
  const uint32_t ip = ParseIPv4(uid, &ok);
  if (ok) { *t = ALZ_NODE_OUTBOUND; *v = ip; return true; }
  const auto it = host_ids_.find(uid);   // a destination keyed by its Host header (data.go:851-854)
  if (it == host_ids_.end()) return false;
  *t = ALZ_NODE_OUTBOUND_HOST;
  *v = it->second;
  return true;
}

bool Aggregator::ToEnds(const EdgeRef& e, alz_edge_ends* out) const {
  *out = alz_edge_ends{};
  return EndOf(e.FromType, e.FromUID, &out->from_type, &out->from) && EndOf(e.ToType, e.ToUID, &out->to_type, &out->to);
}

template <class Row, class Call>
int Aggregator::RunSeries(size_t nm, std::vector<Row>* out, std::vector<alz_rollup_info>* points, Call call) {
  size_t n = 0;
  uint32_t P = 0;
  int rc = call(nullptr, nullptr, 0, &n, &P, nullptr);   // the sizes, then the values
  if (rc != ALZ_OK && rc != ALZ_E_CAPACITY) return rc;
  series_values_.assign(n * P * nm, 0.0);
  series_present_.assign(n * P, 0);
  std::vector<alz_rollup_info> pts(P);
  rc = call(series_values_.data(), series_present_.data(), n, &n, &P, pts.data());
  if (rc != ALZ_OK) return rc;
  out->assign(n, Row{});
  for (size_t i = 0; i < n; ++i) {
    (*out)[i].Present.assign(series_present_.begin() + i * P, series_present_.begin() + (i + 1) * P);
    (*out)[i].Values.assign(series_values_.begin() + i * P * nm, series_values_.begin() + (i + 1) * P * nm);
  }
  if (points) *points = pts;
  return ALZ_OK;
}

int Aggregator::Series(uint32_t source, uint32_t tier, uint32_t k, const std::vector<alz_metric>& metrics,
                       std::vector<EdgeSeries>* out, std::vector<alz_rollup_info>* points) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  const uint32_t nm = (uint32_t)metrics.size();
  int rc = RunSeries(nm, out, points, [&](double* v, uint8_t* p, size_t cap, size_t* n, uint32_t* P,
                                          alz_rollup_info* pts) {
    return alz_edge_series(h_, source == kLastWindow ? ALZ_SOURCE_WINDOW : source, tier, k, metrics.data(), nm, v, p,
                           cap, n, P, pts, nullptr);
  });
  if (rc != ALZ_OK) return rc;
  // the names: the source's rows in its row order, from its top list by count with every row eligible and each
  // row's index (no other call returns a rollup's held rows)
  const size_t n = out->size();
  if (n == 0) return ALZ_OK;
  std::vector<alz_edge_out> ranked(n), rows(n);
  std::vector<uint32_t> index(n);
  const alz_metric count{ALZ_METRIC_COUNT, 0, 0.0};
  const double all = -HUGE_VAL;
  size_t m = 0;
  rc = source == kLastWindow
           ? alz_edge_top(h_, &count, (uint32_t)n, all, ranked.data(), nullptr, index.data(), n, &m, nullptr)
           : alz_edge_top_rollup(h_, source, &count, (uint32_t)n, all, ranked.data(), nullptr, index.data(), n, &m,
                                 nullptr);
  if (rc != ALZ_OK) return rc;
  if (m != n) return ALZ_E_STATE;
  for (size_t j = 0; j < n; ++j) rows[index[j]] = ranked[j];
  const std::vector<EdgeWindow> names = ToEdges(rows.data(), n, nullptr);
  for (size_t i = 0; i < n; ++i) {
    EdgeSeries& e = (*out)[i];
    e.FromType = names[i].FromType; e.FromUID = names[i].FromUID; e.ToType = names[i].ToType; e.ToUID = names[i].ToUID;
  }
  return ALZ_OK;
}

int Aggregator::SeriesFor(const std::vector<EdgeRef>& edges, uint32_t tier, uint32_t k,
                          const std::vector<alz_metric>& metrics, std::vector<EdgeSeries>* out,
                          std::vector<alz_rollup_info>* points) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  // the edges with ids go to the library; the others are absent at every point
  std::vector<alz_edge_ends> keys;
  std::vector<size_t> row_of;   // edge -> row of keys, or SIZE_MAX
  for (const EdgeRef& e : edges) {
    alz_edge_ends k_{};
    if (ToEnds(e, &k_)) { row_of.push_back(keys.size()); keys.push_back(k_); }
    else row_of.push_back(SIZE_MAX);
  }
  const uint32_t nm = (uint32_t)metrics.size();
  std::vector<EdgeSeries> known;
  std::vector<alz_rollup_info> pts;
  const int rc = RunSeries(nm, &known, &pts, [&](double* v, uint8_t* p, size_t cap, size_t* n, uint32_t* P,
                                                 alz_rollup_info* pp) {
    return alz_edge_series_keys(h_, keys.data(), keys.size(), tier, k, metrics.data(), nm, v, p, cap, n, P, pp,
                                nullptr);
  });
  if (rc != ALZ_OK) return rc;
  const size_t P = pts.size();
  out->assign(edges.size(), EdgeSeries{});
  for (size_t i = 0; i < edges.size(); ++i) {
    EdgeSeries& e = (*out)[i];
    if (row_of[i] != SIZE_MAX) e = known[row_of[i]];
    else { e.Present.assign(P, 0); e.Values.assign(P * nm, 0.0); }
    e.FromType = edges[i].FromType; e.FromUID = edges[i].FromUID; e.ToType = edges[i].ToType; e.ToUID = edges[i].ToUID;
  }
  if (points) *points = pts;
  return ALZ_OK;
}

int Aggregator::Trends(uint32_t source, uint32_t tier, uint32_t k, const alz_metric& metric, const alz_trend& trend,
                       uint32_t top, double min_trend, std::vector<EdgeTrend>* out,
                       std::vector<alz_rollup_info>* points) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  return RunEdgeTrends(alz_edge_trends_top, source, tier, k, metric, trend, top, min_trend, out, points);
}

int Aggregator::RunEdgeTrends(EdgeTrendsTop fn, uint32_t source, uint32_t tier, uint32_t k, const alz_metric& metric,
                              const alz_trend& trend, uint32_t top, double min_trend, std::vector<EdgeTrend>* out,
                              std::vector<alz_rollup_info>* points) {
  const uint32_t src = source == kLastWindow ? ALZ_SOURCE_WINDOW : source;
  // a first call sizes the results (ALZ_E_CAPACITY with n = the results, P = the points; nothing written)
  size_t n = 0;
  uint32_t P = 0;
  int rc = fn(h_, src, tier, k, &metric, &trend, top, min_trend, nullptr, nullptr, nullptr, nullptr, 0, &n, &P,
              nullptr, nullptr);
  std::vector<alz_rollup_info> pts(P);
  if (rc == ALZ_E_CAPACITY && n > 0) {
    trends_.resize(n);
    trend_rows_.resize(n);
    trend_values_.resize(n * P);
    trend_present_.resize(n * P);
    rc = fn(h_, src, tier, k, &metric, &trend, top, min_trend, trends_.data(), trend_rows_.data(),
            trend_values_.data(), trend_present_.data(), n, &n, &P, pts.data(), nullptr);
  }
  if (rc != ALZ_OK) return rc;
  const std::vector<EdgeWindow> names = ToEdges(trend_rows_.data(), n, nullptr);
  out->assign(n, EdgeTrend{});
  for (size_t i = 0; i < n; ++i) {
    const alz_edge_trend& r = trends_[i];
    EdgeTrend& e = (*out)[i];
    e.FromType = names[i].FromType; e.FromUID = names[i].FromUID; e.ToType = names[i].ToType; e.ToUID = names[i].ToUID;
    e.Valid = r.valid != 0;
    e.Used = r.used;
    e.Trend = r.trend; e.Recent = r.recent; e.Before = r.before;
    e.Present.assign(trend_present_.begin() + i * P, trend_present_.begin() + (i + 1) * P);
    e.Values.assign(trend_values_.begin() + i * P, trend_values_.begin() + (i + 1) * P);
  }
  if (points) *points = pts;
  return ALZ_OK;
}

std::vector<NodeWindow> Aggregator::ToNodes(const alz_node_out* rows, size_t n, const double* values,
                                            size_t nm) const {
  std::vector<NodeWindow> nodes(n);
  for (size_t i = 0; i < n; ++i) {
    const alz_node_out& o = rows[i];
    NodeWindow& w = nodes[i];
    w.Type = NodeTypeName(o.type);
    w.UID = UidOf(o.type, o.value);
    w.InEdges = o.in_edges;
    w.OutEdges = o.out_edges;
    w.In = o.in;
    w.Out = o.out;
    if (values) w.Values.assign(values + i * nm, values + (i + 1) * nm);
  }
  return nodes;
}

int Aggregator::Nodes(uint32_t source, uint32_t side, const std::vector<alz_metric>& metrics,
                      std::vector<NodeWindow>* out) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  const uint32_t src = source == kLastWindow ? ALZ_SOURCE_WINDOW : source;
  const uint32_t nm = (uint32_t)metrics.size();
  // the node count (ALZ_E_CAPACITY with n = the nodes; nothing written), then the rows and the values
  size_t n = 0;
  int rc = alz_node_rows(h_, src, nullptr, 0, &n);
  if (rc == ALZ_E_CAPACITY) {
    nodes_.resize(n);
    rc = alz_node_rows(h_, src, nodes_.data(), n, &n);
  }
  if (rc != ALZ_OK) return rc;
  node_values_.assign(n * nm, 0.0);
  size_t nv = 0;
  rc = alz_node_metrics(h_, src, side, metrics.data(), nm, node_values_.data(), n, &nv);
  if (rc != ALZ_OK) return rc;
  if (nv != n) return ALZ_E_STATE;
  *out = ToNodes(nodes_.data(), n, node_values_.data(), nm);
  return ALZ_OK;
}

int Aggregator::NodeChanges(uint32_t source, uint32_t side, const alz_metric& metric, uint32_t mode,
                            uint32_t presence, uint32_t k, double min_change, std::vector<NodeChange>* out,
                            alz_change_info* info) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  const uint32_t src = source == kLastWindow ? ALZ_SOURCE_WINDOW : source;
  size_t n = 0;
  const int rc = RunChanges(&node_changes_, &n, [&](alz_node_change* recs, size_t cap, size_t* n_out) {
    return k == 0 ? alz_node_changes(h_, src, side, &metric, mode, presence, recs, cap, n_out, info)
                  : alz_node_changes_top(h_, src, side, &metric, mode, presence, k, min_change, recs, cap, n_out, info);
  });
  if (rc != ALZ_OK) return rc;
  *out = ToNodeChanges(node_changes_.data(), n);
  return ALZ_OK;
}

std::vector<NodeChange> Aggregator::ToNodeChanges(const alz_node_change* recs, size_t n) const {
  std::vector<NodeChange> out(n);
  for (size_t i = 0; i < n; ++i) {
    const alz_node_change& c = recs[i];
    NodeChange& e = out[i];
    e.Type = NodeTypeName(c.type);
    e.UID = UidOf(c.type, c.node);
    e.Presence = c.presence; e.Value = c.value; e.BaseValue = c.base_value; e.Change = c.change;
  }
  return out;
}

int Aggregator::TopNodes(uint32_t source, uint32_t side, const alz_metric& metric, uint32_t k, double min_value,
                         std::vector<NodeWindow>* out, alz_top_info* info) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  const uint32_t src = source == kLastWindow ? ALZ_SOURCE_WINDOW : source;
  // into nodes_ / node_values_, grown once when the results do not fit (ALZ_E_CAPACITY with n = the results)
  auto call = [&](size_t* n) {
    return alz_node_top(h_, src, side, &metric, k, min_value, nodes_.data(), node_values_.data(), nullptr,
                        nodes_.size(), n, info);
  };
  size_t n = 0;
  node_values_.resize(nodes_.size());
  int rc = call(&n);
  if (rc == ALZ_E_CAPACITY && n > nodes_.size()) {
    nodes_.resize(n);
    node_values_.resize(n);
    rc = call(&n);
  }
  if (rc != ALZ_OK) return rc;
  *out = ToNodes(nodes_.data(), n, node_values_.data(), 1);
  return ALZ_OK;
}

int Aggregator::SetGroups(const std::vector<GroupMember>& members) {
  if (!h_) return ALZ_E_STATE;
  std::lock_guard<std::mutex> g(mu_);
  members_ = members;
  for (const GroupMember& m : members_) {
    if (group_ids_.count(m.Group)) continue;
    if (group_names_.size() >= (1u << 29)) return ALZ_E_CAPACITY;
    group_ids_.emplace(m.Group, (uint32_t)group_names_.size());
    group_names_.push_back(m.Group);
  }
  groups_sent_ = false;
  return ALZ_OK;
}

int Aggregator::SyncGroups() {
  const uint64_t changes = pods_.changes + svcs_.changes + host_names_.size();
  if (groups_sent_ && changes == groups_changes_) return ALZ_OK;
  std::vector<alz_node_ends> nodes;
  std::vector<uint32_t> groups;
  std::unordered_map<uint64_t, bool> seen;
  for (const GroupMember& m : members_) {
    alz_node_ends e{};
    if (!EndOf(m.Type, m.UID, &e.type, &e.value)) continue;   // no id now: not in any row the library holds
    if (!seen.emplace(((uint64_t)e.type << 32) | e.value, true).second) continue;
    nodes.push_back(e);
    groups.push_back(group_ids_.at(m.Group));
  }
  const int rc = alz_group_set(h_, nodes.data(), groups.data(), nodes.size());
  if (rc != ALZ_OK) return rc;
  groups_sent_ = true;
  groups_changes_ = changes;
  return ALZ_OK;
}

int Aggregator::GroupEdges(uint32_t source, std::vector<EdgeWindow>* out, alz_group_info* info) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  int rc = SyncGroups();
  if (rc != ALZ_OK) return rc;
  const uint32_t src = source == kLastWindow ? ALZ_SOURCE_WINDOW : source;
  // into roll_, grown once when the rows do not fit (ALZ_E_CAPACITY with n = the rows; nothing written)
  size_t n = 0;
  rc = alz_group_edges(h_, src, roll_.data(), roll_.size(), &n, info);
  if (rc == ALZ_E_CAPACITY && n > roll_.size()) {
    roll_.resize(n);
    rc = alz_group_edges(h_, src, roll_.data(), roll_.size(), &n, info);
  }
  if (rc != ALZ_OK) return rc;
  *out = ToEdges(roll_.data(), n, nullptr);
  return ALZ_OK;
}

int Aggregator::GroupNodes(uint32_t source, uint32_t side, const std::vector<alz_metric>& metrics,
                           std::vector<NodeWindow>* out) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  int rc = SyncGroups();
  if (rc != ALZ_OK) return rc;
  const uint32_t src = source == kLastWindow ? ALZ_SOURCE_WINDOW : source;
  const uint32_t nm = (uint32_t)metrics.size();
  // the node count (ALZ_E_CAPACITY with n = the nodes; nothing written), then the rows and the values
  size_t n = 0;
  rc = alz_group_nodes(h_, src, nullptr, 0, &n);
  if (rc == ALZ_E_CAPACITY) {
    nodes_.resize(n);
    rc = alz_group_nodes(h_, src, nodes_.data(), n, &n);
  }
  if (rc != ALZ_OK) return rc;
  node_values_.assign(n * nm, 0.0);
  size_t nv = 0;
  rc = alz_group_node_metrics(h_, src, side, metrics.data(), nm, node_values_.data(), n, &nv);
  if (rc != ALZ_OK) return rc;
  if (nv != n) return ALZ_E_STATE;
  *out = ToNodes(nodes_.data(), n, node_values_.data(), nm);
  return ALZ_OK;
}

int Aggregator::TopGroupNodes(uint32_t source, uint32_t side, const alz_metric& metric, uint32_t k, double min_value,
                              std::vector<NodeWindow>* out, alz_top_info* info) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  int rc = SyncGroups();
  if (rc != ALZ_OK) return rc;
  const uint32_t src = source == kLastWindow ? ALZ_SOURCE_WINDOW : source;
  // into nodes_ / node_values_, grown once when the results do not fit (ALZ_E_CAPACITY with n = the results)
  auto call = [&](size_t* n) {
    return alz_group_node_top(h_, src, side, &metric, k, min_value, nodes_.data(), node_values_.data(), nullptr,
                              nodes_.size(), n, info);
  };
  size_t n = 0;
  node_values_.resize(nodes_.size());
  rc = call(&n);
  if (rc == ALZ_E_CAPACITY && n > nodes_.size()) {
    nodes_.resize(n);
    node_values_.resize(n);
    rc = call(&n);
  }
  if (rc != ALZ_OK) return rc;
  *out = ToNodes(nodes_.data(), n, node_values_.data(), 1);
  return ALZ_OK;
}

int Aggregator::GroupChanges(uint32_t source, const alz_metric& metric, uint32_t mode, uint32_t presence, uint32_t k,
                             double min_change, std::vector<EdgeChange>* out, alz_change_info* info) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  int rc = SyncGroups();
  if (rc != ALZ_OK) return rc;
  const uint32_t src = source == kLastWindow ? ALZ_SOURCE_WINDOW : source;
  size_t n = 0;
  rc = RunChanges(&changes_, &n, [&](alz_edge_change* recs, size_t cap, size_t* n_out) {
    return k == 0 ? alz_group_edge_changes(h_, src, &metric, mode, presence, recs, cap, n_out, info)
                  : alz_group_edge_changes_top(h_, src, &metric, mode, presence, k, min_change, recs, cap, n_out, info);
  });
  if (rc != ALZ_OK) return rc;
  *out = ToChanges(changes_.data(), n);
  return ALZ_OK;
}

int Aggregator::GroupNodeChanges(uint32_t source, uint32_t side, const alz_metric& metric, uint32_t mode,
                                 uint32_t presence, uint32_t k, double min_change, std::vector<NodeChange>* out,
                                 alz_change_info* info) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  int rc = SyncGroups();
  if (rc != ALZ_OK) return rc;
  const uint32_t src = source == kLastWindow ? ALZ_SOURCE_WINDOW : source;
  size_t n = 0;
  rc = RunChanges(&node_changes_, &n, [&](alz_node_change* recs, size_t cap, size_t* n_out) {
    return k == 0 ? alz_group_node_changes(h_, src, side, &metric, mode, presence, recs, cap, n_out, info)
                  : alz_group_node_changes_top(h_, src, side, &metric, mode, presence, k, min_change, recs, cap,
                                               n_out, info);
  });
  if (rc != ALZ_OK) return rc;
  *out = ToNodeChanges(node_changes_.data(), n);
  return ALZ_OK;
}

int Aggregator::NodeSeries(uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                           const std::vector<alz_metric>& metrics, std::vector<NodeSeriesRow>* out,
                           std::vector<alz_rollup_info>* points) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  const uint32_t src = source == kLastWindow ? ALZ_SOURCE_WINDOW : source;
  const uint32_t nm = (uint32_t)metrics.size();
  int rc = RunSeries(nm, out, points, [&](double* v, uint8_t* p, size_t cap, size_t* n, uint32_t* P,
                                          alz_rollup_info* pts) {
    return alz_node_series(h_, src, side, tier, k, metrics.data(), nm, v, p, cap, n, P, pts, nullptr);
  });
  if (rc != ALZ_OK) return rc;
  // the names: the source's node rows, in the same node order
  const size_t n = out->size();
  if (n == 0) return ALZ_OK;
  nodes_.resize(n);
  size_t m = 0;
  rc = alz_node_rows(h_, src, nodes_.data(), n, &m);
  if (rc != ALZ_OK) return rc;
  if (m != n) return ALZ_E_STATE;
  for (size_t i = 0; i < n; ++i) {
    (*out)[i].Type = NodeTypeName(nodes_[i].type);
    (*out)[i].UID = UidOf(nodes_[i].type, nodes_[i].value);
  }
  return ALZ_OK;
}

int Aggregator::NodeSeriesFor(const std::vector<NodeRef>& nodes, uint32_t side, uint32_t tier, uint32_t k,
                              const std::vector<alz_metric>& metrics, std::vector<NodeSeriesRow>* out,
                              std::vector<alz_rollup_info>* points) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  // the nodes with ids go to the library; the others are absent at every point
  std::vector<alz_node_ends> keys;
  std::vector<size_t> row_of;   // node -> row of keys, or SIZE_MAX
  for (const NodeRef& r : nodes) {
    alz_node_ends k_{};
    if (EndOf(r.Type, r.UID, &k_.type, &k_.value)) { row_of.push_back(keys.size()); keys.push_back(k_); }
    else row_of.push_back(SIZE_MAX);
  }
  const uint32_t nm = (uint32_t)metrics.size();
  std::vector<NodeSeriesRow> known;
  std::vector<alz_rollup_info> pts;
  const int rc = RunSeries(nm, &known, &pts, [&](double* v, uint8_t* p, size_t cap, size_t* n, uint32_t* P,
                                                 alz_rollup_info* pp) {
    return alz_node_series_keys(h_, keys.data(), keys.size(), side, tier, k, metrics.data(), nm, v, p, cap, n, P, pp,
                                nullptr);
  });
  if (rc != ALZ_OK) return rc;
  const size_t P = pts.size();
  out->assign(nodes.size(), NodeSeriesRow{});
  for (size_t i = 0; i < nodes.size(); ++i) {
    NodeSeriesRow& e = (*out)[i];
    if (row_of[i] != SIZE_MAX) e = known[row_of[i]];
    else { e.Present.assign(P, 0); e.Values.assign(P * nm, 0.0); }
    e.Type = nodes[i].Type;
    e.UID = nodes[i].UID;
  }
  if (points) *points = pts;
  return ALZ_OK;
}

int Aggregator::NodeTrends(uint32_t source, uint32_t side, uint32_t tier, uint32_t k, const alz_metric& metric,
                           const alz_trend& trend, uint32_t top, double min_trend, std::vector<NodeTrend>* out,
                           std::vector<alz_rollup_info>* points) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  return RunNodeTrends(alz_node_trends_top, source, side, tier, k, metric, trend, top, min_trend, out, points);
}

int Aggregator::RunNodeTrends(NodeTrendsTop fn, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                              const alz_metric& metric, const alz_trend& trend, uint32_t top, double min_trend,
                              std::vector<NodeTrend>* out, std::vector<alz_rollup_info>* points) {
  const uint32_t src = source == kLastWindow ? ALZ_SOURCE_WINDOW : source;
  // a first call sizes the results (ALZ_E_CAPACITY with n = the results, P = the points; nothing written)
  size_t n = 0;
  uint32_t P = 0;
  int rc = fn(h_, src, side, tier, k, &metric, &trend, top, min_trend, nullptr, nullptr, nullptr, nullptr, 0, &n,
              &P, nullptr, nullptr);
  std::vector<alz_rollup_info> pts(P);
  if (rc == ALZ_E_CAPACITY && n > 0) {
    node_trends_.resize(n);
    node_trend_rows_.resize(n);
    trend_values_.resize(n * P);
    trend_present_.resize(n * P);
    rc = fn(h_, src, side, tier, k, &metric, &trend, top, min_trend, node_trends_.data(), node_trend_rows_.data(),
            trend_values_.data(), trend_present_.data(), n, &n, &P, pts.data(), nullptr);
  }
  if (rc != ALZ_OK) return rc;
  const std::vector<NodeWindow> names = ToNodes(node_trend_rows_.data(), n, nullptr, 0);
  out->assign(n, NodeTrend{});
  for (size_t i = 0; i < n; ++i) {
    const alz_node_trend& r = node_trends_[i];
    NodeTrend& e = (*out)[i];
    e.Node = names[i];
    e.Valid = r.valid != 0;
    e.Used = r.used;
    e.Trend = r.trend; e.Recent = r.recent; e.Before = r.before;
    e.Present.assign(trend_present_.begin() + i * P, trend_present_.begin() + (i + 1) * P);
    e.Values.assign(trend_values_.begin() + i * P, trend_values_.begin() + (i + 1) * P);
  }
  if (points) *points = pts;
  return ALZ_OK;
}

bool Aggregator::GroupEndOf(const std::string& type, const std::string& uid, uint8_t* t, uint32_t* v) const {
  if (type != "group") return EndOf(type, uid, t, v);
  const auto it = group_ids_.find(uid);
  if (it == group_ids_.end()) return false;
  *t = ALZ_NODE_GROUP;
  *v = it->second;
  return true;
}

int Aggregator::GroupSeries(uint32_t source, uint32_t tier, uint32_t k, const std::vector<alz_metric>& metrics,
                            std::vector<EdgeSeries>* out, std::vector<alz_rollup_info>* points) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  int rc = SyncGroups();
  if (rc != ALZ_OK) return rc;
  const uint32_t src = source == kLastWindow ? ALZ_SOURCE_WINDOW : source;
  const uint32_t nm = (uint32_t)metrics.size();
  rc = RunSeries(nm, out, points, [&](double* v, uint8_t* p, size_t cap, size_t* n, uint32_t* P,
                                      alz_rollup_info* pts) {
    return alz_group_edge_series(h_, src, tier, k, metrics.data(), nm, v, p, cap, n, P, pts, nullptr);
  });
  if (rc != ALZ_OK) return rc;
  // the names: the source's group-edge rows, in the same order
  const size_t n = out->size();
  if (n == 0) return ALZ_OK;
  roll_.resize(n);
  size_t m = 0;
  rc = alz_group_edges(h_, src, roll_.data(), n, &m, nullptr);
  if (rc != ALZ_OK) return rc;
  if (m != n) return ALZ_E_STATE;
  const std::vector<EdgeWindow> names = ToEdges(roll_.data(), n, nullptr);
  for (size_t i = 0; i < n; ++i) {
    EdgeSeries& e = (*out)[i];
    e.FromType = names[i].FromType; e.FromUID = names[i].FromUID; e.ToType = names[i].ToType; e.ToUID = names[i].ToUID;
  }
  return ALZ_OK;
}

int Aggregator::GroupSeriesFor(const std::vector<EdgeRef>& edges, uint32_t tier, uint32_t k,
                               const std::vector<alz_metric>& metrics, std::vector<EdgeSeries>* out,
                               std::vector<alz_rollup_info>* points) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  int rc = SyncGroups();
  if (rc != ALZ_OK) return rc;
  // the edges whose ends resolve go to the library; the others are absent at every point
  std::vector<alz_edge_ends> keys;
  std::vector<size_t> row_of;   // edge -> row of keys, or SIZE_MAX
  for (const EdgeRef& e : edges) {
    alz_edge_ends k_{};
    if (GroupEndOf(e.FromType, e.FromUID, &k_.from_type, &k_.from) &&
        GroupEndOf(e.ToType, e.ToUID, &k_.to_type, &k_.to)) {
      row_of.push_back(keys.size());
      keys.push_back(k_);
    } else {
      row_of.push_back(SIZE_MAX);
    }
  }
  const uint32_t nm = (uint32_t)metrics.size();
  std::vector<EdgeSeries> known;
  std::vector<alz_rollup_info> pts;
  rc = RunSeries(nm, &known, &pts, [&](double* v, uint8_t* p, size_t cap, size_t* n, uint32_t* P,
                                       alz_rollup_info* pp) {
    return alz_group_edge_series_keys(h_, keys.data(), keys.size(), tier, k, metrics.data(), nm, v, p, cap, n, P, pp,
                                      nullptr);
  });
  if (rc != ALZ_OK) return rc;
  const size_t P = pts.size();
  out->assign(edges.size(), EdgeSeries{});
  for (size_t i = 0; i < edges.size(); ++i) {
    EdgeSeries& e = (*out)[i];
    if (row_of[i] != SIZE_MAX) e = known[row_of[i]];
    else { e.Present.assign(P, 0); e.Values.assign(P * nm, 0.0); }
    e.FromType = edges[i].FromType; e.FromUID = edges[i].FromUID; e.ToType = edges[i].ToType; e.ToUID = edges[i].ToUID;
  }
  if (points) *points = pts;
  return ALZ_OK;
}

int Aggregator::GroupNodeSeries(uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                const std::vector<alz_metric>& metrics, std::vector<NodeSeriesRow>* out,
                                std::vector<alz_rollup_info>* points) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  int rc = SyncGroups();
  if (rc != ALZ_OK) return rc;
  const uint32_t src = source == kLastWindow ? ALZ_SOURCE_WINDOW : source;
  const uint32_t nm = (uint32_t)metrics.size();
  rc = RunSeries(nm, out, points, [&](double* v, uint8_t* p, size_t cap, size_t* n, uint32_t* P,
                                      alz_rollup_info* pts) {
    return alz_group_node_series(h_, src, side, tier, k, metrics.data(), nm, v, p, cap, n, P, pts, nullptr);
  });
  if (rc != ALZ_OK) return rc;
  // the names: the source's group nodes, in the same node order
  const size_t n = out->size();
  if (n == 0) return ALZ_OK;
  nodes_.resize(n);
  size_t m = 0;
  rc = alz_group_nodes(h_, src, nodes_.data(), n, &m);
  if (rc != ALZ_OK) return rc;
  if (m != n) return ALZ_E_STATE;
  for (size_t i = 0; i < n; ++i) {
    (*out)[i].Type = NodeTypeName(nodes_[i].type);
    (*out)[i].UID = UidOf(nodes_[i].type, nodes_[i].value);
  }
  return ALZ_OK;
}

int Aggregator::Reach(uint32_t source, const std::vector<NodeRef>& seeds, uint32_t dir, uint32_t max_hops,
                      const alz_metric* filter, double min_value, std::vector<ReachNode>* nodes,
                      std::vector<EdgeWindow>* rows, alz_reach_info* info) {
  return RunReach(false, source, seeds, dir, max_hops, filter, min_value, nodes, rows, info);
}

int Aggregator::GroupReach(uint32_t source, const std::vector<NodeRef>& seeds, uint32_t dir, uint32_t max_hops,
                           const alz_metric* filter, double min_value, std::vector<ReachNode>* nodes,
                           std::vector<EdgeWindow>* rows, alz_reach_info* info) {
  return RunReach(true, source, seeds, dir, max_hops, filter, min_value, nodes, rows, info);
}

int Aggregator::RunReach(bool group, uint32_t source, const std::vector<NodeRef>& seeds, uint32_t dir,
                         uint32_t max_hops, const alz_metric* filter, double min_value,
                         std::vector<ReachNode>* nodes, std::vector<EdgeWindow>* rows, alz_reach_info* info) {
  if (!h_) return ALZ_E_STATE;
  if (!nodes || !rows) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  if (info) *info = alz_reach_info{};
  nodes->clear();
  rows->clear();
  if (group) {
    const int rc = SyncGroups();
    if (rc != ALZ_OK) return rc;
  }
  std::vector<alz_node_ends> keys;
  for (const NodeRef& r : seeds) {
    alz_node_ends k_{};
    if (group ? GroupEndOf(r.Type, r.UID, &k_.type, &k_.value) : EndOf(r.Type, r.UID, &k_.type, &k_.value))
      keys.push_back(k_);
  }
  if (keys.empty()) return ALZ_OK;
  const uint32_t src = source == kLastWindow ? ALZ_SOURCE_WINDOW : source;
  // never empty: a null array would not be written (and its cap not checked)
  if (reach_nodes_.empty()) reach_nodes_.resize(1);
  if (reach_index_.empty()) reach_index_.resize(1);
  if (roll_.empty()) roll_.resize(1);
  auto call = [&](size_t* nn, size_t* nr) {
    return (group ? alz_group_reach : alz_reach)(h_, src, keys.data(), keys.size(), dir, max_hops, filter, min_value,
                                                 reach_nodes_.data(), reach_nodes_.size(), nn, reach_index_.data(),
                                                 roll_.data(), std::min(reach_index_.size(), roll_.size()), nr, info);
  };
  // into reach_nodes_ / reach_index_ / roll_, grown once when the results do not fit (ALZ_E_CAPACITY with the counts
  // set; nothing written)
  size_t nn = 0, nr = 0;
  int rc = call(&nn, &nr);
  if (rc == ALZ_E_CAPACITY && (nn > reach_nodes_.size() || nr > reach_index_.size() || nr > roll_.size())) {
    reach_nodes_.resize(std::max(nn, reach_nodes_.size()));
    reach_index_.resize(std::max(nr, reach_index_.size()));
    roll_.resize(std::max(nr, roll_.size()));
    rc = call(&nn, &nr);
  }
  if (rc != ALZ_OK) return rc;
  *rows = ToEdges(roll_.data(), nr, nullptr);
  nodes->resize(nn);
  for (size_t i = 0; i < nn; ++i) {
    const alz_reach_node& r = reach_nodes_[i];
    ReachNode& o = (*nodes)[i];
    o.Type = NodeTypeName(r.type);
    o.UID = UidOf(r.type, r.value);
    o.Hops = r.hops;
    o.Parent = r.parent;
    o.Row = kReachNone;
    if (r.row != kReachNone) {   // the parent's row is listed: its tail is the parent, at hops < max_hops
      o.Row = (uint32_t)(std::lower_bound(reach_index_.begin(), reach_index_.begin() + nr, r.row) -
                         reach_index_.begin());
    }
  }
  return ALZ_OK;
}

int Aggregator::Cycles(uint32_t source, const alz_metric* filter, double min_value, uint32_t min_size,
                       std::vector<CycleNode>* nodes, std::vector<EdgeWindow>* rows, alz_cycle_info* info) {
  return RunCycles(false, source, filter, min_value, min_size, nodes, rows, info);
}

int Aggregator::GroupCycles(uint32_t source, const alz_metric* filter, double min_value, uint32_t min_size,
                            std::vector<CycleNode>* nodes, std::vector<EdgeWindow>* rows, alz_cycle_info* info) {
  return RunCycles(true, source, filter, min_value, min_size, nodes, rows, info);
}

int Aggregator::RunCycles(bool group, uint32_t source, const alz_metric* filter, double min_value, uint32_t min_size,
                          std::vector<CycleNode>* nodes, std::vector<EdgeWindow>* rows, alz_cycle_info* info) {
  if (!h_) return ALZ_E_STATE;
  if (!nodes || !rows) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  if (info) *info = alz_cycle_info{};
  nodes->clear();
  rows->clear();
  if (group) {
    const int rc = SyncGroups();
    if (rc != ALZ_OK) return rc;
  }
  const uint32_t src = source == kLastWindow ? ALZ_SOURCE_WINDOW : source;
  // never empty: a null array would not be written (and its cap not checked)
  if (cycle_nodes_.empty()) cycle_nodes_.resize(1);
  if (cycle_index_.empty()) cycle_index_.resize(1);
  if (roll_.empty()) roll_.resize(1);
  auto call = [&](size_t* nn, size_t* nr) {
    return (group ? alz_group_cycles : alz_cycles)(h_, src, filter, min_value, min_size, cycle_nodes_.data(),
                                                   cycle_nodes_.size(), nn, cycle_index_.data(), roll_.data(),
                                                   std::min(cycle_index_.size(), roll_.size()), nr, info);
  };
  // into cycle_nodes_ / cycle_index_ / roll_, grown once when the results do not fit (ALZ_E_CAPACITY with the counts
  // set; nothing written)
  size_t nn = 0, nr = 0;
  int rc = call(&nn, &nr);
  if (rc == ALZ_E_CAPACITY && (nn > cycle_nodes_.size() || nr > cycle_index_.size() || nr > roll_.size())) {
    cycle_nodes_.resize(std::max(nn, cycle_nodes_.size()));
    cycle_index_.resize(std::max(nr, cycle_index_.size()));
    roll_.resize(std::max(nr, roll_.size()));
    rc = call(&nn, &nr);
  }
  if (rc != ALZ_OK) return rc;
  *rows = ToEdges(roll_.data(), nr, nullptr);
  nodes->resize(nn);
  for (size_t i = 0; i < nn; ++i) {
    const alz_cycle_node& r = cycle_nodes_[i];
    CycleNode& o = (*nodes)[i];
    o.Type = NodeTypeName(r.type);
    o.UID = UidOf(r.type, r.value);
    o.Component = r.component;
    o.Size = r.size;
    o.Depth = r.depth;
    o.Height = r.height;
  }
  return ALZ_OK;
}

int Aggregator::GroupNodeSeriesFor(const std::vector<NodeRef>& nodes, uint32_t side, uint32_t tier, uint32_t k,
                                   const std::vector<alz_metric>& metrics, std::vector<NodeSeriesRow>* out,
                                   std::vector<alz_rollup_info>* points) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  int rc = SyncGroups();
  if (rc != ALZ_OK) return rc;
  // the nodes that resolve go to the library; the others are absent at every point
  std::vector<alz_node_ends> keys;
  std::vector<size_t> row_of;   // node -> row of keys, or SIZE_MAX
  for (const NodeRef& r : nodes) {
    alz_node_ends k_{};
    if (GroupEndOf(r.Type, r.UID, &k_.type, &k_.value)) { row_of.push_back(keys.size()); keys.push_back(k_); }
    else row_of.push_back(SIZE_MAX);
  }
  const uint32_t nm = (uint32_t)metrics.size();
  std::vector<NodeSeriesRow> known;
  std::vector<alz_rollup_info> pts;
  rc = RunSeries(nm, &known, &pts, [&](double* v, uint8_t* p, size_t cap, size_t* n, uint32_t* P,
                                       alz_rollup_info* pp) {
    return alz_group_node_series_keys(h_, keys.data(), keys.size(), side, tier, k, metrics.data(), nm, v, p, cap, n,
                                      P, pp, nullptr);
  });
  if (rc != ALZ_OK) return rc;
  const size_t P = pts.size();
  out->assign(nodes.size(), NodeSeriesRow{});
  for (size_t i = 0; i < nodes.size(); ++i) {
    NodeSeriesRow& e = (*out)[i];
    if (row_of[i] != SIZE_MAX) e = known[row_of[i]];
    else { e.Present.assign(P, 0); e.Values.assign(P * nm, 0.0); }
    e.Type = nodes[i].Type;
    e.UID = nodes[i].UID;
  }
  if (points) *points = pts;
  return ALZ_OK;
}

int Aggregator::GroupTrends(uint32_t source, uint32_t tier, uint32_t k, const alz_metric& metric,
                            const alz_trend& trend, uint32_t top, double min_trend, std::vector<EdgeTrend>* out,
                            std::vector<alz_rollup_info>* points) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  const int rc = SyncGroups();
  if (rc != ALZ_OK) return rc;
  return RunEdgeTrends(alz_group_edge_trends_top, source, tier, k, metric, trend, top, min_trend, out, points);
}

int Aggregator::GroupNodeTrends(uint32_t source, uint32_t side, uint32_t tier, uint32_t k, const alz_metric& metric,
                                const alz_trend& trend, uint32_t top, double min_trend, std::vector<NodeTrend>* out,
                                std::vector<alz_rollup_info>* points) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  const int rc = SyncGroups();
  if (rc != ALZ_OK) return rc;
  return RunNodeTrends(alz_group_node_trends_top, source, side, tier, k, metric, trend, top, min_trend, out, points);
}

int Aggregator::SetHistory(uint32_t depth, uint64_t arena_rows, const std::vector<alz_history_tier>& tiers) {
  if (!h_) return ALZ_E_STATE;
  std::lock_guard<std::mutex> g(mu_);
  // The longest span, in flushed windows, that a retained entry or an open block can reach back: depth windows in
  // the window history; in tier t, depth_t closed entries and the open block, each of factor_1 x ... x factor_t
  // windows (the library keeps that product times depth_t below 2^32). The hold only grows: entries retained under
  // an earlier configuration may still be there.
  uint64_t hold = depth, span = 1;
  for (const alz_history_tier& t : tiers) {
    span = std::min<uint64_t>(span * t.factor, 1ull << 32);
    hold = std::max<uint64_t>(hold, span * ((uint64_t)t.depth + 1u));
  }
  hold_ = std::max(hold_, hold);
  const int rc = alz_window_history(h_, depth, arena_rows);
  if (rc != ALZ_OK) return rc;
  return alz_window_history_tiers(h_, tiers.empty() ? nullptr : tiers.data(), (uint32_t)tiers.size());
}

// call(out, cap, &n) into roll_, grown once when the rows do not fit (ALZ_E_CAPACITY with n = the rows there are;
// nothing was written), with_scores the GNN pass over those rows, then the rows to the data store
template <class Call>
int Aggregator::PersistRollup(uint32_t kind, bool with_scores, Call call) {
  size_t n = 0;
  int rc = call(roll_.data(), roll_.size(), &n);
  if (rc == ALZ_E_CAPACITY && n > roll_.size()) {
    roll_.resize(n + n / 4);
    rc = call(roll_.data(), roll_.size(), &n);
  }
  if (rc != ALZ_OK) return rc;
  if (with_scores && n) {
    scores_.resize(n);
    size_t ns = 0;
    rc = alz_gnn_score_rollup(h_, kind, scores_.data(), n, &ns);
    if (rc != ALZ_OK) return rc;
  }
  return ds_ ? ds_->PersistEdgeWindow(ToEdges(roll_.data(), n, with_scores ? scores_.data() : nullptr)) : ALZ_OK;
}

int Aggregator::Rollup(uint32_t tier, uint32_t k, alz_rollup_info* info, bool with_scores) {
  if (!h_) return ALZ_E_STATE;
  std::lock_guard<std::mutex> g(mu_);
  return PersistRollup(tier == 0 ? ALZ_ROLLUP_WINDOWS : ALZ_ROLLUP_TIER, with_scores,
                       [&](alz_edge_out* out, size_t cap, size_t* n) {
                         return alz_window_rollup_tier(h_, tier, k, out, cap, n, info);
                       });
}

// A span is made of retained entries and open blocks, each inside the span SetHistory's hold covers, so the ids it
// carries are held as those of a tier rollup are.
int Aggregator::RollupSpan(uint64_t windows, uint32_t mode, alz_span_info* info, bool with_scores) {
  if (!h_) return ALZ_E_STATE;
  std::lock_guard<std::mutex> g(mu_);
  return PersistRollup(ALZ_ROLLUP_SPAN, with_scores, [&](alz_edge_out* out, size_t cap, size_t* n) {
    return alz_window_rollup_span(h_, windows, mode, out, cap, n, info);
  });
}

int Aggregator::Stats(alz_stats* out) { return h_ ? alz_get_stats(h_, out) : ALZ_E_STATE; }

int Aggregator::ClearSocketLines(bool send_alive, int64_t check_time_ms) {
  if (!h_) return ALZ_E_STATE;
  std::lock_guard<std::mutex> g(mu_);
  if (send_alive) {
    if (tables_dirty_) {   // the export resolves against the committed tables
      int rc = alz_table_commit(h_);
      if (rc != ALZ_OK) return rc;
      tables_dirty_ = false;
    }
    size_t n = 0;
    if (alive_.empty()) alive_.resize(1u << 12);
    int rc = alz_sock_alive(h_, alive_.data(), alive_.size(), &n);
    if (rc == ALZ_E_CAPACITY) {   // n = the rows there are
      alive_.resize(n + n / 4);
      rc = alz_sock_alive(h_, alive_.data(), alive_.size(), &n);
    }
    if (rc != ALZ_OK) return rc;
    for (size_t i = 0; i < n && ds_; ++i) {
      const alz_alive_conn& c = alive_[i];
      AliveConnection ac;
      ac.CheckTime = check_time_ms;
      ac.FromIP = FormatIPv4(c.from_ip); ac.FromType = "pod"; ac.FromPort = c.from_port;
      ac.FromUID = c.from_id < pods_.names.size() ? pods_.names[c.from_id] : std::string("?");
      ac.ToIP = FormatIPv4(c.to_ip); ac.ToPort = c.to_port;
      ac.ToType = NodeTypeName(c.to_type);
      if (c.to_type == ALZ_NODE_POD) ac.ToUID = c.to_id < pods_.names.size() ? pods_.names[c.to_id] : std::string("?");
      else if (c.to_type == ALZ_NODE_SVC) ac.ToUID = c.to_id < svcs_.names.size() ? svcs_.names[c.to_id] : std::string("?");
      else ac.ToUID = ac.ToIP;                                             // data.go:1672-1673
      ds_->PersistAliveConnection(ac);
    }
  }
  return alz_sock_gc(h_);
}

namespace {
// the library's form of a CorrTarget; Present empty: every point present
alz_corr_target CorrTargetOf(const CorrTarget& t) {
  alz_corr_target c{};
  c.values = t.Values.data();
  c.present = t.Present.empty() ? nullptr : t.Present.data();
  c.n = t.Values.size();
  c.window_last = t.WindowLast;
  return c;
}
// the target a one-row series call gave: its only row and its newest point's window_last
template <class Row>
CorrTarget TargetOfSeries(const std::vector<Row>& rows, const std::vector<alz_rollup_info>& pts) {
  CorrTarget t;
  if (!rows.empty()) {
    t.Values = rows[0].Values;
    t.Present = rows[0].Present;
  }
  t.WindowLast = pts.empty() ? 0 : pts.back().window_last;
  return t;
}
}  // namespace

int Aggregator::RunEdgeCorr(EdgeCorrTop fn, uint32_t source, uint32_t tier, uint32_t k, const alz_metric& metric,
                            const alz_corr& corr, const CorrTarget& target, uint32_t top, double min_score,
                            const EdgeRef* skip, std::vector<EdgeCorr>* out, std::vector<alz_rollup_info>* points) {
  const uint32_t src = source == kLastWindow ? ALZ_SOURCE_WINDOW : source;
  const alz_corr_target t = CorrTargetOf(target);
  const uint32_t ask = skip && top ? top + 1 : top;   // room for the target's own row
  // a first call sizes the results (ALZ_E_CAPACITY with n = the results, P = the points; nothing written)
  size_t n = 0;
  uint32_t P = 0;
  int rc = fn(h_, src, tier, k, &metric, &corr, &t, ask, min_score, nullptr, nullptr, nullptr, nullptr, 0, &n, &P,
              nullptr, nullptr);
  std::vector<alz_rollup_info> pts(P);
  if (rc == ALZ_E_CAPACITY && n > 0) {
    corrs_.resize(n);
    trend_rows_.resize(n);
    trend_values_.resize(n * P);
    trend_present_.resize(n * P);
    rc = fn(h_, src, tier, k, &metric, &corr, &t, ask, min_score, corrs_.data(), trend_rows_.data(),
            trend_values_.data(), trend_present_.data(), n, &n, &P, pts.data(), nullptr);
  }
  if (rc != ALZ_OK) return rc;
  const std::vector<EdgeWindow> names = ToEdges(trend_rows_.data(), n, nullptr);
  out->clear();
  for (size_t i = 0; i < n && out->size() < top; ++i) {
    const EdgeWindow& w = names[i];
    if (skip && w.FromType == skip->FromType && w.FromUID == skip->FromUID && w.ToType == skip->ToType &&
        w.ToUID == skip->ToUID)
      continue;
    const alz_edge_corr& r = corrs_[i];
    EdgeCorr e;
    e.FromType = w.FromType; e.FromUID = w.FromUID; e.ToType = w.ToType; e.ToUID = w.ToUID;
    e.Valid = r.valid != 0;
    e.Lag = r.lag;
    e.Used = r.used;
    e.R = r.r; e.Score = r.score; e.R0 = r.r0;
    e.Present.assign(trend_present_.begin() + i * P, trend_present_.begin() + (i + 1) * P);
    e.Values.assign(trend_values_.begin() + i * P, trend_values_.begin() + (i + 1) * P);
    out->push_back(std::move(e));
  }
  if (points) *points = pts;
  return ALZ_OK;
}

int Aggregator::RunNodeCorr(NodeCorrTop fn, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                            const alz_metric& metric, const alz_corr& corr, const CorrTarget& target, uint32_t top,
                            double min_score, const NodeRef* skip, std::vector<NodeCorr>* out,
                            std::vector<alz_rollup_info>* points) {
  const uint32_t src = source == kLastWindow ? ALZ_SOURCE_WINDOW : source;
  const alz_corr_target t = CorrTargetOf(target);
  const uint32_t ask = skip && top ? top + 1 : top;
  size_t n = 0;
  uint32_t P = 0;
  int rc = fn(h_, src, side, tier, k, &metric, &corr, &t, ask, min_score, nullptr, nullptr, nullptr, nullptr, 0, &n,
              &P, nullptr, nullptr);
  std::vector<alz_rollup_info> pts(P);
  if (rc == ALZ_E_CAPACITY && n > 0) {
    node_corrs_.resize(n);
    node_trend_rows_.resize(n);
    trend_values_.resize(n * P);
    trend_present_.resize(n * P);
    rc = fn(h_, src, side, tier, k, &metric, &corr, &t, ask, min_score, node_corrs_.data(), node_trend_rows_.data(),
            trend_values_.data(), trend_present_.data(), n, &n, &P, pts.data(), nullptr);
  }
  if (rc != ALZ_OK) return rc;
  const std::vector<NodeWindow> names = ToNodes(node_trend_rows_.data(), n, nullptr, 0);
  out->clear();
  for (size_t i = 0; i < n && out->size() < top; ++i) {
    if (skip && names[i].Type == skip->Type && names[i].UID == skip->UID) continue;
    const alz_node_corr& r = node_corrs_[i];
    NodeCorr e;
    e.Node = names[i];
    e.Valid = r.valid != 0;
    e.Lag = r.lag;
    e.Used = r.used;
    e.R = r.r; e.Score = r.score; e.R0 = r.r0;
    e.Present.assign(trend_present_.begin() + i * P, trend_present_.begin() + (i + 1) * P);
    e.Values.assign(trend_values_.begin() + i * P, trend_values_.begin() + (i + 1) * P);
    out->push_back(std::move(e));
  }
  if (points) *points = pts;
  return ALZ_OK;
}

int Aggregator::Correlations(uint32_t source, uint32_t tier, uint32_t k, const alz_metric& metric,
                             const alz_corr& corr, const CorrTarget& target, uint32_t top, double min_score,
                             std::vector<EdgeCorr>* out, std::vector<alz_rollup_info>* points) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  return RunEdgeCorr(alz_edge_correlations_top, source, tier, k, metric, corr, target, top, min_score, nullptr, out,
                     points);
}

int Aggregator::Correlations(uint32_t source, uint32_t tier, uint32_t k, const alz_metric& metric,
                             const alz_corr& corr, const EdgeRef& target, uint32_t top, double min_score,
                             std::vector<EdgeCorr>* out, std::vector<alz_rollup_info>* points) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::vector<EdgeSeries> ser;
  std::vector<alz_rollup_info> pts;
  int rc = SeriesFor({target}, tier, k, {metric}, &ser, &pts);
  if (rc != ALZ_OK) return rc;
  std::lock_guard<std::mutex> g(mu_);
  return RunEdgeCorr(alz_edge_correlations_top, source, tier, k, metric, corr, TargetOfSeries(ser, pts), top,
                     min_score, &target, out, points);
}

int Aggregator::NodeCorrelations(uint32_t source, uint32_t side, uint32_t tier, uint32_t k, const alz_metric& metric,
                                 const alz_corr& corr, const CorrTarget& target, uint32_t top, double min_score,
                                 std::vector<NodeCorr>* out, std::vector<alz_rollup_info>* points) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  return RunNodeCorr(alz_node_correlations_top, source, side, tier, k, metric, corr, target, top, min_score, nullptr,
                     out, points);
}

int Aggregator::NodeCorrelations(uint32_t source, uint32_t side, uint32_t tier, uint32_t k, const alz_metric& metric,
                                 const alz_corr& corr, const NodeRef& target, uint32_t top, double min_score,
                                 std::vector<NodeCorr>* out, std::vector<alz_rollup_info>* points) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::vector<NodeSeriesRow> ser;
  std::vector<alz_rollup_info> pts;
  int rc = NodeSeriesFor({target}, side, tier, k, {metric}, &ser, &pts);
  if (rc != ALZ_OK) return rc;
  std::lock_guard<std::mutex> g(mu_);
  return RunNodeCorr(alz_node_correlations_top, source, side, tier, k, metric, corr, TargetOfSeries(ser, pts), top,
                     min_score, &target, out, points);
}

int Aggregator::GroupCorrelations(uint32_t source, uint32_t tier, uint32_t k, const alz_metric& metric,
                                  const alz_corr& corr, const CorrTarget& target, uint32_t top, double min_score,
                                  std::vector<EdgeCorr>* out, std::vector<alz_rollup_info>* points) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  const int rc = SyncGroups();
  if (rc != ALZ_OK) return rc;
  return RunEdgeCorr(alz_group_edge_correlations_top, source, tier, k, metric, corr, target, top, min_score, nullptr,
                     out, points);
}

int Aggregator::GroupCorrelations(uint32_t source, uint32_t tier, uint32_t k, const alz_metric& metric,
                                  const alz_corr& corr, const EdgeRef& target, uint32_t top, double min_score,
                                  std::vector<EdgeCorr>* out, std::vector<alz_rollup_info>* points) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::vector<EdgeSeries> ser;
  std::vector<alz_rollup_info> pts;
  int rc = GroupSeriesFor({target}, tier, k, {metric}, &ser, &pts);
  if (rc != ALZ_OK) return rc;
  std::lock_guard<std::mutex> g(mu_);
  rc = SyncGroups();
  if (rc != ALZ_OK) return rc;
  return RunEdgeCorr(alz_group_edge_correlations_top, source, tier, k, metric, corr, TargetOfSeries(ser, pts), top,
                     min_score, &target, out, points);
}

int Aggregator::GroupNodeCorrelations(uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                      const alz_metric& metric, const alz_corr& corr, const CorrTarget& target,
                                      uint32_t top, double min_score, std::vector<NodeCorr>* out,
                                      std::vector<alz_rollup_info>* points) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(mu_);
  const int rc = SyncGroups();
  if (rc != ALZ_OK) return rc;
  return RunNodeCorr(alz_group_node_correlations_top, source, side, tier, k, metric, corr, target, top, min_score,
                     nullptr, out, points);
}

int Aggregator::GroupNodeCorrelations(uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                      const alz_metric& metric, const alz_corr& corr, const NodeRef& target,
                                      uint32_t top, double min_score, std::vector<NodeCorr>* out,
                                      std::vector<alz_rollup_info>* points) {
  if (!h_) return ALZ_E_STATE;
  if (!out) return ALZ_E_INVAL;
  std::vector<NodeSeriesRow> ser;
  std::vector<alz_rollup_info> pts;
  int rc = GroupNodeSeriesFor({target}, side, tier, k, {metric}, &ser, &pts);
  if (rc != ALZ_OK) return rc;
  std::lock_guard<std::mutex> g(mu_);
  rc = SyncGroups();
  if (rc != ALZ_OK) return rc;
  return RunNodeCorr(alz_group_node_correlations_top, source, side, tier, k, metric, corr, TargetOfSeries(ser, pts),
                     top, min_score, &target, out, points);
}

}  // namespace alaz
