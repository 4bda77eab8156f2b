// edge_top_adapter_test.cc — the C++ host adapter's edge metrics and top edges (docs/SPEC.md §17): EdgeMetrics and
// TopEdges after Flush, Rollup and RollupSpan agree with the source's own rows as the data store received them, by
// UID, highest first and ties in row order; every quantile equals alz_edge_quantiles of the row.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../alaz_b200/host/alaz_aggregator.hpp"

struct RecordingDataStore : alaz::DataStore {
  std::vector<std::vector<alaz::EdgeWindow>> calls;
  int PersistEdgeWindow(const std::vector<alaz::EdgeWindow>& edges) override { calls.push_back(edges); return 0; }
};

#define CHECK(cond, ...)                                             \
  do {                                                               \
    if (!(cond)) { fprintf(stderr, "FAIL %s:%d: ", __FILE__, __LINE__); fprintf(stderr, __VA_ARGS__); fprintf(stderr, "\n"); return 1; } \
  } while (0)

static void k8s(alaz::Aggregator& a, const char* kind, const char* ev, const char* uid, const char* ip) {
  alaz::K8sResourceMessage m;
  m.ResourceType = kind; m.EventType = ev; m.UID = uid; m.IP = ip;
  a.ProcessK8s(m);
}
static void requests(alaz::Aggregator& a, const char* from, const char* to, int n, uint32_t status, uint64_t dur) {
  for (int i = 0; i < n; ++i) {
    alaz::L7Event e;
    e.Status = status; e.Duration = dur * (uint64_t)(i + 1); e.Protocol = "HTTP"; e.Method = "GET";
    e.Saddr = alaz::Aggregator::ParseIPv4(from, nullptr);
    e.Daddr = alaz::Aggregator::ParseIPv4(to, nullptr);
    e.Sport = (uint16_t)(40000 + i); e.Dport = 80;
    a.ProcessL7(e);
  }
}
static alz_metric metric(uint32_t kind, double q = 0.0) { alz_metric m{}; m.kind = kind; m.q = q; return m; }
// the metric of one row as docs/SPEC.md §17 defines it, with the library's host quantile
static double value_of(const alaz::EdgeWindow& r, const alz_metric& m) {
  switch (m.kind) {
    case ALZ_METRIC_COUNT: return (double)r.Count;
    case ALZ_METRIC_ERR5XX: return (double)r.Err5xx;
    case ALZ_METRIC_ERR_RATE: return r.Count ? (double)r.Err5xx / (double)r.Count : 0.0;
    case ALZ_METRIC_MEAN_NS: return r.Count ? (double)r.LatSumNs / (double)r.Count : 0.0;
    default: {
      alz_edge_out e{};
      memcpy(e.hist, r.Hist, sizeof e.hist);
      double v = -1.0;
      alz_edge_quantiles(&e, &m.q, 1, &v);
      return v;
    }
  }
}
static uint64_t key_of(double v) {   // docs/SPEC.md §17's order key
  uint64_t u;
  memcpy(&u, &v, 8);
  return (u >> 63) ? ~u : u ^ (1ull << 63);
}
static std::string uid(const alaz::EdgeWindow& r) { return r.FromType + ":" + r.FromUID + "->" + r.ToType + ":" + r.ToUID; }
static bool same(const alaz::EdgeWindow& a, const alaz::EdgeWindow& b) {
  return uid(a) == uid(b) && a.Count == b.Count && a.Err5xx == b.Err5xx && a.LatSumNs == b.LatSumNs &&
         memcmp(a.Hist, b.Hist, sizeof a.Hist) == 0;
}
// the first k rows of `rows` (in row order) with value >= min, stably by key desc, each with its Value
static std::vector<alaz::EdgeWindow> best(const std::vector<alaz::EdgeWindow>& rows, const alz_metric& m, size_t k,
                                          double min) {
  std::vector<size_t> idx;
  for (size_t i = 0; i < rows.size(); ++i)
    if (key_of(value_of(rows[i], m)) >= key_of(min)) idx.push_back(i);
  for (size_t i = 1; i < idx.size(); ++i)   // insertion sort: stable, the lists are short
    for (size_t j = i; j > 0 && key_of(value_of(rows[idx[j]], m)) > key_of(value_of(rows[idx[j - 1]], m)); --j)
      std::swap(idx[j], idx[j - 1]);
  std::vector<alaz::EdgeWindow> out;
  for (size_t i = 0; i < idx.size() && i < k; ++i) {
    out.push_back(rows[idx[i]]);
    out.back().Value = value_of(rows[idx[i]], m);
  }
  return out;
}
static int compare(const std::vector<alaz::EdgeWindow>& got, const std::vector<alaz::EdgeWindow>& want, const char* what) {
  CHECK(got.size() == want.size(), "%s: %zu rows, want %zu", what, got.size(), want.size());
  for (size_t i = 0; i < got.size(); ++i) {
    CHECK(same(got[i], want[i]), "%s: row %zu is %s, want %s", what, i, uid(got[i]).c_str(), uid(want[i]).c_str());
    CHECK(memcmp(&got[i].Value, &want[i].Value, 8) == 0, "%s: row %zu value %.17g, want %.17g", what, i,
          got[i].Value, want[i].Value);
  }
  return 0;
}
static int check_metrics(alaz::Aggregator& a, uint32_t source, const std::vector<alaz::EdgeWindow>& rows,
                         const std::vector<alz_metric>& ms, const char* what) {
  std::vector<double> v;
  CHECK(a.EdgeMetrics(source, ms, &v) == ALZ_OK, "%s: EdgeMetrics", what);
  CHECK(v.size() == rows.size() * ms.size(), "%s: %zu values for %zu rows", what, v.size(), rows.size());
  for (size_t i = 0; i < rows.size(); ++i)
    for (size_t j = 0; j < ms.size(); ++j) {
      const double want = value_of(rows[i], ms[j]);
      CHECK(memcmp(&v[i * ms.size() + j], &want, 8) == 0, "%s: row %zu metric %zu", what, i, j);
    }
  return 0;
}

int main() {
  RecordingDataStore ds;
  alaz::AggregatorConfig ac;
  ac.MaxEndpoints = 1u << 10;
  ac.MaxPairs = 1u << 12;
  alaz::Aggregator a(&ds, ac);
  CHECK(a.Ok(), "aggregator: %s", a.LastError().c_str());
  CHECK(a.SetHistory(4, 1u << 12) == ALZ_OK, "SetHistory");
  const std::vector<alz_metric> all = {metric(ALZ_METRIC_COUNT), metric(ALZ_METRIC_ERR5XX),
                                       metric(ALZ_METRIC_ERR_RATE), metric(ALZ_METRIC_MEAN_NS),
                                       metric(ALZ_METRIC_QUANTILE, 0.5), metric(ALZ_METRIC_QUANTILE, 0.99)};
  std::vector<alaz::EdgeWindow> top;
  std::vector<double> v;
  CHECK(a.TopEdges(ALZ_ROLLUP_WINDOWS, all[0], 5, 0.0, &top) == ALZ_E_STATE, "no rollup yet");
  CHECK(a.EdgeMetrics(ALZ_ROLLUP_WINDOWS, all, &v) == ALZ_E_STATE, "no rollup yet");
  CHECK(a.TopEdges(alaz::Aggregator::kLastWindow, all[0], 0, 0.0, &top) == ALZ_E_INVAL, "k = 0");
  CHECK(a.EdgeMetrics(alaz::Aggregator::kLastWindow, {}, &v) == ALZ_E_INVAL, "no metric");

  k8s(a, "Service", "Add", "svc-a", "10.96.0.1");
  k8s(a, "Service", "Add", "svc-b", "10.96.0.2");
  for (int p = 1; p <= 40; ++p) {
    char u[16], ip[16];
    snprintf(u, sizeof u, "pod-%d", p);
    snprintf(ip, sizeof ip, "10.0.0.%d", p);
    k8s(a, "Pod", "Add", u, ip);
  }
  for (int w = 1; w <= 4; ++w) {
    for (int p = w; p <= w + 30; ++p) {
      char ip[16];
      snprintf(ip, sizeof ip, "10.0.0.%d", p);
      requests(a, ip, "10.96.0.1", 1 + (p + w) % 4, (p % 5) ? 200u : 500u, 1000000u * (uint64_t)(w + p % 7));
      if (p % 3 == w % 3) requests(a, ip, "10.96.0.2", 2, 200u, 3000000u);
      if (p % 4 == 0) requests(a, ip, "10.0.0.12", 1, (p % 8) ? 200u : 503u, 500000u);
    }
    CHECK(a.Flush() == ALZ_OK, "flush %d", w);
    const std::vector<alaz::EdgeWindow> rows = ds.calls.back();
    if (check_metrics(a, alaz::Aggregator::kLastWindow, rows, all, "window")) return 1;
    for (const alz_metric& m : all)
      for (size_t k : {(size_t)1, (size_t)7, rows.size() + 5}) {
        alz_top_info info;
        CHECK(a.TopEdges(alaz::Aggregator::kLastWindow, m, (uint32_t)k, 0.0, &top, &info) == ALZ_OK, "window %d", w);
        CHECK(info.scored == rows.size() && info.above == rows.size(), "window %d info", w);
        if (compare(top, best(rows, m, k, 0.0), "window")) return 1;
      }
  }
  for (uint32_t N = 1; N <= 4; ++N) {
    CHECK(a.Rollup(0, N) == ALZ_OK, "Rollup(0, %u)", N);
    std::vector<alaz::EdgeWindow> rows = ds.calls.back();
    if (check_metrics(a, ALZ_ROLLUP_WINDOWS, rows, all, "rollup")) return 1;
    for (const alz_metric& m : all) {
      const double mid = value_of(best(rows, m, rows.size() / 2, 0.0).back(), m);
      CHECK(a.TopEdges(ALZ_ROLLUP_WINDOWS, m, 10, mid, &top) == ALZ_OK, "rollup %u", N);
      if (compare(top, best(rows, m, 10, mid), "rollup")) return 1;
    }
    alz_span_info si;
    CHECK(a.RollupSpan(N, ALZ_SPAN_AT_MOST, &si) == ALZ_OK && si.r.windows == N, "RollupSpan(%u)", N);
    rows = ds.calls.back();
    if (check_metrics(a, ALZ_ROLLUP_SPAN, rows, all, "span")) return 1;
    CHECK(a.TopEdges(ALZ_ROLLUP_SPAN, all[5], 20, 0.0, &top) == ALZ_OK, "span %u", N);
    if (compare(top, best(rows, all[5], 20, 0.0), "span")) return 1;
  }
  printf("edge top adapter ok\n");
  return 0;
}
