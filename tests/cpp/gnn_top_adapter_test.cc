// gnn_top_adapter_test.cc — the C++ host adapter's top anomalous rows (docs/SPEC.md §16): Anomalies after Flush,
// Rollup and RollupSpan returns the scored source's own best rows, by UID, best first and ties in row order.
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
static uint32_t key_of(float s) {   // docs/SPEC.md §16's order key
  uint32_t u;
  memcpy(&u, &s, 4);
  return (u & 0x80000000u) ? ~u : u ^ 0x80000000u;
}
static std::string uid(const alaz::EdgeWindow& r) { return r.FromType + ":" + r.FromUID + "->" + r.ToType + ":" + r.ToUID; }
static bool same(const alaz::EdgeWindow& a, const alaz::EdgeWindow& b) {
  return uid(a) == uid(b) && a.Count == b.Count && a.Err5xx == b.Err5xx && a.LatSumNs == b.LatSumNs &&
         memcmp(a.Hist, b.Hist, sizeof a.Hist) == 0 && memcmp(&a.Score, &b.Score, 4) == 0;
}
// the first k rows of `scored` (the source's rows with scores, in row order) with score >= min, stably by key desc
static std::vector<alaz::EdgeWindow> best(const std::vector<alaz::EdgeWindow>& scored, size_t k, float min) {
  std::vector<size_t> idx;
  for (size_t i = 0; i < scored.size(); ++i)
    if (key_of(scored[i].Score) >= key_of(min)) idx.push_back(i);
  for (size_t i = 1; i < idx.size(); ++i)   // insertion sort: stable, the lists are short
    for (size_t j = i; j > 0 && key_of(scored[idx[j]].Score) > key_of(scored[idx[j - 1]].Score); --j)
      std::swap(idx[j], idx[j - 1]);
  std::vector<alaz::EdgeWindow> out;
  for (size_t i = 0; i < idx.size() && i < k; ++i) out.push_back(scored[idx[i]]);
  return out;
}
static int compare(const std::vector<alaz::EdgeWindow>& got, const std::vector<alaz::EdgeWindow>& want, const char* what) {
  CHECK(got.size() == want.size(), "%s: %zu rows, want %zu", what, got.size(), want.size());
  for (size_t i = 0; i < got.size(); ++i)
    CHECK(same(got[i], want[i]), "%s: row %zu is %s, want %s", what, i, uid(got[i]).c_str(), uid(want[i]).c_str());
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
  std::vector<alaz::EdgeWindow> top;
  CHECK(a.Anomalies(ALZ_ROLLUP_WINDOWS, 5, 0.f, &top) == ALZ_E_STATE, "no rollup yet");
  CHECK(a.Anomalies(alaz::Aggregator::kLastWindow, 0, 0.f, &top) == ALZ_E_INVAL, "k = 0");

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
      requests(a, ip, "10.96.0.1", 1 + (p + w) % 4, (p % 5) ? 200u : 500u, 1000000u * (uint64_t)w);
      if (p % 3 == w % 3) requests(a, ip, "10.96.0.2", 2, 200u, 3000000u);
      if (p % 4 == 0) requests(a, ip, "10.0.0.12", 1, 200u, 500000u);
    }
    CHECK(a.Flush(true) == ALZ_OK, "flush %d", w);
    const std::vector<alaz::EdgeWindow> scored = ds.calls.back();
    for (size_t k : {(size_t)1, (size_t)7, scored.size(), scored.size() + 5}) {
      alz_top_info info;
      CHECK(a.Anomalies(alaz::Aggregator::kLastWindow, (uint32_t)k, 0.f, &top, &info) == ALZ_OK, "window %d", w);
      CHECK(info.scored == scored.size() && info.above == scored.size(), "window %d info", w);
      if (compare(top, best(scored, k, 0.f), "window")) return 1;
    }
  }
  for (uint32_t N = 1; N <= 4; ++N) {
    CHECK(a.Rollup(0, N, nullptr, true) == ALZ_OK, "Rollup(0, %u)", N);
    std::vector<alaz::EdgeWindow> scored = ds.calls.back();
    const float mid = best(scored, scored.size() / 2, 0.f).back().Score;
    for (uint32_t k : {1u, 10u, 1000u}) {
      CHECK(a.Anomalies(ALZ_ROLLUP_WINDOWS, k, mid, &top) == ALZ_OK, "rollup %u k %u", N, k);
      if (compare(top, best(scored, k, mid), "rollup")) return 1;
    }
    alz_span_info si;
    CHECK(a.RollupSpan(N, ALZ_SPAN_AT_MOST, &si, true) == ALZ_OK && si.r.windows == N, "RollupSpan(%u)", N);
    scored = ds.calls.back();
    CHECK(a.Anomalies(ALZ_ROLLUP_SPAN, 20, 0.f, &top) == ALZ_OK, "span %u", N);
    if (compare(top, best(scored, 20, 0.f), "span")) return 1;
  }
  printf("gnn top adapter ok\n");
  return 0;
}
