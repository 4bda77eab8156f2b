// gnn_rollup_adapter_test.cc — the C++ host adapter's scored rollups (docs/SPEC.md §15): Rollup and RollupSpan with
// with_scores fill EdgeWindow::Score through alz_gnn_score_rollup, as Flush(true) does for a window.
#include <cstdio>
#include <cstring>
#include <map>
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
// per edge (by UIDs): its score, as the bits of the float
static std::map<std::string, uint32_t> scores(const std::vector<alaz::EdgeWindow>& rows) {
  std::map<std::string, uint32_t> m;
  for (const auto& r : rows) {
    uint32_t bits;
    memcpy(&bits, &r.Score, 4);
    m[r.FromType + ":" + r.FromUID + "->" + r.ToType + ":" + r.ToUID] = bits;
  }
  return m;
}

int main() {
  RecordingDataStore ds;
  alaz::AggregatorConfig ac;
  ac.MaxEndpoints = 1u << 10;
  ac.MaxPairs = 1u << 12;
  alaz::Aggregator a(&ds, ac);
  CHECK(a.Ok(), "aggregator: %s", a.LastError().c_str());
  CHECK(a.SetHistory(4, 1u << 12) == ALZ_OK, "SetHistory");

  k8s(a, "Service", "Add", "svc-a", "10.96.0.1");
  k8s(a, "Service", "Add", "svc-b", "10.96.0.2");
  for (int p = 1; p <= 12; ++p) {
    char uid[16], ip[16];
    snprintf(uid, sizeof uid, "pod-%d", p);
    snprintf(ip, sizeof ip, "10.0.0.%d", p);
    k8s(a, "Pod", "Add", uid, ip);
  }
  for (int w = 1; w <= 4; ++w) {                                // window w: pods w .. w + 8, to both services
    for (int p = w; p <= w + 8; ++p) {
      char ip[16];
      snprintf(ip, sizeof ip, "10.0.0.%d", p);
      requests(a, ip, "10.96.0.1", 1 + (p + w) % 4, (p % 5) ? 200u : 500u, 1000000u * (uint64_t)w);
      if (p % 3 == w % 3) requests(a, ip, "10.96.0.2", 2, 200u, 3000000u);
      if (p % 4 == 0) requests(a, ip, "10.0.0.12", 1, 200u, 500000u);
    }
    CHECK(a.Flush(true) == ALZ_OK, "flush %d", w);
    const auto win = scores(ds.calls.back());
    CHECK(a.Rollup(0, 1, nullptr, true) == ALZ_OK, "Rollup(0, 1) after window %d", w);
    const auto roll = scores(ds.calls.back());
    CHECK(roll == win && win.size() > 10, "window %d: a 1-window rollup scores %zu rows as the window's %zu", w,
          roll.size(), win.size());
  }
  for (uint32_t N = 1; N <= 4; ++N) {
    alz_span_info si;
    CHECK(a.RollupSpan(N, ALZ_SPAN_AT_MOST, &si, true) == ALZ_OK && si.r.windows == N, "RollupSpan(%u)", N);
    const auto span = scores(ds.calls.back());
    alz_rollup_info ri;
    CHECK(a.Rollup(0, N, &ri, true) == ALZ_OK && ri.windows == N, "Rollup(0, %u)", N);
    const auto roll = scores(ds.calls.back());
    CHECK(span == roll, "span of %u scores as the window rollup of %u", N, N);
    bool some = false;
    for (const auto& kv : roll) some |= kv.second != 0u;
    CHECK(some, "rollup of %u: every score is 0", N);
  }
  CHECK(a.Rollup(0, 3) == ALZ_OK, "Rollup without scores");
  for (const auto& r : ds.calls.back()) CHECK(r.Score == 0.f, "Rollup without scores: %s %g", r.FromUID.c_str(), r.Score);
  CHECK(a.RollupSpan(3, ALZ_SPAN_AT_LEAST) == ALZ_OK, "RollupSpan without scores");
  for (const auto& r : ds.calls.back()) CHECK(r.Score == 0.f, "RollupSpan without scores: %g", r.Score);
  printf("gnn rollup adapter ok\n");
  return 0;
}
