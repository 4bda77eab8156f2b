// span_adapter_test.cc — the C++ host adapter with the window history and tiers on (docs/SPEC.md §14):
// Aggregator::RollupSpan hands the sum of the last N windows, open blocks included, to the sink with the windows it
// covers.
#include <cstdio>
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
static void requests(alaz::Aggregator& a, const char* from, const char* to, int n) {
  for (int i = 0; i < n; ++i) {
    alaz::L7Event e;
    e.Status = 200; e.Duration = 1000; e.Protocol = "HTTP"; e.Method = "GET";
    e.Saddr = alaz::Aggregator::ParseIPv4(from, nullptr);
    e.Daddr = alaz::Aggregator::ParseIPv4(to, nullptr);
    e.Sport = (uint16_t)(40000 + i); e.Dport = 80;
    a.ProcessL7(e);
  }
}
static std::map<std::string, uint64_t> counts(const std::vector<alaz::EdgeWindow>& rows) {
  std::map<std::string, uint64_t> m;
  for (const auto& r : rows) m[r.FromUID + "->" + r.ToUID] += r.Count;
  return m;
}

int main() {
  RecordingDataStore ds;
  alaz::AggregatorConfig ac;
  ac.MaxEndpoints = 1u << 10;
  ac.MaxPairs = 1u << 12;
  alaz::Aggregator a(&ds, ac);
  CHECK(a.Ok(), "aggregator: %s", a.LastError().c_str());
  alz_span_info info;
  CHECK(a.RollupSpan(1, ALZ_SPAN_AT_MOST, &info) == ALZ_E_STATE, "span without a history or tiers");
  // the window history keeps 2 windows; tier 1 sums 4 windows per entry
  CHECK(a.SetHistory(2, 1u << 12, {{4u, 2u, 1u << 12, 1u << 12}}) == ALZ_OK, "SetHistory");

  k8s(a, "Service", "Add", "svc-s", "10.96.0.1");
  for (int w = 1; w <= 6; ++w) {                                // pod-w sends w requests in window w
    char uid[16], ip[16];
    snprintf(uid, sizeof uid, "pod-%d", w);
    snprintf(ip, sizeof ip, "10.0.0.%d", w);
    k8s(a, "Pod", "Add", uid, ip);
    requests(a, ip, "10.96.0.1", w);
    CHECK(a.Flush() == ALZ_OK, "flush %d", w);
  }
  const size_t flushes = ds.calls.size();
  // windows 1..6: the tier-1 entry of windows 1..4 and tier 1's open block of windows 5 and 6
  CHECK(a.RollupSpan(6, ALZ_SPAN_AT_MOST, &info) == ALZ_OK, "RollupSpan(6)");
  CHECK(ds.calls.size() == flushes + 1 && info.r.windows == 6 && info.r.window_first == 1 && info.r.window_last == 6,
        "span of 6: %zu calls, %u windows", ds.calls.size(), info.r.windows);
  CHECK(info.entries[1] == 1 && info.open_blocks == 2u, "span of 6: pieces %u / %u", info.entries[1], info.open_blocks);
  auto s6 = counts(ds.calls.back());
  CHECK(s6.size() == 6, "span of 6: %zu rows", s6.size());
  for (int w = 1; w <= 6; ++w) {
    char key[32];
    snprintf(key, sizeof key, "pod-%d->svc-s", w);
    CHECK(s6[key] == (uint64_t)w, "span of 6: %s %llu", key, (unsigned long long)s6[key]);
  }
  // 3 windows are not coverable (the history has 5 and 6, tier 1's open block 5..6): at least 3 gives 6
  CHECK(a.RollupSpan(3, ALZ_SPAN_AT_MOST, &info) == ALZ_OK && info.r.windows == 2 && info.r.window_first == 5,
        "at most 3: %u windows", info.r.windows);
  CHECK(counts(ds.calls.back()).size() == 2, "at most 3: rows");
  CHECK(a.RollupSpan(3, ALZ_SPAN_AT_LEAST, &info) == ALZ_OK && info.r.windows == 6, "at least 3: %u", info.r.windows);
  CHECK(a.RollupSpan(0, ALZ_SPAN_AT_MOST, &info) == ALZ_E_INVAL, "N = 0");
  printf("span adapter ok\n");
  return 0;
}
