// tier_adapter_test.cc — the C++ host adapter with the window history and tiers on (docs/SPEC.md §12, §13):
// Aggregator::SetHistory / Rollup hand tier rollups to the sink, and an id freed inside the retained span is not
// given to another UID (two pods would otherwise become one row in the entries that cover both).
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
// FromUID -> count of the rows of one sink call
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
  CHECK(a.SetHistory(3, 1u << 12, {{1u, 2u, 1u << 12, 1u << 12}}) == ALZ_E_INVAL, "factor 1 accepted");
  // tier 1: 4 windows per entry, 2 entries: an id can be reached back for (2 + 1) x 4 = 12 windows
  CHECK(a.SetHistory(3, 1u << 12, {{4u, 2u, 1u << 12, 1u << 12}}) == ALZ_OK, "SetHistory");

  k8s(a, "Service", "Add", "svc-s", "10.96.0.1");
  k8s(a, "Pod", "Add", "pod-a", "10.0.0.1");
  requests(a, "10.0.0.1", "10.96.0.1", 3);
  CHECK(a.Flush() == ALZ_OK, "flush 1");                        // window 1: pod-a
  k8s(a, "Pod", "Delete", "pod-a", "10.0.0.1");
  CHECK(a.Flush() == ALZ_OK, "flush 2");                        // window 2: pod-a's id is no longer mapped
  k8s(a, "Pod", "Add", "pod-c", "10.0.0.3");                    // must not take pod-a's id: window 1 is retained
  requests(a, "10.0.0.3", "10.96.0.1", 5);
  CHECK(a.Flush() == ALZ_OK, "flush 3");
  CHECK(a.Flush() == ALZ_OK, "flush 4");                        // closes the tier-1 block of windows 1..4
  CHECK(ds.calls.size() == 4, "%zu sink calls", ds.calls.size());

  alz_rollup_info info;
  CHECK(a.Rollup(1, 1, &info) == ALZ_OK, "Rollup(1, 1)");
  CHECK(ds.calls.size() == 5 && info.windows == 4 && info.window_first == 1 && info.window_last == 4,
        "tier-1 rollup: %zu calls, %u windows", ds.calls.size(), info.windows);
  auto t1 = counts(ds.calls.back());
  CHECK(t1.size() == 2 && t1["pod-a->svc-s"] == 3 && t1["pod-c->svc-s"] == 5,
        "tier-1 entry: %zu rows, pod-a %llu, pod-c %llu", t1.size(), (unsigned long long)t1["pod-a->svc-s"],
        (unsigned long long)t1["pod-c->svc-s"]);

  CHECK(a.Rollup(0, 3, &info) == ALZ_OK, "Rollup(0, 3)");          // windows 2..4 of the window history
  auto t0 = counts(ds.calls.back());
  CHECK(ds.calls.size() == 6 && info.windows == 3 && t0.size() == 1 && t0["pod-c->svc-s"] == 5, "tier-0 rollup");

  // pod-c leaves in window 5; until window 5 + 12 has been flushed its id stays taken, and every pod added
  // meanwhile gets a row of its own in the tier-1 entries
  k8s(a, "Pod", "Delete", "pod-c", "10.0.0.3");
  CHECK(a.Flush() == ALZ_OK, "flush 5");
  for (int w = 6; w <= 8; ++w) {
    char uid[16], ip[16];
    snprintf(uid, sizeof uid, "pod-%d", w);
    snprintf(ip, sizeof ip, "10.0.1.%d", w);
    k8s(a, "Pod", "Add", uid, ip);
    requests(a, ip, "10.96.0.1", w);
    CHECK(a.Flush() == ALZ_OK, "flush %d", w);
  }                                                             // windows 5..8: the second tier-1 entry
  CHECK(a.Rollup(1, 2, &info) == ALZ_OK && info.windows == 8, "Rollup(1, 2)");
  auto t2 = counts(ds.calls.back());
  CHECK(t2.size() == 5 && t2["pod-a->svc-s"] == 3 && t2["pod-c->svc-s"] == 5 && t2["pod-6->svc-s"] == 6 &&
        t2["pod-7->svc-s"] == 7 && t2["pod-8->svc-s"] == 8, "two tier-1 entries: %zu rows", t2.size());
  CHECK(a.SetHistory(0, 0, {}) == ALZ_OK, "SetHistory off");
  CHECK(a.Rollup(1, 1, &info) == ALZ_E_STATE, "Rollup without tiers");
  printf("tier adapter ok\n");
  return 0;
}
