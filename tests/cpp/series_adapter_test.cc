// series_adapter_test.cc — the C++ host adapter's edge series (docs/SPEC.md §19): Series gives every row of a source
// and SeriesFor the edges named by UID, point by point over the window history. A series by UID matches the id series;
// a pod deleted mid-history is present up to its deletion and absent after it, under its own UID and never under the
// UID of a pod added later; an unknown UID gives an absent row.
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../alaz_b200/host/alaz_aggregator.hpp"

#define CHECK(cond, ...)                                             \
  do {                                                               \
    if (!(cond)) { fprintf(stderr, "FAIL %s:%d: ", __FILE__, __LINE__); fprintf(stderr, __VA_ARGS__); fprintf(stderr, "\n"); return 1; } \
  } while (0)

static void k8s(alaz::Aggregator& a, const char* kind, const char* ev, const char* uid, const char* ip) {
  alaz::K8sResourceMessage m;
  m.ResourceType = kind; m.EventType = ev; m.UID = uid; m.IP = ip;
  a.ProcessK8s(m);
}
static void requests(alaz::Aggregator& a, const char* from, const char* to, int n, uint32_t status = 200) {
  for (int i = 0; i < n; ++i) {
    alaz::L7Event e;
    e.Status = status; e.Duration = 1000000; e.Protocol = "HTTP"; e.Method = "GET";
    e.Saddr = alaz::Aggregator::ParseIPv4(from, nullptr);
    e.Daddr = alaz::Aggregator::ParseIPv4(to, nullptr);
    e.Sport = (uint16_t)(40000 + i); e.Dport = 80;
    a.ProcessL7(e);
  }
}
static alz_metric metric(uint32_t kind) { alz_metric m{}; m.kind = kind; return m; }
static std::string counts(const alaz::EdgeSeries& s, size_t nm) {   // "5,3,-" : count per point, '-' when absent
  std::string out;
  for (size_t p = 0; p < s.Present.size(); ++p) {
    if (p) out += ",";
    out += s.Present[p] ? std::to_string((long long)s.Values[p * nm]) : std::string("-");
  }
  return out;
}

int main() {
  alaz::AggregatorConfig cfg;
  cfg.MaxEndpoints = 64;
  cfg.MaxPairs = 1u << 12;
  alaz::Aggregator a(nullptr, cfg);
  CHECK(a.Ok(), "create: %s", a.LastError().c_str());
  CHECK(a.SetHistory(4, 1u << 12) == ALZ_OK, "history");
  const std::vector<alz_metric> ms = {metric(ALZ_METRIC_COUNT), metric(ALZ_METRIC_ERR5XX)};
  k8s(a, "Service", "Add", "svc-s", "10.1.0.1");
  k8s(a, "Pod", "Add", "pod-a", "10.0.0.1");
  k8s(a, "Pod", "Add", "pod-b", "10.0.0.2");
  requests(a, "10.0.0.1", "10.1.0.1", 5);
  requests(a, "10.0.0.2", "10.1.0.1", 4, 503);
  CHECK(a.Flush() == ALZ_OK, "flush 1");
  requests(a, "10.0.0.1", "10.1.0.1", 3);
  requests(a, "10.0.0.2", "10.1.0.1", 2);
  k8s(a, "Pod", "Delete", "pod-b", "10.0.0.2");   // pod-b's edges are in windows 1 and 2 only
  CHECK(a.Flush() == ALZ_OK, "flush 2");
  k8s(a, "Pod", "Add", "pod-c", "10.0.0.3");      // must not take pod-b's id while the history may carry it
  requests(a, "10.0.0.1", "10.1.0.1", 1);
  requests(a, "10.0.0.3", "10.1.0.1", 6);
  CHECK(a.Flush() == ALZ_OK, "flush 3");

  // every row of the last window, by id
  std::vector<alaz::EdgeSeries> by_id;
  std::vector<alz_rollup_info> pts;
  CHECK(a.Series(alaz::Aggregator::kLastWindow, 0, 10, ms, &by_id, &pts) == ALZ_OK, "series: %s", a.LastError().c_str());
  CHECK(pts.size() == 3, "points %zu", pts.size());
  for (size_t j = 0; j < 3; ++j)
    CHECK(pts[j].windows == 1 && pts[j].window_first == j + 1 && pts[j].window_last == j + 1 && pts[j].rows_in == 2,
          "point %zu: windows %u first %llu rows %llu", j, pts[j].windows, (unsigned long long)pts[j].window_first,
          (unsigned long long)pts[j].rows_in);
  std::map<std::string, alaz::EdgeSeries> ids;
  for (const auto& s : by_id) ids[s.FromUID + "->" + s.ToUID] = s;
  CHECK(by_id.size() == 2 && ids.count("pod-a->svc-s") && ids.count("pod-c->svc-s"), "rows %zu", by_id.size());
  CHECK(counts(ids["pod-a->svc-s"], 2) == "5,3,1", "pod-a %s", counts(ids["pod-a->svc-s"], 2).c_str());
  CHECK(counts(ids["pod-c->svc-s"], 2) == "-,-,6", "pod-c %s", counts(ids["pod-c->svc-s"], 2).c_str());
  CHECK(ids["pod-a->svc-s"].FromType == "pod" && ids["pod-a->svc-s"].ToType == "service", "types");

  // by UID, in the caller's order, with a deleted pod, an unknown pod and an unknown outbound host
  const std::vector<alaz::EdgeRef> refs = {{"pod", "pod-c", "service", "svc-s"},
                                           {"pod", "pod-b", "service", "svc-s"},
                                           {"pod", "pod-zzz", "service", "svc-s"},
                                           {"pod", "pod-a", "service", "svc-s"},
                                           {"pod", "pod-a", "outbound", "no-such-host.example"}};
  std::vector<alaz::EdgeSeries> by_uid;
  std::vector<alz_rollup_info> pts2;
  CHECK(a.SeriesFor(refs, 0, 10, ms, &by_uid, &pts2) == ALZ_OK, "series for: %s", a.LastError().c_str());
  CHECK(by_uid.size() == refs.size() && pts2.size() == 3, "rows %zu points %zu", by_uid.size(), pts2.size());
  CHECK(memcmp(pts.data(), pts2.data(), 3 * sizeof(alz_rollup_info)) == 0, "points differ");
  CHECK(by_uid[0].Present == ids["pod-c->svc-s"].Present && by_uid[0].Values == ids["pod-c->svc-s"].Values, "pod-c");
  CHECK(by_uid[3].Present == ids["pod-a->svc-s"].Present && by_uid[3].Values == ids["pod-a->svc-s"].Values, "pod-a");
  CHECK(counts(by_uid[1], 2) == "4,2,-", "pod-b %s", counts(by_uid[1], 2).c_str());
  CHECK(by_uid[1].Values[1] == 4.0 && by_uid[1].Values[3] == 0.0, "pod-b 5xx");
  CHECK(counts(by_uid[2], 2) == "-,-,-" && counts(by_uid[4], 2) == "-,-,-", "unknown");
  for (double v : by_uid[2].Values) CHECK(v == 0.0, "unknown value");
  CHECK(by_uid[1].FromUID == "pod-b" && by_uid[4].ToUID == "no-such-host.example", "names");

  // a bad argument comes back as the library's status
  CHECK(a.SeriesFor(refs, 0, 0, ms, &by_uid) == ALZ_E_INVAL, "k = 0");
  CHECK(a.Series(alaz::Aggregator::kLastWindow, 1, 2, ms, &by_id) == ALZ_E_STATE, "no tiers");
  printf("series adapter ok\n");
  return 0;
}
