// trends_adapter_test.cc — the C++ host adapter's edge trends (docs/SPEC.md §20): Trends ranks a source's rows by a
// trend over the window history and names them by UID, each with its series. A pod deleted mid-history keeps its own
// UID over the points it was seen in, and a pod added later never shows under it.
#include <cmath>
#include <cstdio>
#include <cstring>
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
static std::string counts(const alaz::EdgeTrend& t) {   // "5,3,-" : the value per point, '-' when absent
  std::string out;
  for (size_t p = 0; p < t.Present.size(); ++p) {
    if (p) out += ",";
    out += t.Present[p] ? std::to_string((long long)t.Values[p]) : std::string("-");
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
  k8s(a, "Service", "Add", "svc-s", "10.1.0.1");
  k8s(a, "Pod", "Add", "pod-a", "10.0.0.1");
  k8s(a, "Pod", "Add", "pod-b", "10.0.0.2");
  requests(a, "10.0.0.1", "10.1.0.1", 5);
  requests(a, "10.0.0.2", "10.1.0.1", 2);
  CHECK(a.Flush() == ALZ_OK, "flush 1");
  requests(a, "10.0.0.1", "10.1.0.1", 3);
  requests(a, "10.0.0.2", "10.1.0.1", 6);
  k8s(a, "Pod", "Delete", "pod-b", "10.0.0.2");   // pod-b's edge is in windows 1 and 2 only
  CHECK(a.Flush() == ALZ_OK, "flush 2");
  k8s(a, "Pod", "Add", "pod-c", "10.0.0.3");      // must not take pod-b's id while the history may carry it
  requests(a, "10.0.0.1", "10.1.0.1", 1);
  requests(a, "10.0.0.3", "10.1.0.1", 9);
  CHECK(a.Flush() == ALZ_OK, "flush 3");
  CHECK(a.Rollup(0, 3) == ALZ_OK, "rollup: %s", a.LastError().c_str());   // every edge of the three windows

  alz_metric count{};
  count.kind = ALZ_METRIC_COUNT;
  // the count's slope over the three points, skipping absent ones: pod-b 2 -> 6 is +4 per point, pod-a 5, 3, 1 is -2,
  // pod-c (one point) has none
  alz_trend slope{};
  slope.stat = ALZ_TREND_SLOPE;
  slope.recent = 1;
  std::vector<alaz::EdgeTrend> top;
  std::vector<alz_rollup_info> pts;
  CHECK(a.Trends(ALZ_ROLLUP_WINDOWS, 0, 3, count, slope, 10, -HUGE_VAL, &top, &pts) == ALZ_OK, "trends: %s",
        a.LastError().c_str());
  CHECK(pts.size() == 3, "points %zu", pts.size());
  for (size_t j = 0; j < 3; ++j) CHECK(pts[j].windows == 1 && pts[j].window_first == j + 1, "point %zu", j);
  CHECK(top.size() == 2, "rows %zu", top.size());
  CHECK(top[0].FromUID == "pod-b" && top[0].ToUID == "svc-s" && top[0].FromType == "pod" && top[0].ToType == "service",
        "first %s -> %s", top[0].FromUID.c_str(), top[0].ToUID.c_str());
  CHECK(top[0].Valid && top[0].Trend == 4.0 && top[0].Used == 2 && counts(top[0]) == "2,6,-", "pod-b %g %s",
        top[0].Trend, counts(top[0]).c_str());
  CHECK(top[1].FromUID == "pod-a" && top[1].Trend == -2.0 && counts(top[1]) == "5,3,1", "pod-a %g %s", top[1].Trend,
        counts(top[1]).c_str());

  // absent points as zero, the last point against the two before: pod-c 0, 0 -> 9 is a new edge (+inf), pod-b 4 -> 0
  // falls most
  alz_trend ratio{};
  ratio.stat = ALZ_TREND_RATIO;
  ratio.absent = ALZ_TREND_ABSENT_ZERO;
  ratio.recent = 1;
  CHECK(a.Trends(ALZ_ROLLUP_WINDOWS, 0, 3, count, ratio, 1, 0.0, &top) == ALZ_OK, "ratio");
  CHECK(top.size() == 1 && top[0].FromUID == "pod-c" && std::isinf(top[0].Trend) && counts(top[0]) == "-,-,9",
        "pod-c %s", top.empty() ? "" : top[0].FromUID.c_str());
  ratio.direction = ALZ_TREND_FALLING;
  CHECK(a.Trends(ALZ_ROLLUP_WINDOWS, 0, 3, count, ratio, 3, -HUGE_VAL, &top) == ALZ_OK, "falling");
  CHECK(top.size() == 3 && top[0].FromUID == "pod-b" && std::isinf(top[0].Trend) && top[0].Before == 4.0 &&
            top[0].Recent == 0.0 && top[1].FromUID == "pod-a" && top[1].Trend == 4.0,
        "falling %s %g", top.empty() ? "" : top[0].FromUID.c_str(), top.empty() ? 0.0 : top[0].Trend);

  // a bad argument comes back as the library's status
  CHECK(a.Trends(ALZ_ROLLUP_WINDOWS, 0, 3, count, ratio, 0, 0.0, &top) == ALZ_E_INVAL, "top = 0");
  CHECK(a.Trends(alaz::Aggregator::kLastWindow, 0, 1, count, ratio, 5, 0.0, &top) == ALZ_E_INVAL, "k = 1");
  CHECK(a.Trends(alaz::Aggregator::kLastWindow, 1, 3, count, slope, 5, 0.0, &top) == ALZ_E_STATE, "no tiers");
  printf("trends adapter ok\n");
  return 0;
}
