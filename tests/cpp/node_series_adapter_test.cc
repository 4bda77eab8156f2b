// node_series_adapter_test.cc — the C++ host adapter's node series and trends (docs/SPEC.md §22): NodeSeries names a
// rollup's nodes by UID, NodeSeriesFor takes nodes by UID (one with no id is absent everywhere), and NodeTrends ranks
// nodes with their rows and series. A pod deleted in window 2 shows under its own UID up to its deletion, and a pod
// added after it never shows in the windows before it came.
#include <cmath>
#include <cstdio>
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
static void requests(alaz::Aggregator& a, const char* from, const char* to, int n, uint32_t status = 200,
                     const char* host = nullptr) {
  for (int i = 0; i < n; ++i) {
    alaz::L7Event e;
    e.Status = status; e.Duration = 1000000; e.Protocol = "HTTP"; e.Method = "GET";
    e.Saddr = alaz::Aggregator::ParseIPv4(from, nullptr);
    e.Daddr = alaz::Aggregator::ParseIPv4(to, nullptr);
    e.Sport = (uint16_t)(40000 + i); e.Dport = 80;
    if (host) e.Payload = std::string("GET / HTTP/1.1\r\nHost: ") + host + "\r\n\r\n";
    a.ProcessL7(e);
  }
}
static std::vector<double> counts(const std::vector<double>& v, size_t nm) {
  std::vector<double> c;
  for (size_t p = 0; p < v.size() / nm; ++p) c.push_back(v[p * nm]);
  return c;
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
  requests(a, "10.0.0.2", "10.1.0.1", 2, 503);
  requests(a, "10.0.0.1", "8.8.8.8", 3);                              // an outbound IP
  CHECK(a.Flush() == ALZ_OK, "flush 1");
  requests(a, "10.0.0.2", "10.1.0.1", 4);
  requests(a, "10.0.0.1", "93.184.216.34", 2, 200, "example.com");     // keyed by its Host header
  k8s(a, "Pod", "Delete", "pod-b", "10.0.0.2");                       // pod-b is in windows 1 and 2 only
  CHECK(a.Flush() == ALZ_OK, "flush 2");
  k8s(a, "Pod", "Add", "pod-c", "10.0.0.3");   // must not take pod-b's id while the history may carry it
  requests(a, "10.0.0.3", "10.1.0.1", 6);
  CHECK(a.Flush() == ALZ_OK, "flush 3");
  requests(a, "10.0.0.1", "10.1.0.1", 1);
  CHECK(a.Flush() == ALZ_OK, "flush 4");
  CHECK(a.Rollup(0, 4) == ALZ_OK, "rollup: %s", a.LastError().c_str());

  alz_metric count{}, rate{};
  count.kind = ALZ_METRIC_COUNT;
  rate.kind = ALZ_METRIC_ERR_RATE;
  // every node of the rollup, IN side, 4 points
  std::vector<alaz::NodeSeriesRow> ser;
  std::vector<alz_rollup_info> pts;
  CHECK(a.NodeSeries(ALZ_ROLLUP_WINDOWS, ALZ_SIDE_IN, 0, 4, {count, rate}, &ser, &pts) == ALZ_OK, "series: %s",
        a.LastError().c_str());
  std::map<std::string, alaz::NodeSeriesRow> by;
  for (const auto& r : ser) by[r.Type + "/" + r.UID] = r;
  CHECK(ser.size() == 6 && by.size() == 6 && pts.size() == 4, "nodes %zu points %zu", ser.size(), pts.size());
  for (const auto& p : pts) CHECK(p.windows == 1, "one window per point");
  const alaz::NodeSeriesRow& s = by["service/svc-s"];
  CHECK(s.Present == std::vector<uint8_t>({1, 1, 1, 1}), "svc-s present");
  CHECK(counts(s.Values, 2) == std::vector<double>({7.0, 4.0, 6.0, 1.0}), "svc-s counts");
  CHECK(s.Values[1] == 2.0 / 7.0 && s.Values[3] == 0.0, "svc-s 5xx rate");
  CHECK(by["outbound/8.8.8.8"].Present == std::vector<uint8_t>({1, 0, 0, 0}), "outbound ip");
  CHECK(counts(by["outbound/example.com"].Values, 2) == std::vector<double>({0.0, 2.0, 0.0, 0.0}), "host-keyed");
  CHECK(by["pod/pod-a"].Present == std::vector<uint8_t>({0, 0, 0, 0}), "pod-a is never called");

  // by UID, OUT side: the deleted pod up to its deletion, the pod added after it from its first window, a pod with no
  // id, a node seen only on the other side
  std::vector<alaz::NodeRef> refs = {{"pod", "pod-b"}, {"pod", "pod-c"}, {"pod", "ghost"}, {"service", "svc-s"},
                                     {"pod", "pod-a"}, {"pod", "pod-b"}};
  CHECK(a.NodeSeriesFor(refs, ALZ_SIDE_OUT, 0, 4, {count}, &ser, &pts) == ALZ_OK, "for: %s", a.LastError().c_str());
  CHECK(ser.size() == 6 && pts.size() == 4, "for %zu", ser.size());
  CHECK(ser[0].UID == "pod-b" && ser[0].Present == std::vector<uint8_t>({1, 1, 0, 0}) &&
            ser[0].Values == std::vector<double>({2.0, 4.0, 0.0, 0.0}), "pod-b");
  CHECK(ser[1].Present == std::vector<uint8_t>({0, 0, 1, 0}) && ser[1].Values[2] == 6.0, "pod-c");
  CHECK(ser[2].Type == "pod" && ser[2].UID == "ghost" && ser[2].Present == std::vector<uint8_t>(4, 0) &&
            ser[2].Values == std::vector<double>(4, 0.0), "ghost");
  CHECK(ser[3].Present == std::vector<uint8_t>(4, 0), "svc-s has no OUT rows");
  CHECK(ser[4].Values == std::vector<double>({8.0, 2.0, 0.0, 1.0}), "pod-a");
  CHECK(ser[5].Present == ser[0].Present && ser[5].Values == ser[0].Values, "duplicate");

  // the nodes whose IN count fell most: the last window against the three before
  alz_trend t{};
  t.stat = ALZ_TREND_SHIFT;
  t.direction = ALZ_TREND_FALLING;
  t.absent = ALZ_TREND_ABSENT_ZERO;
  t.recent = 1;
  std::vector<alaz::NodeTrend> top;
  CHECK(a.NodeTrends(ALZ_ROLLUP_WINDOWS, ALZ_SIDE_IN, 0, 4, count, t, 2, -HUGE_VAL, &top, &pts) == ALZ_OK,
        "trends: %s", a.LastError().c_str());
  CHECK(top.size() == 2 && pts.size() == 4, "top %zu", top.size());
  CHECK(top[0].Node.Type == "service" && top[0].Node.UID == "svc-s" && top[0].Valid && top[0].Used == 4, "first");
  CHECK(top[0].Trend == 17.0 / 3.0 - 1.0 && top[0].Recent == 1.0 && top[0].Before == 17.0 / 3.0, "svc-s trend");
  CHECK(top[0].Node.In.count == 18 && top[0].Node.InEdges == 3, "svc-s row");
  CHECK(top[0].Values == std::vector<double>({7.0, 4.0, 6.0, 1.0}), "svc-s series");
  CHECK(top[1].Node.UID == "8.8.8.8" && top[1].Trend == 1.0 && top[1].Present == std::vector<uint8_t>({1, 0, 0, 0}),
        "second %s", top[1].Node.UID.c_str());

  // a bad argument comes back as the library's status
  CHECK(a.NodeTrends(ALZ_ROLLUP_WINDOWS, ALZ_SIDE_IN, 0, 4, count, t, 0, 0.0, &top) == ALZ_E_INVAL, "top = 0");
  CHECK(a.NodeSeries(ALZ_ROLLUP_WINDOWS, 2, 0, 4, {count}, &ser) == ALZ_E_INVAL, "side 2");
  CHECK(a.NodeSeries(ALZ_ROLLUP_SPAN, ALZ_SIDE_IN, 0, 4, {count}, &ser) == ALZ_E_STATE, "no span rollup");
  printf("node series adapter ok\n");
  return 0;
}
