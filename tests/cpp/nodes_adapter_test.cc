// nodes_adapter_test.cc — the C++ host adapter's node metrics (docs/SPEC.md §21): Nodes and TopNodes group a rollup's
// rows by node and name each node by UID: a service, pods, an outbound IP and a Host-keyed destination. A pod deleted
// inside the rollup's span keeps its own UID, and a pod added after it never shows under it.
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
static std::string key(const alaz::NodeWindow& w) { return w.Type + "/" + w.UID; }

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
  requests(a, "10.0.0.1", "8.8.8.8", 3);                        // an outbound IP
  CHECK(a.Flush() == ALZ_OK, "flush 1");
  requests(a, "10.0.0.2", "10.1.0.1", 4);
  requests(a, "10.0.0.1", "93.184.216.34", 2, 200, "example.com");   // keyed by its Host header
  k8s(a, "Pod", "Delete", "pod-b", "10.0.0.2");                 // pod-b is in windows 1 and 2 only
  CHECK(a.Flush() == ALZ_OK, "flush 2");
  k8s(a, "Pod", "Add", "pod-c", "10.0.0.3");                    // must not take pod-b's id while the history may carry it
  requests(a, "10.0.0.3", "10.1.0.1", 6);
  CHECK(a.Flush() == ALZ_OK, "flush 3");
  CHECK(a.Rollup(0, 3) == ALZ_OK, "rollup: %s", a.LastError().c_str());

  alz_metric count{}, rate{};
  count.kind = ALZ_METRIC_COUNT;
  rate.kind = ALZ_METRIC_ERR_RATE;
  std::vector<alaz::NodeWindow> nodes;
  CHECK(a.Nodes(ALZ_ROLLUP_WINDOWS, ALZ_SIDE_IN, {count, rate}, &nodes) == ALZ_OK, "nodes: %s", a.LastError().c_str());
  std::map<std::string, alaz::NodeWindow> by;
  for (const auto& w : nodes) by[key(w)] = w;
  CHECK(nodes.size() == 6 && by.size() == 6, "nodes %zu", nodes.size());
  const alaz::NodeWindow& s = by["service/svc-s"];
  CHECK(s.InEdges == 3 && s.OutEdges == 0 && s.In.count == 17 && s.In.err5xx == 2, "svc-s %u %llu", s.InEdges,
        (unsigned long long)s.In.count);
  CHECK(s.Values.size() == 2 && s.Values[0] == 17.0 && s.Values[1] == 2.0 / 17.0, "svc-s values");
  const alaz::NodeWindow& pa = by["pod/pod-a"];
  CHECK(pa.OutEdges == 3 && pa.InEdges == 0 && pa.Out.count == 10 && pa.Values[0] == 0.0, "pod-a");
  const alaz::NodeWindow& pb = by["pod/pod-b"];   // deleted in window 2, still under its own UID
  CHECK(pb.OutEdges == 1 && pb.Out.count == 6 && pb.Out.err5xx == 2, "pod-b %u %llu", pb.OutEdges,
        (unsigned long long)pb.Out.count);
  CHECK(by["pod/pod-c"].Out.count == 6, "pod-c");
  CHECK(by["outbound/8.8.8.8"].In.count == 3 && by["outbound/8.8.8.8"].InEdges == 1, "outbound ip");
  CHECK(by["outbound/example.com"].In.count == 2, "host-keyed");

  // the busiest callers, then the services by 5xx rate
  std::vector<alaz::NodeWindow> top;
  alz_top_info info{};
  CHECK(a.TopNodes(ALZ_ROLLUP_WINDOWS, ALZ_SIDE_OUT, count, 2, 0.0, &top, &info) == ALZ_OK, "top out");
  CHECK(top.size() == 2 && key(top[0]) == "pod/pod-a" && top[0].Values[0] == 10.0 && info.scored == 6 &&
            info.above == 6, "top out %s", top.empty() ? "" : key(top[0]).c_str());
  CHECK(key(top[1]) == "pod/pod-b" || key(top[1]) == "pod/pod-c", "second %s", key(top[1]).c_str());
  CHECK(a.TopNodes(ALZ_ROLLUP_WINDOWS, ALZ_SIDE_IN, rate, 10, 0.1, &top, &info) == ALZ_OK, "top rate");
  CHECK(top.size() == 1 && key(top[0]) == "service/svc-s" && info.above == 1, "rate");

  // the last window alone: pod-b is gone, pod-c calls the service
  CHECK(a.Nodes(alaz::Aggregator::kLastWindow, ALZ_SIDE_OUT, {count}, &nodes) == ALZ_OK, "window");
  CHECK(nodes.size() == 2 && key(nodes[0]) == "pod/pod-c" && nodes[0].Values[0] == 6.0, "window %zu", nodes.size());

  // a bad argument comes back as the library's status
  CHECK(a.TopNodes(ALZ_ROLLUP_WINDOWS, ALZ_SIDE_IN, count, 0, 0.0, &top) == ALZ_E_INVAL, "k = 0");
  CHECK(a.Nodes(ALZ_ROLLUP_WINDOWS, 2, {count}, &nodes) == ALZ_E_INVAL, "side 2");
  CHECK(a.Nodes(ALZ_ROLLUP_SPAN, ALZ_SIDE_IN, {count}, &nodes) == ALZ_E_STATE, "no span rollup");
  printf("nodes adapter ok\n");
  return 0;
}
