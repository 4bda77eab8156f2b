// node_changes_adapter_test.cc — the C++ host adapter's node changes (docs/SPEC.md §23): NodeChanges names the nodes
// of a window and of the pinned baseline by UID. A pod deleted after the pin is GONE under its own UID, a pod added
// after it is NEW under its own (PinBaseline's hold keeps the deleted pod's id from going to it), a caller on both
// sides is BOTH, and the top call ranks by change.
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

int main() {
  alaz::AggregatorConfig cfg;
  cfg.MaxEndpoints = 64;
  cfg.MaxPairs = 1u << 12;
  alaz::Aggregator a(nullptr, cfg);
  CHECK(a.Ok(), "create: %s", a.LastError().c_str());
  k8s(a, "Service", "Add", "svc-s", "10.1.0.1");
  k8s(a, "Pod", "Add", "pod-a", "10.0.0.1");
  k8s(a, "Pod", "Add", "pod-b", "10.0.0.2");
  requests(a, "10.0.0.1", "10.1.0.1", 5);
  requests(a, "10.0.0.2", "10.1.0.1", 2, 503);
  CHECK(a.Flush() == ALZ_OK, "flush 1");
  alz_rollup_info pinned{};
  CHECK(a.PinBaseline(alaz::Aggregator::kLastWindow, &pinned) == ALZ_OK, "pin: %s", a.LastError().c_str());
  CHECK(pinned.windows == 1, "pinned windows");
  k8s(a, "Pod", "Delete", "pod-b", "10.0.0.2");
  k8s(a, "Pod", "Add", "pod-c", "10.0.0.3");   // must not take pod-b's id while the baseline carries it
  requests(a, "10.0.0.1", "10.1.0.1", 3);
  requests(a, "10.0.0.3", "10.1.0.1", 6);
  CHECK(a.Flush() == ALZ_OK, "flush 2");

  alz_metric count{}, rate{};
  count.kind = ALZ_METRIC_COUNT;
  rate.kind = ALZ_METRIC_ERR_RATE;
  std::vector<alaz::NodeChange> ch;
  alz_change_info info{};
  // the callers (OUT side): pod-a in both, pod-b gone, pod-c new, in node order
  CHECK(a.NodeChanges(alaz::Aggregator::kLastWindow, ALZ_SIDE_OUT, count, ALZ_CHANGE_DELTA, 7, 0, 0.0, &ch, &info) ==
            ALZ_OK, "changes: %s", a.LastError().c_str());
  std::map<std::string, alaz::NodeChange> by;
  for (const auto& c : ch) by[c.Type + "/" + c.UID] = c;
  CHECK(ch.size() == 3 && by.size() == 3, "callers %zu", ch.size());
  CHECK(info.both == 1 && info.added == 1 && info.gone == 1 && info.source_rows == 2 && info.base_rows == 2, "info");
  const alaz::NodeChange& pa = by["pod/pod-a"];
  CHECK(pa.Presence == ALZ_PRESENT_BOTH && pa.Value == 3.0 && pa.BaseValue == 5.0 && pa.Change == -2.0, "pod-a");
  const alaz::NodeChange& pb = by["pod/pod-b"];
  CHECK(pb.Presence == ALZ_PRESENT_GONE && pb.Value == 0.0 && pb.BaseValue == 2.0 && pb.Change == -2.0, "pod-b");
  const alaz::NodeChange& pc = by["pod/pod-c"];
  CHECK(pc.Presence == ALZ_PRESENT_NEW && pc.Value == 6.0 && pc.BaseValue == 0.0 && pc.Change == 6.0, "pod-c");
  // the served side (IN): only the service, whose error rate fell from 2/7 to 0
  CHECK(a.NodeChanges(alaz::Aggregator::kLastWindow, ALZ_SIDE_IN, rate, ALZ_CHANGE_DROP, 7, 0, 0.0, &ch, &info) ==
            ALZ_OK, "served");
  CHECK(ch.size() == 1 && ch[0].Type == "service" && ch[0].UID == "svc-s" && ch[0].Presence == ALZ_PRESENT_BOTH,
        "svc-s");
  CHECK(ch[0].Value == 0.0 && ch[0].BaseValue == 2.0 / 7.0 && ch[0].Change == 2.0 / 7.0, "svc-s rate");
  // the top caller by count change, and only the new and gone callers
  CHECK(a.NodeChanges(alaz::Aggregator::kLastWindow, ALZ_SIDE_OUT, count, ALZ_CHANGE_DELTA, 7, 1, -INFINITY, &ch,
                      &info) == ALZ_OK, "top");
  CHECK(ch.size() == 1 && ch[0].UID == "pod-c" && info.above == 3, "top caller");
  CHECK(a.NodeChanges(alaz::Aggregator::kLastWindow, ALZ_SIDE_OUT, count, ALZ_CHANGE_DELTA,
                      ALZ_PRESENT_NEW | ALZ_PRESENT_GONE, 0, 0.0, &ch, &info) == ALZ_OK, "filtered");
  CHECK(ch.size() == 2 && info.listed == 2 && info.both == 1, "filtered count");
  CHECK(a.ClearBaseline() == ALZ_OK, "clear");
  CHECK(a.NodeChanges(alaz::Aggregator::kLastWindow, ALZ_SIDE_OUT, count, ALZ_CHANGE_DELTA, 7, 0, 0.0, &ch) ==
            ALZ_E_STATE, "no baseline");
  printf("node changes adapter ok\n");
  return 0;
}
