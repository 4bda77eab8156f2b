// group_changes_adapter_test.cc — the C++ host adapter's group changes (docs/SPEC.md §25) through a rollout: web
// calls deployment api's pods api-1 and api-2 in window 1, which is pinned; the rollout replaces them with api-3 and
// api-4 before window 2. Per pod, NodeChanges lists api-1 and api-2 as GONE and api-3 and api-4 as NEW; per
// deployment, GroupNodeChanges lists group/api as BOTH with its count and p99 change, and GroupChanges lists
// web -> api as BOTH. The deleted pods stay members under PinBaseline's hold; api-3 and api-4 have no id when
// SetGroups names them.
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
static void requests(alaz::Aggregator& a, const char* from, const char* to, int n, uint64_t duration_ns) {
  for (int i = 0; i < n; ++i) {
    alaz::L7Event e;
    e.Status = 200; e.Duration = duration_ns; e.Protocol = "HTTP"; e.Method = "GET";
    e.Saddr = alaz::Aggregator::ParseIPv4(from, nullptr);
    e.Daddr = alaz::Aggregator::ParseIPv4(to, nullptr);
    e.Sport = (uint16_t)(40000 + i); e.Dport = 80;
    a.ProcessL7(e);
  }
}

int main() {
  alaz::AggregatorConfig cfg;
  cfg.MaxEndpoints = 64;
  cfg.MaxPairs = 1u << 12;
  alaz::Aggregator a(nullptr, cfg);
  CHECK(a.Ok(), "create: %s", a.LastError().c_str());
  CHECK(a.SetGroups({{"pod", "api-1", "api"}, {"pod", "api-2", "api"}, {"pod", "api-3", "api"},
                     {"pod", "api-4", "api"}, {"pod", "web", "web"}}) == ALZ_OK, "set groups");
  k8s(a, "Pod", "Add", "web", "10.0.0.10");
  k8s(a, "Pod", "Add", "api-1", "10.0.0.1");
  k8s(a, "Pod", "Add", "api-2", "10.0.0.2");
  requests(a, "10.0.0.10", "10.0.0.1", 60, 1000000);     // 1 ms
  requests(a, "10.0.0.10", "10.0.0.2", 35, 2000000);     // 2 ms
  CHECK(a.Flush() == ALZ_OK, "flush 1");
  CHECK(a.PinBaseline(alaz::Aggregator::kLastWindow) == ALZ_OK, "pin: %s", a.LastError().c_str());
  k8s(a, "Pod", "Delete", "api-1", "10.0.0.1");          // the rollout
  k8s(a, "Pod", "Delete", "api-2", "10.0.0.2");
  k8s(a, "Pod", "Add", "api-3", "10.0.0.3");
  k8s(a, "Pod", "Add", "api-4", "10.0.0.4");
  requests(a, "10.0.0.10", "10.0.0.3", 3, 16000000);     // 16 ms
  requests(a, "10.0.0.10", "10.0.0.4", 2, 64000000);     // 64 ms
  CHECK(a.Flush() == ALZ_OK, "flush 2");

  alz_metric count{}, p99{};
  count.kind = ALZ_METRIC_COUNT;
  p99.kind = ALZ_METRIC_QUANTILE;
  p99.q = 0.99;
  const uint32_t last = alaz::Aggregator::kLastWindow;
  std::vector<alaz::NodeChange> ch;
  alz_change_info info{};
  CHECK(a.NodeChanges(last, ALZ_SIDE_IN, count, ALZ_CHANGE_DELTA, 7, 0, 0.0, &ch, &info) == ALZ_OK, "pods: %s",
        a.LastError().c_str());
  std::map<std::string, alaz::NodeChange> by;
  for (const auto& c : ch) by[c.Type + "/" + c.UID] = c;
  CHECK(ch.size() == 4 && info.both == 0, "pods %zu", ch.size());
  CHECK(by["pod/api-1"].Presence == ALZ_PRESENT_GONE && by["pod/api-2"].Presence == ALZ_PRESENT_GONE, "gone");
  CHECK(by["pod/api-3"].Presence == ALZ_PRESENT_NEW && by["pod/api-4"].Presence == ALZ_PRESENT_NEW, "new");

  CHECK(a.GroupNodeChanges(last, ALZ_SIDE_IN, count, ALZ_CHANGE_DELTA, 7, 0, 0.0, &ch, &info) == ALZ_OK,
        "group nodes: %s", a.LastError().c_str());
  CHECK(ch.size() == 1 && ch[0].Type == "group" && ch[0].UID == "api" && ch[0].Presence == ALZ_PRESENT_BOTH &&
            ch[0].Value == 5.0 && ch[0].BaseValue == 95.0 && ch[0].Change == -90.0, "group/api count %zu", ch.size());
  CHECK(info.both == 1 && info.source_rows == 1 && info.base_rows == 1, "group info");
  CHECK(a.GroupNodeChanges(last, ALZ_SIDE_IN, p99, ALZ_CHANGE_DELTA, 7, 0, 0.0, &ch) == ALZ_OK, "p99");
  CHECK(ch.size() == 1 && ch[0].UID == "api" && ch[0].Presence == ALZ_PRESENT_BOTH && ch[0].Value > 16e6 &&
            ch[0].BaseValue < 4e6 && ch[0].Change == ch[0].Value - ch[0].BaseValue, "p99 %g %g", ch[0].Value,
        ch[0].BaseValue);
  std::vector<alaz::NodeChange> top;
  CHECK(a.GroupNodeChanges(last, ALZ_SIDE_OUT, count, ALZ_CHANGE_DROP, 7, 5, 0.0, &top) == ALZ_OK, "top");
  CHECK(top.size() == 1 && top[0].Type == "group" && top[0].UID == "web" && top[0].Change == 90.0, "web out");

  std::vector<alaz::EdgeChange> edges;
  CHECK(a.GroupChanges(last, count, ALZ_CHANGE_DELTA, 7, 0, 0.0, &edges, &info) == ALZ_OK, "group edges: %s",
        a.LastError().c_str());
  CHECK(edges.size() == 1 && edges[0].FromType == "group" && edges[0].FromUID == "web" && edges[0].ToType == "group" &&
            edges[0].ToUID == "api" && edges[0].Presence == ALZ_PRESENT_BOTH && edges[0].Change == -90.0,
        "web -> api %zu", edges.size());
  std::vector<alaz::EdgeChange> pod_edges;
  CHECK(a.Changes(last, count, ALZ_CHANGE_DELTA, 7, 0, 0.0, &pod_edges) == ALZ_OK, "pod edges");
  for (const auto& e : pod_edges) CHECK(e.Presence != ALZ_PRESENT_BOTH, "a pod edge %s is BOTH", e.ToUID.c_str());

  CHECK(a.ClearBaseline() == ALZ_OK, "clear");
  CHECK(a.GroupChanges(last, count, ALZ_CHANGE_DELTA, 7, 0, 0.0, &edges) == ALZ_E_STATE, "no baseline");
  printf("group changes adapter ok\n");
  return 0;
}
