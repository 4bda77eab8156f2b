// groups_adapter_test.cc — the C++ host adapter's groups (docs/SPEC.md §24) through a rolling deploy: deployment api
// runs pods api-1 and api-2 in window 1 and api-3 and api-4 in window 2, and web calls whichever run. Over the
// two-window rollup, grouped by owner, api is one node: its IN count is the four pods' sum, its p99 is the quantile of
// their summed histogram (which is no pod's p99), and the pods deleted after window 1 stay in api under SetHistory's id
// hold. The members api-3 and api-4 have no id when SetGroups names them; the map is sent again once they do.
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
static std::string key(const alaz::NodeWindow& w) { return w.Type + "/" + w.UID; }

int main() {
  alaz::AggregatorConfig cfg;
  cfg.MaxEndpoints = 64;
  cfg.MaxPairs = 1u << 12;
  alaz::Aggregator a(nullptr, cfg);
  CHECK(a.Ok(), "create: %s", a.LastError().c_str());
  CHECK(a.SetHistory(4, 1u << 12) == ALZ_OK, "history");
  CHECK(a.SetGroups({{"pod", "api-1", "api"}, {"pod", "api-2", "api"}, {"pod", "api-3", "api"},
                     {"pod", "api-4", "api"}, {"pod", "web", "web"}}) == ALZ_OK, "set groups");
  k8s(a, "Pod", "Add", "web", "10.0.0.10");
  k8s(a, "Pod", "Add", "api-1", "10.0.0.1");
  k8s(a, "Pod", "Add", "api-2", "10.0.0.2");
  requests(a, "10.0.0.10", "10.0.0.1", 60, 1000000);     // 1 ms
  requests(a, "10.0.0.10", "10.0.0.2", 35, 2000000);     // 2 ms
  k8s(a, "Pod", "Delete", "api-1", "10.0.0.1");          // the rollout replaces both pods after window 1
  k8s(a, "Pod", "Delete", "api-2", "10.0.0.2");
  CHECK(a.Flush() == ALZ_OK, "flush 1");
  std::vector<alaz::EdgeWindow> edges;
  CHECK(a.GroupEdges(alaz::Aggregator::kLastWindow, &edges) == ALZ_OK, "group edges 1: %s", a.LastError().c_str());
  CHECK(edges.size() == 1 && edges[0].FromType == "group" && edges[0].FromUID == "web" && edges[0].ToUID == "api" &&
            edges[0].Count == 95, "window 1 %zu", edges.size());
  k8s(a, "Pod", "Add", "api-3", "10.0.0.3");
  k8s(a, "Pod", "Add", "api-4", "10.0.0.4");
  requests(a, "10.0.0.10", "10.0.0.3", 3, 16000000);     // 16 ms
  requests(a, "10.0.0.10", "10.0.0.4", 2, 64000000);     // 64 ms
  CHECK(a.Flush() == ALZ_OK, "flush 2");
  CHECK(a.Rollup(0, 2) == ALZ_OK, "rollup: %s", a.LastError().c_str());

  alz_metric count{}, p99{};
  count.kind = ALZ_METRIC_COUNT;
  p99.kind = ALZ_METRIC_QUANTILE;
  p99.q = 0.99;
  alz_group_info info{};
  CHECK(a.GroupEdges(ALZ_ROLLUP_WINDOWS, &edges, &info) == ALZ_OK, "group edges: %s", a.LastError().c_str());
  CHECK(edges.size() == 1 && edges[0].FromUID == "web" && edges[0].ToType == "group" && edges[0].ToUID == "api" &&
            edges[0].Count == 100, "rollup edges %zu", edges.size());
  CHECK(info.source_rows == 4 && info.mapped_ends == 8 && info.edges == 1 && info.internal == 0, "info");

  std::vector<alaz::NodeWindow> groups, pods;
  CHECK(a.GroupNodes(ALZ_ROLLUP_WINDOWS, ALZ_SIDE_IN, {count, p99}, &groups) == ALZ_OK, "group nodes");
  CHECK(groups.size() == 2 && key(groups[0]) == "group/api" && key(groups[1]) == "group/web", "groups %zu",
        groups.size());
  const alaz::NodeWindow& api = groups[0];
  CHECK(api.InEdges == 1 && api.In.count == 100 && api.Values[0] == 100.0, "api in %llu",
        (unsigned long long)api.In.count);
  CHECK(a.Nodes(ALZ_ROLLUP_WINDOWS, ALZ_SIDE_IN, {count, p99}, &pods) == ALZ_OK, "pod nodes");
  std::map<std::string, alaz::NodeWindow> by;
  for (const auto& w : pods) by[key(w)] = w;
  uint64_t sum = 0;
  for (const char* p : {"pod/api-1", "pod/api-2", "pod/api-3", "pod/api-4"}) {   // deleted pods under their own UIDs
    CHECK(by.count(p) == 1, "%s missing", p);
    sum += by[p].In.count;
    CHECK(by[p].Values[1] != api.Values[1], "%s p99 %g equals the group's", p, by[p].Values[1]);
  }
  CHECK(sum == api.In.count, "sum %llu", (unsigned long long)sum);

  std::vector<alaz::NodeWindow> top;
  alz_top_info tinfo{};
  CHECK(a.TopGroupNodes(ALZ_ROLLUP_WINDOWS, ALZ_SIDE_IN, p99, 20, 0.0, &top, &tinfo) == ALZ_OK, "top");
  CHECK(top.size() == 2 && key(top[0]) == "group/api" && top[0].Values[0] == api.Values[1] && tinfo.scored == 2,
        "top %zu", top.size());

  // an empty map: the pods again, as Nodes names them
  CHECK(a.SetGroups({}) == ALZ_OK, "clear");
  CHECK(a.GroupNodes(ALZ_ROLLUP_WINDOWS, ALZ_SIDE_IN, {count}, &groups) == ALZ_OK, "cleared");
  CHECK(groups.size() == pods.size() && key(groups[0]) == key(pods[0]), "cleared %zu", groups.size());
  CHECK(a.TopGroupNodes(ALZ_ROLLUP_WINDOWS, ALZ_SIDE_IN, count, 0, 0.0, &top) == ALZ_E_INVAL, "k = 0");
  CHECK(a.GroupEdges(ALZ_ROLLUP_SPAN, &edges) == ALZ_E_STATE, "no span rollup");
  printf("groups adapter ok\n");
  return 0;
}
