// reach_adapter_test.cc — the C++ host adapter's Reach and GroupReach (docs/SPEC.md §27) on a three-tier service map:
// pod web calls pods api-1 and api-2 (deployment api), and both call pod db; web -> api-2 and api-2 -> db return 500.
// Reach by UID: down from web every pod, db through api-1 (the parent of smaller index) with the row api-1 -> db; up
// from db every caller, an unknown UID skipped; following 5xx only, web -> api-2 -> db. GroupReach by group name: the
// deployments web -> api -> db, a group name SetGroups never gave skipped, no seed at all giving empty results.
#include <cstdio>
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
static void requests(alaz::Aggregator& a, const char* from, const char* to, int n, uint32_t status) {
  for (int i = 0; i < n; ++i) {
    alaz::L7Event e;
    e.Status = status; e.Duration = 1000000; e.Protocol = "HTTP"; e.Method = "GET";
    e.Saddr = alaz::Aggregator::ParseIPv4(from, nullptr);
    e.Daddr = alaz::Aggregator::ParseIPv4(to, nullptr);
    e.Sport = (uint16_t)(40000 + i); e.Dport = 80;
    a.ProcessL7(e);
  }
}
static std::string names(const std::vector<alaz::ReachNode>& v) {
  std::string s;
  for (const alaz::ReachNode& n : v) s += n.Type + "/" + n.UID + ":" + std::to_string(n.Hops) + " ";
  return s;
}

int main() {
  alaz::AggregatorConfig cfg;
  cfg.MaxEndpoints = 64;
  cfg.MaxPairs = 1u << 12;
  alaz::Aggregator a(nullptr, cfg);
  CHECK(a.Ok(), "create: %s", a.LastError().c_str());
  k8s(a, "Pod", "Add", "web", "10.0.0.10");
  k8s(a, "Pod", "Add", "api-1", "10.0.0.1");
  k8s(a, "Pod", "Add", "api-2", "10.0.0.2");
  k8s(a, "Pod", "Add", "db", "10.0.0.20");
  CHECK(a.SetGroups({{"pod", "web", "web"}, {"pod", "api-1", "api"}, {"pod", "api-2", "api"}, {"pod", "db", "db"}}) ==
            ALZ_OK, "set groups");
  requests(a, "10.0.0.10", "10.0.0.1", 10, 200);
  requests(a, "10.0.0.10", "10.0.0.2", 20, 500);
  requests(a, "10.0.0.1", "10.0.0.20", 5, 200);
  requests(a, "10.0.0.2", "10.0.0.20", 6, 500);
  CHECK(a.Flush() == ALZ_OK, "flush");
  const uint32_t last = alaz::Aggregator::kLastWindow, none = alaz::Aggregator::kReachNone;

  std::vector<alaz::ReachNode> nodes;
  std::vector<alaz::EdgeWindow> rows;
  alz_reach_info info{};
  // dependencies of web
  CHECK(a.Reach(last, {{"pod", "web"}}, ALZ_REACH_DOWN, 64, nullptr, 0.0, &nodes, &rows, &info) == ALZ_OK,
        "down: %s", a.LastError().c_str());
  CHECK(names(nodes) == "pod/web:0 pod/api-1:1 pod/api-2:1 pod/db:2 ", "down nodes %s", names(nodes).c_str());
  CHECK(rows.size() == 4 && info.rows == 4 && info.levels == 2 && info.cut == 0 && info.seeds_found == 1,
        "down rows %zu", rows.size());
  CHECK(nodes[0].Parent == none && nodes[0].Row == none && nodes[3].Parent == 1, "db's parent %u", nodes[3].Parent);
  CHECK(rows[nodes[3].Row].FromUID == "api-1" && rows[nodes[3].Row].ToUID == "db", "db's row");
  CHECK(rows[nodes[2].Row].FromUID == "web" && rows[nodes[2].Row].ToUID == "api-2" && rows[nodes[2].Row].Count == 20,
        "api-2's row");
  // one hop: db is cut off
  CHECK(a.Reach(last, {{"pod", "web"}}, ALZ_REACH_DOWN, 1, nullptr, 0.0, &nodes, &rows, &info) == ALZ_OK, "one hop");
  CHECK(nodes.size() == 3 && rows.size() == 2 && info.cut == 2, "one hop %zu %zu %llu", nodes.size(), rows.size(),
        (unsigned long long)info.cut);
  // callers of db; a UID with no id is skipped
  CHECK(a.Reach(last, {{"pod", "no-such-pod"}, {"pod", "db"}}, ALZ_REACH_UP, 64, nullptr, 0.0, &nodes, &rows,
                &info) == ALZ_OK, "up: %s", a.LastError().c_str());
  CHECK(names(nodes) == "pod/db:0 pod/api-1:1 pod/api-2:1 pod/web:2 ", "up nodes %s", names(nodes).c_str());
  CHECK(info.seeds_found == 1, "seeds found");
  // failing calls only
  alz_metric err{};
  err.kind = ALZ_METRIC_ERR5XX;
  CHECK(a.Reach(last, {{"pod", "web"}}, ALZ_REACH_DOWN, 64, &err, 1.0, &nodes, &rows, &info) == ALZ_OK, "5xx");
  CHECK(names(nodes) == "pod/web:0 pod/api-2:1 pod/db:2 ", "5xx nodes %s", names(nodes).c_str());
  CHECK(rows.size() == 2 && info.traversable == 2, "5xx rows %zu", rows.size());

  // deployments, by group name
  CHECK(a.GroupReach(last, {{"group", "web"}, {"group", "no-such-group"}}, ALZ_REACH_DOWN, 64, nullptr, 0.0, &nodes,
                     &rows, &info) == ALZ_OK, "group down: %s", a.LastError().c_str());
  CHECK(names(nodes) == "group/web:0 group/api:1 group/db:2 ", "group nodes %s", names(nodes).c_str());
  CHECK(rows.size() == 2 && rows[0].FromUID == "web" && rows[0].ToUID == "api" && rows[0].Count == 30 &&
            rows[1].FromUID == "api" && rows[1].ToUID == "db" && rows[1].Count == 11, "group rows %zu", rows.size());
  CHECK(nodes[2].Parent == 1 && rows[nodes[2].Row].ToUID == "db", "group db's parent");
  CHECK(a.GroupReach(last, {{"group", "db"}}, ALZ_REACH_UP, 1, nullptr, 0.0, &nodes, &rows, &info) == ALZ_OK,
        "group up");
  CHECK(names(nodes) == "group/db:0 group/api:1 " && info.cut == 1, "group up %s", names(nodes).c_str());
  // no seed resolves: empty results
  CHECK(a.GroupReach(last, {{"group", "no-such-group"}}, ALZ_REACH_ANY, 3, nullptr, 0.0, &nodes, &rows, &info) ==
            ALZ_OK && nodes.empty() && rows.empty() && info.rows == 0, "no seed");
  CHECK(a.Reach(last, {{"pod", "web"}}, 3, 64, nullptr, 0.0, &nodes, &rows, &info) == ALZ_E_INVAL, "bad dir");
  printf("reach adapter ok\n");
  return 0;
}
