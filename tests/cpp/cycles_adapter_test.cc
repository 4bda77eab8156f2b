// cycles_adapter_test.cc — the C++ host adapter's Cycles and GroupCycles (docs/SPEC.md §28) on a small service map:
// pod web calls pods api-1 and api-2 (deployment api), api-1 calls db and api-2, and db calls api-1 back with 500s.
// Cycles: the loop {api-1, db} with depth 1 and height 1 under web, the two rows inside it, every node with min_size
// 0, no loop along 5xx only. GroupCycles: the deployments api and db call each other; api's internal row is a self row.
#include <algorithm>
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
static std::string names(const std::vector<alaz::CycleNode>& v) {
  std::string s;
  for (const alaz::CycleNode& n : v)
    s += n.Type + "/" + n.UID + ":" + std::to_string(n.Size) + "," + std::to_string(n.Depth) + "," +
         std::to_string(n.Height) + " ";
  return s;
}
static std::string pairs(const std::vector<alaz::EdgeWindow>& v) {
  std::vector<std::string> p;
  for (const alaz::EdgeWindow& e : v) p.push_back(e.FromUID + ">" + e.ToUID);
  std::sort(p.begin(), p.end());
  std::string s;
  for (const std::string& x : p) s += x + " ";
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
  requests(a, "10.0.0.1", "10.0.0.2", 4, 200);
  requests(a, "10.0.0.20", "10.0.0.1", 3, 500);
  CHECK(a.Flush() == ALZ_OK, "flush");
  const uint32_t last = alaz::Aggregator::kLastWindow;

  std::vector<alaz::CycleNode> nodes;
  std::vector<alaz::EdgeWindow> rows;
  alz_cycle_info info{};
  // the services on a loop
  CHECK(a.Cycles(last, nullptr, 0.0, 2, &nodes, &rows, &info) == ALZ_OK, "cycles: %s", a.LastError().c_str());
  CHECK(nodes.size() == 2 && nodes[0].Component == nodes[1].Component, "loop %s", names(nodes).c_str());
  CHECK((names(nodes) == "pod/api-1:2,1,1 pod/db:2,1,1 " || names(nodes) == "pod/db:2,1,1 pod/api-1:2,1,1 "),
        "loop %s", names(nodes).c_str());
  CHECK(pairs(rows) == "api-1>db db>api-1 ", "loop rows %s", pairs(rows).c_str());
  CHECK(info.rows == 5 && info.nodes == 4 && info.components == 3 && info.cyclic == 1 && info.cyclic_nodes == 2 &&
            info.largest == 2 && info.cycle_rows == 2 && info.depth == 2 && info.self_rows == 0, "info");
  // every node, with its layer
  CHECK(a.Cycles(last, nullptr, 0.0, 0, &nodes, &rows, &info) == ALZ_OK && nodes.size() == 4, "all nodes");
  for (const alaz::CycleNode& n : nodes) {
    if (n.UID == "web") CHECK(n.Size == 1 && n.Depth == 0 && n.Height == 2, "web %s", names(nodes).c_str());
    if (n.UID == "api-2") CHECK(n.Size == 1 && n.Depth == 2 && n.Height == 0, "api-2 %s", names(nodes).c_str());
  }
  CHECK(rows.size() == 2, "rows with min_size 0");
  // failing calls only: no loop
  alz_metric err{};
  err.kind = ALZ_METRIC_ERR5XX;
  CHECK(a.Cycles(last, &err, 1.0, 2, &nodes, &rows, &info) == ALZ_OK, "5xx");
  CHECK(nodes.empty() && rows.empty() && info.traversable == 2 && info.cyclic == 0, "5xx %s", names(nodes).c_str());

  // deployments
  CHECK(a.GroupCycles(last, nullptr, 0.0, 2, &nodes, &rows, &info) == ALZ_OK, "group: %s", a.LastError().c_str());
  CHECK((names(nodes) == "group/api:2,1,0 group/db:2,1,0 " || names(nodes) == "group/db:2,1,0 group/api:2,1,0 "),
        "group loop %s", names(nodes).c_str());
  CHECK(pairs(rows) == "api>db db>api ", "group rows %s", pairs(rows).c_str());
  CHECK(info.self_rows == 1 && info.components == 2 && info.cyclic == 1 && info.depth == 1, "group info");
  CHECK(a.Cycles(7, nullptr, 0.0, 2, &nodes, &rows, &info) == ALZ_E_INVAL, "bad source");
  printf("cycles adapter ok\n");
  return 0;
}
