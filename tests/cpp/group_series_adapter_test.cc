// group_series_adapter_test.cc — the C++ host adapter's group series and trends (docs/SPEC.md §26) through a rolling
// deploy: web calls deployment api's pods api-1 and api-2 in windows 1 and 2; the rollout replaces them with api-3 and
// api-4 before windows 3 and 4. Per pod (NodeSeriesFor), each pod is present in its own two windows only; per
// deployment (GroupNodeSeriesFor by group name, GroupNodeSeries by source), group/api is present at all four points
// with its members' summed counts, and so is the group edge web -> api. A group name SetGroups never gave and a mapped
// pod are absent everywhere. GroupNodeTrends and GroupTrends rank the groups over the four points.
#include <cmath>
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
static bool same(const std::vector<double>& v, const std::vector<double>& w) { return v == w; }

int main() {
  alaz::AggregatorConfig cfg;
  cfg.MaxEndpoints = 64;
  cfg.MaxPairs = 1u << 12;
  alaz::Aggregator a(nullptr, cfg);
  CHECK(a.Ok(), "create: %s", a.LastError().c_str());
  CHECK(a.SetHistory(8, 1u << 12) == ALZ_OK, "history: %s", a.LastError().c_str());
  CHECK(a.SetGroups({{"pod", "api-1", "api"}, {"pod", "api-2", "api"}, {"pod", "api-3", "api"},
                     {"pod", "api-4", "api"}, {"pod", "web", "web"}}) == ALZ_OK, "set groups");
  k8s(a, "Pod", "Add", "web", "10.0.0.10");
  k8s(a, "Pod", "Add", "api-1", "10.0.0.1");
  k8s(a, "Pod", "Add", "api-2", "10.0.0.2");
  requests(a, "10.0.0.10", "10.0.0.1", 10, 1000000);
  requests(a, "10.0.0.10", "10.0.0.2", 20, 2000000);
  CHECK(a.Flush() == ALZ_OK, "flush 1");
  requests(a, "10.0.0.10", "10.0.0.1", 5, 1000000);
  requests(a, "10.0.0.10", "10.0.0.2", 5, 2000000);
  CHECK(a.Flush() == ALZ_OK, "flush 2");
  k8s(a, "Pod", "Delete", "api-1", "10.0.0.1");          // the rollout
  k8s(a, "Pod", "Delete", "api-2", "10.0.0.2");
  k8s(a, "Pod", "Add", "api-3", "10.0.0.3");
  k8s(a, "Pod", "Add", "api-4", "10.0.0.4");
  requests(a, "10.0.0.10", "10.0.0.3", 7, 4000000);
  requests(a, "10.0.0.10", "10.0.0.4", 8, 8000000);
  CHECK(a.Flush() == ALZ_OK, "flush 3");
  requests(a, "10.0.0.10", "10.0.0.3", 9, 4000000);
  requests(a, "10.0.0.10", "10.0.0.4", 1, 8000000);
  CHECK(a.Flush() == ALZ_OK, "flush 4");

  alz_metric count{};
  count.kind = ALZ_METRIC_COUNT;
  const uint32_t last = alaz::Aggregator::kLastWindow;
  const std::vector<double> api = {30, 10, 15, 10};
  std::vector<alz_rollup_info> pts;

  // per pod: each present in its own windows only
  std::vector<alaz::NodeSeriesRow> rows;
  CHECK(a.NodeSeriesFor({{"pod", "api-1"}, {"pod", "api-3"}}, ALZ_SIDE_IN, 0, 4, {count}, &rows, &pts) == ALZ_OK,
        "pods: %s", a.LastError().c_str());
  CHECK(pts.size() == 4 && rows.size() == 2, "pods %zu %zu", pts.size(), rows.size());
  CHECK((rows[0].Present == std::vector<uint8_t>{1, 1, 0, 0}) && (rows[1].Present == std::vector<uint8_t>{0, 0, 1, 1}),
        "pod presence");

  // per deployment, by group name: present at every point with the members' summed counts
  CHECK(a.GroupNodeSeriesFor({{"group", "api"}, {"group", "no-such-group"}, {"pod", "api-1"}, {"group", "api"}},
                             ALZ_SIDE_IN, 0, 4, {count}, &rows, &pts) == ALZ_OK,
        "group nodes for: %s", a.LastError().c_str());
  CHECK(rows.size() == 4 && pts.size() == 4, "rows %zu", rows.size());
  CHECK(rows[0].Type == "group" && rows[0].UID == "api" && (rows[0].Present == std::vector<uint8_t>{1, 1, 1, 1}) &&
            same(rows[0].Values, api), "group/api %g %g %g %g", rows[0].Values[0], rows[0].Values[1],
        rows[0].Values[2], rows[0].Values[3]);
  CHECK(rows[1].UID == "no-such-group" && (rows[1].Present == std::vector<uint8_t>{0, 0, 0, 0}) &&
            same(rows[1].Values, {0, 0, 0, 0}), "unknown group");
  CHECK(rows[2].Type == "pod" && (rows[2].Present == std::vector<uint8_t>{0, 0, 0, 0}), "a mapped pod is absent");
  CHECK(rows[3].Present == rows[0].Present && same(rows[3].Values, rows[0].Values), "duplicate");

  // by source: the last window's group nodes, named as GroupNodes names them
  CHECK(a.GroupNodeSeries(last, ALZ_SIDE_IN, 0, 4, {count}, &rows) == ALZ_OK, "group nodes: %s",
        a.LastError().c_str());
  CHECK(rows.size() == 2 && rows[0].Type == "group" && rows[0].UID == "api" && same(rows[0].Values, api) &&
            rows[1].UID == "web" && (rows[1].Present == std::vector<uint8_t>{0, 0, 0, 0}), "group nodes %zu",
        rows.size());
  CHECK(a.GroupNodeSeries(last, ALZ_SIDE_OUT, 0, 4, {count}, &rows) == ALZ_OK, "group nodes out");
  CHECK(rows.size() == 2 && rows[1].UID == "web" && same(rows[1].Values, api), "web out");

  // group edges, by source and by name
  std::vector<alaz::EdgeSeries> edges;
  CHECK(a.GroupSeries(last, 0, 4, {count}, &edges) == ALZ_OK, "group edges: %s", a.LastError().c_str());
  CHECK(edges.size() == 1 && edges[0].FromType == "group" && edges[0].FromUID == "web" && edges[0].ToType == "group" &&
            edges[0].ToUID == "api" && same(edges[0].Values, api), "web -> api %zu", edges.size());
  CHECK(a.GroupSeriesFor({{"group", "web", "group", "api"}, {"group", "web", "pod", "api-3"},
                          {"group", "web", "group", "no-such-group"}}, 0, 4, {count}, &edges) == ALZ_OK,
        "group edges for: %s", a.LastError().c_str());
  CHECK(edges.size() == 3 && same(edges[0].Values, api) && (edges[0].Present == std::vector<uint8_t>{1, 1, 1, 1}),
        "web -> api by name");
  CHECK((edges[1].Present == std::vector<uint8_t>{0, 0, 0, 0}) &&
            (edges[2].Present == std::vector<uint8_t>{0, 0, 0, 0}), "absent group edges");

  // trends over the four points
  alz_trend slope{};
  slope.stat = ALZ_TREND_SLOPE;
  slope.recent = 1;
  std::vector<alaz::NodeTrend> nt;
  CHECK(a.GroupNodeTrends(last, ALZ_SIDE_IN, 0, 4, count, slope, 5, -HUGE_VAL, &nt) == ALZ_OK, "node trends: %s",
        a.LastError().c_str());
  CHECK(nt.size() == 1 && nt[0].Node.Type == "group" && nt[0].Node.UID == "api" && nt[0].Valid && nt[0].Used == 4 &&
            nt[0].Trend == -5.5 && same(nt[0].Values, api), "group/api trend %zu %g", nt.size(),
        nt.empty() ? 0.0 : nt[0].Trend);
  std::vector<alaz::EdgeTrend> et;
  CHECK(a.GroupTrends(last, 0, 4, count, slope, 5, -HUGE_VAL, &et) == ALZ_OK, "edge trends: %s",
        a.LastError().c_str());
  CHECK(et.size() == 1 && et[0].FromUID == "web" && et[0].ToType == "group" && et[0].ToUID == "api" &&
            et[0].Trend == -5.5 && same(et[0].Values, api), "web -> api trend %zu", et.size());
  printf("group series adapter ok\n");
  return 0;
}
