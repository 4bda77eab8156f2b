// corr_adapter_test.cc — the C++ host adapter's correlations (docs/SPEC.md §29) on a small service map: frontend pod
// calls checkout, checkout's pod calls payments, and payments' latency leads checkout's by one window. Correlations,
// NodeCorrelations, GroupCorrelations and GroupNodeCorrelations each find the dependency at lag 1 when the target is
// the caller's p99, and leave the target itself out of the result.
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

int main() {
  alaz::AggregatorConfig cfg;
  cfg.MaxEndpoints = 64;
  cfg.MaxPairs = 1u << 12;
  alaz::Aggregator a(nullptr, cfg);
  CHECK(a.Ok(), "create: %s", a.LastError().c_str());
  CHECK(a.SetHistory(8, 1u << 12) == ALZ_OK, "history");
  k8s(a, "Service", "Add", "svc-checkout", "10.1.0.1");
  k8s(a, "Service", "Add", "svc-payments", "10.1.0.2");
  k8s(a, "Service", "Add", "svc-search", "10.1.0.3");
  k8s(a, "Pod", "Add", "pod-frontend", "10.0.0.1");
  k8s(a, "Pod", "Add", "pod-checkout", "10.0.0.2");
  k8s(a, "Pod", "Add", "pod-search", "10.0.0.3");
  // payments' latency (ms) in each window; checkout's is payments' of the window before; search's is unrelated
  const uint64_t pay[7] = {1, 16, 2, 64, 4, 32, 8};
  const uint64_t search[7] = {8, 8, 1, 2, 64, 4, 16};
  for (int w = 0; w < 7; ++w) {
    requests(a, "10.0.0.2", "10.1.0.2", 20, pay[w] * 1000000);
    requests(a, "10.0.0.1", "10.1.0.1", 20, (w ? pay[w - 1] : 128) * 1000000);
    requests(a, "10.0.0.3", "10.1.0.3", 20, search[w] * 1000000);
    CHECK(a.Flush() == ALZ_OK, "flush %d", w);
  }
  CHECK(a.Rollup(0, 7) == ALZ_OK, "rollup: %s", a.LastError().c_str());

  alz_metric p99{};
  p99.kind = ALZ_METRIC_QUANTILE;
  p99.q = 0.99;
  alz_corr corr{};
  corr.direction = ALZ_CORR_POSITIVE;
  corr.absent = ALZ_CORR_ABSENT_SKIP;
  corr.max_lag = 2;
  corr.min_points = 3;

  // edges: the target is frontend -> checkout
  const alaz::EdgeRef caller{"pod", "pod-frontend", "service", "svc-checkout"};
  std::vector<alaz::EdgeCorr> ec;
  std::vector<alz_rollup_info> pts;
  CHECK(a.Correlations(ALZ_ROLLUP_WINDOWS, 0, 7, p99, corr, caller, 5, -HUGE_VAL, &ec, &pts) == ALZ_OK,
        "edges: %s", a.LastError().c_str());
  CHECK(pts.size() == 7, "points %zu", pts.size());
  CHECK(!ec.empty() && ec[0].FromUID == "pod-checkout" && ec[0].ToUID == "svc-payments", "first %s -> %s",
        ec.empty() ? "" : ec[0].FromUID.c_str(), ec.empty() ? "" : ec[0].ToUID.c_str());
  CHECK(ec[0].Valid && ec[0].Lag == 1 && ec[0].Used == 6 && ec[0].R > 0.999999 && ec[0].R0 < 0.9, "lag %u r %g r0 %g",
        ec[0].Lag, ec[0].R, ec[0].R0);
  CHECK(ec[0].Values.size() == 7 && ec[0].Present.size() == 7, "series");
  for (const alaz::EdgeCorr& e : ec)
    CHECK(!(e.FromUID == "pod-frontend" && e.ToUID == "svc-checkout"), "the target is in the result");
  // the same through an explicit target: the caller's own row is then listed, at lag 0 with r = 1
  std::vector<alaz::EdgeSeries> ser;
  CHECK(a.SeriesFor({caller}, 0, 7, {p99}, &ser, &pts) == ALZ_OK, "series for");
  alaz::CorrTarget t{ser[0].Values, ser[0].Present, pts.back().window_last};
  std::vector<alaz::EdgeCorr> all;
  CHECK(a.Correlations(ALZ_ROLLUP_WINDOWS, 0, 7, p99, corr, t, 5, -HUGE_VAL, &all) == ALZ_OK, "explicit");
  bool self = false;
  for (const alaz::EdgeCorr& e : all)
    if (e.FromUID == "pod-frontend" && e.ToUID == "svc-checkout") self = e.Lag == 0 && e.R > 0.999999;
  CHECK(self, "the explicit target's own row");
  // nodes, side IN: the target is checkout's inbound p99; payments' inbound leads it
  const alaz::NodeRef checkout{"service", "svc-checkout"};
  std::vector<alaz::NodeCorr> nc;
  corr.max_lag = 3;
  CHECK(a.NodeCorrelations(ALZ_ROLLUP_WINDOWS, ALZ_SIDE_IN, 0, 7, p99, corr, checkout, 5, -HUGE_VAL, &nc) == ALZ_OK,
        "nodes: %s", a.LastError().c_str());
  CHECK(!nc.empty() && nc[0].Node.UID == "svc-payments" && nc[0].Lag == 1, "nodes first %s lag %u",
        nc.empty() ? "" : nc[0].Node.UID.c_str(), nc.empty() ? 0u : nc[0].Lag);
  for (const alaz::NodeCorr& e : nc) CHECK(e.Node.UID != "svc-checkout", "the target node is in the result");

  // groups: frontend, checkout (its pod and its service) and payments
  CHECK(a.SetGroups({{"pod", "pod-frontend", "frontend"}, {"pod", "pod-checkout", "checkout"},
                     {"service", "svc-checkout", "checkout"}, {"service", "svc-payments", "payments"},
                     {"pod", "pod-search", "search"}, {"service", "svc-search", "search"}}) == ALZ_OK,
        "groups");
  const alaz::EdgeRef gcaller{"group", "frontend", "group", "checkout"};
  CHECK(a.GroupCorrelations(ALZ_ROLLUP_WINDOWS, 0, 7, p99, corr, gcaller, 5, -HUGE_VAL, &ec) == ALZ_OK,
        "group edges: %s", a.LastError().c_str());
  CHECK(!ec.empty() && ec[0].FromUID == "checkout" && ec[0].ToUID == "payments" && ec[0].Lag == 1 &&
            ec[0].FromType == "group",
        "group edges first %s -> %s lag %u", ec.empty() ? "" : ec[0].FromUID.c_str(),
        ec.empty() ? "" : ec[0].ToUID.c_str(), ec.empty() ? 0u : ec[0].Lag);
  for (const alaz::EdgeCorr& e : ec)
    CHECK(!(e.FromUID == "frontend" && e.ToUID == "checkout"), "the target group edge is in the result");
  const alaz::NodeRef gcheckout{"group", "checkout"};
  CHECK(a.GroupNodeCorrelations(ALZ_ROLLUP_WINDOWS, ALZ_SIDE_IN, 0, 7, p99, corr, gcheckout, 5, -HUGE_VAL, &nc) ==
            ALZ_OK,
        "group nodes: %s", a.LastError().c_str());
  CHECK(!nc.empty() && nc[0].Node.UID == "payments" && nc[0].Node.Type == "group" && nc[0].Lag == 1,
        "group nodes first %s lag %u", nc.empty() ? "" : nc[0].Node.UID.c_str(), nc.empty() ? 0u : nc[0].Lag);
  for (const alaz::NodeCorr& e : nc) CHECK(e.Node.UID != "checkout", "the target group is in the result");

  // a bad argument comes back as the library's status
  corr.min_points = 2;
  CHECK(a.Correlations(ALZ_ROLLUP_WINDOWS, 0, 7, p99, corr, caller, 5, 0.0, &ec) == ALZ_E_INVAL, "min_points 2");
  // a target taken before a flush is stale
  corr.min_points = 3;
  requests(a, "10.0.0.1", "10.1.0.1", 5, 1000000);
  CHECK(a.Flush() == ALZ_OK, "flush");
  CHECK(a.Correlations(alaz::Aggregator::kLastWindow, 0, 7, p99, corr, t, 5, -HUGE_VAL, &all) == ALZ_E_STATE,
        "stale target");
  printf("corr adapter ok\n");
  return 0;
}
