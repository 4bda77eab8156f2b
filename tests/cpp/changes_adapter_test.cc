// changes_adapter_test.cc — the C++ host adapter's edge changes (docs/SPEC.md §18): PinBaseline and Changes return the
// new, gone and changed edges by UID, full and top; and while a baseline is pinned, a deleted pod's id is not handed to
// a new pod, whether it was freed before or after the pin, so the deleted pod's edge shows as gone under its own UID
// and the new pod's edge as new. ClearBaseline releases the hold, and a pin over an id already reused is refused.
#include <cstdio>
#include <cstring>
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
static alz_metric metric(uint32_t kind) { alz_metric m{}; m.kind = kind; return m; }
static std::map<std::string, alaz::EdgeChange> by_uid(const std::vector<alaz::EdgeChange>& v) {
  std::map<std::string, alaz::EdgeChange> out;
  for (const auto& c : v) out[c.FromUID + "->" + c.ToUID] = c;
  return out;
}

// A pod deleted in the window that is then pinned: its id was already free when the baseline was pinned, and the pin
// takes it back, so a pod added afterwards does not take over its edge.
static int freed_before_the_pin(const alaz::AggregatorConfig& cfg) {
  alaz::Aggregator a(nullptr, cfg);
  CHECK(a.Ok(), "create: %s", a.LastError().c_str());
  const alz_metric count = metric(ALZ_METRIC_COUNT);
  k8s(a, "Service", "Add", "svc-s", "10.1.0.1");
  k8s(a, "Pod", "Add", "pod-a", "10.0.0.1");
  k8s(a, "Pod", "Add", "pod-b", "10.0.0.2");
  requests(a, "10.0.0.1", "10.1.0.1", 5);
  requests(a, "10.0.0.2", "10.1.0.1", 4);
  k8s(a, "Pod", "Delete", "pod-b", "10.0.0.2");           // in the same window: its id is free after this flush
  CHECK(a.Flush() == ALZ_OK, "flush 1");
  CHECK(a.PinBaseline(alaz::Aggregator::kLastWindow) == ALZ_OK, "pin");
  k8s(a, "Pod", "Add", "pod-d", "10.0.0.4");
  requests(a, "10.0.0.1", "10.1.0.1", 5);
  requests(a, "10.0.0.4", "10.1.0.1", 3);
  CHECK(a.Flush() == ALZ_OK, "flush 2");
  std::vector<alaz::EdgeChange> ch;
  CHECK(a.Changes(alaz::Aggregator::kLastWindow, count, ALZ_CHANGE_DELTA, 7, 0, 0.0, &ch) == ALZ_OK, "changes");
  auto m = by_uid(ch);
  CHECK(ch.size() == 3, "rows %zu", ch.size());
  CHECK(m.count("pod-a->svc-s") && m["pod-a->svc-s"].Presence == ALZ_PRESENT_BOTH, "pod-a both");
  CHECK(m.count("pod-b->svc-s") && m["pod-b->svc-s"].Presence == ALZ_PRESENT_GONE, "pod-b gone under its own UID");
  CHECK(m.count("pod-d->svc-s") && m["pod-d->svc-s"].Presence == ALZ_PRESENT_NEW, "pod-d new");
  return 0;
}

// ClearBaseline releases the hold: after it, a new pod takes the deleted pod's id, so a held rollup that still carries
// the deleted pod's edge can no longer be pinned (ALZ_E_STATE). Were the hold never released, the new pod would get a
// fresh id and the pin would succeed.
static int released_by_clear(const alaz::AggregatorConfig& cfg) {
  alaz::Aggregator a(nullptr, cfg);
  CHECK(a.Ok(), "create: %s", a.LastError().c_str());
  CHECK(a.SetHistory(1, 1u << 12) == ALZ_OK, "history");   // holds a freed id for one more window
  k8s(a, "Service", "Add", "svc-s", "10.1.0.1");
  k8s(a, "Pod", "Add", "pod-b", "10.0.0.2");
  requests(a, "10.0.0.2", "10.1.0.1", 4);
  k8s(a, "Pod", "Delete", "pod-b", "10.0.0.2");
  CHECK(a.Flush() == ALZ_OK, "flush 1");
  CHECK(a.Rollup(0, 1) == ALZ_OK, "rollup");               // the window rollup's rows carry pod-b's id
  CHECK(a.PinBaseline(ALZ_ROLLUP_WINDOWS) == ALZ_OK, "pin");
  CHECK(a.Flush() == ALZ_OK, "flush 2");
  CHECK(a.Flush() == ALZ_OK, "flush 3");                   // the history's own hold is over
  k8s(a, "Pod", "Add", "pod-d", "10.0.0.4");               // still held: a fresh id
  CHECK(a.PinBaseline(ALZ_ROLLUP_WINDOWS) == ALZ_OK, "re-pin while held");
  CHECK(a.ClearBaseline() == ALZ_OK, "clear");
  k8s(a, "Pod", "Add", "pod-e", "10.0.0.5");               // takes pod-b's id
  CHECK(a.PinBaseline(ALZ_ROLLUP_WINDOWS) == ALZ_E_STATE, "pin over a reused id is refused");
  std::vector<alaz::EdgeChange> ch;
  CHECK(a.Changes(alaz::Aggregator::kLastWindow, metric(ALZ_METRIC_COUNT), ALZ_CHANGE_DELTA, 7, 0, 0.0, &ch) ==
            ALZ_E_STATE, "a refused pin leaves no baseline");
  return 0;
}

int main() {
  alaz::AggregatorConfig cfg;
  cfg.MaxEndpoints = 1024;
  cfg.MaxPairs = 1u << 12;
  cfg.BatchSize = 256;
  alaz::Aggregator a(nullptr, cfg);
  CHECK(a.Ok(), "create: %s", a.LastError().c_str());
  const alz_metric count = metric(ALZ_METRIC_COUNT);
  std::vector<alaz::EdgeChange> ch;
  CHECK(a.Changes(alaz::Aggregator::kLastWindow, count, ALZ_CHANGE_DELTA, 7, 0, 0.0, &ch) == ALZ_E_STATE, "no baseline");

  k8s(a, "Service", "Add", "svc-s", "10.1.0.1");
  k8s(a, "Pod", "Add", "pod-a", "10.0.0.1");
  k8s(a, "Pod", "Add", "pod-b", "10.0.0.2");
  requests(a, "10.0.0.1", "10.1.0.1", 10);
  requests(a, "10.0.0.2", "10.1.0.1", 4, 500);
  CHECK(a.Flush() == ALZ_OK, "flush 1");
  alz_rollup_info info{};
  CHECK(a.PinBaseline(alaz::Aggregator::kLastWindow, &info) == ALZ_OK, "pin");
  CHECK(info.windows == 1 && info.window_first == 1 && info.rows_in == 2, "pin info %u %lu %lu", info.windows,
        (unsigned long)info.window_first, (unsigned long)info.rows_in);

  // pod-b goes; its id must not go to pod-d while the baseline (which holds pod-b's edge) is pinned
  k8s(a, "Pod", "Delete", "pod-b", "10.0.0.2");
  requests(a, "10.0.0.1", "10.1.0.1", 7);
  CHECK(a.Flush() == ALZ_OK, "flush 2");
  CHECK(a.Flush() == ALZ_OK, "flush 3");                 // without the hold, pod-b's id would be free by now
  k8s(a, "Pod", "Add", "pod-d", "10.0.0.4");
  requests(a, "10.0.0.1", "10.1.0.1", 13);
  requests(a, "10.0.0.4", "10.1.0.1", 3);
  CHECK(a.Flush() == ALZ_OK, "flush 4");

  alz_change_info ci{};
  CHECK(a.Changes(alaz::Aggregator::kLastWindow, count, ALZ_CHANGE_DELTA, 7, 0, 0.0, &ch, &ci) == ALZ_OK, "changes");
  CHECK(ch.size() == 3 && ci.both == 1 && ci.added == 1 && ci.gone == 1, "rows %zu both %lu added %lu gone %lu",
        ch.size(), (unsigned long)ci.both, (unsigned long)ci.added, (unsigned long)ci.gone);
  auto m = by_uid(ch);
  CHECK(m.count("pod-a->svc-s") && m["pod-a->svc-s"].Presence == ALZ_PRESENT_BOTH && m["pod-a->svc-s"].Change == 3.0,
        "pod-a");
  CHECK(m.count("pod-b->svc-s") && m["pod-b->svc-s"].Presence == ALZ_PRESENT_GONE && m["pod-b->svc-s"].Change == -4.0,
        "pod-b is gone under its own UID");
  CHECK(m.count("pod-d->svc-s") && m["pod-d->svc-s"].Presence == ALZ_PRESENT_NEW && m["pod-d->svc-s"].Value == 3.0,
        "pod-d is new");
  CHECK(m["pod-a->svc-s"].FromType == "pod" && m["pod-a->svc-s"].ToType == "service", "types");

  // top: the largest drop in 5xx first
  CHECK(a.Changes(alaz::Aggregator::kLastWindow, metric(ALZ_METRIC_ERR5XX), ALZ_CHANGE_DROP, 7, 1, 0.0, &ch, &ci) ==
            ALZ_OK, "top");
  CHECK(ch.size() == 1 && ch[0].FromUID == "pod-b" && ch[0].Change == 4.0 && ci.above == 3, "top drop %zu", ch.size());
  // only new edges
  CHECK(a.Changes(alaz::Aggregator::kLastWindow, count, ALZ_CHANGE_RATIO, ALZ_PRESENT_NEW, 0, 0.0, &ch) == ALZ_OK,
        "new only");
  CHECK(ch.size() == 1 && ch[0].FromUID == "pod-d" && ch[0].Change > 1e308, "new only: %zu", ch.size());

  // more windows, another new pod: the hold lasts until ClearBaseline
  k8s(a, "Pod", "Add", "pod-g", "10.0.0.7");
  requests(a, "10.0.0.7", "10.1.0.1", 2);
  CHECK(a.Flush() == ALZ_OK, "flush 5");
  CHECK(a.Changes(alaz::Aggregator::kLastWindow, count, ALZ_CHANGE_DELTA, 7, 0, 0.0, &ch) == ALZ_OK, "changes 5");
  m = by_uid(ch);
  CHECK(m.count("pod-b->svc-s") && m["pod-b->svc-s"].Presence == ALZ_PRESENT_GONE, "pod-b still gone");
  CHECK(m.count("pod-g->svc-s") && m["pod-g->svc-s"].Presence == ALZ_PRESENT_NEW, "pod-g new");

  CHECK(a.ClearBaseline() == ALZ_OK, "clear");
  CHECK(a.Changes(alaz::Aggregator::kLastWindow, count, ALZ_CHANGE_DELTA, 7, 0, 0.0, &ch) == ALZ_E_STATE, "cleared");

  // a new pin holds the ids of its own window: pod-d goes, pod-h comes, and pod-d's edge stays pod-d's
  requests(a, "10.0.0.4", "10.1.0.1", 6);
  CHECK(a.Flush() == ALZ_OK, "flush 6");
  CHECK(a.PinBaseline(alaz::Aggregator::kLastWindow) == ALZ_OK, "re-pin");
  k8s(a, "Pod", "Delete", "pod-d", "10.0.0.4");
  CHECK(a.Flush() == ALZ_OK, "flush 7");
  CHECK(a.Flush() == ALZ_OK, "flush 8");
  k8s(a, "Pod", "Add", "pod-h", "10.0.0.8");
  k8s(a, "Pod", "Add", "pod-i", "10.0.0.9");
  requests(a, "10.0.0.8", "10.1.0.1", 1);
  requests(a, "10.0.0.9", "10.1.0.1", 1);
  CHECK(a.Flush() == ALZ_OK, "flush 9");
  CHECK(a.Changes(alaz::Aggregator::kLastWindow, count, ALZ_CHANGE_DELTA, 7, 0, 0.0, &ch) == ALZ_OK, "changes 9");
  m = by_uid(ch);
  CHECK(ch.size() == 3, "rows %zu", ch.size());
  CHECK(m.count("pod-d->svc-s") && m["pod-d->svc-s"].Presence == ALZ_PRESENT_GONE && m["pod-d->svc-s"].Change == -6.0,
        "pod-d gone under its own UID");
  CHECK(m.count("pod-h->svc-s") && m.count("pod-i->svc-s"), "pod-h and pod-i new");
  if (freed_before_the_pin(cfg) || released_by_clear(cfg)) return 1;
  printf("changes adapter ok\n");
  return 0;
}
