// alaz_aggregator.hpp — host side of the path above the C ABI, in C++ (the reference is Go and no Go
// toolchain exists here; INTEGRATION.md shows the cgo equivalent). It mirrors the aggregator's seam:
// the same event types go in (only the fields this path reads), a DataStore-shaped sink comes out.
//
//   reference                                              here
//   NewAggregator(ctx, ct, k8sChan, events, ...)           alaz::Aggregator(ds, cfg)      aggregator/data.go:135-140
//   processk8s -> processPod / processSvc                  ProcessK8s(msg)                aggregator/persist.go:25-131
//   processEbpf -> processL7                               ProcessL7(ev)                  aggregator/data.go:310-337, 1364
//   processEbpfTcp -> processTcpConnect                    ProcessTcpConnect(ev)          aggregator/data.go:404-506
//   ds.PersistRequest(row) per event                       ds->PersistEdgeWindow(edges)   datastore/datastore.go:13
#pragma once
#include <cstdint>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/alazgpu.h"

namespace alaz {

// ebpf/l7_req/l7.go:396-421 (fields read on this path)
struct L7Event {
  uint64_t Fd = 0;
  uint32_t Pid = 0;
  uint32_t Status = 0;
  uint64_t Duration = 0;
  std::string Protocol;   // "HTTP", "AMQP", ... (l7.go:32-42)
  bool Tls = false;
  std::string Method;     // "GET", "DELIVER", "PUSHED_EVENT", ...
  uint64_t WriteTimeNs = 0;
  uint32_t Saddr = 0, Daddr = 0;
  uint16_t Sport = 0, Dport = 0;
  bool PayloadRejected = false;   // the Go-side SQL/Mongo parser returned an error (data.go:1252, 1288, 1328)
  std::string Payload;            // HTTP only: Payload[0:PayloadSize], read for its Host header (data.go:1213)
};

// ebpf/tcp_state/tcp.go:75-84
struct TcpConnectEvent {
  uint64_t Fd = 0, Timestamp = 0;
  std::string Type_;      // "EVENT_TCP_ESTABLISHED", "EVENT_TCP_CLOSED", ... (tcp.go:27-60)
  uint32_t Pid = 0;
  uint16_t SPort = 0, DPort = 0;
  std::string SAddr, DAddr;   // dotted quad (tcp.go:241-242)
};

// k8s/informer.go:236-240, reduced to what processPod/processSvc write into ClusterInfo
struct K8sResourceMessage {
  std::string ResourceType;   // "Pod" | "Service" (k8s/informer.go:26-36)
  std::string EventType;      // "Add" | "Update" | "Delete"
  std::string UID;
  std::string IP;             // pod.Status.PodIP or service.Spec.ClusterIP; empty pod IP is skipped (persist.go:37-40)
};

struct EdgeWindow {
  std::string FromType, FromUID, ToType, ToUID;   // "pod" | "service" | "outbound" (data.go:42-44)
  uint64_t Count = 0, Err5xx = 0, LatSumNs = 0;
  uint32_t Hist[ALZ_NB] = {0};
  float Score = 0.f;                              // GNN anomaly score when requested
  double Value = 0.0;                             // the ranking metric's value (TopEdges)
};

// one row of a change list (docs/SPEC.md §18): the edge by UID, where it is (ALZ_PRESENT_*) and the metric's value on
// each side with their change
struct EdgeChange {
  std::string FromType, FromUID, ToType, ToUID;
  uint32_t Presence = 0;
  double Value = 0.0, BaseValue = 0.0, Change = 0.0;
};

// one node of a node change list (docs/SPEC.md §23): the node by UID as NodeWindow names it, where it is
// (ALZ_PRESENT_*) and the metric's value of one side on each side of the comparison with their change
struct NodeChange {
  std::string Type, UID;
  uint32_t Presence = 0;
  double Value = 0.0, BaseValue = 0.0, Change = 0.0;
};

// an edge named by UID, as EdgeWindow names it: FromType / ToType "pod" | "service" | "outbound"; an outbound end's UID
// is its dotted quad or its Host header text
struct EdgeRef {
  std::string FromType, FromUID, ToType, ToUID;
};

// one edge's series (docs/SPEC.md §19): per point, oldest first, whether that entry holds the edge and the metrics'
// values on its row there (every value 0 where it does not)
struct EdgeSeries {
  std::string FromType, FromUID, ToType, ToUID;
  std::vector<uint8_t> Present;   // [points]
  std::vector<double> Values;     // [points * metrics]: metric j at point p is Values[p * metrics + j]
};

// one edge's trend (docs/SPEC.md §20) with the series it was computed from: per point, oldest first, whether that
// entry holds the edge and the metric's value there (0 where it does not)
struct EdgeTrend {
  std::string FromType, FromUID, ToType, ToUID;
  bool Valid = false;
  uint32_t Used = 0;                  // points used
  double Trend = 0.0, Recent = 0.0, Before = 0.0;
  std::vector<uint8_t> Present;       // [points]
  std::vector<double> Values;         // [points]
};

// one node of a source (docs/SPEC.md §21) by UID: Type "pod" | "service" | "outbound" as EdgeWindow names an end (an
// outbound node's UID is its dotted quad or its Host header text), the rows into it (In) and out of it (Out) with their
// sums, and metric values of one side
struct NodeWindow {
  std::string Type, UID;
  uint32_t InEdges = 0, OutEdges = 0;
  alz_node_sums In{}, Out{};
  std::vector<double> Values;   // Nodes: the metrics in the caller's order; TopNodes: the ranking metric's value
};

// a node named by UID, as NodeWindow names it: Type "pod" | "service" | "outbound"; an outbound node's UID is its
// dotted quad or its Host header text
struct NodeRef {
  std::string Type, UID;
};

// a member of a caller-defined group (docs/SPEC.md §24): the node by Type ("pod" | "service" | "outbound") and UID as
// NodeRef names it, and its group's name (a deployment, a namespace)
struct GroupMember {
  std::string Type, UID, Group;
};

// one node a reach (docs/SPEC.md §27) listed: named as Nodes / GroupNodes name it, its hops from the nearest seed, the
// position in the result of its parent on one shortest path and the position in the rows of the row used from that
// parent (both kReachNone for a seed)
struct ReachNode {
  std::string Type, UID;
  uint32_t Hops = 0, Parent = 0, Row = 0;
};

// one node of a cycles call (docs/SPEC.md §28): named as Nodes / GroupNodes name it, its component's number, node
// count, depth (the most rows between components on a path that ends at it) and height (on a path that starts at it)
struct CycleNode {
  std::string Type, UID;
  uint32_t Component = 0, Size = 0, Depth = 0, Height = 0;
};

// one node's series (docs/SPEC.md §22): per point, oldest first, whether that entry holds a row on the side of the
// node and the metrics' values of the side's sums there (every value 0 where it does not)
struct NodeSeriesRow {
  std::string Type, UID;
  std::vector<uint8_t> Present;   // [points]
  std::vector<double> Values;     // [points * metrics]: metric j at point p is Values[p * metrics + j]
};

// one node's trend (docs/SPEC.md §22) with the series it was computed from, and the node's row in the source
struct NodeTrend {
  NodeWindow Node;                    // Type, UID, edge counts and both sides' sums in the source (Values empty)
  bool Valid = false;
  uint32_t Used = 0;                  // points used
  double Trend = 0.0, Recent = 0.0, Before = 0.0;
  std::vector<uint8_t> Present;       // [points]
  std::vector<double> Values;         // [points]
};

// a target series for the correlation calls (docs/SPEC.md §29): per point, oldest first, its value and whether it is
// present (empty Present: every point), aligned to the ring and k of the call; WindowLast is the window_last of its
// newest point, as the *SeriesFor calls' points report it
struct CorrTarget {
  std::vector<double> Values;
  std::vector<uint8_t> Present;
  uint64_t WindowLast = 0;
};

// one edge's correlation with a target (docs/SPEC.md §29) and the series it was computed from
struct EdgeCorr {
  std::string FromType, FromUID, ToType, ToUID;
  bool Valid = false;
  uint32_t Lag = 0;                   // the best lag: the edge leads the target by this many points
  uint32_t Used = 0;                  // pairs used at it
  double R = 0.0, Score = 0.0, R0 = 0.0;   // r and the score at the best lag, r at lag 0
  std::vector<uint8_t> Present;       // [points]
  std::vector<double> Values;         // [points]
};

// one node's correlation with a target (docs/SPEC.md §29), its node row in the source and its series
struct NodeCorr {
  NodeWindow Node;                    // Type, UID, edge counts and both sides' sums in the source (Values empty)
  bool Valid = false;
  uint32_t Lag = 0, Used = 0;
  double R = 0.0, Score = 0.0, R0 = 0.0;
  std::vector<uint8_t> Present;       // [points]
  std::vector<double> Values;         // [points]
};

// datastore/dto.go AliveConnection, as sendOpenConnection fills it (aggregator/data.go:1649-1675)
struct AliveConnection {
  int64_t CheckTime = 0;   // unix ms
  std::string FromIP, FromType, FromUID;
  uint16_t FromPort = 0;
  std::string ToIP, ToType, ToUID;
  uint16_t ToPort = 0;
};

// the sink, next to DataStore.PersistRequest (datastore/datastore.go:13)
class DataStore {
 public:
  virtual ~DataStore() = default;
  virtual int PersistEdgeWindow(const std::vector<EdgeWindow>& edges) = 0;
  virtual int PersistAliveConnection(const AliveConnection&) { return 0; }   // datastore/datastore.go:19
};

struct AggregatorConfig {
  int Device = 0;
  uint32_t MaxEndpoints = 1u << 16;
  uint32_t MaxPairs = 1u << 18;
  size_t BatchSize = 1u << 16;   // records per alz_submit_l7
};

class Aggregator {
 public:
  Aggregator(DataStore* ds, const AggregatorConfig& cfg);
  ~Aggregator();
  Aggregator(const Aggregator&) = delete;
  Aggregator& operator=(const Aggregator&) = delete;

  bool Ok() const { return h_ != nullptr; }
  const std::string& LastError() const { return err_; }
  // events dropped because a submit failed (capacity, CUDA error): the reference only logs such errors too
  // (aggregator/data.go:1244-1247), but the count is kept
  uint64_t DroppedEvents() const { return dropped_events_; }

  // All Process* methods and Flush may be called from several threads (the reference runs 4*NumCPU processL7
  // workers, aggregator/data.go:230-232); the batch buffer is guarded by one mutex, the library below is
  // thread-safe on its own.

  void ProcessK8s(const K8sResourceMessage& m);
  void ProcessL7(const L7Event& e);
  void ProcessTcpConnect(const TcpConnectEvent& e);
  // close the window: rows grouped by edge go to ds->PersistEdgeWindow. Returns 0 or an alz_status.
  int Flush(bool with_scores = false);
  // Rolling windows and tiered history (docs/SPEC.md §12, §13): keep the last `depth` flushed windows (depth 0: off)
  // and the tiers (empty: off) on the device. Rows are summed by id, so from here on a freed pod or service id is
  // not handed to another UID while a retained entry or an open block can still contain it.
  // Returns 0 or the status of the call that refused its part (alz_window_history, alz_window_history_tiers).
  int SetHistory(uint32_t depth, uint64_t arena_rows, const std::vector<alz_history_tier>& tiers = {});
  // the last k entries of `tier` (0: flushed windows, 1..n: the tiers) added up per edge go to
  // ds->PersistEdgeWindow, as a flush's rows do. info may be null. with_scores: each row's Score is the GNN anomaly
  // score of the row in the rollup's graph (docs/SPEC.md §15), as Flush(true) scores a window. Returns 0 or an
  // alz_status.
  int Rollup(uint32_t tier, uint32_t k, alz_rollup_info* info = nullptr, bool with_scores = false);
  // the last `windows` flushed windows up to now (docs/SPEC.md §14: ALZ_SPAN_AT_MOST or ALZ_SPAN_AT_LEAST; the span
  // covered is info->r.windows), summed from every retained piece, go to ds->PersistEdgeWindow as a flush's rows do.
  // info may be null; with_scores as in Rollup. Returns 0 or an alz_status.
  int RollupSpan(uint64_t windows, uint32_t mode, alz_span_info* info = nullptr, bool with_scores = false);
  // Anomalies' source for the last flushed window; the other sources are the rollup kinds ALZ_ROLLUP_*
  static constexpr uint32_t kLastWindow = 0xFFFFFFFFu;
  // the k rows of `source` with the highest GNN anomaly scores >= min_score (docs/SPEC.md §16: fewer when fewer
  // qualify), best first, ties by row order, Score set, into *out (not to the data store). A rollup source is the
  // last Rollup / RollupSpan of that kind. info may be null. Returns 0 or an alz_status.
  int Anomalies(uint32_t source, uint32_t k, float min_score, std::vector<EdgeWindow>* out,
                alz_top_info* info = nullptr);
  // Edge metrics (docs/SPEC.md §17) of `source` (kLastWindow or a rollup kind, as in Anomalies): (*values)[i * m.size()
  // + j] is metric j of row i, in the source's row order. Returns 0 or an alz_status.
  int EdgeMetrics(uint32_t source, const std::vector<alz_metric>& metrics, std::vector<double>* values);
  // the k rows of `source` with the highest values of `metric` >= min_value (fewer when fewer qualify), highest
  // first, ties by row order, Value set, into *out (not to the data store): "the slowest / most failing edges".
  // info may be null. Returns 0 or an alz_status.
  int TopEdges(uint32_t source, const alz_metric& metric, uint32_t k, double min_value, std::vector<EdgeWindow>* out,
               alz_top_info* info = nullptr);
  // Edge changes (docs/SPEC.md §18). PinBaseline copies the rows of `source` (kLastWindow or a rollup kind, as in
  // Anomalies) into the library's baseline; info may be null. Rows are matched by id, so while a baseline is pinned
  // no pod or service id unmapped in the oldest window it covers or later is handed to another UID, including ids
  // that were already free when it was pinned; ClearBaseline or another pin releases that hold. A source in which
  // such an id has already gone to another UID (a rollup result older than SetHistory's hold) cannot be compared by
  // id: the pin is refused with ALZ_E_STATE and no baseline is left. Returns 0 or an alz_status.
  int PinBaseline(uint32_t source, alz_rollup_info* info = nullptr);
  int ClearBaseline();
  // The rows of `source` and the baseline whose presence is in `presence` (ALZ_PRESENT_* mask) with one metric's
  // change by `mode` (ALZ_CHANGE_*), into *out: k = 0 every such row in key order, else the k largest changes >=
  // min_change, largest first, ties in key order. info may be null. Returns 0 or an alz_status.
  int Changes(uint32_t source, const alz_metric& metric, uint32_t mode, uint32_t presence, uint32_t k,
              double min_change, std::vector<EdgeChange>* out, alz_change_info* info = nullptr);
  // Node changes (docs/SPEC.md §23): the nodes with rows on side `side` (ALZ_SIDE_*) of `source` (kLastWindow or a
  // rollup kind, as in Anomalies) and of the baseline whose presence is in `presence`, with one metric's change of that
  // side by `mode`, into *out: k = 0 every such node in node order, else the k largest changes >= min_change, largest
  // first, ties in node order: "what changed since the deploy, per service". Nodes are matched by id and named as
  // Nodes names them; PinBaseline's hold makes that correct by UID, so a pod deleted after the pin is GONE under its
  // own UID and a pod added since is NEW under its own. info may be null. Returns 0 or an alz_status.
  int NodeChanges(uint32_t source, uint32_t side, const alz_metric& metric, uint32_t mode, uint32_t presence,
                  uint32_t k, double min_change, std::vector<NodeChange>* out, alz_change_info* info = nullptr);
  // Edge series (docs/SPEC.md §19) over the last k entries of `tier` (0: flushed windows, 1..n: the tiers), oldest
  // first; *points (may be null) gets what a rollup of each entry alone reports. Series gives one series per row of
  // `source` (kLastWindow or a rollup kind, as in Anomalies), in its row order. SeriesFor gives one per edge named by
  // UID, in the caller's order; an edge whose UID has no id (never seen, or freed) is absent at every point. Both match
  // rows by id. That is correct by UID because SetHistory's hold never hands an id to another UID while a retained
  // entry may carry it: a deleted pod's id stays its own until no entry covers the window it was deleted in, so its
  // edges show under its UID up to its deletion and under no other UID. Series names the source's rows through
  // alz_edge_top*, so the library's metric results refer to that call afterwards. Returns 0 or an alz_status.
  int Series(uint32_t source, uint32_t tier, uint32_t k, const std::vector<alz_metric>& metrics,
             std::vector<EdgeSeries>* out, std::vector<alz_rollup_info>* points = nullptr);
  int SeriesFor(const std::vector<EdgeRef>& edges, uint32_t tier, uint32_t k, const std::vector<alz_metric>& metrics,
                std::vector<EdgeSeries>* out, std::vector<alz_rollup_info>* points = nullptr);
  // Edge trends (docs/SPEC.md §20): the `top` rows of `source` (kLastWindow or a rollup kind, as in Anomalies) with the
  // largest valid trends >= min_trend of one metric over the last k entries of `tier`, largest first, ties in row
  // order, each with its series, into *out; *points (may be null) as in Series. Rows are named by UID as Series names
  // them, which SetHistory's hold makes correct over the whole retained history. top = 0: ALZ_E_INVAL. Returns 0 or an
  // alz_status.
  int Trends(uint32_t source, uint32_t tier, uint32_t k, const alz_metric& metric, const alz_trend& trend,
             uint32_t top, double min_trend, std::vector<EdgeTrend>* out,
             std::vector<alz_rollup_info>* points = nullptr);
  // Node metrics (docs/SPEC.md §21) of `source` (kLastWindow or a rollup kind, as in Anomalies): every node of its rows
  // with both sides' sums and `metrics` of side `side` (ALZ_SIDE_IN: the requests a node served; ALZ_SIDE_OUT: the ones
  // it made), in node order. Nodes are grouped and named by id; that is correct by UID over a rollup because
  // SetHistory's hold never hands an id to another UID while a retained entry or an open block can carry it, so a pod
  // deleted inside the rollup's span still shows under its own UID. Returns 0 or an alz_status.
  int Nodes(uint32_t source, uint32_t side, const std::vector<alz_metric>& metrics, std::vector<NodeWindow>* out);
  // the k nodes of `source` with the highest values of `metric` on side `side` >= min_value (fewer when fewer qualify),
  // highest first, ties in node order, Values = {the value}: "the slowest / most failing services". Named as Nodes
  // names them. info may be null. Returns 0 or an alz_status.
  int TopNodes(uint32_t source, uint32_t side, const alz_metric& metric, uint32_t k, double min_value,
               std::vector<NodeWindow>* out, alz_top_info* info = nullptr);
  // Node series (docs/SPEC.md §22) of side `side` over the last k entries of `tier` (0: flushed windows, 1..n: the
  // tiers), oldest first; *points (may be null) as in Series. NodeSeries gives one series per node of `source`
  // (kLastWindow or a rollup kind, as in Anomalies), in node order, named as Nodes names them. NodeSeriesFor gives one
  // per node named by UID, in the caller's order; a node whose UID has no id (never seen, or freed) is absent at every
  // point. Both group rows by id, which SetHistory's hold makes correct by UID over the whole retained history: a
  // deleted pod's points show under its UID up to its deletion and under no other UID. Returns 0 or an alz_status.
  int NodeSeries(uint32_t source, uint32_t side, uint32_t tier, uint32_t k, const std::vector<alz_metric>& metrics,
                 std::vector<NodeSeriesRow>* out, std::vector<alz_rollup_info>* points = nullptr);
  int NodeSeriesFor(const std::vector<NodeRef>& nodes, uint32_t side, uint32_t tier, uint32_t k,
                    const std::vector<alz_metric>& metrics, std::vector<NodeSeriesRow>* out,
                    std::vector<alz_rollup_info>* points = nullptr);
  // Node trends (docs/SPEC.md §22): the `top` nodes of `source` with the largest valid trends >= min_trend of one
  // metric of side `side` over the last k entries of `tier`, largest first, ties in node order, each with its node row
  // and its series, into *out; named as Nodes names them. top = 0: ALZ_E_INVAL. Returns 0 or an alz_status.
  int NodeTrends(uint32_t source, uint32_t side, uint32_t tier, uint32_t k, const alz_metric& metric,
                 const alz_trend& trend, uint32_t top, double min_trend, std::vector<NodeTrend>* out,
                 std::vector<alz_rollup_info>* points = nullptr);
  // Groups (docs/SPEC.md §24). SetGroups replaces the group map: each member's node goes to its group, named by a
  // string the adapter interns; an empty list clears the map. A member is resolved by UID whenever the map is sent:
  // before the next group call after SetGroups, and again before a group call whenever an id was handed out or freed
  // since the last send. A member whose UID has no id then is skipped, and the first of repeated members counts.
  // SetHistory's hold keeps a deleted pod's id, and so its membership, for every retained row that carries it.
  int SetGroups(const std::vector<GroupMember>& members);
  // the group-edge rows of `source` (kLastWindow or a rollup kind, as in Anomalies) into *out, in the library's order:
  // a group end is Type "group", UID the group's name; an unmapped end is named as ToEdges names it. info may be null.
  // Returns 0 or an alz_status.
  int GroupEdges(uint32_t source, std::vector<EdgeWindow>* out, alz_group_info* info = nullptr);
  // the §21 nodes of the group-edge rows with `metrics` of side `side`, in node order (groups last), named as
  // GroupEdges names the ends: "what is deployment checkout's inbound p99 over the last hour"
  int GroupNodes(uint32_t source, uint32_t side, const std::vector<alz_metric>& metrics, std::vector<NodeWindow>* out);
  // the k group nodes with the highest values of `metric` on side `side` >= min_value, as TopNodes ranks nodes
  int TopGroupNodes(uint32_t source, uint32_t side, const alz_metric& metric, uint32_t k, double min_value,
                    std::vector<NodeWindow>* out, alz_top_info* info = nullptr);
  // Group changes (docs/SPEC.md §25): Changes and NodeChanges over the group-edge rows and group nodes of `source` and
  // of the baseline, both grouped by the map SetGroups gave, resolved by UID as for every group call: "what changed
  // since the deploy, per deployment". A rolling deploy's pods are NEW and GONE under their own UIDs; their group is
  // BOTH, with quantiles of the summed histograms on each side. GroupChanges names ends as GroupEdges does,
  // GroupNodeChanges nodes as GroupNodes does. The map is the current one on both sides: a baseline pod stays
  // resolvable by UID after its deletion through PinBaseline's hold, but a member dropped from the list since the pin
  // no longer maps, and its baseline rows then show under the pod's own UID. info may be null. Returns 0 or an
  // alz_status.
  int GroupChanges(uint32_t source, const alz_metric& metric, uint32_t mode, uint32_t presence, uint32_t k,
                   double min_change, std::vector<EdgeChange>* out, alz_change_info* info = nullptr);
  int GroupNodeChanges(uint32_t source, uint32_t side, const alz_metric& metric, uint32_t mode, uint32_t presence,
                       uint32_t k, double min_change, std::vector<NodeChange>* out, alz_change_info* info = nullptr);
  // Group series and trends (docs/SPEC.md §26): Series, SeriesFor, NodeSeries, NodeSeriesFor, Trends and NodeTrends
  // over groups, with every retained entry grouped by the map SetGroups gave, resolved by UID as for every group call:
  // "what was deployment checkout's inbound p99, minute by minute", "which deployments are getting worse". GroupSeries
  // and GroupTrends name ends as GroupEdges does, GroupNodeSeries and GroupNodeTrends nodes as GroupNodes does. In the
  // For forms a ref of Type "group" names a group by the name SetGroups gave it; a name SetGroups never gave, like a
  // UID with no id, is absent at every point. The map is the current one for every point: a rolled-out pod keeps
  // contributing to its deployment's earlier points only while it stays in the member list, and SetHistory's hold
  // keeps its id resolvable for as long as a retained entry carries it. *points (may be null) as in Series. Returns 0
  // or an alz_status.
  int GroupSeries(uint32_t source, uint32_t tier, uint32_t k, const std::vector<alz_metric>& metrics,
                  std::vector<EdgeSeries>* out, std::vector<alz_rollup_info>* points = nullptr);
  int GroupSeriesFor(const std::vector<EdgeRef>& edges, uint32_t tier, uint32_t k,
                     const std::vector<alz_metric>& metrics, std::vector<EdgeSeries>* out,
                     std::vector<alz_rollup_info>* points = nullptr);
  int GroupNodeSeries(uint32_t source, uint32_t side, uint32_t tier, uint32_t k, const std::vector<alz_metric>& metrics,
                      std::vector<NodeSeriesRow>* out, std::vector<alz_rollup_info>* points = nullptr);
  int GroupNodeSeriesFor(const std::vector<NodeRef>& nodes, uint32_t side, uint32_t tier, uint32_t k,
                         const std::vector<alz_metric>& metrics, std::vector<NodeSeriesRow>* out,
                         std::vector<alz_rollup_info>* points = nullptr);
  int GroupTrends(uint32_t source, uint32_t tier, uint32_t k, const alz_metric& metric, const alz_trend& trend,
                  uint32_t top, double min_trend, std::vector<EdgeTrend>* out,
                  std::vector<alz_rollup_info>* points = nullptr);
  int GroupNodeTrends(uint32_t source, uint32_t side, uint32_t tier, uint32_t k, const alz_metric& metric,
                      const alz_trend& trend, uint32_t top, double min_trend, std::vector<NodeTrend>* out,
                      std::vector<alz_rollup_info>* points = nullptr);
  // Correlations (docs/SPEC.md §29): the `top` rows (Correlations), nodes of side `side` (NodeCorrelations), group
  // edges (GroupCorrelations) or group nodes of side `side` (GroupNodeCorrelations) of `source` whose series of
  // `metric` over the last k entries of `tier` followed a target most closely at the best lag up to corr.max_lag,
  // valid scores >= min_score, largest first, ties in source order, each with its series; named as Trends,
  // NodeTrends, GroupTrends and GroupNodeTrends name them. The target is a CorrTarget, or the series of one edge, node
  // or group named as the matching *SeriesFor call names it; in that form the target's own row is left out of the
  // result (top others are returned). "Who moved with checkout's inbound p99, and a point earlier?" A flush between the
  // target's series and the call: ALZ_E_STATE. *points (may be null) as in Series. Returns 0 or an alz_status.
  int Correlations(uint32_t source, uint32_t tier, uint32_t k, const alz_metric& metric, const alz_corr& corr,
                   const CorrTarget& target, uint32_t top, double min_score, std::vector<EdgeCorr>* out,
                   std::vector<alz_rollup_info>* points = nullptr);
  int Correlations(uint32_t source, uint32_t tier, uint32_t k, const alz_metric& metric, const alz_corr& corr,
                   const EdgeRef& target, uint32_t top, double min_score, std::vector<EdgeCorr>* out,
                   std::vector<alz_rollup_info>* points = nullptr);
  int NodeCorrelations(uint32_t source, uint32_t side, uint32_t tier, uint32_t k, const alz_metric& metric,
                       const alz_corr& corr, const CorrTarget& target, uint32_t top, double min_score,
                       std::vector<NodeCorr>* out, std::vector<alz_rollup_info>* points = nullptr);
  int NodeCorrelations(uint32_t source, uint32_t side, uint32_t tier, uint32_t k, const alz_metric& metric,
                       const alz_corr& corr, const NodeRef& target, uint32_t top, double min_score,
                       std::vector<NodeCorr>* out, std::vector<alz_rollup_info>* points = nullptr);
  int GroupCorrelations(uint32_t source, uint32_t tier, uint32_t k, const alz_metric& metric, const alz_corr& corr,
                        const CorrTarget& target, uint32_t top, double min_score, std::vector<EdgeCorr>* out,
                        std::vector<alz_rollup_info>* points = nullptr);
  int GroupCorrelations(uint32_t source, uint32_t tier, uint32_t k, const alz_metric& metric, const alz_corr& corr,
                        const EdgeRef& target, uint32_t top, double min_score, std::vector<EdgeCorr>* out,
                        std::vector<alz_rollup_info>* points = nullptr);
  int GroupNodeCorrelations(uint32_t source, uint32_t side, uint32_t tier, uint32_t k, const alz_metric& metric,
                            const alz_corr& corr, const CorrTarget& target, uint32_t top, double min_score,
                            std::vector<NodeCorr>* out, std::vector<alz_rollup_info>* points = nullptr);
  int GroupNodeCorrelations(uint32_t source, uint32_t side, uint32_t tier, uint32_t k, const alz_metric& metric,
                            const alz_corr& corr, const NodeRef& target, uint32_t top, double min_score,
                            std::vector<NodeCorr>* out, std::vector<alz_rollup_info>* points = nullptr);
  // Reach (docs/SPEC.md §27): the nodes of `source` within max_hops rows of the seeds, in direction dir
  // (ALZ_REACH_DOWN: what the seeds call; ALZ_REACH_UP: who calls them; ALZ_REACH_ANY), in (hops, node key) order, and
  // the rows crossed, in the source's order, named as ToEdges names ends. filter (may be null): only rows whose value
  // of that metric is >= min_value are followed ("follow the calls that return 5xx"). A seed whose UID has no id is
  // skipped like a seed no row holds; when no seed resolves, *nodes and *rows are empty and info counts nothing. info
  // may be null. Returns 0 or an alz_status.
  int Reach(uint32_t source, const std::vector<NodeRef>& seeds, uint32_t dir, uint32_t max_hops,
            const alz_metric* filter, double min_value, std::vector<ReachNode>* nodes, std::vector<EdgeWindow>* rows,
            alz_reach_info* info = nullptr);
  // Reach over the group-edge rows of `source` under the map SetGroups gave (sent first, as for every group call):
  // "which deployments does checkout depend on". A seed of Type "group" names a group by its SetGroups name; a name
  // SetGroups never gave is skipped like a UID with no id. Nodes and rows are named as GroupNodes / GroupEdges name
  // them.
  int GroupReach(uint32_t source, const std::vector<NodeRef>& seeds, uint32_t dir, uint32_t max_hops,
                 const alz_metric* filter, double min_value, std::vector<ReachNode>* nodes,
                 std::vector<EdgeWindow>* rows, alz_reach_info* info = nullptr);
  static constexpr uint32_t kReachNone = 0xFFFFFFFFu;   // ReachNode.Parent / Row of a seed
  // Cycles (docs/SPEC.md §28): the strongly connected components of `source`'s nodes, following rows from caller to
  // callee. *nodes lists the nodes of every component of at least min_size nodes (2: the services on a loop) in
  // (component, node index) order; *rows the rows inside the listed loops, by component then source order, named as
  // ToEdges names ends. filter (may be null): only rows whose value of that metric is >= min_value are followed
  // ("loops of failing calls"). info may be null. Returns 0 or an alz_status.
  int Cycles(uint32_t source, const alz_metric* filter, double min_value, uint32_t min_size,
             std::vector<CycleNode>* nodes, std::vector<EdgeWindow>* rows, alz_cycle_info* info = nullptr);
  // Cycles over the group-edge rows of `source` under the map SetGroups gave (sent first, as for every group call):
  // "which deployments call each other in a loop". A group's internal rows never make it a loop. Nodes and rows are
  // named as GroupNodes / GroupEdges name them.
  int GroupCycles(uint32_t source, const alz_metric* filter, double min_value, uint32_t min_size,
                  std::vector<CycleNode>* nodes, std::vector<EdgeWindow>* rows, alz_cycle_info* info = nullptr);
  int Stats(alz_stats* out);
  // one tick of clearSocketLines (aggregator/data.go:1681-1716, every 120 s there): with send_alive (the
  // reference's SEND_ALIVE_TCP_CONNECTIONS) every open connection with a pod at its source goes to
  // ds->PersistAliveConnection, then every socket line is garbage-collected (SocketLine.DeleteUnused)
  int ClearSocketLines(bool send_alive, int64_t check_time_ms = 0);

  static uint32_t ParseIPv4(const std::string& s, bool* ok);   // "a.b.c.d" -> the integer IntToIPv4 takes
  static std::string FormatIPv4(uint32_t ip);
  // parseHttpPayload's hostHeader (aggregator/data.go:508-531): "" when the reference finds none
  static std::string ParseHttpHostHeader(const std::string& payload);

 private:
  int SubmitBatch();   // requires mu_
  // a rollup call(out, cap, &n) of `kind` (ALZ_ROLLUP_*) into roll_, with_scores its GNN scores, then its rows to
  // ds->PersistEdgeWindow; requires mu_
  template <class Call>
  int PersistRollup(uint32_t kind, bool with_scores, Call call);
  // rows -> EdgeWindow with the UIDs the interners hold (scores: one per row, or null)
  std::vector<EdgeWindow> ToEdges(const alz_edge_out* rows, size_t n, const float* scores) const;
  // the UID of an edge end or node (type, id) as the interners and the Host table hold it
  std::string UidOf(uint8_t type, uint32_t id) const;
  // a change call(recs, cap, &n) into *recs (changes_ or node_changes_), grown once when the records do not fit
  // (ALZ_E_CAPACITY with n = the records; nothing written); requires mu_
  template <class Rec, class Call>
  int RunChanges(std::vector<Rec>* recs, size_t* n, Call call);
  // change records -> EdgeChange / NodeChange with the UIDs the interners and the group names hold
  std::vector<EdgeChange> ToChanges(const alz_edge_change* recs, size_t n) const;
  std::vector<NodeChange> ToNodeChanges(const alz_node_change* recs, size_t n) const;
  // node rows -> NodeWindow (values: nm per row, or null)
  std::vector<NodeWindow> ToNodes(const alz_node_out* rows, size_t n, const double* values, size_t nm) const;
  // the library's (type, id) of an edge end or node named by UID; false when the UID has no id
  bool EndOf(const std::string& type, const std::string& uid, uint8_t* t, uint32_t* v) const;
  // EndOf, and a group (Type "group") by the name SetGroups gave it; false for a name it never gave
  bool GroupEndOf(const std::string& type, const std::string& uid, uint8_t* t, uint32_t* v) const;
  // Reach and GroupReach: the seeds resolved by EndOf (group false) or GroupEndOf, the call, the results named
  int RunReach(bool group, uint32_t source, const std::vector<NodeRef>& seeds, uint32_t dir, uint32_t max_hops,
               const alz_metric* filter, double min_value, std::vector<ReachNode>* nodes,
               std::vector<EdgeWindow>* rows, alz_reach_info* info);
  // Cycles and GroupCycles: the call, the results named
  int RunCycles(bool group, uint32_t source, const alz_metric* filter, double min_value, uint32_t min_size,
                std::vector<CycleNode>* nodes, std::vector<EdgeWindow>* rows, alz_cycle_info* info);
  // ends -> the library's key of an edge named by UID; false when a UID has no id
  bool ToEnds(const EdgeRef& e, alz_edge_ends* out) const;
  // a series call(values, present, cap, &n, &P, points) into series_values_ / series_present_, then each series
  // row's Present and Values in *out (EdgeSeries or NodeSeriesRow; the names are the caller's); requires mu_
  template <class Row, class Call>
  int RunSeries(size_t nm, std::vector<Row>* out, std::vector<alz_rollup_info>* points, Call call);
  // the edge trends_top call `fn` (alz_edge_trends_top, alz_group_edge_trends_top) into trends_ and its rows named,
  // and the node one (alz_node_trends_top, alz_group_node_trends_top) into node_trends_; require mu_
  using EdgeTrendsTop = int (*)(alz_handle*, uint32_t, uint32_t, uint32_t, const alz_metric*, const alz_trend*,
                                uint32_t, double, alz_edge_trend*, alz_edge_out*, double*, uint8_t*, size_t, size_t*,
                                uint32_t*, alz_rollup_info*, alz_trend_info*);
  using NodeTrendsTop = int (*)(alz_handle*, uint32_t, uint32_t, uint32_t, uint32_t, const alz_metric*,
                                const alz_trend*, uint32_t, double, alz_node_trend*, alz_node_out*, double*, uint8_t*,
                                size_t, size_t*, uint32_t*, alz_rollup_info*, alz_trend_info*);
  int RunEdgeTrends(EdgeTrendsTop fn, uint32_t source, uint32_t tier, uint32_t k, const alz_metric& metric,
                    const alz_trend& trend, uint32_t top, double min_trend, std::vector<EdgeTrend>* out,
                    std::vector<alz_rollup_info>* points);
  int RunNodeTrends(NodeTrendsTop fn, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                    const alz_metric& metric, const alz_trend& trend, uint32_t top, double min_trend,
                    std::vector<NodeTrend>* out, std::vector<alz_rollup_info>* points);
  // the edge correlations_top call `fn` (alz_edge_correlations_top, alz_group_edge_correlations_top) into corrs_ and
  // its rows named, and the node one into node_corrs_; a row named `skip` (not null) is left out and top + 1 asked
  // for; require mu_
  using EdgeCorrTop = int (*)(alz_handle*, uint32_t, uint32_t, uint32_t, const alz_metric*, const alz_corr*,
                              const alz_corr_target*, uint32_t, double, alz_edge_corr*, alz_edge_out*, double*,
                              uint8_t*, size_t, size_t*, uint32_t*, alz_rollup_info*, alz_corr_info*);
  using NodeCorrTop = int (*)(alz_handle*, uint32_t, uint32_t, uint32_t, uint32_t, const alz_metric*, const alz_corr*,
                              const alz_corr_target*, uint32_t, double, alz_node_corr*, alz_node_out*, double*,
                              uint8_t*, size_t, size_t*, uint32_t*, alz_rollup_info*, alz_corr_info*);
  int RunEdgeCorr(EdgeCorrTop fn, uint32_t source, uint32_t tier, uint32_t k, const alz_metric& metric,
                  const alz_corr& corr, const CorrTarget& target, uint32_t top, double min_score,
                  const EdgeRef* skip, std::vector<EdgeCorr>* out, std::vector<alz_rollup_info>* points);
  int RunNodeCorr(NodeCorrTop fn, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                  const alz_metric& metric, const alz_corr& corr, const CorrTarget& target, uint32_t top,
                  double min_score, const NodeRef* skip, std::vector<NodeCorr>* out,
                  std::vector<alz_rollup_info>* points);
  // the group map resolved by UID sent to the library when SetGroups changed it or an interner handed out or freed an
  // id since the last send; requires mu_
  int SyncGroups();
  // UID <-> dense id (< 2^29). An id whose last IP mapping went away while window w was open may be carried by
  // window w, and by every retained entry and open block that covers w: it is recycled once `hold` more windows
  // have been flushed after w (hold 0: when w is flushed).
  struct Interner {
    std::unordered_map<std::string, uint32_t> ids;
    std::vector<std::string> names;
    std::vector<uint32_t> refs;                       // IP entries currently mapping to the id
    std::unordered_map<uint32_t, uint32_t> ip_to_id;  // mirror of the device table's value per IP
    std::vector<uint64_t> unmapped_in;                // the window that was open when refs last fell to 0
    std::vector<uint32_t> free_ids, pending_free;
    std::vector<uint32_t> held;                       // freed ids taken back while a pinned baseline may carry them
    std::vector<uint64_t> reused_after;               // unmapped_in of the id when another UID last took it (0: never)
    uint64_t changes = 0;                             // ids handed out or freed so far
    uint32_t Acquire(const std::string& uid);
    void Map(uint32_t ip, uint32_t id, uint64_t open_window);
    void Unmap(uint32_t ip, uint64_t open_window);
    // pinned_from: no id unmapped in that window or later is freed (0: no baseline pinned); held ids outside it are
    // freed again
    void EndWindow(uint64_t flushed, uint64_t hold, uint64_t pinned_from);
    // whether no id unmapped in window pinned_from or later has gone to another UID since
    bool CanHold(uint64_t pinned_from) const;
    // the free ids unmapped in window pinned_from or later are held
    void Hold(uint64_t pinned_from);
  };

  DataStore* ds_;
  alz_handle* h_ = nullptr;
  std::string err_;
  AggregatorConfig cfg_;
  alz_l7_rec* batch_ = nullptr;   // pinned (alz_pinned_alloc)
  size_t batch_n_ = 0;
  bool tables_dirty_ = false;
  std::mutex mu_;
  uint64_t dropped_events_ = 0;
  uint64_t windows_ = 0;          // windows flushed through Flush
  uint64_t hold_ = 0;             // windows a retained entry or open block can reach back (SetHistory)
  uint64_t pinned_from_ = 0;      // the oldest window the pinned baseline covers; 0: none pinned
  Interner pods_, svcs_;
  std::unordered_map<std::string, uint32_t> host_ids_;   // Host header text -> dense id (ALZ_NODE_OUTBOUND_HOST)
  std::vector<std::string> host_names_;
  std::vector<alz_edge_out> out_;
  std::vector<alz_edge_out> roll_;   // rows of the last Rollup, Anomalies or TopEdges
  std::vector<float> scores_;
  std::vector<double> values_;       // values of the last TopEdges
  std::vector<alz_alive_conn> alive_;
  std::vector<alz_edge_change> changes_;   // records of the last Changes
  std::vector<double> series_values_;      // values and presence of the last Series / SeriesFor / NodeSeries*
  std::vector<uint8_t> series_present_;
  std::vector<alz_edge_trend> trends_;     // records, rows, series and presence of the last Trends
  std::vector<alz_edge_out> trend_rows_;
  std::vector<double> trend_values_;
  std::vector<uint8_t> trend_present_;
  std::vector<alz_node_out> nodes_;       // node rows, values and indices of the last Nodes / TopNodes
  std::vector<double> node_values_;
  std::vector<alz_node_change> node_changes_;   // records of the last NodeChanges
  std::vector<alz_node_trend> node_trends_;   // records, node rows, series and presence of the last NodeTrends
  std::vector<alz_node_out> node_trend_rows_;
  std::vector<alz_edge_corr> corrs_;          // records of the last Correlations / GroupCorrelations (rows, series and
  std::vector<alz_node_corr> node_corrs_;     // presence in trend_rows_ / node_trend_rows_ / trend_values_ / ...)
  std::vector<alz_reach_node> reach_nodes_;   // the records and row positions of the last Reach / GroupReach
  std::vector<uint32_t> reach_index_;
  std::vector<alz_cycle_node> cycle_nodes_;   // the records and row positions of the last Cycles / GroupCycles
  std::vector<uint32_t> cycle_index_;
  std::vector<GroupMember> members_;                    // the group map as SetGroups gave it
  std::unordered_map<std::string, uint32_t> group_ids_;  // group name -> dense id (ALZ_NODE_GROUP)
  std::vector<std::string> group_names_;
  bool groups_sent_ = true;                             // the library holds members_ as resolved at groups_changes_
  uint64_t groups_changes_ = 0;                         // the interners' changes at the last send
};

}  // namespace alaz
