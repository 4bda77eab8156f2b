// alz_trends.cu — edge trends (docs/SPEC.md §20): one statistic per source row over its §19 series of one metric,
// and the top rows by it with their series; node trends (§22): the same per source node over its node series; group
// trends (§26): the same per group edge or group node of the source over its group series.
//
//   series  the §19 path (alz_series.cu: keys, match, the §17 metric kernels over the slots) with nm = 1, into the
//           trend state's own SeriesBufs, so a trend call leaves the series calls' device results alone; for nodes
//           the §22 path (alz_node_series.cu) into the node trend state's own NodeSeriesBufs; for groups the §26
//           path (alz_group_series.cu) into the group trend state's own GroupSeriesBufs, whose group-edge rows are the
//           edge records' heads and the selection's rows
//   trend   one thread per series row walks its P values and presence bytes in the SPEC's order: the sums of the
//           used, recent and earlier points, then a second pass for Sxy / Sxx or the squared deviations. It writes
//           the 48-byte record and, for a top call, an 8-byte selection value: the trend's bits for a valid row, all
//           ones (a negative NaN, key 0) otherwise. A non-NaN min_trend has key >= key(-inf) > 0, so an invalid row is
//           never eligible. A warp-reduced count of the valid rows goes to a pinned word that the call's wait reads.
//           An edge record and a node record differ only in their first 16 bytes (EdgeHead, NodeHead).
//   top     the §17 selection over those values, which gathers the source rows (for nodes, a gather of the source's
//           node rows follows), then one gather of the selected records and their P-point series and presence
// The orchestration (series, pass, selection, gather, waits) is scored_series_locked, which the correlations
// (alz_corr.cu) share with their own pass.
// Every SPEC operation is rounded on its own: nvcc would contract s + a * b into a fused multiply-add, so the
// arithmetic is written with the round-to-nearest intrinsics. Waits: a full-list edge call waits once, at its end (the
// ring's clocks and the valid count, and a host call's results); a top call adds the selection's wait. A node call
// adds the node series' waits (the source's node count, the entries' present slots) before those.
#include <algorithm>
#include <cmath>
#include <mutex>
#include <string>

#include "alz_metrics.cuh"

using namespace alz;
using namespace alz::metrics;

static_assert(sizeof(alz_edge_trend) == 48, "alz_edge_trend is three 16-byte stores");
static_assert(sizeof(alz_trend) == 24, "alz_trend is 24 bytes");
static_assert(sizeof(alz_node_trend) == sizeof(alz_edge_trend), "a node record is written as an edge record");
static_assert(offsetof(alz_node_trend, valid) == offsetof(alz_edge_trend, valid) &&
                  offsetof(alz_node_trend, value) == offsetof(alz_edge_trend, from) &&
                  offsetof(alz_node_trend, _pad2) == offsetof(alz_edge_trend, to) &&
                  offsetof(alz_node_trend, index) == offsetof(alz_edge_trend, index) &&
                  offsetof(alz_node_trend, used) == offsetof(alz_edge_trend, used) &&
                  offsetof(alz_node_trend, trend) == offsetof(alz_edge_trend, trend) &&
                  offsetof(alz_node_trend, recent) == offsetof(alz_edge_trend, recent) &&
                  offsetof(alz_node_trend, before) == offsetof(alz_edge_trend, before),
              "from `valid` on, alz_node_trend is laid out as alz_edge_trend (NodeHead writes the first 16 bytes)");

namespace {

constexpr uint64_t kInvalidValue = ~0ull;   // a negative NaN: key 0, below every non-NaN min_trend

struct TrendArgs {
  uint32_t n, points;
  const double* values;      // values[i * points + j]
  const uint8_t* present;    // present[i * points + j]
  uint32_t stat, falling, zero, recent, min_points;
};

__device__ __forceinline__ double pos_inf() { return __longlong_as_double(0x7FF0000000000000ll); }
__device__ __forceinline__ double neg_inf() { return __longlong_as_double((long long)0xFFF0000000000000ull); }

// num / den with the §18 RATIO zero rule: den = 0 gives +inf when num > 0, else 1.0
__device__ __forceinline__ double ratio_of(double num, double den) {
  if (den > 0.0) return __ddiv_rn(num, den);
  return num > 0.0 ? pos_inf() : 1.0;
}

struct Stat {
  double t, recent, before;
  uint32_t used;
  bool ok;
};

// The SPEC §20 statistic of series row i
__device__ __forceinline__ Stat trend_of(const TrendArgs& a, uint32_t i) {
  const uint32_t P = a.points;
  const uint32_t lo = P > a.recent ? P - a.recent : 0u;   // B = U ∩ [0, lo), R = U ∩ [lo, P)
  const double* __restrict__ y = a.values + (size_t)i * P;
  const uint8_t* __restrict__ pr = a.present + (size_t)i * P;
  // pass 1: the sums of U, B and R in ascending j, and the exact sum of U's point indices
  double su = 0.0, sb = 0.0, sr = 0.0;
  uint32_t nu = 0, nb = 0, nr = 0;
  uint64_t sj = 0;
  for (uint32_t j = 0; j < P; ++j) {
    if (!(a.zero || pr[j])) continue;
    const double v = y[j];
    su = __dadd_rn(su, v);
    sj += j;
    ++nu;
    if (j < lo) { sb = __dadd_rn(sb, v); ++nb; } else { sr = __dadd_rn(sr, v); ++nr; }
  }
  const double before = nb ? __ddiv_rn(sb, (double)nb) : 0.0;
  const double recent = nr ? __ddiv_rn(sr, (double)nr) : 0.0;
  double t = 0.0;
  bool ok;
  if (a.stat == ALZ_TREND_SLOPE) {
    ok = nu >= 2u;
    if (ok) {   // pass 2: Sxy and Sxx about the means
      const double xm = __ddiv_rn((double)sj, (double)nu);
      const double ym = __ddiv_rn(su, (double)nu);
      double sxy = 0.0, sxx = 0.0;
      for (uint32_t j = 0; j < P; ++j) {
        if (!(a.zero || pr[j])) continue;
        const double dx = __dsub_rn((double)j, xm);
        sxy = __dadd_rn(sxy, __dmul_rn(dx, __dsub_rn(y[j], ym)));
        sxx = __dadd_rn(sxx, __dmul_rn(dx, dx));
      }
      t = __ddiv_rn(sxy, sxx);
      if (a.falling) t = __dsub_rn(0.0, t);
    }
  } else if (a.stat == ALZ_TREND_SHIFT) {
    ok = nr >= 1u && nb >= 1u;
    if (ok) t = a.falling ? __dsub_rn(before, recent) : __dsub_rn(recent, before);
  } else if (a.stat == ALZ_TREND_RATIO) {
    ok = nr >= 1u && nb >= 1u;
    if (ok) t = a.falling ? ratio_of(before, recent) : ratio_of(recent, before);
  } else {   // ALZ_TREND_ZSCORE
    ok = nr >= 1u && nb >= 2u;
    if (ok) {   // pass 2: the squared deviations of B about its mean
      double ss = 0.0;
      for (uint32_t j = 0; j < lo; ++j) {
        if (!(a.zero || pr[j])) continue;
        const double d = __dsub_rn(y[j], before);
        ss = __dadd_rn(ss, __dmul_rn(d, d));
      }
      const double sd = __dsqrt_rn(__ddiv_rn(ss, (double)nb));
      const double d = a.falling ? __dsub_rn(before, recent) : __dsub_rn(recent, before);
      if (sd > 0.0) t = __ddiv_rn(d, sd);
      else t = d > 0.0 ? pos_inf() : (d < 0.0 ? neg_inf() : 0.0);
    }
  }
  ok = ok && nu >= a.min_points;
  if (!ok) t = 0.0;
  return Stat{t, recent, before, nu, ok};
}

// Thread i: series row i. rec[i] its record; with sel, sel[i] its selection value; *valid += the valid rows.
template <class Head>
__global__ void __launch_bounds__(256) trend_kernel(const __grid_constant__ TrendArgs a, const Head head,
                                                    alz_edge_trend* __restrict__ rec, uint64_t* __restrict__ sel,
                                                    uint32_t* __restrict__ valid_cnt) {
  const uint32_t stride = gridDim.x * blockDim.x;
  uint32_t n_valid = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += stride) {
    const Stat r = trend_of(a, i);
    n_valid += r.ok;
    const uint64_t tb = (uint64_t)__double_as_longlong(r.t), rb = (uint64_t)__double_as_longlong(r.recent),
                   bb = (uint64_t)__double_as_longlong(r.before);
    uint4* o = reinterpret_cast<uint4*>(rec + i);
    o[0] = head(i, r.ok);
    o[1] = make_uint4(i, r.used, (uint32_t)tb, (uint32_t)(tb >> 32));
    o[2] = make_uint4((uint32_t)rb, (uint32_t)(rb >> 32), (uint32_t)bb, (uint32_t)(bb >> 32));
    if (sel) sel[i] = r.ok ? tb : kInvalidValue;
  }
  n_valid = __reduce_add_sync(0xFFFFFFFFu, n_valid);   // every lane of the warp leaves the loop to get here
  if ((threadIdx.x & 31u) == 0 && n_valid) atomicAdd(valid_cnt, n_valid);
}

// Result j: the record, the series and the presence of source row idx[j]. Thread t: word w = t % (P + 3) of result
// t / (P + 3), w < 3 a 16-byte word of the record, else point w - 3.
__global__ void __launch_bounds__(256) trend_gather_kernel(const uint32_t* __restrict__ idx, uint32_t m, uint32_t P,
                                                           const alz_edge_trend* __restrict__ rec,
                                                           const double* __restrict__ values,
                                                           const uint8_t* __restrict__ present,
                                                           alz_edge_trend* __restrict__ top_rec,
                                                           double* __restrict__ top_values,
                                                           uint8_t* __restrict__ top_present) {
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t per = P + 3u;
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < m * per; t += stride) {
    const uint32_t j = t / per, w = t - j * per;
    const uint32_t i = idx[j];
    if (w < 3u) {
      reinterpret_cast<uint4*>(top_rec + j)[w] = reinterpret_cast<const uint4*>(rec + i)[w];
    } else {
      const uint32_t p = w - 3u;
      top_values[(size_t)j * P + p] = values[(size_t)i * P + p];
      top_present[(size_t)j * P + p] = present[(size_t)i * P + p];
    }
  }
}

}  // namespace

void alz::metrics::free_scored_state(alz_trend_state*& s) {
  if (!s) return;
  s->ser.free();
  s->nser.free();
  s->gser.free();
  free_bufs({&s->rec, &s->sel_val, &s->valid_cnt, &s->top_rec, &s->top_values, &s->top_present, &s->top_nodes,
             &s->target});
  s->sel.free();
  if (s->h_valid) cudaFreeHost(s->h_valid);
  if (s->h_target) cudaFreeHost(s->h_target);
  delete s;
  s = nullptr;
}

void alz_internal_free_trends(alz_handle* h) { free_scored_state(h->trends); }
void alz_internal_free_node_trends(alz_handle* h) { free_scored_state(h->node_trends); }
void alz_internal_free_group_trends(alz_handle* h) { free_scored_state(h->group_trends); }

int alz::metrics::scored_series_locked(alz_handle* h, alz_trend_state*& sp, const char* what, const ScoredCall& c,
                                       size_t cap, void* copy_out, ScorePass& pass, ScoredResult* res,
                                       uint32_t* n_points, alz_rollup_info* points, alz_trend_info* info) {
  CK(cudaSetDevice(h->device));
  const alz_edge_out* rows = h->d_out;
  size_t n = h->last_n_edges;
  if (c.given) {
    n = c.given_n;
    if (n > kMaxRows || (uint64_t)n * c.given_points > kMaxRows) return ALZ_E_CAPACITY;
  } else if (c.node || c.group) {
    const int rc = node_source(h, c.source, &rows, &n);
    if (rc != ALZ_OK) return rc;
  } else {
    if (c.source != ALZ_SOURCE_WINDOW) {
      const int rc = alz_internal_rollup_rows(h, c.source, &rows, &n);
      if (rc != ALZ_OK) return rc;
    }
    if (n > kMaxRows) return ALZ_E_CAPACITY;
  }
  if (!sp) sp = new alz_trend_state();
  alz_trend_state* s = sp;
  if (!s->h_valid) {
    void* p = nullptr;
    if (cudaMallocHost(&p, sizeof(uint32_t)) != cudaSuccess) {
      h->last_err = std::string(what) + ": " + cudaGetErrorString(cudaGetLastError());
      return ALZ_E_NOMEM;
    }
    s->h_valid = static_cast<uint32_t*>(p);
  }
  size_t n_rows = 0;   // series rows: the source's rows, or its nodes
  uint64_t rows_in = 0;
  const size_t room = c.top ? SIZE_MAX : cap;
  int rc = ALZ_OK;
  if (c.given) {
    n_rows = n;
    *n_points = c.given_points;
    if (n > room) rc = ALZ_E_CAPACITY;
  } else {
    rc = c.group  ? run_group_series_rows(h, s->gser, rows, n, c.node, c.side, c.tier, c.k, c.ms, c.top, room,
                                          &n_rows, n_points, &rows_in)
         : c.node ? run_node_series_rows(h, s->nser, rows, n, c.side, c.tier, c.k, c.ms, c.top, room, &n_rows,
                                         n_points, &rows_in)
                  : run_series_rows(h, s->ser, rows, n, c.tier, c.k, c.ms, room, &n_rows, n_points, &rows_in);
  }
  res->m = c.top ? 0 : n_rows;
  if (rc != ALZ_OK) return rc;
  const uint32_t P = *n_points;
  const size_t N = n_rows;
  const NodeSeriesBufs& nser = c.group ? s->gser.s : s->nser;   // node or group series
  if (c.group && !c.node) rows = static_cast<const alz_edge_out*>(s->gser.edges.p);   // the series rows
  const double* values = c.given ? c.given_values
                                 : static_cast<const double*>(c.node || c.group ? nser.values.p : s->ser.values.p);
  const uint8_t* present = c.given ? c.given_present
                                   : static_cast<const uint8_t*>(c.node || c.group ? nser.present.p
                                                                                    : s->ser.present.p);
  rc = reserve(h, {{&s->rec, std::max<size_t>(N, 1) * sizeof(alz_edge_trend)},
                   {&s->sel_val, c.top ? std::max<size_t>(N, 1) * 8 : 0},
                   {&s->valid_cnt, 4}});
  if (rc != ALZ_OK) return rc;
  cudaStream_t st = h->stream;
  uint32_t* d_valid = static_cast<uint32_t*>(s->valid_cnt.p);
  CK(cudaMemsetAsync(d_valid, 0, 4, st));
  alz_edge_trend* d_rec = static_cast<alz_edge_trend*>(s->rec.p);
  ScoredInput in;
  in.n = N;
  in.points = P;
  in.values = values;
  in.present = present;
  if (c.given) rows = nullptr;
  else if (c.node) in.keys = static_cast<const uint64_t*>(nser.keys.p);
  else in.rows = rows;
  rc = pass.launch(h, *s, in, d_rec, c.top ? static_cast<uint64_t*>(s->sel_val.p) : nullptr, d_valid);
  if (rc != ALZ_OK) return rc;
  CK(cudaMemcpyAsync(s->h_valid, d_valid, 4, cudaMemcpyDeviceToHost, st));   // read after the call's wait
  uint64_t above = 0;
  bool waited = false;
  if (c.top) {
    size_t m = 0;
    rc = select_top(h, s->sel, static_cast<const uint64_t*>(s->sel_val.p), (uint32_t)N, c.n_top, c.min_value,
                    c.node ? nullptr : rows, &m, &above);
    if (rc != ALZ_OK) return rc;
    waited = N > 0;   // the selection waited for its control block
    rc = reserve(h, {{&s->top_rec, std::max<size_t>(m, 1) * sizeof(alz_edge_trend)},
                     {&s->top_values, std::max<size_t>(m * P, 1) * 8},
                     {&s->top_present, std::max<size_t>(m * P, 1)},
                     {&s->top_nodes, c.node ? std::max<size_t>(m, 1) * sizeof(alz_node_out) : 0}});
    if (rc != ALZ_OK) return rc;
    const uint32_t* top_index = static_cast<const uint32_t*>(s->sel.top_index.p);
    if (m) {
      const uint64_t items = (uint64_t)m * (P + 3u);   // m <= n and m x P <= 2^30: fits
      trend_gather_kernel<<<(unsigned)std::min<uint64_t>((items + 255) / 256, (uint64_t)h->sms * 4), 256, 0, st>>>(
          top_index, (uint32_t)m, P, d_rec, values, present, static_cast<alz_edge_trend*>(s->top_rec.p),
          static_cast<double*>(s->top_values.p), static_cast<uint8_t*>(s->top_present.p));
      h->launches += 1;
      CK(cudaGetLastError());
      if (c.node) {
        rc = node_gather(h, top_index, (uint32_t)m, static_cast<const alz_node_out*>(nser.src_rows.p),
                         static_cast<alz_node_out*>(s->top_nodes.p));
        if (rc != ALZ_OK) return rc;
      }
    }
    res->rec = s->top_rec.p;
    res->rows = c.node ? s->top_nodes.p : s->sel.top_rows.p;
    res->index = top_index;
    res->values = static_cast<const double*>(s->top_values.p);
    res->present = static_cast<const uint8_t*>(s->top_present.p);
    res->m = m;
  } else {
    res->rec = d_rec;
    if (N && copy_out) CK(cudaMemcpyAsync(copy_out, d_rec, N * sizeof(alz_edge_trend), cudaMemcpyDeviceToHost, st));
  }
  if (!waited) CK(cudaStreamSynchronize(st));   // a full-list call's last wait: its results, the clocks, the count
  if (points && !c.given) alz_internal_ring_points(h, c.tier, c.k, points);
  if (info) {
    *info = alz_trend_info{};
    info->edges = N;
    info->rows_in = rows_in;
    info->valid = *s->h_valid;
    info->above = above;
    info->points = P;
    info->tier = c.tier;
  }
  return ALZ_OK;
}

namespace {

struct TrendCall : ScoredCall {
  bool device = false;
  alz_trend t{};
};

// The §20 pass: one trend_kernel thread per series row
struct TrendPass final : ScorePass {
  alz_trend t{};
  int launch(alz_handle* h, alz_trend_state&, const ScoredInput& in, void* rec, uint64_t* sel,
             uint32_t* valid_cnt) override {
    if (!in.n) return ALZ_OK;
    const TrendArgs ta{(uint32_t)in.n, in.points, in.values, in.present, t.stat, t.direction,
                       t.absent == ALZ_TREND_ABSENT_ZERO ? 1u : 0u, t.recent, t.min_points};
    const unsigned grid = std::min<unsigned>((unsigned)((in.n + 255) / 256), (unsigned)h->sms * 8);
    alz_edge_trend* d_rec = static_cast<alz_edge_trend*>(rec);
    if (in.keys)
      trend_kernel<<<grid, 256, 0, h->stream>>>(ta, NodeHead{in.keys}, d_rec, sel, valid_cnt);
    else
      trend_kernel<<<grid, 256, 0, h->stream>>>(ta, EdgeHead{in.rows}, d_rec, sel, valid_cnt);
    h->launches += 1;
    CK(cudaGetLastError());
    return ALZ_OK;
  }
};

bool valid_trend(const alz_trend* t, uint32_t k) {
  return t && k >= 2 && t->stat <= ALZ_TREND_ZSCORE && t->direction <= ALZ_TREND_FALLING &&
         t->absent <= ALZ_TREND_ABSENT_ZERO && t->recent >= 1 && t->recent <= k - 1;
}

// The eight entry points. A host full-list call's records are copied before its last wait; a host top call copies
// its results after the selection, with one more wait. Device calls: *dev (required) gets the device results.
int trends_entry(alz_handle* h, TrendCall c, const alz_metric* m, const alz_trend* t, void* out, void* rows,
                 double* series, uint8_t* present, size_t cap, ScoredResult* dev, size_t* n_out, uint32_t* n_points,
                 alz_rollup_info* points, alz_trend_info* info) {
  if (!h || !n_out || !n_points) {
    if (n_out) *n_out = 0;
    if (n_points) *n_points = 0;
    return ALZ_E_INVAL;
  }
  *n_out = 0;
  *n_points = 0;
  if (info) *info = alz_trend_info{};
  if (!valid_trend(t, c.k) || !valid_metrics(m, 1, &c.ms)) return ALZ_E_INVAL;
  c.t = *t;
  if (c.source != ALZ_SOURCE_WINDOW && c.source > ALZ_ROLLUP_SPAN) return ALZ_E_INVAL;
  if (c.node && c.side > ALZ_SIDE_OUT) return ALZ_E_INVAL;
  if (c.top && (c.n_top == 0 || std::isnan(c.min_value))) return ALZ_E_INVAL;
  if (c.device ? !dev : (!c.top && !out && cap)) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  ScoredResult res;
  alz_trend_info ti{};
  TrendPass pass;
  pass.t = c.t;
  const int rc = scored_series_locked(h, c.group ? h->group_trends : c.node ? h->node_trends : h->trends,
                                      c.group ? "group trends" : c.node ? "node trends" : "edge trends", c,
                                      c.device ? SIZE_MAX : cap, c.device || c.top ? nullptr : out, pass, &res,
                                      n_points, points, info ? &ti : nullptr);
  *n_out = res.m;
  if (rc != ALZ_OK) return rc;
  if (info) *info = ti;
  const size_t mm = res.m, P = *n_points;
  if (c.device) {
    *dev = res;
    return ALZ_OK;
  }
  if (!c.top) return ALZ_OK;   // the records came with the call's wait
  if (mm > cap) return ALZ_E_CAPACITY;
  cudaStream_t st = h->stream;
  const size_t row_bytes = c.node ? sizeof(alz_node_out) : sizeof(alz_edge_out);
  if (mm && out) CK(cudaMemcpyAsync(out, res.rec, mm * sizeof(alz_edge_trend), cudaMemcpyDeviceToHost, st));
  if (mm && rows) CK(cudaMemcpyAsync(rows, res.rows, mm * row_bytes, cudaMemcpyDeviceToHost, st));
  if (mm * P && series) CK(cudaMemcpyAsync(series, res.values, mm * P * 8, cudaMemcpyDeviceToHost, st));
  if (mm * P && present) CK(cudaMemcpyAsync(present, res.present, mm * P, cudaMemcpyDeviceToHost, st));
  if (mm) CK(cudaStreamSynchronize(st));
  return ALZ_OK;
}

// The device entry points: trends_entry, then its results as the caller's pointer types
template <class Rec, class Row>
int trends_device(alz_handle* h, const TrendCall& c, const alz_metric* m, const alz_trend* t, const Rec** dev_out,
                  const Row** dev_rows, const double** dev_series, const uint8_t** dev_present, size_t* n_out,
                  uint32_t* n_points, alz_rollup_info* points, alz_trend_info* info) {
  ScoredResult r;
  const int rc = trends_entry(h, c, m, t, nullptr, nullptr, nullptr, nullptr, 0, dev_out ? &r : nullptr, n_out,
                              n_points, points, info);
  if (rc != ALZ_OK) return rc;
  *dev_out = static_cast<const Rec*>(r.rec);
  if (dev_rows) *dev_rows = static_cast<const Row*>(r.rows);
  if (dev_series) *dev_series = r.values;
  if (dev_present) *dev_present = r.present;
  return ALZ_OK;
}

TrendCall call_of(bool device, bool top, uint32_t source, uint32_t tier, uint32_t k, uint32_t n_top, double min_trend) {
  TrendCall c;
  c.device = device;
  c.top = top;
  c.source = source;
  c.tier = tier;
  c.k = k;
  c.n_top = n_top;
  c.min_value = min_trend;
  return c;
}

TrendCall node_call_of(bool device, bool top, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                       uint32_t n_top, double min_trend) {
  TrendCall c = call_of(device, top, source, tier, k, n_top, min_trend);
  c.node = true;
  c.side = side;
  return c;
}

TrendCall group_call_of(bool node, bool device, bool top, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                        uint32_t n_top, double min_trend) {
  TrendCall c = node ? node_call_of(device, top, source, side, tier, k, n_top, min_trend)
                     : call_of(device, top, source, tier, k, n_top, min_trend);
  c.group = true;
  return c;
}

}  // namespace

extern "C" int alz_edge_trends(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                               const alz_trend* t, alz_edge_trend* out, size_t cap, size_t* n_out, uint32_t* n_points,
                               alz_rollup_info* points, alz_trend_info* info) {
  return trends_entry(h, call_of(false, false, source, tier, k, 0, 0.0), m, t, out, nullptr, nullptr, nullptr, cap,
                      nullptr, n_out, n_points, points, info);
}

extern "C" int alz_edge_trends_device(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                                      const alz_trend* t, const alz_edge_trend** dev_out, size_t* n_out,
                                      uint32_t* n_points, alz_rollup_info* points, alz_trend_info* info) {
  return trends_device<alz_edge_trend, alz_edge_out>(h, call_of(true, false, source, tier, k, 0, 0.0), m, t, dev_out,
                                                     nullptr, nullptr, nullptr, n_out, n_points, points, info);
}

extern "C" int alz_edge_trends_top(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                                   const alz_trend* t, uint32_t top, double min_trend, alz_edge_trend* out,
                                   alz_edge_out* rows, double* series, uint8_t* present, size_t cap, size_t* n_out,
                                   uint32_t* n_points, alz_rollup_info* points, alz_trend_info* info) {
  return trends_entry(h, call_of(false, true, source, tier, k, top, min_trend), m, t, out, rows, series, present, cap,
                      nullptr, n_out, n_points, points, info);
}

extern "C" int alz_edge_trends_top_device(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k,
                                          const alz_metric* m, const alz_trend* t, uint32_t top, double min_trend,
                                          const alz_edge_trend** dev_out, const alz_edge_out** dev_rows,
                                          const double** dev_series, const uint8_t** dev_present, size_t* n_out,
                                          uint32_t* n_points, alz_rollup_info* points, alz_trend_info* info) {
  return trends_device(h, call_of(true, true, source, tier, k, top, min_trend), m, t, dev_out, dev_rows, dev_series,
                       dev_present, n_out, n_points, points, info);
}

extern "C" int alz_node_trends(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                               const alz_metric* m, const alz_trend* t, alz_node_trend* out, size_t cap, size_t* n_out,
                               uint32_t* n_points, alz_rollup_info* points, alz_trend_info* info) {
  return trends_entry(h, node_call_of(false, false, source, side, tier, k, 0, 0.0), m, t, out, nullptr, nullptr,
                      nullptr, cap, nullptr, n_out, n_points, points, info);
}

extern "C" int alz_node_trends_device(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                      const alz_metric* m, const alz_trend* t, const alz_node_trend** dev_out,
                                      size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                                      alz_trend_info* info) {
  return trends_device<alz_node_trend, alz_node_out>(h, node_call_of(true, false, source, side, tier, k, 0, 0.0), m,
                                                     t, dev_out, nullptr, nullptr, nullptr, n_out, n_points, points,
                                                     info);
}

extern "C" int alz_node_trends_top(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                   const alz_metric* m, const alz_trend* t, uint32_t top, double min_trend,
                                   alz_node_trend* out, alz_node_out* nodes, double* series, uint8_t* present,
                                   size_t cap, size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                                   alz_trend_info* info) {
  return trends_entry(h, node_call_of(false, true, source, side, tier, k, top, min_trend), m, t, out, nodes, series,
                      present, cap, nullptr, n_out, n_points, points, info);
}

extern "C" int alz_node_trends_top_device(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                          const alz_metric* m, const alz_trend* t, uint32_t top, double min_trend,
                                          const alz_node_trend** dev_out, const alz_node_out** dev_nodes,
                                          const double** dev_series, const uint8_t** dev_present, size_t* n_out,
                                          uint32_t* n_points, alz_rollup_info* points, alz_trend_info* info) {
  return trends_device(h, node_call_of(true, true, source, side, tier, k, top, min_trend), m, t, dev_out, dev_nodes,
                       dev_series, dev_present, n_out, n_points, points, info);
}

extern "C" int alz_group_edge_trends(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                                     const alz_trend* t, alz_edge_trend* out, size_t cap, size_t* n_out,
                                     uint32_t* n_points, alz_rollup_info* points, alz_trend_info* info) {
  return trends_entry(h, group_call_of(false, false, false, source, 0, tier, k, 0, 0.0), m, t, out, nullptr, nullptr,
                      nullptr, cap, nullptr, n_out, n_points, points, info);
}

extern "C" int alz_group_edge_trends_device(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k,
                                            const alz_metric* m, const alz_trend* t, const alz_edge_trend** dev_out,
                                            size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                                            alz_trend_info* info) {
  return trends_device<alz_edge_trend, alz_edge_out>(h, group_call_of(false, true, false, source, 0, tier, k, 0, 0.0),
                                                     m, t, dev_out, nullptr, nullptr, nullptr, n_out, n_points, points,
                                                     info);
}

extern "C" int alz_group_edge_trends_top(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k,
                                         const alz_metric* m, const alz_trend* t, uint32_t top, double min_trend,
                                         alz_edge_trend* out, alz_edge_out* rows, double* series, uint8_t* present,
                                         size_t cap, size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                                         alz_trend_info* info) {
  return trends_entry(h, group_call_of(false, false, true, source, 0, tier, k, top, min_trend), m, t, out, rows,
                      series, present, cap, nullptr, n_out, n_points, points, info);
}

extern "C" int alz_group_edge_trends_top_device(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k,
                                                const alz_metric* m, const alz_trend* t, uint32_t top,
                                                double min_trend, const alz_edge_trend** dev_out,
                                                const alz_edge_out** dev_rows, const double** dev_series,
                                                const uint8_t** dev_present, size_t* n_out, uint32_t* n_points,
                                                alz_rollup_info* points, alz_trend_info* info) {
  return trends_device(h, group_call_of(false, true, true, source, 0, tier, k, top, min_trend), m, t, dev_out,
                       dev_rows, dev_series, dev_present, n_out, n_points, points, info);
}

extern "C" int alz_group_node_trends(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                     const alz_metric* m, const alz_trend* t, alz_node_trend* out, size_t cap,
                                     size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                                     alz_trend_info* info) {
  return trends_entry(h, group_call_of(true, false, false, source, side, tier, k, 0, 0.0), m, t, out, nullptr,
                      nullptr, nullptr, cap, nullptr, n_out, n_points, points, info);
}

extern "C" int alz_group_node_trends_device(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                            const alz_metric* m, const alz_trend* t, const alz_node_trend** dev_out,
                                            size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                                            alz_trend_info* info) {
  return trends_device<alz_node_trend, alz_node_out>(
      h, group_call_of(true, true, false, source, side, tier, k, 0, 0.0), m, t, dev_out, nullptr, nullptr, nullptr,
      n_out, n_points, points, info);
}

extern "C" int alz_group_node_trends_top(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                         const alz_metric* m, const alz_trend* t, uint32_t top, double min_trend,
                                         alz_node_trend* out, alz_node_out* nodes, double* series, uint8_t* present,
                                         size_t cap, size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                                         alz_trend_info* info) {
  return trends_entry(h, group_call_of(true, false, true, source, side, tier, k, top, min_trend), m, t, out, nodes,
                      series, present, cap, nullptr, n_out, n_points, points, info);
}

extern "C" int alz_group_node_trends_top_device(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier,
                                                uint32_t k, const alz_metric* m, const alz_trend* t, uint32_t top,
                                                double min_trend, const alz_node_trend** dev_out,
                                                const alz_node_out** dev_nodes, const double** dev_series,
                                                const uint8_t** dev_present, size_t* n_out, uint32_t* n_points,
                                                alz_rollup_info* points, alz_trend_info* info) {
  return trends_device(h, group_call_of(true, true, true, source, side, tier, k, top, min_trend), m, t, dev_out,
                       dev_nodes, dev_series, dev_present, n_out, n_points, points, info);
}
