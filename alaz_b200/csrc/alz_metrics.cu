// alz_metrics.cu — edge metrics on the device (docs/SPEC.md §17): per-row counts, 5xx, 5xx rate, mean latency and
// histogram quantiles of a window or a rollup, and the top rows by one of them (the selection of alz_top.cu on the
// 64-bit keys of the float64 values). Reads the source rows only; touches no GNN state.
//
//   metrics  with a quantile: a warp per row, lane l owns buckets 2l and 2l+1 (one 8-byte load), one inclusive scan
//            of the counts serves every quantile of the row; without one: a thread per row, which reads the row's
//            three 8-byte sums and not its histogram
//   top      the metrics kernel with one metric writes the row's 8-byte value, and the selection ranks its bits
//
// Every value is bit for bit what the host computes (alz_edge_quantiles, SPEC §5), which rounds each operation on its
// own. nvcc would contract q * total and lo + f * (hi - lo) into fused multiply-adds, so the quantile arithmetic is
// written with the round-to-nearest intrinsics.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <mutex>
#include <string>

#include "alz_metrics.cuh"
#include "alz_top.cuh"

using namespace alz;
using namespace alz::metrics;

namespace {

// docs/SPEC.md §4/§5 bucket bounds, float64 (exact)
__device__ __forceinline__ double bucket_lo(uint32_t b) {
  if (b == 0) return 0.0;
  const double base = (double)(1ull << (8 + b / 2));
  return (b & 1u) ? base * 1.5 : base;
}
__device__ __forceinline__ double bucket_hi(uint32_t b) { return b == ALZ_NB - 1 ? (double)(1ull << 40) : bucket_lo(b + 1); }

__device__ __forceinline__ double scalar_metric(uint32_t kind, uint64_t count, uint64_t err, uint64_t lat) {
  switch (kind) {
    case ALZ_METRIC_COUNT: return (double)count;
    case ALZ_METRIC_ERR5XX: return (double)err;
    case ALZ_METRIC_ERR_RATE: return count ? (double)err / (double)count : 0.0;
    default: return count ? (double)lat / (double)count : 0.0;   // ALZ_METRIC_MEAN_NS
  }
}

// Output row i reads the row rows(i). With RowOf::kMayBeAbsent, rows(i) may be null: every value of output row i is
// +0.0, and rows.mark(i, present) records which it was.
struct PlainRows {
  static constexpr bool kMayBeAbsent = false;
  const alz_edge_out* e;
  __device__ __forceinline__ const alz_edge_out* operator()(uint32_t i) const { return e + i; }
};

// a thread per row: the three sums only
template <class RowOf>
__global__ void __launch_bounds__(256) edge_metrics_sums_kernel(const RowOf rows, uint32_t n, MetricSet ms,
                                                                double* __restrict__ out) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const alz_edge_out* __restrict__ r = rows(i);
    if constexpr (RowOf::kMayBeAbsent) {
      rows.mark(i, r != nullptr);
      if (!r) {
#pragma unroll
        for (uint32_t j = 0; j < ALZ_MAX_METRICS; ++j)
          if (j < ms.nm) out[(size_t)i * ms.nm + j] = 0.0;
        continue;
      }
    }
    const uint64_t count = r->count, err = r->err5xx, lat = r->lat_sum_ns;
#pragma unroll
    for (uint32_t j = 0; j < ALZ_MAX_METRICS; ++j)   // unrolled: ms stays in the parameter space, no local copy
      if (j < ms.nm) out[(size_t)i * ms.nm + j] = scalar_metric(ms.kind[j], count, err, lat);
  }
}

// a warp per row: one read of the histogram for every metric of the row; lane j < nm writes metric j
template <class RowOf>
__global__ void __launch_bounds__(256) edge_metrics_hist_kernel(const RowOf rows, uint32_t n, MetricSet ms,
                                                                double* __restrict__ out) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t warps_per_grid = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps_per_grid) {
    const alz_edge_out* __restrict__ r = rows(i);
    if constexpr (RowOf::kMayBeAbsent) {   // the same row in every lane: the warp stays converged
      if (lane == 0) rows.mark(i, r != nullptr);
      if (!r) {
        if (lane < ms.nm) out[(size_t)i * ms.nm + lane] = 0.0;
        continue;
      }
    }
    const uint2 cc = *reinterpret_cast<const uint2*>(&r->hist[2 * lane]);
    const uint64_t c0 = cc.x, c1 = cc.y;
    uint64_t incl = c0 + c1;                      // integer sums: exact, as the host's float64 sums of the cells are
    for (int o = 1; o < 32; o <<= 1) {
      const uint64_t t = __shfl_up_sync(0xFFFFFFFFu, (unsigned long long)incl, o);
      if ((int)lane >= o) incl += t;
    }
    const uint64_t total = __shfl_sync(0xFFFFFFFFu, (unsigned long long)incl, 31);
    const uint64_t before = incl - (c0 + c1);
    const uint64_t count = r->count, err = r->err5xx, lat = r->lat_sum_ns;
    double mine = 0.0;
#pragma unroll
    for (uint32_t j = 0; j < ALZ_MAX_METRICS; ++j) {   // unrolled: ms stays in the parameter space, no local copy
      if (j >= ms.nm) break;                            // ms is the same in every lane: the warp stays converged
      double v;
      if (ms.kind[j] == ALZ_METRIC_QUANTILE) {
        // the first bucket with c > 0 and cum + c >= target, interpolated as alz_edge_quantiles does
        const double target = __dmul_rn(ms.q[j], (double)total);
        const bool h0 = c0 > 0 && (double)(before + c0) >= target;
        const bool h1 = c1 > 0 && (double)(before + c0 + c1) >= target;
        const uint32_t m = __ballot_sync(0xFFFFFFFFu, h0 || h1);
        double val = total ? bucket_hi(ALZ_NB - 1) : 0.0;
        const int owner = m ? __ffs(m) - 1 : 0;
        if (m && (int)lane == owner) {
          const uint32_t b = h0 ? 2u * lane : 2u * lane + 1u;
          const double cum = (double)(h0 ? before : before + c0);
          const double cb = (double)(h0 ? c0 : c1);
          double f = __ddiv_rn(__dsub_rn(target, cum), cb);
          if (f < 0.0) f = 0.0;
          const double lo = bucket_lo(b), hi = bucket_hi(b);
          val = __dadd_rn(lo, __dmul_rn(f, __dsub_rn(hi, lo)));
        }
        v = __shfl_sync(0xFFFFFFFFu, val, owner);
      } else {
        v = scalar_metric(ms.kind[j], count, err, lat);
      }
      if (lane == j) mine = v;
    }
    if (lane < ms.nm) out[(size_t)i * ms.nm + lane] = mine;
  }
}

}  // namespace

// Buffers of the metric calls, each grown on demand and never shrunk; freed in alz_destroy
struct alz_metrics_state {
  DevBuf values;                 // rows x nm float64 values
  Selection sel;                 // the top call's selection and results
};

void alz_internal_free_metrics(alz_handle* h) {
  alz_metrics_state* s = h->metrics;
  if (!s) return;
  free_bufs({&s->values});
  s->sel.free();
  delete s;
  h->metrics = nullptr;
}

namespace alz {
namespace metrics {

void free_bufs(std::initializer_list<DevBuf*> bufs) {
  for (DevBuf* b : bufs) {
    cudaFree(b->p);
    *b = DevBuf{};
  }
}

void Selection::free() {
  free_bufs({&words, &tile_cnt, &cand_key, &cand_idx, &sorted_key, &sorted_idx, &tmp, &top_rows, &top_values,
             &top_index});
}

int reserve(alz_handle* h, std::initializer_list<std::pair<DevBuf*, size_t>> need) {
  bool waited = false;
  for (const auto& [b, bytes] : need) {
    if (bytes <= b->bytes) continue;
    if (!waited) { CK(cudaStreamSynchronize(h->stream)); waited = true; }
    cudaFree(b->p);
    b->p = nullptr;
    b->bytes = 0;
    if (cudaMalloc(&b->p, bytes) != cudaSuccess) {
      b->p = nullptr;
      h->last_err = std::string("edge metrics: ") + cudaGetErrorString(cudaGetLastError());
      return ALZ_E_NOMEM;
    }
    b->bytes = bytes;
  }
  return ALZ_OK;
}

bool valid_metrics(const alz_metric* m, uint32_t nm, MetricSet* ms) {
  if (!m || nm == 0 || nm > ALZ_MAX_METRICS) return false;
  *ms = MetricSet{};
  ms->nm = nm;
  for (uint32_t j = 0; j < nm; ++j) {
    if (m[j].kind > ALZ_METRIC_QUANTILE) return false;
    if (m[j].kind == ALZ_METRIC_QUANTILE && !(m[j].q >= 0.0 && m[j].q <= 1.0)) return false;   // NaN fails too
    ms->kind[j] = m[j].kind;
    ms->q[j] = m[j].kind == ALZ_METRIC_QUANTILE ? m[j].q : 0.0;
  }
  return true;
}

}  // namespace metrics
}  // namespace alz

namespace {

template <class RowOf>
int launch_metrics(alz_handle* h, const RowOf& rows, uint32_t n, const MetricSet& ms, double* out) {
  if (n == 0) return ALZ_OK;
  bool quant = false;
  for (uint32_t j = 0; j < ms.nm; ++j) quant |= ms.kind[j] == ALZ_METRIC_QUANTILE;
  if (quant) {
    const unsigned grid = std::min<unsigned>((n + 7) / 8, (unsigned)h->sms * 8);
    edge_metrics_hist_kernel<<<grid, 256, 0, h->stream>>>(rows, n, ms, out);
  } else {
    const unsigned grid = std::min<unsigned>((n + 255) / 256, (unsigned)h->sms * 8);
    edge_metrics_sums_kernel<<<grid, 256, 0, h->stream>>>(rows, n, ms, out);
  }
  h->launches += 1;
  CK(cudaGetLastError());
  return ALZ_OK;
}

}  // namespace

namespace alz {
namespace metrics {

int run_metrics(alz_handle* h, const alz_edge_out* rows, uint32_t n, const MetricSet& ms, double* out) {
  return launch_metrics(h, PlainRows{rows}, n, ms, out);
}

int run_metrics_series(alz_handle* h, const SeriesRows& rows, uint32_t n, const MetricSet& ms, double* out) {
  return launch_metrics(h, rows, n, ms, out);
}

int run_metrics_nodes(alz_handle* h, const NodeRows& rows, uint32_t n, const MetricSet& ms, double* out) {
  return launch_metrics(h, rows, n, ms, out);
}

int run_metrics_node_series(alz_handle* h, const NodeSeriesRows& rows, uint32_t n, const MetricSet& ms, double* out) {
  return launch_metrics(h, rows, n, ms, out);
}

int select_top(alz_handle* h, Selection& s, const uint64_t* vals, uint32_t n, uint32_t k, double min_value,
               const alz_edge_out* rows, size_t* m_out, uint64_t* above) {
  *m_out = 0;
  *above = 0;
  if (n == 0) return ALZ_OK;
  const uint32_t m_max = std::min(n, k);
  int rc = reserve(h, {{&s.words, top::kWordsBytes},
                       {&s.tile_cnt, (size_t)top::tiles(n) * 8},
                       {&s.cand_key, (size_t)m_max * 8},
                       {&s.cand_idx, (size_t)m_max * 4},
                       {&s.sorted_key, (size_t)m_max * 8},
                       {&s.sorted_idx, (size_t)m_max * 4},
                       {&s.tmp, top::tmp_bytes<uint64_t>(n, m_max)}});
  if (rc != ALZ_OK) return rc;
  const top::Scratch sc{static_cast<uint32_t*>(s.words.p), static_cast<uint64_t*>(s.tile_cnt.p), s.cand_key.p,
                        static_cast<uint32_t*>(s.cand_idx.p), s.sorted_key.p, static_cast<uint32_t*>(s.sorted_idx.p),
                        s.tmp.p, s.tmp.bytes};
  uint64_t min_bits;
  memcpy(&min_bits, &min_value, 8);
  top::Ctl<uint64_t> c;
  rc = top::select_candidates<uint64_t>(h, vals, n, k, min_bits, sc, &c);
  if (rc != ALZ_OK) return rc;
  *above = c.above;
  if (c.m == 0) return ALZ_OK;
  rc = reserve(h, {{&s.top_rows, rows ? (size_t)c.m * sizeof(alz_edge_out) : 0}, {&s.top_values, (size_t)c.m * 8},
                   {&s.top_index, (size_t)c.m * 4}});
  if (rc != ALZ_OK) return rc;
  rc = top::select_results<uint64_t>(h, vals, n, c, rows, sc, static_cast<uint32_t*>(s.top_index.p),
                                     static_cast<uint64_t*>(s.top_values.p),
                                     rows ? static_cast<alz_edge_out*>(s.top_rows.p) : nullptr);
  if (rc != ALZ_OK) return rc;
  *m_out = c.m;
  return ALZ_OK;
}

}  // namespace metrics
}  // namespace alz

namespace {

// allocated on first use; its buffers start empty
void metrics_state(alz_handle* h) {
  if (!h->metrics) h->metrics = new alz_metrics_state();
}

// the rows of the last flushed window (rollup false) or of the last rollup of `kind`; caller holds h->mu
int source_rows(alz_handle* h, bool rollup, uint32_t kind, const alz_edge_out** rows, size_t* n) {
  *rows = h->d_out;
  *n = h->last_n_edges;
  if (rollup) return alz_internal_rollup_rows(h, kind, rows, n);
  return ALZ_OK;
}

// the metrics of n rows into the values buffer, on the stream; no wait
int run_metrics_values(alz_handle* h, const alz_edge_out* rows, uint32_t n, const MetricSet& ms) {
  alz_metrics_state* s = h->metrics;
  const int rc = reserve(h, {{&s->values, std::max<size_t>((size_t)n * ms.nm, 1) * 8}});
  if (rc != ALZ_OK) return rc;
  return run_metrics(h, rows, n, ms, static_cast<double*>(s->values.p));
}

// The metrics of a source or of caller rows (dev_rows, n). Device variant: values null, *dev set. Host variant:
// cap rows in values, one wait. Caller holds h->mu.
int metrics_call(alz_handle* h, const alz_edge_out* rows, size_t n, const MetricSet& ms, double* values, size_t cap,
                 const double** dev, size_t* n_out) {
  if (n > kMaxRows) return ALZ_E_CAPACITY;
  *n_out = n;
  if (!dev && n > cap) return ALZ_E_CAPACITY;
  metrics_state(h);
  const int rc = run_metrics_values(h, rows, (uint32_t)n, ms);
  if (rc != ALZ_OK) { *n_out = 0; return rc; }
  if (dev) {
    *dev = static_cast<const double*>(h->metrics->values.p);
    return ALZ_OK;
  }
  if (n) CK(cudaMemcpyAsync(values, h->metrics->values.p, n * ms.nm * 8, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return ALZ_OK;
}

int metrics_entry(alz_handle* h, bool rollup, uint32_t kind, const alz_metric* m, uint32_t nm, double* values,
                  size_t cap, const double** dev, size_t* n_out) {
  if (!h || !n_out) return ALZ_E_INVAL;
  *n_out = 0;
  MetricSet ms;
  if (!valid_metrics(m, nm, &ms) || (!dev && !values && cap)) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  const alz_edge_out* rows = nullptr;
  size_t n = 0;
  const int rc = source_rows(h, rollup, kind, &rows, &n);
  if (rc != ALZ_OK) return rc;
  return metrics_call(h, rows, n, ms, values, cap, dev, n_out);
}

// The top call over a source: the one metric's values, then the selection. Caller holds h->mu; *n_out = results.
int top_call(alz_handle* h, bool rollup, uint32_t kind, const alz_metric* m, uint32_t k, double min_value,
             size_t* n_out, alz_top_info* info) {
  MetricSet ms;
  if (k == 0 || std::isnan(min_value) || !valid_metrics(m, 1, &ms)) return ALZ_E_INVAL;
  CK(cudaSetDevice(h->device));
  const alz_edge_out* rows = nullptr;
  size_t n = 0;
  int rc = source_rows(h, rollup, kind, &rows, &n);
  if (rc != ALZ_OK) return rc;
  if (n > kMaxRows) return ALZ_E_CAPACITY;
  metrics_state(h);
  rc = run_metrics_values(h, rows, (uint32_t)n, ms);
  if (rc != ALZ_OK) return rc;
  uint64_t above = 0;
  rc = select_top(h, h->metrics->sel, static_cast<const uint64_t*>(h->metrics->values.p), (uint32_t)n, k, min_value,
                  rows, n_out, &above);
  if (rc != ALZ_OK) return rc;
  if (info) { info->scored = n; info->above = above; }
  return ALZ_OK;
}

int top_entry(alz_handle* h, bool rollup, uint32_t kind, const alz_metric* m, uint32_t k, double min_value,
              alz_edge_out* rows, double* values, uint32_t* index, size_t cap, const alz_edge_out** dev_rows,
              const double** dev_values, const uint32_t** dev_index, bool device, size_t* n_out, alz_top_info* info) {
  if (!h || !n_out) return ALZ_E_INVAL;
  *n_out = 0;
  if (info) *info = alz_top_info{};
  std::lock_guard<std::mutex> g(h->mu);
  const int rc = top_call(h, rollup, kind, m, k, min_value, n_out, info);
  if (rc != ALZ_OK) { *n_out = 0; return rc; }
  const Selection& s = h->metrics->sel;
  if (device) {
    if (dev_rows) *dev_rows = static_cast<const alz_edge_out*>(s.top_rows.p);
    if (dev_values) *dev_values = static_cast<const double*>(s.top_values.p);
    if (dev_index) *dev_index = static_cast<const uint32_t*>(s.top_index.p);
    return ALZ_OK;
  }
  const size_t n = *n_out;
  if (n > cap) return ALZ_E_CAPACITY;
  cudaStream_t st = h->stream;
  if (n && rows) CK(cudaMemcpyAsync(rows, s.top_rows.p, n * sizeof(alz_edge_out), cudaMemcpyDeviceToHost, st));
  if (n && values) CK(cudaMemcpyAsync(values, s.top_values.p, n * 8, cudaMemcpyDeviceToHost, st));
  if (n && index) CK(cudaMemcpyAsync(index, s.top_index.p, n * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return ALZ_OK;
}

}  // namespace

extern "C" int alz_edge_metrics(alz_handle* h, const alz_metric* m, uint32_t nm, double* values, size_t cap,
                                size_t* n_out) {
  return metrics_entry(h, false, 0, m, nm, values, cap, nullptr, n_out);
}

extern "C" int alz_edge_metrics_device(alz_handle* h, const alz_metric* m, uint32_t nm, const double** dev_values,
                                       size_t* n_out) {
  if (!dev_values) return n_out ? (*n_out = 0, ALZ_E_INVAL) : ALZ_E_INVAL;
  return metrics_entry(h, false, 0, m, nm, nullptr, 0, dev_values, n_out);
}

extern "C" int alz_edge_metrics_rollup(alz_handle* h, uint32_t kind, const alz_metric* m, uint32_t nm, double* values,
                                       size_t cap, size_t* n_out) {
  return metrics_entry(h, true, kind, m, nm, values, cap, nullptr, n_out);
}

extern "C" int alz_edge_metrics_rollup_device(alz_handle* h, uint32_t kind, const alz_metric* m, uint32_t nm,
                                              const double** dev_values, size_t* n_out) {
  if (!dev_values) return n_out ? (*n_out = 0, ALZ_E_INVAL) : ALZ_E_INVAL;
  return metrics_entry(h, true, kind, m, nm, nullptr, 0, dev_values, n_out);
}

extern "C" int alz_edge_top(alz_handle* h, const alz_metric* m, uint32_t k, double min_value, alz_edge_out* rows,
                            double* values, uint32_t* index, size_t cap, size_t* n_out, alz_top_info* info) {
  return top_entry(h, false, 0, m, k, min_value, rows, values, index, cap, nullptr, nullptr, nullptr, false, n_out,
                   info);
}

extern "C" int alz_edge_top_device(alz_handle* h, const alz_metric* m, uint32_t k, double min_value,
                                   const alz_edge_out** dev_rows, const double** dev_values,
                                   const uint32_t** dev_index, size_t* n_out, alz_top_info* info) {
  return top_entry(h, false, 0, m, k, min_value, nullptr, nullptr, nullptr, 0, dev_rows, dev_values, dev_index, true,
                   n_out, info);
}

extern "C" int alz_edge_top_rollup(alz_handle* h, uint32_t kind, const alz_metric* m, uint32_t k, double min_value,
                                   alz_edge_out* rows, double* values, uint32_t* index, size_t cap, size_t* n_out,
                                   alz_top_info* info) {
  return top_entry(h, true, kind, m, k, min_value, rows, values, index, cap, nullptr, nullptr, nullptr, false, n_out,
                   info);
}

extern "C" int alz_edge_top_rollup_device(alz_handle* h, uint32_t kind, const alz_metric* m, uint32_t k,
                                          double min_value, const alz_edge_out** dev_rows, const double** dev_values,
                                          const uint32_t** dev_index, size_t* n_out, alz_top_info* info) {
  return top_entry(h, true, kind, m, k, min_value, nullptr, nullptr, nullptr, 0, dev_rows, dev_values, dev_index, true,
                   n_out, info);
}

extern "C" int alz_debug_edge_metrics_rows(alz_handle* h, const alz_edge_out* dev_rows, size_t n, const alz_metric* m,
                                           uint32_t nm, double* values, size_t cap, size_t* n_out) {
  if (!h || !n_out) return ALZ_E_INVAL;
  *n_out = 0;
  MetricSet ms;
  if (!valid_metrics(m, nm, &ms) || (!dev_rows && n) || (!values && cap)) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  return metrics_call(h, dev_rows, n, ms, values, cap, nullptr, n_out);
}

extern "C" int alz_debug_top_keys64(alz_handle* h, const double* dev_values, size_t n, uint32_t k, double min_value,
                                    uint32_t* index, size_t cap, size_t* n_out, uint64_t* above) {
  if (!h || !n_out || (!dev_values && n)) return ALZ_E_INVAL;
  *n_out = 0;
  if (above) *above = 0;
  if (k == 0 || std::isnan(min_value)) return ALZ_E_INVAL;
  if (n > kMaxRows) return ALZ_E_CAPACITY;
  std::lock_guard<std::mutex> g(h->mu);
  CK(cudaSetDevice(h->device));
  metrics_state(h);
  uint64_t ab = 0;
  const int rc = select_top(h, h->metrics->sel, reinterpret_cast<const uint64_t*>(dev_values), (uint32_t)n, k, min_value,
                            nullptr, n_out, &ab);
  if (rc != ALZ_OK) { *n_out = 0; return rc; }
  if (above) *above = ab;
  if (*n_out > cap) return ALZ_E_CAPACITY;
  if (*n_out && index)
    CK(cudaMemcpyAsync(index, h->metrics->sel.top_index.p, *n_out * 4, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return ALZ_OK;
}
