// alz_corr.cu — correlations (docs/SPEC.md §29): how closely each series row of a source followed a target series the
// caller supplies, at the best lag, and the top rows by it with their series. The rows are a source's edges (§19
// series), nodes (§22) or group edges and group nodes (§26).
//
//   skeleton  scored_series_locked (alz_trends.cu), which the trends share: the level's series path into the
//             correlation state's own buffers (so a correlation call leaves the series and trend device results
//             alone), this file's pass, then for a top call the §17 selection and trend_gather_kernel over the 48-byte
//             records
//   target    checked on the host (n = P, the ring's newest window_last, finite values within 2^64), then staged
//             through pinned memory with absent points as +0.0 and presence as 0 / 1
//   corr      one block of kRows threads per kRows series rows, one thread per row. A row-major tile of rows over
//             kTile points is staged in shared memory, transposed with a padded pitch so the threads' reads do not
//             conflict: when a tile is whole rows it is one contiguous span of values and of presence bytes, read with
//             16-byte loads; otherwise each row's run is read with consecutive 8-byte loads. The tile of the target
//             (the points the tile's pairs reach at every lag up to max_lag) comes with it. Each thread then walks its
//             row for every lag: pass 1 the sums of the used pairs, pass 2 Sxx, Syy and Sxy about the means, in
//             ascending j and with the round-to-nearest intrinsics (no contraction), carrying the sums across tiles.
//             A row of at most kTile points is loaded once per block; a longer one once per tile, lag and pass.
//             Writes the record and, for a top call, the selection value (the score's bits when valid, all ones
//             otherwise); a warp-reduced count of the valid rows goes to a pinned word.
// Waits: as trends (a full-list call once at its end, a top call adds the selection's wait); the target's checks read
// host records only.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "alz_metrics.cuh"

using namespace alz;
using namespace alz::metrics;

static_assert(sizeof(alz_edge_corr) == sizeof(alz_edge_trend), "a correlation record is gathered as a trend record");
static_assert(sizeof(alz_corr) == 16 && sizeof(alz_corr_target) == 32 && sizeof(alz_corr_info) == 48,
              "alz_corr, alz_corr_target and alz_corr_info sizes");
static_assert(offsetof(alz_edge_corr, valid) == offsetof(alz_edge_trend, valid) &&
                  offsetof(alz_edge_corr, lag) == 3 && offsetof(alz_edge_corr, index) == offsetof(alz_edge_trend, index) &&
                  offsetof(alz_edge_corr, used) == offsetof(alz_edge_trend, used) &&
                  offsetof(alz_edge_corr, r) == 24 && offsetof(alz_edge_corr, score) == 32 &&
                  offsetof(alz_edge_corr, r0) == 40,
              "alz_edge_corr's head is laid out as alz_edge_trend's (EdgeHead writes its first 16 bytes)");
static_assert(sizeof(alz_node_corr) == sizeof(alz_edge_corr) &&
                  offsetof(alz_node_corr, valid) == offsetof(alz_edge_corr, valid) &&
                  offsetof(alz_node_corr, lag) == offsetof(alz_edge_corr, lag) &&
                  offsetof(alz_node_corr, value) == offsetof(alz_edge_corr, from) &&
                  offsetof(alz_node_corr, index) == offsetof(alz_edge_corr, index) &&
                  offsetof(alz_node_corr, r0) == offsetof(alz_edge_corr, r0),
              "from `valid` on, alz_node_corr is laid out as alz_edge_corr (NodeHead writes the first 16 bytes)");

namespace {

constexpr uint64_t kInvalidValue = ~0ull;   // a negative NaN: key 0, below every non-NaN min_score
constexpr uint32_t kRows = 64;              // series rows per block, one per thread
constexpr uint32_t kTile = 64;              // points per tile
constexpr uint32_t kPitch = kRows + 1;      // the value tile's pitch in doubles: thread r reads bank pair r + c

struct CorrArgs {
  uint32_t n, points;
  const double* values;      // values[i * points + j]
  const uint8_t* present;    // present[i * points + j]
  const double* y;           // the target, absent points +0.0
  const uint8_t* yp;         // its presence, 0 / 1
  uint32_t direction, zero, max_lag, min_points;
};

// The first 16 bytes of a record of caller series (the hook): zero but `valid`
struct BareHead {
  __device__ __forceinline__ uint4 operator()(uint32_t, bool ok) const {
    return make_uint4((ok ? 1u : 0u) << 16, 0u, 0u, 0u);
  }
};

// The dynamic shared memory of a launch: the value tile (w x kPitch doubles), the target tile (tw doubles), the
// presence tile (w x kRows bytes), the target's presence (tw bytes)
struct Smem {
  double* x;
  double* y;
  uint8_t* xp;
  uint8_t* yp;
};
__host__ __device__ inline size_t smem_bytes(uint32_t w, uint32_t tw) {
  return ((size_t)w * kPitch + tw) * 8 + (size_t)w * kRows + tw;
}

// Tile t of the block's rows [row0, row0 + rows) and of the target into shared memory; every thread calls it
__device__ void load_tile(const CorrArgs& a, const Smem& s, uint32_t row0, uint32_t rows, uint32_t t) {
  const uint32_t P = a.points, a0 = t * kTile, w = min(kTile, P - a0);
  const uint32_t tid = threadIdx.x;
  __syncthreads();   // every thread is done with the last tile
  // presence first: the values read it to write an absent point as +0.0
  if (w == P) {   // whole rows: one contiguous span of rows x P <= kRows x kTile bytes
    const uint32_t cnt = rows * P;
    const uint8_t* g = a.present + (size_t)row0 * P;
    const uint32_t head = min((16u - (uint32_t)((uintptr_t)g & 15u)) & 15u, cnt);
    const uint32_t vecs = (cnt - head) / 16;
    auto put = [&](uint32_t e, uint32_t b) {
      const uint32_t r = e / P, c = e - r * P;
      s.xp[c * kRows + r] = b != 0;
    };
    if (tid < head) put(tid, g[tid]);
    for (uint32_t q = tid; q < vecs; q += kRows) {
      const uint4 v = *reinterpret_cast<const uint4*>(g + head + q * 16);
      const uint32_t wd[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (uint32_t b = 0; b < 16; ++b) put(head + q * 16 + b, (wd[b >> 2] >> ((b & 3u) * 8)) & 0xFFu);
    }
    for (uint32_t e = head + vecs * 16 + tid; e < cnt; e += kRows) put(e, g[e]);
  } else {
    for (uint32_t e = tid; e < rows * w; e += kRows) {
      const uint32_t r = e / w, c = e - r * w;
      s.xp[c * kRows + r] = a.present[(size_t)(row0 + r) * P + a0 + c] != 0;
    }
  }
  const uint32_t tw = min(w + a.max_lag, P - a0);
  for (uint32_t e = tid; e < tw; e += kRows) {
    s.y[e] = a.y[a0 + e];
    s.yp[e] = a.yp[a0 + e];
  }
  __syncthreads();
  if (w == P) {   // the values: one contiguous span of rows x P doubles, 16-byte loads from the first aligned one
    const uint32_t cnt = rows * P;
    const double* g = a.values + (size_t)row0 * P;
    const uint32_t head = min(((uintptr_t)g & 15u) ? 1u : 0u, cnt);
    const uint32_t pairs = (cnt - head) / 2;
    auto put = [&](uint32_t e, double v) {
      const uint32_t r = e / P, c = e - r * P;
      s.x[c * kPitch + r] = s.xp[c * kRows + r] ? v : 0.0;
    };
    if (tid < head) put(0, g[0]);
    for (uint32_t q = tid; q < pairs; q += kRows) {
      const double2 v = *reinterpret_cast<const double2*>(g + head + 2 * q);
      put(head + 2 * q, v.x);
      put(head + 2 * q + 1, v.y);
    }
    if (tid == 0 && head + 2 * pairs < cnt) put(cnt - 1, g[cnt - 1]);
  } else {
    for (uint32_t e = tid; e < rows * w; e += kRows) {
      const uint32_t r = e / w, c = e - r * w;
      const double v = a.values[(size_t)(row0 + r) * P + a0 + c];
      s.x[c * kPitch + r] = s.xp[c * kRows + r] ? v : 0.0;
    }
  }
  __syncthreads();
}

// Block b: series rows [b * kRows, +kRows), thread r row b * kRows + r. rec[i] its record; with sel, sel[i] its
// selection value; *valid_cnt += the valid rows.
template <class Head>
__global__ void __launch_bounds__(kRows) corr_kernel(const __grid_constant__ CorrArgs a, const Head head,
                                                     alz_edge_corr* __restrict__ rec, uint64_t* __restrict__ sel,
                                                     uint32_t* __restrict__ valid_cnt) {
  extern __shared__ __align__(16) unsigned char smem[];
  const uint32_t P = a.points, w = min(kTile, P), tw = min(w + a.max_lag, P);
  const Smem s{reinterpret_cast<double*>(smem), reinterpret_cast<double*>(smem) + (size_t)w * kPitch,
               smem + ((size_t)w * kPitch + tw) * 8, smem + ((size_t)w * kPitch + tw) * 8 + (size_t)w * kRows};
  const uint32_t row0 = blockIdx.x * kRows, rows = min(kRows, a.n - row0);
  const uint32_t r = threadIdx.x, i = row0 + r;
  const bool mine = r < rows;
  int resident = -1;   // the tile in shared memory (block-uniform)
  bool valid = false;
  uint32_t best_lag = 0, best_used = 0, used0 = 0;
  double best_r = 0.0, best_score = 0.0, r0 = 0.0;
  for (uint32_t L = 0; L <= a.max_lag; ++L) {
    const uint32_t A = P > L ? P - L : 0u;   // pairs (x[j - L], y[j]) for j in [L, P): x index a in [0, A)
    double sx = 0.0, sy = 0.0;
    uint32_t u = 0;
    for (uint32_t t = 0; t * kTile < A; ++t) {   // pass 1: the sums of the used pairs
      if ((int)t != resident) {
        load_tile(a, s, row0, rows, t);
        resident = (int)t;
      }
      const uint32_t cw = min(kTile, A - t * kTile);
      if (mine) {
        for (uint32_t c = 0; c < cw; ++c) {
          if (!(a.zero || (s.xp[c * kRows + r] & s.yp[c + L]))) continue;
          sx = __dadd_rn(sx, s.x[c * kPitch + r]);
          sy = __dadd_rn(sy, s.y[c + L]);
          ++u;
        }
      }
    }
    const double mx = u ? __ddiv_rn(sx, (double)u) : 0.0, my = u ? __ddiv_rn(sy, (double)u) : 0.0;
    double sxx = 0.0, syy = 0.0, sxy = 0.0;
    for (uint32_t t = 0; t * kTile < A; ++t) {   // pass 2: the sums of squares and products about the means
      if ((int)t != resident) {
        load_tile(a, s, row0, rows, t);
        resident = (int)t;
      }
      const uint32_t cw = min(kTile, A - t * kTile);
      if (mine) {
        for (uint32_t c = 0; c < cw; ++c) {
          if (!(a.zero || (s.xp[c * kRows + r] & s.yp[c + L]))) continue;
          const double dx = __dsub_rn(s.x[c * kPitch + r], mx), dy = __dsub_rn(s.y[c + L], my);
          sxx = __dadd_rn(sxx, __dmul_rn(dx, dx));
          syy = __dadd_rn(syy, __dmul_rn(dy, dy));
          sxy = __dadd_rn(sxy, __dmul_rn(dx, dy));
        }
      }
    }
    const double den = __dmul_rn(__dsqrt_rn(sxx), __dsqrt_rn(syy));
    const bool defined = u >= a.min_points && den > 0.0;
    double rl = 0.0;
    if (defined) {
      rl = fmin(fmax(__ddiv_rn(sxy, den), -1.0), 1.0);
      const double sc = a.direction == ALZ_CORR_POSITIVE   ? rl
                        : a.direction == ALZ_CORR_NEGATIVE ? __dsub_rn(0.0, rl)
                                                           : fabs(rl);
      if (!valid || sc > best_score) {
        valid = true;
        best_lag = L;
        best_used = u;
        best_r = rl;
        best_score = sc;
      }
    }
    if (L == 0) {
      used0 = u;
      r0 = rl;
    }
  }
  uint32_t n_valid = 0;
  if (mine) {
    n_valid = valid;
    const uint64_t rb = (uint64_t)__double_as_longlong(best_r), sb = (uint64_t)__double_as_longlong(best_score),
                   zb = (uint64_t)__double_as_longlong(r0);
    uint4 h0 = head(i, valid);
    h0.x |= best_lag << 24;
    uint4* o = reinterpret_cast<uint4*>(rec + i);
    o[0] = h0;
    o[1] = make_uint4(i, valid ? best_used : used0, (uint32_t)rb, (uint32_t)(rb >> 32));
    o[2] = make_uint4((uint32_t)sb, (uint32_t)(sb >> 32), (uint32_t)zb, (uint32_t)(zb >> 32));
    if (sel) sel[i] = valid ? sb : kInvalidValue;
  }
  n_valid = __reduce_add_sync(0xFFFFFFFFu, n_valid);   // kRows is a multiple of 32: every lane gets here
  if ((threadIdx.x & 31u) == 0 && n_valid) atomicAdd(valid_cnt, n_valid);
}

// The pass of one correlation call: the target's staleness checks, its upload, corr_kernel
struct CorrPass final : ScorePass {
  alz_corr corr{};
  const alz_corr_target* target = nullptr;
  bool given = false;   // caller series: the target's window_last is not read
  uint32_t tier = 0;
  uint32_t target_used = 0;   // out: the target's present points
  int launch(alz_handle* h, alz_trend_state& s, const ScoredInput& in, void* rec, uint64_t* sel,
             uint32_t* valid_cnt) override {
    const uint32_t P = in.points;
    if (target->n != P) return ALZ_E_STATE;
    if (!given && P && target->window_last != alz_internal_ring_last(h, tier)) return ALZ_E_STATE;
    const size_t bytes = (size_t)P * 9;
    if (s.h_target_bytes < bytes) {
      if (s.h_target) cudaFreeHost(s.h_target);
      s.h_target = nullptr;
      s.h_target_bytes = 0;
      if (cudaMallocHost(&s.h_target, bytes) != cudaSuccess) {
        h->last_err = std::string("correlations: ") + cudaGetErrorString(cudaGetLastError());
        s.h_target = nullptr;
        return ALZ_E_NOMEM;
      }
      s.h_target_bytes = bytes;
    }
    int rc = reserve(h, {{&s.target, std::max<size_t>(bytes, 16)}});
    if (rc != ALZ_OK) return rc;
    // the last call's copies are done: every call ends with a wait
    double* hy = static_cast<double*>(s.h_target);
    uint8_t* hp = reinterpret_cast<uint8_t*>(hy + P);
    target_used = 0;
    for (uint32_t j = 0; j < P; ++j) {
      const bool p = !target->present || target->present[j];
      hy[j] = p ? target->values[j] : 0.0;
      hp[j] = p ? 1u : 0u;
      target_used += p;
    }
    if (!in.n) return ALZ_OK;
    cudaStream_t st = h->stream;
    CK(cudaMemcpyAsync(s.target.p, s.h_target, bytes, cudaMemcpyHostToDevice, st));
    const double* dy = static_cast<const double*>(s.target.p);
    const CorrArgs ca{(uint32_t)in.n, P, in.values, in.present, dy, reinterpret_cast<const uint8_t*>(dy + P),
                      corr.direction, corr.absent == ALZ_CORR_ABSENT_ZERO ? 1u : 0u, corr.max_lag, corr.min_points};
    const uint32_t w = std::min(kTile, P), tw = std::min(w + corr.max_lag, P);
    const size_t sm = smem_bytes(w, tw);
    const unsigned grid = (unsigned)((in.n + kRows - 1) / kRows);
    alz_edge_corr* d_rec = static_cast<alz_edge_corr*>(rec);
    if (in.keys)
      corr_kernel<<<grid, kRows, sm, st>>>(ca, NodeHead{in.keys}, d_rec, sel, valid_cnt);
    else if (in.rows)
      corr_kernel<<<grid, kRows, sm, st>>>(ca, EdgeHead{in.rows}, d_rec, sel, valid_cnt);
    else
      corr_kernel<<<grid, kRows, sm, st>>>(ca, BareHead{}, d_rec, sel, valid_cnt);
    h->launches += 1;
    CK(cudaGetLastError());
    return ALZ_OK;
  }
};

}  // namespace

void alz_internal_free_corr(alz_handle* h) {
  free_scored_state(h->corr);
  free_scored_state(h->node_corr);
  free_scored_state(h->group_corr);
}

namespace {

// 2^64: the largest |value| of a §17 metric, and of a target value
constexpr double kMaxAbs = 18446744073709551616.0;

struct CorrCall : ScoredCall {
  bool device = false;
  alz_corr corr{};
};

bool valid_corr(const alz_corr* c, uint32_t k) {
  return c && k >= 1 && c->direction <= ALZ_CORR_ABS && c->absent <= ALZ_CORR_ABSENT_ZERO &&
         c->max_lag <= ALZ_CORR_MAX_LAG && c->max_lag < k && c->min_points >= 3;
}

bool valid_target(const alz_corr_target* t) {
  if (!t || (t->n && !t->values)) return false;
  for (size_t j = 0; j < t->n; ++j) {
    if (t->present && !t->present[j]) continue;
    const double v = t->values[j];
    if (!std::isfinite(v) || std::fabs(v) > kMaxAbs) return false;
  }
  return true;
}

alz_corr_info info_of(const alz_trend_info& ti, uint32_t target_used) {
  alz_corr_info ci{};
  ci.rows = ti.edges;
  ci.rows_in = ti.rows_in;
  ci.valid = ti.valid;
  ci.above = ti.above;
  ci.points = ti.points;
  ci.tier = ti.tier;
  ci.target_used = target_used;
  return ci;
}

// The 16 entry points. A host full-list call's records are copied before its last wait; a host top call copies its
// results after the selection, with one more wait. Device calls: *dev (required) gets the device results.
int corr_entry(alz_handle* h, CorrCall c, const alz_metric* m, const alz_corr* corr, const alz_corr_target* target,
               void* out, void* rows, double* series, uint8_t* present, size_t cap, ScoredResult* dev, size_t* n_out,
               uint32_t* n_points, alz_rollup_info* points, alz_corr_info* info) {
  if (!h || !n_out || !n_points) {
    if (n_out) *n_out = 0;
    if (n_points) *n_points = 0;
    return ALZ_E_INVAL;
  }
  *n_out = 0;
  *n_points = 0;
  if (info) *info = alz_corr_info{};
  if (!valid_corr(corr, c.k) || !valid_metrics(m, 1, &c.ms) || !valid_target(target)) return ALZ_E_INVAL;
  c.corr = *corr;
  if (c.source != ALZ_SOURCE_WINDOW && c.source > ALZ_ROLLUP_SPAN) return ALZ_E_INVAL;
  if (c.node && c.side > ALZ_SIDE_OUT) return ALZ_E_INVAL;
  if (c.top && (c.n_top == 0 || std::isnan(c.min_value))) return ALZ_E_INVAL;
  if (c.device ? !dev : (!c.top && !out && cap)) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  ScoredResult res;
  alz_trend_info ti{};
  CorrPass pass;
  pass.corr = c.corr;
  pass.target = target;
  pass.tier = c.tier;
  const int rc = scored_series_locked(h, c.group ? h->group_corr : c.node ? h->node_corr : h->corr,
                                      c.group ? "group correlations" : c.node ? "node correlations"
                                                                              : "edge correlations",
                                      c, c.device ? SIZE_MAX : cap, c.device || c.top ? nullptr : out, pass, &res,
                                      n_points, points, &ti);
  *n_out = res.m;
  if (rc != ALZ_OK) return rc;
  if (info) *info = info_of(ti, pass.target_used);
  const size_t mm = res.m, P = *n_points;
  if (c.device) {
    *dev = res;
    return ALZ_OK;
  }
  if (!c.top) return ALZ_OK;   // the records came with the call's wait
  if (mm > cap) return ALZ_E_CAPACITY;
  cudaStream_t st = h->stream;
  const size_t row_bytes = c.node ? sizeof(alz_node_out) : sizeof(alz_edge_out);
  if (mm && out) CK(cudaMemcpyAsync(out, res.rec, mm * sizeof(alz_edge_corr), cudaMemcpyDeviceToHost, st));
  if (mm && rows) CK(cudaMemcpyAsync(rows, res.rows, mm * row_bytes, cudaMemcpyDeviceToHost, st));
  if (mm * P && series) CK(cudaMemcpyAsync(series, res.values, mm * P * 8, cudaMemcpyDeviceToHost, st));
  if (mm * P && present) CK(cudaMemcpyAsync(present, res.present, mm * P, cudaMemcpyDeviceToHost, st));
  if (mm) CK(cudaStreamSynchronize(st));
  return ALZ_OK;
}

// The device entry points: corr_entry, then its results as the caller's pointer types
template <class Rec, class Row>
int corr_device(alz_handle* h, const CorrCall& c, const alz_metric* m, const alz_corr* corr,
                const alz_corr_target* target, const Rec** dev_out, const Row** dev_rows, const double** dev_series,
                const uint8_t** dev_present, size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                alz_corr_info* info) {
  ScoredResult r;
  const int rc = corr_entry(h, c, m, corr, target, nullptr, nullptr, nullptr, nullptr, 0, dev_out ? &r : nullptr,
                            n_out, n_points, points, info);
  if (rc != ALZ_OK) return rc;
  *dev_out = static_cast<const Rec*>(r.rec);
  if (dev_rows) *dev_rows = static_cast<const Row*>(r.rows);
  if (dev_series) *dev_series = r.values;
  if (dev_present) *dev_present = r.present;
  return ALZ_OK;
}

CorrCall call_of(bool device, bool top, bool node, bool group, uint32_t source, uint32_t side, uint32_t tier,
                 uint32_t k, uint32_t n_top, double min_score) {
  CorrCall c;
  c.device = device;
  c.top = top;
  c.node = node;
  c.group = group;
  c.source = source;
  c.side = side;
  c.tier = tier;
  c.k = k;
  c.n_top = n_top;
  c.min_value = min_score;
  return c;
}

}  // namespace

extern "C" int alz_edge_correlations(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k, const alz_metric* m,
                                     const alz_corr* corr, const alz_corr_target* target, alz_edge_corr* out,
                                     size_t cap, size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                                     alz_corr_info* info) {
  return corr_entry(h, call_of(false, false, false, false, source, 0, tier, k, 0, 0.0), m, corr, target, out, nullptr,
                    nullptr, nullptr, cap, nullptr, n_out, n_points, points, info);
}

extern "C" int alz_edge_correlations_device(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k,
                                            const alz_metric* m, const alz_corr* corr, const alz_corr_target* target,
                                            const alz_edge_corr** dev_out, size_t* n_out, uint32_t* n_points,
                                            alz_rollup_info* points, alz_corr_info* info) {
  return corr_device<alz_edge_corr, alz_edge_out>(h, call_of(true, false, false, false, source, 0, tier, k, 0, 0.0), m,
                                                  corr, target, dev_out, nullptr, nullptr, nullptr, n_out, n_points,
                                                  points, info);
}

extern "C" int alz_edge_correlations_top(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k,
                                         const alz_metric* m, const alz_corr* corr, const alz_corr_target* target,
                                         uint32_t top, double min_score, alz_edge_corr* out, alz_edge_out* rows,
                                         double* series, uint8_t* present, size_t cap, size_t* n_out,
                                         uint32_t* n_points, alz_rollup_info* points, alz_corr_info* info) {
  return corr_entry(h, call_of(false, true, false, false, source, 0, tier, k, top, min_score), m, corr, target, out,
                    rows, series, present, cap, nullptr, n_out, n_points, points, info);
}

extern "C" int alz_edge_correlations_top_device(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k,
                                                const alz_metric* m, const alz_corr* corr,
                                                const alz_corr_target* target, uint32_t top, double min_score,
                                                const alz_edge_corr** dev_out, const alz_edge_out** dev_rows,
                                                const double** dev_series, const uint8_t** dev_present, size_t* n_out,
                                                uint32_t* n_points, alz_rollup_info* points, alz_corr_info* info) {
  return corr_device(h, call_of(true, true, false, false, source, 0, tier, k, top, min_score), m, corr, target,
                     dev_out, dev_rows, dev_series, dev_present, n_out, n_points, points, info);
}

extern "C" int alz_node_correlations(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                     const alz_metric* m, const alz_corr* corr, const alz_corr_target* target,
                                     alz_node_corr* out, size_t cap, size_t* n_out, uint32_t* n_points,
                                     alz_rollup_info* points, alz_corr_info* info) {
  return corr_entry(h, call_of(false, false, true, false, source, side, tier, k, 0, 0.0), m, corr, target, out,
                    nullptr, nullptr, nullptr, cap, nullptr, n_out, n_points, points, info);
}

extern "C" int alz_node_correlations_device(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                            const alz_metric* m, const alz_corr* corr, const alz_corr_target* target,
                                            const alz_node_corr** dev_out, size_t* n_out, uint32_t* n_points,
                                            alz_rollup_info* points, alz_corr_info* info) {
  return corr_device<alz_node_corr, alz_node_out>(h, call_of(true, false, true, false, source, side, tier, k, 0, 0.0),
                                                  m, corr, target, dev_out, nullptr, nullptr, nullptr, n_out,
                                                  n_points, points, info);
}

extern "C" int alz_node_correlations_top(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                         const alz_metric* m, const alz_corr* corr, const alz_corr_target* target,
                                         uint32_t top, double min_score, alz_node_corr* out, alz_node_out* nodes,
                                         double* series, uint8_t* present, size_t cap, size_t* n_out,
                                         uint32_t* n_points, alz_rollup_info* points, alz_corr_info* info) {
  return corr_entry(h, call_of(false, true, true, false, source, side, tier, k, top, min_score), m, corr, target, out,
                    nodes, series, present, cap, nullptr, n_out, n_points, points, info);
}

extern "C" int alz_node_correlations_top_device(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier,
                                                uint32_t k, const alz_metric* m, const alz_corr* corr,
                                                const alz_corr_target* target, uint32_t top, double min_score,
                                                const alz_node_corr** dev_out, const alz_node_out** dev_nodes,
                                                const double** dev_series, const uint8_t** dev_present, size_t* n_out,
                                                uint32_t* n_points, alz_rollup_info* points, alz_corr_info* info) {
  return corr_device(h, call_of(true, true, true, false, source, side, tier, k, top, min_score), m, corr, target,
                     dev_out, dev_nodes, dev_series, dev_present, n_out, n_points, points, info);
}

extern "C" int alz_group_edge_correlations(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k,
                                           const alz_metric* m, const alz_corr* corr, const alz_corr_target* target,
                                           alz_edge_corr* out, size_t cap, size_t* n_out, uint32_t* n_points,
                                           alz_rollup_info* points, alz_corr_info* info) {
  return corr_entry(h, call_of(false, false, false, true, source, 0, tier, k, 0, 0.0), m, corr, target, out, nullptr,
                    nullptr, nullptr, cap, nullptr, n_out, n_points, points, info);
}

extern "C" int alz_group_edge_correlations_device(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k,
                                                  const alz_metric* m, const alz_corr* corr,
                                                  const alz_corr_target* target, const alz_edge_corr** dev_out,
                                                  size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                                                  alz_corr_info* info) {
  return corr_device<alz_edge_corr, alz_edge_out>(h, call_of(true, false, false, true, source, 0, tier, k, 0, 0.0), m,
                                                  corr, target, dev_out, nullptr, nullptr, nullptr, n_out, n_points,
                                                  points, info);
}

extern "C" int alz_group_edge_correlations_top(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k,
                                               const alz_metric* m, const alz_corr* corr,
                                               const alz_corr_target* target, uint32_t top, double min_score,
                                               alz_edge_corr* out, alz_edge_out* rows, double* series,
                                               uint8_t* present, size_t cap, size_t* n_out, uint32_t* n_points,
                                               alz_rollup_info* points, alz_corr_info* info) {
  return corr_entry(h, call_of(false, true, false, true, source, 0, tier, k, top, min_score), m, corr, target, out,
                    rows, series, present, cap, nullptr, n_out, n_points, points, info);
}

extern "C" int alz_group_edge_correlations_top_device(alz_handle* h, uint32_t source, uint32_t tier, uint32_t k,
                                                      const alz_metric* m, const alz_corr* corr,
                                                      const alz_corr_target* target, uint32_t top, double min_score,
                                                      const alz_edge_corr** dev_out, const alz_edge_out** dev_rows,
                                                      const double** dev_series, const uint8_t** dev_present,
                                                      size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                                                      alz_corr_info* info) {
  return corr_device(h, call_of(true, true, false, true, source, 0, tier, k, top, min_score), m, corr, target,
                     dev_out, dev_rows, dev_series, dev_present, n_out, n_points, points, info);
}

extern "C" int alz_group_node_correlations(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier, uint32_t k,
                                           const alz_metric* m, const alz_corr* corr, const alz_corr_target* target,
                                           alz_node_corr* out, size_t cap, size_t* n_out, uint32_t* n_points,
                                           alz_rollup_info* points, alz_corr_info* info) {
  return corr_entry(h, call_of(false, false, true, true, source, side, tier, k, 0, 0.0), m, corr, target, out,
                    nullptr, nullptr, nullptr, cap, nullptr, n_out, n_points, points, info);
}

extern "C" int alz_group_node_correlations_device(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier,
                                                  uint32_t k, const alz_metric* m, const alz_corr* corr,
                                                  const alz_corr_target* target, const alz_node_corr** dev_out,
                                                  size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                                                  alz_corr_info* info) {
  return corr_device<alz_node_corr, alz_node_out>(h, call_of(true, false, true, true, source, side, tier, k, 0, 0.0),
                                                  m, corr, target, dev_out, nullptr, nullptr, nullptr, n_out,
                                                  n_points, points, info);
}

extern "C" int alz_group_node_correlations_top(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier,
                                               uint32_t k, const alz_metric* m, const alz_corr* corr,
                                               const alz_corr_target* target, uint32_t top, double min_score,
                                               alz_node_corr* out, alz_node_out* nodes, double* series,
                                               uint8_t* present, size_t cap, size_t* n_out, uint32_t* n_points,
                                               alz_rollup_info* points, alz_corr_info* info) {
  return corr_entry(h, call_of(false, true, true, true, source, side, tier, k, top, min_score), m, corr, target, out,
                    nodes, series, present, cap, nullptr, n_out, n_points, points, info);
}

extern "C" int alz_group_node_correlations_top_device(alz_handle* h, uint32_t source, uint32_t side, uint32_t tier,
                                                      uint32_t k, const alz_metric* m, const alz_corr* corr,
                                                      const alz_corr_target* target, uint32_t top, double min_score,
                                                      const alz_node_corr** dev_out, const alz_node_out** dev_nodes,
                                                      const double** dev_series, const uint8_t** dev_present,
                                                      size_t* n_out, uint32_t* n_points, alz_rollup_info* points,
                                                      alz_corr_info* info) {
  return corr_device(h, call_of(true, true, true, true, source, side, tier, k, top, min_score), m, corr, target,
                     dev_out, dev_nodes, dev_series, dev_present, n_out, n_points, points, info);
}

extern "C" int alz_debug_corr_series(alz_handle* h, const double* dev_values, const uint8_t* dev_present, size_t n,
                                     uint32_t P, const alz_corr_target* target, const alz_corr* corr, uint32_t top,
                                     double min_score, alz_edge_corr* out, uint32_t* top_index, size_t cap,
                                     size_t* n_out, uint64_t* valid, uint64_t* above) {
  if (!h || !n_out) return ALZ_E_INVAL;
  *n_out = 0;
  if (!valid_corr(corr, UINT32_MAX) || !valid_target(target)) return ALZ_E_INVAL;
  if (n && P && (!dev_values || !dev_present)) return ALZ_E_INVAL;
  if (top && std::isnan(min_score)) return ALZ_E_INVAL;
  if (!out && cap) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  CorrCall c;
  c.top = top > 0;
  c.n_top = top;
  c.min_value = min_score;
  c.given = true;
  c.given_values = dev_values;
  c.given_present = dev_present;
  c.given_n = n;
  c.given_points = P;
  CorrPass pass;
  pass.corr = *corr;
  pass.target = target;
  pass.given = true;
  ScoredResult res;
  alz_trend_info ti{};
  uint32_t n_points = 0;
  const int rc = scored_series_locked(h, h->corr, "edge correlations", c, SIZE_MAX, nullptr, pass, &res, &n_points,
                                      nullptr, &ti);
  *n_out = res.m;
  if (rc != ALZ_OK) return rc;
  if (valid) *valid = ti.valid;
  if (above) *above = ti.above;
  if (res.m > cap) return ALZ_E_CAPACITY;
  cudaStream_t st = h->stream;
  if (res.m) CK(cudaMemcpyAsync(out, res.rec, res.m * sizeof(alz_edge_corr), cudaMemcpyDeviceToHost, st));
  if (res.m && c.top && top_index)
    CK(cudaMemcpyAsync(top_index, res.index, res.m * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return ALZ_OK;
}
