// alz_gnn.cu — GNN anomaly pass over the flushed service graph (docs/SPEC.md §6;
// not in the reference: north_star's extension). 2-layer GraphSAGE-mean, d = 64,
// fixed seeded weights, per-edge score. The same pass scores a window, tier or span
// rollup's rows (docs/SPEC.md §15): it is a function of the rows it is given.
//
//   nodes   : 2 node keys per edge -> sort -> unique (ascending (kind,value))
//   stats   : per-node in/out count, 5xx, latency sum, degree  (u64 atomics: exact,
//             order-independent, so the float features are deterministic)
//   CSR     : in-edges grouped by destination (stable sort by dst index, row
//             offsets = exclusive scan of the in-degrees)
//   layer   : mean of the in-neighbours' rows (coalesced 256-B row reads) ->
//             [h_v || m_v] (128) x W (128 x 64) + b, ReLU; the GEMM runs on wgmma
//             (sage_layer_tc_kernel, 3xTF32), an FP32 FFMA version is kept for comparison
//   score   : sigma(a . [h2_u || h2_v || e_uv] + c), e_uv from the edge's
//             integers and float64 histogram quantiles
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <string>
#include <mutex>
#include <vector>

#include <cub/block/block_scan.cuh>

#include "alz_handle.h"
#include "alz_mbar.cuh"
#include "alz_top.cuh"

using namespace alz;

namespace {

constexpr int D = 64;
constexpr uint64_t kGnnSeed = 0xA1A26E6Eull;

// ---- weights: pure integer -> double -> float, restated in tests/gnn_ref.py -----
inline double unit(uint64_t idx) {
  const uint64_t r = alz_splitmix64(kGnnSeed + idx);
  return (double)(r >> 11) * (1.0 / 9007199254740992.0) * 2.0 - 1.0;   // [-1, 1)
}

struct Weights {
  std::vector<float> W[2], b[2], a;   // W[l][k*64 + j], k in [0,128)
  float c;
};
Weights make_weights() {
  Weights w;
  const double sw = 1.0 / std::sqrt(128.0), sa = 1.0 / std::sqrt(132.0);
  uint64_t idx = 0;
  for (int l = 0; l < 2; ++l) {
    w.W[l].resize(128 * D);
    w.b[l].resize(D);
    for (int k = 0; k < 128; ++k)
      for (int j = 0; j < D; ++j) w.W[l][k * D + j] = (float)(unit(idx++) * sw);
    for (int j = 0; j < D; ++j) w.b[l][j] = (float)(unit(idx++) * 0.01);
  }
  w.a.resize(132);
  for (int k = 0; k < 132; ++k) w.a[k] = (float)(unit(idx++) * sa);
  w.c = 0.0f;
  return w;
}

// host-side cvt.rna.tf32.f32: round to nearest (ties away) on the 13 dropped mantissa bits
inline float tf32_round(float x) {
  uint32_t u;
  memcpy(&u, &x, 4);
  u = (u + 0x1000u) & 0xFFFFE000u;
  float r;
  memcpy(&r, &u, 4);
  return r;
}

__global__ void edge_node_keys_kernel(const alz_edge_out* __restrict__ e, uint32_t n_e, uint64_t* __restrict__ out) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_e; i += stride) {
    out[2 * i] = node_key(e[i].from_type, e[i].from);
    out[2 * i + 1] = node_key(e[i].to_type, e[i].to);
  }
}

// per node: [out_count, in_count, out_err, in_err, out_lat, in_lat, out_deg, in_deg]
// the node count stays on the device: every consumer reads it from there, the host never waits for it
__global__ void node_count_kernel(const uint32_t* __restrict__ pos, const uint32_t* __restrict__ flags, uint32_t n2,
                                  uint32_t* __restrict__ n_v) {
  if (threadIdx.x == 0 && blockIdx.x == 0) *n_v = n2 ? pos[n2 - 1] + flags[n2 - 1] : 0u;
}

__global__ void edge_stats_kernel(const alz_edge_out* __restrict__ e, uint32_t n_e, const uint64_t* __restrict__ nodes,
                                  const uint32_t* __restrict__ n_v_ptr, uint32_t* __restrict__ src_idx,
                                  uint64_t* __restrict__ dst_key, unsigned long long* __restrict__ stats,
                                  uint32_t* __restrict__ in_deg) {
  const uint32_t n_v = *n_v_ptr;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_e; i += stride) {
    const uint32_t u = lower_bound_u64(nodes, n_v, node_key(e[i].from_type, e[i].from));
    const uint32_t v = lower_bound_u64(nodes, n_v, node_key(e[i].to_type, e[i].to));
    src_idx[i] = u;
    dst_key[i] = v;
    atomicAdd(&stats[(size_t)u * 8 + 0], (unsigned long long)e[i].count);
    atomicAdd(&stats[(size_t)v * 8 + 1], (unsigned long long)e[i].count);
    if (e[i].err5xx) {
      atomicAdd(&stats[(size_t)u * 8 + 2], (unsigned long long)e[i].err5xx);
      atomicAdd(&stats[(size_t)v * 8 + 3], (unsigned long long)e[i].err5xx);
    }
    atomicAdd(&stats[(size_t)u * 8 + 4], (unsigned long long)e[i].lat_sum_ns);
    atomicAdd(&stats[(size_t)v * 8 + 5], (unsigned long long)e[i].lat_sum_ns);
    atomicAdd(&stats[(size_t)u * 8 + 6], 1ull);
    atomicAdd(&stats[(size_t)v * 8 + 7], 1ull);
    atomicAdd(&in_deg[v], 1u);
  }
}

__global__ void csr_cols_kernel(const uint32_t* __restrict__ sorted_edge, const uint32_t* __restrict__ src_idx,
                                uint32_t n_e, uint32_t* __restrict__ col) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_e; i += stride) col[i] = src_idx[sorted_edge[i]];
}

__device__ __forceinline__ double ratio(uint64_t a, uint64_t b) { return b ? (double)a / (double)b : 0.0; }

__global__ void node_features_kernel(const uint64_t* __restrict__ nodes, const unsigned long long* __restrict__ stats,
                                     const uint32_t* __restrict__ n_v_ptr, float* __restrict__ h0) {
  const uint32_t n_v = *n_v_ptr;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n_v; v += stride) {
    const unsigned long long* s = stats + (size_t)v * 8;
    float* o = h0 + (size_t)v * D;
    const uint32_t kind = (uint32_t)(nodes[v] >> 32);
    float f[12];
    f[0] = (float)log1p((double)s[0]);
    f[1] = (float)log1p((double)s[1]);
    f[2] = (float)ratio(s[2], s[0]);
    f[3] = (float)ratio(s[3], s[1]);
    f[4] = (float)log1p(ratio(s[4], s[0]));
    f[5] = (float)log1p(ratio(s[5], s[1]));
    f[6] = (float)log1p((double)s[6]);
    f[7] = (float)log1p((double)s[7]);
    f[8] = kind == ALZ_NODE_POD ? 1.f : 0.f;
    f[9] = kind == ALZ_NODE_SVC ? 1.f : 0.f;
    f[10] = kind >= ALZ_NODE_OUTBOUND ? 1.f : 0.f;   // outbound, keyed by address or by Host header
    f[11] = 1.f;
    for (int j = 0; j < D; ++j) o[j] = j < 12 ? f[j] : 0.f;
  }
}

// one GraphSAGE-mean layer, FP32 SIMT: warp per node, W (32 KB) in shared memory
__global__ void __launch_bounds__(256) sage_layer_kernel(const float* __restrict__ h_in, float* __restrict__ h_out,
                                                         const uint32_t* __restrict__ rowptr,
                                                         const uint32_t* __restrict__ col, const float* __restrict__ W,
                                                         const float* __restrict__ b, const uint32_t* __restrict__ n_v_ptr) {
  const uint32_t n_v = *n_v_ptr;
  __shared__ float sW[128 * D];
  __shared__ float sz[8][128];
  for (int i = threadIdx.x; i < 128 * D; i += blockDim.x) sW[i] = W[i];
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t warps_per_grid = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; v < n_v; v += warps_per_grid) {
    const uint32_t beg = rowptr[v], end = rowptr[v + 1];
    double m0 = 0.0, m1 = 0.0;                       // float64: a hub's many similar rows do not drift (SPEC §6)
    for (uint32_t p = beg; p < end; ++p) {          // CSR order: deterministic sum
      const float* hu = h_in + (size_t)col[p] * D;
      m0 += (double)hu[lane];
      m1 += (double)hu[32 + lane];
    }
    const double inv = end > beg ? 1.0 / (double)(end - beg) : 0.0;
    const float* hv = h_in + (size_t)v * D;
    sz[warp][lane] = hv[lane];
    sz[warp][32 + lane] = hv[32 + lane];
    sz[warp][64 + lane] = (float)(m0 * inv);
    sz[warp][96 + lane] = (float)(m1 * inv);
    __syncwarp();
    float a0 = b[lane], a1 = b[32 + lane];
#pragma unroll 8
    for (int k = 0; k < 128; ++k) {
      const float z = sz[warp][k];
      a0 = fmaf(z, sW[k * D + lane], a0);
      a1 = fmaf(z, sW[k * D + 32 + lane], a1);
    }
    h_out[(size_t)v * D + lane] = fmaxf(a0, 0.f);
    h_out[(size_t)v * D + 32 + lane] = fmaxf(a1, 0.f);
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------
// The same layer on the Hopper tensor cores: the feature update
//   [h_v || mean_{u in N_in(v)} h_u]  (128 nodes x 128)  x  W (128 x 64)
// is the path's one dense contraction. One persistent CTA per SM, tile = 128 nodes:
//   gather   8 warps build the tile's 128 x 128 operand directly in shared memory in
//            the wgmma K-major / no-swizzle layout (8 x 16-byte core matrices)
//   MMA      each of the two warpgroups issues wgmma.mma_async m64n64k8 .tf32 on its
//            64 rows of the tile, accumulator in registers (32 fp32 per thread)
//   epilogue every thread adds the bias to its accumulator fragment, ReLU, stores
// Precision: tf32 keeps 10 mantissa bits, which would miss the 1e-5 bound, so
// both operands are split x = hi + lo (hi = cvt.rna.tf32, lo = x - hi, exact) and
// the product is accumulated as hi*hi + hi*lo + lo*hi (3xTF32): 48 wgmma per warpgroup per tile.
// ---------------------------------------------------------------------------
namespace tc {
constexpr uint32_t TM = 128, TK = 128, TN = 64;
constexpr uint32_t WG_M = 64;                             // rows of the tile per warpgroup
constexpr uint32_t A_BYTES = TM * TK * 4, B_BYTES = TN * TK * 4;
constexpr uint32_t A_LBO = (TM / 8) * 128, A_SBO = 128;   // K-adjacent cores TM/8 cores apart; row groups adjacent
constexpr uint32_t B_LBO = (TN / 8) * 128, B_SBO = 128;

// byte offset of element (row r, k) in a K-major no-swizzle operand with R rows:
// core matrix = 8 rows x 16 B; cores of one K-slice are contiguous over the row groups
__host__ __device__ inline uint32_t op_off(uint32_t r, uint32_t k, uint32_t rows) {
  return (k >> 2) * (rows / 8) * 128 + (r >> 3) * 128 + (r & 7) * 16 + (k & 3) * 4;
}
// wgmma shared-memory descriptor (sm_90): start >> 4 at bit 0, LBO >> 4 at bit 16 (K-adjacent core matrices),
// SBO >> 4 at bit 32 (adjacent 8-row groups), base offset 0, layout type 0 (no swizzle) at bit 62
__device__ __forceinline__ uint64_t smem_desc(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(sbo >> 4) << 32);
}

__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return u;
}
// D (64 x 64 fp32, this warpgroup's fragment) += A (64 x 8) * B (8 x 64), both tf32 K-major in shared memory
__device__ __forceinline__ void wgmma_tf32(float* d, uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db)
      : "memory");
}

// ---- TMA-staged neighbour gather ---------------------------------------------------------
// A warp builds 16 rows of the tile's operand. Every 256-byte feature row it needs — its nodes' own rows (16
// consecutive rows of h_in: two bulk copies) and then the rows of their in-neighbours in CSR order — is fetched
// by the TMA (cp.async.bulk global -> shared, completion on an mbarrier) into a two-slot ring of 8 rows per
// warp: while the warp sums the rows of one slot, the copies of the next 8 neighbours are in flight, 16 rows
// per warp regardless of the nodes' degrees (the edge range of the warp's rows is walked as one stream and cut
// at the row boundaries). No register holds a row in flight, unlike plain loads.
constexpr uint32_t RING_ROWS = 8, RING_BYTES = RING_ROWS * 256;
constexpr uint32_t SMEM_TC = 2 * A_BYTES + 2 * B_BYTES + 8 * 2 * RING_BYTES + 256;

__device__ __forceinline__ void tma_row(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// operand row r, columns kbase + lane and kbase + 32 + lane <- (z0, z1), split hi/lo in the wgmma layout
__device__ __forceinline__ void put_pair(uint8_t* sA_hi, uint8_t* sA_lo, uint32_t r, uint32_t kbase, uint32_t lane,
                                         float z0, float z1) {
  const float z[2] = {z0, z1};
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const uint32_t k = kbase + (uint32_t)q * 32 + lane;
    const uint32_t hi = to_tf32(z[q]);
    const uint32_t lo = to_tf32(z[q] - __uint_as_float(hi));
    const uint32_t off = op_off(r, k, TM);
    *reinterpret_cast<uint32_t*>(sA_hi + off) = hi;
    *reinterpret_cast<uint32_t*>(sA_lo + off) = lo;
  }
}

__global__ void __launch_bounds__(256, 1) sage_layer_tc_kernel(const float* __restrict__ h_in, float* __restrict__ h_out,
                                                               const uint32_t* __restrict__ rowptr,
                                                               const uint32_t* __restrict__ col,
                                                               const uint8_t* __restrict__ Wcan,   // B_hi then B_lo
                                                               const float* __restrict__ bias,
                                                               const uint32_t* __restrict__ n_v_ptr) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t n_v = *n_v_ptr;
  const uint32_t zero_rt = n_v >> 31;                    // node counts are < 2^31
  uint8_t* sA_hi = smem;
  uint8_t* sA_lo = smem + A_BYTES;
  uint8_t* sB = smem + 2 * A_BYTES;                      // B_hi, then B_lo
  uint8_t* rings = smem + 2 * A_BYTES + 2 * B_BYTES;     // per warp: 2 slots of RING_ROWS rows
  uint64_t* bars = reinterpret_cast<uint64_t*>(rings + 8 * 2 * RING_BYTES);   // [2w + slot] ring slots
  const uint32_t tid = threadIdx.x, warp = tid >> 5, lane = tid & 31u;
  const uint32_t wg = warp >> 2;                         // warpgroup: rows 64 wg .. 64 wg + 63 of the tile
  const float* ring = reinterpret_cast<const float*>(rings + warp * 2 * RING_BYTES);
  const uint32_t ring_a = smem_u32(ring);
  const uint32_t rbar = smem_u32(bars + 2 * warp);
  uint32_t ring_uses[2] = {0u, 0u};

  for (uint32_t i = tid; i < 2 * B_BYTES / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(sB)[i] = reinterpret_cast<const uint4*>(Wcan)[i];
  if (lane == 0) { mbar_init(rbar, 1u); mbar_init(rbar + 8u, 1u); }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();

  for (uint32_t tile = blockIdx.x; tile * TM < n_v; tile += gridDim.x) {
    // ---- gather: warp w builds rows 16w .. 16w+15 of the operand (hi and lo parts)
    const uint32_t v0 = tile * TM + warp * 16;
    const uint32_t n_rows = v0 < n_v ? min(16u, n_v - v0) : 0u;
    // (1) the nodes' own rows: two bulk copies of up to 8 consecutive rows each
    for (uint32_t half = 0; half < 2; ++half) {
      const uint32_t cnt = n_rows > half * 8 ? min(8u, n_rows - half * 8) : 0u;
      if (lane == 0 && cnt) {
        mbar_expect_tx(rbar + half * 8u, cnt * 256u);
        tma_row(ring_a + half * RING_BYTES, h_in + (size_t)(v0 + half * 8) * D, cnt * 256u, rbar + half * 8u);
      }
    }
    for (uint32_t half = 0; half < 2; ++half) {
      const uint32_t cnt = n_rows > half * 8 ? min(8u, n_rows - half * 8) : 0u;
      if (cnt) { mbar_wait(rbar + half * 8u, ring_uses[half] & 1u); ring_uses[half]++; }
      for (uint32_t j = 0; j < 8; ++j) {
        const float* row = ring + (half * RING_ROWS + j) * D;
        const bool on = j < cnt;
        put_pair(sA_hi, sA_lo, warp * 16 + half * 8 + j, 0u, lane, on ? row[lane] : 0.f, on ? row[32 + lane] : 0.f);
      }
      __syncwarp();
    }
    // (2) the in-neighbours of the warp's rows, as one stream of edges cut at the row boundaries
    const uint32_t e_beg = n_rows ? rowptr[v0] : 0u, e_end = n_rows ? rowptr[v0 + n_rows] : 0u;
    const uint32_t n_chunks = (e_end - e_beg + RING_ROWS - 1) / RING_ROWS;
    // `dep` is always 0 but derived from the last word this lane read out of the slot (zero_rt is a run-time 0 the
    // compiler cannot see through): the copies that refill a slot cannot be issued before its reads have returned
    auto issue = [&](uint32_t c, uint32_t dep) {
      const uint32_t slot = c & 1u, first = e_beg + c * RING_ROWS, cnt = min(RING_ROWS, e_end - first);
      if (lane == 0) mbar_expect_tx(rbar + slot * 8u, cnt * 256u + dep);
      __syncwarp();
      if (lane < cnt) tma_row(ring_a + (slot * RING_ROWS + lane) * 256u, h_in + (size_t)col[first + lane] * D, 256u + dep, rbar + slot * 8u);
    };
    if (n_chunks > 0) issue(0, 0u);
    if (n_chunks > 1) issue(1, 0u);
    uint32_t r = 0;                                   // current row of the warp
    uint32_t row_end = n_rows ? rowptr[v0 + 1] : 0u, row_beg = e_beg;
    double m0 = 0.0, m1 = 0.0;                        // float64 neighbour sums (SPEC §6), as in the SIMT layer
    auto close_rows_until = [&](uint32_t e) {         // rows that end at or before edge e are complete
      while (r < n_rows && row_end <= e) {
        const double inv = row_end > row_beg ? 1.0 / (double)(row_end - row_beg) : 0.0;
        put_pair(sA_hi, sA_lo, warp * 16 + r, 64u, lane, (float)(m0 * inv), (float)(m1 * inv));
        m0 = m1 = 0.0;
        ++r;
        row_beg = row_end;
        if (r < n_rows) row_end = rowptr[v0 + r + 1];
      }
    };
    for (uint32_t c = 0; c < n_chunks; ++c) {
      const uint32_t slot = c & 1u, first = e_beg + c * RING_ROWS, cnt = min(RING_ROWS, e_end - first);
      mbar_wait(rbar + slot * 8u, ring_uses[slot] & 1u);
      ring_uses[slot]++;
      float last = 0.f;
      for (uint32_t j = 0; j < cnt; ++j) {          // CSR order: deterministic sum
        close_rows_until(first + j);
        const float* row = ring + (slot * RING_ROWS + j) * D;
        last = row[lane];
        m0 += (double)last;
        m1 += (double)row[32 + lane];
      }
      __syncwarp();
      if (c + 2 < n_chunks) issue(c + 2, __float_as_uint(last) & zero_rt);   // the slot goes back to the TMA
    }
    close_rows_until(e_end);                          // the last rows, and rows without in-edges
    for (uint32_t rr = n_rows; rr < 16; ++rr) {       // rows past the end of the graph: zeros
      put_pair(sA_hi, sA_lo, warp * 16 + rr, 0u, lane, 0.f, 0.f);
      put_pair(sA_hi, sA_lo, warp * 16 + rr, 64u, lane, 0.f, 0.f);
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> tensor-core (async proxy) reads
    __syncthreads();
    // ---- MMA: each warpgroup, 3 passes x 16 K-steps of M64 N64 K8 over its 64 rows (8 row groups = 1 KB in)
    float acc[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[j] = 0.f;
    {
      const uint32_t a_off = wg * (WG_M / 8) * 128;
      const uint32_t a_hi = smem_u32(sA_hi) + a_off, a_lo = smem_u32(sA_lo) + a_off;
      const uint32_t b_hi = smem_u32(sB), b_lo = smem_u32(sB + B_BYTES);
      const uint32_t pa[3] = {a_hi, a_hi, a_lo}, pb[3] = {b_hi, b_lo, b_hi};
      asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
      for (int ps = 0; ps < 3; ++ps) {
#pragma unroll
        for (uint32_t ks = 0; ks < TK / 8; ++ks) {
          const uint64_t da = smem_desc(pa[ps] + ks * 2 * A_LBO, A_LBO, A_SBO);
          const uint64_t db = smem_desc(pb[ps] + ks * 2 * B_LBO, B_LBO, B_SBO);
          wgmma_tf32(acc, da, db);
        }
      }
      asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
      asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
    }
    // ---- epilogue: accumulator fragment of warp w (of the warpgroup), lane l: rows 16w + l/4 (+8),
    // columns 8j + 2 (l % 4) (+1) in acc[4j + {0,1}] (+ {2,3} for the row 8 further down)
    {
      const uint32_t r0 = tile * TM + wg * WG_M + (warp & 3u) * 16 + (lane >> 2);
#pragma unroll
      for (uint32_t half = 0; half < 2; ++half) {
        const uint32_t v = r0 + half * 8;
        if (v < n_v) {
          float* orow = h_out + (size_t)v * D;
#pragma unroll
          for (uint32_t j = 0; j < TN / 8; ++j) {
            const uint32_t c = 8 * j + 2 * (lane & 3u);
            float2 o;
            o.x = fmaxf(acc[4 * j + 2 * half + 0] + bias[c + 0], 0.f);
            o.y = fmaxf(acc[4 * j + 2 * half + 1] + bias[c + 1], 0.f);
            *reinterpret_cast<float2*>(orow + c) = o;
          }
        }
      }
    }
    __syncthreads();   // the operand tile is free again
  }
}
}  // namespace tc

// docs/SPEC.md §4/§5 on the device, float64
__device__ __forceinline__ double bucket_lo(uint32_t b) {
  if (b == 0) return 0.0;
  const double base = (double)(1ull << (8 + b / 2));
  return (b & 1u) ? base * 1.5 : base;
}
__device__ __forceinline__ double bucket_hi(uint32_t b) { return b == ALZ_NB - 1 ? (double)(1ull << 40) : bucket_lo(b + 1); }
__global__ void __launch_bounds__(256) edge_score_kernel(const alz_edge_out* __restrict__ e, uint32_t n_e,
                                                         const uint32_t* __restrict__ src_idx,
                                                         const uint64_t* __restrict__ dst_key,
                                                         const float* __restrict__ h2, const float* __restrict__ a,
                                                         float c, float* __restrict__ scores) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t warps_per_grid = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n_e; i += warps_per_grid) {
    const float* hu = h2 + (size_t)src_idx[i] * D;
    const float* hv = h2 + (size_t)dst_key[i] * D;
    float acc = hu[lane] * a[lane] + hu[32 + lane] * a[32 + lane] + hv[lane] * a[64 + lane] +
                hv[32 + lane] * a[96 + lane];
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xFFFFFFFFu, acc, o);
    // quantiles with the whole warp: lane l owns buckets 2l and 2l+1; an inclusive scan of the
    // (exactly representable) counts finds the bucket each quantile falls into, then the one
    // lane that owns it interpolates exactly like hist_quantile() / SPEC §5
    const double c0 = (double)e[i].hist[2 * lane], c1 = (double)e[i].hist[2 * lane + 1];
    double incl = c0 + c1;
    for (int o = 1; o < 32; o <<= 1) {
      const double t = __shfl_up_sync(0xFFFFFFFFu, incl, o);
      if ((int)lane >= o) incl += t;
    }
    const double total = __shfl_sync(0xFFFFFFFFu, incl, 31);
    const double before = incl - (c0 + c1);
    double qv[2];
#pragma unroll
    for (int qi = 0; qi < 2; ++qi) {
      const double target = (qi == 0 ? 0.5 : 0.99) * total;
      // first bucket with c > 0 and cum + c >= target
      const bool h0 = c0 > 0.0 && before + c0 >= target;
      const bool h1 = c1 > 0.0 && before + c0 + c1 >= target;
      const uint32_t m = __ballot_sync(0xFFFFFFFFu, h0 || h1);
      double val = total > 0.0 ? bucket_hi(ALZ_NB - 1) : 0.0;
      const int owner = m ? __ffs(m) - 1 : 0;
      if (m && (int)lane == owner) {
        const uint32_t b = h0 ? 2u * lane : 2u * lane + 1u;
        const double cum = h0 ? before : before + c0;
        const double cb = h0 ? c0 : c1;
        double f = (target - cum) / cb;
        if (f < 0.0) f = 0.0;
        val = bucket_lo(b) + f * (bucket_hi(b) - bucket_lo(b));
      }
      qv[qi] = __shfl_sync(0xFFFFFFFFu, val, owner);
    }
    if (lane == 0) {
      const float f0 = (float)log1p((double)e[i].count);
      const float f1 = (float)ratio(e[i].err5xx, e[i].count);
      const float f2 = (float)log1p(qv[0]);
      const float f3 = (float)log1p(qv[1]);
      const float z = acc + f0 * a[128] + f1 * a[129] + f2 * a[130] + f3 * a[131] + c;
      scores[i] = 1.0f / (1.0f + expf(-z));
    }
  }
}

}  // namespace

struct alz_gnn_state {
  uint32_t cap_e = 0, cap_v = 0;
  uint64_t *d_nk = nullptr, *d_nk_sorted = nullptr, *d_nodes = nullptr, *d_dst_key = nullptr, *d_dst_sorted = nullptr;
  uint32_t *d_flags = nullptr, *d_pos = nullptr, *d_iota = nullptr, *d_vals = nullptr, *d_src_idx = nullptr;
  uint32_t *d_in_deg = nullptr, *d_rowptr = nullptr, *d_col = nullptr, *d_sorted_edge = nullptr;
  unsigned long long* d_stats = nullptr;
  float *d_h[3] = {nullptr, nullptr, nullptr}, *d_W[2] = {nullptr, nullptr}, *d_b[2] = {nullptr, nullptr};
  float *d_a = nullptr, *d_scores = nullptr;
  uint8_t* d_Wcan[2] = {nullptr, nullptr};   // per layer: W^T split hi/lo in the wgmma operand layout (64 KB)
  bool use_tc = true;
  float c = 0.f;
  void* d_tmp = nullptr;
  size_t tmp_bytes = 0;
  uint32_t n_v = 0, n_e = 0;
  bool n_v_known = true;
  uint32_t* d_nv = nullptr;      // node count of the last pass, on the device
  // top anomalous rows (docs/SPEC.md §16): the result of the last selection, top_cap rows each; grown on demand
  alz_edge_out* d_top_rows = nullptr;
  float* d_top_scores = nullptr;
  uint32_t* d_top_index = nullptr;
  size_t top_cap = 0;
};

// The buffers sized by rows (cap_e) and nodes (cap_v = 2 cap_e), and the CUB scratch of the sorts and scans over
// up to cap_v + 1 items. The first failed allocation's status; what was allocated stays for free_row_buffers.
static cudaError_t alloc_row_buffers(alz_gnn_state* g, uint32_t cap_e) {
  g->cap_e = cap_e;
  g->cap_v = 2 * cap_e;
  const size_t E = g->cap_e, V = g->cap_v;
  cudaError_t e = cudaSuccess;
  auto get = [&e](auto** p, size_t bytes) { if (e == cudaSuccess) e = cudaMalloc(p, bytes); };
  get(&g->d_nk, V * 8);
  get(&g->d_nk_sorted, V * 8);
  get(&g->d_nodes, V * 8);
  get(&g->d_dst_key, E * 8);
  get(&g->d_dst_sorted, E * 8);
  get(&g->d_flags, V * 4);
  get(&g->d_pos, V * 4);
  get(&g->d_iota, V * 4);
  get(&g->d_vals, V * 4);
  get(&g->d_src_idx, E * 4);
  get(&g->d_in_deg, (V + 1) * 4);
  get(&g->d_rowptr, (V + 1) * 4);
  get(&g->d_col, E * 4);
  get(&g->d_sorted_edge, E * 4);
  get(&g->d_stats, V * 8 * 8);
  for (int i = 0; i < 3; ++i) get(&g->d_h[i], V * D * 4);
  get(&g->d_scores, E * 4);
  g->tmp_bytes = std::max(sort_pairs_temp_bytes((uint32_t)V), scan_temp_bytes((uint32_t)V + 1));
  get(&g->d_tmp, g->tmp_bytes);
  return e;
}

static void free_row_buffers(alz_gnn_state* g) {
  cudaFree(g->d_nk); cudaFree(g->d_nk_sorted); cudaFree(g->d_nodes); cudaFree(g->d_dst_key); cudaFree(g->d_dst_sorted);
  cudaFree(g->d_flags); cudaFree(g->d_pos); cudaFree(g->d_iota); cudaFree(g->d_vals); cudaFree(g->d_src_idx);
  cudaFree(g->d_in_deg); cudaFree(g->d_rowptr); cudaFree(g->d_col); cudaFree(g->d_sorted_edge); cudaFree(g->d_stats);
  for (int i = 0; i < 3; ++i) cudaFree(g->d_h[i]);
  cudaFree(g->d_scores); cudaFree(g->d_tmp);
  g->d_nk = g->d_nk_sorted = g->d_nodes = g->d_dst_key = g->d_dst_sorted = nullptr;
  g->d_flags = g->d_pos = g->d_iota = g->d_vals = g->d_src_idx = nullptr;
  g->d_in_deg = g->d_rowptr = g->d_col = g->d_sorted_edge = nullptr;
  g->d_stats = nullptr;
  g->d_h[0] = g->d_h[1] = g->d_h[2] = nullptr;
  g->d_scores = nullptr;
  g->d_tmp = nullptr;
  g->cap_e = g->cap_v = 0;
  g->tmp_bytes = 0;
}

static int gnn_init_impl(alz_handle* h) {
  alz_gnn_state* g = new alz_gnn_state();
  h->gnn = g;
  CK(alloc_row_buffers(g, h->cfg.max_edges));
  CK(cudaMalloc(&g->d_nv, 4));
  const Weights w = make_weights();
  for (int l = 0; l < 2; ++l) {
    CK(cudaMalloc(&g->d_W[l], 128 * D * 4));
    CK(cudaMalloc(&g->d_b[l], D * 4));
    CK(cudaMemcpyAsync(g->d_W[l], w.W[l].data(), 128 * D * 4, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(g->d_b[l], w.b[l].data(), D * 4, cudaMemcpyHostToDevice, h->stream));
  }
  {
    const char* simt = getenv("ALZ_GNN_SIMT");   // comparison knob: FP32 FFMA layer instead of wgmma
    g->use_tc = !(simt && simt[0] == '1');
    std::vector<float> can(2 * tc::TN * tc::TK);
    for (int l = 0; l < 2; ++l) {
      for (uint32_t n = 0; n < tc::TN; ++n)
        for (uint32_t k = 0; k < tc::TK; ++k) {
          const float x = w.W[l][k * D + n];               // B[n][k] = W[k][n]
          const float hi = tf32_round(x), lo = tf32_round(x - hi);
          const uint32_t off = tc::op_off(n, k, tc::TN) / 4;
          can[off] = hi;
          can[tc::TN * tc::TK + off] = lo;
        }
      CK(cudaMalloc(&g->d_Wcan[l], 2 * tc::B_BYTES));
      CK(cudaMemcpyAsync(g->d_Wcan[l], can.data(), 2 * tc::B_BYTES, cudaMemcpyHostToDevice, h->stream));
      CK(cudaStreamSynchronize(h->stream));   // `can` is rewritten for the next layer
    }
    CK(cudaFuncSetAttribute(tc::sage_layer_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc::SMEM_TC));
  }
  CK(cudaMalloc(&g->d_a, 132 * 4));
  CK(cudaMemcpyAsync(g->d_a, w.a.data(), 132 * 4, cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));     // the host-side weight vectors die with this frame
  g->c = w.c;
  return ALZ_OK;
}

void alz_internal_free_gnn(alz_handle* h);
// a half-built state never stays published: a failed allocation frees everything and the next call retries
static int gnn_init(alz_handle* h) {
  if (h->gnn) return ALZ_OK;
  const int rc = gnn_init_impl(h);
  if (rc != ALZ_OK) alz_internal_free_gnn(h);
  return rc;
}

void alz_internal_free_gnn(alz_handle* h) {
  alz_gnn_state* g = h->gnn;
  if (!g) return;
  free_row_buffers(g);
  for (int l = 0; l < 2; ++l) { cudaFree(g->d_W[l]); cudaFree(g->d_b[l]); cudaFree(g->d_Wcan[l]); }
  cudaFree(g->d_a); cudaFree(g->d_nv);
  cudaFree(g->d_top_rows); cudaFree(g->d_top_scores); cudaFree(g->d_top_index);
  delete g;
  h->gnn = nullptr;
}

// The CUB calls take int item counts over 2 * n_e node keys: at most 2^30 - 1 rows per pass.
constexpr uint32_t kMaxRows = (1u << 30) - 1u;

// A rollup can have more rows than max_edges (docs/SPEC.md §12). The row- and node-sized buffers and the CUB scratch
// then grow to n + n/2 rows; the weights, the layer path and the node count stay. The state never shrinks. A failed
// growth frees the whole state, as a failed gnn_init does, and the next call rebuilds it at max_edges.
static int gnn_grow(alz_handle* h, uint32_t n_e) {
  alz_gnn_state* g = h->gnn;
  CK(cudaStreamSynchronize(h->stream));   // the last pass may still read the buffers
  free_row_buffers(g);
  if (alloc_row_buffers(g, (uint32_t)std::min<uint64_t>(kMaxRows, (uint64_t)n_e + n_e / 2u)) != cudaSuccess) {
    h->last_err = std::string("alz_gnn_score_rollup: ") + cudaGetErrorString(cudaGetLastError());
    alz_internal_free_gnn(h);
    return ALZ_E_NOMEM;
  }
  return ALZ_OK;
}

// CSR build + 2 layers + scoring over n_e edge rows in device memory: the last flushed window (h->d_out) or a
// rollup's rows (docs/SPEC.md §15). Nothing here waits for the device unless the state grows: the node count lives
// in device memory and every kernel reads it there; buffers and grids are sized by the bound 2 * n_e the host knows.
// Sorts only cover the key bits that can differ.
static int bits_for(uint64_t x) { int b = 1; while (b < 64 && (x >> b) != 0) ++b; return b; }

// a GNN state whose row-sized buffers hold at least n_rows rows
static int gnn_reserve(alz_handle* h, size_t n_rows) {
  const int rc = gnn_init(h);
  if (rc != ALZ_OK) return rc;
  if (n_rows > kMaxRows) return ALZ_E_CAPACITY;
  return n_rows > h->gnn->cap_e ? gnn_grow(h, (uint32_t)n_rows) : ALZ_OK;
}

// scratch_rows: the state holds at least that many rows as well (the top-row selection's scratch, below)
static int gnn_run(alz_handle* h, const alz_edge_out* rows, size_t n_rows, size_t scratch_rows = 0) {
  const int rc = gnn_reserve(h, std::max(n_rows, scratch_rows));
  if (rc != ALZ_OK) return rc;
  alz_gnn_state* g = h->gnn;
  cudaStream_t s = h->stream;
  const uint32_t n_e = (uint32_t)n_rows;
  g->n_e = n_e;
  g->n_v = 0;
  g->n_v_known = n_e == 0;
  if (n_e == 0) { CK(cudaMemsetAsync(g->d_nv, 0, 4, s)); return ALZ_OK; }
  const unsigned grid = (unsigned)h->sms * 4;
  const uint32_t n2 = 2 * n_e;   // bound on the node count
  // nodes: (kind 2 bits << 32 | value 32 bits): 34 key bits
  edge_node_keys_kernel<<<grid, 256, 0, s>>>(rows, n_e, g->d_nk);
  launch_iota(g->d_iota, n2, h->sms, s);
  CK(sort_pairs(g->d_tmp, g->tmp_bytes, g->d_nk, g->d_nk_sorted, g->d_iota, g->d_vals, n2, s, 34));
  CK(launch_unique_sorted(g->d_nk_sorted, n2, g->d_flags, g->d_pos, g->d_nodes, g->d_tmp, g->tmp_bytes, h->sms, s));
  node_count_kernel<<<1, 32, 0, s>>>(g->d_pos, g->d_flags, n2, g->d_nv);
  // stats + CSR by destination (destination index < n2)
  CK(cudaMemsetAsync(g->d_stats, 0, (size_t)n2 * 64, s));
  CK(cudaMemsetAsync(g->d_in_deg, 0, ((size_t)n2 + 1) * 4, s));
  edge_stats_kernel<<<grid, 256, 0, s>>>(rows, n_e, g->d_nodes, g->d_nv, g->d_src_idx, g->d_dst_key, g->d_stats,
                                         g->d_in_deg);
  launch_iota(g->d_iota, n_e, h->sms, s);
  CK(sort_pairs(g->d_tmp, g->tmp_bytes, g->d_dst_key, g->d_dst_sorted, g->d_iota, g->d_sorted_edge, n_e, s,
                bits_for(n2)));
  csr_cols_kernel<<<grid, 256, 0, s>>>(g->d_sorted_edge, g->d_src_idx, n_e, g->d_col);
  CK(exclusive_scan_u32(g->d_tmp, g->tmp_bytes, g->d_in_deg, g->d_rowptr, n2 + 1, s));
  // features, layers, scores
  node_features_kernel<<<grid, 256, 0, s>>>(g->d_nodes, g->d_stats, g->d_nv, g->d_h[0]);
  for (int l = 0; l < 2; ++l) {
    if (g->use_tc) {
      const unsigned tiles = (n2 + tc::TM - 1) / tc::TM;
      tc::sage_layer_tc_kernel<<<std::min<unsigned>(tiles, (unsigned)h->sms), 256, tc::SMEM_TC, s>>>(
          g->d_h[l], g->d_h[l + 1], g->d_rowptr, g->d_col, g->d_Wcan[l], g->d_b[l], g->d_nv);
    } else {
      sage_layer_kernel<<<grid, 256, 0, s>>>(g->d_h[l], g->d_h[l + 1], g->d_rowptr, g->d_col, g->d_W[l], g->d_b[l], g->d_nv);
    }
  }
  edge_score_kernel<<<grid, 256, 0, s>>>(rows, n_e, g->d_src_idx, g->d_dst_key, g->d_h[2], g->d_a, g->c,
                                         g->d_scores);
  h->launches += 12;
  CK(cudaGetLastError());
  return ALZ_OK;
}

// Top anomalous rows (docs/SPEC.md §16): the selection of alz_top.cu over the float32 score bits. Its scratch is the
// pass's: histogram and control block in d_flags, tile counts in d_pos, candidates in d_nk / d_iota, sorted in
// d_nk_sorted / d_vals, CUB in d_tmp. The node keys, h2, the node count and the scores are not touched.
constexpr uint32_t kTopScratchRows = (uint32_t)((top::kWordsBytes / 4 + 1) / 2);   // d_flags holds 2 words per row
// The rows of GNN state the selection of at most k of n scores needs: at most min(k, n) candidates, 2 words of d_pos
// per tile, the histogram and the control block. A pass over n rows already holds n.
static size_t top_scratch_rows(size_t n, uint32_t k) {
  return std::max<size_t>({std::min<size_t>(n, k), n / top::kTile + 1, kTopScratchRows});
}

// The result buffers hold at least m rows: grown on demand, never shrunk; freed with the GNN state
static int top_reserve(alz_handle* h, size_t m) {
  alz_gnn_state* g = h->gnn;
  if (m <= g->top_cap) return ALZ_OK;
  cudaFree(g->d_top_rows); cudaFree(g->d_top_scores); cudaFree(g->d_top_index);
  g->d_top_rows = nullptr; g->d_top_scores = nullptr; g->d_top_index = nullptr;
  g->top_cap = 0;
  const size_t cap = std::max<size_t>(m, 64);
  if (cudaMalloc(&g->d_top_rows, cap * sizeof(alz_edge_out)) != cudaSuccess ||
      cudaMalloc(&g->d_top_scores, cap * 4) != cudaSuccess || cudaMalloc(&g->d_top_index, cap * 4) != cudaSuccess) {
    h->last_err = std::string("top anomalous rows: ") + cudaGetErrorString(cudaGetLastError());
    cudaFree(g->d_top_rows); cudaFree(g->d_top_scores); cudaFree(g->d_top_index);
    g->d_top_rows = nullptr; g->d_top_scores = nullptr; g->d_top_index = nullptr;
    return ALZ_E_NOMEM;
  }
  g->top_cap = cap;
  return ALZ_OK;
}

// The selection over n scores on the device (rows: n rows to gather from, or null). The state holds at least
// top_scratch_rows(n, k) rows. *m_out = results, *above = eligible scores. One wait, for m.
static int top_select(alz_handle* h, const float* scores, uint32_t n, uint32_t k, float min_score,
                      const alz_edge_out* rows, size_t* m_out, uint64_t* above) {
  alz_gnn_state* g = h->gnn;
  *m_out = 0;
  *above = 0;
  const top::Scratch sc{g->d_flags, reinterpret_cast<uint64_t*>(g->d_pos), g->d_nk, g->d_iota, g->d_nk_sorted,
                        g->d_vals, g->d_tmp, g->tmp_bytes};
  const uint32_t* bits = reinterpret_cast<const uint32_t*>(scores);
  uint32_t min_bits;
  memcpy(&min_bits, &min_score, 4);
  top::Ctl<uint32_t> c;
  int rc = top::select_candidates<uint32_t>(h, bits, n, k, min_bits, sc, &c);
  if (rc != ALZ_OK) return rc;
  *above = c.above;
  if (c.m == 0) return ALZ_OK;
  rc = top_reserve(h, c.m);
  if (rc != ALZ_OK) return rc;
  rc = top::select_results<uint32_t>(h, bits, n, c, rows, sc, g->d_top_index,
                                     reinterpret_cast<uint32_t*>(g->d_top_scores), g->d_top_rows);
  if (rc != ALZ_OK) return rc;
  *m_out = c.m;
  return ALZ_OK;
}

// the pass over rows; *n_out = its rows (0 without a GNN state). Caller holds h->mu.
static int gnn_score_locked(alz_handle* h, const alz_edge_out* rows, size_t n_rows, const float** dev_scores,
                            size_t* n_out) {
  CK(cudaSetDevice(h->device));
  int rc = gnn_run(h, rows, n_rows);
  *n_out = h->gnn ? n_rows : 0;
  if (rc != ALZ_OK) return rc;
  if (dev_scores) *dev_scores = h->gnn->d_scores;
  return ALZ_OK;
}

// the pass over the rows the last rollup of `kind` returned (docs/SPEC.md §15)
static int gnn_score_rollup_locked(alz_handle* h, uint32_t kind, const float** dev_scores, size_t* n_out) {
  *n_out = 0;
  const alz_edge_out* rows = nullptr;
  size_t n_rows = 0;
  const int rc = alz_internal_rollup_rows(h, kind, &rows, &n_rows);
  if (rc != ALZ_OK) return rc;
  return gnn_score_locked(h, rows, n_rows, dev_scores, n_out);
}

// scores on the device into `scores` (cap of them) and a wait; the usual cap rule
static int copy_scores(alz_handle* h, const float* d, float* scores, size_t cap, size_t n) {
  if (n > cap) return ALZ_E_CAPACITY;
  if (n) CK(cudaMemcpyAsync(scores, d, n * 4, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return ALZ_OK;
}

extern "C" int alz_gnn_score_device(alz_handle* h, const float** dev_scores, size_t* n_out) {
  if (!h || !n_out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  return gnn_score_locked(h, h->d_out, h->last_n_edges, dev_scores, n_out);
}

extern "C" int alz_gnn_score(alz_handle* h, float* edge_scores, size_t cap, size_t* n_out) {
  if (!h || !n_out || (!edge_scores && cap)) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  const float* d = nullptr;
  int rc = gnn_score_locked(h, h->d_out, h->last_n_edges, &d, n_out);
  if (rc != ALZ_OK) return rc;
  return copy_scores(h, d, edge_scores, cap, *n_out);
}

extern "C" int alz_gnn_score_rollup_device(alz_handle* h, uint32_t kind, const float** dev_scores, size_t* n_out) {
  if (!h || !n_out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  return gnn_score_rollup_locked(h, kind, dev_scores, n_out);
}

extern "C" int alz_gnn_score_rollup(alz_handle* h, uint32_t kind, float* scores, size_t cap, size_t* n_out) {
  if (!h || !n_out || (!scores && cap)) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  const float* d = nullptr;
  int rc = gnn_score_rollup_locked(h, kind, &d, n_out);
  if (rc != ALZ_OK) return rc;
  return copy_scores(h, d, scores, cap, *n_out);
}

// ---- top anomalous rows (docs/SPEC.md §16) ------------------------------------------------------------------------
// the pass over rows, then the selection; *n_out = results, on the device in the GNN state. Caller holds h->mu.
static int gnn_top_locked(alz_handle* h, const alz_edge_out* rows, size_t n_rows, uint32_t k, float min_score,
                          size_t* n_out, alz_top_info* info) {
  CK(cudaSetDevice(h->device));
  int rc = gnn_run(h, rows, n_rows, top_scratch_rows(n_rows, k));
  if (rc != ALZ_OK) return rc;
  uint64_t above = 0;
  rc = top_select(h, h->gnn->d_scores, (uint32_t)n_rows, k, min_score, rows, n_out, &above);
  if (rc != ALZ_OK) return rc;
  if (info) { info->scored = n_rows; info->above = above; }
  return ALZ_OK;
}

// the rows of the last flushed window (rollup false) or of the last rollup of `kind`
static int gnn_top_call(alz_handle* h, bool rollup, uint32_t kind, uint32_t k, float min_score, size_t* n_out,
                        alz_top_info* info) {
  *n_out = 0;
  if (info) *info = alz_top_info{};
  if (k == 0 || std::isnan(min_score)) return ALZ_E_INVAL;
  const alz_edge_out* rows = h->d_out;
  size_t n_rows = h->last_n_edges;
  if (rollup) {
    const int rc = alz_internal_rollup_rows(h, kind, &rows, &n_rows);
    if (rc != ALZ_OK) return rc;
  }
  return gnn_top_locked(h, rows, n_rows, k, min_score, n_out, info);
}

static void top_device_out(alz_handle* h, const alz_edge_out** dev_rows, const float** dev_scores,
                           const uint32_t** dev_index) {
  if (dev_rows) *dev_rows = h->gnn->d_top_rows;
  if (dev_scores) *dev_scores = h->gnn->d_top_scores;
  if (dev_index) *dev_index = h->gnn->d_top_index;
}

// the results into the caller's buffers (each may be null) and a wait; the usual cap rule
static int top_host_out(alz_handle* h, size_t n, alz_edge_out* rows, float* scores, uint32_t* index, size_t cap) {
  if (n > cap) return ALZ_E_CAPACITY;
  alz_gnn_state* g = h->gnn;
  if (n && rows) CK(cudaMemcpyAsync(rows, g->d_top_rows, n * sizeof(alz_edge_out), cudaMemcpyDeviceToHost, h->stream));
  if (n && scores) CK(cudaMemcpyAsync(scores, g->d_top_scores, n * 4, cudaMemcpyDeviceToHost, h->stream));
  if (n && index) CK(cudaMemcpyAsync(index, g->d_top_index, n * 4, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return ALZ_OK;
}

extern "C" int alz_gnn_top(alz_handle* h, uint32_t k, float min_score, alz_edge_out* rows, float* scores,
                           uint32_t* index, size_t cap, size_t* n_out, alz_top_info* info) {
  if (!h || !n_out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  const int rc = gnn_top_call(h, false, 0, k, min_score, n_out, info);
  return rc != ALZ_OK ? rc : top_host_out(h, *n_out, rows, scores, index, cap);
}

extern "C" int alz_gnn_top_device(alz_handle* h, uint32_t k, float min_score, const alz_edge_out** dev_rows,
                                  const float** dev_scores, const uint32_t** dev_index, size_t* n_out,
                                  alz_top_info* info) {
  if (!h || !n_out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  const int rc = gnn_top_call(h, false, 0, k, min_score, n_out, info);
  if (rc == ALZ_OK) top_device_out(h, dev_rows, dev_scores, dev_index);
  return rc;
}

extern "C" int alz_gnn_top_rollup(alz_handle* h, uint32_t kind, uint32_t k, float min_score, alz_edge_out* rows,
                                  float* scores, uint32_t* index, size_t cap, size_t* n_out, alz_top_info* info) {
  if (!h || !n_out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  const int rc = gnn_top_call(h, true, kind, k, min_score, n_out, info);
  return rc != ALZ_OK ? rc : top_host_out(h, *n_out, rows, scores, index, cap);
}

extern "C" int alz_gnn_top_rollup_device(alz_handle* h, uint32_t kind, uint32_t k, float min_score,
                                         const alz_edge_out** dev_rows, const float** dev_scores,
                                         const uint32_t** dev_index, size_t* n_out, alz_top_info* info) {
  if (!h || !n_out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  const int rc = gnn_top_call(h, true, kind, k, min_score, n_out, info);
  if (rc == ALZ_OK) top_device_out(h, dev_rows, dev_scores, dev_index);
  return rc;
}

// debug/test: the selection of alz_gnn_top over n scores in device memory, with the GNN state's scratch (grown to
// top_scratch_rows(n, k) rows when smaller; a growth leaves no pass for alz_gnn_nodes to report). index: the
// results' indices, or null.
extern "C" int alz_debug_top_scores(alz_handle* h, const float* dev_scores, size_t n, uint32_t k, float min_score,
                                    uint32_t* index, size_t cap, size_t* n_out, uint64_t* above) {
  if (!h || !n_out || (!dev_scores && n)) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  *n_out = 0;
  if (above) *above = 0;
  if (k == 0 || std::isnan(min_score)) return ALZ_E_INVAL;
  CK(cudaSetDevice(h->device));
  int rc = gnn_init(h);
  if (rc != ALZ_OK) return rc;
  if (n > kMaxRows) return ALZ_E_CAPACITY;
  const size_t need = top_scratch_rows(n, k);
  const bool grows = need > h->gnn->cap_e;
  rc = gnn_reserve(h, need);
  if (rc != ALZ_OK) return rc;
  if (grows) {                              // the buffers of the last pass are gone
    h->gnn->n_e = h->gnn->n_v = 0;
    h->gnn->n_v_known = true;
    CK(cudaMemsetAsync(h->gnn->d_nv, 0, 4, h->stream));
  }
  uint64_t ab = 0;
  rc = top_select(h, dev_scores, (uint32_t)n, k, min_score, nullptr, n_out, &ab);
  if (rc != ALZ_OK) return rc;
  if (above) *above = ab;
  return top_host_out(h, *n_out, nullptr, nullptr, index, cap);
}

// debug/test: node keys ((kind << 32) | value, ascending) and the layer-2 embeddings of the last GNN pass, over a
// window or a rollup
extern "C" int alz_gnn_nodes(alz_handle* h, uint64_t* node_keys, float* h2, size_t cap, size_t* n_out) {
  if (!h || !n_out) return ALZ_E_INVAL;
  std::lock_guard<std::mutex> g(h->mu);
  if (!h->gnn) return ALZ_E_STATE;
  CK(cudaSetDevice(h->device));
  if (!h->gnn->n_v_known) {   // the pass itself never needed the count on the host
    CK(cudaMemcpyAsync(&h->gnn->n_v, h->gnn->d_nv, 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    h->gnn->n_v_known = true;
  }
  *n_out = h->gnn->n_v;
  if (h->gnn->n_v > cap) return ALZ_E_CAPACITY;
  if (h->gnn->n_v) {
    if (node_keys) CK(cudaMemcpyAsync(node_keys, h->gnn->d_nodes, (size_t)h->gnn->n_v * 8, cudaMemcpyDeviceToHost, h->stream));
    if (h2) CK(cudaMemcpyAsync(h2, h->gnn->d_h[2], (size_t)h->gnn->n_v * D * 4, cudaMemcpyDeviceToHost, h->stream));
  }
  CK(cudaStreamSynchronize(h->stream));
  return ALZ_OK;
}

// SPEC §5 on the host: the same interpolation, float64
extern "C" int alz_edge_quantiles(const alz_edge_out* e, const double* qs, size_t nq, double* out_ns) {
  if (!e || (!qs && nq) || (!out_ns && nq)) return ALZ_E_INVAL;
  uint64_t total = 0;
  for (int b = 0; b < ALZ_NB; ++b) total += e->hist[b];
  auto lo = [](uint32_t b) -> double {
    if (b == 0) return 0.0;
    const double base = (double)(1ull << (8 + b / 2));
    return (b & 1u) ? base * 1.5 : base;
  };
  auto hi = [&](uint32_t b) -> double { return b == ALZ_NB - 1 ? (double)(1ull << 40) : lo(b + 1); };
  for (size_t i = 0; i < nq; ++i) {
    double r = total ? hi(ALZ_NB - 1) : 0.0;
    if (total) {
      const double target = qs[i] * (double)total;
      double cum = 0.0;
      for (uint32_t b = 0; b < ALZ_NB; ++b) {
        const double c = (double)e->hist[b];
        if (c > 0.0 && cum + c >= target) {
          double f = (target - cum) / c;
          if (f < 0.0) f = 0.0;
          r = lo(b) + f * (hi(b) - lo(b));
          break;
        }
        cum += c;
      }
    }
    out_ns[i] = r;
  }
  return ALZ_OK;
}
