// wgmma GEMM / implicit-GEMM 3x3 convolution for sm_90a — warp-specialised, one output tile per CTA, optionally on CTA
// pairs (2-CTA clusters sharing the weight tile by TMA multicast) and with split-K reduced inside a thread-block
// cluster through distributed shared memory.
//
//   grid        : one CTA (or CTA pair) per 128 x BN output tile, M fastest, so CTAs running side by side read the same
//                 weight tile from L2. Cluster split-K: one cluster per output tile, one CTA (pair) per K slice.
//   warp 8      : A producer (one elected lane) — A tile [128 rows x 64 ch] via 4-D NHWC tensor maps (3x3 taps are
//                 shifted boxes; out-of-image reads are zero-filled by TMA = conv padding; stride-2 convs traverse the
//                 input with element strides {1,2,2,1}; up to four A sources are concatenated along K: UNet skip
//                 concat, or hi/lo fp16 splits of one fp32 activation). STAGES-deep mbarrier ring.
//   warp 9      : B producer — B tile [BN x 64] from the K-major weight matrix.
//   warps 0..7  : two consumer warpgroups. Main loop: warpgroup g issues wgmma (M = 64, N = BN, K = 16) for rows
//                 64 g .. 64 g + 63 straight from the swizzled stage buffers, fp32 accumulators in registers. Epilogue:
//                 the accumulators go to a shared-memory tile (the idle ring), then each warp takes accumulator rows
//                 (one row per thread, 32-column chunks), fused alpha/bias/FiLM/residual/activation in registers,
//                 16-byte stores into a swizzled staging tile, TMA store (cp.async.bulk.tensor) of each 32x32 block
//                 to the NHWC output: fp16 (optionally a hi+lo pair) and/or fp32. Outputs whose row pitch TMA cannot
//                 address (N = 3, 4 ...) take a scalar transposed path.
//
//   CTA pair (CG = 2): the two CTAs of a cluster compute the two 128-row halves of a 256 x BN tile. Each loads its own
//   A rows and HALF of the B tile (BN/2 weight rows), multicast into the shared memory of both CTAs, so the L2 -> SM
//   weight traffic per CTA and K step drops from BN to BN/2 rows.
//
//   Cluster split-K: the S (x CG) CTAs of a cluster take K slices of one tile, exchange fp32 partials through
//   distributed shared memory (rows scattered to their owner CTA), and each owner reduces its rows in a fixed order and
//   runs the fused epilogue - no partial planes in HBM, no second kernel, deterministic.
//
//   GroupNorm statistics of the output are written as per-tile partial sums {sum, sum of squares} per channel group
//   (plain stores into [sample][tile][N / group] - no atomics, no zeroing, bit-reproducible); the consumer folds them.
//
// Replaces cuDNN/cuBLAS calls behind nn.Conv2d / nn.Linear in the reference
// (ldm/modules/diffusionmodules/openaimodel.py:204,230,241,519,685; ldm/modules/attention.py:40-60,161-168,233-248).
#pragma once
#include "../../include/sdb200.h"
#include "host.h"
#include "ptx.cuh"

#include <algorithm>
#include <stdlib.h>

namespace sdb {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int A_BYTES = BM * BK * 2;
constexpr int MAX_SRC = 4;
constexpr int EPI_WARPS = 8;          // the two consumer warpgroups (MMA, then epilogue)
constexpr int STG_WARP_BYTES = 8192;  // per epilogue warp: 2 x 4 KB fp32 tiles, or 2 x (2 KB hi + 2 KB lo) fp16 tiles
constexpr int STAGING_BYTES = EPI_WARPS * STG_WARP_BYTES;
constexpr int A_WARP = EPI_WARPS;      // activation (A) tile producer
constexpr int B_WARP = EPI_WARPS + 1;  // weight (B) tile producer
constexpr int GEMM_THREADS = 32 * (EPI_WARPS + 2);

struct TmapPack {
  CUtensorMap a[MAX_SRC];
  CUtensorMap b;     // box {64, BN / CG}
  CUtensorMap o32;   // fp32 output (or the split-K workspace), 5-D [C, W, H, NB, S], box {32, bw, bh, bn, 1}, SWIZZLE_128B
  CUtensorMap o16;   // fp16 output, same geometry, SWIZZLE_64B
  CUtensorMap o16lo; // fp16 low half
  CUtensorMap ows;   // split-K fp32 partial planes [C, W, H, NB, splits]
};

struct GemmArgs {
  int M, N;
  int taps, nsrc;
  int cb[MAX_SRC + 1];  // cumulative 64-channel chunk boundaries of the A sources; cb[nsrc] = chunks per tap
  int H, W, NB;
  int TW, TH, TN, tiles_x, tiles_y;
  int lw, lh;           // log2(TW), log2(TH): the spatial tile sides are powers of two
  int k_iters, iters_per_split, splits;
  int m_tiles, n_tiles;
  int m_units;          // m_tiles for single CTAs, ceil(m_tiles / 2) for CTA pairs
  int csk;              // cluster split-K: the `splits` (x CG) CTAs of a cluster share one output tile
  float alpha;
  const float* bias;
  const float* film;
  int ldf;
  int rows_per_sample;
  const float* residual;
  int ldr;
  __half* out_f16;
  __half* out_f16_lo;
  float* out_f32;
  int ldo;
  float* ws;
  int act;
  float2* stats;    // optional per-tile GroupNorm partials [n_samples][stats_T][N / stats_sg] {sum, sum of squares}
  int stats_halves; // 1: the 128 rows of a tile belong to one sample; 2: rows 0-63 / 64-127 to two samples
  int stats_T;      // partial slots per sample
  int stats_sg;     // channels per statistics entry
  int stats_tps;    // 3x3 geometry: tiles per sample (tiles_x * tiles_y)
  int n_samples;
  int b_static;     // B is a weight matrix: safe to prefetch before griddepcontrol.wait
  int fast;         // outputs go through the TMA-store epilogue
  int bw, bh;       // store box: bw x bh x (32 / (bw*bh)) output pixels per epilogue warp
  int cstride, cshift;   // 3x3 conv: input pixel = cstride * o + tap - 1 + cshift (per axis)
  int film_table;   // 1: rows 0-63 / 64-127 of every tile belong to one sample each, so bias + FiLM fold into a
                    // per-tile shared-memory column table; 0: FiLM is read per row from global memory
  unsigned long long* trace;  // debug: per-CTA phase timestamps (sdb_debug_trace), NULL in production
  int dbg;                    // debug (env SDB_DBG): bit 0 no statistics loop, 1 no statistics flush, 2 no TMA stores,
                              // 3 no B loads, 4 no MMAs, 5 no A loads (timing experiments; results are garbage)
};

// Exact-erf GELU (attention.py:44, F.gelu default) with erf from Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7, far
// below the fp16 rounding of the GEGLU output): one MUFU.RCP + one MUFU.EX2 + 7 FMA instead of erff's branchy ~30.
__device__ __forceinline__ float gelu_erf(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
  float poly = fmaf(fmaf(fmaf(fmaf(1.061405429f, t, -1.453152027f), t, 1.421413741f), t, -0.284496736f), t, 0.254829592f) * t;
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-z * z * 1.4426950408889634f));
  const float erf_abs = fmaf(-poly, e, 1.0f);
  return 0.5f * x * (1.0f + copysignf(erf_abs, x));
}
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + __expf(-x)); }
__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == SDB_ACT_QUICK_GELU) return x * sigmoidf_(1.702f * x);
  if (act == SDB_ACT_SILU) return x * sigmoidf_(x);
  if (act == SDB_ACT_GELU) return gelu_erf(x);
  return x;
}
// The activation of an epilogue of kind KIND: kind 4 carries only the ReLU family (SDB_ACT_RELU, SDB_ACT_LEAKY_RELU),
// so the other kinds compile exactly the code they had before it existed. Both keep a NaN (and -0), as torch.relu and
// F.leaky_relu do: fmaxf(x, 0) would turn a NaN into 0.
template <int KIND>
__device__ __forceinline__ float epi_act(float x, int act) {
  if (KIND == 4) return act == SDB_ACT_RELU ? (x < 0.0f ? 0.0f : x) : (x > 0.0f ? x : 0.2f * x);
  return apply_act(x, act);
}

// Output row of accumulator row r of tile m_tile. 3x3 geometry: a tile is TW x TH x TN output pixels (powers of two, so
// the row decomposes with shifts); its origin (TileGeo) costs three integer divisions and is computed once per tile.
struct TileGeo {
  int gx0, gy0, gn0;
};
__device__ __forceinline__ TileGeo tile_geo(const GemmArgs& p, int m_tile) {
  TileGeo g{0, 0, 0};
  if (p.taps != 1) {
    const int t2 = m_tile / p.tiles_x;
    const int tx = m_tile - t2 * p.tiles_x;
    const int tn = t2 / p.tiles_y;
    const int ty = t2 - tn * p.tiles_y;
    g.gx0 = tx * p.TW;
    g.gy0 = ty * p.TH;
    g.gn0 = tn * p.TN;
  }
  return g;
}
__device__ __forceinline__ bool map_row(const GemmArgs& p, const TileGeo& g, int m_tile, int r, int& out_row) {
  if (p.taps == 1) {
    out_row = m_tile * BM + r;
    return out_row < p.M;
  }
  const int x = r & (p.TW - 1);
  const int y = (r >> p.lw) & (p.TH - 1);
  const int nl = r >> (p.lw + p.lh);
  const int gx = g.gx0 + x, gy = g.gy0 + y, gn = g.gn0 + nl;
  out_row = (gn * p.H + gy) * p.W + gx;
  return gy < p.H && gn < p.NB;
}
__device__ __forceinline__ bool map_row(const GemmArgs& p, int m_tile, int r, int& out_row) {
  return map_row(p, tile_geo(p, m_tile), m_tile, r, out_row);
}

// One element of the fused epilogue (after alpha/bias which are column-only).
template <int KIND = 2>
__device__ __forceinline__ void store_elem(const GemmArgs& p, float x, int orow, int sample, int col, bool finish) {
  if (finish) {
    if (p.film) x += p.film[static_cast<size_t>(sample) * p.ldf + col];
    if (p.residual) x += p.residual[static_cast<size_t>(orow) * p.ldr + col];
    x = epi_act<KIND>(x, p.act);
  }
  size_t o = static_cast<size_t>(orow) * p.ldo + col;
  if (p.out_f32) p.out_f32[o] = x;
  if (p.out_f16) {
    __half h = __float2half_rn(x);
    p.out_f16[o] = h;
    if (p.out_f16_lo) p.out_f16_lo[o] = __float2half_rn(x - __half2float(h));
  }
}

// Drain one 32x32 fp32 chunk that sits in the warp's padded staging tile (row = accumulator row, col = chunk column) to
// global memory with row-contiguous accesses: 16 lanes x 2 columns per row, two rows per instruction.
//   mode 0: fused epilogue (alpha, bias, FiLM, residual, activation)   mode 1: raw split-K partial   mode 2: values
//   already final (GEGLU computed in row layout)
template <int KIND = 2>
__device__ __forceinline__ void drain_chunk(const GemmArgs& p, const float* stage, int lane, int my_row, int my_sample,
                                            bool my_valid, int ocol0, int ncols, int mode, int split) {
  const int l16 = lane & 15, rsel = lane >> 4;
  const int col = ocol0 + 2 * l16;
  const bool c0 = col < ncols, c1 = col + 1 < ncols;
  float b0 = 0.f, b1 = 0.f;
  if (mode == 0 && p.bias) {
    if (c0) b0 = __ldg(p.bias + col);
    if (c1) b1 = __ldg(p.bias + col + 1);
  }
  const bool vec = c1 && ((p.ldo & 1) == 0) && (!p.residual || (p.ldr & 1) == 0) && (!p.film || (p.ldf & 1) == 0);
#pragma unroll 4
  for (int it = 0; it < 16; ++it) {
    const int r = it * 2 + rsel;
    const int orow = __shfl_sync(0xffffffffu, my_row, r);
    const int sample = __shfl_sync(0xffffffffu, my_sample, r);
    const bool valid = __shfl_sync(0xffffffffu, my_valid ? 1 : 0, r) != 0;
    if (!valid || !c0) continue;
    float x0 = stage[r * 33 + 2 * l16];
    float x1 = stage[r * 33 + 2 * l16 + 1];
    if (mode == 1) {
      float* dst = p.ws + (static_cast<size_t>(split) * p.M + orow) * p.N + col;
      if (c1 && (p.N & 1) == 0) {
        *reinterpret_cast<float2*>(dst) = make_float2(x0, x1);
      } else {
        dst[0] = x0;
        if (c1) dst[1] = x1;
      }
      continue;
    }
    if (mode == 0) {
      x0 = x0 * p.alpha + b0;
      x1 = x1 * p.alpha + b1;
    }
    if (!vec) {
      store_elem<KIND>(p, x0, orow, sample, col, mode == 0);
      if (c1) store_elem<KIND>(p, x1, orow, sample, col + 1, mode == 0);
      continue;
    }
    if (mode == 0) {
      if (p.film) {
        float2 f = *reinterpret_cast<const float2*>(p.film + static_cast<size_t>(sample) * p.ldf + col);
        x0 += f.x;
        x1 += f.y;
      }
      if (p.residual) {
        float2 rv = *reinterpret_cast<const float2*>(p.residual + static_cast<size_t>(orow) * p.ldr + col);
        x0 += rv.x;
        x1 += rv.y;
      }
      x0 = epi_act<KIND>(x0, p.act);
      x1 = epi_act<KIND>(x1, p.act);
    }
    const size_t o = static_cast<size_t>(orow) * p.ldo + col;
    if (p.out_f32) *reinterpret_cast<float2*>(p.out_f32 + o) = make_float2(x0, x1);
    if (p.out_f16) {
      __half2 h = __floats2half2_rn(x0, x1);
      *reinterpret_cast<__half2*>(p.out_f16 + o) = h;
      if (p.out_f16_lo) {
        float2 hf = __half22float2(h);
        *reinterpret_cast<__half2*>(p.out_f16_lo + o) = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
      }
    }
  }
}

__device__ __forceinline__ unsigned long long gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// debug trace: word w of this CTA's record (8 words per CTA after an 8-word launch header)
#ifdef SDB_TRACE
#define SDB_TRACE_ENABLED 1
#else
#define SDB_TRACE_ENABLED 0
#endif
#define SDB_TR(w, val)                                                                             \
  do {                                                                                             \
    if (SDB_TRACE_ENABLED && trace && blockIdx.x < 160) trace[8 + blockIdx.x * 8 + (w)] = (val);   \
  } while (0)

// Every CTA computes exactly ONE tile (the grid is one CTA per tile, or per tile and K slice). Once both consumer
// warpgroups are past their last MMA the operand ring is idle, so the fp32 accumulator tile (ring head) and the
// epilogue's staging tiles (ring tail) alias it and the whole shared memory is pipeline during the main loop.
template <int BN, int CG>
struct GemmCfg {
  static constexpr int B_ROWS = BN / CG;            // weight rows of the tile this CTA loads (multicast to the pair)
  static constexpr int B_BYTES = BN * BK * 2;       // every CTA holds the whole B tile
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int ACC_BYTES = BN * BM * 4;
  static constexpr int STAGES = (200 * 1024) / STAGE_BYTES < 10 ? (200 * 1024) / STAGE_BYTES : 10;
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES;
  static constexpr int SMEM = RING_BYTES + 1024;
  static_assert(RING_BYTES >= ACC_BYTES + STAGING_BYTES, "accumulator tile (or cluster split-K receive area) + staging must fit the ring");
};

struct EpiRows {   // the output rows one epilogue warp handles: row per lane + the TMA store box origin
  int row, sample;
  bool valid;
  int sx, sy, sn;
};

// KIND selects what is compiled into an instantiation. Every instruction of an epilogue runs once per CTA from a cold
// instruction cache, so the activation / GEGLU / scalar-store code of the general kernel is compiled out of the
// instantiations the UNet launches most.
//   0 lean   : no activation, TMA-store epilogue, bias / FiLM through the column table  (almost every UNet GEMM)
//   1 geglu  : GEGLU with fp16 output only (the feed-forward up-projection)
//   2 general: everything (activations, scalar-store epilogue for odd widths, per-row FiLM, fp32 + fp16 hi/lo outputs)
//   3 lean + cluster split-K (kind 0 is compiled without the cluster exchange, kind 3 without the single-CTA epilogue)
//   4 general with the ReLU family instead of the other activations (SDB_ACT_RELU / SDB_ACT_LEAKY_RELU; never split:
//     the split-K second pass applies kind 2's activations only)
template <int BN, int CG, int KIND>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_tc_kernel(const __grid_constant__ TmapPack tm, const GemmArgs p) {
  // compile-time specialisation of the descriptor fields the KIND fixes (dead branches fold away)
  const int act = (KIND == 0 || KIND == 3) ? SDB_ACT_NONE : (KIND == 1 ? SDB_ACT_GEGLU : p.act);
  const bool fast = (KIND == 2 || KIND == 4) ? (p.fast != 0) : true;
  const bool film_row = (KIND == 2 || KIND == 4) && p.film && !p.film_table;
  // debug hooks (phase stamps, SDB_DBG switches) exist only in a -DSDB_TRACE build (SDB_BUILD_TRACE=1 python build.py)
  const int dbg = SDB_TRACE_ENABLED ? p.dbg : 0;
  unsigned long long* const trace = SDB_TRACE_ENABLED ? p.trace : nullptr;
  // lean kinds: 0 = no cluster split-K, 3 = cluster split-K; kind 4 never splits
  const int csk = (KIND == 0 || KIND == 4) ? 0 : (KIND == 3 ? 1 : p.csk);
  using Cfg = GemmCfg<BN, CG>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int B_ROWS = Cfg::B_ROWS;
  constexpr int STAGE_BYTES = Cfg::STAGE_BYTES;
  constexpr int NCH = BN / 32;   // 32-column chunks of the accumulator

  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment by offset (keeps the shared address space visible to the compiler: LDS/STS, not generic)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* staging = smem + Cfg::RING_BYTES - STAGING_BYTES;   // aliases the last stages (idle by then)
  // accumulator tile after the main loop, ring head: 4 KB blocks [lane group][chunk] of 32 rows x 32 fp32, row r at
  // r * 128 bytes, 16-byte granule q at (q ^ (r & 7)) << 4 (row-per-lane reads and fragment writes stay conflict-light)
  uint8_t* accbuf = smem;
  __shared__ uint64_t full_bar[STAGES];
  __shared__ uint64_t empty_bar[STAGES];
  // fused GroupNorm statistics: [lane group][column][sum, sum of squares]; one writer per slot per tile, fixed-order
  // fold at the flush, plain stores of the per-tile partials (deterministic)
  __shared__ __align__(16) float colsum[4 * BN * 2];
  // per-tile column constants of the fused epilogue: bias[col] (+ FiLM[sample of the row half][col]), so the chunk
  // loop reads them from shared memory instead of paying a global-load latency per chunk
  __shared__ __align__(16) float coltab[2 * BN];

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  pdl_launch_dependents();   // the next kernel may start its prologue while this one runs
  const long long clk0 = clock64();

  // ---- cluster coordinates. CTA pair: ranks (2k, 2k+1), the even one leads. Cluster split-K: rank / CG = K slice.
  const bool clustered = (CG == 2) || (csk != 0);
  const uint32_t crank = clustered ? cluster_ctarank() : 0u;
  const uint32_t pr = CG == 2 ? (crank & 1u) : 0u;
  const uint32_t lead = crank - pr;
  const int csplit = csk ? static_cast<int>(crank) / CG : 0;
  const int unit0 = csk ? static_cast<int>(blockIdx.x) / (p.splits * CG) : static_cast<int>(blockIdx.x) / CG;
  int m_tile, n_tile, split;
  {
    const int mu = unit0 % p.m_units;
    const int rest = unit0 / p.m_units;
    n_tile = rest % p.n_tiles;
    split = csk ? csplit : rest / p.n_tiles;
    m_tile = mu * CG + static_cast<int>(pr);
  }
  const int it_begin = split * p.iters_per_split;
  const int it_end = min(p.k_iters, it_begin + p.iters_per_split);
  if (trace && threadIdx.x == 0) {
    SDB_TR(0, gtimer());
    if (blockIdx.x == 0) {
      trace[0] = gridDim.x;
      trace[1] = BN + 1000 * CG;
      trace[2] = p.splits + 100 * csk;
      trace[3] = p.k_iters;
      trace[4] = p.M;
      trace[5] = p.N;
      trace[6] = p.taps;
      trace[7] = p.m_units * p.n_tiles * (csk ? 1 : p.splits);
    }
  }

  if (warp == A_WARP && lane == 0) {
    for (int i = 0; i < p.nsrc; ++i) tma_prefetch_desc(&tm.a[i]);
    tma_prefetch_desc(&tm.b);
    if (fast) {
      if (p.ws) tma_prefetch_desc(&tm.ows);
      if (p.out_f32) tma_prefetch_desc(&tm.o32);
      if (p.out_f16) tma_prefetch_desc(&tm.o16);
      if (p.out_f16_lo) tma_prefetch_desc(&tm.o16lo);
    }
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], EPI_WARPS * CG);   // CTA pair: a slot is refilled once the consumers of BOTH CTAs freed it
    }
    fence_barrier_init();
  }
  if (csk && p.stats) {   // lane groups this CTA does not own contribute zeros to its statistics
    for (int i = threadIdx.x; i < 4 * BN * 2; i += GEMM_THREADS) colsum[i] = 0.f;
  }
  if (clustered) cluster_sync_all();   // barrier inits visible to the peer before any remote arrive / multicast
  else __syncthreads();
  if (threadIdx.x == 0 && !(dbg & 64)) SDB_TR(2, clock64() - clk0);

  // ---------------------------------------------------------------- epilogue state and helpers (warps 0..7)
  const int ew = warp & 7;
  const int lg = warp >> 1;      // 32-row lane group of the tile: the rows of warps 2 lg, 2 lg + 1 in the MMA layout
  const int par = warp & 1;      // the two warps of a lane group alternate chunks
  const int et = threadIdx.x;
  uint8_t* stg = staging + ew * STG_WARP_BYTES;
  const bool geglu = (KIND == 0 || KIND == 3 || KIND == 4) ? false : (KIND == 1 ? true : ((p.act == SDB_ACT_GEGLU) && !p.ws));
  constexpr int HALF = BN / 2;
  const int n_chunks = geglu ? HALF / 32 : BN / 32;
  const int n_lim = geglu ? p.N / 2 : p.N;   // output columns that exist
  const bool st32 = p.ws || p.out_f32;       // an fp32 tile is staged in some phase (output or split-K partial)
  const bool st16 = p.out_f16 != nullptr;
  // staging buffers per chunk parity: fp32 tiles 4 KB each; fp16 hi 2 KB + lo 2 KB each (fp32+fp16 together: single)
  const bool dbl = !(st32 && st16);
  const bool split_fast = p.ws && fast;    // raw fp32 partial planes; finished by splitk_epilogue_kernel
  const bool use_tab = fast && !split_fast;
  const bool pre_res = use_tab && !geglu && p.residual != nullptr;
  uint32_t flip = 0;
  bool tr_chunk = false;   // debug (SDB_DBG bit 6): sub-phase stamps of the first chunk of epilogue warp 0

  auto rows_of = [&](int m_tile, int lgx) {
    EpiRows rw;
    const TileGeo geo = tile_geo(p, m_tile);
    rw.valid = map_row(p, geo, m_tile, lgx * 32 + lane, rw.row);
    rw.sample = rw.valid ? rw.row / p.rows_per_sample : 0;
    if (p.taps == 1) {
      rw.sx = m_tile * BM + lgx * 32;
      rw.sy = 0;
      rw.sn = 0;
    } else {
      const int r0 = lgx * 32;
      rw.sx = geo.gx0 + (r0 & (p.TW - 1));
      rw.sy = geo.gy0 + ((r0 >> p.lw) & (p.TH - 1));
      rw.sn = geo.gn0 + (r0 >> (p.lw + p.lh));
    }
    return rw;
  };
  // column table of a tile: bias (+ FiLM of the sample each row half belongs to); all epilogue warps take part
  auto fill_coltab = [&](int m_tile, int n_tile) {
    const TileGeo geo = tile_geo(p, m_tile);
    for (int i = et; i < 2 * BN; i += 32 * EPI_WARPS) {
      const int hsel = i / BN, cl = i - hsel * BN;
      const int col = n_tile * BN + cl;
      float t = 0.f;
      if (col < p.N) {
        if (p.bias) t = __ldg(p.bias + col);
        if (p.film && p.film_table) {
          int prow;
          if (map_row(p, geo, m_tile, hsel * 64, prow))
            t += __ldg(p.film + static_cast<size_t>(prow / p.rows_per_sample) * p.ldf + col);
        }
      }
      coltab[i] = t;
    }
    asm volatile("bar.sync 1, %0;" ::"n"(32 * EPI_WARPS) : "memory");
  };
  // residual rows of one 32-column chunk -> registers (row per thread, 128 contiguous bytes)
  auto load_res = [&](const EpiRows& rw, int n_tile, int c, float4 (&r)[8]) {
    const int oc = n_tile * BN + c * 32;
    if (rw.valid && oc < n_lim) {
      const float4* rp = reinterpret_cast<const float4*>(p.residual + static_cast<size_t>(rw.row) * p.ldr + oc);
#pragma unroll
      for (int q = 0; q < 8; ++q) r[q] = rp[q];
    } else {
#pragma unroll
      for (int q = 0; q < 8; ++q) r[q] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  // one 32-column chunk of this warp's lane group from the accumulator tile: row lg * 32 + lane, columns c*32 .. +31
  auto acc_ld32 = [&](int c, uint32_t (&r)[32]) {
    const uint8_t* blk = accbuf + (lg * NCH + c) * 4096 + lane * 128;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const uint4 t = *reinterpret_cast<const uint4*>(blk + ((q ^ (lane & 7)) << 4));
      r[4 * q] = t.x;
      r[4 * q + 1] = t.y;
      r[4 * q + 2] = t.z;
      r[4 * q + 3] = t.w;
    }
  };
  // fused epilogue + staging + TMA store of one 32x32 chunk held in registers (row per thread); lgx = lane group of
  // the rows (selects the sample half of the column table and the statistics slot)
  auto emit = [&](float (&v)[32], int ocol0, int n_tile, int split, const EpiRows& rw, int lgx, bool fuse,
                  bool raw_partial, const float4 (&res)[8]) {
    if (fuse) {
      // alpha * acc + (bias [+ FiLM]) from the tile's column table; all pointers are 16-byte aligned on this path
      const float4* tp = reinterpret_cast<const float4*>(coltab + (lgx >= 2 ? BN : 0) + (ocol0 - n_tile * BN));
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float4 t = tp[q];
        v[4 * q] = fmaf(v[4 * q], p.alpha, t.x);
        v[4 * q + 1] = fmaf(v[4 * q + 1], p.alpha, t.y);
        v[4 * q + 2] = fmaf(v[4 * q + 2], p.alpha, t.z);
        v[4 * q + 3] = fmaf(v[4 * q + 3], p.alpha, t.w);
      }
      if (film_row) {   // rows of a tile half span several samples: FiLM per row from global
        const float4* fp = reinterpret_cast<const float4*>(p.film + static_cast<size_t>(rw.sample) * p.ldf + ocol0);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          float4 t = __ldg(fp + q);
          v[4 * q] += t.x;
          v[4 * q + 1] += t.y;
          v[4 * q + 2] += t.z;
          v[4 * q + 3] += t.w;
        }
      }
      if (p.residual) {   // prefetched (zeros for rows outside the problem)
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          v[4 * q] += res[q].x;
          v[4 * q + 1] += res[q].y;
          v[4 * q + 2] += res[q].z;
          v[4 * q + 3] += res[q].w;
        }
      }
      if (act != SDB_ACT_NONE) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = epi_act<KIND>(v[j], act);
      }
    }
    if (tr_chunk) SDB_TR(4, clock64() - clk0);
    const bool w32 = raw_partial || p.out_f32;
    const bool w16 = !raw_partial && p.out_f16;
    const bool w16lo = w16 && p.out_f16_lo;
    // staging buffer for this chunk; make sure the TMA store that last read it has finished reading
    const uint32_t bsel = dbl ? (flip & 1) : 0;
    if (lane == 0) {
      if (dbl) tma_store_wait_read<1>();
      else tma_store_wait_read<0>();
    }
    __syncwarp();
    uint8_t* s32 = stg + bsel * 4096;
    uint8_t* s16 = st32 ? stg + 4096 : stg + bsel * 4096;
    uint8_t* s16l = s16 + 2048;
    if (w32) {
#pragma unroll
      for (int q = 0; q < 8; ++q)
        *reinterpret_cast<float4*>(s32 + lane * 128 + ((q ^ (lane & 7)) << 4)) =
            make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
    }
    if (w16) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        __half2 h[4];
        uint4 u, ul;
#pragma unroll
        for (int e = 0; e < 4; ++e) h[e] = __floats2half2_rn(v[8 * q + 2 * e], v[8 * q + 2 * e + 1]);
        u.x = *reinterpret_cast<uint32_t*>(&h[0]);
        u.y = *reinterpret_cast<uint32_t*>(&h[1]);
        u.z = *reinterpret_cast<uint32_t*>(&h[2]);
        u.w = *reinterpret_cast<uint32_t*>(&h[3]);
        const uint32_t off = lane * 64 + ((q ^ ((lane >> 1) & 3)) << 4);
        *reinterpret_cast<uint4*>(s16 + off) = u;
        if (w16lo) {
          __half2 l[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            float2 hf = __half22float2(h[e]);
            l[e] = __floats2half2_rn(v[8 * q + 2 * e] - hf.x, v[8 * q + 2 * e + 1] - hf.y);
          }
          ul.x = *reinterpret_cast<uint32_t*>(&l[0]);
          ul.y = *reinterpret_cast<uint32_t*>(&l[1]);
          ul.z = *reinterpret_cast<uint32_t*>(&l[2]);
          ul.w = *reinterpret_cast<uint32_t*>(&l[3]);
          *reinterpret_cast<uint4*>(s16l + off) = ul;
        }
      }
    }
    fence_proxy_async();
    __syncwarp();
    if (tr_chunk) SDB_TR(5, clock64() - clk0);
    if (lane == 0 && !(dbg & 4)) {
      if (raw_partial) {
        tma_store_5d(&tm.ows, s32, ocol0, rw.sx, rw.sy, rw.sn, split);
      } else {
        if (w32) tma_store_5d(&tm.o32, s32, ocol0, rw.sx, rw.sy, rw.sn, 0);
        if (w16) tma_store_5d(&tm.o16, s16, ocol0, rw.sx, rw.sy, rw.sn, 0);
        if (w16lo) tma_store_5d(&tm.o16lo, s16l, ocol0, rw.sx, rw.sy, rw.sn, 0);
      }
      tma_store_commit();
    }
    if (!raw_partial && p.stats && w32 && !(dbg & 1)) {
      // GroupNorm statistics of the value just produced, from the staged 32x32 fp32 tile: lane l reads the 16-byte
      // granule (l & 7) of rows (l >> 3) + 4k (8 independent LDS.128, conflict-free), two butterfly steps fold the four
      // row classes, lanes 0-7 then hold the sums of columns 4*(l & 7) .. +3 and write the CTA's shared column sums
      // (flushed once per tile)
      const uint32_t vmask = __ballot_sync(0xffffffffu, rw.valid);
      const int gq = lane & 7, rb = lane >> 3;
      float cs[4] = {0.f, 0.f, 0.f, 0.f}, cq[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int r = rb + 4 * k;
        float4 x = *reinterpret_cast<const float4*>(s32 + r * 128 + ((gq ^ (r & 7)) << 4));
        const float keep = ((vmask >> r) & 1u) ? 1.0f : 0.0f;   // rows outside the problem hold bias-only garbage
        x.x *= keep;
        x.y *= keep;
        x.z *= keep;
        x.w *= keep;
        cs[0] += x.x;
        cs[1] += x.y;
        cs[2] += x.z;
        cs[3] += x.w;
        cq[0] = fmaf(x.x, x.x, cq[0]);
        cq[1] = fmaf(x.y, x.y, cq[1]);
        cq[2] = fmaf(x.z, x.z, cq[2]);
        cq[3] = fmaf(x.w, x.w, cq[3]);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        cs[j] += __shfl_xor_sync(0xffffffffu, cs[j], 8);
        cq[j] += __shfl_xor_sync(0xffffffffu, cq[j], 8);
        cs[j] += __shfl_xor_sync(0xffffffffu, cs[j], 16);
        cq[j] += __shfl_xor_sync(0xffffffffu, cq[j], 16);
      }
      if (lane < 8) {
        const int cl = ocol0 - n_tile * BN + 4 * gq;
#pragma unroll
        for (int j = 0; j < 4; ++j)
          *reinterpret_cast<float2*>(&colsum[(lgx * BN + cl + j) * 2]) = make_float2(cs[j], cq[j]);
      }
    }
    if (tr_chunk) SDB_TR(2, clock64() - clk0);
    ++flip;
  };
  // per-tile flush of the fused GroupNorm column sums: one {sum, sum of squares} entry per group of stats_sg
  // channels, stored (not accumulated) into the slot only this tile owns
  auto flush_stats = [&](int m_tile, int n_tile) {
    asm volatile("bar.sync 1, %0;" ::"n"(32 * EPI_WARPS) : "memory");   // all smem column sums of this tile are in
    const int sg = p.stats_sg;
    const int gpt = BN / sg;       // BN % sg == 0 (checked on the host)
    const int E = p.N / sg;
    const int halves = p.stats_halves;
    const TileGeo geo = tile_geo(p, m_tile);
    for (int i = et; i < halves * gpt; i += 32 * EPI_WARPS) {
      const int hsel = i / gpt, g = i - hsel * gpt;
      const int col0 = n_tile * BN + g * sg;
      int prow;
      const bool pv = map_row(p, geo, m_tile, hsel * 64, prow);   // first tile row of this half
      if (pv && col0 < p.N) {
        const int s = prow / p.rows_per_sample;
        int t;
        if (p.taps == 1) t = halves == 1 ? (prow % p.rows_per_sample) / BM : 0;
        else t = m_tile % p.stats_tps;   // spatial tile position (each half of a two-sample tile has its own sample)
        if (csk) t = t * p.splits + csplit;
        float a = 0.f, b = 0.f;
#pragma unroll 1
        for (int j = 0; j < sg; ++j) {
          const int cl = g * sg + j;
          if (halves == 2) {
            a += colsum[((2 * hsel) * BN + cl) * 2] + colsum[((2 * hsel + 1) * BN + cl) * 2];
            b += colsum[((2 * hsel) * BN + cl) * 2 + 1] + colsum[((2 * hsel + 1) * BN + cl) * 2 + 1];
          } else {
            a += (colsum[cl * 2] + colsum[(BN + cl) * 2]) + (colsum[(2 * BN + cl) * 2] + colsum[(3 * BN + cl) * 2]);
            b += (colsum[cl * 2 + 1] + colsum[(BN + cl) * 2 + 1]) +
                 (colsum[(2 * BN + cl) * 2 + 1] + colsum[(3 * BN + cl) * 2 + 1]);
          }
        }
        p.stats[(static_cast<size_t>(s) * p.stats_T + t) * E + col0 / sg] = make_float2(a, b);
      }
    }
  };

  // ---------------------------------------------------------------- roles
  if (warp == A_WARP || warp == B_WARP) {
    // Two single-thread producers: warp 8 streams the activation (A) tiles and arms the stage barriers, warp 9 streams
    // the weight (B) tiles. All loop state is advanced incrementally (no division in the loop). Static weights do not
    // depend on the previous kernel: their producer never executes griddepcontrol.wait and runs ahead under
    // programmatic dependent launch.
    if (elect_one()) {
      // CTA pair: each CTA loads its own 128 A rows and HALF of the B tile, multicast into both CTAs' rings; every CTA
      // arms its own full barrier with the bytes of its A tile and of the whole B tile. Completions of the peer's
      // multicast that overtake the arming just drive the transaction count negative for a moment.
      const bool is_a = warp == A_WARP;
      const uint32_t full_base = smem_u32(&full_bar[0]);
      const uint32_t arm_bytes = ((dbg & 8) ? 0u : Cfg::B_BYTES) + ((dbg & 32) ? 0u : A_BYTES);
      const uint32_t smem_base =
          smem_u32(smem) + (is_a ? 0u : static_cast<uint32_t>(A_BYTES) + pr * static_cast<uint32_t>(B_ROWS * BK * 2));
      const uint16_t mc_mask = static_cast<uint16_t>(3u << lead);   // the two CTAs of this pair
      int s = 0;
      uint32_t ph = 0;
      bool ring_pass = false;
      uint32_t dst = smem_base, bar = full_base;
      const int cpt = p.cb[p.nsrc];
      // A: position inside the (tap, source, 64-channel chunk) sequence, advanced per K step
      int x0 = 0, y0 = 0, n0 = 0;
      if (p.taps == 1) {
        x0 = m_tile * BM;
      } else {
        int tx = m_tile % p.tiles_x;
        int t2 = m_tile / p.tiles_x;
        x0 = tx * p.TW * p.cstride + p.cshift;
        y0 = (t2 % p.tiles_y) * p.TH * p.cstride + p.cshift;
        n0 = (t2 / p.tiles_y) * p.TN;
      }
      int tap = it_begin / cpt, cc = it_begin - tap * cpt;
      int dx = 0, dy = 0;
      if (p.taps == 9) {
        dy = tap / 3 - 1;
        dx = tap - (tap / 3) * 3 - 1;
      }
      int src = 0;
      while (src + 1 < p.nsrc && cc >= p.cb[src + 1]) ++src;
      int cend = p.cb[src + 1];
      int c0 = (cc - p.cb[src]) * BK;
      const CUtensorMap* amap = &tm.a[src];
      int kb = it_begin * BK;
      const int nrow = n_tile * BN + static_cast<int>(pr) * B_ROWS;
      // the dependency wait sits right before this thread's first load: the tile decode / tap geometry above (cold
      // code with integer divisions) overlaps the predecessor's tail instead of following it
      if (is_a || !p.b_static) {
        pdl_wait();
        if (is_a && !(dbg & 64)) SDB_TR(3, clock64() - clk0);
      }
      for (int it = it_begin; it < it_end; ++it) {
        if (ring_pass) mbar_wait_mma(&empty_bar[s], ph ^ 1);   // (first pass over the ring: every slot is free)
        if (is_a) {
          mbar_arrive_expect_tx(&full_bar[s], arm_bytes);
          if (!(dbg & 32)) tma_load_4d_addr(dst, amap, bar, c0, x0 + dx, y0 + dy, n0);
          // next K step: chunk -> source -> tap
          c0 += BK;
          if (++cc == cend) {
            if (cc == cpt) {
              cc = 0;
              src = 0;
              if (++dx == 2) {
                dx = -1;
                ++dy;
              }
            } else {
              ++src;
            }
            c0 = 0;
            cend = p.cb[src + 1];
            amap = &tm.a[src];
          }
        } else {
          if (!(dbg & 8)) {
            if (CG == 2) tma_load_2d_mc_addr(dst, &tm.b, bar, kb, nrow, mc_mask);
            else tma_load_2d_addr(dst, &tm.b, bar, kb, nrow);
          }
          kb += BK;
        }
        dst += STAGE_BYTES;
        bar += 8;
        if (++s == STAGES) {
          s = 0;
          ph ^= 1;
          dst = smem_base;
          bar = full_base;
          ring_pass = true;
        }
      }
    }
    __syncwarp();
    if (csk) {   // the consumers' two cluster barriers around the split-K exchange
      cluster_sync_all();
      cluster_sync_all();
    }
  } else {
    // ---- main loop: two consumer warpgroups, warpgroup g computes rows 64 g .. 64 g + 63 of the tile with wgmma
    // (M = 64, N = BN, K = 16) straight from the swizzled stage buffers; one MMA group stays in flight while the
    // previous stage is handed back to the producers
    pdl_wait();   // residual / FiLM reads and all output writes come after the previous kernel has completed
    float acc[BN / 2];   // rows 16 warp + lane / 4 (+ 8) of the tile, wgmma fragment layout (see wgmma.cuh)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    const uint32_t a_off = static_cast<uint32_t>((warp >> 2) * 64 * 128);
    const uint32_t peer_empty = CG == 2 ? mapa_shared(smem_u32(&empty_bar[0]), crank ^ 1u) : 0u;
    auto release = [&](int s) {
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&empty_bar[s]);
        if (CG == 2) mbar_arrive_cluster(peer_empty + 8u * s);
      }
    };
    int s = 0, prev = -1;
    uint32_t ph = 0;
    wgmma_hold(acc);
    for (int it = it_begin; it < it_end; ++it) {
      mbar_wait_mma(&full_bar[s], ph);
      if (it == it_begin && threadIdx.x == 0 && !(dbg & 64)) SDB_TR(4, clock64() - clk0);
      const uint32_t base = smem_u32(smem) + static_cast<uint32_t>(s * STAGE_BYTES);
      wgmma_fence();
      if (!(dbg & 16)) {
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          WgmmaSS<BN>::mma(acc, wg_desc(base + a_off + 32 * k), wg_desc(base + A_BYTES + 32 * k), 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0) release(prev);
      prev = s;
      if (++s == STAGES) {
        s = 0;
        ph ^= 1;
      }
    }
    wgmma_wait<0>();
    wgmma_hold(acc);
    if (prev >= 0) release(prev);
    if (threadIdx.x == 0 && !(dbg & 64)) SDB_TR(5, clock64() - clk0);
    // both warpgroups are past their last MMA and every load of the tile has landed: the ring is free
    asm volatile("bar.sync 1, %0;" ::"n"(32 * EPI_WARPS) : "memory");

    if (csk) {
      // ---- cluster split-K: exchange + owner epilogue. S K-slices of ONE tile sit in the registers of the cluster's
      // CTAs. Rows are scattered to their owner (K slice o owns lane groups [o * 4/S, (o+1) * 4/S) of its pair-rank's
      // 128 rows) through distributed shared memory into the (now idle) stage ring; the owner sums the S partials in
      // slice order and runs the fused epilogue. The producer warps take part in the two cluster barriers.
      const int S = p.splits;
      const int lgs_per = 4 / S;
      const int n_tasks = lgs_per * n_chunks;   // (owned lane group, chunk) pairs; <= 2 per epilogue warp
      EpiRows rw0{}, rw1{};
      float4 r0[8], r1[8];
      {
        fill_coltab(m_tile, n_tile);
        if (ew < n_tasks) {
          rw0 = rows_of(m_tile, csplit * lgs_per + ew / n_chunks);
          if (p.residual) load_res(rw0, n_tile, ew % n_chunks, r0);
        }
        if (ew + 8 < n_tasks) {
          rw1 = rows_of(m_tile, csplit * lgs_per + (ew + 8) / n_chunks);
          if (p.residual) load_res(rw1, n_tile, (ew + 8) % n_chunks, r1);
        }
      }
      __syncwarp();
      cluster_sync_all();   // every CTA of the cluster is past its main loop: the stage rings are free
      {
        const int owner = lg / lgs_per, lgsub = lg - owner * lgs_per;
        const int rl = 16 * (warp & 1) + (lane >> 2);
        const uint32_t dst = mapa_shared(smem_u32(smem), static_cast<uint32_t>(owner * CG) + pr) +
                             static_cast<uint32_t>((csplit * lgs_per + lgsub) * NCH) * 4096u + rl * 128u + (lane & 1) * 8u;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int q = 2 * (j & 3) + ((lane & 3) >> 1);
          const uint32_t a = dst + static_cast<uint32_t>(j >> 2) * 4096u + ((q ^ (lane >> 2)) << 4);
          st_cluster_f32x2(a, acc[4 * j], acc[4 * j + 1]);
          st_cluster_f32x2(a + 8u * 128u, acc[4 * j + 2], acc[4 * j + 3]);
        }
      }
      __syncwarp();
      cluster_sync_all();   // partials have landed (release / acquire at cluster scope)
      {
#pragma unroll 1
        for (int k = 0; k < 2; ++k) {
          const int t = ew + 8 * k;
          if (t >= n_tasks) break;
          const int lgsub = t / n_chunks, c = t - lgsub * n_chunks;
          float v[32];
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = 0.f;
          for (int src = 0; src < S; ++src) {   // fixed order: deterministic
            const uint8_t* rp = smem + static_cast<size_t>((src * lgs_per + lgsub) * n_chunks + c) * 4096 + lane * 128;
#pragma unroll
            for (int q = 0; q < 8; ++q) {
              const float4 t4 = *reinterpret_cast<const float4*>(rp + ((q ^ (lane & 7)) << 4));
              v[4 * q] += t4.x;
              v[4 * q + 1] += t4.y;
              v[4 * q + 2] += t4.z;
              v[4 * q + 3] += t4.w;
            }
          }
          const int ocol0 = n_tile * BN + c * 32;
          if (ocol0 < n_lim) emit(v, ocol0, n_tile, 0, k ? rw1 : rw0, csplit * lgs_per + lgsub, true, false, k ? r1 : r0);
        }
        if (p.stats) flush_stats(m_tile, n_tile);
      }
    } else {
      // accumulator fragments -> accumulator tile in shared memory (see accbuf), then the row-per-lane epilogue
      {
        const int rl = 16 * (warp & 1) + (lane >> 2);
        uint8_t* blk = accbuf + lg * NCH * 4096 + rl * 128 + (lane & 1) * 8;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int q = 2 * (j & 3) + ((lane & 3) >> 1);
          uint8_t* a = blk + (j >> 2) * 4096 + ((q ^ (lane >> 2)) << 4);
          *reinterpret_cast<float2*>(a) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(a + 8 * 128) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
      }
      const EpiRows rw = rows_of(m_tile, lg);
      if (use_tab) fill_coltab(m_tile, n_tile);   // (its barrier also publishes the accumulator tile)
      else asm volatile("bar.sync 1, %0;" ::"n"(32 * EPI_WARPS) : "memory");
      if (threadIdx.x == 0) SDB_TR(6, clock64() - clk0);
      float* stage = reinterpret_cast<float*>(stg);  // scalar path: [32][33] floats
      if (KIND == 1 || (geglu && fast && !p.out_f32 && !p.out_f16_lo)) {
        // GEGLU tiles (fp16 output): value and gate halves of a chunk are two accumulator reads
#pragma unroll 1
        for (int c = par; c < n_chunks; c += 2) {
          uint32_t xr[32], gr[32], hp[16];
          acc_ld32(c, xr);
          acc_ld32(HALF / 32 + c, gr);
          const float* tb = coltab + c * 32;   // bias of the value half; gate half at +HALF
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const float x0 = fmaf(__uint_as_float(xr[2 * j]), p.alpha, tb[2 * j]);
            const float g0 = fmaf(__uint_as_float(gr[2 * j]), p.alpha, tb[HALF + 2 * j]);
            const float x1 = fmaf(__uint_as_float(xr[2 * j + 1]), p.alpha, tb[2 * j + 1]);
            const float g1 = fmaf(__uint_as_float(gr[2 * j + 1]), p.alpha, tb[HALF + 2 * j + 1]);
            const __half2 h = __floats2half2_rn(x0 * gelu_erf(g0), x1 * gelu_erf(g1));
            hp[j] = *reinterpret_cast<const uint32_t*>(&h);
          }
          const int ocol0 = n_tile * HALF + c * 32;
          if (ocol0 < n_lim) {
            uint8_t* s16 = stg + (flip & 1) * 4096;
            if (lane == 0) tma_store_wait_read<1>();   // the bulk store that last read this staging buffer is done with it
            __syncwarp();
#pragma unroll
            for (int q = 0; q < 4; ++q)
              *reinterpret_cast<uint4*>(s16 + lane * 64 + ((q ^ ((lane >> 1) & 3)) << 4)) =
                  make_uint4(hp[4 * q], hp[4 * q + 1], hp[4 * q + 2], hp[4 * q + 3]);
            fence_proxy_async();
            __syncwarp();
            if (lane == 0 && !(dbg & 4)) {
              tma_store_5d(&tm.o16, s16, ocol0, rw.sx, rw.sy, rw.sn, 0);
              tma_store_commit();
            }
            ++flip;
          }
        }
      } else {
        float4 rcur[8];
        if (pre_res && par < n_chunks) load_res(rw, n_tile, par, rcur);
#pragma unroll 1
        for (int c = par; c < n_chunks; c += 2) {
          float v[32];
          float4 rnxt[8];
          int ocol0;
          const bool has_next = pre_res && (c + 2 < n_chunks);
          if (geglu) {
            uint32_t xr[32], gr[32];
            acc_ld32(c, xr);
            acc_ld32(HALF / 32 + c, gr);
            const float* tb = coltab + c * 32;   // bias of the value half; gate half at +HALF
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              const float x = fmaf(__uint_as_float(xr[j]), p.alpha, tb[j]);
              const float g = fmaf(__uint_as_float(gr[j]), p.alpha, tb[HALF + j]);
              v[j] = x * gelu_erf(g);
            }
            ocol0 = n_tile * HALF + c * 32;
          } else {
            uint32_t rr[32];
            if (has_next) load_res(rw, n_tile, c + 2, rnxt);   // next chunk's residual rows: in flight across this chunk's work
            acc_ld32(c, rr);
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(rr[j]);
            ocol0 = n_tile * BN + c * 32;
          }
          tr_chunk = trace && (dbg & 64) && threadIdx.x == 0 && c == par;
          if (tr_chunk) SDB_TR(3, clock64() - clk0);
          if (!fast) {
            // scalar transposed path (row pitch not TMA-addressable); split-K partials are finished by
            // splitk_epilogue_kernel on this path
#pragma unroll
            for (int j = 0; j < 32; ++j) stage[lane * 33 + j] = v[j];
            __syncwarp();
            drain_chunk<KIND>(p, stage, lane, rw.row, rw.sample, rw.valid, ocol0, geglu ? p.N / 2 : p.N,
                        geglu ? 2 : (p.ws ? 1 : 0), split);
            __syncwarp();
            continue;
          }
          if (ocol0 < n_lim) emit(v, ocol0, n_tile, split, rw, lg, !geglu && !split_fast, split_fast, rcur);
          if (has_next) {
#pragma unroll
            for (int q = 0; q < 8; ++q) rcur[q] = rnxt[q];
          }
        }
      }
      if (p.stats && !p.ws && !(dbg & 2)) flush_stats(m_tile, n_tile);
    }
  }

  if (warp < EPI_WARPS) {
    // smem may be released once the bulk stores have READ it; their global writes complete with the grid
    if (lane == 0) tma_store_wait_read<0>();
    if (threadIdx.x == 0) SDB_TR(7, clock64() - clk0);
  }
  __syncwarp();
  if (clustered) cluster_sync_all();   // the peer's multicast writes / remote arrives into this CTA are done
  if (threadIdx.x == 0) SDB_TR(1, gtimer());
}

// split-K second pass (workspace mode): sum the fp32 partial planes and apply the fused epilogue. Block = 32 rows x
// (4 * CQ) columns (thread: 4 adjacent columns of rows ty, ty+8, ty+16, ty+24); the GroupNorm column sums of the
// result fold through shared memory into per-(32-row block, channel group) partial entries (plain stores).
template <int CQ>
__global__ void __launch_bounds__(CQ * 8) splitk_epilogue_kernel(const GemmArgs p, int splits) {
  constexpr int CB = CQ * 4;
  __shared__ float red[8][CB][2];
  pdl_launch_dependents();
  const int tx = threadIdx.x % CQ, ty = threadIdx.x / CQ;
  const int col = blockIdx.x * CB + tx * 4;
  const size_t plane = static_cast<size_t>(p.M) * p.N;
  float cs[4] = {0.f, 0.f, 0.f, 0.f}, cq[4] = {0.f, 0.f, 0.f, 0.f};
  float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
  if (col < p.N && p.bias) bv = *reinterpret_cast<const float4*>(p.bias + col);   // weights: before the dependency wait
  pdl_wait();
  if (col < p.N) {
    // All four rows of a thread are summed in ONE loop over the planes, before anything is stored: the output pointers
    // may alias the workspace as far as the compiler knows, so a row-by-row version reloads only after the previous
    // row's stores - four rows x (planes / 4) dependent L2 round trips (10 us for 12 planes of a 128 x 1280 output).
    // Here: planes / 4 round trips of sixteen loads each.
    float4 accs[4];
    const float* srcs[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int row = min(blockIdx.y * 32 + ty + 8 * i, p.M - 1);   // rows past M: a valid address, result unused
      srcs[i] = p.ws + static_cast<size_t>(row) * p.N + col;
      accs[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll 1
    for (int sp0 = 0; sp0 < splits; sp0 += 4) {   // sixteen 16-byte loads in flight per thread; plane order: deterministic
      float4 t[4][4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (sp0 + u < splits) {
#pragma unroll
          for (int i = 0; i < 4; ++i) t[u][i] = __ldcg(reinterpret_cast<const float4*>(srcs[i] + (sp0 + u) * plane));
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (sp0 + u < splits) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            accs[i].x += t[u][i].x;
            accs[i].y += t[u][i].y;
            accs[i].z += t[u][i].z;
            accs[i].w += t[u][i].w;
          }
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int row = blockIdx.y * 32 + ty + 8 * i;
      if (row >= p.M) continue;
      const float4 acc = accs[i];
      float x[4] = {acc.x * p.alpha + bv.x, acc.y * p.alpha + bv.y, acc.z * p.alpha + bv.z, acc.w * p.alpha + bv.w};
      const int sample = row / p.rows_per_sample;
      if (p.film) {
        float4 f = *reinterpret_cast<const float4*>(p.film + static_cast<size_t>(sample) * p.ldf + col);
        x[0] += f.x; x[1] += f.y; x[2] += f.z; x[3] += f.w;
      }
      if (p.residual) {
        float4 r = *reinterpret_cast<const float4*>(p.residual + static_cast<size_t>(row) * p.ldr + col);
        x[0] += r.x; x[1] += r.y; x[2] += r.z; x[3] += r.w;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        x[j] = apply_act(x[j], p.act);
        cs[j] += x[j];
        cq[j] = fmaf(x[j], x[j], cq[j]);
      }
      const size_t o = static_cast<size_t>(row) * p.ldo + col;
      if (p.out_f32) *reinterpret_cast<float4*>(p.out_f32 + o) = make_float4(x[0], x[1], x[2], x[3]);
      if (p.out_f16) {
        __half2 h0 = __floats2half2_rn(x[0], x[1]), h1 = __floats2half2_rn(x[2], x[3]);
        uint2 u;
        u.x = *reinterpret_cast<uint32_t*>(&h0);
        u.y = *reinterpret_cast<uint32_t*>(&h1);
        *reinterpret_cast<uint2*>(p.out_f16 + o) = u;
        if (p.out_f16_lo) {
          float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
          __half2 l0 = __floats2half2_rn(x[0] - f0.x, x[1] - f0.y), l1 = __floats2half2_rn(x[2] - f1.x, x[3] - f1.y);
          uint2 w;
          w.x = *reinterpret_cast<uint32_t*>(&l0);
          w.y = *reinterpret_cast<uint32_t*>(&l1);
          *reinterpret_cast<uint2*>(p.out_f16_lo + o) = w;
        }
      }
    }
  }
  if (p.stats) {   // rows of one block belong to one sample (rows_per_sample % 32 == 0, checked on the host)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      red[ty][tx * 4 + j][0] = cs[j];
      red[ty][tx * 4 + j][1] = cq[j];
    }
    __syncthreads();
    const int sg = p.stats_sg;
    const int g = threadIdx.x;                       // channel group inside this column block (CB % sg == 0)
    const int c0 = blockIdx.x * CB + g * sg;
    const int row0 = blockIdx.y * 32;
    if (g < CB / sg && c0 < p.N && row0 < p.M) {
      float a = 0.f, b = 0.f;
      for (int j = 0; j < sg; ++j) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          a += red[k][g * sg + j][0];
          b += red[k][g * sg + j][1];
        }
      }
      const int sample = row0 / p.rows_per_sample;
      const int t = (row0 - sample * p.rows_per_sample) / 32;
      p.stats[(static_cast<size_t>(sample) * p.stats_T + t) * (p.N / sg) + c0 / sg] = make_float2(a, b);
    }
  }
}

// scalar variant for outputs whose width is not a multiple of 4 (no fused statistics)
static __global__ void __launch_bounds__(256) splitk_epilogue_scalar_kernel(const GemmArgs p, int splits) {
  const size_t total = static_cast<size_t>(p.M) * p.N;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int row = static_cast<int>(idx / p.N);
    const int col = static_cast<int>(idx - static_cast<size_t>(row) * p.N);
    float acc = 0.f;
    for (int sp = 0; sp < splits; ++sp) acc += p.ws[static_cast<size_t>(sp) * total + idx];
    float x = acc * p.alpha + (p.bias ? p.bias[col] : 0.f);
    store_elem(p, x, row, row / p.rows_per_sample, col, true);
  }
}

// one CTA per tile (and K slice); CTA pairs and cluster split-K launch as thread-block clusters
template <int BN, int CG, int KIND>
static int launch_gemm(const TmapPack& tm, const GemmArgs& p, cudaStream_t st) {
  using Cfg = GemmCfg<BN, CG>;
  auto kern = gemm_tc_kernel<BN, CG, KIND>;
  static bool configured = false;
  if (!configured) {
    SDB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM));
    configured = true;
  }
  const int grid = p.m_units * p.n_tiles * p.splits * CG;
  const int cluster = p.csk ? p.splits * CG : CG;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = Cfg::SMEM;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (pdl_enabled()) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  if (cluster > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = cluster;
    attr[na].val.clusterDim.y = 1;
    attr[na].val.clusterDim.z = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  SDB_CUDA(cudaLaunchKernelEx(&cfg, kern, tm, p));
  SDB_LAUNCH_CHECK();
  return 0;
}

// all tile shapes of one KIND (one translation unit per KIND: gemm_k0.cu .. gemm_k4.cu)
template <int KIND>
static int launch_gemm_kind(int bn, int cg, const TmapPack& tm, const GemmArgs& p, cudaStream_t st) {
  if (cg == 2) {
    switch (bn) {
      case 128: return launch_gemm<128, 2, KIND>(tm, p, st);
      case 160:
        if (KIND != 1) return launch_gemm<160, 2, KIND>(tm, p, st);
        break;
      case 256: return launch_gemm<256, 2, KIND>(tm, p, st);
      default: break;
    }
    SDB_CHECK(false, "sdb_gemm: CTA pairs need block_n 128, 160 or 256 (got %d)", bn);
  }
  switch (bn) {
    case 32:
      if (KIND != 1) return launch_gemm<32, 1, KIND>(tm, p, st);
      break;
    case 64:
      if (KIND != 1) return launch_gemm<64, 1, KIND>(tm, p, st);
      break;
    case 128: return launch_gemm<128, 1, KIND>(tm, p, st);
    case 160:
      if (KIND != 1) return launch_gemm<160, 1, KIND>(tm, p, st);
      break;
    case 256: return launch_gemm<256, 1, KIND>(tm, p, st);
    default: break;
  }
  SDB_CHECK(false, "sdb_gemm: unsupported block_n %d for this epilogue kind", bn);
}
int launch_gemm_kind0(int bn, int cg, const TmapPack& tm, const GemmArgs& p, cudaStream_t st);
int launch_gemm_kind1(int bn, int cg, const TmapPack& tm, const GemmArgs& p, cudaStream_t st);
int launch_gemm_kind2(int bn, int cg, const TmapPack& tm, const GemmArgs& p, cudaStream_t st);
int launch_gemm_kind3(int bn, int cg, const TmapPack& tm, const GemmArgs& p, cudaStream_t st);
int launch_gemm_kind4(int bn, int cg, const TmapPack& tm, const GemmArgs& p, cudaStream_t st);

}  // namespace sdb
