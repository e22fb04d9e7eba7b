// GroupNorm(32)[+SiLU] over (optionally concatenated) NHWC fp32 activations, LayerNorm, row softmax.
// HBM/L2-bound streaming kernels: fp32 statistics (fp64 cross-block combine), fp16 operand output for the
// tensor-core kernels. Reference: ldm/modules/diffusionmodules/util.py:199-216 (GroupNorm32, fp32),
// ldm/modules/attention.py:76-77 (Normalize, eps 1e-6), :203-205 (LayerNorm), ldm/modules/diffusionmodules/model.py:38-39.
#include "../../include/sdb200.h"
#include "host.h"
#include "ptx.cuh"
#include <cuda_fp16.h>

namespace sdb {

constexpr int GN_THREADS = 256;
constexpr int GN_CPT = 12;      // channels per thread of the statistics pass: C <= 3072
constexpr int GN_MAX_CPT = 14;  // C <= 3584 (the retrieval-augmented UNet's widest skip concat) takes a 14-channel variant

constexpr int GN_MAX_SLABS = 128;

// pass 1: per (sample, group) mean / rstd. grid = (slabs, nb). Thread t owns channel (t % cw) [+ k*cw] of rows
// (t / cw) + k * (256 / cw): consecutive threads read consecutive channels (coalesced), four rows in flight per
// thread. Sums are taken around a per-(sample, group) pivot (x at row 0, the group's first channel) that every block
// reads alike, so a mean far from zero does not cancel away the variance: fp32 E[(x-p)^2] - E[x-p]^2 keeps its
// accuracy where E[x^2] - E[x]^2 would lose (mean/std)^2 of it. Each row lane parks its per-channel partials in its
// own shared-memory slot and a fixed-order sum combines them (bit-reproducible: shared-memory float atomics from
// more than two lanes would add in scheduling order); each group is reduced by one warp and written as per-block
// partials; the last block of each sample (ticket counter) folds the partials in fp64 and publishes mean / rstd.
// Three resident blocks per SM (80 registers, no spills).
template <int CPT>
__global__ void __launch_bounds__(GN_THREADS, 3)
    gn_stats_kernel(const float* __restrict__ x0, const float* __restrict__ x1, int c0, int c1, int hw, int groups,
                    int rows_per_block, int cw, float eps, float* __restrict__ partial,
                    unsigned int* __restrict__ counter, float* __restrict__ meanrstd) {
  extern __shared__ float gn_smem[];  // [2][rstep][C] partials | [C] pivot of each channel's group
  __shared__ bool is_last;
  __shared__ float piv[64];
  const int C = c0 + c1;
  const int cpg = C / groups;
  const int n = blockIdx.y;
  const int slabs = gridDim.x;
  const int r0 = blockIdx.x * rows_per_block;
  const int r1 = min(hw, r0 + rows_per_block);
  const int tc = threadIdx.x % cw;
  const int tr = threadIdx.x / cw;
  const int rstep = GN_THREADS / cw;
  float* sum_s = gn_smem;
  float* sum_q = gn_smem + rstep * C;
  float* piv_c = gn_smem + 2 * rstep * C;
  const size_t base = static_cast<size_t>(n) * hw;
  if (threadIdx.x < groups) {
    const int c = threadIdx.x * cpg;
    piv[threadIdx.x] = c < c0 ? x0[base * c0 + c] : x1[base * c1 + (c - c0)];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += GN_THREADS) piv_c[c] = piv[c / cpg];
  __syncthreads();
  float s[CPT], q[CPT];
#pragma unroll
  for (int j = 0; j < CPT; ++j) s[j] = q[j] = 0.f;
  for (int r = r0 + tr; r < r1; r += 4 * rstep) {
#pragma unroll
    for (int j = 0; j < CPT; ++j) {
      const int c = tc + j * cw;
      if (c < C) {
        const float p = piv_c[c];
        float v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int rr = r + u * rstep;
          v[u] = 0.f;
          if (rr < r1) v[u] = (c < c0 ? x0[(base + rr) * c0 + c] : x1[(base + rr) * c1 + (c - c0)]) - p;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          s[j] += v[u];
          q[j] += v[u] * v[u];
        }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < CPT; ++j) {
    const int c = tc + j * cw;
    if (c < C) {
      sum_s[tr * C + c] = s[j];
      sum_q[tr * C + c] = q[j];
    }
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* my_part = partial + (static_cast<size_t>(n) * GN_MAX_SLABS + blockIdx.x) * groups * 2;
  for (int g = warp; g < groups; g += GN_THREADS / 32) {
    float a = 0.f, b = 0.f;
    for (int c = lane; c < cpg; c += 32) {
      for (int k = 0; k < rstep; ++k) {
        a += sum_s[k * C + g * cpg + c];
        b += sum_q[k * C + g * cpg + c];
      }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      a += __shfl_xor_sync(0xffffffffu, a, o);
      b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    if (lane == 0) {
      my_part[g * 2] = a;
      my_part[g * 2 + 1] = b;
    }
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(&counter[n], 1u) == static_cast<unsigned>(slabs - 1);
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  const double cnt = static_cast<double>(hw) * cpg;
  for (int g = warp; g < groups; g += GN_THREADS / 32) {
    double a = 0.0, b = 0.0;
    for (int sl = lane; sl < slabs; sl += 32) {
      const float* pp = partial + ((static_cast<size_t>(n) * GN_MAX_SLABS + sl) * groups + g) * 2;
      a += static_cast<double>(__ldcg(pp));
      b += static_cast<double>(__ldcg(pp + 1));
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      a += __shfl_xor_sync(0xffffffffu, a, o);
      b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    if (lane == 0) {
      const double d = a / cnt;   // mean - pivot
      double v = b / cnt - d * d;
      if (v < 0) v = 0;
      meanrstd[(static_cast<size_t>(n) * groups + g) * 2] = static_cast<float>(static_cast<double>(piv[g]) + d);
      meanrstd[(static_cast<size_t>(n) * groups + g) * 2 + 1] = static_cast<float>(1.0 / sqrt(v + static_cast<double>(eps)));
    }
  }
}

// Fold of the per-tile statistics partials when a sample has many tile slots (large images: one slot per 128 output
// pixels): grid = (groups, nb); a block sums every entry / slot of its group in a fixed thread-strided order (fp64),
// tree-reduces and publishes mean / rstd, so the apply blocks read 8 bytes per group instead of the whole slot list.
__global__ void __launch_bounds__(GN_THREADS)
    gn_fold_kernel(const float2* __restrict__ cs0, int T0, const float2* __restrict__ cs1, int T1, int sg, int c0, int c1,
                   int groups, int hw, float eps, float* __restrict__ meanrstd) {
  __shared__ double ra[GN_THREADS / 32], rb[GN_THREADS / 32];
  const int g = blockIdx.x, n = blockIdx.y;
  const int C = c0 + c1, cpg = C / groups;
  pdl_launch_dependents();
  pdl_wait();
  double a = 0.0, b = 0.0;
  for (int c = g * cpg; c < (g + 1) * cpg; c += sg) {
    const bool first = c < c0;
    const float2* src = first ? cs0 : cs1;
    const int T = first ? T0 : T1;
    const int E = (first ? c0 : c1) / sg;
    const int e = (first ? c : c - c0) / sg;
    for (int t = threadIdx.x; t < T; t += GN_THREADS) {
      const float2 v = src[(static_cast<size_t>(n) * T + t) * E + e];
      a += static_cast<double>(v.x);
      b += static_cast<double>(v.y);
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  if ((threadIdx.x & 31) == 0) {
    ra[threadIdx.x >> 5] = a;
    rb[threadIdx.x >> 5] = b;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    a = 0.0;
    b = 0.0;
    for (int k = 0; k < GN_THREADS / 32; ++k) {
      a += ra[k];
      b += rb[k];
    }
    const double cnt = static_cast<double>(hw) * cpg;
    const double m = a / cnt;
    double v = b / cnt - m * m;
    if (v < 0) v = 0;
    meanrstd[(static_cast<size_t>(n) * groups + g) * 2] = static_cast<float>(m);
    meanrstd[(static_cast<size_t>(n) * groups + g) * 2 + 1] = static_cast<float>(1.0 / sqrt(v + static_cast<double>(eps)));
  }
}

// pass 2: normalise (+SiLU) -> fp16, optional raw fp16 cast. grid = (slabs, nb); dynamic smem: float2[C] per-channel
// {scale, shift} so the streaming loop is one FMA (+ SiLU) per element. The element loop keeps four independent 16-byte
// loads in flight per thread and walks (row, channel quad) incrementally (no integer division per element).
__device__ __forceinline__ float silu_fast(float y) { return __fdividef(y, 1.0f + __expf(-y)); }

__global__ void __launch_bounds__(GN_THREADS)
    gn_apply_kernel(const float* __restrict__ x0, const float* __restrict__ x1, int c0, int c1, int hw, int groups,
                    int rows_per_block, const float* __restrict__ meanrstd, const float* __restrict__ gamma,
                    const float* __restrict__ beta, float eps, int silu, __half* __restrict__ out,
                    __half* __restrict__ raw, __half* __restrict__ out_lo, __half* __restrict__ raw_lo,
                    const float2* __restrict__ cs0, int T0, const float2* __restrict__ cs1, int T1, int sg) {
  extern __shared__ float2 gn_ab[];   // [C] {rstd * gamma, beta - mean * rstd * gamma}
  const int C = c0 + c1;
  const int cpg = C / groups;
  const int n = blockIdx.y;
  __shared__ float mean_s[64], rstd_s[64];
  pdl_launch_dependents();
  // gamma / beta are weights: park them in the table before the dependency wait (one L2 round trip off the chain)
  for (int c = threadIdx.x; c < C; c += GN_THREADS) gn_ab[c] = make_float2(__ldg(gamma + c), __ldg(beta + c));
  pdl_wait();
  if (cs0) {
    // per-tile partial {sum, sum of squares} per sg-channel entry, stored by the producing GEMM epilogues
    // (sdb_gemm.stats_out, [sample][T][C / sg]): fold the entries and tile slots of each group in a fixed order, fp64
    // (8 lanes per group, then a butterfly: the result does not depend on scheduling)
    const int g = threadIdx.x >> 3, sub = threadIdx.x & 7;
    if (g < groups) {
      double a = 0.0, b = 0.0;
      for (int c = g * cpg; c < (g + 1) * cpg; c += sg) {
        const bool first = c < c0;
        const float2* src = first ? cs0 : cs1;
        const int T = first ? T0 : T1;
        const int E = (first ? c0 : c1) / sg;
        const int e = (first ? c : c - c0) / sg;
        for (int t = sub; t < T; t += 8) {
          const float2 v = src[(static_cast<size_t>(n) * T + t) * E + e];
          a += static_cast<double>(v.x);
          b += static_cast<double>(v.y);
        }
      }
#pragma unroll
      for (int o = 4; o; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
      }
      if (sub == 0) {
        const double cnt = static_cast<double>(hw) * cpg;
        double m = a / cnt;
        double v = b / cnt - m * m;
        if (v < 0) v = 0;
        mean_s[g] = static_cast<float>(m);
        rstd_s[g] = static_cast<float>(1.0 / sqrt(v + static_cast<double>(eps)));
      }
    }
  } else if (threadIdx.x < groups) {
    mean_s[threadIdx.x] = meanrstd[(static_cast<size_t>(n) * groups + threadIdx.x) * 2];
    rstd_s[threadIdx.x] = meanrstd[(static_cast<size_t>(n) * groups + threadIdx.x) * 2 + 1];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += GN_THREADS) {   // each thread rewrites the entries it parked above
    const int g = c / cpg;
    const float2 gb = gn_ab[c];
    const float a = rstd_s[g] * gb.x;
    gn_ab[c] = make_float2(a, fmaf(-mean_s[g], a, gb.y));
  }
  __syncthreads();
  const int r0 = blockIdx.x * rows_per_block;
  const int r1 = min(hw, r0 + rows_per_block);
  const int c4n = C >> 2;  // C is a multiple of 4 (checked on the host); c0 too
  const int total = (r1 - r0) * c4n;
  // position of element quad i = tid + k * GN_THREADS: (row, quad) advanced by (dr, dq) with one conditional carry
  const int dr = GN_THREADS / c4n, dq = GN_THREADS - dr * c4n;
  int row = r0 + threadIdx.x / c4n, quad = threadIdx.x % c4n;
  const size_t base = static_cast<size_t>(n) * hw;
  constexpr int U = 4;
  for (int i = threadIdx.x; i < total; i += U * GN_THREADS) {
    float4 v[U];
    int rr[U], qq[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      rr[u] = row;
      qq[u] = quad;
      if (i + u * GN_THREADS < total) {
        const int c = quad * 4;
        const size_t r = base + row;
        v[u] = c < c0 ? *reinterpret_cast<const float4*>(x0 + r * c0 + c)
                      : *reinterpret_cast<const float4*>(x1 + r * c1 + (c - c0));
      }
      row += dr;
      quad += dq;
      if (quad >= c4n) {
        quad -= c4n;
        ++row;
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (i + u * GN_THREADS >= total) break;
      const int c = qq[u] * 4;
      const size_t o = (base + rr[u]) * C + c;
      const float4 ab01 = *reinterpret_cast<const float4*>(&gn_ab[c]);       // {a0, b0, a1, b1}
      const float4 ab23 = *reinterpret_cast<const float4*>(&gn_ab[c + 2]);   // {a2, b2, a3, b3}
      const float in[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
      float y[4] = {fmaf(in[0], ab01.x, ab01.y), fmaf(in[1], ab01.z, ab01.w), fmaf(in[2], ab23.x, ab23.y),
                    fmaf(in[3], ab23.z, ab23.w)};
      if (silu) {
#pragma unroll
        for (int j = 0; j < 4; ++j) y[j] = silu_fast(y[j]);
      }
      __half2 h0 = __floats2half2_rn(y[0], y[1]), h1 = __floats2half2_rn(y[2], y[3]);
      uint2 w;
      w.x = *reinterpret_cast<uint32_t*>(&h0);
      w.y = *reinterpret_cast<uint32_t*>(&h1);
      *reinterpret_cast<uint2*>(out + o) = w;
      if (out_lo) {  // low halves of the hi/lo operand split: fp16(y - float(fp16(y)))
        float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
        __half2 l0 = __floats2half2_rn(y[0] - f0.x, y[1] - f0.y), l1 = __floats2half2_rn(y[2] - f1.x, y[3] - f1.y);
        w.x = *reinterpret_cast<uint32_t*>(&l0);
        w.y = *reinterpret_cast<uint32_t*>(&l1);
        *reinterpret_cast<uint2*>(out_lo + o) = w;
      }
      if (raw) {
        __half2 r0h = __floats2half2_rn(in[0], in[1]), r1h = __floats2half2_rn(in[2], in[3]);
        w.x = *reinterpret_cast<uint32_t*>(&r0h);
        w.y = *reinterpret_cast<uint32_t*>(&r1h);
        *reinterpret_cast<uint2*>(raw + o) = w;
        if (raw_lo) {
          float2 f0 = __half22float2(r0h), f1 = __half22float2(r1h);
          __half2 l0 = __floats2half2_rn(in[0] - f0.x, in[1] - f0.y), l1 = __floats2half2_rn(in[2] - f1.x, in[3] - f1.y);
          w.x = *reinterpret_cast<uint32_t*>(&l0);
          w.y = *reinterpret_cast<uint32_t*>(&l1);
          *reinterpret_cast<uint2*>(raw_lo + o) = w;
        }
      }
    }
  }
}

// LayerNorm: one warp per row, row held in registers. Vector variant (C a multiple of 64): NP float2 per lane,
// coalesced 8-byte loads / 4-byte fp16x2 stores; the scalar variant covers every other width.
template <int NP>
__global__ void __launch_bounds__(256)
    layernorm_v2_kernel(const float* __restrict__ x, int rows, int C, const float* __restrict__ gamma,
                        const float* __restrict__ beta, float eps, __half* __restrict__ out, float* __restrict__ out32) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  pdl_launch_dependents();
  // gamma / beta are weights: fetch them while the producer of x drains
  float2 gm[NP], bt[NP];
#pragma unroll
  for (int j = 0; j < NP; ++j) {
    gm[j] = __ldg(reinterpret_cast<const float2*>(gamma) + lane + j * 32);
    bt[j] = __ldg(reinterpret_cast<const float2*>(beta) + lane + j * 32);
  }
  pdl_wait();
  if (warp >= rows) return;
  const float2* p = reinterpret_cast<const float2*>(x + static_cast<size_t>(warp) * C);
  float2 v[NP];
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < NP; ++j) {
    v[j] = p[lane + j * 32];
    s += v[j].x + v[j].y;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / C;
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < NP; ++j) {
    const float dx = v[j].x - mean, dy = v[j].y - mean;
    q = fmaf(dx, dx, q);
    q = fmaf(dy, dy, q);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / C + eps);
#pragma unroll
  for (int j = 0; j < NP; ++j) {
    const float y0 = (v[j].x - mean) * rstd * gm[j].x + bt[j].x;
    const float y1 = (v[j].y - mean) * rstd * gm[j].y + bt[j].y;
    const size_t o = static_cast<size_t>(warp) * C + 2 * (lane + j * 32);
    if (out) *reinterpret_cast<__half2*>(out + o) = __floats2half2_rn(y0, y1);
    if (out32) *reinterpret_cast<float2*>(out32 + o) = make_float2(y0, y1);
  }
}

template <int NPL>
__global__ void __launch_bounds__(256)
    layernorm_kernel(const float* __restrict__ x, int rows, int C, const float* __restrict__ gamma,
                     const float* __restrict__ beta, float eps, __half* __restrict__ out, float* __restrict__ out32) {
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  pdl_launch_dependents();
  pdl_wait();
  if (warp >= rows) return;
  const float* p = x + static_cast<size_t>(warp) * C;
  float v[NPL];
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < NPL; ++j) {
    int c = lane + j * 32;
    v[j] = c < C ? p[c] : 0.f;
    s += v[j];
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  float mean = s / C;
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < NPL; ++j) {
    int c = lane + j * 32;
    float d = c < C ? v[j] - mean : 0.f;
    q += d * d;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  float rstd = rsqrtf(q / C + eps);
#pragma unroll
  for (int j = 0; j < NPL; ++j) {
    int c = lane + j * 32;
    if (c < C) {
      float y = (v[j] - mean) * rstd * gamma[c] + beta[c];
      if (out) out[static_cast<size_t>(warp) * C + c] = __float2half_rn(y);
      if (out32) out32[static_cast<size_t>(warp) * C + c] = y;
    }
  }
}

// Row softmax: one block per row.
__global__ void __launch_bounds__(256)
    softmax_rows_kernel(const float* __restrict__ x, int cols, float scale, __half* __restrict__ out) {
  const float* p = x + static_cast<size_t>(blockIdx.x) * cols;
  __half* o = out + static_cast<size_t>(blockIdx.x) * cols;
  __shared__ float red[32];
  float m = -INFINITY;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) m = fmaxf(m, p[c] * scale);
  for (int k = 16; k; k >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, k));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
  for (int w = 1; w < (blockDim.x >> 5); ++w) m = fmaxf(m, red[w]);
  __syncthreads();
  float s = 0.f;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) s += __expf(p[c] * scale - m);
  for (int k = 16; k; k >>= 1) s += __shfl_xor_sync(0xffffffffu, s, k);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  s = 0.f;
  for (int w = 0; w < (blockDim.x >> 5); ++w) s += red[w];
  float inv = 1.0f / s;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) o[c] = __float2half_rn(__expf(p[c] * scale - m) * inv);
}

// GroupNorm(32) of an NHWC fp32 tensor -> one per-(sample, channel) affine -> SiLU -> optional 2x2 resample -> fp16.
// Modulation (ResBlock.out_layers with use_scale_shift_norm, openaimodel.py:267-271): GN(h) * (1 + scale) + shift is
// folded into a = rstd gamma (1 + scale), b = (beta - mean rstd gamma)(1 + scale) + shift; scale / shift are strided
// column slices of the FiLM GEMV output (row stride ldm). Resample (ResBlock up / down, openaimodel.py:256-261, with
// Downsample / Upsample(use_conv=False)): the activated values are written 2x2 average-pooled (1) or nearest-2x
// upsampled (2), so the full-resolution fp16 tensor never reaches HBM. grid = (slabs of output pixels, nb).
__global__ void __launch_bounds__(GN_THREADS)
    gn_mod_apply_kernel(const float* __restrict__ x, int C, int h, int w, int groups, int pix_per_block,
                        const float* __restrict__ meanrstd, const float* __restrict__ gamma,
                        const float* __restrict__ beta, const float* __restrict__ scale, const float* __restrict__ shift,
                        int ldm, int silu, int resample, __half* __restrict__ out) {
  extern __shared__ float2 gn_ab[];   // [C] {a, b}
  const int n = blockIdx.y;
  const int cpg = C / groups;
  pdl_launch_dependents();
  pdl_wait();
  for (int c = threadIdx.x; c < C; c += GN_THREADS) {
    const int g = c / cpg;
    const float mean = meanrstd[(static_cast<size_t>(n) * groups + g) * 2];
    const float rstd = meanrstd[(static_cast<size_t>(n) * groups + g) * 2 + 1];
    float a = rstd * __ldg(gamma + c);
    float b = fmaf(-mean, a, __ldg(beta + c));
    if (scale) {
      const float s1 = 1.0f + scale[static_cast<size_t>(n) * ldm + c];
      a *= s1;
      b = fmaf(b, s1, shift[static_cast<size_t>(n) * ldm + c]);
    }
    gn_ab[c] = make_float2(a, b);
  }
  __syncthreads();
  const int ho = resample == 1 ? h / 2 : resample == 2 ? 2 * h : h;
  const int wo = resample == 1 ? w / 2 : resample == 2 ? 2 * w : w;
  const int c4n = C >> 2;
  const long p0 = static_cast<long>(blockIdx.x) * pix_per_block;
  const long p1 = min(static_cast<long>(ho) * wo, p0 + pix_per_block);
  const float* xs = x + static_cast<size_t>(n) * h * w * C;
  __half* os = out + static_cast<size_t>(n) * ho * wo * C;
  for (long i = p0 * c4n + threadIdx.x; i < p1 * c4n; i += GN_THREADS) {
    const int c = static_cast<int>(i % c4n) * 4;
    const long p = i / c4n;
    const int oy = static_cast<int>(p / wo), ox = static_cast<int>(p % wo);
    const float4 ab01 = *reinterpret_cast<const float4*>(&gn_ab[c]);
    const float4 ab23 = *reinterpret_cast<const float4*>(&gn_ab[c + 2]);
    auto act = [&](float4 v, float y[4]) {
      y[0] = fmaf(v.x, ab01.x, ab01.y);
      y[1] = fmaf(v.y, ab01.z, ab01.w);
      y[2] = fmaf(v.z, ab23.x, ab23.y);
      y[3] = fmaf(v.w, ab23.z, ab23.w);
      if (silu) {
#pragma unroll
        for (int j = 0; j < 4; ++j) y[j] = silu_fast(y[j]);
      }
    };
    float y[4];
    if (resample == 1) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int t = 0; t < 4; ++t) {   // avg_pool2d order: rows, then columns
        const int iy = 2 * oy + (t >> 1), ix = 2 * ox + (t & 1);
        float yt[4];
        act(*reinterpret_cast<const float4*>(xs + (static_cast<size_t>(iy) * w + ix) * C + c), yt);
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[j] += yt[j];
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) y[j] = acc[j] * 0.25f;
    } else {
      const int iy = resample == 2 ? oy >> 1 : oy, ix = resample == 2 ? ox >> 1 : ox;
      act(*reinterpret_cast<const float4*>(xs + (static_cast<size_t>(iy) * w + ix) * C + c), y);
    }
    __half2 h0 = __floats2half2_rn(y[0], y[1]), h1 = __floats2half2_rn(y[2], y[3]);
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&h0);
    u.y = *reinterpret_cast<uint32_t*>(&h1);
    *reinterpret_cast<uint2*>(os + p * C + c) = u;
  }
}

}  // namespace sdb

using namespace sdb;

extern "C" int sdb_groupnorm(const float* x0, const float* x1, int32_t c0, int32_t c1, int32_t nb, int32_t hw,
                             int32_t groups, const float* gamma, const float* beta, float eps, int32_t silu,
                             void* out_f16, void* raw_f16, void* out_lo_f16, void* raw_lo_f16, void* stats_ws,
                             const void* chan_stats0, const void* chan_stats1, int32_t stats_t0, int32_t stats_t1,
                             int32_t stats_group, sdb_stream_t stream) {
  SDB_REC(sdb_groupnorm(x0, x1, c0, c1, nb, hw, groups, gamma, beta, eps, silu, out_f16, raw_f16, out_lo_f16, raw_lo_f16, stats_ws, chan_stats0, chan_stats1, stats_t0, stats_t1, stats_group, s_));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int C = c0 + c1;
  SDB_CHECK(x0 && out_f16 && stats_ws && gamma && beta, "sdb_groupnorm: null pointer");
  SDB_CHECK((c1 == 0) == (x1 == nullptr), "sdb_groupnorm: x1/c1 mismatch");
  SDB_CHECK(groups > 0 && groups <= 64 && C % groups == 0, "sdb_groupnorm: C=%d not divisible by groups=%d", C, groups);
  SDB_CHECK(c0 % 4 == 0 && c1 % 4 == 0, "sdb_groupnorm: channel counts must be multiples of 4");
  SDB_CHECK(C <= GN_THREADS * GN_MAX_CPT, "sdb_groupnorm: C=%d too large", C);
  // the apply pass reads x as float4 and writes fp16 quads as 8-byte words
  SDB_CHECK(((reinterpret_cast<uintptr_t>(x0) | reinterpret_cast<uintptr_t>(x1)) & 15) == 0,
            "sdb_groupnorm: x0 / x1 must be 16-byte aligned");
  SDB_CHECK(((reinterpret_cast<uintptr_t>(out_f16) | reinterpret_cast<uintptr_t>(raw_f16) |
              reinterpret_cast<uintptr_t>(out_lo_f16) | reinterpret_cast<uintptr_t>(raw_lo_f16)) & 7) == 0,
            "sdb_groupnorm: fp16 outputs must be 8-byte aligned");
  // workspace layout: [nb][GN_MAX_SLABS][groups][2] float partials | [nb][groups][2] float mean/rstd | [nb] tickets
  float* partial = static_cast<float*>(stats_ws);
  float* meanrstd = partial + static_cast<size_t>(nb) * GN_MAX_SLABS * groups * 2;
  unsigned int* counter = reinterpret_cast<unsigned int*>(meanrstd + static_cast<size_t>(nb) * groups * 2);
  const int sg = stats_group > 0 ? stats_group : 1;
  const bool fused_stats = chan_stats0 != nullptr && (c1 == 0 || chan_stats1 != nullptr) && groups <= 32;
  if (fused_stats)
    SDB_CHECK(stats_t0 > 0 && (c1 == 0 || stats_t1 > 0) && (C / groups) % sg == 0 && c0 % sg == 0 && c1 % sg == 0,
              "sdb_groupnorm: statistics entries of %d channels do not tile the groups (C %d + %d, %d groups)", sg, c0, c1,
              groups);
  if (!fused_stats) SDB_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned int) * nb, st));
  SDB_CHECK(!raw_lo_f16 || raw_f16, "sdb_groupnorm: raw_lo needs raw");
  // channel-lane width: threads of a block cover cw channels x (256 / cw) rows at a time
  int cw = GN_THREADS;
  while (cw > 32 && cw / 2 >= C) cw /= 2;
  const int rstep = GN_THREADS / cw;
  int target_blocks = sm_count() * 4;
  int slabs = std::max(1, std::min(std::min((hw + rstep - 1) / rstep, GN_MAX_SLABS), (target_blocks + nb - 1) / nb));
  int rows_per_block = (hw + slabs - 1) / slabs;
  slabs = (hw + rows_per_block - 1) / rows_per_block;
  dim3 grid(slabs, nb);
  if (!fused_stats) {
    (C > GN_THREADS * GN_CPT ? gn_stats_kernel<GN_MAX_CPT> : gn_stats_kernel<GN_CPT>)<<<grid, GN_THREADS, (2 * rstep + 1) * C * sizeof(float), st>>>(x0, x1, c0, c1, hw, groups, rows_per_block, cw,
                                                                      eps, partial, counter, meanrstd);
    SDB_LAUNCH_CHECK();
  }
  // many tile slots per sample (large images): fold them once, the apply blocks then read mean / rstd
  bool in_kernel_fold = fused_stats;
  if (fused_stats && static_cast<long>(std::max(stats_t0, stats_t1)) * ((C / groups) / sg) > 512) {
    SDB_CUDA(launch_pdl(gn_fold_kernel, dim3(groups, nb), dim3(GN_THREADS), 0, st, static_cast<const float2*>(chan_stats0),
                        static_cast<int>(stats_t0), static_cast<const float2*>(chan_stats1), static_cast<int>(stats_t1), sg,
                        c0, c1, groups, hw, eps, meanrstd));
    SDB_LAUNCH_CHECK();
    in_kernel_fold = false;
  }
  // apply: about four resident blocks per SM (each re-derives the group statistics from a few KB of partials), down to
  // one row per block at small resolutions
  int aslabs = std::max(1, std::min(hw, (sm_count() * 4 + nb - 1) / nb));
  int arows = (hw + aslabs - 1) / aslabs;
  aslabs = (hw + arows - 1) / arows;
  dim3 agrid(aslabs, nb);
  SDB_CUDA(launch_pdl(gn_apply_kernel, agrid, dim3(GN_THREADS), static_cast<size_t>(C) * sizeof(float2), st, x0, x1, c0, c1,
                      hw, groups, arows,
                      static_cast<const float*>(meanrstd), gamma, beta, eps, silu, static_cast<__half*>(out_f16),
                      static_cast<__half*>(raw_f16), static_cast<__half*>(out_lo_f16),
                      static_cast<__half*>(raw_lo_f16),
                      in_kernel_fold ? static_cast<const float2*>(chan_stats0) : static_cast<const float2*>(nullptr),
                      static_cast<int>(stats_t0), static_cast<const float2*>(chan_stats1), static_cast<int>(stats_t1), sg));
  SDB_LAUNCH_CHECK();
  return 0;
}

extern "C" int sdb_layernorm(const float* x, int32_t rows, int32_t c, const float* gamma, const float* beta, float eps,
                             void* out_f16, float* out_f32, sdb_stream_t stream) {
  SDB_REC(sdb_layernorm(x, rows, c, gamma, beta, eps, out_f16, out_f32, s_));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  SDB_CHECK(x && gamma && beta && (out_f16 || out_f32), "sdb_layernorm: null pointer");
  SDB_CHECK(c <= 32 * 56, "sdb_layernorm: C=%d too large", c);
  // one warp per row; fewer warps per block at small row counts so the grid still covers the machine
  int warps_per_block = rows >= 8 * 2 * sm_count() ? 8 : rows >= 4 * 2 * sm_count() ? 4 : rows >= 2 * 2 * sm_count() ? 2 : 1;
  int blocks = (rows + warps_per_block - 1) / warps_per_block;
  __half* o16 = static_cast<__half*>(out_f16);
  const int npl = (c + 31) / 32;
  const bool al8 = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(beta) |
                     reinterpret_cast<uintptr_t>(out_f32)) & 7) == 0 && (reinterpret_cast<uintptr_t>(o16) & 3) == 0;
#define SDB_LN2(N) SDB_CUDA(launch_pdl(layernorm_v2_kernel<N>, dim3(blocks), dim3(warps_per_block * 32), 0, st, x, rows, c, gamma, beta, eps, o16, out_f32))
  if (c % 64 == 0 && al8 && (c == 320 || c == 640 || c == 768 || c == 1280 || c == 512)) {
    switch (c / 64) {
      case 5: SDB_LN2(5); break;
      case 8: SDB_LN2(8); break;
      case 10: SDB_LN2(10); break;
      case 12: SDB_LN2(12); break;
      default: SDB_LN2(20); break;
    }
    SDB_LAUNCH_CHECK();
    return 0;
  }
#undef SDB_LN2
#define SDB_LN(N) SDB_CUDA(launch_pdl(layernorm_kernel<N>, dim3(blocks), dim3(warps_per_block * 32), 0, st, x, rows, c, gamma, beta, eps, o16, out_f32))
  if (npl <= 2) SDB_LN(2);
  else if (npl <= 4) SDB_LN(4);
  else if (npl <= 10) SDB_LN(10);
  else if (npl <= 20) SDB_LN(20);
  else if (npl <= 24) SDB_LN(24);
  else if (npl <= 40) SDB_LN(40);
  else if (npl <= 48) SDB_LN(48);
  else SDB_LN(56);   // the retrieval-augmented UNet's middle block (1792)
#undef SDB_LN
  SDB_LAUNCH_CHECK();
  return 0;
}

extern "C" int sdb_softmax_rows(const float* x, int32_t rows, int32_t cols, float scale, void* out_f16,
                                sdb_stream_t stream) {
  SDB_REC(sdb_softmax_rows(x, rows, cols, scale, out_f16, s_));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  SDB_CHECK(x && out_f16, "sdb_softmax_rows: null pointer");
  softmax_rows_kernel<<<rows, 256, 0, st>>>(x, cols, scale, static_cast<__half*>(out_f16));
  SDB_LAUNCH_CHECK();
  return 0;
}

extern "C" int sdb_groupnorm_mod(const float* x, int32_t c, int32_t nb, int32_t h, int32_t w, int32_t groups,
                                 const float* gamma, const float* beta, float eps, int32_t silu, const float* scale,
                                 const float* shift, int32_t ldm, int32_t resample, void* out_f16, void* stats_ws,
                                 const void* chan_stats, int32_t stats_t, int32_t stats_group, sdb_stream_t stream) {
  SDB_REC(sdb_groupnorm_mod(x, c, nb, h, w, groups, gamma, beta, eps, silu, scale, shift, ldm, resample, out_f16, stats_ws,
                            chan_stats, stats_t, stats_group, s_));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  SDB_CHECK(x && out_f16 && stats_ws && gamma && beta, "sdb_groupnorm_mod: null pointer");
  SDB_CHECK(nb > 0 && h > 0 && w > 0, "sdb_groupnorm_mod: bad sizes");
  SDB_CHECK(groups > 0 && groups <= 32 && c % groups == 0, "sdb_groupnorm_mod: C=%d not divisible by groups=%d", c, groups);
  SDB_CHECK(c % 4 == 0 && c <= GN_THREADS * GN_MAX_CPT, "sdb_groupnorm_mod: C=%d must be a multiple of 4, <= %d", c,
            GN_THREADS * GN_MAX_CPT);
  // the apply pass reads x as float4 and writes fp16 quads as 8-byte words
  SDB_CHECK((reinterpret_cast<uintptr_t>(x) & 15) == 0, "sdb_groupnorm_mod: x must be 16-byte aligned");
  SDB_CHECK((reinterpret_cast<uintptr_t>(out_f16) & 7) == 0, "sdb_groupnorm_mod: out must be 8-byte aligned");
  SDB_CHECK((scale == nullptr) == (shift == nullptr), "sdb_groupnorm_mod: scale and shift go together");
  SDB_CHECK(!scale || ldm >= c, "sdb_groupnorm_mod: modulation row stride %d < C %d", ldm, c);
  SDB_CHECK(resample >= 0 && resample <= 2, "sdb_groupnorm_mod: resample %d (0 none, 1 down, 2 up)", resample);
  SDB_CHECK(resample != 1 || (h % 2 == 0 && w % 2 == 0), "sdb_groupnorm_mod: 2x2 average pool needs even sides (%dx%d)",
            h, w);
  const int hw = h * w;
  const int cpg = c / groups;
  const int sg = stats_group > 0 ? stats_group : 1;
  // workspace layout as sdb_groupnorm: [nb][GN_MAX_SLABS][groups][2] partials | [nb][groups][2] mean/rstd | [nb] tickets
  float* partial = static_cast<float*>(stats_ws);
  float* meanrstd = partial + static_cast<size_t>(nb) * GN_MAX_SLABS * groups * 2;
  unsigned int* counter = reinterpret_cast<unsigned int*>(meanrstd + static_cast<size_t>(nb) * groups * 2);
  if (chan_stats) {
    SDB_CHECK(stats_t > 0 && cpg % sg == 0 && c % sg == 0,
              "sdb_groupnorm_mod: statistics entries of %d channels do not tile the groups (C %d, %d groups)", sg, c, groups);
    SDB_CUDA(launch_pdl(gn_fold_kernel, dim3(groups, nb), dim3(GN_THREADS), 0, st, static_cast<const float2*>(chan_stats),
                        static_cast<int>(stats_t), static_cast<const float2*>(nullptr), 0, sg, c, 0, groups, hw, eps,
                        meanrstd));
    SDB_LAUNCH_CHECK();
  } else {
    SDB_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned int) * nb, st));
    int cw = GN_THREADS;
    while (cw > 32 && cw / 2 >= c) cw /= 2;
    const int rstep = GN_THREADS / cw;
    int slabs = std::max(1, std::min(std::min((hw + rstep - 1) / rstep, GN_MAX_SLABS), (sm_count() * 4 + nb - 1) / nb));
    int rows_per_block = (hw + slabs - 1) / slabs;
    slabs = (hw + rows_per_block - 1) / rows_per_block;
    (c > GN_THREADS * GN_CPT ? gn_stats_kernel<GN_MAX_CPT> : gn_stats_kernel<GN_CPT>)<<<dim3(slabs, nb), GN_THREADS, (2 * rstep + 1) * c * sizeof(float), st>>>(x, nullptr, c, 0, hw, groups,
                                                                                 rows_per_block, cw, eps, partial, counter,
                                                                                 meanrstd);
    SDB_LAUNCH_CHECK();
  }
  const long opix = resample == 1 ? static_cast<long>(hw) / 4 : resample == 2 ? static_cast<long>(hw) * 4 : hw;
  long slabs = std::max(1L, std::min(opix, static_cast<long>((sm_count() * 4 + nb - 1) / nb)));
  long ppb = (opix + slabs - 1) / slabs;
  slabs = (opix + ppb - 1) / ppb;
  SDB_CUDA(launch_pdl(gn_mod_apply_kernel, dim3(static_cast<unsigned>(slabs), nb), dim3(GN_THREADS),
                      static_cast<size_t>(c) * sizeof(float2), st, x, static_cast<int>(c), static_cast<int>(h),
                      static_cast<int>(w), static_cast<int>(groups), static_cast<int>(ppb), static_cast<const float*>(meanrstd),
                      gamma, beta, scale, shift, static_cast<int>(ldm), static_cast<int>(silu), static_cast<int>(resample),
                      static_cast<__half*>(out_f16)));
  SDB_LAUNCH_CHECK();
  return 0;
}
