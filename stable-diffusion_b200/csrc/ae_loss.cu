// The layers around the tensor-core convs of the first-stage loss (include/sdb200_ae_loss.h): LPIPS input scaling,
// VGG max-pooling, the LPIPS per-layer head, the discriminator's k x k im2col, and the per-sample loss reductions.
// All are HBM-bound streams. The reductions are fp64 in an order fixed by the sample's shape: the LPIPS head sums
// per-chunk partials (the chunk grid depends on the sample's size alone), folded by one warp per sample in a fixed tree;
// the loss terms run one CTA per sample.
#include <cuda_fp16.h>

#include "../../include/sdb200_ae_loss.h"
#include "host.h"

namespace sdb {

constexpr int kAeThreads = 256;
constexpr int kHeadChunk = 256;    // pixels per lpips_head partial

static int ae_grid(size_t total) {
  const size_t blocks = (total + kAeThreads - 1) / kAeThreads, cap = static_cast<size_t>(sm_count()) * 16;
  return static_cast<int>(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

__global__ void lpips_scale_kernel(const float* __restrict__ in0, const float* __restrict__ in1, int nb, int hw,
                                   const float* __restrict__ shift, const float* __restrict__ scale,
                                   float* __restrict__ out) {
  const size_t total = static_cast<size_t>(2 * nb) * hw * 3;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % 3);
    const size_t pix = i / 3;
    const int p = static_cast<int>(pix % hw);
    const int s = static_cast<int>(pix / hw);
    const float* src = s < nb ? in0 + static_cast<size_t>(s) * 3 * hw : in1 + static_cast<size_t>(s - nb) * 3 * hw;
    out[i] = __fdiv_rn(__fsub_rn(src[static_cast<size_t>(c) * hw + p], shift[c]), scale[c]);
  }
}

__device__ __forceinline__ __half2 hmax2_nan(__half2 a, __half2 b) { return __hmax2_nan(a, b); }

// one thread per 8 channels of one output pixel
__global__ void maxpool2x2_kernel(const __half* __restrict__ x, int nb, int h, int w, int c, __half* __restrict__ out) {
  const int ho = h / 2, wo = w / 2, c8 = c / 8;
  const size_t total = static_cast<size_t>(nb) * ho * wo * c8;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int cv = static_cast<int>(i % c8);
    const size_t pix = i / c8;
    const int ox = static_cast<int>(pix % wo);
    const int oy = static_cast<int>((pix / wo) % ho);
    const size_t n = pix / (static_cast<size_t>(wo) * ho);
    const __half* p = x + ((n * h + 2 * oy) * w + 2 * ox) * c + cv * 8;
    const uint4 a = *reinterpret_cast<const uint4*>(p);
    const uint4 b = *reinterpret_cast<const uint4*>(p + c);
    const uint4 d = *reinterpret_cast<const uint4*>(p + static_cast<size_t>(w) * c);
    const uint4 e = *reinterpret_cast<const uint4*>(p + static_cast<size_t>(w) * c + c);
    const __half2* A = reinterpret_cast<const __half2*>(&a);
    const __half2* B = reinterpret_cast<const __half2*>(&b);
    const __half2* D = reinterpret_cast<const __half2*>(&d);
    const __half2* E = reinterpret_cast<const __half2*>(&e);
    uint4 r;
    __half2* R = reinterpret_cast<__half2*>(&r);
#pragma unroll
    for (int j = 0; j < 4; ++j) R[j] = hmax2_nan(hmax2_nan(A[j], B[j]), hmax2_nan(D[j], E[j]));
    *reinterpret_cast<uint4*>(out + pix * c + cv * 8) = r;
  }
}

// Fixed-tree fold of one fp64 value over the lanes of a group of G (power of two, aligned) lanes; every lane of the
// group ends with the same bits.
template <int G>
__device__ __forceinline__ double group_sum(double v) {
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// LPIPS head partials: CTA (chunk, sample) covers pixels [chunk * kHeadChunk, +kHeadChunk) of one sample. G lanes per
// pixel, each holding V 8-channel vectors of both feature maps. Group g sums the values of pixels g, g + GROUPS, ... of
// the chunk in order, then thread 0 sums the groups in order.
template <int G, int V>
__global__ void __launch_bounds__(kAeThreads) lpips_head_partial_kernel(const __half* __restrict__ f, int nb, int hw,
                                                                        const float* __restrict__ lin_w,
                                                                        double* __restrict__ work) {
  constexpr int C = G * V * 8;
  constexpr int GROUPS = kAeThreads / G;
  __shared__ double gsum[GROUPS];
  const int chunk = blockIdx.x, b = blockIdx.y;
  const int g = threadIdx.x / G, lane = threadIdx.x % G;
  float wv[V][8];
#pragma unroll
  for (int v = 0; v < V; ++v)
#pragma unroll
    for (int j = 0; j < 8; ++j) wv[v][j] = lin_w[(v * G + lane) * 8 + j];
  const __half* f0 = f + static_cast<size_t>(b) * hw * C;
  const __half* f1 = f + static_cast<size_t>(b + nb) * hw * C;
  const int p_end = min(hw, (chunk + 1) * kHeadChunk);
  double acc = 0.0;
  // every warp runs the same trip count (the group shuffles below are warp-wide); pixels past the chunk read as zero
  for (int p0 = chunk * kHeadChunk; p0 < p_end; p0 += GROUPS) {
    const int p = p0 + g;
    const bool valid = p < p_end;
    float x0[V][8], x1[V][8];
    double s0 = 0.0, s1 = 0.0;
#pragma unroll
    for (int v = 0; v < V; ++v) {
      uint4 a = make_uint4(0u, 0u, 0u, 0u), q = a;
      if (valid) {
        a = *reinterpret_cast<const uint4*>(f0 + static_cast<size_t>(p) * C + (v * G + lane) * 8);
        q = *reinterpret_cast<const uint4*>(f1 + static_cast<size_t>(p) * C + (v * G + lane) * 8);
      }
      const __half* ah = reinterpret_cast<const __half*>(&a);
      const __half* qh = reinterpret_cast<const __half*>(&q);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        x0[v][j] = __half2float(ah[j]);
        x1[v][j] = __half2float(qh[j]);
        s0 += static_cast<double>(x0[v][j]) * x0[v][j];
        s1 += static_cast<double>(x1[v][j]) * x1[v][j];
      }
    }
    s0 = group_sum<G>(s0);
    s1 = group_sum<G>(s1);
    const float n0 = __fadd_rn(static_cast<float>(sqrt(s0)), 1e-10f);
    const float n1 = __fadd_rn(static_cast<float>(sqrt(s1)), 1e-10f);
    double t = 0.0;
#pragma unroll
    for (int v = 0; v < V; ++v)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = __fsub_rn(__fdiv_rn(x0[v][j], n0), __fdiv_rn(x1[v][j], n1));
        t += static_cast<double>(wv[v][j]) * __fmul_rn(d, d);
      }
    t = group_sum<G>(t);
    if (valid) acc += t;   // every lane of the group holds the same sum
  }
  if (lane == 0) gsum[g] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < GROUPS; ++i) s += gsum[i];
    work[static_cast<size_t>(b) * gridDim.x + chunk] = s;
  }
}

// one warp per sample: lane l sums partials l, l + 32, ..., then a fixed xor tree
__global__ void lpips_head_fold_kernel(const double* __restrict__ work, int nb, int chunks, int hw, int first,
                                       double* __restrict__ acc, float* __restrict__ out) {
  const int b = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x % 32;
  if (b >= nb) return;
  double s = 0.0;
  for (int i = lane; i < chunks; i += 32) s += work[static_cast<size_t>(b) * chunks + i];
  s = group_sum<32>(s);
  if (lane == 0) {
    const double tap = s / static_cast<double>(hw);
    const double a = first ? tap : acc[b] + tap;
    acc[b] = a;
    if (out) out[b] = static_cast<float>(a);
  }
}

__global__ void im2col_kernel(const __half* __restrict__ x, int nb, int h, int w, int c, int k, int stride, int pad,
                              int ho, int wo, int kpad, __half* __restrict__ out) {
  const int vec = (c % 8 == 0) ? 8 : 1;
  const int per_row = kpad / vec;
  const size_t total = static_cast<size_t>(nb) * ho * wo * per_row;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int col = static_cast<int>(i % per_row) * vec;
    const size_t row = i / per_row;
    const int ox = static_cast<int>(row % wo);
    const int oy = static_cast<int>((row / wo) % ho);
    const size_t n = row / (static_cast<size_t>(wo) * ho);
    const int tap = col / c, ch = col - tap * c;
    const int iy = oy * stride - pad + tap / k, ix = ox * stride - pad + tap % k;
    const bool in = tap < k * k && iy >= 0 && iy < h && ix >= 0 && ix < w;
    const __half* src = x + ((n * h + iy) * w + ix) * c + ch;
    if (vec == 8) {
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (in) v = *reinterpret_cast<const uint4*>(src);
      *reinterpret_cast<uint4*>(out + row * kpad + col) = v;
    } else {
      out[row * kpad + col] = in ? *src : __float2half_rn(0.f);
    }
  }
}

__device__ __forceinline__ float softplus_(float x) { return x > 20.f ? x : log1pf(expf(x)); }
// torch.clamp and F.relu keep a NaN; fminf / fmaxf would replace it with the other operand
__device__ __forceinline__ float clamp_nan(float x, float lo, float hi) { return x < lo ? lo : (x > hi ? hi : x); }
__device__ __forceinline__ float relu_nan(float x) { return x < 0.f ? 0.f : x; }

// ae_loss_terms: one CTA per sample (the terms are small next to the convs); thread j sums elements j, j + 256, ... in
// fp64, then a fixed shuffle tree per warp and the eight warp sums in order, as sdb_diffusion_loss does
template <int KIND>
__global__ void __launch_bounds__(kAeThreads) ae_terms_kernel(const float* __restrict__ a, const float* __restrict__ bb,
                                                              size_t n, int cc, double* __restrict__ out) {
  constexpr int R = KIND == 3 ? 5 : 1;
  __shared__ double ws[R][kAeThreads / 32];
  const int b = blockIdx.x, nb = gridDim.x;
  double acc[R];
#pragma unroll
  for (int r = 0; r < R; ++r) acc[r] = 0.0;
  for (size_t i = threadIdx.x; i < n; i += kAeThreads) {
    if (KIND == 1) {
      const size_t e = static_cast<size_t>(b) * n + i;
      acc[0] += static_cast<double>(fabsf(__fsub_rn(a[e], bb[e])));
    } else if (KIND == 2) {
      // sample b holds n / cc pixels of 2 * cc moments: mean channel ch, logvar channel cc + ch
      const size_t pix = static_cast<size_t>(b) * (n / cc) + i / cc;
      const int ch = static_cast<int>(i % cc);
      const float m = a[pix * 2 * cc + ch];
      const float lv = clamp_nan(a[pix * 2 * cc + cc + ch], -30.f, 20.f);
      acc[0] += static_cast<double>(__fsub_rn(__fsub_rn(__fadd_rn(__fmul_rn(m, m), expf(lv)), 1.f), lv));
    } else {
      const float l = a[(static_cast<size_t>(b) * n + i) * cc];
      acc[0] += static_cast<double>(l);
      acc[1] += static_cast<double>(relu_nan(__fsub_rn(1.f, l)));
      acc[2] += static_cast<double>(relu_nan(__fadd_rn(1.f, l)));
      acc[3] += static_cast<double>(softplus_(-l));
      acc[4] += static_cast<double>(softplus_(l));
    }
  }
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const double s = group_sum<32>(acc[r]);
    if ((threadIdx.x & 31) == 0) ws[r][threadIdx.x >> 5] = s;
  }
  __syncthreads();
  if (threadIdx.x < R) {
    double s = 0.0;
    for (int w = 0; w < kAeThreads / 32; ++w) s += ws[threadIdx.x][w];
    out[threadIdx.x * nb + b] = KIND == 2 ? 0.5 * s : s;
  }
}

}  // namespace sdb

using namespace sdb;
#define ST static_cast<cudaStream_t>(stream)

static bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" int sdb_lpips_scale(const float* in0, const float* in1, int32_t nb, int32_t h, int32_t w,
                               const float* shift, const float* scale, float* out, sdb_stream_t stream) {
  SDB_REC(sdb_lpips_scale(in0, in1, nb, h, w, shift, scale, out, s_));
  SDB_CHECK(in0 && in1 && shift && scale && out, "sdb_lpips_scale: null pointer");
  SDB_CHECK(nb > 0 && h > 0 && w > 0, "sdb_lpips_scale: empty input (nb %d, h %d, w %d)", nb, h, w);
  const size_t total = static_cast<size_t>(2 * nb) * h * w * 3;
  lpips_scale_kernel<<<ae_grid(total), kAeThreads, 0, ST>>>(in0, in1, nb, h * w, shift, scale, out);
  SDB_LAUNCH_CHECK();
  return 0;
}

extern "C" int sdb_maxpool2x2(const void* x, int32_t nb, int32_t h, int32_t w, int32_t c, void* out,
                              sdb_stream_t stream) {
  SDB_REC(sdb_maxpool2x2(x, nb, h, w, c, out, s_));
  SDB_CHECK(x && out, "sdb_maxpool2x2: null pointer");
  SDB_CHECK(nb > 0 && h >= 2 && w >= 2 && c > 0 && c % 8 == 0,
            "sdb_maxpool2x2: need nb > 0, h, w >= 2 and c a positive multiple of 8 (nb %d, h %d, w %d, c %d)", nb, h,
            w, c);
  SDB_CHECK(al16(x) && al16(out), "sdb_maxpool2x2: x and out must be 16-byte aligned");
  const size_t total = static_cast<size_t>(nb) * (h / 2) * (w / 2) * (c / 8);
  maxpool2x2_kernel<<<ae_grid(total), kAeThreads, 0, ST>>>(static_cast<const __half*>(x), nb, h, w, c,
                                                          static_cast<__half*>(out));
  SDB_LAUNCH_CHECK();
  return 0;
}

extern "C" int64_t sdb_lpips_head_work(int32_t nb, int32_t hw) {
  return static_cast<int64_t>(nb) * ((static_cast<int64_t>(hw) + kHeadChunk - 1) / kHeadChunk);
}

extern "C" int sdb_lpips_head(const void* f, int32_t nb, int32_t hw, int32_t c, const float* lin_w, int32_t first,
                              double* work, double* acc, float* out, sdb_stream_t stream) {
  SDB_REC(sdb_lpips_head(f, nb, hw, c, lin_w, first, work, acc, out, s_));
  SDB_CHECK(f && lin_w && work && acc, "sdb_lpips_head: null pointer");
  SDB_CHECK(nb > 0 && hw > 0, "sdb_lpips_head: empty input (nb %d, hw %d)", nb, hw);
  SDB_CHECK(al16(f), "sdb_lpips_head: f must be 16-byte aligned");
  const int chunks = (hw + kHeadChunk - 1) / kHeadChunk;
  const dim3 grid(chunks, nb);
  const __half* fh = static_cast<const __half*>(f);
  switch (c) {
    case 64: lpips_head_partial_kernel<8, 1><<<grid, kAeThreads, 0, ST>>>(fh, nb, hw, lin_w, work); break;
    case 128: lpips_head_partial_kernel<16, 1><<<grid, kAeThreads, 0, ST>>>(fh, nb, hw, lin_w, work); break;
    case 256: lpips_head_partial_kernel<32, 1><<<grid, kAeThreads, 0, ST>>>(fh, nb, hw, lin_w, work); break;
    case 512: lpips_head_partial_kernel<32, 2><<<grid, kAeThreads, 0, ST>>>(fh, nb, hw, lin_w, work); break;
    default: SDB_CHECK(false, "sdb_lpips_head: c %d (64, 128, 256 or 512)", c);
  }
  SDB_LAUNCH_CHECK();
  lpips_head_fold_kernel<<<(nb + 7) / 8, kAeThreads, 0, ST>>>(work, nb, chunks, hw, first, acc, out);
  SDB_LAUNCH_CHECK();
  return 0;
}

extern "C" int sdb_im2col(const void* x, int32_t nb, int32_t h, int32_t w, int32_t c, int32_t k, int32_t stride,
                          int32_t pad, int32_t ho, int32_t wo, int32_t kpad, void* out, sdb_stream_t stream) {
  SDB_REC(sdb_im2col(x, nb, h, w, c, k, stride, pad, ho, wo, kpad, out, s_));
  SDB_CHECK(x && out, "sdb_im2col: null pointer");
  SDB_CHECK(nb > 0 && h > 0 && w > 0 && c > 0 && k > 0 && stride > 0 && pad >= 0 && ho > 0 && wo > 0,
            "sdb_im2col: bad geometry (nb %d, h %d, w %d, c %d, k %d, stride %d, pad %d, ho %d, wo %d)", nb, h, w, c,
            k, stride, pad, ho, wo);
  SDB_CHECK(kpad % 8 == 0 && static_cast<int64_t>(k) * k * c <= kpad, "sdb_im2col: kpad %d (need >= %d, %% 8 == 0)",
            kpad, k * k * c);
  SDB_CHECK(c % 8 != 0 || (al16(x) && al16(out)), "sdb_im2col: x and out must be 16-byte aligned when c %% 8 == 0");
  const size_t total = static_cast<size_t>(nb) * ho * wo * (c % 8 == 0 ? kpad / 8 : kpad);
  im2col_kernel<<<ae_grid(total), kAeThreads, 0, ST>>>(static_cast<const __half*>(x), nb, h, w, c, k, stride, pad, ho,
                                                      wo, kpad, static_cast<__half*>(out));
  SDB_LAUNCH_CHECK();
  return 0;
}

extern "C" int sdb_ae_loss_terms(const float* a, const float* bb, int32_t kind, int32_t nb, int64_t n, int32_t cc,
                                 double* out, sdb_stream_t stream) {
  SDB_REC(sdb_ae_loss_terms(a, bb, kind, nb, n, cc, out, s_));
  SDB_CHECK(kind == 1 || kind == 2 || kind == 3, "sdb_ae_loss_terms: kind %d (1 = |a - b|, 2 = KL, 3 = logits)", kind);
  SDB_CHECK(a && out && (kind != 1 || bb), "sdb_ae_loss_terms: null pointer");
  SDB_CHECK(nb > 0 && n > 0, "sdb_ae_loss_terms: empty batch (nb %d, n %lld)", nb, static_cast<long long>(n));
  SDB_CHECK(kind == 1 || (cc > 0 && (kind != 2 || n % cc == 0)), "sdb_ae_loss_terms: cc %d for n %lld", cc,
            static_cast<long long>(n));
  const size_t un = static_cast<size_t>(n);
  if (kind == 1) ae_terms_kernel<1><<<nb, kAeThreads, 0, ST>>>(a, bb, un, cc, out);
  else if (kind == 2) ae_terms_kernel<2><<<nb, kAeThreads, 0, ST>>>(a, bb, un, cc, out);
  else ae_terms_kernel<3><<<nb, kAeThreads, 0, ST>>>(a, bb, un, cc, out);
  SDB_LAUNCH_CHECK();
  return 0;
}
