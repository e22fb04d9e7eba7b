// The cond stage of the LDM semantic-synthesis models (models/ldm/semantic_synthesis{256,512}): SpatialRescaler
// (ldm/modules/encoders/modules.py:106-134), i.e. n_stages bilinear x0.5 interpolations followed by an optional 1x1 conv
// (channel_mapper), on a float NCHW map or straight from a uint8 label map (the one-hot the reference's data pipeline
// builds, never materialised).
//
// With scale_factor 0.5 and align_corners False every output pixel o reads source 2o + 0.5: input pixels 2o and 2o + 1
// at weight 0.5 each, both always inside the input (side -> floor(side / 2)). n stages therefore read the
// 2^n x 2^n window at 2^n * o. Each stage is computed in the order of torch's CUDA bilinear kernel,
// 0.5 (0.5 a + 0.5 b) + 0.5 (0.5 c + 0.5 d); every product by 0.5 is exact, so contraction cannot change the result.
// The channel map accumulates fma(W[o, k], v_k, acc) over k ascending from +0, then adds the bias. For one-hot input
// every v_k is count_k / 4^n exactly and absent classes add exact zeros, so the label kernel, which visits only the
// classes present, gives the float kernel's bits.
#include "../../include/sdb200.h"
#include "host.h"

namespace sdb {

constexpr int kRescaleMaxStages = 3;   // windows up to 8 x 8; every reference config uses 2
constexpr int kRescaleOutGroup = 4;    // output channels accumulated per pass over the input channels

static inline int semantic_grid(size_t n, int threads) {
  size_t b = (n + threads - 1) / threads;
  size_t cap = static_cast<size_t>(sm_count()) * 16;
  return static_cast<int>(b < 1 ? 1 : (b > cap ? cap : b));
}

__device__ __forceinline__ float half_bilerp(float a, float b, float c, float d) {
  const float top = __fadd_rn(__fmul_rn(0.5f, a), __fmul_rn(0.5f, b));
  const float bot = __fadd_rn(__fmul_rn(0.5f, c), __fmul_rn(0.5f, d));
  return __fadd_rn(__fmul_rn(0.5f, top), __fmul_rn(0.5f, bot));
}

// N bilinear x0.5 stages of the 2^N x 2^N window at p (row pitch w), stage by stage as interpolate computes them
template <int N>
__device__ __forceinline__ float downscale(const float* __restrict__ p, int w) {
  if constexpr (N == 0) {
    return __ldg(p);
  } else {
    constexpr int s = 1 << (N - 1);
    const float a = downscale<N - 1>(p, w), b = downscale<N - 1>(p + s, w);
    const float c = downscale<N - 1>(p + static_cast<size_t>(s) * w, w);
    const float d = downscale<N - 1>(p + static_cast<size_t>(s) * w + s, w);
    return half_bilerp(a, b, c, d);
  }
}

// x fp32 [nb, cin, h, w] -> out fp32 [nb, cout, ho, wo]; weight == nullptr: cout = cin, out = the downscaled input
template <int N>
__global__ void spatial_rescale_kernel(const float* __restrict__ x, int nb, int cin, int h, int w,
                                       const float* __restrict__ weight, const float* __restrict__ bias, int cout,
                                       int ho, int wo, float* __restrict__ out) {
  const size_t ohw = static_cast<size_t>(ho) * wo;
  const size_t ihw = static_cast<size_t>(h) * w;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < nb * ohw;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t n = i / ohw, p = i % ohw;
    const int oy = static_cast<int>(p / wo), ox = static_cast<int>(p % wo);
    const float* src = x + n * cin * ihw + (static_cast<size_t>(oy) << N) * w + (static_cast<size_t>(ox) << N);
    float* dst = out + n * cout * ohw + p;
    if (weight == nullptr) {
      for (int k = 0; k < cin; ++k) dst[k * ohw] = downscale<N>(src + k * ihw, w);
      continue;
    }
    for (int o0 = 0; o0 < cout; o0 += kRescaleOutGroup) {
      float acc[kRescaleOutGroup];
#pragma unroll
      for (int j = 0; j < kRescaleOutGroup; ++j) acc[j] = 0.0f;
      for (int k = 0; k < cin; ++k) {
        const float v = downscale<N>(src + k * ihw, w);
#pragma unroll
        for (int j = 0; j < kRescaleOutGroup; ++j)
          if (o0 + j < cout) acc[j] = __fmaf_rn(__ldg(weight + static_cast<size_t>(o0 + j) * cin + k), v, acc[j]);
      }
#pragma unroll
      for (int j = 0; j < kRescaleOutGroup; ++j)
        if (o0 + j < cout) dst[(o0 + j) * ohw] = bias ? __fadd_rn(acc[j], __ldg(bias + o0 + j)) : acc[j];
    }
  }
}

// labels uint8 [nb, h, w] (ids < cin) -> out fp32 [nb, cout, ho, wo]: the channel map of the downscaled one-hot. The
// window's labels sit in registers; each pass picks the next larger class id present and its count.
template <int N>
__global__ void seg_labels_rescale_kernel(const uint8_t* __restrict__ labels, int nb, int cin, int h, int w,
                                          const float* __restrict__ weight, const float* __restrict__ bias, int cout,
                                          int ho, int wo, float* __restrict__ out) {
  constexpr int S = 1 << N;
  const float inv = 1.0f / static_cast<float>(S * S);    // a power of two: count * inv is exact
  const size_t ohw = static_cast<size_t>(ho) * wo;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < nb * ohw;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t n = i / ohw, p = i % ohw;
    const int oy = static_cast<int>(p / wo), ox = static_cast<int>(p % wo);
    const uint8_t* src = labels + n * static_cast<size_t>(h) * w + (static_cast<size_t>(oy) << N) * w +
                         (static_cast<size_t>(ox) << N);
    int lab[S * S];
#pragma unroll
    for (int r = 0; r < S; ++r)
#pragma unroll
      for (int c = 0; c < S; ++c) lab[r * S + c] = __ldg(src + static_cast<size_t>(r) * w + c);
    float* dst = out + n * cout * ohw + p;
    for (int o0 = 0; o0 < cout; o0 += kRescaleOutGroup) {
      float acc[kRescaleOutGroup];
#pragma unroll
      for (int j = 0; j < kRescaleOutGroup; ++j) acc[j] = 0.0f;
      int prev = -1;
      while (true) {
        int k = 256, cnt = 0;
#pragma unroll
        for (int q = 0; q < S * S; ++q) k = lab[q] > prev ? min(k, lab[q]) : k;
        if (k == 256) break;
#pragma unroll
        for (int q = 0; q < S * S; ++q) cnt += lab[q] == k;
        const float v = __fmul_rn(static_cast<float>(cnt), inv);
#pragma unroll
        for (int j = 0; j < kRescaleOutGroup; ++j)
          if (o0 + j < cout) acc[j] = __fmaf_rn(__ldg(weight + static_cast<size_t>(o0 + j) * cin + k), v, acc[j]);
        prev = k;
      }
#pragma unroll
      for (int j = 0; j < kRescaleOutGroup; ++j)
        if (o0 + j < cout) dst[(o0 + j) * ohw] = bias ? __fadd_rn(acc[j], __ldg(bias + o0 + j)) : acc[j];
    }
  }
}

}  // namespace sdb

using namespace sdb;
#define ST static_cast<cudaStream_t>(stream)

#define SDB_RESCALE_DISPATCH(kernel, n_stages, grid, threads, ...)              \
  switch (n_stages) {                                                            \
    case 0: kernel<0><<<grid, threads, 0, ST>>>(__VA_ARGS__); break;             \
    case 1: kernel<1><<<grid, threads, 0, ST>>>(__VA_ARGS__); break;             \
    case 2: kernel<2><<<grid, threads, 0, ST>>>(__VA_ARGS__); break;             \
    default: kernel<3><<<grid, threads, 0, ST>>>(__VA_ARGS__); break;            \
  }

static int rescale_sizes(const char* what, int32_t nb, int32_t cin, int32_t h, int32_t w, int32_t n_stages,
                         int32_t* ho, int32_t* wo) {
  SDB_CHECK(n_stages >= 0 && n_stages <= kRescaleMaxStages, "%s: n_stages %d outside [0, %d]", what, n_stages,
            kRescaleMaxStages);
  SDB_CHECK(nb > 0 && cin > 0 && h > 0 && w > 0, "%s: bad sizes (nb=%d cin=%d %dx%d)", what, nb, cin, h, w);
  *ho = h >> n_stages;
  *wo = w >> n_stages;
  SDB_CHECK(*ho > 0 && *wo > 0, "%s: %dx%d is smaller than the 2^%d window", what, h, w, n_stages);
  return 0;
}

extern "C" int sdb_spatial_rescale(const float* x_nchw, int32_t nb, int32_t cin, int32_t h, int32_t w,
                                   int32_t n_stages, const float* weight, const float* bias, int32_t cout,
                                   float* out_nchw, sdb_stream_t stream) {
  SDB_REC(sdb_spatial_rescale(x_nchw, nb, cin, h, w, n_stages, weight, bias, cout, out_nchw, s_));
  SDB_CHECK(x_nchw && out_nchw, "sdb_spatial_rescale: null pointer");
  int32_t ho, wo;
  if (rescale_sizes("sdb_spatial_rescale", nb, cin, h, w, n_stages, &ho, &wo)) return 1;
  SDB_CHECK(weight ? cout > 0 : (cout == cin && bias == nullptr),
            "sdb_spatial_rescale: without a channel map cout must equal cin (%d vs %d) and bias be NULL", cout, cin);
  const size_t n = static_cast<size_t>(nb) * ho * wo;
  const int grid = semantic_grid(n, 128);
  SDB_RESCALE_DISPATCH(spatial_rescale_kernel, n_stages, grid, 128, x_nchw, nb, cin, h, w, weight, bias, cout, ho,
                       wo, out_nchw);
  SDB_LAUNCH_CHECK();
  return 0;
}

extern "C" int sdb_seg_labels_rescale(const uint8_t* labels, int32_t nb, int32_t cin, int32_t h, int32_t w,
                                      int32_t n_stages, const float* weight, const float* bias, int32_t cout,
                                      float* out_nchw, sdb_stream_t stream) {
  SDB_REC(sdb_seg_labels_rescale(labels, nb, cin, h, w, n_stages, weight, bias, cout, out_nchw, s_));
  SDB_CHECK(labels && weight && out_nchw, "sdb_seg_labels_rescale: null pointer (the channel map is required)");
  SDB_CHECK(cin <= 256 && cout > 0, "sdb_seg_labels_rescale: bad channels (cin=%d <= 256, cout=%d)", cin, cout);
  int32_t ho, wo;
  if (rescale_sizes("sdb_seg_labels_rescale", nb, cin, h, w, n_stages, &ho, &wo)) return 1;
  const size_t n = static_cast<size_t>(nb) * ho * wo;
  const int grid = semantic_grid(n, 128);
  SDB_RESCALE_DISPATCH(seg_labels_rescale_kernel, n_stages, grid, 128, labels, nb, cin, h, w, weight, bias, cout, ho,
                       wo, out_nchw);
  SDB_LAUNCH_CHECK();
  return 0;
}
