// The forward half of the LDM training objective (include/sdb200_eval.h): per-sample-t forward noising and the fused
// per-sample loss reduction. Both are HBM-bound streams over the latent; the loss is one CTA per sample so that its
// summation order depends on the sample's size alone.
#include "../../include/sdb200_eval.h"
#include "host.h"

namespace sdb {

constexpr int kLossThreads = 256;

__global__ void q_sample_t_kernel(const float* __restrict__ x0, const float* __restrict__ noise,
                                  const int64_t* __restrict__ t, const float* __restrict__ sqrt_ac,
                                  const float* __restrict__ sqrt_1m_ac, size_t per, size_t total,
                                  float* __restrict__ out) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int64_t tb = t[i / per];
    out[i] = __fadd_rn(__fmul_rn(sqrt_ac[tb], x0[i]), __fmul_rn(sqrt_1m_ac[tb], noise[i]));
  }
}

// one CTA per sample: thread j sums elements j, j + 256, ... in fp64, then a fixed shuffle tree per warp and the eight
// warp sums in order
__global__ void __launch_bounds__(kLossThreads) diffusion_loss_kernel(
    const float* __restrict__ pred, const float* __restrict__ target, int kind, const int64_t* __restrict__ t,
    const float* __restrict__ logvar, const float* __restrict__ lvlb_weights, int nb, size_t n,
    float* __restrict__ out) {
  __shared__ double warp_sum[kLossThreads / 32];
  const int b = blockIdx.x;
  const float* p = pred + static_cast<size_t>(b) * n;
  const float* q = target + static_cast<size_t>(b) * n;
  double acc = 0.0;
  for (size_t i = threadIdx.x; i < n; i += kLossThreads) {
    const float d = __fsub_rn(q[i], p[i]);
    acc += kind == 1 ? static_cast<double>(fabsf(d)) : static_cast<double>(__fmul_rn(d, d));
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < kLossThreads / 32; ++w) s += warp_sum[w];
    const float simple = static_cast<float>(s / static_cast<double>(n));
    const int64_t tb = t[b];
    const float lv = logvar[tb];
    out[b] = simple;
    out[nb + b] = __fadd_rn(__fdiv_rn(simple, expf(lv)), lv);
    out[2 * nb + b] = __fmul_rn(lvlb_weights[tb], simple);
  }
}

}  // namespace sdb

using namespace sdb;
#define ST static_cast<cudaStream_t>(stream)

extern "C" int sdb_q_sample_t(const float* x0, const float* noise, const int64_t* t, const float* sqrt_ac,
                              const float* sqrt_1m_ac, int32_t nb, int64_t n, float* out, sdb_stream_t stream) {
  SDB_REC(sdb_q_sample_t(x0, noise, t, sqrt_ac, sqrt_1m_ac, nb, n, out, s_));
  SDB_CHECK(x0 && noise && t && sqrt_ac && sqrt_1m_ac && out, "sdb_q_sample_t: null pointer");
  SDB_CHECK(nb > 0 && n > 0, "sdb_q_sample_t: empty batch (nb %d, n %lld)", nb, static_cast<long long>(n));
  const size_t total = static_cast<size_t>(nb) * static_cast<size_t>(n);
  const size_t blocks = (total + 255) / 256, cap = static_cast<size_t>(sm_count()) * 16;
  q_sample_t_kernel<<<static_cast<int>(blocks < cap ? blocks : cap), 256, 0, ST>>>(
      x0, noise, t, sqrt_ac, sqrt_1m_ac, static_cast<size_t>(n), total, out);
  SDB_LAUNCH_CHECK();
  return 0;
}

extern "C" int sdb_diffusion_loss(const float* pred, const float* target, int32_t kind, const int64_t* t,
                                  const float* logvar, const float* lvlb_weights, int32_t nb, int64_t n, float* out,
                                  sdb_stream_t stream) {
  SDB_REC(sdb_diffusion_loss(pred, target, kind, t, logvar, lvlb_weights, nb, n, out, s_));
  SDB_CHECK(pred && target && t && logvar && lvlb_weights && out, "sdb_diffusion_loss: null pointer");
  SDB_CHECK(kind == 1 || kind == 2, "sdb_diffusion_loss: kind %d (1 = l1, 2 = l2)", kind);
  SDB_CHECK(nb > 0 && n > 0, "sdb_diffusion_loss: empty batch (nb %d, n %lld)", nb, static_cast<long long>(n));
  diffusion_loss_kernel<<<nb, kLossThreads, 0, ST>>>(pred, target, kind, t, logvar, lvlb_weights, nb,
                                                     static_cast<size_t>(n), out);
  SDB_LAUNCH_CHECK();
  return 0;
}
