// Inpainting with a concat-conditioned UNet (scripts/inpaint.py of the reference, models/ldm/inpainting_big):
// the UNet's conv_in im2col read from two NCHW sources, and the per-image pre- / post-processing of make_batch and the
// composite. Elementwise fp32 math uses explicit __f*_rn ops in the reference's operation order, so results are bit-exact.
#include "../../include/sdb200.h"
#include "host.h"
#include <cuda_fp16.h>

namespace sdb {

static inline int inpaint_grid(size_t n, int threads = 256) {
  size_t b = (n + threads - 1) / threads;
  size_t cap = static_cast<size_t>(sm_count()) * 16;
  return static_cast<int>(b < 1 ? 1 : (b > cap ? cap : b));
}
#define GRID_STRIDE(i, n)                                                                      \
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < (n); \
       i += static_cast<size_t>(gridDim.x) * blockDim.x)

// 3x3 / stride 1 / pad 1 im2col of cat([x, cond], 1) without materialising the concat: row = (n, oy, ox),
// k = (ky*3+kx)*(cx+cc) + ch, channel ch < cx read from x, the rest from cond; zero beyond 9*(cx+cc).
__global__ void im2col3x3_concat_kernel(const float* __restrict__ x, int cx, const float* __restrict__ cond, int cc,
                                        int nb, int h, int w, int kpad, __half* __restrict__ out) {
  const int ct = cx + cc;
  const size_t total = static_cast<size_t>(nb) * h * w * kpad;
  const size_t hw = static_cast<size_t>(h) * w;
  GRID_STRIDE(i, total) {
    const int k = static_cast<int>(i % kpad);
    const size_t row = i / kpad;
    float v = 0.f;
    if (k < 9 * ct) {
      const int tap = k / ct, ch = k - tap * ct;
      const int ox = static_cast<int>(row % w);
      const int oy = static_cast<int>((row / w) % h);
      const size_t n = row / hw;
      const int iy = oy + tap / 3 - 1, ix = ox + tap % 3 - 1;
      if (iy >= 0 && iy < h && ix >= 0 && ix < w) {
        const size_t p = static_cast<size_t>(iy) * w + ix;
        v = ch < cx ? x[(n * cx + ch) * hw + p] : cond[(n * cc + (ch - cx)) * hw + p];
      }
    }
    out[i] = __float2half_rn(v);
  }
}

// make_batch: m01 = (u8 / 255 >= 0.5); masked = ((1 - m01) * (u / 255)) * 2 - 1, NCHW fp32 (the VQ encoder's input).
__global__ void inpaint_masked_image_kernel(const uint8_t* __restrict__ img, const uint8_t* __restrict__ mask, int nb,
                                            int h, int w, float* __restrict__ masked) {
  const size_t hw = static_cast<size_t>(h) * w;
  GRID_STRIDE(i, static_cast<size_t>(nb) * 3 * hw) {
    const size_t p = i % hw;
    const int c = static_cast<int>((i / hw) % 3);
    const size_t n = i / (3 * hw);
    const float m = __fdiv_rn(static_cast<float>(mask[n * hw + p]), 255.0f) >= 0.5f ? 1.0f : 0.0f;
    const float u = __fdiv_rn(static_cast<float>(img[(n * hw + p) * 3 + c]), 255.0f);
    masked[i] = __fsub_rn(__fmul_rn(__fmul_rn(__fsub_rn(1.0f, m), u), 2.0f), 1.0f);
  }
}

// F.interpolate(mask * 2 - 1, size=(hc, wc)) (mode "nearest": src = min(floor(dst * (float)in / out), in - 1)) into
// channel `ch` of the conditioning buffer [nb, cond_c, hc, wc].
__global__ void inpaint_mask_channel_kernel(const uint8_t* __restrict__ mask, int nb, int h, int w, int hc, int wc,
                                            float* __restrict__ cond, int cond_c, int ch) {
  const float sy = __fdiv_rn(static_cast<float>(h), static_cast<float>(hc));
  const float sx = __fdiv_rn(static_cast<float>(w), static_cast<float>(wc));
  const size_t hwc = static_cast<size_t>(hc) * wc;
  GRID_STRIDE(i, static_cast<size_t>(nb) * hwc) {
    const int ox = static_cast<int>(i % wc);
    const int oy = static_cast<int>((i / wc) % hc);
    const size_t n = i / hwc;
    const int iy = hc == h ? oy : min(static_cast<int>(floorf(__fmul_rn(static_cast<float>(oy), sy))), h - 1);
    const int ix = wc == w ? ox : min(static_cast<int>(floorf(__fmul_rn(static_cast<float>(ox), sx))), w - 1);
    const float u = __fdiv_rn(static_cast<float>(mask[(n * h + iy) * w + ix]), 255.0f);
    const float m = u >= 0.5f ? 1.0f : 0.0f;
    cond[(n * cond_c + ch) * hwc + static_cast<size_t>(oy) * wc + ox] = __fsub_rn(__fmul_rn(m, 2.0f), 1.0f);
  }
}

__device__ __forceinline__ float clamp01(float v) { return fminf(fmaxf(v, 0.0f), 1.0f); }

// inpaint.py's composite on the ±1 batch entries: image = clamp((image + 1) / 2), mask = clamp((mask + 1) / 2),
// predicted = clamp((x + 1) / 2); (1 - mask) * image + mask * predicted, * 255, truncated to uint8. HWC in / out.
__global__ void inpaint_composite_kernel(const float* __restrict__ x, const uint8_t* __restrict__ img,
                                         const uint8_t* __restrict__ mask, size_t npix, uint8_t* __restrict__ out) {
  GRID_STRIDE(i, npix * 3) {
    const size_t p = i / 3;
    const float m01 = __fdiv_rn(static_cast<float>(mask[p]), 255.0f) >= 0.5f ? 1.0f : 0.0f;
    const float m = clamp01(__fdiv_rn(__fadd_rn(__fsub_rn(__fmul_rn(m01, 2.0f), 1.0f), 1.0f), 2.0f));
    const float u = __fsub_rn(__fmul_rn(__fdiv_rn(static_cast<float>(img[i]), 255.0f), 2.0f), 1.0f);
    const float im = clamp01(__fdiv_rn(__fadd_rn(u, 1.0f), 2.0f));
    const float pr = clamp01(__fdiv_rn(__fadd_rn(x[i], 1.0f), 2.0f));
    const float v = __fadd_rn(__fmul_rn(__fsub_rn(1.0f, m), im), __fmul_rn(m, pr));
    out[i] = static_cast<uint8_t>(__fmul_rn(v, 255.0f));
  }
}

}  // namespace sdb

using namespace sdb;
#define ST static_cast<cudaStream_t>(stream)

extern "C" int sdb_im2col3x3_concat(const float* x, int32_t nb, int32_t cx, int32_t h, int32_t w, const float* cond,
                                    int32_t cond_nb, int32_t cc, int32_t cond_h, int32_t cond_w, int32_t kpad,
                                    void* out_f16, sdb_stream_t stream) {
  SDB_REC(sdb_im2col3x3_concat(x, nb, cx, h, w, cond, cond_nb, cc, cond_h, cond_w, kpad, out_f16, s_));
  SDB_CHECK(x && cond && out_f16, "sdb_im2col3x3_concat: null pointer");
  SDB_CHECK(nb > 0 && h > 0 && w > 0 && cx > 0 && cc > 0, "sdb_im2col3x3_concat: bad sizes (nb=%d cx=%d cc=%d %dx%d)",
            nb, cx, cc, h, w);
  SDB_CHECK(cond_nb == nb && cond_h == h && cond_w == w,
            "sdb_im2col3x3_concat: conditioning [%d, %d, %d, %d] does not match x [%d, %d, %d, %d]", cond_nb, cc, cond_h,
            cond_w, nb, cx, h, w);
  SDB_CHECK(kpad % 64 == 0 && 9 * (cx + cc) <= kpad, "sdb_im2col3x3_concat: 9 * (%d + %d) channels exceed kpad %d",
            cx, cc, kpad);
  const size_t total = static_cast<size_t>(nb) * h * w * kpad;
  im2col3x3_concat_kernel<<<inpaint_grid(total), 256, 0, ST>>>(x, cx, cond, cc, nb, h, w, kpad,
                                                               static_cast<__half*>(out_f16));
  SDB_LAUNCH_CHECK();
  return 0;
}

extern "C" int sdb_inpaint_prepare(const uint8_t* image_u8, const uint8_t* mask_u8, int32_t nb, int32_t h, int32_t w,
                                   float* masked_nchw, float* cond, int32_t cond_c, int32_t cond_h, int32_t cond_w,
                                   int32_t mask_channel, sdb_stream_t stream) {
  SDB_REC(sdb_inpaint_prepare(image_u8, mask_u8, nb, h, w, masked_nchw, cond, cond_c, cond_h, cond_w, mask_channel, s_));
  SDB_CHECK(image_u8 && mask_u8 && masked_nchw && cond, "sdb_inpaint_prepare: null pointer");
  SDB_CHECK(nb > 0 && h > 0 && w > 0 && cond_h > 0 && cond_w > 0, "sdb_inpaint_prepare: bad sizes");
  SDB_CHECK(mask_channel >= 0 && mask_channel < cond_c, "sdb_inpaint_prepare: mask channel %d of %d", mask_channel,
            cond_c);
  const size_t n = static_cast<size_t>(nb) * 3 * h * w;
  inpaint_masked_image_kernel<<<inpaint_grid(n), 256, 0, ST>>>(image_u8, mask_u8, nb, h, w, masked_nchw);
  SDB_LAUNCH_CHECK();
  const size_t nc = static_cast<size_t>(nb) * cond_h * cond_w;
  inpaint_mask_channel_kernel<<<inpaint_grid(nc), 256, 0, ST>>>(mask_u8, nb, h, w, cond_h, cond_w, cond, cond_c,
                                                                mask_channel);
  SDB_LAUNCH_CHECK();
  return 0;
}

extern "C" int sdb_inpaint_composite(const float* x_nhwc, const uint8_t* image_u8, const uint8_t* mask_u8,
                                     int64_t npix, uint8_t* out_u8, sdb_stream_t stream) {
  SDB_REC(sdb_inpaint_composite(x_nhwc, image_u8, mask_u8, npix, out_u8, s_));
  SDB_CHECK(x_nhwc && image_u8 && mask_u8 && out_u8 && npix > 0, "sdb_inpaint_composite: bad arguments");
  inpaint_composite_kernel<<<inpaint_grid(static_cast<size_t>(npix) * 3), 256, 0, ST>>>(
      x_nhwc, image_u8, mask_u8, static_cast<size_t>(npix), out_u8);
  SDB_LAUNCH_CHECK();
  return 0;
}
