// Super-resolution with the LDM-BSR model (models/ldm/bsr_sr, notebook_helpers.py): the low-resolution image's conversion
// to the UNet's conditioning, and the patch tiling of LatentDiffusion's split_input_params path (ddpm.py:564-651,
// 705-763, 891-992): unfold a latent into overlapping tiles, and stitch tile outputs back with the delta_border weighting.
// Elementwise fp32 math uses explicit __f*_rn ops in the reference's operation order.
#include "../../include/sdb200.h"
#include "host.h"

namespace sdb {

static inline int superres_grid(size_t n, int threads = 256) {
  size_t b = (n + threads - 1) / threads;
  size_t cap = static_cast<size_t>(sm_count()) * 16;
  return static_cast<int>(b < 1 ? 1 : (b > cap ? cap : b));
}
#define GRID_STRIDE(i, n)                                                                      \
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < (n); \
       i += static_cast<size_t>(gridDim.x) * blockDim.x)

// get_cond("superresolution"): ToTensor (u / 255) then 2c - 1; uint8 HWC RGB in, fp32 NCHW out.
__global__ void lr_prepare_kernel(const uint8_t* __restrict__ img, int nb, int h, int w, float* __restrict__ out) {
  const size_t hw = static_cast<size_t>(h) * w;
  GRID_STRIDE(i, static_cast<size_t>(nb) * 3 * hw) {
    const size_t p = i % hw;
    const int c = static_cast<int>((i / hw) % 3);
    const size_t n = i / (3 * hw);
    const float u = __fdiv_rn(static_cast<float>(img[(n * hw + p) * 3 + c]), 255.0f);
    out[i] = __fsub_rn(__fmul_rn(2.0f, u), 1.0f);
  }
}

// nn.Unfold(kernel (kh, kw), stride (sy, sx)) + view: x [nb, c, h, w] -> tiles [ly*lx*nb, c, kh, kw], tile index
// l*nb + n with l = ty*lx + tx (Unfold's block order). A copy.
__global__ void patch_unfold_kernel(const float* __restrict__ x, int nb, int c, int h, int w, int kh, int kw, int sy,
                                    int sx, int lx, size_t total, float* __restrict__ out) {
  const size_t khw = static_cast<size_t>(kh) * kw;
  GRID_STRIDE(i, total) {
    const int px = static_cast<int>(i % kw);
    const int py = static_cast<int>((i / kw) % kh);
    const int ch = static_cast<int>((i / khw) % c);
    const size_t tn = i / (khw * c);
    const int n = static_cast<int>(tn % nb);
    const int l = static_cast<int>(tn / nb);
    const int y = (l / lx) * sy + py, xx = (l % lx) * sx + px;
    out[i] = x[((static_cast<size_t>(n) * c + ch) * h + y) * w + xx];
  }
}

// fold(o * weight) / norm, output-stationary: every output pixel sums the tiles that cover it, in the order
// nn.Fold's CPU col2im accumulates them (kernel offset ascending, i.e. tile row then tile column descending), from 0.
// No atomics: the result does not depend on scheduling. Tiles NCHW [L*nb, c, kh, kw] or NHWC [L*nb, kh, kw, c].
__global__ void patch_fold_kernel(const float* __restrict__ tiles, int nhwc, int nb, int c, int kh, int kw, int ly,
                                  int lx, int sy, int sx, const float* __restrict__ weight,
                                  const float* __restrict__ norm, int h, int w, float* __restrict__ out) {
  const size_t hw = static_cast<size_t>(h) * w;
  const size_t khw = static_cast<size_t>(kh) * kw;
  GRID_STRIDE(i, static_cast<size_t>(nb) * c * hw) {
    const int x = static_cast<int>(i % w);
    const int y = static_cast<int>((i / w) % h);
    const int ch = static_cast<int>((i / hw) % c);
    const int n = static_cast<int>(i / (hw * c));
    // tiles ty with ty*sy <= y < ty*sy + kh
    const int ty1 = min(y / sy, ly - 1), tx1 = min(x / sx, lx - 1);
    const int ty0 = y >= kh ? (y - kh) / sy + 1 : 0, tx0 = x >= kw ? (x - kw) / sx + 1 : 0;
    float acc = 0.0f;
    for (int ty = ty1; ty >= ty0; --ty) {
      const int py = y - ty * sy;
      for (int tx = tx1; tx >= tx0; --tx) {
        const int px = x - tx * sx;
        const int l = ty * lx + tx;
        const size_t t = static_cast<size_t>(l) * nb + n;
        const size_t pix = static_cast<size_t>(py) * kw + px;
        const float v = nhwc ? tiles[(t * khw + pix) * c + ch] : tiles[(t * c + ch) * khw + pix];
        acc = __fadd_rn(acc, __fmul_rn(v, weight[static_cast<size_t>(l) * khw + pix]));
      }
    }
    out[i] = __fdiv_rn(acc, norm[static_cast<size_t>(y) * w + x]);
  }
}

}  // namespace sdb

using namespace sdb;
#define ST static_cast<cudaStream_t>(stream)

extern "C" int sdb_lr_prepare(const uint8_t* image_u8, int32_t nb, int32_t h, int32_t w, float* out_nchw,
                              sdb_stream_t stream) {
  SDB_REC(sdb_lr_prepare(image_u8, nb, h, w, out_nchw, s_));
  SDB_CHECK(image_u8 && out_nchw, "sdb_lr_prepare: null pointer");
  SDB_CHECK(nb > 0 && h > 0 && w > 0, "sdb_lr_prepare: bad sizes (nb=%d %dx%d)", nb, h, w);
  const size_t n = static_cast<size_t>(nb) * 3 * h * w;
  lr_prepare_kernel<<<superres_grid(n), 256, 0, ST>>>(image_u8, nb, h, w, out_nchw);
  SDB_LAUNCH_CHECK();
  return 0;
}

extern "C" int sdb_patch_unfold(const float* x, int32_t nb, int32_t c, int32_t h, int32_t w, int32_t kh, int32_t kw,
                                int32_t sy, int32_t sx, float* tiles, sdb_stream_t stream) {
  SDB_REC(sdb_patch_unfold(x, nb, c, h, w, kh, kw, sy, sx, tiles, s_));
  SDB_CHECK(x && tiles, "sdb_patch_unfold: null pointer");
  SDB_CHECK(nb > 0 && c > 0 && kh > 0 && kw > 0 && sy > 0 && sx > 0,
            "sdb_patch_unfold: bad sizes (nb=%d c=%d kernel %dx%d stride %dx%d)", nb, c, kh, kw, sy, sx);
  SDB_CHECK(kh <= h && kw <= w, "sdb_patch_unfold: kernel %dx%d larger than the input %dx%d", kh, kw, h, w);
  const int ly = (h - kh) / sy + 1, lx = (w - kw) / sx + 1;
  const size_t total = static_cast<size_t>(ly) * lx * nb * c * kh * kw;
  patch_unfold_kernel<<<superres_grid(total), 256, 0, ST>>>(x, nb, c, h, w, kh, kw, sy, sx, lx, total, tiles);
  SDB_LAUNCH_CHECK();
  return 0;
}

extern "C" int sdb_patch_fold(const float* tiles, int32_t tiles_nhwc, int32_t nb, int32_t c, int32_t kh, int32_t kw,
                              int32_t ly, int32_t lx, int32_t sy, int32_t sx, const float* weight, const float* norm,
                              int32_t h, int32_t w, float* out_nchw, sdb_stream_t stream) {
  SDB_REC(sdb_patch_fold(tiles, tiles_nhwc, nb, c, kh, kw, ly, lx, sy, sx, weight, norm, h, w, out_nchw, s_));
  SDB_CHECK(tiles && weight && norm && out_nchw, "sdb_patch_fold: null pointer");
  SDB_CHECK(nb > 0 && c > 0 && kh > 0 && kw > 0 && ly > 0 && lx > 0 && sy > 0 && sx > 0,
            "sdb_patch_fold: bad sizes (nb=%d c=%d kernel %dx%d tiles %dx%d stride %dx%d)", nb, c, kh, kw, ly, lx, sy,
            sx);
  SDB_CHECK(h == (ly - 1) * sy + kh && w == (lx - 1) * sx + kw,
            "sdb_patch_fold: %dx%d tiles of %dx%d at stride %dx%d do not cover the output %dx%d exactly", ly, lx, kh,
            kw, sy, sx, h, w);
  const size_t n = static_cast<size_t>(nb) * c * h * w;
  patch_fold_kernel<<<superres_grid(n), 256, 0, ST>>>(tiles, tiles_nhwc ? 1 : 0, nb, c, kh, kw, ly, lx, sy, sx,
                                                        weight, norm, h, w, out_nchw);
  SDB_LAUNCH_CHECK();
  return 0;
}
