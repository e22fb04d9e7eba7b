// CLIP image embedding of retrieval databases (the reference's FrozenClipImageEmbedder, ldm/modules/encoders/
// modules.py:197-229): the preprocessing of a ragged batch straight into the patch-embedding GEMM's operand, the
// assembly of the token sequence after that GEMM, and the class-token gather before ln_post.
//
// Preprocessing restates kornia.geometry.resize(x, (S, S), 'bicubic', align_corners=True, antialias=False), which is
// F.interpolate(mode='bicubic', align_corners=True): torch's CUDA kernel (UpSampleBicubic2d.cu) with A = -0.75,
// source coordinate scale * dst with scale = (in - 1) / (out - 1) in fp32, border taps clamped, a plain copy when
// both sides already match; the four row interpolations at the source column first, then the one down the column.
// Then (x + 1) / 2 and (x - mean) / std, rounded to fp16 in the patch layout of CLIPVisionEmbeddings.patch_embedding
// (k = (c * P + py) * P + px, zero-padded to kpad). Each image is read in place from one packed buffer at its own
// size: fp32 NCHW in [-1, 1], or uint8 HWC converted as x / 127.5 - 1 (IEEE division) as each tap is read.
#include <cuda_fp16.h>

#include "../../include/sdb200.h"
#include "host.h"

namespace sdb {

static inline int cgrid(size_t n, int threads = 256) {
  size_t b = (n + threads - 1) / threads;
  size_t cap = static_cast<size_t>(sm_count()) * 16;
  return static_cast<int>(b < 1 ? 1 : (b > cap ? cap : b));
}

__device__ __forceinline__ float cubic1(float x, float A) { return ((A + 2) * x - (A + 3)) * x * x + 1; }
__device__ __forceinline__ float cubic2(float x, float A) { return ((A * x - 5 * A) * x + 8 * A) * x - 4 * A; }

__device__ __forceinline__ float cubic_interp1d(float x0, float x1, float x2, float x3, float t) {
  const float A = -0.75f;
  const float c0 = cubic2(t + 1.0f, A), c1 = cubic1(t, A);
  const float u = 1.0f - t;
  const float c2 = cubic1(u, A), c3 = cubic2(u + 1.0f, A);
  return x0 * c0 + x1 * c1 + x2 * c2 + x3 * c3;
}

template <bool U8>
__device__ __forceinline__ float tap(const void* src, long long off, int c, int y, int x, int h, int w) {
  y = min(max(y, 0), h - 1);
  x = min(max(x, 0), w - 1);
  if (U8) {
    const uint8_t v = static_cast<const uint8_t*>(src)[off + (static_cast<long long>(y) * w + x) * 3 + c];
    return __fsub_rn(__fdiv_rn(static_cast<float>(v), 127.5f), 1.0f);
  }
  return static_cast<const float*>(src)[off + (static_cast<long long>(c) * h + y) * w + x];
}

// One thread per element of the patch matrix [nb * g * g, kpad] (g = size / patch); table int64 [nb, 3] = (H, W,
// element offset of the image in src). resized (optional) fp32 [nb, 3, size, size] receives the interpolated values
// before (x + 1) / 2 and the normalisation.
template <bool U8>
__global__ void clip_resize_patches_kernel(const void* __restrict__ src, const int64_t* __restrict__ table, int nb,
                                           int size, int patch, int kpad, float m0, float m1, float m2, float s0,
                                           float s1, float s2, __half* __restrict__ patches, float* __restrict__ resized) {
  const int g = size / patch;
  const int kval = 3 * patch * patch;
  const size_t total = static_cast<size_t>(nb) * g * g * kpad;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(i % kpad);
    if (k >= kval) {
      patches[i] = __float2half_rn(0.f);
      continue;
    }
    size_t r = i / kpad;
    const int gx = static_cast<int>(r % g);
    r /= g;
    const int gy = static_cast<int>(r % g);
    const int b = static_cast<int>(r / g);
    const int px = k % patch, py = (k / patch) % patch, c = k / (patch * patch);
    const int oy = gy * patch + py, ox = gx * patch + px;
    const int h = static_cast<int>(table[3 * b]), w = static_cast<int>(table[3 * b + 1]);
    const long long off = table[3 * b + 2];
    float v;
    if (h == size && w == size) {
      v = tap<U8>(src, off, c, oy, ox, h, w);
    } else {
      const float sh = size > 1 ? static_cast<float>(h - 1) / static_cast<float>(size - 1) : 0.f;
      const float sw = size > 1 ? static_cast<float>(w - 1) / static_cast<float>(size - 1) : 0.f;
      const float ry = sh * oy, rx = sw * ox;
      const int iy = static_cast<int>(floorf(ry)), ix = static_cast<int>(floorf(rx));
      const float ty = ry - iy, tx = rx - ix;
      float rows[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int y = iy - 1 + j;
        rows[j] = cubic_interp1d(tap<U8>(src, off, c, y, ix - 1, h, w), tap<U8>(src, off, c, y, ix, h, w),
                                 tap<U8>(src, off, c, y, ix + 1, h, w), tap<U8>(src, off, c, y, ix + 2, h, w), tx);
      }
      v = cubic_interp1d(rows[0], rows[1], rows[2], rows[3], ty);
    }
    if (resized) resized[((static_cast<size_t>(b) * 3 + c) * size + oy) * size + ox] = v;
    const float mean = c == 0 ? m0 : (c == 1 ? m1 : m2), sd = c == 0 ? s0 : (c == 1 ? s1 : s2);
    patches[i] = __float2half_rn((((v + 1.0f) / 2.0f) - mean) / sd);
  }
}

// CLIPVisionEmbeddings after the patch GEMM: x [nb, np + 1, h] with row 0 = cls_pos (class embedding + pos[0]) and
// row 1 + p = pe[b * np + p] + pos_patches[p]. h % 4 == 0: float4 lanes.
__global__ void vit_embed_kernel(const float4* __restrict__ pe, const float4* __restrict__ cls_pos,
                                 const float4* __restrict__ pos_patches, int nb, int np, int h4, float4* __restrict__ x) {
  const size_t total = static_cast<size_t>(nb) * (np + 1) * h4;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int col = static_cast<int>(i % h4);
    const size_t row = i / h4;
    const int t = static_cast<int>(row % (np + 1));
    const size_t b = row / (np + 1);
    if (t == 0) {
      x[i] = cls_pos[col];
    } else {
      const float4 a = pe[(b * np + t - 1) * h4 + col], p = pos_patches[static_cast<size_t>(t - 1) * h4 + col];
      x[i] = make_float4(a.x + p.x, a.y + p.y, a.z + p.z, a.w + p.w);
    }
  }
}

// out[r] = x[r * row_stride], rows of dim floats
__global__ void rows_gather_kernel(const float* __restrict__ x, int rows, long long row_stride, int dim,
                                   float* __restrict__ out) {
  const size_t total = static_cast<size_t>(rows) * dim;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t r = i / dim;
    out[i] = x[r * row_stride * dim + i % dim];
  }
}

}  // namespace sdb

using namespace sdb;

extern "C" int sdb_clip_resize_patches(const void* src, int32_t src_u8, const int64_t* table, int32_t nb, int32_t size,
                                       int32_t patch, int32_t kpad, float m0, float m1, float m2, float s0, float s1,
                                       float s2, void* patches_f16, float* resized, sdb_stream_t stream) {
  SDB_REC(sdb_clip_resize_patches(src, src_u8, table, nb, size, patch, kpad, m0, m1, m2, s0, s1, s2, patches_f16, resized, s_));
  SDB_CHECK(src && table && patches_f16, "sdb_clip_resize_patches: null pointer");
  SDB_CHECK(nb > 0 && patch > 0 && size >= patch && size % patch == 0 && kpad >= 3 * patch * patch && kpad % 64 == 0,
            "sdb_clip_resize_patches: bad sizes (nb %d size %d patch %d kpad %d)", nb, size, patch, kpad);
  const size_t total = static_cast<size_t>(nb) * (size / patch) * (size / patch) * kpad;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (src_u8)
    clip_resize_patches_kernel<true><<<cgrid(total), 256, 0, st>>>(src, table, nb, size, patch, kpad, m0, m1, m2, s0,
                                                                    s1, s2, static_cast<__half*>(patches_f16), resized);
  else
    clip_resize_patches_kernel<false><<<cgrid(total), 256, 0, st>>>(src, table, nb, size, patch, kpad, m0, m1, m2, s0,
                                                                     s1, s2, static_cast<__half*>(patches_f16), resized);
  SDB_LAUNCH_CHECK();
  return 0;
}

extern "C" int sdb_vit_embed(const float* pe, const float* cls_pos, const float* pos_patches, int32_t nb, int32_t np,
                             int32_t dim, float* x, sdb_stream_t stream) {
  SDB_REC(sdb_vit_embed(pe, cls_pos, pos_patches, nb, np, dim, x, s_));
  SDB_CHECK(pe && cls_pos && pos_patches && x, "sdb_vit_embed: null pointer");
  SDB_CHECK(nb > 0 && np > 0 && dim > 0 && dim % 4 == 0, "sdb_vit_embed: bad sizes (nb %d np %d dim %d)", nb, np, dim);
  SDB_CHECK(((reinterpret_cast<uintptr_t>(pe) | reinterpret_cast<uintptr_t>(cls_pos) |
              reinterpret_cast<uintptr_t>(pos_patches) | reinterpret_cast<uintptr_t>(x)) & 15) == 0,
            "sdb_vit_embed: pointers must be 16-byte aligned");
  const size_t total = static_cast<size_t>(nb) * (np + 1) * (dim / 4);
  vit_embed_kernel<<<cgrid(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(pe), reinterpret_cast<const float4*>(cls_pos),
      reinterpret_cast<const float4*>(pos_patches), nb, np, dim / 4, reinterpret_cast<float4*>(x));
  SDB_LAUNCH_CHECK();
  return 0;
}

extern "C" int sdb_rows_gather(const float* x, int32_t rows, int64_t row_stride, int32_t dim, float* out,
                               sdb_stream_t stream) {
  SDB_REC(sdb_rows_gather(x, rows, row_stride, dim, out, s_));
  SDB_CHECK(x && out && rows > 0 && row_stride > 0 && dim > 0, "sdb_rows_gather: bad arguments");
  const size_t total = static_cast<size_t>(rows) * dim;
  rows_gather_kernel<<<cgrid(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, rows, row_stride, dim, out);
  SDB_LAUNCH_CHECK();
  return 0;
}
