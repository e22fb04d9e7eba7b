/*
 * sdb200 first-stage loss ABI: the forward half of the KL autoencoders' training objective
 * (ldm/modules/losses/contperceptual.py LPIPSWithDiscriminator, called from AutoencoderKL.validation_step,
 * ldm/models/autoencoder.py:372-383): the LPIPS perceptual distance over a VGG16 trunk, the PatchGAN discriminator's
 * 4x4 convs, and the per-sample reductions of the loss terms. The convs themselves run in sdb_gemm (include/sdb200.h,
 * SDB_ACT_RELU / SDB_ACT_LEAKY_RELU epilogues); the entry points here are the layers around them. Nothing here is on the
 * sampling path, so they live apart from sdb200.h and its entry-point table; they use its stream type and follow its
 * conventions: device pointers, 0 on success, sdb_last_error() for the message, and every call is recorded into an
 * open plan (sdb_plan_begin) like the entry points of sdb200.h.
 *
 * Every per-sample sum below is taken in fp64 in an order fixed by the shape alone (the sample's own size, never the
 * batch size), so a sample's value is the same bits alone, inside a batch and on a rerun.
 */
#ifndef SDB200_AE_LOSS_H
#define SDB200_AE_LOSS_H

#include "sdb200.h"

#ifdef __cplusplus
extern "C" {
#endif

/*
 * LPIPS ScalingLayer of both LPIPS inputs: out[s, y, x, c] = (in[s, c, y, x] - shift[c]) / scale[c] as one fp32
 * subtraction and one true fp32 division (taming lpips.py ScalingLayer.forward). in0 / in1: NCHW fp32 [nb, 3, h, w];
 * out: NHWC fp32 [2 * nb, h, w, 3], the in0 images first, then the in1 images (the operand of conv1_1 through
 * sdb_im2col3x3); shift / scale: fp32 [3] device tables.
 */
int sdb_lpips_scale(const float* in0, const float* in1, int32_t nb, int32_t h, int32_t w, const float* shift,
                    const float* scale, float* out, sdb_stream_t stream);

/*
 * MaxPool2d(kernel 2, stride 2) over NHWC fp16 [nb, h, w, c] -> [nb, h / 2, w / 2, c] (odd trailing rows / columns are
 * dropped, as torch floors). Exact; a NaN in a window propagates. c % 8 == 0; x and out 16-byte aligned.
 */
int sdb_maxpool2x2(const void* x, int32_t nb, int32_t h, int32_t w, int32_t c, void* out, sdb_stream_t stream);

/*
 * One LPIPS layer (taming lpips.py LPIPS.forward) for the two feature maps of one batch, f fp16 [2 * nb, hw, c] NHWC
 * (samples 0 .. nb-1 from in0, nb .. 2nb-1 from in1):
 *   per pixel p:  n = sqrt(sum_c f[p, c]^2) + 1e-10              (normalize_tensor; sum in fp64, sqrt rounded to fp32)
 *                 d_c = (f0[p, c] / n0 - f1[p, c] / n1)^2         (fp32 roundings as the reference)
 *                 v_p = sum_c lin_w[c] * d_c                       (lin{k}: 1x1 conv, no bias; fp64 sum)
 *   tap_b = (sum_p v_p) / hw                                       (spatial_average; fp64)
 *   acc[b] = tap_b (first != 0) or acc[b] + tap_b, and out[b] = (float)acc[b] when out is not NULL.
 * lin_w: fp32 [c]; acc: fp64 [nb]; out: fp32 [nb] or NULL; work: fp64 scratch of sdb_lpips_head_work(nb, hw)
 * elements. c in {64, 128, 256, 512}; f 16-byte aligned. Two launches: per-chunk partials, then a per-sample fold.
 */
int64_t sdb_lpips_head_work(int32_t nb, int32_t hw);
int sdb_lpips_head(const void* f, int32_t nb, int32_t hw, int32_t c, const float* lin_w, int32_t first, double* work,
                   double* acc, float* out, sdb_stream_t stream);

/*
 * General im2col for the k x k convs the TMA path does not take (the discriminator's 4x4 stride-2 / stride-1 convs,
 * taming discriminator/model.py NLayerDiscriminator): x fp16 NHWC [nb, h, w, c] -> out fp16 [nb * ho * wo, kpad],
 * column (ky * k + kx) * c + ch holding x[n, oy * stride - pad + ky, ox * stride - pad + kx, ch] (zero outside the
 * image), columns k * k * c .. kpad - 1 zero. A copy: exact. k * k * c <= kpad, kpad % 8 == 0; when c % 8 == 0, x and
 * out must be 16-byte aligned.
 */
int sdb_im2col(const void* x, int32_t nb, int32_t h, int32_t w, int32_t c, int32_t k, int32_t stride, int32_t pad,
               int32_t ho, int32_t wo, int32_t kpad, void* out, sdb_stream_t stream);

/*
 * Per-sample fp64 sums of LPIPSWithDiscriminator's terms (contperceptual.py:47-119), for nb samples:
 *   kind 1: out[b] = sum_i |a[b, i] - bb[b, i]|, a / bb fp32 [nb, n] (each difference one fp32 rounding, :49)
 *   kind 2: out[b] = 0.5 * sum (mean^2 + exp(lv) - 1 - lv), lv = clamp(logvar, -30, 20), the posterior KL against N(0, I)
 *           (distributions.py:34-45) with the element value in fp32 as the reference computes it; a = the NHWC moments
 *           fp32 [nb * n / cc, 2 * cc] (per pixel: cc means, then cc logvars); n = h * w * cc; bb unused
 *   kind 3: the discriminator logits l = a[(b * n + i) * cc] (column 0 of rows cc floats apart), n per sample:
 *           out[0*nb + b] = sum l, out[1*nb + b] = sum relu(1 - l), out[2*nb + b] = sum relu(1 + l),
 *           out[3*nb + b] = sum softplus(-l), out[4*nb + b] = sum softplus(l)      (g_loss, hinge_d_loss,
 *           vanilla_d_loss of taming vqperceptual.py; softplus as F.softplus: x > 20 ? x : log1p(exp(x)))
 * out: fp64 [1 or 5, nb]. The batch means and the weighting are left to the host. A NaN element makes its sample's sum
 * NaN, as in the reference: the clamp of kind 2 and the relu of kind 3 keep a NaN (torch.clamp, F.relu).
 */
int sdb_ae_loss_terms(const float* a, const float* bb, int32_t kind, int32_t nb, int64_t n, int32_t cc, double* out,
                      sdb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* SDB200_AE_LOSS_H */
