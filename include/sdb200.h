/*
 * sdb200 — C ABI of the H100-native latent-diffusion kernels.
 *
 * The reference (CompVis/stable-diffusion) has no FFI: its plug-in boundary is `instantiate_from_config`
 * (ldm/util.py:78-93) plus the duck-typed nn.Module contracts around the denoising loop. This header is the
 * boundary a maintainer binds instead (ctypes stub in INTEGRATION.md): plain pointers and sizes, no torch
 * types. Every entry point enqueues work on `stream` and returns immediately; 0 = OK, non-zero = error
 * (text via sdb_last_error()). All device pointers are owned by the caller.
 *
 * Each function cites the reference operation(s) it replaces.
 */
#ifndef SDB200_H
#define SDB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* sdb_stream_t; /* cudaStream_t */

const char* sdb_last_error(void);
int sdb_version(void);
int sdb_sm_count(void);
long long sdb_launch_count(void); /* kernels launched through this library since load */
/* Debug only: subsequent sdb_gemm launches write per-CTA phase timestamps (8-word launch header + 8 words per CTA,
 * 1288 words per launch) into the device buffer `buf` of n_words uint64; NULL switches tracing off. Returns the
 * number of words handed out since the previous call. Used by scripts/timeline_unet.py. The stamps are written only by
 * a library built with -DSDB_TRACE (SDB_BUILD_TRACE=1 python build.py); the production build leaves the buffer untouched. */
long long sdb_debug_trace(void* buf, int64_t n_words);

/* ---- epilogue activations ---- */
enum {
  SDB_ACT_NONE = 0,
  SDB_ACT_GEGLU = 1,      /* out[:, j] = x_j * gelu_erf(gate_j); ldm/modules/attention.py:37-45 (weights packed
                             so each accumulator tile holds [x half | gate half]) */
  SDB_ACT_QUICK_GELU = 2, /* x * sigmoid(1.702 x): CLIP MLP (transformers CLIPMLP, quick_gelu) */
  SDB_ACT_SILU = 3,       /* x * sigmoid(x): time_embed MLP, openaimodel.py:506-511 */
  SDB_ACT_GELU = 4,       /* gelu_erf(x) = 0.5 x (1 + erf(x / sqrt 2)), exact nn.GELU: the BERTEmbedder feed-forward
                             (x_transformer.py:199-202) */
                          /* 5 is not an activation: sdb_gemm rejects it, as it rejects every value not listed here */
  SDB_ACT_RELU = 6,       /* x < 0 ? 0 : x: the LPIPS VGG16 trunk's ReLUs (include/sdb200_ae_loss.h); a NaN stays NaN,
                             as in torch.relu */
  SDB_ACT_LEAKY_RELU = 7  /* x > 0 ? x : 0.2 x: the PatchGAN discriminator's LeakyReLU(0.2); a NaN stays NaN. The two
                             ReLU activations run in their own epilogue instantiation and never split K: a requested
                             split-K factor resolves to 1 */
};

/*
 * Tensor-core GEMM / implicit-GEMM convolution (wgmma + TMA), fp16 operands, fp32 accumulate:
 *
 *   acc[m, n] = sum_k A[m, k] * B[n, k]
 *   v         = alpha * acc + bias[n] + film[m / rows_per_sample, n] + residual[m, n]
 *   out       = act(v)   written as fp16 and/or fp32, row stride ldo
 *
 * A is one to four NHWC fp16 tensors concatenated along channels: the UNet skip concat (openaimodel.py:736) folded
 * into the K loop, or the hi/lo fp16 halves of one fp32 activation ([A_hi | A_lo | A_hi] against [W_hi | W_hi | W_lo]
 * recovers ~fp32 operand precision for the few 1x1 convs that act on the raw residual stream). taps = 1: plain [rows, C] matrix (nn.Linear, 1x1 conv:
 * attention.py:161-168,233-248; openaimodel.py:241). taps = 9: 3x3 conv, stride 1, zero pad 1
 * (openaimodel.py:204,230,519,685; model.py:44-50,94-118) with B laid out [n, 9*(c0+c1)], k = tap*(c0+c1)+c.
 * All channel counts must be multiples of 64.
 */
typedef struct sdb_gemm_desc {
  const void* a0;        /* fp16 [nb, h, w, c0] */
  const void* a1;        /* fp16 [nb, h, w, c1] or NULL; further sources a2, a3 likewise (contiguous from a0) */
  const void* a2;
  const void* a3;
  int32_t c0, c1, c2, c3;
  int32_t nb, h, w;      /* rows M = nb*h*w */
  int32_t taps;          /* 1 or 9 */
  const void* b;         /* fp16 [n, taps*(c0+c1)]. Unless b_dynamic is set, b is streamed ahead of the programmatic-
                            launch wait (griddepcontrol.wait), while earlier kernels of the stream may still run: it must
                            not be written by any kernel still in flight (in practice: packed weights) */
  int32_t n;
  float alpha;
  const float* bias;     /* [n] or NULL. Read ahead of the programmatic-launch wait by the split-K second pass: it must not
                            be written by any kernel still in flight (in practice: packed weights) */
  const float* film;     /* [M / rows_per_sample, ldf] or NULL (timestep FiLM add, openaimodel.py:271-274) */
  int32_t ldf;           /* row stride of film (0 = n) */
  int32_t rows_per_sample;
  const float* residual; /* fp32 [M, ldr] or NULL */
  int32_t ldr;
  int32_t act;           /* SDB_ACT_* */
  void* out_f16;         /* fp16 [M, ldo] or NULL */
  void* out_f16_lo;      /* optional fp16 [M, ldo]: fp16(v - float(out_f16)), the low half of a hi/lo operand split */
  float* out_f32;        /* fp32 [M, ldo] or NULL */
  int32_t ldo;           /* 0 = dense (n, or n/2 for GEGLU) */
  int32_t block_n;       /* 0 = auto; else one of 32,64,128,160,256 */
  int32_t splits;        /* split-K factor: >1 explicit, 0/1 none, -1 auto (picked with block_n by the tile model,
                            bounded by workspace_floats); split-K needs workspace of splits*M*n floats */
  float* workspace;
  int64_t workspace_floats;
  void* stats_out;       /* optional fp32 [M / rows_per_sample, T, n / stats_group, 2]: per-tile partial {sum, sum of squares}
                            of the fp32 output per channel group, STORED by the epilogue of the tile that owns the slot
                            (no atomics, no zeroing, bit-reproducible) — the GroupNorm statistics of the tensor being
                            produced, so no separate reduction pass reads it again. T comes from sdb_gemm_plan; the
                            consumer (sdb_groupnorm) folds the T slots */
  int32_t stats_prezeroed; /* unused (kept for layout compatibility) */
  int32_t b_dynamic;       /* non-zero: b is read only after the programmatic-launch wait. Required whenever b may be
                              written by a kernel that can still be in flight: not just the preceding one, but any
                              earlier kernel of an unbroken chain of programmatic launches, since every kernel lets its
                              successor start before it finishes (e.g. V^T = W_v . X^T, which swaps the operand roles) */
  int32_t conv_stride;     /* taps = 9 only. 0/1: stride 1. 2: stride-2 conv read straight from the NHWC input through
                              strided TMA boxes (no im2col): Downsample, openaimodel.py:149-153; model.py:72-76 */
  int32_t conv_shift;      /* input pixel of output o, tap t (per axis) = stride*o + t - 1 + conv_shift: 0 = zero pad 1
                              on every side (UNet), 1 = pad only right/bottom (the VAE's asymmetric F.pad, model.py:73) */
  int32_t in_h, in_w;      /* input height / width when they differ from the output's h / w (stride 2); 0 = h, w */
  int32_t pair;            /* 0 auto, 1 single CTAs, 2 CTA pairs: two CTAs of a cluster compute one 256 x block_n tile
                              as a 2-CTA cluster, each loading half of the weight tile and multicasting it to both (block_n 128/160/256) */
  int32_t splitk_mode;     /* how split-K partials meet. 0 auto, 1 fp32 planes in `workspace` + a second kernel,
                              2 inside a thread-block cluster through distributed shared memory (2 or 4 slices, no
                              workspace traffic, fused epilogue in the same kernel) */
  int32_t stats_group;     /* channels per statistics entry (0/1 = per channel); must divide n and the tile width */
} sdb_gemm_desc;

int sdb_gemm(const sdb_gemm_desc* d, sdb_stream_t stream);
/* The tile configuration sdb_gemm would use for `d` (explicit requests honoured): out[0..4] = block_n, CTAs per tile
 * (1 | 2), split-K factor, split-K mode (0 none | 1 workspace | 2 cluster), statistics slots per sample T (0 when
 * stats_out is NULL). stats_out, when set, is written as fp32 [samples][T][n / stats_group][2]. */
int sdb_gemm_plan(const sdb_gemm_desc* d, int32_t* out);

/*
 * Fused multi-head attention (flash-style, S/P/O in registers), replaces CrossAttention.forward's
 * einsum -> scale -> softmax -> einsum (ldm/modules/attention.py:178-192) without materialising N x N.
 *   q  : fp16 [batch, nq,  heads*hs]     (row stride ldq elements; head h at column h*hs)
 *   k  : fp16 [batch, nkv, heads*hs]     (row stride ldk)
 *   vt : fp16 [batch, heads*hs, ldvt]    (V transposed: channel-major, head h at row h*hs, nkv valid columns)
 *   out: fp16 [batch, nq, heads*d]       (row stride ldo; unpadded head dim d)
 * hs = head_stride, the elements between consecutive heads (a multiple of 8, >= d; 0 means dpad). head_stride = d is
 * the packed layout the projections produce; elements d .. hs-1 of a head, if any, are never read.
 * dpad in {64,128,192}: d rounded up to the kernel's 64-column K panels.
 * dpad in {384,512,576,960}: the single-head kernels (the AutoencoderKL AttnBlock at 512, the num_heads-1
 * SpatialTransformers of the class-conditional ImageNet LDM at 384 / 576 / 960); they require heads == 1, d == dpad,
 * causal == 0, head_stride 0 or d, and ldq, ldk, ldvt, ldo, o_batch_stride multiples of 8.
 * Any other descriptor returns nonzero with a message in sdb_last_error() and launches nothing.
 * scale multiplies q.k before softmax (applied after the dot product, attention.py:180); it must be positive and
 * finite (the kernel takes the row maximum before scaling).
 * causal != 0 masks kv index > q index (CLIP text encoder).
 */
typedef struct sdb_attn_desc {
  const void* q;
  const void* k;
  const void* vt;
  void* out;
  int32_t batch, heads, nq, nkv, d, dpad;
  int32_t ldq, ldk, ldvt, ldo;
  int64_t q_batch_stride, k_batch_stride, vt_batch_stride, o_batch_stride; /* elements */
  float scale;
  int32_t causal;
  int32_t head_stride;
} sdb_attn_desc;

int sdb_attention(const sdb_attn_desc* d, sdb_stream_t stream);

/*
 * GroupNorm(32) [+ SiLU] over NHWC fp32 input that may be the channel concat of two tensors
 * (ldm/modules/diffusionmodules/util.py:199-216 GroupNorm32 in fp32; attention.py:76-77 Normalize eps 1e-6;
 * model.py:38-39). Statistics: fp32 per-block partials, folded in fp64 by the last block of each sample. Writes the normalised fp16 operand
 * for the following conv and optionally a raw fp16 cast of the (concatenated) input for the 1x1 skip conv.
 */
int sdb_groupnorm(const float* x0, const float* x1, int32_t c0, int32_t c1, int32_t nb, int32_t hw, int32_t groups,
                  const float* gamma /* gamma / beta are read ahead of the programmatic-launch wait, while earlier
                                        kernels of the stream may still run: they must not be written by any kernel
                                        still in flight (in practice: packed weights) */,
                  const float* beta, float eps, int32_t silu, void* out_f16, void* raw_f16,
                  void* out_lo_f16 /* optional low half of the normalised output (hi/lo split) */,
                  void* raw_lo_f16 /* optional low half of the raw cast */,
                  void* stats_ws /* scratch: nb * (128*groups*2 + groups*2 + 1) * 4 bytes */,
                  const void* chan_stats0 /* optional fp32 [nb, stats_t0, c0 / stats_group, 2] from sdb_gemm.stats_out
                                             (skips the stats pass) */,
                  const void* chan_stats1 /* same for x1, [nb, stats_t1, c1 / stats_group, 2] */,
                  int32_t stats_t0, int32_t stats_t1 /* partial slots per sample (sdb_gemm_plan) */,
                  int32_t stats_group /* channels per entry; must divide c0, c1 and (c0 + c1) / groups */,
                  sdb_stream_t stream);

/*
 * GroupNorm(32) [+ SiLU] of one NHWC fp32 tensor [nb, h, w, c] with the two options of the attention-block UNet's
 * ResBlock (openaimodel.py:255-275), writing the fp16 operand of the following 3x3 conv:
 *   modulation (scale, shift non-NULL; use_scale_shift_norm, :267-271): GN(x) * (1 + scale[n, c]) + shift[n, c], with
 *     scale / shift rows ldm floats apart (column slices of the FiLM output);
 *   resample (up / down ResBlocks, :256-261): 0 none, 1 the activated output 2x2 average-pooled ([nb, h/2, w/2, c]),
 *     2 nearest-2x upsampled ([nb, 2h, 2w, c]).
 * Statistics come from chan_stats (fused GEMM statistics, as in sdb_groupnorm; groups <= 32) or, when NULL, from a
 * reduction pass. stats_ws as in sdb_groupnorm.
 */
int sdb_groupnorm_mod(const float* x, int32_t c, int32_t nb, int32_t h, int32_t w, int32_t groups, const float* gamma,
                      const float* beta, float eps, int32_t silu, const float* scale, const float* shift, int32_t ldm,
                      int32_t resample, void* out_f16, void* stats_ws, const void* chan_stats, int32_t stats_t,
                      int32_t stats_group, sdb_stream_t stream);

/* LayerNorm over the last dim of fp32 [rows, c] -> fp16 (attention.py:203-205, eps 1e-5). gamma / beta are read ahead
 * of the programmatic-launch wait (c = 320, 512, 640, 768, 1280 with 8-byte aligned operands), while earlier kernels of
 * the stream may still run: they must not be written by any kernel still in flight (in practice: packed weights). */
int sdb_layernorm(const float* x, int32_t rows, int32_t c, const float* gamma, const float* beta, float eps,
                  void* out_f16, float* out_f32 /* optional */, sdb_stream_t stream);

/* Row softmax of fp32 [rows, cols] * scale -> fp16 (VAE AttnBlock, model.py:191-194). */
int sdb_softmax_rows(const float* x, int32_t rows, int32_t cols, float scale, void* out_f16, sdb_stream_t stream);

/* ---- layout / elementwise helpers ---- */
/* NCHW fp32 -> NHWC fp32 (+ optional fp16 copy); NHWC fp32 -> NCHW fp32 */
int sdb_nchw_to_nhwc(const float* x, int32_t nb, int32_t c, int32_t hw, float* out_f32, void* out_f16,
                     sdb_stream_t stream);
int sdb_nhwc_to_nchw(const float* x, int32_t nb, int32_t c, int32_t hw, float* out, sdb_stream_t stream);
/* explicit im2col for the few convs the TMA path does not cover (C_in not a multiple of 64, stride 2,
 * asymmetric pad): out fp16 [nb*ho*wo, kpad], k = (ky*3+kx)*c + ch, zero padded to kpad.
 * pad_lo applies top/left, bottom/right pad is implied by ho/wo (openaimodel.py:149-153; model.py:72-76). */
int sdb_im2col3x3(const float* x, int32_t nb, int32_t h, int32_t w, int32_t c, int32_t stride, int32_t pad_lo,
                  int32_t ho, int32_t wo, int32_t kpad, void* out_f16, sdb_stream_t stream);
/* im2col of a concat-conditioned UNet's conv_in (DiffusionWrapper "concat", ddpm.py:1405-1407) straight from the two
 * NCHW fp32 sources x [nb, cx, h, w] and cond [cond_nb, cc, cond_h, cond_w] (their dims must agree): 3x3, stride 1,
 * pad 1, out fp16 [nb*h*w, kpad], k = (ky*3+kx)*(cx+cc) + ch, channels cx.. read from cond; 9*(cx+cc) <= kpad.
 * Values equal im2col3x3 of the NHWC concat bit for bit. */
int sdb_im2col3x3_concat(const float* x, int32_t nb, int32_t cx, int32_t h, int32_t w, const float* cond,
                         int32_t cond_nb, int32_t cc, int32_t cond_h, int32_t cond_w, int32_t kpad, void* out_f16,
                         sdb_stream_t stream);
/* nearest 2x upsample NHWC fp32 -> fp16 (openaimodel.py:116; model.py:54). c % 4 == 0; x 16-byte and out_f16 8-byte
 * aligned. */
int sdb_upsample2x(const float* x, int32_t nb, int32_t h, int32_t w, int32_t c, void* out_f16, sdb_stream_t stream);
/* fp32 -> fp16 cast, optional transpose of [rows, cols] per batch into [cols, ldo] */
int sdb_cast_f16(const float* x, int64_t n, void* out_f16, sdb_stream_t stream);
int sdb_transpose_f16(const void* x, int32_t batch, int32_t rows, int32_t cols, int32_t ldx, void* out,
                      int32_t ldo, sdb_stream_t stream);
/* sinusoidal timestep embedding [cos | sin] (util.py:151-171): t[n] -> fp16 [n, dim] */
int sdb_timestep_embedding(const float* t, int32_t n, int32_t dim, float max_period, void* out_f16,
                           sdb_stream_t stream);
/* fp32 variant of the above, and the small-M fp32-activation linear (time_embed MLP + all emb_layers,
 * openaimodel.py:506-511,217-223): out[m, j] = act(x[m, :] . w[j, :] + bias[j]), w fp16 [n, k], act NONE|SILU */
int sdb_timestep_embedding_f32(const float* t, int32_t n, int32_t dim, float max_period, float* out,
                               sdb_stream_t stream);
int sdb_linear_small(const float* x, int32_t m, int32_t k, const void* w_f16, int32_t n, const float* bias,
                     int32_t act, float* out_f32, void* out_f16, sdb_stream_t stream);
/* y = silu(x) fp32 -> fp16 */
int sdb_silu_f16(const float* x, int64_t n, void* out_f16, sdb_stream_t stream);

/*
 * One fused sampler update (classifier-free guidance + PLMS / DDIM step), replacing ~25 elementwise
 * launches per step (ldm/models/diffusion/plms.py:182-186,199-236; ddim.py:174-204).
 *   eps2   : fp32 [2, n] = [e_uncond; e_cond] (or [1, n] when guidance is off: scale==1)
 *   e_t    = e_uncond + scale * (e_cond - e_uncond)
 *   order 0: e' = e_t (DDIM / first PLMS half-step); 1..3: Adams-Bashforth with old eps h1,h2,h3
 *   order 4 (PLMS step 0 second half): e' = (e_t_old + e_t)/2 where e_t_old = h1
 *   pred_x0 = (x - sqrt(1-a_t) e') / sqrt(a_t);  x_prev = sqrt(a_prev) pred_x0 + sqrt(1-a_prev-sigma^2) e' + sigma*noise
 * coef = {a_t, a_prev, sigma_t, sqrt_one_minus_a_t}; e_t is written to e_out (for the multistep history).
 */
int sdb_sampler_step(const float* x, const float* eps2, const float* eps_cond /* NULL: eps2 + n. Otherwise the
                     conditional half lives elsewhere - e.g. in the peer GPU's buffer mapped over NVLink (CFG halves
                     evaluated on two GPUs, SURVEY 8f-2): the exchange is then the kernel's own peer loads */,
                     int32_t guided, float scale, int32_t order, const float* h1,
                     const float* h2, const float* h3, const float* noise, float a_t, float a_prev, float sigma_t,
                     float sqrt_one_minus_a_t, int64_t n, float* x_prev, float* x_prev2 /* optional second copy: the
                     cond half of the guidance-doubled latent batch */, float* pred_x0, float* e_out,
                     sdb_stream_t stream);

/*
 * DPM-Solver++ (multistep, order <= 2, data prediction) update fused with classifier-free guidance and the
 * noise -> x0 conversion: replaces model_wrapper.model_fn + DPM_Solver.data_prediction_fn +
 * dpm_solver_first_update / multistep_dpm_solver_second_update
 * (ldm/models/diffusion/dpm_solver/dpm_solver.py:321-346, 386-399, 504-533, 755-789).
 *   e   = e_uncond + scale (e_cond - e_uncond)            (eps2 as in sdb_sampler_step)
 *   m0  = (x - sigma_s e) / alpha_s                        -> m_out (the history entry for the next step)
 *   order 1: x_t = c_x x - c_m m0                          c_x = sigma_t / sigma_s, c_m = alpha_t * expm1(-h)
 *   order 2: x_t = c_x x - c_m m0 - (c_m / 2) inv_r0 (m0 - m_prev)      c_m = alpha_t * (exp(-h) - 1)
 * The host computes the scalars in fp32 exactly as the reference's schedule tensors do.
 */
int sdb_dpm_solver_step(const float* x, const float* eps2, const float* eps_cond /* as in sdb_sampler_step */,
                        int32_t guided, float scale, float sigma_s, float alpha_s,
                        int32_t order, const float* m_prev, float c_x, float c_m, float inv_r0, int64_t n,
                        float* m_out, float* x_out, float* x_out2 /* optional second copy */, sdb_stream_t stream);

/* Inpainting blend of the samplers' mask branch (plms.py:147-150, ddim.py:144-147), in place:
 * img = img_orig * mask + (1 - mask) * img; mask fp32 [nb, 1 or c, hw]; img2: optional second copy of the result. */
int sdb_mask_blend(const float* img_orig, const float* mask, int32_t mask_channels, int32_t nb, int32_t c, int64_t hw,
                   float* img, float* img2, sdb_stream_t stream);

/* VAE posterior sample + scale (distributions.py:24-37, ddpm.py:542-549): moments NHWC fp32 [rows, 8]
 * -> z NCHW. And image post-process clamp((x+1)/2,0,1)*255 -> uint8 NHWC (txt2img.py:314-324). */
int sdb_vae_sample(const float* moments, const float* noise_nchw, int32_t nb, int32_t hw, float scale_factor,
                   float* z_nchw, sdb_stream_t stream);
int sdb_to_uint8(const float* x_nhwc, int64_t n, uint8_t* out, sdb_stream_t stream);
/* 2x2 resample of the fp32 residual stream (ResBlock.x_upd, openaimodel.py:209-214,260): NHWC [nb, h, w, c] ->
 * mode 1: 2x2 average pool [nb, h/2, w/2, c] (summed in avg_pool2d's order, then / 4); mode 2: nearest 2x [nb, 2h, 2w, c].
 * c % 4 == 0; x and out 16-byte aligned. */
int sdb_resample_f32(const float* x, int32_t nb, int32_t h, int32_t w, int32_t c, int32_t mode, float* out,
                     sdb_stream_t stream);
/* Ancestral DDPM step, LatentDiffusion.p_sample with clip_denoised=False (ddpm.py:1047-1108), one timestep per call:
 *   x0 = sqrt_recip_ac * x - sqrt_recipm1_ac * eps;  mean = coef1 * x0 + coef2 * x;  x' = mean + sigma * noise
 * with sigma = nonzero_mask * exp(0.5 * posterior_log_variance_clipped[t]) (noise NULL: x' = mean). fp32, rounded per
 * operation as the reference's tensor ops; x0 optionally written (the intermediates). */
int sdb_ddpm_step(const float* x, const float* eps, const float* noise, float sqrt_recip_alphas_cumprod,
                  float sqrt_recipm1_alphas_cumprod, float posterior_mean_coef1, float posterior_mean_coef2, float sigma,
                  int64_t n, float* x_out, float* x0_out, sdb_stream_t stream);
/* Vector quantizer of a VQ first stage (taming VectorQuantizer2.forward, legacy, no remap): z fp32 NHWC [m, e_dim],
 * first multiplied by `scale` (1 / scale_factor of decode_first_stage); codebook fp32 [n_e, e_dim] with code_sq[j] =
 * sum(codebook[j]^2) precomputed once per weight load. Index = argmin_j sum(z^2) + code_sq[j] - 2 z.e_j, the lowest
 * index on ties; z_q = z + (e - z) in fp32 (the straight-through value, not always e bit for bit). indices (int64 [m])
 * may be NULL. e_dim 1 .. 8, any n_e (the codebook streams through shared memory). */
int sdb_vq_quantize(const float* z, int64_t m, int32_t e_dim, float scale, const float* codebook, const float* code_sq,
                    int32_t n_e, float* z_q, int64_t* indices, sdb_stream_t stream);
/* Inpainting pre-processing (scripts/inpaint.py make_batch + the interpolated mask channel), fp32 in the reference's
 * operation order: image uint8 RGB [nb, h, w, 3], mask uint8 L [nb, h, w], m = (mask / 255 >= 0.5).
 * masked_nchw fp32 [nb, 3, h, w] = ((1 - m) * (image / 255)) * 2 - 1 (the VQ encoder's input); channel mask_channel of
 * cond fp32 [nb, cond_c, cond_h, cond_w] = nearest-resized m * 2 - 1 (F.interpolate's src = floor(dst * (float)in / out)).
 * The other channels of cond are not written. */
int sdb_inpaint_prepare(const uint8_t* image_u8, const uint8_t* mask_u8, int32_t nb, int32_t h, int32_t w,
                        float* masked_nchw, float* cond, int32_t cond_c, int32_t cond_h, int32_t cond_w,
                        int32_t mask_channel, sdb_stream_t stream);
/* Inpainting composite (scripts/inpaint.py): x_nhwc fp32 [npix, 3] the decoded image, image uint8 [npix, 3], mask
 * uint8 [npix]; out uint8 [npix, 3] = trunc(255 * ((1 - m) * clamp(((image / 255) * 2 - 1 + 1) / 2) + m * clamp((x + 1) / 2)))
 * with m = (mask / 255 >= 0.5), fp32 in the reference's order. */
int sdb_inpaint_composite(const float* x_nhwc, const uint8_t* image_u8, const uint8_t* mask_u8, int64_t npix,
                          uint8_t* out_u8, sdb_stream_t stream);
/* Super-resolution conditioning (notebook_helpers.py get_cond): image uint8 RGB [nb, h, w, 3] -> out fp32
 * [nb, 3, h, w] = 2 * (image / 255) - 1, fp32 in the reference's order (ToTensor, then 2c - 1). */
int sdb_lr_prepare(const uint8_t* image_u8, int32_t nb, int32_t h, int32_t w, float* out_nchw, sdb_stream_t stream);
/* Patch tiling of LatentDiffusion's split_input_params path (ddpm.py:611-651): nn.Unfold(kernel (kh, kw), stride
 * (sy, sx)) of x fp32 [nb, c, h, w] viewed as tiles fp32 [L*nb, c, kh, kw], tile index l*nb + n, l = ty*lx + tx,
 * ly = (h - kh) / sy + 1, lx = (w - kw) / sx + 1 (rows / columns the tiles miss are dropped, as by Unfold). A copy. */
int sdb_patch_unfold(const float* x, int32_t nb, int32_t c, int32_t h, int32_t w, int32_t kh, int32_t kw, int32_t sy,
                     int32_t sx, float* tiles, sdb_stream_t stream);
/* The stitch of the split path: out fp32 [nb, c, h, w] = fold(tiles * weight) / norm with nn.Fold(kernel (kh, kw),
 * stride (sy, sx)); tiles fp32 [ly*lx*nb, c, kh, kw] (tiles_nhwc 0) or [ly*lx*nb, kh, kw, c] (1) in sdb_patch_unfold's
 * order, weight fp32 [ly*lx, kh, kw] (get_weighting, per tile), norm fp32 [h, w] (fold of the weights). The tiles must
 * cover the output exactly: h = (ly - 1) * sy + kh, w = (lx - 1) * sx + kw. Each output element sums its covering tiles
 * in a fixed order (no atomics): deterministic. */
int sdb_patch_fold(const float* tiles, int32_t tiles_nhwc, int32_t nb, int32_t c, int32_t kh, int32_t kw, int32_t ly,
                   int32_t lx, int32_t sy, int32_t sx, const float* weight, const float* norm, int32_t h, int32_t w,
                   float* out_nchw, sdb_stream_t stream);
/* SpatialRescaler (ldm/modules/encoders/modules.py:106-134) with method 'bilinear', multiplier 0.5: n_stages
 * (0..3) x F.interpolate(scale_factor=0.5, mode='bilinear') of x fp32 [nb, cin, h, w] (each stage floor(side / 2),
 * computed as torch's CUDA kernel orders it), then the optional channel_mapper 1x1 conv: weight fp32 [cout, cin],
 * bias fp32 [cout] or NULL, accumulated by fma over cin ascending, bias last. weight NULL: no mapper, cout = cin.
 * out fp32 [nb, cout, h >> n_stages, w >> n_stages]. */
int sdb_spatial_rescale(const float* x_nchw, int32_t nb, int32_t cin, int32_t h, int32_t w, int32_t n_stages,
                        const float* weight, const float* bias, int32_t cout, float* out_nchw, sdb_stream_t stream);
/* The same SpatialRescaler applied to the one-hot of uint8 label ids [nb, h, w] (ids < cin <= 256; the caller checks
 * them), without materialising it: each output pixel sums W[o, k] * count_k / 4^n_stages over the classes k present in
 * its window, ascending. Bit-identical to sdb_spatial_rescale on the one-hot. The channel map (weight) is required. */
int sdb_seg_labels_rescale(const uint8_t* labels, int32_t nb, int32_t cin, int32_t h, int32_t w, int32_t n_stages,
                           const float* weight, const float* bias, int32_t cout, float* out_nchw, sdb_stream_t stream);
/* Exact top-k by inner product (knn.cu; the score_brute_force searcher of scripts/knn2img.py): db fp16 [n, dim]
 * row-major (n < 2^31), queries fp16 [b, dim]; dim a multiple of 64, <= 768; 1 <= b <= 64; 1 <= k <= min(64, n).
 * out_score fp32 [b, k] and out_idx int64 [b, k] hold each query's k best rows by fp32 dot product, score descending,
 * the lower row first on equal scores. Two launches: per-CTA candidate lists into the workspace (ws_score fp32 and
 * ws_idx int32, ws_entries >= sdb_knn_workspace(n, b, k) each), then their merge. Deterministic, no atomics. */
int64_t sdb_knn_workspace(int64_t n, int32_t b, int32_t k);
int sdb_knn_topk(const void* db, int64_t n, int32_t dim, const void* queries, int32_t b, int32_t k, float* ws_score,
                 int32_t* ws_idx, int64_t ws_entries, float* out_score, int64_t* out_idx, sdb_stream_t stream);
/* Row pooling of CLIP's text embedding (FrozenCLIPTextEmbedder): out fp32 [b, dim] = x fp32 row
 * b * n_ctx + argmax(ids[b, :n_ctx]) (the EOT token; the first maximum) when ids (int64 [b, n_ctx]) is given, else
 * row b; normalize != 0 divides each row by its L2 norm in fp32. */
int sdb_rows_pool(const float* x, const int64_t* ids, int32_t b, int32_t n_ctx, int32_t dim, int32_t normalize,
                  float* out, sdb_stream_t stream);
/* ---- CLIP image embedding of retrieval databases (clip_image.cu; FrozenClipImageEmbedder, modules.py:197-229) ----
 * Preprocessing of a ragged batch straight into the patch-embedding GEMM's operand: each image is resized to
 * size x size as F.interpolate(mode='bicubic', align_corners=True) does on CUDA (kornia.geometry.resize with
 * antialias=False; A = -0.75, border taps clamped, a copy when both sides match), then (x + 1) / 2 and (x - m) / s per
 * channel, rounded to fp16 patch rows [nb * (size/patch)^2, kpad], k = (c * patch + py) * patch + px, zero-padded to
 * kpad (a multiple of 64). table int64 [nb, 3] (device) = (H, W, element offset in src) per image. src is fp32 NCHW
 * [3, H, W] per image in [-1, 1] (src_u8 0) or uint8 HWC [H, W, 3] (src_u8 1), read as x / 127.5 - 1.
 * resized (optional) fp32 [nb, 3, size, size] receives the interpolated values before (x + 1) / 2. */
int sdb_clip_resize_patches(const void* src, int32_t src_u8, const int64_t* table, int32_t nb, int32_t size,
                            int32_t patch, int32_t kpad, float m0, float m1, float m2, float s0, float s1, float s2,
                            void* patches_f16, float* resized, sdb_stream_t stream);
/* CLIPVisionEmbeddings after the patch GEMM: x fp32 [nb, np + 1, dim], row 0 = cls_pos [dim] (class embedding +
 * pos[0]), row 1 + p = pe[b * np + p] + pos_patches[p]; pe fp32 [nb * np, dim]. dim % 4 == 0, 16-byte aligned. */
int sdb_vit_embed(const float* pe, const float* cls_pos, const float* pos_patches, int32_t nb, int32_t np, int32_t dim,
                  float* x, sdb_stream_t stream);
/* out fp32 [rows, dim] = x row r * row_stride (the class token of each sequence before ln_post) */
int sdb_rows_gather(const float* x, int32_t rows, int64_t row_stride, int32_t dim, float* out, sdb_stream_t stream);
/* out = a*x + b (latent scaling z/0.18215, ddpm.py:713) */
int sdb_axpby(const float* x, float a, float b, int64_t n, float* out, sdb_stream_t stream);
/* out = a*x + b*y (DDIMSampler.stochastic_encode, ddim.py:206-220; q_sample, ddpm.py:274-277) */
int sdb_axpby2(const float* x, const float* y, float a, float b, int64_t n, float* out, sdb_stream_t stream);

/* 1x1 conv with <= 128 channels in and out, fp32 (post_quant_conv 4->4 with the 1/scale_factor folded in as alpha,
 * quant_conv 8->8, KL-f16's 32->32, KL-f32's 128->128 and 64->64; autoencoder.py:302-303,326,331):
 * out[p, j] = sum_c (alpha x[p, c]) w[j, c] + b[j] */
int sdb_pointwise_small(const float* x, int64_t npix, int32_t cin, int32_t cout, const float* w, const float* b,
                        float alpha, float* out, sdb_stream_t stream);
/* CLIP token + position embedding gather (transformers CLIPTextEmbeddings): ids int64 [rows] -> fp32 [rows, dim] */
int sdb_embed_tokens(const int64_t* ids, int32_t rows, int32_t n_ctx, int32_t dim, int32_t vocab, const float* tok,
                     const float* pos, float* out, sdb_stream_t stream);

/* ---- post-processing of the decoded image: safety checker (scripts/txt2img.py:26-29, 88-95, 319) ----
 * The reference delegates to third-party code: transformers' CLIPFeatureExtractor (PIL bicubic resize of the shorter
 * side to 224, centre crop, 1/255, mean/std) and diffusers' StableDiffusionSafetyChecker (CLIP ViT-L/14 vision tower +
 * projection, cosine distance to 17 concept and 3 special-care embeddings). The vision tower runs on sdb_gemm /
 * sdb_attention / sdb_layernorm; these are the pieces around it. */
/* One pass of PIL's 8-bit ImagingResample over interleaved [n_img, H, W, 3] images: horizontal (vertical = 0: lines =
 * rows, in_size / out_size = widths) or vertical (vertical = 1: lines = columns, other_size_in = the row length W).
 * bounds int32 [out_size, 2] = {first source index, tap count}, coefs int32 [out_size, ksize] = 22-bit fixed-point
 * weights, both computed by the host exactly as PIL's precompute_coeffs / normalize_coeffs_8bpc. The source is uint8,
 * or fp32 in [0, 1] converted as numpy_to_pil does ((x * 255).round()). */
int sdb_resample_u8(const void* src_u8, const float* src_f32, int32_t n_img, int32_t lines, int32_t in_size,
                    int32_t out_size, int32_t ksize, const int32_t* bounds, const int32_t* coefs, int32_t vertical,
                    int32_t other_size_in, void* out_u8, sdb_stream_t stream);
/* centre crop to size x size, x / 255, (x - mean) / std: uint8 [nb, h, w, 3] -> fp32 NCHW [nb, 3, size, size] */
int sdb_clip_normalize(const void* img_u8, int32_t nb, int32_t h, int32_t w, int32_t size, float m0, float m1, float m2,
                       float s0, float s1, float s2, float* out_nchw, sdb_stream_t stream);
/* ViT patch extraction: NCHW fp32 [nb, 3, size, size] -> fp16 [nb * (size/patch)^2, kpad], k = (c * patch + py) * patch + px
 * (the flattening of CLIPVisionEmbeddings.patch_embedding.weight), zero-padded to kpad (multiple of 64) */
int sdb_patchify(const float* x_nchw, int32_t nb, int32_t size, int32_t patch, int32_t kpad, void* out_f16,
                 sdb_stream_t stream);
/* StableDiffusionSafetyChecker decision: scores fp32 [nb, n_special + n_concept] (rounded to 3 decimals as the
 * library does), flagged int32 [nb] */
int sdb_safety_scores(const float* image_embeds, int32_t nb, int32_t dim, const float* special_embeds,
                      const float* special_weights, int32_t n_special, const float* concept_embeds,
                      const float* concept_weights, int32_t n_concept, float* scores, int32_t* flagged,
                      sdb_stream_t stream);
/* images[i] = 0 for flagged images (fp32, per_image elements each) */
int sdb_blank_flagged(float* images, int64_t per_image, int32_t nb, const int32_t* flagged, sdb_stream_t stream);

/* Invisible watermark of scripts/txt2img.py:69-74, 261-264, 324 (third-party `invisible-watermark`: WatermarkEncoder
 * .encode(bgr, 'dwtDct') = EmbedMaxDct, scales [0, 36, 36], block 4) on uint8 RGB images [nb, h, w, 3]: cv2's 8-bit
 * RGB -> YUV, one watermark bit per 4x4 block of the Haar approximation band of U, YUV -> RGB. bits: uint8 [n_bits]
 * (0 / 1; "StableDiffusionV1" MSB first = 136 bits); yuv_scratch: nb*h*w*3 bytes. */
int sdb_watermark_dwtdct(const void* rgb_u8, int32_t nb, int32_t h, int32_t w, const void* bits_u8, int32_t n_bits,
                         float scale, void* yuv_scratch_u8, void* out_rgb_u8, sdb_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Handle-level entry points: the engine, not just its kernels.
 *
 * A plan is the ordered list of sdb_* launches of one pass over the model, recorded (arguments copied by value) while
 * the host side walks the model once between sdb_plan_begin and sdb_plan_end - the calls still execute, so the
 * recording pass doubles as the warm-up. sdb_plan_launch replays it as ONE CUDA graph (captured on first use on a
 * private stream). Every pointer inside is a caller-owned static buffer (weights, workspaces, I/O) that must outlive
 * the plan. Recording is per host thread.
 */
typedef struct sdb_plan sdb_plan;
int sdb_plan_begin(sdb_plan** out);
int sdb_plan_end(sdb_plan* plan);
int sdb_plan_size(const sdb_plan* plan);                 /* recorded launches (-1: NULL) */
int sdb_plan_run(sdb_plan* plan, sdb_stream_t stream);    /* eager replay, call by call */
int sdb_plan_launch(sdb_plan* plan, sdb_stream_t stream); /* graph replay */
int sdb_plan_destroy(sdb_plan* plan);
int sdb_fill_f32(float* x, int64_t n, float value, sdb_stream_t stream);

/*
 * One guided UNet evaluation as a handle: replaces sampler -> LatentDiffusion.apply_model -> DiffusionWrapper.forward
 * -> UNetModel.forward (ldm/models/diffusion/ddpm.py:891-992,1393-1421; ldm/modules/diffusionmodules/openaimodel.py:
 * 710-742). `plan` was recorded over one evaluation whose first kernel reads x_static [n, c_in, h, w] (NCHW fp32) and
 * t_static [n] and whose last kernel writes eps_static [n, c_out, h, w]; the cross-attention context is baked into the
 * plan (its K / V buffers are static: re-fill them to change the prompt). sdb_unet_forward copies x / t in when they
 * are not the static buffers themselves (NULL = already in place), launches the graph and copies eps out (NULL = leave
 * it in eps_static).
 */
typedef struct sdb_unet sdb_unet;
int sdb_unet_create(sdb_plan* plan, float* x_static, float* t_static, float* eps_static, int32_t n, int32_t c_in,
                    int32_t c_out, int32_t h, int32_t w, sdb_unet** out);
int sdb_unet_forward(sdb_unet* unet, const float* x, const float* t, float* eps, sdb_stream_t stream);
int sdb_unet_destroy(sdb_unet* unet);

/*
 * A whole PLMS trajectory (ldm/models/diffusion/plms.py:98-236, eta = 0) on the device: per step one sdb_unet_forward
 * (two on the first step: pseudo improved Euler) and one fused sdb_sampler_step. The schedule is passed as host arrays
 * indexed like the reference's ddim_* arrays (index 0 = the LAST step taken); timesteps are the ddim_timesteps as
 * floats. `unet` evaluates 2 * batch samples when guided ([uncond; cond] halves of the latent), else batch.
 */
typedef struct sdb_plms_desc {
  sdb_unet* unet;
  const float* x;          /* x_T, fp32 [batch, c, h, w] (device) */
  float* x_out;            /* final latent [batch, c, h, w] (device; may alias x) */
  float* pred_x0_out;      /* optional: last predicted x0 */
  float* work;             /* device scratch: (5 + 2 * rep) * batch*c*h*w floats, rep = guided ? 2 : 1 */
  int32_t batch, n_steps, guided;
  float scale;             /* unconditional_guidance_scale */
  const float* timesteps;  /* host [n_steps] */
  const float* alphas;     /* host [n_steps] ddim_alphas */
  const float* alphas_prev;
  const float* sqrt_one_minus_alphas;
  const float* sigmas;     /* host [n_steps] or NULL (eta = 0) */
} sdb_plms_desc;
int sdb_sample_plms(const sdb_plms_desc* d, sdb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* SDB200_H */
