/*
 * sdb200 evaluation ABI: the forward half of the LDM training objective (ldm/models/diffusion/ddpm.py), for computing
 * the denoising loss a trained model reaches (val/loss_simple, val/loss_vlb, val/loss). Nothing here is on the
 * sampling path, so these entry points live apart from include/sdb200.h and its entry-point table; they use its stream
 * type and follow its conventions: device pointers, 0 on success, sdb_last_error() for the message, and every call is
 * recorded into an open plan (sdb_plan_begin) like the entry points of sdb200.h.
 */
#ifndef SDB200_EVAL_H
#define SDB200_EVAL_H

#include "sdb200.h"

#ifdef __cplusplus
extern "C" {
#endif

/*
 * q(x_t | x_0) with one timestep per sample (DDPM.q_sample, ddpm.py:274-277):
 *   out[b, i] = sqrt_ac[t[b]] * x0[b, i] + sqrt_1m_ac[t[b]] * noise[b, i]
 * as __fadd_rn(__fmul_rn(a, x), __fmul_rn(s, n)) (extract_into_tensor(a, t, .) * x_start + extract_into_tensor(s, t,
 * .) * noise), so at a uniform t the result equals sdb_axpby2's bit for bit. x0 / noise / out: fp32 [nb, n] (NCHW
 * samples of n = c*h*w elements); t: int64 [nb] on the device, each in [0, T) (not checked here: the caller validates);
 * sqrt_ac / sqrt_1m_ac: fp32 [T] device tables (sqrt_alphas_cumprod, sqrt_one_minus_alphas_cumprod).
 */
int sdb_q_sample_t(const float* x0, const float* noise, const int64_t* t, const float* sqrt_ac, const float* sqrt_1m_ac,
                   int32_t nb, int64_t n, float* out, sdb_stream_t stream);

/*
 * Per-sample denoising loss of LatentDiffusion.p_losses (ddpm.py:1012-1045) for pred, target fp32 [nb, n]:
 *   out[0*nb + b] = loss_simple_b = mean_i |target - pred| (kind 1, l1) or mean_i (target - pred)^2 (kind 2, l2)
 *                   (get_loss(mean=False).mean([1, 2, 3]), ddpm.py:1016-1030)
 *   out[1*nb + b] = loss_simple_b / exp(logvar[t_b]) + logvar[t_b]                       (:1032-1033)
 *   out[2*nb + b] = lvlb_weights[t_b] * loss_simple_b                                    (:1040-1041)
 * Each difference and square is one fp32 rounding, as in the reference; the sum over a sample is in fp64 in an order
 * fixed by n alone (one CTA per sample, fixed thread strides, fixed fold tree), so a sample's three values do not depend
 * on nb, on the other samples of the batch or on the run. The batch means and the l_simple_weight /
 * original_elbo_weight combination are left to the host (ddpm.py:1031, 1036-1043). t: int64 [nb] in [0, T) (the
 * caller validates); logvar / lvlb_weights: fp32 [T] device tables. out: fp32 [3, nb].
 */
int sdb_diffusion_loss(const float* pred, const float* target, int32_t kind, const int64_t* t, const float* logvar,
                       const float* lvlb_weights, int32_t nb, int64_t n, float* out, sdb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* SDB200_EVAL_H */
