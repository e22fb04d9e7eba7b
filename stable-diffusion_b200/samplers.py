"""PLMS, DDIM and DPM-Solver++ samplers with the reference's API surface (ldm/models/diffusion/plms.py:10-236,
ldm/models/diffusion/ddim.py:12-241, ldm/models/diffusion/dpm_solver/sampler.py:8-82): `Sampler(model,
schedule="linear")`, `.make_schedule`, `.sample(...) -> (samples, intermediates)`, DDIM's `.stochastic_encode` /
`.decode`, and the `mask` / `x0` inpainting branch of the PLMS / DDIM loops (plms.py:147-150, ddim.py:144-147).

The per-step update (classifier-free guidance + Adams-Bashforth / DDIM step, ~25 elementwise launches and four
host->device scalar fills per step in the reference, plms.py:182-236) is ONE fused kernel (sdb_sampler_step) taking
the schedule scalars as kernel arguments: no device-side torch.full, no host sync. The [uncond; cond] batch is
kept in a persistent doubled latent buffer that the step kernel writes directly (no torch.cat per step).

`model` is the facade the reference samplers read (plms.py:15,29-35,121,180-190): num_timesteps, betas,
alphas_cumprod, alphas_cumprod_prev, device, apply_model(x, t, c).
"""
from __future__ import annotations

import numpy as np
import torch

from . import ops


def make_ddim_timesteps(ddim_discr_method, num_ddim_timesteps, num_ddpm_timesteps, verbose=True):
    """util.py:46-60."""
    if ddim_discr_method == "uniform":
        c = num_ddpm_timesteps // num_ddim_timesteps
        ddim_timesteps = np.asarray(list(range(0, num_ddpm_timesteps, c)))
    elif ddim_discr_method == "quad":
        ddim_timesteps = ((np.linspace(0, np.sqrt(num_ddpm_timesteps * .8), num_ddim_timesteps)) ** 2).astype(int)
    else:
        raise NotImplementedError(f'There is no ddim discretization method called "{ddim_discr_method}"')
    steps_out = ddim_timesteps + 1
    if verbose:
        print(f"Selected timesteps for ddim sampler: {steps_out}")
    return steps_out


def make_ddim_sampling_parameters(alphacums, ddim_timesteps, eta, verbose=True):
    """util.py:63-74; alphacums is the fp32 cumulative-alpha table (host numpy)."""
    if int(ddim_timesteps.max()) >= len(alphacums):
        raise IndexError(f"timestep {int(ddim_timesteps.max())} out of range for {len(alphacums)} training steps")
    alphas = alphacums[ddim_timesteps]
    alphas_prev = np.asarray([alphacums[0]] + alphacums[ddim_timesteps[:-1]].tolist())
    sigmas = eta * np.sqrt((1 - alphas_prev) / (1 - alphas) * (1 - alphas / alphas_prev))
    if verbose:
        print(f"Selected alphas for ddim sampler: a_t: {alphas}; a_(t-1): {alphas_prev}")
        print(f"For the chosen value of eta, which is {eta}, this results in the following sigma_t schedule "
              f"for ddim sampler {sigmas}")
    return sigmas, alphas, alphas_prev


class _SamplerBase:
    name = "sampler"

    def __init__(self, model, schedule="linear", cfg_parallel=None, **kwargs):
        self.model = model
        self.ddpm_num_timesteps = model.num_timesteps
        self.schedule = schedule
        self.cfg_parallel = cfg_parallel   # dist.CFGParallel: guidance halves on two GPUs (latency mode)

    # -- schedule (host side; fp32 values exactly as the reference's device tensors hold them)
    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0., verbose=True):
        self.ddim_timesteps = make_ddim_timesteps(ddim_discretize, ddim_num_steps, self.ddpm_num_timesteps, verbose)
        ac = self.model.alphas_cumprod.detach().to("cpu", torch.float32).numpy()
        assert ac.shape[0] == self.ddpm_num_timesteps, "alphas have to be defined for each timestep"
        self.alphas_cumprod = ac
        sigmas, alphas, alphas_prev = make_ddim_sampling_parameters(ac, self.ddim_timesteps, ddim_eta, verbose)
        f32 = lambda a: np.asarray(a, dtype=np.float64).astype(np.float32)
        self.ddim_sigmas = f32(sigmas)
        self.ddim_alphas = f32(alphas)
        self.ddim_alphas_prev = f32(alphas_prev)
        self.ddim_sqrt_one_minus_alphas = np.sqrt(np.float32(1.0) - self.ddim_alphas).astype(np.float32)
        self.ddim_eta = ddim_eta

    # -- model evaluation on the (optionally) guidance-doubled batch
    def _setup_guidance(self, cond, uc, scale, b):
        self._guided = not (uc is None or scale == 1.)
        if cond is None and self._guided:
            raise ValueError("classifier-free guidance needs a conditioning")
        self._scale = float(scale)
        if isinstance(cond, dict):
            raise NotImplementedError("dict conditioning (hybrid/concat) is outside the SD-v1 crossattn path")
        self._split = self._guided and self.cfg_parallel is not None
        if self._split:
            self._c_in = self.cfg_parallel.select(uc, cond).contiguous()   # this GPU evaluates one half only
        else:
            # unconditional models (cond None, sample_diffusion.py): no context, no doubled batch
            self._c_in = torch.cat([uc, cond]).contiguous() if self._guided else \
                (cond.contiguous() if cond is not None else None)
        self._rep = 2 if (self._guided and not self._split) else 1
        setter = getattr(self.model, "set_context", None)
        if setter is not None:
            setter(self._c_in)   # cross-attention K/V once per prompt batch instead of once per step

    def _eval(self, x2, step, b):
        """x2: persistent [2b or b, C, H, W] latent buffer; returns eps for the whole (doubled) batch."""
        nb = x2.shape[0]
        ts = self._ts_cache.get((int(step), nb))
        if ts is None:
            ts = torch.full((nb,), int(step), device=x2.device, dtype=torch.long)
            self._ts_cache[(int(step), nb)] = ts
        return self._exchange(self.model.apply_model(x2, ts, self._c_in))

    def _exchange(self, eps):
        """-> (eps2, eps_cond): the [uncond; cond] pair, or two pointers when the halves live on two GPUs."""
        return self.cfg_parallel.exchange(eps) if self._split else (eps, None)

    def _step(self, x2, eps2, index, order, hist, b, noise=None, e_out=None, write_x=True):
        eps2, eps_cond = eps2
        x = x2[:b]
        pred_x0 = torch.empty_like(x)
        x_prev = torch.empty_like(x2) if write_x else None
        xp, p0, e = ops.sampler_step(
            x, eps2, eps_cond=eps_cond, guided=self._guided, scale=self._scale, order=order, hist=hist, noise=noise,
            a_t=float(self.ddim_alphas[index]), a_prev=float(self.ddim_alphas_prev[index]),
            sigma_t=float(self.ddim_sigmas[index]),
            sqrt_one_minus_a_t=float(self.ddim_sqrt_one_minus_alphas[index]),
            x_prev=x_prev, pred_x0=pred_x0, e_out=e_out, dup=self._rep == 2)
        return xp, p0, e

    def _blend_mask(self, x2, mask, x0, step, b):
        """img = q_sample(x0, ts) * mask + (1 - mask) * img on the persistent (doubled) latent buffer, in place."""
        ts = self._ts_cache.get((int(step), b))
        if ts is None:
            ts = self._ts_cache[(int(step), b)] = torch.full((b,), int(step), device=x2.device, dtype=torch.long)
        img_orig = self.model.q_sample(x0, ts)
        ops.mask_blend(img_orig.contiguous().float(), mask, x2, b, dup=self._rep == 2)

    @staticmethod
    def _prep_mask(mask, x0, device):
        if mask is None:
            return None, None
        return (mask.to(device=device, dtype=torch.float32).contiguous(),
                x0.to(device=device, dtype=torch.float32).contiguous())

    def _check_args(self, **kw):
        for k in ("score_corrector", "corrector_kwargs", "normals_sequence"):
            if kw.get(k) is not None:
                raise NotImplementedError(f"{k} is outside the txt2img/img2img hot path of this engine")
        if kw.get("mask") is not None:
            assert kw.get("x0") is not None   # plms.py:148 / ddim.py:145
        if kw.get("quantize_x0"):
            raise NotImplementedError("quantize_x0 is not implemented (it would split the fused sampler update)")
        if kw.get("noise_dropout", 0.) != 0.:
            raise NotImplementedError("noise_dropout")


class PLMSSampler(_SamplerBase):
    name = "plms"

    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0., verbose=True):
        if ddim_eta != 0:
            raise ValueError("ddim_eta must be 0 for PLMS")
        super().make_schedule(ddim_num_steps, ddim_discretize, ddim_eta, verbose)

    @torch.no_grad()
    def sample(self, S, batch_size, shape, conditioning=None, callback=None, normals_sequence=None,
               img_callback=None, quantize_x0=False, eta=0., mask=None, x0=None, temperature=1., noise_dropout=0.,
               score_corrector=None, corrector_kwargs=None, verbose=True, x_T=None, log_every_t=100,
               unconditional_guidance_scale=1., unconditional_conditioning=None, **kwargs):
        self._check_args(mask=mask, x0=x0, score_corrector=score_corrector, corrector_kwargs=corrector_kwargs,
                         normals_sequence=normals_sequence, quantize_x0=quantize_x0, noise_dropout=noise_dropout)
        if conditioning is not None and conditioning.shape[0] != batch_size:
            print(f"Warning: Got {conditioning.shape[0]} conditionings but batch-size is {batch_size}")
        self.make_schedule(ddim_num_steps=S, ddim_eta=eta, verbose=verbose)
        C, H, W = shape
        size = (batch_size, C, H, W)
        if verbose:
            print(f"Data shape for PLMS sampling is {size}")
        return self.plms_sampling(conditioning, size, callback=callback, img_callback=img_callback, x_T=x_T,
                                  log_every_t=log_every_t, temperature=temperature, mask=mask, x0=x0,
                                  unconditional_guidance_scale=unconditional_guidance_scale,
                                  unconditional_conditioning=unconditional_conditioning)

    @torch.no_grad()
    def plms_sampling(self, cond, shape, x_T=None, callback=None, img_callback=None, log_every_t=100,
                      temperature=1., unconditional_guidance_scale=1., unconditional_conditioning=None, mask=None,
                      x0=None, **kw):
        device = self.model.device
        b = shape[0]
        mask, x0 = self._prep_mask(mask, x0, device)
        img = torch.randn(shape, device=device) if x_T is None else x_T.to(device=device, dtype=torch.float32)
        self._setup_guidance(cond, unconditional_conditioning, unconditional_guidance_scale, b)
        self._ts_cache = {}
        rep = self._rep
        x2 = img.repeat(rep, 1, 1, 1).contiguous() if rep == 2 else img.contiguous().clone()
        time_range = np.flip(self.ddim_timesteps)
        total_steps = time_range.shape[0]
        intermediates = {"x_inter": [img], "pred_x0": [img]}
        old_eps = []
        for i, step in enumerate(time_range):
            index = total_steps - i - 1
            step_next = time_range[min(i + 1, total_steps - 1)]
            if mask is not None:
                self._blend_mask(x2, mask, x0, step, b)
            eps2 = self._eval(x2, step, b)
            if len(old_eps) == 0:
                # pseudo improved Euler: x_prev from e_t, second evaluation at t_next, e' = (e_t + e_t_next)/2
                e_t = torch.empty_like(x2[:b])
                xp, _, _ = self._step(x2, eps2, index, 0, [], b, e_out=e_t)
                eps2n = self._eval(xp, step_next, b)
                x2, pred_x0, _ = self._step(x2, eps2n, index, 4, [e_t], b)
            else:
                order = min(len(old_eps), 3)
                e_t = torch.empty_like(x2[:b])
                hist = [old_eps[-1 - j] for j in range(order)]
                x2, pred_x0, _ = self._step(x2, eps2, index, order, hist, b, e_out=e_t)
            old_eps.append(e_t)
            if len(old_eps) >= 4:
                old_eps.pop(0)
            if callback:
                callback(i)
            if img_callback:
                img_callback(pred_x0, i)
            if index % log_every_t == 0 or index == total_steps - 1:
                intermediates["x_inter"].append(x2[:b].clone() if mask is not None else x2[:b])
                intermediates["pred_x0"].append(pred_x0)
        return x2[:b].clone(), intermediates


class DDIMSampler(_SamplerBase):
    name = "ddim"

    @torch.no_grad()
    def sample(self, S, batch_size, shape, conditioning=None, callback=None, normals_sequence=None,
               img_callback=None, quantize_x0=False, eta=0., mask=None, x0=None, temperature=1., noise_dropout=0.,
               score_corrector=None, corrector_kwargs=None, verbose=True, x_T=None, log_every_t=100,
               unconditional_guidance_scale=1., unconditional_conditioning=None, **kwargs):
        self._check_args(mask=mask, x0=x0, score_corrector=score_corrector, corrector_kwargs=corrector_kwargs,
                         normals_sequence=normals_sequence, quantize_x0=quantize_x0, noise_dropout=noise_dropout)
        if conditioning is not None and conditioning.shape[0] != batch_size:
            print(f"Warning: Got {conditioning.shape[0]} conditionings but batch-size is {batch_size}")
        self.make_schedule(ddim_num_steps=S, ddim_eta=eta, verbose=verbose)
        C, H, W = shape
        size = (batch_size, C, H, W)
        if verbose:
            print(f"Data shape for DDIM sampling is {size}, eta {eta}")
        return self.ddim_sampling(conditioning, size, callback=callback, img_callback=img_callback, x_T=x_T,
                                  log_every_t=log_every_t, temperature=temperature, mask=mask, x0=x0,
                                  unconditional_guidance_scale=unconditional_guidance_scale,
                                  unconditional_conditioning=unconditional_conditioning)

    def _run(self, img, cond, timesteps, scale, uc, temperature=1., callback=None, img_callback=None,
             log_every_t=100, intermediates=None, mask=None, x0=None):
        b = img.shape[0]
        mask, x0 = self._prep_mask(mask, x0, img.device)
        self._setup_guidance(cond, uc, scale, b)
        self._ts_cache = {}
        rep = self._rep
        x2 = img.repeat(rep, 1, 1, 1).contiguous() if rep == 2 else img.contiguous().clone()
        time_range = np.flip(timesteps)
        total_steps = time_range.shape[0]
        for i, step in enumerate(time_range):
            index = total_steps - i - 1
            if mask is not None:
                self._blend_mask(x2, mask, x0, step, b)
            eps2 = self._eval(x2, step, b)
            noise = None
            if self.ddim_sigmas[index] != 0:
                noise = torch.randn_like(x2[:b]) * temperature   # noise_like, util.py:264-267
            x2, pred_x0, _ = self._step(x2, eps2, index, 0, [], b, noise=noise)
            if callback:
                callback(i)
            if img_callback:
                img_callback(pred_x0, i)
            if intermediates is not None and (index % log_every_t == 0 or index == total_steps - 1):
                intermediates["x_inter"].append(x2[:b].clone() if mask is not None else x2[:b])
                intermediates["pred_x0"].append(pred_x0)
        return x2[:b].clone()

    @torch.no_grad()
    def ddim_sampling(self, cond, shape, x_T=None, callback=None, img_callback=None, log_every_t=100,
                      temperature=1., unconditional_guidance_scale=1., unconditional_conditioning=None, mask=None,
                      x0=None, **kw):
        device = self.model.device
        img = torch.randn(shape, device=device) if x_T is None else x_T.to(device=device, dtype=torch.float32)
        intermediates = {"x_inter": [img], "pred_x0": [img]}
        out = self._run(img, cond, self.ddim_timesteps, unconditional_guidance_scale, unconditional_conditioning,
                        temperature, callback, img_callback, log_every_t, intermediates, mask=mask, x0=x0)
        return out, intermediates

    @torch.no_grad()
    def stochastic_encode(self, x0, t, use_original_steps=False, noise=None):
        """ddim.py:206-220: z_t = sqrt(a[t]) x0 + sqrt(1 - a[t]) eps, indexing the DDIM arrays (per-sample t)."""
        assert not use_original_steps
        if noise is None:
            noise = torch.randn_like(x0)
        t_host = t.detach().to("cpu").long().numpy() if torch.is_tensor(t) else np.asarray(t)
        assert (t_host == t_host[0]).all(), "per-sample t_enc differing within a batch is not used by img2img.py"
        idx = int(t_host[0])
        a = float(np.sqrt(self.ddim_alphas[idx]))
        s = float(self.ddim_sqrt_one_minus_alphas[idx])
        return ops.axpby2(x0.contiguous().float(), noise.contiguous().float(), a, s)

    @torch.no_grad()
    def decode(self, x_latent, cond, t_start, unconditional_guidance_scale=1.0, unconditional_conditioning=None,
               use_original_steps=False):
        """ddim.py:222-241."""
        assert not use_original_steps
        timesteps = self.ddim_timesteps[:t_start]
        return self._run(x_latent.float(), cond, timesteps, unconditional_guidance_scale, unconditional_conditioning)


class DiscreteVPSchedule:
    """NoiseScheduleVP('discrete', alphas_cumprod=...) of the reference (dpm_solver.py:99-108, 125-156) on the host:
    log alpha_t is the piecewise-linear interpolant (interpolate_fn, dpm_solver.py:1132-1171) of
    0.5 log(alphas_cumprod) over t_n = n/N; everything in fp32 torch ops in the reference's order."""

    def __init__(self, alphas_cumprod):
        ac = torch.as_tensor(alphas_cumprod).detach().to("cpu", torch.float32)
        self.log_alpha = 0.5 * torch.log(ac)
        self.total_N = int(ac.numel())
        self.T = 1.
        self.t_array = torch.linspace(0., 1., self.total_N + 1)[1:]

    def marginal_log_mean_coeff(self, t):
        xp, yp, K = self.t_array, self.log_alpha, self.total_N
        idx = torch.searchsorted(xp, t.contiguous(), right=False)       # keypoints strictly below t
        lo = torch.where(idx == 0, torch.zeros_like(idx), torch.where(idx == K, torch.full_like(idx, K - 2), idx - 1))
        return yp[lo] + (t - xp[lo]) * (yp[lo + 1] - yp[lo]) / (xp[lo + 1] - xp[lo])

    def marginal_alpha(self, t):
        return torch.exp(self.marginal_log_mean_coeff(t))

    def marginal_std(self, t):
        return torch.sqrt(1. - torch.exp(2. * self.marginal_log_mean_coeff(t)))

    def marginal_lambda(self, t):
        lm = self.marginal_log_mean_coeff(t)
        return lm - 0.5 * torch.log(1. - torch.exp(2. * lm))


def dpm_solver_plan(alphas_cumprod, steps, order=2, lower_order_final=True):
    """Per-evaluation scalars of DPM_Solver.sample(steps, skip_type='time_uniform', method='multistep', order=2,
    lower_order_final=True) in data-prediction mode (dpm_solver.py:965-1108, 504-533, 755-789): evaluation i happens at
    continuous time t_i (model input (t_i - 1/N) * 1000, dpm_solver.py:278-287) and is followed by the update to t_{i+1}.
    Returns a list of dicts {t_input, sigma_s, alpha_s, order, c_x, c_m, inv_r0}, python floats holding fp32 values."""
    assert order == 2 and steps >= order
    ns = DiscreteVPSchedule(alphas_cumprod)
    ts = torch.linspace(ns.T, 1. / ns.total_N, steps + 1)
    lam, la, sig = ns.marginal_lambda(ts), ns.marginal_log_mean_coeff(ts), ns.marginal_std(ts)
    alpha = torch.exp(la)
    t_in = (ts - 1. / ns.total_N) * 1000.
    plan = []
    for i in range(steps):                      # update from t_i to t_{i+1}; "step" of the reference loop = i + 1
        step = i + 1
        o = 1 if i == 0 else (min(order, steps + 1 - step) if (lower_order_final and steps < 15) else order)
        h = lam[i + 1] - lam[i]
        e = dict(t_input=float(t_in[i]), sigma_s=float(sig[i]), alpha_s=float(alpha[i]), order=o,
                 c_x=float(sig[i + 1] / sig[i]), inv_r0=0.0)
        if o == 1:
            e["c_m"] = float(alpha[i + 1] * torch.expm1(-h))
        else:
            r0 = (lam[i] - lam[i - 1]) / h
            e["c_m"] = float(alpha[i + 1] * (torch.exp(-h) - 1.))
            e["inv_r0"] = float(1. / r0)
        plan.append(e)
    return plan


class DPMSolverSampler(_SamplerBase):
    """dpm_solver/sampler.py:8-82: DPM-Solver++ multistep order 2 on the model's discrete schedule with classifier-free
    guidance. Each step is one UNet evaluation (float timestep) + ONE fused kernel (guidance, eps -> x0, update)."""
    name = "dpm_solver"

    def __init__(self, model, **kwargs):
        super().__init__(model, **kwargs)
        self.alphas_cumprod = model.alphas_cumprod.detach().to("cpu", torch.float32)

    @torch.no_grad()
    def sample(self, S, batch_size, shape, conditioning=None, callback=None, normals_sequence=None,
               img_callback=None, quantize_x0=False, eta=0., mask=None, x0=None, temperature=1., noise_dropout=0.,
               score_corrector=None, corrector_kwargs=None, verbose=True, x_T=None, log_every_t=100,
               unconditional_guidance_scale=1., unconditional_conditioning=None, **kwargs):
        if conditioning is not None and conditioning.shape[0] != batch_size:
            print(f"Warning: Got {conditioning.shape[0]} conditionings but batch-size is {batch_size}")
        C, H, W = shape
        device = self.model.betas.device
        img = torch.randn((batch_size, C, H, W), device=device) if x_T is None else x_T.to(device=device, dtype=torch.float32)
        b = batch_size
        self._setup_guidance(conditioning, unconditional_conditioning, unconditional_guidance_scale, b)
        plan = dpm_solver_plan(self.alphas_cumprod, S)
        rep = self._rep
        x2 = img.repeat(rep, 1, 1, 1).contiguous() if rep == 2 else img.contiguous().clone()
        m_prev = None
        for i, p in enumerate(plan):
            ts = torch.full((x2.shape[0],), p["t_input"], device=device, dtype=torch.float32)
            eps2, eps_cond = self._exchange(self.model.apply_model(x2, ts, self._c_in))
            x2, m_prev = ops.dpm_solver_step(
                x2[:b], eps2, eps_cond=eps_cond, guided=self._guided, scale=self._scale, sigma_s=p["sigma_s"], alpha_s=p["alpha_s"],
                order=p["order"], m_prev=m_prev, c_x=p["c_x"], c_m=p["c_m"], inv_r0=p["inv_r0"],
                x_out=torch.empty_like(x2), dup=rep == 2)
            if callback:
                callback(i)
            if img_callback:
                img_callback(m_prev, i)
        return x2[:b].clone(), None
