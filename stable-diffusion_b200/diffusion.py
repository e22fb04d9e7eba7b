"""LatentDiffusion facade: the inference surface of `ldm.models.diffusion.ddpm.LatentDiffusion` that the scripts and
samplers use (ddpm.py): register_schedule (:117-169), apply_model (:891-992 plain path) through a DiffusionWrapper
(:1393-1421 crossattn branch), get_learned_conditioning (:551-562), encode_first_stage (:825-863),
get_first_stage_encoding (:542-549), decode_first_stage (:705-763, KL and VQ first stages), q_sample (:274-277), ema_scope (:171-184).
Sub-modules keep the reference attribute names so checkpoint prefixes resolve:
`model.diffusion_model.*`, `first_stage_model.*`, `cond_stage_model.transformer.*`, `model_ema.*`.
Unconditional models (cond_stage_config "__is_unconditional__", e.g. LSUN-Churches) sample through DDIM with no
conditioning, or through the ancestral sampler (p_sample_loop / progressive_denoising, ddpm.py:1047-1213) whose update
is one fused kernel per step (sdb_ddpm_step).
The denoising objective is evaluated forward-only: p_losses / get_loss (:1012-1045, :279-293), forward (:870-879),
get_input (:654-705), shared_step (:865-868) and validation_step (:358-364), with the noising at one timestep per sample
(sdb_q_sample_t) and the per-sample reduction (sdb_diffusion_loss) as kernels. Training itself (gradients, optimizers,
EMA updates, logging) is out of scope.
"""
from __future__ import annotations

from contextlib import contextmanager

import numpy as np
import torch
import torch.nn as nn

from . import ops
from .util import instantiate_from_config, remap_config
from .vq import VQModelInterface


# ------------------------------------------------------------------ patch tiling (split_input_params, ddpm.py:564-651)
# cond_stage_keys whose conditioning is an image at the latent size, tiled together with x (ddpm.py:916-927)
SPLIT_COND_KEYS = ("image", "LR_image", "segmentation", "bbox_img")
# Upper bounds on the device memory one tile needs, in bytes per pixel of the tile per channel of the widest full-resolution
# level: the UNet keeps its skips, fp16 hi / lo operands and fp32 outputs at that level alive together; the decoder holds
# a few fp32 / fp16 copies of its last level. Tiles are batched up to half the free memory.
_UNET_TILE_BYTES, _DECODER_TILE_BYTES = 256, 48


def border_distance(h, w):
    """delta_border (ddpm.py:571-582): each pixel's normalized distance to the nearest tile border, fp32 [h, w], 0 at
    the border and 0.5 at the centre. The same fp32 operations as the reference, so the tables match it bit for bit."""
    ay = (torch.arange(h, dtype=torch.float32) / float(h - 1)).view(h, 1)
    ax = (torch.arange(w, dtype=torch.float32) / float(w - 1)).view(1, w)
    return torch.minimum(torch.minimum(ay, ax), torch.minimum(1 - ay, 1 - ax))


def split_geometry(h, w, params, uf=1):
    """Tile geometry of the split path for a latent of h x w: (ks, stride, (ly, lx)). uf == 1 is apply_model's, uf > 1
    decode_first_stage's, which first shrinks ks and stride to the latent as the reference does. Raises ValueError where
    the reference has no finite result: a kernel larger than the latent (apply_model), tiles that leave rows or columns
    uncovered (the reference divides by a zero normalization there), a non-square kernel at uf > 1 (the reference's
    fold kernel is ks[0] on both sides), and tie_braker with a single row or column of tiles (delta_border of a 1-wide
    grid divides 0 by 0)."""
    ks, stride = tuple(int(v) for v in params["ks"]), tuple(int(v) for v in params["stride"])
    if uf > 1:
        ks = (min(ks[0], h), min(ks[1], w))
        if stride[0] > h or stride[1] > w:
            stride = (min(stride[0], h), min(stride[1], w))
        if ks[0] != ks[1]:
            raise ValueError(f"split decode: kernel {ks} is not square, and the reference folds {uf}x-upsampled tiles "
                             "with a square kernel of ks[0]")
    elif ks[0] > h or ks[1] > w:
        raise ValueError(f"split apply_model: kernel {ks} is larger than the {h}x{w} latent")
    if (h - ks[0]) % stride[0] or (w - ks[1]) % stride[1]:
        raise ValueError(f"split path: tiles of {ks} at stride {stride} do not cover the {h}x{w} latent "
                         "((side - ks) % stride must be 0)")
    grid = ((h - ks[0]) // stride[0] + 1, (w - ks[1]) // stride[1] + 1)
    if params.get("tie_braker") and min(grid) == 1:
        raise ValueError(f"split path: tie_braker needs at least two rows and columns of tiles, got {grid}")
    return ks, stride, grid


def split_tables(ks, stride, grid, params, uf=1):
    """get_weighting / fold(weighting) (ddpm.py:584-624) on the CPU in fp32: the per-tile weights [ly*lx, kh, kw] and
    the normalization [(ly - 1)*sy + kh, (lx - 1)*sx + kw], at tile size (kh, kw) = ks*uf and stride (sy, sx) =
    stride*uf."""
    kh, kw = ks[0] * uf, ks[1] * uf
    L = grid[0] * grid[1]
    wt = torch.clip(border_distance(kh, kw), params["clip_min_weight"], params["clip_max_weight"])
    weight = wt.view(1, kh * kw, 1).repeat(1, 1, L)
    if params.get("tie_braker"):
        lw = torch.clip(border_distance(*grid), params["clip_min_tie_weight"], params["clip_max_tie_weight"])
        weight = weight * lw.view(1, 1, L)
    sy, sx = stride[0] * uf, stride[1] * uf
    size = ((grid[0] - 1) * sy + kh, (grid[1] - 1) * sx + kw)
    norm = torch.nn.functional.fold(weight, size, kernel_size=(kh, kw), stride=(sy, sx)).view(*size)
    return weight[0].t().contiguous().view(L, kh, kw), norm


class DiffusionWrapper(nn.Module):
    def __init__(self, diff_model_config, conditioning_key):
        super().__init__()
        self.diffusion_model = instantiate_from_config(remap_config(diff_model_config))
        self.conditioning_key = conditioning_key
        assert self.conditioning_key in [None, "concat", "crossattn", "hybrid", "adm"]
        if self.conditioning_key in ("hybrid", "adm"):
            raise NotImplementedError(f"conditioning_key {self.conditioning_key!r}: supported are crossattn (SD v1), "
                                      "concat (inpainting) and None (unconditional)")

    def forward(self, x, t, c_concat=None, c_crossattn=None):
        if self.conditioning_key is None:
            return self.diffusion_model(x, t)
        if self.conditioning_key == "concat":
            # the UNet reads x and the conditioning as two sources (no cat([x] + c_concat) per step)
            c = c_concat[0] if len(c_concat) == 1 else torch.cat(c_concat, 1)
            return self.diffusion_model(x, t, concat=c)
        cc = c_crossattn[0] if len(c_crossattn) == 1 else torch.cat(c_crossattn, 1)
        return self.diffusion_model(x, t, context=cc)


class _EmaWeights(nn.Module):
    """Receives the `model_ema.*` tensors of a checkpoint (LitEma, ldm/modules/ema.py: buffer names are the
    DiffusionWrapper parameter names with the dots removed, plus `decay` and `num_updates`) and hands them to the UNet
    as its "ema" weight set. Holds no tensors of its own: the UNet packs the set it runs on."""

    def __init__(self, unet):
        super().__init__()
        self._unet = [unet]       # not a sub-module: its tensors belong to model.diffusion_model
        self.loaded = False

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                              error_msgs):
        unet = self._unet[0]
        names = {("diffusion_model." + k).replace(".", ""): k for k in unet.shapes}
        sub = {k[len(prefix):]: v for k, v in state_dict.items() if k.startswith(prefix)}
        unexpected_keys.extend(prefix + k for k in sub if k not in names and k not in ("decay", "num_updates"))
        if not any(k in sub for k in names):
            return        # a checkpoint without EMA copies: ema_scope() keeps the raw weights
        absent = [prefix + k for k in names if k not in sub]
        if absent:
            missing_keys.extend(absent)
            return
        unet.set_weight_set("ema", {names[k]: v for k, v in sub.items() if k in names})
        self.loaded = True


class LatentDiffusion(nn.Module):
    def __init__(self, first_stage_config, cond_stage_config, unet_config, timesteps=1000, beta_schedule="linear",
                 linear_start=1e-4, linear_end=2e-2, cosine_s=8e-3, num_timesteps_cond=None, cond_stage_key="image",
                 cond_stage_trainable=False, concat_mode=True, cond_stage_forward=None, conditioning_key=None,
                 scale_factor=1.0, scale_by_std=False, parameterization="eps", use_ema=True, image_size=256,
                 channels=3, first_stage_key="image", log_every_t=100, monitor=None, v_posterior=0.,
                 scheduler_config=None, loss_type="l2", l_simple_weight=1., original_elbo_weight=0.,
                 learn_logvar=False, logvar_init=0., **ignored):
        super().__init__()
        assert parameterization == "eps" and beta_schedule == "linear"
        if learn_logvar:
            raise NotImplementedError("learn_logvar: a learned per-timestep logvar is a training parameter; no "
                                      "published config sets it")
        if loss_type not in ops.LOSS_KINDS:
            raise NotImplementedError(f"unknown loss type '{loss_type}'")
        self.loss_type = loss_type
        self.l_simple_weight, self.original_elbo_weight = float(l_simple_weight), float(original_elbo_weight)
        self.learn_logvar, self.logvar_init = False, float(logvar_init)
        self.cond_stage_trainable = bool(cond_stage_trainable)
        if conditioning_key is None:
            conditioning_key = "concat" if concat_mode else "crossattn"
        if cond_stage_config == "__is_unconditional__":      # ddpm.py:447-448, 501-504
            conditioning_key = None
        self.parameterization = parameterization
        self.image_size, self.channels = image_size, channels
        self.scale_by_std = scale_by_std
        if scale_by_std:        # a buffer loaded from the checkpoint (ddpm.py:461-464)
            self.register_buffer("scale_factor", torch.tensor(scale_factor))
        else:
            self.scale_factor = float(scale_factor)
        self.use_ema = use_ema
        self.log_every_t = log_every_t
        self.clip_denoised = False
        self.cond_stage_key, self.first_stage_key = cond_stage_key, first_stage_key
        self.model = DiffusionWrapper(unet_config, conditioning_key)
        if use_ema:
            self.model_ema = _EmaWeights(self.model.diffusion_model)
        self.first_stage_model = instantiate_from_config(remap_config(first_stage_config))
        if cond_stage_config == "__is_first_stage__":      # ddpm.py:511-513: one module under both prefixes
            self.cond_stage_model = self.first_stage_model
        else:
            self.cond_stage_model = instantiate_from_config(remap_config(cond_stage_config))
        self.register_schedule(timesteps, linear_start, linear_end)

    # -- schedule: fp64 numpy -> fp32 buffers (ddpm.py:117-169, util.py:21-25)
    def register_schedule(self, timesteps=1000, linear_start=1e-4, linear_end=2e-2):
        betas = (torch.linspace(linear_start ** 0.5, linear_end ** 0.5, timesteps, dtype=torch.float64) ** 2).numpy()
        alphas = 1. - betas
        alphas_cumprod = np.cumprod(alphas, axis=0)
        alphas_cumprod_prev = np.append(1., alphas_cumprod[:-1])
        self.num_timesteps = int(timesteps)
        self.linear_start, self.linear_end = linear_start, linear_end
        to_torch = lambda a: torch.tensor(a, dtype=torch.float32)
        self.register_buffer("betas", to_torch(betas))
        self.register_buffer("alphas_cumprod", to_torch(alphas_cumprod))
        self.register_buffer("alphas_cumprod_prev", to_torch(alphas_cumprod_prev))
        self.register_buffer("sqrt_alphas_cumprod", to_torch(np.sqrt(alphas_cumprod)))
        self.register_buffer("sqrt_one_minus_alphas_cumprod", to_torch(np.sqrt(1. - alphas_cumprod)))
        # q(x_{t-1} | x_t, x_0) for the ancestral sampler (v_posterior 0); recomputed from the config, not loaded
        nonp = dict(persistent=False)
        self.register_buffer("sqrt_recip_alphas_cumprod", to_torch(np.sqrt(1. / alphas_cumprod)), **nonp)
        self.register_buffer("sqrt_recipm1_alphas_cumprod", to_torch(np.sqrt(1. / alphas_cumprod - 1)), **nonp)
        posterior_variance = betas * (1. - alphas_cumprod_prev) / (1. - alphas_cumprod)
        self.register_buffer("posterior_variance", to_torch(posterior_variance), **nonp)
        self.register_buffer("posterior_log_variance_clipped",
                             to_torch(np.log(np.maximum(posterior_variance, 1e-20))), **nonp)
        self.register_buffer("posterior_mean_coef1",
                             to_torch(betas * np.sqrt(alphas_cumprod_prev) / (1. - alphas_cumprod)), **nonp)
        self.register_buffer("posterior_mean_coef2",
                             to_torch((1. - alphas_cumprod_prev) * np.sqrt(alphas) / (1. - alphas_cumprod)), **nonp)
        # the loss weights of p_losses (ddpm.py:158-169, 87-89), formed in fp32 from the fp32 buffers as the reference
        # does; neither is in a checkpoint
        lvlb_weights = self.betas ** 2 / (2 * self.posterior_variance * to_torch(alphas) * (1 - self.alphas_cumprod))
        lvlb_weights[0] = lvlb_weights[1]
        self.register_buffer("lvlb_weights", lvlb_weights, **nonp)
        self.register_buffer("logvar", torch.full(fill_value=self.logvar_init, size=(self.num_timesteps,)),
                             **nonp)

    @property
    def device(self):
        return self.betas.device

    @contextmanager
    def ema_scope(self, context=None):
        """ddpm.py:171-184: inside the scope the UNet runs on the checkpoint's EMA weights (use_ema, e.g. the LSUN
        config's default); SD v1 has use_ema False and the scope is a no-op."""
        unet = self.model.diffusion_model
        swap = self.use_ema and unet.has_weight_set("ema")
        if swap:
            unet.use_weight_set("ema")
            if context is not None:
                print(f"{context}: Switched to EMA weights")
        try:
            yield None
        finally:
            if swap:
                unet.use_weight_set("raw")
                if context is not None:
                    print(f"{context}: Restored training weights")

    # -- denoiser
    def apply_model(self, x_noisy, t, cond, return_ids=False):
        if isinstance(cond, dict):
            pass
        else:
            if not isinstance(cond, list):
                cond = [cond]
            cond = {"c_concat" if self.model.conditioning_key == "concat" else "c_crossattn": cond}
        if getattr(self, "split_input_params", None) is not None:
            assert not return_ids
            return self._apply_split(x_noisy, t, cond)
        x_recon = self.model(x_noisy, t, **cond)
        if isinstance(x_recon, tuple) and not return_ids:
            return x_recon[0]
        return x_recon

    def _split_plan(self, shape, uf, device):
        """Geometry, weight / normalization tables (on the device) and tile-batch size of the split path for a latent of
        `shape`, computed once per geometry. The batch of tiles is cut into equal chunks when it would not fit in half
        the free device memory (a bound from memory, fixed per geometry so every step replays one captured graph)."""
        p = self.split_input_params
        key = (tuple(shape), uf, str(device), tuple(sorted((k, str(v)) for k, v in p.items())))
        cache = self.__dict__.setdefault("_split_cache", {})
        if key not in cache:
            nb, _, h, w = shape
            ks, stride, grid = split_geometry(h, w, p, uf)
            weight, norm = split_tables(ks, stride, grid, p, uf)
            n = grid[0] * grid[1] * nb
            if uf == 1:
                per_tile = ks[0] * ks[1] * self.model.diffusion_model.model_channels * _UNET_TILE_BYTES
            else:
                dd = self.first_stage_model.cfg["ddconfig"]
                per_tile = ks[0] * ks[1] * uf * uf * dd["ch"] * dd["ch_mult"][0] * _DECODER_TILE_BYTES
            cap = max(1, int(torch.cuda.mem_get_info(device)[0] // 2 // per_tile))
            chunks = -(-n // cap)
            cache[key] = dict(ks=ks, stride=stride, grid=grid, n=n, chunk=-(-n // chunks), chunks=chunks,
                              weight=weight.to(device), norm=norm.to(device))
        return cache[key]

    def _apply_split(self, x, t, cond):
        """The split apply_model (ddpm.py:891-992, concat conditioning or none): every tile of every sample in one UNet
        batch (tile l*nb + n; GroupNorm and attention are per sample, so this is the reference's per-tile loop), stitched
        by sdb_patch_fold. The conditioning tiles are gathered once per conditioning tensor, not per step."""
        if len(cond) != 1:
            raise NotImplementedError("split apply_model takes one conditioning")
        key = self.model.conditioning_key
        c = None
        if key is not None:
            if key != "concat" or self.cond_stage_key not in SPLIT_COND_KEYS:
                raise NotImplementedError(f"split apply_model with {key!r} conditioning and cond_stage_key "
                                          f"{self.cond_stage_key!r}: supported are concat conditioning on {SPLIT_COND_KEYS}")
            cl = cond["c_concat"]
            c = cl[0] if len(cl) == 1 else torch.cat(cl, 1)
        x = x.contiguous().float()
        plan = self._split_plan(x.shape, 1, x.device)
        ks, stride, n, chunk, chunks = plan["ks"], plan["stride"], plan["n"], plan["chunk"], plan["chunks"]
        unet = self.model.diffusion_model
        ct = None if c is None else self._cond_tiles(c, plan, chunk * chunks)
        ts = t.reshape(-1).repeat(n // x.shape[0])
        if chunks == 1:
            # graph mode: x_t's tiles go straight into the captured graph's static input
            bufs = unet.graph_inputs((n, x.shape[1], *ks), None if ct is None else tuple(ct.shape))
            xt = ops.patch_unfold(x, ks, stride, out=None if bufs is None else bufs[0])
        else:
            xt = torch.zeros((chunk * chunks, x.shape[1], *ks), dtype=torch.float32, device=x.device)
            ops.patch_unfold(x, ks, stride, out=xt[:n])
            ts = torch.cat([ts, ts[:1].expand(chunk * chunks - n)])
        eps = []
        for i in range(chunks):
            s = slice(i * chunk, (i + 1) * chunk)
            eps.append(self.model(xt[s], ts[s]) if ct is None else self.model(xt[s], ts[s], c_concat=[ct[s]]))
        eps = eps[0] if chunks == 1 else torch.cat(eps)[:n]
        return ops.patch_fold(eps.contiguous().float(), plan["weight"], plan["norm"], plan["grid"], stride)

    def _cond_tiles(self, c, plan, rows):
        """The conditioning's tiles ([rows, c, kh, kw], zero rows after the last tile), cached for the tensor they came
        from: the conditioning is constant over a sampling run."""
        key = (c.data_ptr(), c._version, tuple(c.shape), plan["ks"], plan["stride"], rows)
        hit = self.__dict__.get("_split_cond")
        if hit is None or hit[0] != key:
            ct = torch.zeros((rows, c.shape[1], *plan["ks"]), dtype=torch.float32, device=c.device)
            ops.patch_unfold(c.contiguous().float(), plan["ks"], plan["stride"], out=ct[:plan["n"]])
            hit = (key, ct, c)        # c is kept alive, so its address is not reused by another tensor
            self._split_cond = hit
        return hit[1]

    def _decode_split(self, z, force_not_quantize):
        """The split decode_first_stage (ddpm.py:705-763): quantize and post_quant_conv once on the whole latent (both
        act per pixel, so this equals the reference's per-tile quantize), cut tiles, decode them in memory-bounded equal
        chunks, and stitch the vqf-times larger tiles with sdb_patch_fold straight from the decoder's NHWC output."""
        fs = self.first_stage_model
        uf = int(self.split_input_params["vqf"])
        z = z.contiguous().float()
        plan = self._split_plan(z.shape, uf, z.device)
        scale = 1. / float(self.scale_factor)
        if isinstance(fs, VQModelInterface):
            q = fs.post_quant(z, force_not_quantize=force_not_quantize, scale=scale)
        else:
            q = fs.post_quant(z, scale=scale)
        qt, _ = ops.nchw_to_nhwc(ops.patch_unfold(ops.nhwc_to_nchw(q), plan["ks"], plan["stride"]))
        chunk = plan["chunk"]
        outs = [fs._decoder(qt[i:i + chunk]) for i in range(0, plan["n"], chunk)]
        o = outs[0] if len(outs) == 1 else torch.cat(outs)
        stride = (plan["stride"][0] * uf, plan["stride"][1] * uf)
        return ops.patch_fold(o, plan["weight"], plan["norm"], plan["grid"], stride, nhwc=True)

    def set_context(self, c):
        """Fast path used by sdb200 samplers: cross-attention K/V of the (guidance-doubled) context, once per batch. A
        concat model has no cross-attention: its conditioning reaches the UNet through apply_model on every step."""
        if c is not None and self.model.conditioning_key == "crossattn":
            self.model.diffusion_model.set_context(c)

    def get_learned_conditioning(self, c):
        enc = getattr(self.cond_stage_model, "encode", None)
        if callable(enc):
            c = enc(c)
            if not torch.is_tensor(c) and hasattr(c, "mode"):   # DiagonalGaussianDistribution (ddpm.py:555-556)
                c = c.mode()
        else:
            c = self.cond_stage_model(c)
        return c

    # -- first stage
    def encode_first_stage(self, x):
        return self.first_stage_model.encode(x)

    def get_first_stage_encoding(self, encoder_posterior, noise=None):
        if hasattr(encoder_posterior, "sample"):
            return encoder_posterior.sample(noise=noise, scale=float(self.scale_factor))
        if torch.is_tensor(encoder_posterior):
            return float(self.scale_factor) * encoder_posterior
        raise NotImplementedError(f"encoder_posterior of type '{type(encoder_posterior)}' not yet implemented")

    def decode_first_stage(self, z, predict_cids=False, force_not_quantize=False):
        if predict_cids:
            raise NotImplementedError("decode_first_stage(predict_cids=True): codebook-index latents are not supported")
        sp = getattr(self, "split_input_params", None)
        if sp is not None and sp["patch_distributed_vq"]:
            return self._decode_split(z, force_not_quantize)
        if isinstance(self.first_stage_model, VQModelInterface):     # ddpm.py:753-761: quantize, then decode
            return self.first_stage_model.decode(z, force_not_quantize=force_not_quantize,
                                                 scale=1. / float(self.scale_factor))
        return self.first_stage_model.decode(z, scale=1. / float(self.scale_factor))

    def q_sample(self, x_start, t, noise=None):
        if noise is None:
            noise = torch.randn_like(x_start)
        t_host = t.detach().to("cpu").long()
        assert bool((t_host == t_host[0]).all()), "q_sample: one timestep per call"
        a = float(self.sqrt_alphas_cumprod[int(t_host[0])])
        s = float(self.sqrt_one_minus_alphas_cumprod[int(t_host[0])])
        return ops.axpby2(x_start.contiguous().float(), noise.contiguous().float(), a, s)

    def _q_sample_per_sample(self, x_start, t, noise):
        """q_sample at one timestep per sample: the uniform-t route of q_sample when every t is equal (so the result
        does not depend on which route ran), sdb_q_sample_t otherwise."""
        t = t.to(self.device, torch.long).reshape(-1).contiguous()
        t_host = t.cpu()
        if bool((t_host == t_host[0]).all()):
            if not 0 <= int(t_host[0]) < self.num_timesteps:
                raise IndexError(f"timesteps must lie in [0, {self.num_timesteps}), got {int(t_host[0])}")
            return self.q_sample(x_start, t_host, noise)
        return ops.q_sample_t(x_start.contiguous().float(), noise.contiguous().float(), t,
                              self.sqrt_alphas_cumprod, self.sqrt_one_minus_alphas_cumprod)

    # -- denoising objective, forward only (ddpm.py:279-293, 654-705, 865-880, 1012-1045, 358-364)
    def get_loss(self, pred, target, mean=True):
        """get_loss (ddpm.py:279-293) with mean=True: the l1 / l2 mean over every element, from the per-sample means
        of sdb_diffusion_loss (every sample has the same size, so their mean is the overall mean). The elementwise form
        (mean=False) is not materialized: p_losses reduces per sample inside the kernel."""
        if not mean:
            raise NotImplementedError("get_loss(mean=False): elementwise losses are not materialized; p_losses reduces "
                                      "them per sample with sdb_diffusion_loss")
        t = torch.zeros(pred.shape[0], dtype=torch.long, device=pred.device)
        per = ops.diffusion_loss(pred.contiguous().float(), target.contiguous().float(), self.loss_type, t,
                                 self.logvar, self.lvlb_weights)
        return per[0].cpu().double().mean().float()

    def p_losses(self, x_start, cond, t, noise=None):
        """ddpm.py:1012-1045: noise x_start to t (one timestep per sample), predict eps with apply_model, and reduce.
        Returns (loss, loss_dict) with the reference's keys under train/ or val/ (from self.training); the values are
        0-d fp32 CPU tensors, the batch means formed on the host in the reference's order."""
        x_start = x_start.to(self.device).contiguous().float()
        if noise is None:
            noise = torch.randn_like(x_start)
        noise = noise.to(self.device).contiguous().float()
        t = t.to(self.device, torch.long).reshape(-1).contiguous()
        x_noisy = self._q_sample_per_sample(x_start, t, noise)
        model_output = self.apply_model(x_noisy, t, cond)
        per = ops.diffusion_loss(model_output.contiguous().float(), noise, self.loss_type, t, self.logvar,
                                 self.lvlb_weights).cpu()
        prefix = "train" if self.training else "val"
        loss_simple, loss, loss_vlb = per[0], per[1], per[2]
        loss_dict = {f"{prefix}/loss_simple": loss_simple.mean()}
        loss = self.l_simple_weight * loss.mean()
        loss_vlb = loss_vlb.mean()
        loss_dict[f"{prefix}/loss_vlb"] = loss_vlb
        loss = loss + self.original_elbo_weight * loss_vlb
        loss_dict[f"{prefix}/loss"] = loss
        return loss, loss_dict

    def forward(self, x, c, *args, **kwargs):
        """ddpm.py:870-879: a uniformly drawn timestep per sample, then p_losses."""
        t = torch.randint(0, self.num_timesteps, (x.shape[0],), device=self.device).long()
        if self.model.conditioning_key is not None:
            assert c is not None
            if self.cond_stage_trainable:
                c = self.get_learned_conditioning(c)
        return self.p_losses(x, c, t, *args, **kwargs)

    @staticmethod
    def _batch_image(batch, k):
        """DDPM.get_input (ddpm.py:329-335): a [B, H, W(, C)] tensor to NCHW fp32."""
        x = batch[k]
        if not torch.is_tensor(x):
            raise TypeError(f"get_input: batch[{k!r}] must be a [B, H, W, C] tensor, got {type(x).__name__}")
        if x.dim() == 3:
            x = x[..., None]
        return x.permute(0, 3, 1, 2).contiguous().float()

    @torch.no_grad()
    def get_input(self, batch, k, return_first_stage_outputs=False, force_c_encode=False, cond_key=None,
                  return_original_cond=False, bs=None):
        """ddpm.py:654-705: encode batch[k] ([B, H, W, C] in [-1, 1]) with the first stage (a KL posterior is sampled
        with noise drawn on the CPU generator, as the reference does) and build the conditioning from the batch:
        `caption` (a list of strings, tokenized by the cond stage), `class_label` (the whole batch goes to
        ClassEmbedder) or an image-like key such as `segmentation` or `LR_image`. Returns [z, c] (+ [x, xrec] + [xc])."""
        conditional = self.model.conditioning_key is not None
        cond_key = self.cond_stage_key if cond_key is None else cond_key
        if conditional and cond_key in ("txt", "coordinates_bbox", "nix"):
            raise NotImplementedError(f"get_input: cond_stage_key {cond_key!r} has no conditioning path in the "
                                      "reference's get_input (ddpm.py:664-672)")
        if conditional and cond_key == "masked_image":
            raise NotImplementedError(
                "get_input: 'masked_image' conditioning is built by scripts/inpaint.py (masked image encoded by the "
                "first stage, concatenated with the downsampled mask); pass that conditioning to p_losses instead")
        x = self._batch_image(batch, k)
        if bs is not None:
            x = x[:bs]
        x = x.to(self.device)
        z = self.get_first_stage_encoding(self.encode_first_stage(x))
        xc = c = None
        if conditional:
            if cond_key != self.first_stage_key:
                if cond_key == "caption":
                    xc = batch[cond_key]
                elif cond_key == "class_label":
                    xc = batch
                else:
                    xc = self._batch_image(batch, cond_key).to(self.device)
            else:
                xc = x
            if not self.cond_stage_trainable or force_c_encode:
                c = self.get_learned_conditioning(xc)
            else:
                c = xc
            if bs is not None:
                c = c[:bs]
        out = [z, c]
        if return_first_stage_outputs:
            out.extend([x, self.decode_first_stage(z)])
        if return_original_cond:
            out.append(xc)
        return out

    @torch.no_grad()
    def shared_step(self, batch, **kwargs):
        x, c = self.get_input(batch, self.first_stage_key)
        return self(x, c)

    @torch.no_grad()
    def validation_step(self, batch, batch_idx):
        """ddpm.py:358-364 without the logger: the raw weights' loss_dict merged with the EMA weights' (keys + '_ema'),
        each from its own shared_step (its own t, noise and posterior sample). Runs in eval mode, so the keys carry
        the val/ prefix as under Lightning's validation loop."""
        was_training = self.training
        self.eval()
        try:
            _, loss_dict_no_ema = self.shared_step(batch)
            with self.ema_scope():
                _, loss_dict_ema = self.shared_step(batch)
                loss_dict_ema = {key + "_ema": loss_dict_ema[key] for key in loss_dict_ema}
        finally:
            self.train(was_training)
        return {**loss_dict_no_ema, **loss_dict_ema}

    # -- ancestral sampler (ddpm.py:1047-1213), unconditional models
    def _p_step(self, img, t, noise):
        """LatentDiffusion.p_sample (clip_denoised=False, one timestep for the batch) as one fused kernel; the scalars
        are the fp32 schedule entries, and sigma is formed as the reference does: nonzero_mask * exp(0.5 * logvar)."""
        b = img.shape[0]
        ts = torch.full((b,), t, device=img.device, dtype=torch.long)
        eps = self.apply_model(img, ts, None).contiguous().float()
        cpu = lambda k: getattr(self, k)[t].detach().to("cpu", torch.float32)
        sigma = (torch.tensor(1.0 if t != 0 else 0.0) * (0.5 * cpu("posterior_log_variance_clipped")).exp()).item()
        return ops.ddpm_step(img, eps, noise, sqrt_recip_ac=cpu("sqrt_recip_alphas_cumprod").item(),
                             sqrt_recipm1_ac=cpu("sqrt_recipm1_alphas_cumprod").item(),
                             coef1=cpu("posterior_mean_coef1").item(), coef2=cpu("posterior_mean_coef2").item(),
                             sigma=sigma)

    def _check_uncond(self, cond):
        if cond is not None or self.model.conditioning_key is not None:
            raise NotImplementedError("the ancestral sampler runs unconditional models (cond None) only")

    @torch.no_grad()
    def p_sample_loop(self, cond, shape, return_intermediates=False, x_T=None, verbose=True, callback=None,
                      timesteps=None, quantize_denoised=False, mask=None, x0=None, img_callback=None, start_T=None,
                      log_every_t=None):
        """ddpm.py:1165-1213 (no mask): ancestral steps T-1 .. 0; intermediates are the latents."""
        self._check_uncond(cond)
        assert mask is None and not quantize_denoised
        log_every_t = log_every_t or self.log_every_t
        img = torch.randn(shape, device=self.device) if x_T is None else x_T.to(self.device, torch.float32).contiguous()
        intermediates = [img]
        timesteps = self.num_timesteps if timesteps is None else timesteps
        if start_T is not None:
            timesteps = min(timesteps, start_T)
        for i in reversed(range(0, timesteps)):
            img, _ = self._p_step(img, i, torch.randn(img.shape, device=img.device))
            if i % log_every_t == 0 or i == timesteps - 1:
                intermediates.append(img)
            if callback:
                callback(i)
            if img_callback:
                img_callback(img, i)
        return (img, intermediates) if return_intermediates else img

    @torch.no_grad()
    def progressive_denoising(self, cond, shape, verbose=True, callback=None, quantize_denoised=False, img_callback=None,
                              mask=None, x0=None, temperature=1., noise_dropout=0., score_corrector=None,
                              corrector_kwargs=None, batch_size=None, x_T=None, start_T=None, log_every_t=None):
        """ddpm.py:1110-1163 (no mask): ancestral steps T-1 .. 0; intermediates are the x0 predictions."""
        self._check_uncond(cond)
        assert mask is None and not quantize_denoised and noise_dropout == 0. and score_corrector is None
        log_every_t = log_every_t or self.log_every_t
        timesteps = self.num_timesteps
        if batch_size is not None:
            shape = [batch_size] + list(shape)
        img = torch.randn(shape, device=self.device) if x_T is None else x_T.to(self.device, torch.float32).contiguous()
        if start_T is not None:
            timesteps = min(timesteps, start_T)
        if isinstance(temperature, float):
            temperature = [temperature] * timesteps
        intermediates = []
        for i in reversed(range(0, timesteps)):
            noise = torch.randn(img.shape, device=img.device)       # noise_like, util.py:264-267
            if temperature[i] != 1.:
                noise = noise * temperature[i]
            img, x0_partial = self._p_step(img, i, noise)
            if i % log_every_t == 0 or i == timesteps - 1:
                intermediates.append(x0_partial)
            if callback:
                callback(i)
            if img_callback:
                img_callback(img, i)
        return img, intermediates
