"""One eager forward of each model with random weights: the workloads whose kernel launches the sweeps record
(test_norm_sweep_gpu.py, test_attention_sweep_gpu.py, test_elementwise_sweep_gpu.py, test_gemm_plans_gpu.py, all four
over the first stages in test_first_stage_sweep_gpu.py, and the GEMM plan sweeps in the model test files). Each table
maps a name to a function of the device; a problem's operands are seeded by its index in the recorded list, so an
entry's shapes and call order are part of what a sweep checks. Each function returns what it computes (tensors,
possibly nested in lists and tuples), which test_pdl_order_gpu.py digests bit for bit."""
import torch

import helpers  # noqa: F401  (puts the repository on sys.path)
from sdb200 import arch, ops


def _sd(shapes_fn, cfg, seed, dev):
    return arch.random_state_dict(shapes_fn(cfg), seed, device=dev)


def _unet(cfg, dev):
    import sdb200
    return sdb200.UNetModel(**cfg).load_weights(_sd(arch.unet_param_shapes, cfg, 11, dev), dev)


def _run_unet(cfg, shapes, dev, ctx=None, concat=0):
    """One UNet evaluation per shape; concat > 0 passes the last `concat` channels as the concat conditioning."""
    net = _unet(cfg, dev)
    g = torch.Generator(device=dev).manual_seed(0)
    outs = []
    for s in shapes:
        x = torch.randn(*s, generator=g, device=dev)
        t = torch.linspace(1, 981, s[0], device=dev).round()
        c = None if ctx is None else torch.randn(s[0], *ctx, generator=g, device=dev)
        if concat:
            outs.append(net(x[:, :s[1] - concat].contiguous(), t, concat=x[:, s[1] - concat:].contiguous()))
        else:
            outs.append(net(x, t, context=c))
    del net
    return outs


def _vae(cfg, dev):
    import sdb200
    return sdb200.AutoencoderKL(**cfg).load_weights(_sd(arch.vae_param_shapes, cfg, 12, dev), dev)


def _vq(cfg, dev):
    import sdb200
    return sdb200.VQModelInterface(**cfg).load_weights(_sd(arch.vq_param_shapes, cfg, 12, dev), dev)


def _clip(cfg, dev, ids):
    import sdb200
    cls = sdb200.FrozenCLIPTextEmbedder if "projection_dim" in cfg else sdb200.FrozenCLIPEmbedder
    shapes = arch.clip_text_proj_param_shapes if "projection_dim" in cfg else arch.clip_param_shapes
    enc = cls(config=cfg).load_weights(_sd(shapes, cfg, 13, dev), dev)
    return enc.encode_ids(ids)


def _bert(cfg, dev, ids):
    import sdb200
    return sdb200.BERTEmbedder(**cfg, use_tokenizer=False).load_weights(_sd(arch.bert_param_shapes, cfg, 13, dev),
                                                                 dev).encode_ids(ids)


def _clip_image_embedder(cfg, dev):
    import sdb200
    e = sdb200.FrozenClipImageEmbedder("ViT-L/14", config=cfg)
    return e.load_weights(arch.random_state_dict(e.shapes, 16, device=dev), dev)


def _clip_image(cfg, dev, B):
    e = _clip_image_embedder(cfg, dev)
    g = torch.Generator(device=dev).manual_seed(5)
    return e(torch.rand(B, 3, 224, 224, generator=g, device=dev) * 2 - 1)


def _ids(vocab, B, dev):
    g = torch.Generator(device=dev).manual_seed(3)
    return torch.randint(1, vocab - 2, (B, 77), generator=g, device=dev)


def _wl_sdv1_first(dev):
    import sdb200
    g = torch.Generator(device=dev).manual_seed(1)
    vae = _vae(arch.SD_V1_VAE, dev)
    img = vae.decode(torch.randn(1, 4, 64, 64, generator=g, device=dev))
    post = vae.encode(torch.rand(1, 3, 512, 512, generator=g, device=dev) * 2 - 1)
    del vae
    c = _clip(arch.SD_V1_CLIP, dev, _ids(49408, 2, dev))
    chk = sdb200.StableDiffusionSafetyChecker(config=arch.SD_V1_SAFETY).load_weights(
        _sd(arch.safety_param_shapes, arch.SD_V1_SAFETY, 14, dev), dev)
    return img, post, c, chk.image_embeds(torch.randn(1, 3, 224, 224, generator=g, device=dev))


def _wl_laion(dev, text_batch, unet_batches):
    return (_bert(arch.LAION_BERT, dev, _ids(30522, text_batch, dev)),
            _run_unet(arch.LAION_UNET, [(nb, 4, 64, 64) for nb in unet_batches], dev, ctx=(77, 1280)))


def _wl_rdm_unet_kl(dev, nb):
    g = torch.Generator(device=dev).manual_seed(2)
    return (_run_unet(arch.RDM_UNET, [(nb, 16, 48, 48)], dev, ctx=(11, 768)),
            _vae(arch.KL_F16, dev).decode(torch.randn(1, 16, 24, 24, generator=g, device=dev)))


def _wl_rdm(dev):
    return (_wl_rdm_unet_kl(dev, 2), _clip(arch.CLIP_TEXT_PROJ, dev, _ids(49408, 2, dev)),
            _clip_image(arch.CLIP_VISION_PROJ, dev, 2))


def _wl_celebahq(dev, nb):
    g = torch.Generator(device=dev).manual_seed(2)
    return (_run_unet(arch.CELEBAHQ_UNET, [(nb, 3, 64, 64)], dev),
            _vq(arch.VQ_F4, dev).decode(torch.randn(1, 3, 64, 64, generator=g, device=dev)))


def _wl_cin_f8(dev, nb):
    g = torch.Generator(device=dev).manual_seed(2)
    return (_run_unet(arch.CIN256_F8_UNET, [(nb, 4, 32, 32)], dev, ctx=(1, 512)),
            _vq(arch.VQ_F8, dev).decode(torch.randn(1, 4, 32, 32, generator=g, device=dev)))


def _wl_inpaint(dev, batches):
    g = torch.Generator(device=dev).manual_seed(3)
    eps = _run_unet(arch.INPAINTING_BIG_UNET, [(nb, 7, 128, 128) for nb in batches], dev, concat=4)
    m = _vq(arch.VQ_F4_NOATTN, dev)
    return (eps, m.encode(torch.rand(1, 3, 512, 512, generator=g, device=dev) * 2 - 1),
            m.decode(torch.randn(1, 3, 128, 128, generator=g, device=dev)))


def _wl_bsr(dev):
    g = torch.Generator(device=dev).manual_seed(3)
    return (_run_unet(arch.BSR_SR_UNET, [(1, 6, 128, 128)], dev, concat=3),
            _vq(arch.VQ_F4, dev).decode(torch.randn(1, 3, 64, 96, generator=g, device=dev)))


def _wl_bsr_tiled(dev):
    """The UNet at a tiled sampling batch of 9 and the tiled decode's tile batch: a 192² latent, 2 x 2 tiles of 128²."""
    g = torch.Generator(device=dev).manual_seed(3)
    eps = _run_unet(arch.BSR_SR_UNET, [(9, 6, 128, 128)], dev, concat=3)
    vq = _vq(arch.VQ_F4, dev)
    q = vq.post_quant(torch.randn(1, 3, 192, 192, generator=g, device=dev))
    tiles, _ = ops.nchw_to_nhwc(ops.patch_unfold(ops.nhwc_to_nchw(q), (128, 128), (64, 64)))
    return eps, vq._decoder(tiles)


def _wl_vq_sr_tile(dev):
    g = torch.Generator(device=dev).manual_seed(6)
    return _vq(arch.VQ_F4, dev).decode(torch.randn(1, 3, 128, 128, generator=g, device=dev))


def text2img256(dev):
    """text2img256: BERT-640 on the cond + uncond ids of a batch of 3 (6 x 77 tokens), the UNet at the guidance batches
    2 and 8, and one VQ-f4 decode of a 64² latent (the model's scale_factor is 1)."""
    g = torch.Generator(device=dev).manual_seed(2)
    return (_bert(arch.TEXT2IMG256_BERT, dev, _ids(30522, 6, dev)),
            _run_unet(arch.TEXT2IMG256_UNET, [(2, 3, 64, 64), (8, 3, 64, 64)], dev, ctx=(77, 640)),
            _vq(arch.VQ_F4, dev).decode(torch.randn(1, 3, 64, 64, generator=g, device=dev)))


def _wl_clip_image_tower(dev):
    """The ViT-L/14 tower from patch rows at B = 1, 64 and 256 images (M = 256 B patch rows, 257 B token rows)."""
    e = _clip_image_embedder(arch.CLIP_VISION_PROJ, dev)
    g = torch.Generator(device=dev).manual_seed(0)
    return [e.embed_patches(torch.randn(B * 256, e.W["kpad"], generator=g, device=dev).half(), B) for B in (1, 64, 256)]


def _wl_tiny(dev):
    g = torch.Generator(device=dev).manual_seed(4)
    out = [_run_unet(arch.TINY_UNET, [(2, 4, 16, 16), (1, 4, 16, 24)], dev, ctx=(77, 64)),
           _run_unet(arch.TINY_ATTN_UNET, [(2, 4, 16, 16)], dev),
           _run_unet(arch.TINY_LAION_UNET, [(2, 4, 16, 16)], dev, ctx=(77, 128)),
           _run_unet(arch.TINY_RDM_UNET, [(2, 16, 16, 16)], dev, ctx=(3, 64))]
    vae = _vae(arch.TINY_VAE, dev)
    out.append(vae.decode(torch.randn(1, 4, 8, 8, generator=g, device=dev)))
    out.append(vae.encode(torch.rand(1, 3, 64, 64, generator=g, device=dev) * 2 - 1))
    out.append(_vae(arch.TINY_KL_F16, dev).decode(torch.randn(1, 16, 4, 4, generator=g, device=dev)))
    out.append(_vq(arch.TINY_VQ, dev).decode(torch.randn(1, 3, 8, 8, generator=g, device=dev)))
    out.append(_vq(arch.TINY_VQ_F8, dev).decode(torch.randn(1, 4, 8, 8, generator=g, device=dev)))
    out.append(_clip(arch.TINY_CLIP, dev, _ids(1000, 2, dev)))
    out.append(_clip(arch.TINY_CLIP_TEXT_PROJ, dev, _ids(1000, 2, dev)))
    out.append(_bert(arch.TINY_BERT, dev, _ids(1000, 2, dev)))
    out.append(_clip_image(arch.TINY_CLIP_VISION_PROJ, dev, 2))
    return out


# the norm sweep
WORKLOADS = {
    "sdv1_unet_b2": lambda dev: _run_unet(arch.SD_V1_UNET, [(2, 4, 64, 64), (2, 4, 64, 96)], dev, ctx=(77, 768)),
    "sdv1_vae_clip_safety": _wl_sdv1_first,
    "laion": lambda dev: _wl_laion(dev, 2, [2]),
    "rdm": _wl_rdm,
    "lsun": lambda dev: _run_unet(arch.LSUN_CHURCHES_UNET, [(2, 4, 32, 32)], dev),
    "celebahq": lambda dev: _wl_celebahq(dev, 2),
    "cin256_v2": lambda dev: _run_unet(arch.CIN256_V2_UNET, [(2, 3, 64, 64)], dev, ctx=(1, 512)),
    "cin256_f8": lambda dev: _wl_cin_f8(dev, 2),
    "inpaint": lambda dev: _wl_inpaint(dev, [1]),
    "bsr": _wl_bsr,
    "semantic": lambda dev: _run_unet(arch.SEMANTIC_SYNTHESIS_UNET, [(1, 6, 64, 64)], dev, concat=3),
    "tiny": _wl_tiny,
}

# the attention sweep
ATTENTION_WORKLOADS = {
    **WORKLOADS,
    "vq_f4_128x128_latent": _wl_vq_sr_tile,                                    # 16384 tokens at d = 512
    "vit_l14_b37": lambda dev: _clip_image(arch.CLIP_VISION_PROJ, dev, 37),
    "rdm_one_token_context": lambda dev: _run_unet(arch.RDM_UNET, [(2, 16, 48, 48)], dev, ctx=(1, 768)),
}

def _wl_cin256_class_embedder(dev):
    """The ClassEmbedder on all 1001 labels (1000: the unconditional one): embed_tokens with a one-row position table,
    then the one-token-context projection of every SpatialTransformer (UNetModel.context_kv)."""
    import sdb200
    cfg = arch.CIN256_V2_COND
    emb = sdb200.ClassEmbedder(**cfg).load_weights(_sd(arch.class_embedder_param_shapes, cfg, 15, dev), dev)
    c = emb({cfg["key"]: torch.arange(cfg["n_classes"], device=dev).flip(0)})
    return c, _unet(arch.CIN256_V2_UNET, dev).context_kv(c)


def _wl_sdv1_vae_sample(dev):
    """SD-v1 VAE encode with a posterior sample (vae_sample) at 512² and 512x768."""
    g = torch.Generator(device=dev).manual_seed(7)
    vae = _vae(arch.SD_V1_VAE, dev)
    return [vae.encode(torch.rand(1, 3, h, w, generator=g, device=dev) * 2 - 1).sample(
            noise=torch.randn(1, 4, h // 8, w // 8, generator=g, device=dev), scale=0.18215)
            for h, w in ((512, 512), (512, 768))]


def _wl_sdv1_decode_uint8(dev):
    """SD-v1 decodes to uint8 images as the txt2img / img2img pipelines return them: 2 x 512² and 1 x 512x768."""
    g = torch.Generator(device=dev).manual_seed(8)
    vae = _vae(arch.SD_V1_VAE, dev)
    return [ops.to_uint8(vae.decode(torch.randn(*s, generator=g, device=dev), scale=1 / 0.18215, nhwc=True))
            for s in ((2, 4, 64, 64), (1, 4, 64, 96))]


# the elementwise sweep: what a plain forward of the tables above does not reach
ELEMENTWISE_WORKLOADS = {
    **ATTENTION_WORKLOADS,
    "cin256_class_embedder": _wl_cin256_class_embedder,
    "sdv1_vae_sample": _wl_sdv1_vae_sample,
    "vit_l14_b256": lambda dev: _clip_image(arch.CLIP_VISION_PROJ, dev, 256),  # rows_gather stride 257, projection M 256
    "sdv1_decode_uint8": _wl_sdv1_decode_uint8,
}

# test_gemm_plans_gpu.py
GEMM_WORKLOADS = {
    "sdv1_unet_b2": lambda dev: _run_unet(arch.SD_V1_UNET, [(2, 4, 64, 64), (2, 4, 64, 96), (2, 4, 96, 64)], dev,
                                          ctx=(77, 768)),
    "sdv1_unet_b16": lambda dev: _run_unet(arch.SD_V1_UNET, [(16, 4, 64, 64)], dev, ctx=(77, 768)),
    "sdv1_vae_clip_safety": _wl_sdv1_first,
    "lsun": lambda dev: _run_unet(arch.LSUN_CHURCHES_UNET, [(10, 4, 32, 32)], dev),
    "celebahq": lambda dev: _wl_celebahq(dev, 10),
    "cin256": lambda dev: _run_unet(arch.CIN256_V2_UNET, [(12, 3, 64, 64), (2, 3, 32, 32)], dev, ctx=(1, 512)),
    "inpaint": lambda dev: _wl_inpaint(dev, [1, 4]),
}

# the GEMM plan sweeps of the model test files, one entry per file
GEMM_MODEL_WORKLOADS = {
    "rdm": lambda dev: _wl_rdm_unet_kl(dev, 6),
    "cin256_f8": lambda dev: _wl_cin_f8(dev, 6),
    "clip_image": _wl_clip_image_tower,
    "laion": lambda dev: _wl_laion(dev, 6, [2, 6]),
    "bsr_sr": _wl_bsr_tiled,
    "semantic": lambda dev: _run_unet(arch.SEMANTIC_SYNTHESIS_UNET, [(8, 6, 64, 64), (1, 6, 128, 128)], dev, concat=3),
}

# test_first_stage_sweep_gpu.py: every first stage of arch.FIRST_STAGES, kept out of the tables above so that their
# sweeps and the PDL digest child (pdl_child.ALL) do not grow
DECODE_SCALE = 1.3     # decode(z, scale): not 1, so the quantizer and the 1x1 head see a scale


def first_stage_geometries(f):
    """(batch, height, width) of the images a first stage of factor f runs: 256² (the configs' training size); 256x384
    at batch 2 (non-square, batch strides; every level attention of the nine configs has a token count divisible by 8
    there, e.g. KL-f32 at 16x24 and 8x12); and the thin f x 8f, whose 1 x 8 latent makes the last stride-2 conv run
    2 x 16 -> 1 x 8 with pad (0, 1, 0, 1), the mid attention run at 8 tokens and the last GroupNorms at 8 pixels."""
    return ((1, 256, 256), (2, 256, 384), (1, f, 8 * f))


def _wl_first_stage(cfg, dev):
    """At each geometry: encode (the posterior's mode for KL, VQModel.encode with indices for VQ), decode of a seeded
    latent at DECODE_SCALE (VQModelInterface.decode, which re-quantizes at that scale) and, for VQ, decode_code of the
    indices the encode chose."""
    import sdb200
    f = 2 ** (len(cfg["ddconfig"]["ch_mult"]) - 1)
    g = torch.Generator(device=dev).manual_seed(9)
    if "n_embed" in cfg:
        sd = _sd(arch.vq_param_shapes, cfg, 12, dev)
        vq, vqi = sdb200.VQModel(**cfg).load_weights(sd, dev), sdb200.VQModelInterface(**cfg).load_weights(sd, dev)
    else:
        kl = _vae(cfg, dev)
    outs = []
    for nb, h, w in first_stage_geometries(f):
        x = torch.rand(nb, 3, h, w, generator=g, device=dev) * 2 - 1
        z = torch.randn(nb, cfg["embed_dim"], h // f, w // f, generator=g, device=dev)
        if "n_embed" in cfg:
            quant, loss, (_, _, idx) = vq.encode(x)
            outs += [quant, loss, idx, vqi.decode(z, scale=DECODE_SCALE), vq.decode_code(idx.view(nb, h // f, w // f))]
        else:
            outs += [kl.encode(x).mode(), kl.decode(z, scale=DECODE_SCALE)]
    return outs


FIRST_STAGE_WORKLOADS = {name: (lambda cfg: lambda dev: _wl_first_stage(cfg, dev))(cfg)
                         for name, cfg in arch.FIRST_STAGES.items()}


# test_ae_loss_sweep_gpu.py: the KL autoencoders' validation loss (seeded LPIPSWithDiscriminator weights), kept out of
# the tables above for the same reason
AE_DISC_START = 50


def _wl_ae_loss(dev, nb, h, w):
    """Both LPIPSWithDiscriminator calls (optimizer_idx 0: rec / LPIPS / KL / g_loss; 1: the hinge discriminator loss)
    on each side of disc_start, for an nb x h x w image pair and a KL-f8 posterior with logvar drawn across both clamps."""
    import sdb200
    from sdb200 import ae_loss
    from sdb200.vae import DiagonalGaussianDistribution
    m = sdb200.LPIPSWithDiscriminator(disc_start=AE_DISC_START, kl_weight=1e-6, disc_weight=0.5)
    m.load_state_dict(ae_loss.random_loss_state_dict(ae_loss.loss_param_shapes(), 21))
    m = m.to(dev).eval()
    g = torch.Generator(device=dev).manual_seed(10)
    x = torch.rand(nb, 3, h, w, generator=g, device=dev) * 2 - 1
    xr = (x + 0.2 * torch.randn(nb, 3, h, w, generator=g, device=dev)).clamp(-1, 1)
    zh, zw = h // 8, w // 8
    mom = torch.randn(nb * zh * zw, 8, generator=g, device=dev)
    mom[:, 4:] *= 25
    post = DiagonalGaussianDistribution(mom, nb, zh, zw, 4)
    outs = []
    for idx in (0, 1):
        for gs in (AE_DISC_START - 1, AE_DISC_START):
            loss, log = m(x, xr, post, idx, gs, split="val")
            outs += [loss] + [log[k] for k in sorted(log)]
    return outs


def _wl_lpips_min_side(dev):
    """LPIPS at the smallest side it takes (four 2x2 pools leave one pixel): 16² at batch 3 and 16x24 at batch 1."""
    import sdb200
    from sdb200 import ae_loss
    lp = sdb200.LPIPS().load_weights(ae_loss.random_loss_state_dict(ae_loss.lpips_param_shapes(), 22), dev)
    g = torch.Generator(device=dev).manual_seed(11)
    s = ae_loss.LPIPS_MIN_SIDE
    return [lp(torch.rand(nb, 3, s, w, generator=g, device=dev) * 2 - 1, torch.rand(nb, 3, s, w, generator=g,
                                                                                    device=dev) * 2 - 1)
            for nb, w in ((3, s), (1, s + 8))]


AE_LOSS_WORKLOADS = {
    "ae_loss_256": lambda dev: _wl_ae_loss(dev, 4, 256, 256),        # scripts/eval_autoencoder.py's default batch
    "ae_loss_72x104": lambda dev: _wl_ae_loss(dev, 2, 72, 104),      # pools 9 x 13 -> 4 x 6: odd row and column dropped
    "lpips_min_side": _wl_lpips_min_side,
}
