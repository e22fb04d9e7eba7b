"""One eager forward of each model with random weights: the workloads whose kernel launches the sweeps record
(test_norm_sweep_gpu.py, test_attention_sweep_gpu.py). WORKLOADS maps a name to a function of the device."""
import torch

import helpers  # noqa: F401  (puts the repository on sys.path)
from sdb200 import arch


def _sd(shapes_fn, cfg, seed, dev):
    return arch.random_state_dict(shapes_fn(cfg), seed, device=dev)


def _run_unet(cfg, shapes, dev, ctx=None, concat=False):
    import sdb200
    net = sdb200.UNetModel(**cfg).load_weights(_sd(arch.unet_param_shapes, cfg, 11, dev), dev)
    g = torch.Generator(device=dev).manual_seed(0)
    for s in shapes:
        x = torch.randn(*s, generator=g, device=dev)
        t = torch.linspace(1, 981, s[0], device=dev).round()
        c = None if ctx is None else torch.randn(s[0], *ctx, generator=g, device=dev)
        if concat:
            half = s[1] // 2 if concat is True else concat
            net(x[:, :s[1] - half].contiguous(), t, concat=x[:, s[1] - half:].contiguous())
        else:
            net(x, t, context=c)
    del net


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
    enc.encode_ids(ids)


def _bert(cfg, dev, ids):
    import sdb200
    sdb200.BERTEmbedder(**cfg, use_tokenizer=False).load_weights(_sd(arch.bert_param_shapes, cfg, 13, dev),
                                                                 dev).encode_ids(ids)


def _clip_image(cfg, dev, B):
    import sdb200
    e = sdb200.FrozenClipImageEmbedder("ViT-L/14", config=cfg)
    e = e.load_weights(arch.random_state_dict(e.shapes, 16, device=dev), dev)
    g = torch.Generator(device=dev).manual_seed(5)
    e(torch.rand(B, 3, 224, 224, generator=g, device=dev) * 2 - 1)


def _ids(vocab, B, dev):
    g = torch.Generator(device=dev).manual_seed(3)
    return torch.randint(1, vocab - 2, (B, 77), generator=g, device=dev)


def _wl_sdv1_first(dev):
    import sdb200
    g = torch.Generator(device=dev).manual_seed(1)
    vae = _vae(arch.SD_V1_VAE, dev)
    vae.decode(torch.randn(1, 4, 64, 64, generator=g, device=dev))
    vae.encode(torch.rand(1, 3, 512, 512, generator=g, device=dev) * 2 - 1)
    del vae
    _clip(arch.SD_V1_CLIP, dev, _ids(49408, 2, dev))
    chk = sdb200.StableDiffusionSafetyChecker(config=arch.SD_V1_SAFETY).load_weights(
        _sd(arch.safety_param_shapes, arch.SD_V1_SAFETY, 14, dev), dev)
    chk.image_embeds(torch.randn(1, 3, 224, 224, generator=g, device=dev))


def _wl_laion(dev):
    _bert(arch.LAION_BERT, dev, _ids(30522, 2, dev))
    _run_unet(arch.LAION_UNET, [(2, 4, 64, 64)], dev, ctx=(77, 1280))


def _wl_rdm(dev):
    g = torch.Generator(device=dev).manual_seed(2)
    _run_unet(arch.RDM_UNET, [(2, 16, 48, 48)], dev, ctx=(11, 768))
    _vae(arch.KL_F16, dev).decode(torch.randn(1, 16, 24, 24, generator=g, device=dev))
    _clip(arch.CLIP_TEXT_PROJ, dev, _ids(49408, 2, dev))
    _clip_image(arch.CLIP_VISION_PROJ, dev, 2)


def _wl_celebahq(dev):
    g = torch.Generator(device=dev).manual_seed(2)
    _run_unet(arch.CELEBAHQ_UNET, [(2, 3, 64, 64)], dev)
    _vq(arch.VQ_F4, dev).decode(torch.randn(1, 3, 64, 64, generator=g, device=dev))


def _wl_cin_f8(dev):
    g = torch.Generator(device=dev).manual_seed(2)
    _run_unet(arch.CIN256_F8_UNET, [(2, 4, 32, 32)], dev, ctx=(1, 512))
    _vq(arch.VQ_F8, dev).decode(torch.randn(1, 4, 32, 32, generator=g, device=dev))


def _wl_inpaint(dev):
    g = torch.Generator(device=dev).manual_seed(3)
    _run_unet(arch.INPAINTING_BIG_UNET, [(1, 7, 128, 128)], dev, concat=4)
    m = _vq(arch.VQ_F4_NOATTN, dev)
    m.encode(torch.rand(1, 3, 512, 512, generator=g, device=dev) * 2 - 1)
    m.decode(torch.randn(1, 3, 128, 128, generator=g, device=dev))


def _wl_bsr(dev):
    g = torch.Generator(device=dev).manual_seed(3)
    _run_unet(arch.BSR_SR_UNET, [(1, 6, 128, 128)], dev, concat=3)
    _vq(arch.VQ_F4, dev).decode(torch.randn(1, 3, 64, 96, generator=g, device=dev))


def _wl_tiny(dev):
    g = torch.Generator(device=dev).manual_seed(4)
    _run_unet(arch.TINY_UNET, [(2, 4, 16, 16), (1, 4, 16, 24)], dev, ctx=(77, 64))
    _run_unet(arch.TINY_ATTN_UNET, [(2, 4, 16, 16)], dev)
    _run_unet(arch.TINY_LAION_UNET, [(2, 4, 16, 16)], dev, ctx=(77, 128))
    _run_unet(arch.TINY_RDM_UNET, [(2, 16, 16, 16)], dev, ctx=(3, 64))
    vae = _vae(arch.TINY_VAE, dev)
    vae.decode(torch.randn(1, 4, 8, 8, generator=g, device=dev))
    vae.encode(torch.rand(1, 3, 64, 64, generator=g, device=dev) * 2 - 1)
    _vae(arch.TINY_KL_F16, dev).decode(torch.randn(1, 16, 4, 4, generator=g, device=dev))
    _vq(arch.TINY_VQ, dev).decode(torch.randn(1, 3, 8, 8, generator=g, device=dev))
    _vq(arch.TINY_VQ_F8, dev).decode(torch.randn(1, 4, 8, 8, generator=g, device=dev))
    _clip(arch.TINY_CLIP, dev, _ids(1000, 2, dev))
    _clip(arch.TINY_CLIP_TEXT_PROJ, dev, _ids(1000, 2, dev))
    _bert(arch.TINY_BERT, dev, _ids(1000, 2, dev))
    _clip_image(arch.TINY_CLIP_VISION_PROJ, dev, 2)


WORKLOADS = {
    "sdv1_unet_b2": lambda dev: _run_unet(arch.SD_V1_UNET, [(2, 4, 64, 64), (2, 4, 64, 96)], dev, ctx=(77, 768)),
    "sdv1_vae_clip_safety": _wl_sdv1_first,
    "laion": _wl_laion,
    "rdm": _wl_rdm,
    "lsun": lambda dev: _run_unet(arch.LSUN_CHURCHES_UNET, [(2, 4, 32, 32)], dev),
    "celebahq": _wl_celebahq,
    "cin256_v2": lambda dev: _run_unet(arch.CIN256_V2_UNET, [(2, 3, 64, 64)], dev, ctx=(1, 512)),
    "cin256_f8": _wl_cin_f8,
    "inpaint": _wl_inpaint,
    "bsr": _wl_bsr,
    "semantic": lambda dev: _run_unet(arch.SEMANTIC_SYNTHESIS_UNET, [(1, 6, 64, 64)], dev, concat=3),
    "tiny": _wl_tiny,
}
