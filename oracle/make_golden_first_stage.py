"""ORACLE tooling: generate tests/golden/first_stage.pt by running the UNMODIFIED reference (located by ref_harness.py) on
CPU fp32 for the first-stage autoencoders of models/first_stage_models/*/config.yaml.

Run in the build container:  python oracle/make_golden_first_stage.py

Stored:
- `yamls`: all nine config.yaml files as parsed data (model and data nodes), so no test reads the reference;
- `keys`: the reference's state-dict (key, shape) list of each, built from the YAML's params by the reference's own
  AutoencoderKL / VQModel with the training loss replaced by torch.nn.Identity (LPIPS is not importable here);
- `cases`: for the four geometries no LDM uses (KL-f4, KL-f32, VQ-f8-n256, VQ-f16), at full width with weights from
  arch.random_state_dict(WEIGHT_SEED) and a 128x128 input regenerated from its seed (gen(shape, seed).clamp(-1, 1)):
  KL: the posterior parameters (moments) and decode(mean); VQ: encode_to_prequant, the indices and emb_loss of encode,
  forward's dec (every IMAGE_STRIDE-th pixel) and, per latent pixel, the two smallest of the quantizer's distances
  sum(z^2) + sum(e^2) - 2 z.e, i.e. how close each index decision is.
The quantizer is oracle/vq_oracle.py's restatement of taming's VectorQuantizer2 (ref_harness.install()); the reference's
VQModel is built here (build_vq_model), next to the one generator that needs it. Every vector is also evaluated with the
oracle restatements (rdm_oracle / cin_f8_oracle) and the error printed.
"""
from __future__ import annotations

import contextlib
import io
import os
import sys

import torch
import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import cin_f8_oracle as F8  # noqa: E402
import rdm_oracle as RO  # noqa: E402
import ref_harness as R  # noqa: E402
from ref_harness import gen, rel  # noqa: E402
from sdb200 import arch  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
WEIGHT_SEED = 41
# decoded VQ images are stored at every IMAGE_STRIDE-th pixel in both directions, which keeps the file small; the tests
# decode in full and compare the same pixels
IMAGE_STRIDE = 2
# (name, input shape, input seed): one image for KL; four for VQ, so the index statistics cover 256 / 1024 latent pixels
NEW = (("kl-f4", (1, 3, 128, 128), 950), ("kl-f32", (1, 3, 128, 128), 951),
       ("vq-f8-n256", (4, 3, 128, 128), 952), ("vq-f16", (4, 3, 128, 128), 953))


def build_vq_model(cfg):
    """The reference's standalone VQModel (autoencoder.py:14-122), the target of models/first_stage_models/vq-*, with
    the training loss replaced by torch.nn.Identity as ref_harness's builders do."""
    R.install()
    from ldm.models.autoencoder import VQModel
    with contextlib.redirect_stdout(io.StringIO()):
        m = VQModel(embed_dim=cfg["embed_dim"], n_embed=cfg["n_embed"], ddconfig=cfg["ddconfig"],
                    lossconfig={"target": "torch.nn.Identity"})
    return m.eval()


def _model(cfg):
    return build_vq_model(cfg) if "n_embed" in cfg else R.build_vae(cfg)


def _cfg_of(node):
    p = node["params"]
    cfg = dict(embed_dim=p["embed_dim"], ddconfig=p["ddconfig"])
    if "n_embed" in p:
        cfg["n_embed"] = p["n_embed"]
    return cfg


def top2_distances(z, codebook):
    """The reference quantizer's distances (vq_oracle.VectorQuantizer2.forward), the two smallest per latent pixel."""
    zf = z.permute(0, 2, 3, 1).reshape(-1, codebook.shape[1])
    d = torch.sum(zf ** 2, dim=1, keepdim=True) + torch.sum(codebook ** 2, dim=1) - \
        2 * torch.einsum("bd,dn->bn", zf, codebook.t())
    return torch.topk(d, 2, dim=1, largest=False).values


@torch.no_grad()
def main():
    out = {"weight_seed": WEIGHT_SEED, "image_stride": IMAGE_STRIDE, "yamls": {}, "keys": {}, "cases": {}}
    for name in sorted(arch.FIRST_STAGES):
        with open(os.path.join(R.REF, "models", "first_stage_models", name, "config.yaml")) as f:
            y = yaml.safe_load(f)
        out["yamls"][name] = y
        cfg = _cfg_of(y["model"])
        assert cfg == arch.FIRST_STAGES[name], name
        m = _model(cfg)
        out["keys"][name] = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
        print(f"{name}: {y['model']['target']}, {len(out['keys'][name])} tensors")
        del m
    for name, shape, seed in NEW:
        cfg = arch.FIRST_STAGES[name]
        kl = "n_embed" not in cfg
        shapes = arch.vae_param_shapes(cfg) if kl else arch.vq_param_shapes(cfg)
        sd = arch.random_state_dict(shapes, WEIGHT_SEED)
        m = _model(cfg)
        m.load_state_dict(sd, strict=True)
        x = gen(shape, seed).clamp(-1, 1)
        case = dict(shape=shape, seed=seed)
        if kl:
            post = m.encode(x)
            case["moments"] = post.parameters.clone()
            case["dec"] = m.decode(post.mean)
            print(f"{name} {shape}: moments {tuple(post.parameters.shape)} oracle rel "
                  f"{rel(RO.kl_encode_moments(sd, x), post.parameters):.2e}; decode(mean) oracle rel "
                  f"{rel(RO.kl_decode(sd, post.mean), case['dec']):.2e}")
        else:
            h = m.encode_to_prequant(x)
            quant, emb_loss, (_, _, ind) = m.encode(x)
            dec, diff = m(x)
            assert torch.equal(diff, emb_loss) and torch.equal(dec, m.decode(quant))
            d2 = top2_distances(h, m.quantize.embedding.weight)
            case.update(h=h, indices=ind, emb_loss=emb_loss.clone(), d_top2=d2,
                        dec=dec[..., ::IMAGE_STRIDE, ::IMAGE_STRIDE].contiguous())
            gap = d2[:, 1] - d2[:, 0]
            print(f"{name} {shape}: latent {tuple(h.shape)} oracle rel {rel(F8.vq_encode(sd, x), h):.2e}; "
                  f"emb_loss {float(emb_loss):.4f}; {len(set(ind.tolist()))} distinct codes; top-two gap min "
                  f"{float(gap.min()):.2e} median {float(gap.median()):.2e}; dec oracle rel "
                  f"{rel(F8.vq_decode(sd, h), dec):.2e}")
        out["cases"][name] = case
        del m
    path = os.path.join(OUT, "first_stage.pt")
    torch.save(out, path)
    print(f"  wrote first_stage.pt ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    main()
