"""Checkpoint ingest on the H100: a reference-format checkpoint (fp16 safetensors and pickled .ckpt) loaded through
`load_model_from_config` evaluates like the oracle on the very tensors the file holds."""
import pytest
import torch

from helpers import rel_l2
from sdb200 import arch, checkpoint
from test_checkpoint_cpu import _full_sd, _tiny_yaml

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]


@pytest.mark.parametrize("fmt,dtype", [("safetensors", torch.float16), ("ckpt", torch.float32)])
def test_checkpoint_to_eps_and_image(cuda_dev, tmp_path, fmt, dtype):
    import ldm_oracle as O
    sd = _full_sd(dtype)
    path = str(tmp_path / f"model.{fmt}")
    if fmt == "ckpt":
        torch.save({"state_dict": sd, "global_step": 1}, path)
    else:
        checkpoint.write_safetensors(path, sd)
    model = checkpoint.load_model_from_config(_tiny_yaml(tmp_path), path, device=cuda_dev)
    g = torch.Generator().manual_seed(21)
    x = torch.randn(2, 4, 16, 16, generator=g)
    ctx = torch.randn(2, 77, arch.TINY_UNET["context_dim"], generator=g)
    t = torch.tensor([801, 41])
    eps = model.apply_model(x.to(cuda_dev), t.to(cuda_dev), ctx.to(cuda_dev))
    usd = {k[len("model.diffusion_model."):]: v.float() for k, v in sd.items() if k.startswith("model.diffusion_model.")}
    ref = O.unet_forward(usd, x, t, ctx, num_heads=arch.TINY_UNET["num_heads"])
    assert rel_l2(eps, ref) < 2e-3, rel_l2(eps, ref)
    vsd = {k[len("first_stage_model."):]: v.float() for k, v in sd.items() if k.startswith("first_stage_model.")}
    z = torch.randn(1, 4, 8, 8, generator=g)
    img = model.decode_first_stage(z.to(cuda_dev))
    assert rel_l2(img, O.decode_first_stage(vsd, z)) < 3e-3
