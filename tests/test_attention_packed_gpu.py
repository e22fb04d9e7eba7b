"""sdb_attention with heads packed at stride d (head_stride = d, the layout the UNet projections produce) against an
fp64 restatement, and against the head-padded layout (head_stride = dpad) of the same data: the tensor cores see the
same operands either way (the tensor maps read columns d .. 63 of a panel as zeros), so the outputs are bit-identical.
Memory the kernel must not read holds NaN."""
import pytest
import torch

import sdb200 as S
from sdb200 import arch

from helpers import rel_l2

pytestmark = pytest.mark.gpu

NAN = float("nan")


def _ref(q, k, v, scale, causal):   # [B, H, n, d] fp16 -> fp64 [B, nq, H*d]
    s = torch.einsum("bhid,bhjd->bhij", q.double(), k.double()) * scale
    if causal:
        nq, nkv = s.shape[-2:]
        s = s.masked_fill(torch.ones(nq, nkv, dtype=torch.bool, device=s.device).triu(1), float("-inf"))
    o = torch.einsum("bhij,bhjd->bhid", s.softmax(-1), v.double())
    B, H, nq, d = o.shape
    return o.permute(0, 2, 1, 3).reshape(B, nq, H * d)


def _tokens(t, hs, extra):
    """[B, H, n, d] -> [B, n, H*hs + extra] view of a NaN-filled buffer; per-head columns d .. hs-1 and the row tail
    beyond H*hs stay NaN."""
    B, H, n, d = t.shape
    buf = torch.full((B, n, H * hs + extra), NAN, dtype=torch.float16, device=t.device)
    buf[:, :, :H * hs].view(B, n, H, hs)[..., :d] = t.permute(0, 2, 1, 3)
    return buf[:, :, :H * hs]


def _vt(v, hs, ld):
    """[B, H, nkv, d] -> V^T [B, H*hs, ld]; rows d .. hs-1 of each head and columns nkv .. ld-1 hold NaN."""
    B, H, nkv, d = v.shape
    vt = torch.full((B, H * hs, ld), NAN, dtype=torch.float16, device=v.device)
    vt.view(B, H, hs, ld)[:, :, :d, :nkv] = v.transpose(2, 3)
    return vt


CASES = [  # B, H, nq, nkv, d, causal
    (2, 8, 4096, 4096, 40, False),   # SD-v1 64x64 self-attention
    (2, 8, 4096, 77, 40, False),     # and its cross-attention
    (2, 8, 1024, 1024, 80, False), (2, 8, 1024, 77, 80, False),
    (2, 8, 256, 256, 160, False), (2, 8, 256, 77, 160, False),
    (2, 4, 1024, 1024, 32, False), (2, 4, 256, 77, 64, False),
    (2, 8, 256, 256, 24, False), (1, 8, 300, 300, 8, False),
    (2, 12, 77, 77, 64, True), (1, 2, 300, 97, 40, True),   # causal (CLIP), ragged
    (1, 3, 200, 333, 80, False), (1, 2, 130, 45, 24, False), (1, 2, 65, 129, 160, False),   # ragged nq / nkv
]


@pytest.mark.parametrize("B,H,nq,nkv,d,causal", CASES)
def test_packed_heads(cuda_dev, B, H, nq, nkv, d, causal):
    dpad = (d + 63) // 64 * 64
    g = torch.Generator(device=cuda_dev).manual_seed(nq * 7 + nkv + d)
    rnd = lambda *s: torch.randn(*s, generator=g, device=cuda_dev).half()
    q, k, v = rnd(B, H, nq, d), rnd(B, H, nkv, d), rnd(B, H, nkv, d)
    scale = d ** -0.5
    ld = (nkv + 7) // 8 * 8 + 8
    outs = {}
    for hs in (d, dpad):
        wide = torch.full((B, nq, H * d + 16), NAN, dtype=torch.float16, device=cuda_dev)
        out = wide[:, :, :H * d]
        S.ops.attention(_tokens(q, hs, 24), _tokens(k, hs, 24), _vt(v, hs, ld), heads=H, d=d, dpad=dpad, nq=nq,
                        nkv=nkv, scale=scale, causal=causal, out=out, head_stride=hs)
        torch.cuda.synchronize()
        assert bool(torch.isfinite(out).all()), f"head_stride {hs}: NaN the kernel must not read reached the output"
        assert bool(torch.isnan(wide[:, :, H * d:]).all()), f"head_stride {hs}: columns beyond heads*d were written"
        outs[hs] = out.clone()
    assert torch.equal(outs[d], outs[dpad]), "packed and padded layouts differ"
    err = rel_l2(outs[d].cpu(), _ref(q, k, v, scale, causal).cpu())
    assert err < 2e-3, err


def test_head_stride_validation(cuda_dev):
    q = torch.zeros(1, 64, 2 * 40, dtype=torch.float16, device=cuda_dev)
    vt = torch.zeros(1, 2 * 40, 64, dtype=torch.float16, device=cuda_dev)
    for hs in (36, 44):   # below d; not a multiple of 8
        with pytest.raises(RuntimeError, match="head_stride"):
            S.ops.attention(q, q, vt, heads=2, d=40, dpad=64, nq=64, nkv=64, scale=1.0, head_stride=hs)


def test_sdv1_graph_and_handle_bit_equal(cuda_dev):
    """SD-v1 UNet (packed heads at d = 40 / 80 / 160) at (2, 4, 32, 32): graph replay and the C handle reproduce the
    Python-sequenced forward bit for bit."""
    net = S.UNetModel(**arch.SD_V1_UNET).load_weights(
        arch.random_state_dict(arch.unet_param_shapes(arch.SD_V1_UNET), 5, device=cuda_dev), cuda_dev)
    g = torch.Generator(device=cuda_dev).manual_seed(0)
    x = torch.randn(2, 4, 32, 32, generator=g, device=cuda_dev)
    ctx = torch.randn(2, 77, 768, generator=g, device=cuda_dev)
    t = torch.tensor([981.0, 500.0], device=cuda_dev)
    h = net.c_handle(tuple(x.shape), ctx)
    ref = net(x, t, context=ctx)
    net.use_cuda_graph = True
    first = net(x, t, context=ctx)
    replay = net(x, t, context=ctx)
    out = h.forward(x, t)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(ref).all())
    assert torch.equal(first, ref) and torch.equal(replay, ref)
    assert torch.equal(out, ref), rel_l2(out.cpu(), ref.cpu())
    h.close()
