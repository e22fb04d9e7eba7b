"""SURVEY 8(f) rows on the H100: DPM-Solver++ sampler and the inpainting (mask) branch of PLMS / DDIM — the fused
step kernels bit for bit against the oracle on replayed eps, and the whole loop on the tiny model against the
reference's own outputs (tests/golden/samplers_ext.pt)."""
import pytest
import torch

from helpers import golden, rel_l2
from test_pipeline_gpu import _ReplayModel, _tiny_ld

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def _standin(rec):
    def model_fn(x, t, cc):
        e = torch.tanh(0.7 * x + 1e-4 * t.float()[:, None, None, None]) + 0.05 * cc.mean(dim=(1, 2))[:, None, None, None]
        rec.append(e)
        return e
    return model_fn


@pytest.mark.parametrize("S,scale", [(10, 7.5), (20, 7.5), (12, 1.0)])
def test_dpm_solver_arithmetic_bit_exact(cuda_dev, S, scale):
    import ldm_oracle as O
    import sdb200
    g = torch.Generator().manual_seed(6)
    B, shape = 2, (4, 8, 8)
    x_T, c = torch.randn(B, *shape, generator=g), torch.randn(B, 77, 64, generator=g)
    uc = torch.randn(B, 77, 64, generator=g) if scale != 1.0 else None
    rec = []
    ref = O.dpm_solver_sample(_standin(rec), x_T, c, uc, scale, S=S)
    model = _ReplayModel(O.register_schedule(), rec, cuda_dev)
    seen_t = []

    def apply_model(x, t, cc):
        assert t.dtype == torch.float32 and x.shape[0] == (2 * B if uc is not None else B)
        seen_t.append(float(t[0]))
        model.calls.append((tuple(x.shape), 0))
        return model.eps[len(model.calls) - 1]
    model.apply_model = apply_model
    out, inter = sdb200.DPMSolverSampler(model).sample(
        S=S, conditioning=c.to(cuda_dev), batch_size=B, shape=list(shape), verbose=False,
        unconditional_guidance_scale=scale, unconditional_conditioning=None if uc is None else uc.to(cuda_dev),
        x_T=x_T.to(cuda_dev))
    assert inter is None and len(model.calls) == S          # one UNet evaluation per step, none after the last
    assert abs(seen_t[0] - 999.0) < 1e-3 and all(a > b for a, b in zip(seen_t, seen_t[1:]))
    assert torch.equal(out.cpu(), ref), float((out.cpu() - ref).abs().max())


@pytest.mark.parametrize("kind", ["plms", "ddim"])
def test_masked_sampler_arithmetic_bit_exact(cuda_dev, kind):
    import ldm_oracle as O
    import sdb200
    g = torch.Generator().manual_seed(8)
    B, shape = 2, (4, 8, 8)
    x_T, c, uc = torch.randn(B, *shape, generator=g), torch.randn(B, 77, 64, generator=g), torch.randn(B, 77, 64, generator=g)
    x0 = torch.randn(B, *shape, generator=g)
    mask = (torch.randn(B, 1, 8, 8, generator=g) > 0).float()
    qn = [torch.randn(B, *shape, generator=g) for _ in range(10)]
    rec = []
    fn = O.masked_plms_sample if kind == "plms" else O.masked_ddim_sample
    ref = fn(_standin(rec), x_T, c, uc, 7.5, mask, x0, qn, S=10)
    sched = O.register_schedule()
    model = _ReplayModel(sched, rec, cuda_dev)
    sa, s1 = sched["sqrt_alphas_cumprod"], sched["sqrt_one_minus_alphas_cumprod"]
    qcalls = []

    def q_sample(x_start, t, noise=None):   # the reference facade's q_sample (ddpm.py:274-277) with recorded draws
        n = qn[len(qcalls)].to(cuda_dev)
        qcalls.append(int(t[0]))
        ti = t.cpu()
        return (sa[ti].reshape(-1, 1, 1, 1).to(cuda_dev) * x_start + s1[ti].reshape(-1, 1, 1, 1).to(cuda_dev) * n)
    model.q_sample = q_sample
    S_ = sdb200.PLMSSampler(model) if kind == "plms" else sdb200.DDIMSampler(model)
    out, inter = S_.sample(S=10, conditioning=c.to(cuda_dev), batch_size=B, shape=list(shape), verbose=False,
                           unconditional_guidance_scale=7.5, unconditional_conditioning=uc.to(cuda_dev), eta=0.0,
                           x_T=x_T.to(cuda_dev), mask=mask.to(cuda_dev), x0=x0.to(cuda_dev))
    assert qcalls == [901, 801, 701, 601, 501, 401, 301, 201, 101, 1]
    assert torch.equal(out.cpu(), ref), float((out.cpu() - ref).abs().max())
    with pytest.raises(AssertionError):      # mask without x0 (plms.py:148)
        S_.sample(S=10, conditioning=c.to(cuda_dev), batch_size=B, shape=list(shape), verbose=False, mask=mask.to(cuda_dev))


def test_mask_blend_full_channel_mask(cuda_dev):
    from sdb200 import ops
    g = torch.Generator().manual_seed(2)
    a, img = torch.randn(3, 4, 6, 6, generator=g), torch.randn(3, 4, 6, 6, generator=g)
    for mc in (1, 4):
        m = torch.rand(3, mc, 6, 6, generator=g)
        buf = torch.cat([img, torch.zeros_like(img)]).to(cuda_dev)
        ops.mask_blend(a.to(cuda_dev), m.to(cuda_dev), buf, 3, dup=True)
        ref = a * m + (1. - m) * img
        assert torch.equal(buf[:3].cpu(), ref) and torch.equal(buf[3:].cpu(), ref)


def test_dpm_solver_and_inpainting_vs_reference_tiny(cuda_dev):
    """Whole loops on the tiny LatentDiffusion (sdb200 UNet) against the reference run: fp16-operand error accumulated
    over the trajectory, same bounds as the PLMS / DDIM rows in test_pipeline_gpu.py."""
    import sdb200
    g = golden("samplers_ext.pt")
    ld = _tiny_ld(cuda_dev)
    dev = cuda_dev
    c, uc, x_T = g["c"].to(dev), g["uc"].to(dev), g["x_T"].to(dev)
    errs = {}
    for S, scale in ((20, 7.5), (10, 7.5), (15, 1.0)):
        s, _ = sdb200.DPMSolverSampler(ld).sample(S=S, conditioning=c, batch_size=2, shape=[4, 16, 16], verbose=False,
                                                  unconditional_guidance_scale=scale,
                                                  unconditional_conditioning=uc if scale != 1.0 else None, x_T=x_T)
        errs[f"dpm{S}_s{scale}"] = rel_l2(s, g[f"dpm{S}_s{scale}"])
    # inpainting with the reference's recorded q_sample draws
    for name, cls in (("plms", sdb200.PLMSSampler), ("ddim", sdb200.DDIMSampler)):
        draws = list(g[f"masked_{name}10_qnoise"])
        k = [0]
        real_q = ld.q_sample

        def q_sample(x_start, t, noise=None):
            n = draws[k[0]].to(dev)
            k[0] += 1
            return real_q(x_start, t, noise=n)
        ld.q_sample = q_sample
        try:
            s, _ = cls(ld).sample(S=10, conditioning=c, batch_size=2, shape=[4, 16, 16], verbose=False,
                                  unconditional_guidance_scale=7.5, unconditional_conditioning=uc, eta=0.0, x_T=x_T,
                                  mask=g["mask"].to(dev), x0=g["x0"].to(dev))
        finally:
            del ld.q_sample
        assert k[0] == 10
        errs[f"masked_{name}10"] = rel_l2(s, g[f"masked_{name}10"])
    print({k_: f"{v:.2e}" for k_, v in errs.items()})
    assert all(v < 3e-2 for v in errs.values()), errs
