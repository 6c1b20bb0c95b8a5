"""The whole sampling chain of one StreamingSVD chunk on the project's GPU path — B200EulerEDMSampler x B200StreamingWrapper
x B200VaeDecoder — against the golden produced by the UNMODIFIED reference classes (EulerEDMSampler + Denoiser +
StreamingWrapper + VideoDecoder, oracle/make_golden_chain.py) on identical noise, conditioning and weights.

Tolerance (SURVEY.md section 8c): after 30 Euler steps, latent rel-L2 <= 3e-2 and decoded-frame pixel MSE <= 1e-3 on
[-1, 1].  The fixture also carries the reference's own bf16-autocast-vs-fp32 self-discrepancy on the same chain; it
is printed next to ours."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "chain_tiny_t8_16x16.npz")
LATENT_TOL, PIXEL_MSE_TOL = 3e-2, 1e-3


def _build(cuda_dev):
    from oracle.make_golden_chain import SCALE_FACTOR, SEED, STEPS, T, chain_inputs
    from streamingt2v_b200 import arch
    from streamingt2v_b200.sampler import B200EulerEDMSampler
    from streamingt2v_b200.vae import B200VaeDecoder
    from streamingt2v_b200.wrapper import B200StreamingWrapper
    cfg, vcfg = arch.TINY, arch.VaeConfig()
    sd_u = arch.synth_state_dict(arch.unet_param_shapes(cfg), seed=SEED)
    sd_c = arch.synth_state_dict(arch.controlnet_param_shapes(cfg), seed=SEED + 1000)
    sd_v = arch.synth_state_dict(arch.vae_decoder_param_shapes(vcfg), seed=SEED + 2000)
    model = B200StreamingWrapper(cfg, sd_u, sd_c, cuda_dev)
    dec = B200VaeDecoder(vcfg, sd_v, cuda_dev)
    sampler = B200EulerEDMSampler(num_steps=STEPS, num_frames=T)
    noise, cond, uc, extra = chain_inputs(cfg)
    to = lambda d: {k: (v.to(cuda_dev) if torch.is_tensor(v) else v) for k, v in d.items()}  # noqa: E731
    return model, dec, sampler, noise.to(cuda_dev), to(cond), to(uc), to(extra), SCALE_FACTOR, T


def test_thirty_step_chain_vs_reference_golden(cuda_dev):
    g = np.load(GOLDEN)
    z_ref = torch.from_numpy(g["latent"])
    x_ref = torch.from_numpy(g["frames"].astype(np.float32))
    model, dec, sampler, noise, cond, uc, extra, sf, T = _build(cuda_dev)
    z = sampler(model, noise, cond, uc, **extra)
    x = dec.decode(z / sf, timesteps=T).clamp(-1.0, 1.0)
    torch.cuda.synchronize()
    z, x = z.float().cpu(), x.float().cpu()
    assert torch.isfinite(z).all() and torch.isfinite(x).all()
    rel = ((z - z_ref).norm() / z_ref.norm()).item()
    mse = ((x - x_ref) ** 2).mean().item()
    sz, sx = (float(v) for v in g["reference_bf16_autocast_vs_fp32"])
    print(f"[chain] 30 Euler steps + decode vs REFERENCE chain golden: latent rel-L2 {rel:.4e} (tol {LATENT_TOL}), "
          f"pixel MSE {mse:.4e} (tol {PIXEL_MSE_TOL}); the reference's own bf16-autocast run vs its fp32 run: "
          f"latent rel-L2 {sz:.4e}, pixel MSE {sx:.4e}")
    assert rel <= LATENT_TOL, rel
    assert mse <= PIXEL_MSE_TOL, mse
    # the chain is deterministic run to run (graph replay included)
    z2 = sampler(model, noise, cond, uc, **extra).float().cpu()
    assert torch.equal(z, z2)
