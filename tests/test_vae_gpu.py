"""GPU parity of the temporal VAE decoder (B200VaeDecoder.decode == first_stage_model.decode) against the golden
vectors produced by the UNMODIFIED reference VideoDecoder (tests/golden/vae_*.npz, oracle/make_golden_vae.py).
Tolerance (bf16 activations, fp32 accumulate, vs the reference's fp32 result): pixel MSE <= 1e-3 on the decoder output
range, relative L2 <= 3e-2 overall and per block against the oracle."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


@pytest.mark.parametrize("name", ["vae_t4_8x16", "vae_t3_16x8"])
def test_vae_decode_vs_reference_golden(cuda_dev, name):
    from oracle import vae_decoder_oracle as vorc
    from oracle.make_golden_vae import make_latent
    from streamingt2v_b200 import arch
    from streamingt2v_b200.vae import B200VaeDecoder
    g = np.load(os.path.join(GOLDEN, f"{name}.npz"))
    T, h, w, seed = (int(v) for v in g["meta"])
    cfg = arch.VaeConfig()
    sd = arch.synth_state_dict(arch.vae_decoder_param_shapes(cfg), seed=seed)
    z = make_latent(T, h, w, seed)
    dec = B200VaeDecoder(cfg, sd, cuda_dev)
    dec.debug_taps = {}
    out = dec.decode(z.to(cuda_dev), timesteps=T)
    torch.cuda.synchronize()
    out = out.cpu()
    ref = torch.from_numpy(g["out"])
    r, mse = _rel(out, ref), ((out - ref) ** 2).mean().item()
    print(f"[{name}] vs REFERENCE golden: rel_l2={r:.4e} pixel_mse={mse:.3e} max_abs={(out - ref).abs().max():.3e}")
    assert torch.isfinite(out).all() and out.shape == ref.shape
    taps = {}
    with torch.no_grad():
        vorc.decode(sd, cfg, z, T, taps=taps)
    for tname, (tt, n, hh, ww) in dec.debug_taps.items():
        mine = tt.float().cpu().reshape(n, hh, ww, -1).permute(0, 3, 1, 2)
        rr = _rel(mine, taps[tname])
        print(f"   {tname:20s} rel_l2={rr:.4e}")
        assert rr < 3e-2, (tname, rr)
    assert r < 3e-2 and mse < 1e-3
    assert torch.equal(out, dec.decode(z.to(cuda_dev), timesteps=T).cpu()), "decode is not deterministic"


def test_softmax_rows_and_transpose(cuda_dev):
    from streamingt2v_b200 import ops
    s = torch.randn(300, 1000, device=cuda_dev) * 3
    p = ops.softmax_rows(s)
    x = torch.randn(77, 200, device=cuda_dev).to(torch.bfloat16)
    xt = ops.transpose(x)
    torch.cuda.synchronize()
    ref = F.softmax(s.double(), dim=-1)
    # per element: bf16 rounding (2^-8 p) plus __expf and the fp32 row sum (2^-16 p at this logit spread)
    assert ((p.double() - ref).abs() <= (2 ** -8 + 2 ** -16) * ref).all()
    assert torch.equal(xt, x.t().contiguous())


def test_attention_single_head(cuda_dev):
    from streamingt2v_b200 import ops
    n, s, c = 2, 160, 512
    g = torch.Generator().manual_seed(0)
    q, k, v = ((torch.randn(n * s, c, generator=g) * 1.2).to(cuda_dev).to(torch.bfloat16) for _ in range(3))
    o = ops.attention_single_head(q, k, v, n, s)
    torch.cuda.synchronize()
    ref = F.scaled_dot_product_attention(q.float().reshape(n, 1, s, c), k.float().reshape(n, 1, s, c),
                                         v.float().reshape(n, 1, s, c)).reshape(n * s, c)
    err = (o.float() - ref).abs()
    assert (err <= 2e-2 + 2 ** -6 * ref.abs()).all(), err.max().item()


@pytest.mark.parametrize("name", ["vae_enc_2_64x96", "vae_enc_1_128x64"])
def test_vae_encode_vs_reference_golden(cuda_dev, name):
    """B200VaeEncoder.encode == mode(quant_conv(Encoder(x))) of the unmodified reference (conditioner's SD-VAE encoder,
    SURVEY.md section 8 row f1).  Same tolerance as the decoder: relative L2 <= 3e-2 overall and per block."""
    from oracle import vae_encoder_oracle as eorc
    from oracle.make_golden_vae_enc import make_image
    from streamingt2v_b200 import arch
    from streamingt2v_b200.vae import B200VaeEncoder
    g = np.load(os.path.join(GOLDEN, f"{name}.npz"))
    n, H, W, seed = (int(v) for v in g["meta"])
    cfg = arch.VaeConfig()
    sd = arch.synth_state_dict(arch.vae_encoder_param_shapes(cfg), seed=seed)
    x = make_image(n, H, W, seed)
    enc = B200VaeEncoder(cfg, sd, cuda_dev)
    enc.debug_taps = {}
    out = enc.encode(x.to(cuda_dev))
    torch.cuda.synchronize()
    out = out.cpu()
    ref = torch.from_numpy(g["out"])
    r = _rel(out, ref)
    print(f"[{name}] vs REFERENCE golden: rel_l2={r:.4e} max_abs={(out - ref).abs().max():.3e}")
    assert torch.isfinite(out).all() and out.shape == ref.shape
    taps = {}
    with torch.no_grad():
        eorc.encode(sd, cfg, x, taps=taps)
    for tname, (tt, nn_, hh, ww) in enc.debug_taps.items():
        mine = tt.float().cpu().reshape(nn_, hh, ww, -1).permute(0, 3, 1, 2)
        rr = _rel(mine, taps[tname])
        assert rr < 3e-2, (tname, rr)
    assert r < 3e-2
    assert torch.equal(out, enc.encode(x.to(cuda_dev)).cpu()), "encode is not deterministic"
