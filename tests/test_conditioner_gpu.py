"""GPU: the SVD conditioner on the project's kernels — CLIP preprocessing, head-dim-80 FlashAttention, the ViT-H/14
image tower, the assembled (c, uc) against the reference's GeneralConditioner (tests/golden/cond_full_576x1024.npz,
oracle/make_golden_conditioner.py), and one stage run with the real conditioner.

Bounds:
  preprocess     |out - ref| <= 2^-8 |ref| + 1e-5 per element (bf16 rounding of an fp32 result; the fp32 restatement
                 is oracle/clip_image_oracle.py); padding columns 588..591 exactly 0.
  attention d80  |out - ref| <= 2^-8 |ref| + 2^-7 (softmax(Q K^T) |V|) against float64 (as tests/test_kernel_edges_gpu.py)
                 and relative L2 <= 1e-2; outputs inside NaN guard bands; two runs bitwise equal.
  tower / conditioner  relative L2 <= 3e-2 (bf16 activations through 32 pre-LN blocks, fp32 accumulation)."""
import math
import os

import numpy as np
import pytest
import torch

from test_kernel_edges_gpu import Guarded

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm()).item()


def _frame(n, H, W, seed):
    rng = np.random.default_rng([seed, 77])                  # oracle/make_golden_conditioner.py make_frame
    return torch.from_numpy(rng.uniform(-1, 1, size=(n, 3, H, W)).astype(np.float32))


# ---------------------------------------------------------------------------------------------------------------------
# preprocessing
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2])
@pytest.mark.parametrize("hw", [(576, 1024), (224, 224), (128, 300), (448, 320)], ids=lambda v: f"{v[0]}x{v[1]}")
def test_clip_preprocess(cuda_dev, hw, n):
    from oracle import clip_image_oracle as co
    from streamingt2v_b200 import ops
    from streamingt2v_b200.conditioner import antialias_taps
    H, W = hw
    x = (torch.rand(n, 3, H, W, generator=torch.Generator().manual_seed(H * W + n)) * 2 - 1).to(cuda_dev)
    ty, tx = antialias_taps(H, W)
    out = ops.clip_preprocess(x, ty, tx)
    ref = co.patch_rows(co.preprocess(x)).double()
    assert out.shape == (n * 256, 592)
    got = out.double()
    assert torch.equal(got[:, 588:], torch.zeros_like(got[:, 588:]))
    err = (got[:, :588] - ref).abs()
    bound = 2.0 ** -8 * ref.abs() + 1e-5
    assert bool((err <= bound).all()), f"max err/bound {(err / bound).max().item():.3f}"
    if (H, W) == (224, 224):                                   # no blur, identity resize
        ref_id = co.patch_rows(co.normalize((x + 1) / 2)).double()
        assert torch.equal(got[:, :588], ref_id.to(torch.bfloat16).double())


# ---------------------------------------------------------------------------------------------------------------------
# head-dim-80 FlashAttention
# ---------------------------------------------------------------------------------------------------------------------
def _attn64(qkv, n, s, heads):
    q, k, v = (t.double().reshape(n, s, heads, 80).permute(0, 2, 1, 3) for t in qkv.chunk(3, dim=1))
    p = torch.softmax((q @ k.transpose(-1, -2)) / math.sqrt(80), dim=-1)
    o = (p @ v).permute(0, 2, 1, 3).reshape(n * s, heads * 80)
    oa = (p @ v.abs()).permute(0, 2, 1, 3).reshape(n * s, heads * 80)
    return o, oa


@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("heads", [2, 16])
@pytest.mark.parametrize("S", [1, 17, 128, 129, 256, 257])
def test_flash_attn_d80(cuda_dev, S, heads, n):
    from streamingt2v_b200 import ops
    C = heads * 80
    g = torch.Generator(device=cuda_dev).manual_seed(S * 100 + heads * 10 + n)
    qkv = Guarded((n * S, 3 * C), torch.bfloat16, cuda_dev, pad=16)
    qkv.fill((torch.randn(n * S, 3 * C, generator=g, device=cuda_dev) * 1.5).to(torch.bfloat16))
    out = Guarded((n * S, C), torch.bfloat16, cuda_dev, pad=8).snapshot()
    ops.flash_attn_d80(qkv.view, n, S, heads, out=out.view)
    torch.cuda.synchronize()
    out.check("flash_attn_d80")
    ref, ref_abs = _attn64(qkv.view, n, S, heads)
    got = out.view.double()
    err = (got - ref).abs()
    bound = 2.0 ** -8 * ref.abs() + 2.0 ** -7 * ref_abs
    assert bool((err <= bound).all()), f"max err/bound {(err / bound).max().item():.3f}"
    assert _rel(got, ref) <= 1e-2
    again = ops.flash_attn_d80(qkv.view, n, S, heads)
    assert torch.equal(again, out.view)


@pytest.mark.parametrize("S", [1, 128, 129, 257])
def test_flash_attn_d80_key_coverage_probe(cuda_dev, S):
    """Q = 0: every key gets weight 1/S.  V holds key-block indicators in head columns b and 64 + b (the two TMA boxes
    of a row) and the head index in column 20, so each output column is (keys in that block) / S exactly; the one-key
    ragged block of S = 257 must count 1, a mask off by one or an unmasked zero-filled key changes the sum."""
    from streamingt2v_b200 import ops
    n, heads = 2, 3
    C = heads * 80
    qkv = torch.zeros(n * S, 3 * C, dtype=torch.bfloat16, device=cuda_dev)
    j = torch.arange(S, device=cuda_dev)
    for f in range(n):
        for h in range(heads):
            v = qkv[f * S:(f + 1) * S, 2 * C + h * 80:2 * C + (h + 1) * 80]
            v[j, j // 128] = 1.0
            v[j, 64 + j // 128] = 1.0
            v[:, 20] = float(h + 1)
            qkv[f * S:(f + 1) * S, C + h * 80:C + (h + 1) * 80] = (j % 7).float()[:, None].to(torch.bfloat16)
    out = ops.flash_attn_d80(qkv, n, S, heads)
    colsum = qkv[:, 2 * C:].float().view(n, S, C).sum(1)                                  # exact small integers
    expect = (colsum * (1.0 / torch.tensor(float(S), device=cuda_dev)))[:, None, :].expand(n, S, C)
    assert torch.equal(out.view(n, S, C), expect.to(torch.bfloat16))


# ---------------------------------------------------------------------------------------------------------------------
# tower and conditioner
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["clip_tiny_2_448x320", "clip_tiny_1_128x300"])
def test_clip_tower_tiny_taps(cuda_dev, case):
    from streamingt2v_b200 import arch
    from streamingt2v_b200.conditioner import B200ClipImageEncoder
    g = np.load(os.path.join(GOLDEN, case + ".npz"))
    n, H, W, seed, wseed = (int(v) for v in g["meta"])
    cfg = arch.CLIP_TINY
    enc = B200ClipImageEncoder(cfg, arch.synth_state_dict(arch.clip_visual_param_shapes(cfg), wseed), cuda_dev)
    enc.debug_taps = {}
    out = enc.encode(_frame(n, H, W, seed).to(cuda_dev))
    torch.cuda.synchronize()
    for k, v in enc.debug_taps.items():
        ref = torch.from_numpy(g["tap_" + k].astype(np.float32))
        got = v.float().cpu().reshape(ref.shape)
        assert _rel(got, ref) <= 3e-2, (k, _rel(got, ref))
    assert out.dtype == torch.float32 and out.shape == (n, 1024)
    assert _rel(out, torch.from_numpy(g["out"])) <= 3e-2


@pytest.fixture(scope="module")
def full_conditioner(cuda_dev):
    from streamingt2v_b200 import arch
    from streamingt2v_b200.conditioner import B200ClipImageEncoder, B200SVDConditioner
    from streamingt2v_b200.vae import B200VaeEncoder
    g = np.load(os.path.join(GOLDEN, "cond_full_576x1024.npz"))
    H, W, T, seed, clip_seed, vae_seed = (int(v) for v in g["meta"])
    ccfg, vcfg = arch.ClipVisionConfig(), arch.VaeConfig()
    clip = B200ClipImageEncoder(ccfg, arch.synth_state_dict(arch.clip_visual_param_shapes(ccfg), clip_seed), cuda_dev)
    vae = B200VaeEncoder(vcfg, arch.synth_state_dict(arch.vae_encoder_param_shapes(vcfg), vae_seed), cuda_dev)
    frame = _frame(1, H, W, seed)[0]
    assert abs(frame.double().sum().item() - float(g["frame_sum"][0])) < 1e-6
    return clip, vae, frame, g


def test_clip_tower_full(full_conditioner, cuda_dev):
    clip, _, frame, g = full_conditioner
    out = clip.encode(frame[None].to(cuda_dev))
    r = _rel(out, torch.from_numpy(g["crossattn"][:, 0]))
    assert r <= 3e-2, r


def test_conditioner_matches_reference(full_conditioner, cuda_dev):
    from streamingt2v_b200.conditioner import B200SVDConditioner
    clip, vae, frame, g = full_conditioner
    T, seed = int(g["meta"][2]), int(g["meta"][3])
    runs = []
    for _ in range(2):
        cond = B200SVDConditioner(clip, vae, generator=torch.Generator().manual_seed(seed))
        c, uc = cond(frame.to(cuda_dev), T)
        torch.cuda.synchronize()
        runs.append((c, uc))
    c, uc = runs[0]
    assert c["crossattn"].shape == (1, 1, 1024) and c["concat"].shape == g["concat"].shape
    assert c["vector"].shape == (T, 768)
    for k in ("crossattn", "concat", "vector"):
        assert c[k].dtype == torch.float32 and c[k].device.type == "cuda"
    assert _rel(c["crossattn"], torch.from_numpy(g["crossattn"])) <= 3e-2
    assert _rel(c["concat"], torch.from_numpy(g["concat"])) <= 3e-2
    assert float((c["vector"].cpu() - torch.from_numpy(g["vector"])).abs().max()) <= 2.0 ** -8
    assert not uc["crossattn"].any() and not uc["concat"].any()
    assert torch.equal(uc["vector"], c["vector"])
    c2, uc2 = runs[1]
    for k in ("crossattn", "concat", "vector"):
        assert torch.equal(c[k], c2[k]) and torch.equal(uc[k], uc2[k])


def test_stage_runs_with_real_conditioner(cuda_dev):
    """test_stage.py::test_stage_runs_on_real_components with `B200SVDConditioner` (CLIP_TINY tower, real VAE encoder)
    in place of the random conditioning callable: shapes, ranges, finiteness, determinism."""
    import dataclasses

    from streamingt2v_b200 import arch
    from streamingt2v_b200.conditioner import B200ClipImageEncoder, B200SVDConditioner
    from streamingt2v_b200.sampler import B200EulerEDMSampler
    from streamingt2v_b200.stage import B200StreamingSVDStage
    from streamingt2v_b200.vae import B200VaeDecoder, B200VaeEncoder
    from streamingt2v_b200.wrapper import B200StreamingWrapper
    Tg, ncond = 8, 3
    cfg = dataclasses.replace(arch.TINY, num_frame_conditioning=ncond)
    wrapper = B200StreamingWrapper(cfg, arch.synth_state_dict(arch.unet_param_shapes(cfg), 1),
                                   arch.synth_state_dict(arch.controlnet_param_shapes(cfg), 2), cuda_dev)
    vcfg = arch.VaeConfig()
    dec = B200VaeDecoder(vcfg, arch.synth_state_dict(arch.vae_decoder_param_shapes(vcfg), 3), cuda_dev)
    enc = B200VaeEncoder(vcfg, arch.synth_state_dict(arch.vae_encoder_param_shapes(vcfg), 4), cuda_dev)
    clip = B200ClipImageEncoder(arch.CLIP_TINY, arch.synth_state_dict(arch.clip_visual_param_shapes(arch.CLIP_TINY), 5),
                                cuda_dev)
    conditioner = B200SVDConditioner(clip, enc)
    sampler = B200EulerEDMSampler(num_steps=2, num_frames=Tg)
    stage = B200StreamingSVDStage(wrapper, sampler, dec, conditioner, num_conditional_frames=ncond, device=cuda_dev)
    first = torch.rand(Tg, 3, 128, 128, generator=torch.Generator().manual_seed(1)) * 2 - 1
    outs = []
    for _ in range(2):
        conditioner.generator = torch.Generator().manual_seed(6)
        video = stage.autoregressive_generation(first.to(cuda_dev), 1, generator=torch.Generator().manual_seed(9))
        torch.cuda.synchronize()
        outs.append(video.cpu())
    video = outs[0]
    assert video.shape == (Tg + (Tg - ncond), 3, 128, 128)
    assert torch.isfinite(video).all() and float(video.min()) >= 0.0 and float(video.max()) <= 255.0
    assert torch.equal(outs[0], outs[1])
    assert torch.allclose(video[:Tg], (first + 1) * 127.5, atol=1e-3)
    assert float(video[Tg:].std()) > 0.0
