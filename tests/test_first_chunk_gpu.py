"""GPU: the first chunk of an image-to-video request on the kernels.

- b200svd_frames_quantize is bit-exact against the numpy / PIL / ToTensor round trip on edge and random values.
- The tiny pipeline matches the golden of oracle/make_golden_first_chunk.py before the 8-bit round trip
  (rel-L2 <= 3e-2, the tolerance of test_denoiser_gpu.py).
- At full size (576 x 1024, 25 frames, synthetic weights, 2 steps) the conditioning and the decoded chunk match the
  fp32 oracle run on the GPU.
- `from_diffusers` builds from a pipeline-shaped object (renamed synthetic state dicts, transformers' CLIP model).
- One `image_to_video` call with one autoregressive generation returns finite frames of the right shape."""
import dataclasses
import os
import types

import numpy as np
import pytest
import torch

from test_first_chunk import GOLDEN, _diffusers_vae_sd, edge_frames, quantize_like_reference

pytestmark = pytest.mark.gpu
REL_TOL = 3e-2


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm()).item()


def test_frames_quantize_bit_exact(cuda_dev):
    from streamingt2v_b200 import ops
    x = edge_frames()
    assert torch.equal(ops.frames_quantize(x.to(cuda_dev)).cpu(), quantize_like_reference(x))
    y = torch.randn(25, 3, 72, 128, generator=torch.Generator().manual_seed(4)) * 0.8
    out = ops.frames_quantize(y.to(cuda_dev)).cpu()
    assert torch.equal(out, quantize_like_reference(y))
    yd = y.to(cuda_dev)
    ops.frames_quantize(yd, out=yd)                                   # in place
    assert torch.equal(yd.cpu(), out)


def _pipeline(cuda_dev, unet_cfg, sd_u, clip_cfg, sd_c, vcfg, sd_e, sd_d):
    from streamingt2v_b200.conditioner import B200ClipImageEncoder, B200SVDConditioner
    from streamingt2v_b200.first_chunk import B200SVDImageToVideo
    from streamingt2v_b200.vae import B200VaeDecoder, B200VaeEncoder
    from streamingt2v_b200.wrapper import B200StreamingWrapper
    cond = B200SVDConditioner(B200ClipImageEncoder(clip_cfg, sd_c, cuda_dev), B200VaeEncoder(vcfg, sd_e, cuda_dev),
                              noise="gaussian")
    return B200SVDImageToVideo(B200StreamingWrapper(unet_cfg, sd_u, None, cuda_dev), cond,
                               B200VaeDecoder(vcfg, sd_d, cuda_dev), device=cuda_dev)


def test_tiny_pipeline_matches_golden(cuda_dev):
    from oracle import make_golden_first_chunk as mg
    from streamingt2v_b200 import arch
    g = np.load(GOLDEN)
    T, H, W, steps, seed = (int(v) for v in g["meta"][:5])
    sd_u, sd_c, sd_e, sd_d = mg.weights()
    p = _pipeline(cuda_dev, arch.TINY, sd_u, arch.CLIP_TINY, sd_c, arch.VaeConfig(), sd_e, sd_d)
    image = mg.make_image(seed)
    kw = dict(num_frames=T, num_inference_steps=steps, min_guidance_scale=1.0, max_guidance_scale=3.0, fps=7,
              motion_bucket_id=127, noise_aug_strength=0.02)
    c, _ = p.conditioner.condition(image.to(cuda_dev) * 2.0 - 1.0, T, fps_id=6, motion_bucket_id=127, cond_aug=0.02,
                                   generator=torch.Generator().manual_seed(seed))
    z = p.sample(image, generator=torch.Generator().manual_seed(seed), **kw)
    frames = p.decode(z, 8)
    out = p(image, generator=torch.Generator().manual_seed(seed), **kw)
    torch.cuda.synchronize()
    for k in ("crossattn", "concat"):
        r = _rel(c[k].cpu(), torch.from_numpy(g[k]))
        print(f"{k}: rel_l2 {r:.3e}")
        assert r < REL_TOL, k
    rz = _rel(z.cpu(), torch.from_numpy(g["latents"]))
    rf = _rel(frames.cpu(), torch.from_numpy(g["frames"].astype(np.float32)))
    print(f"latents rel_l2 {rz:.3e}; frames rel_l2 {rf:.3e}")
    assert rz < REL_TOL and rf < REL_TOL
    assert torch.equal(out.cpu(), quantize_like_reference(frames.cpu()))   # __call__ = decode + frames_quantize


def test_full_size_conditioning_and_decode_match_oracle(cuda_dev):
    """576 x 1024, 25 frames, full-size CLIP / VAE / UNet with synthetic weights, 2 Karras steps: the conditioning and
    the decoded chunk (of the pipeline's own latents) against the fp32 oracle on the GPU."""
    from oracle import svd_pipeline_oracle as spo
    from streamingt2v_b200 import arch
    T, H, W = 25, 576, 1024
    ucfg, ccfg, vcfg = arch.UNetConfig(), arch.ClipVisionConfig(), arch.VaeConfig()
    sd_u = arch.synth_state_dict_device(arch.plain_unet_param_shapes(ucfg), cuda_dev, 1)
    sd_c = arch.synth_state_dict_device(arch.clip_visual_param_shapes(ccfg), cuda_dev, 2)
    sd_e = arch.synth_state_dict_device(arch.vae_encoder_param_shapes(vcfg), cuda_dev, 3)
    sd_d = arch.synth_state_dict_device(arch.vae_decoder_param_shapes(vcfg), cuda_dev, 4)
    p = _pipeline(cuda_dev, ucfg, sd_u, ccfg, sd_c, vcfg, sd_e, sd_d)
    image = torch.rand(3, H, W, generator=torch.Generator().manual_seed(6))
    seed = 8
    c, _ = p.conditioner.condition(image.to(cuda_dev) * 2.0 - 1.0, T, fps_id=6, motion_bucket_id=127, cond_aug=0.02,
                                   generator=torch.Generator().manual_seed(seed))
    z = p.sample(image, num_frames=T, num_inference_steps=2, min_guidance_scale=1.0, max_guidance_scale=3.0, fps=7,
                 motion_bucket_id=127, noise_aug_strength=0.02, generator=torch.Generator().manual_seed(seed))
    frames = p.decode(z, 8)
    torch.cuda.synchronize()
    assert z.shape == (T, 4, H // 8, W // 8) and torch.isfinite(z).all()
    noise = torch.randn((1, 3, H, W), generator=torch.Generator().manual_seed(seed)).to(cuda_dev)
    with torch.no_grad():
        ca, co_, vec = spo.conditioning(sd_c, ccfg, sd_e, vcfg, image.to(cuda_dev), noise, T)
    for name, mine, ref in (("crossattn", c["crossattn"], ca), ("concat", c["concat"], co_)):
        r = _rel(mine, ref)
        print(f"{name}: rel_l2 {r:.3e}")
        assert r < REL_TOL, name
    assert (c["vector"] - vec).abs().max().item() <= 2.0 ** -8
    # decode of the pipeline's latents in groups of 8: compare group by group (the fp32 oracle holds one group at a time)
    zs = 1.0 / 0.18215 * z
    worst = 0.0
    for i in range(0, T, 8):
        with torch.no_grad():
            ref = spo.vdo.decode(sd_d, vcfg, zs[i:i + 8], len(zs[i:i + 8]))
        worst = max(worst, _rel(frames[i:i + 8], ref))
        del ref
    print(f"decoded chunk: worst group rel_l2 {worst:.3e}")
    assert worst < REL_TOL


def _sd_to_module(sd, config):
    return types.SimpleNamespace(state_dict=lambda: sd, config=config)


def test_from_diffusers_builds_from_a_pipeline_object(cuda_dev):
    """A pipeline-shaped object with the diffusers / transformers state dicts (renamed synthetic weights) and a real
    transformers CLIPVisionModelWithProjection builds the same pipeline as the SGM-named constructor path."""
    pytest.importorskip("transformers")
    from oracle import make_golden_conditioner as mgc
    from oracle import make_golden_first_chunk as mg
    from streamingt2v_b200 import arch
    from streamingt2v_b200.first_chunk import B200SVDImageToVideo
    sd_u, sd_c, sd_e, sd_d = mg.weights()
    vcfg = arch.VaeConfig()
    m = arch.sgm_to_diffusers_svd_keys(arch.TINY)
    unet_cfg = types.SimpleNamespace(block_out_channels=(320, 320, 640, 640), num_attention_heads=(5, 5, 10, 10),
                                     layers_per_block=2, in_channels=8, out_channels=4, cross_attention_dim=1024,
                                     projection_class_embeddings_input_dim=768,
                                     down_block_types=("CrossAttnDownBlockSpatioTemporal",) * 3 + ("DownBlockSpatioTemporal",))
    vae_cfg = types.SimpleNamespace(block_out_channels=(128, 256, 512, 512), layers_per_block=2, latent_channels=4,
                                    out_channels=3, scaling_factor=0.18215)
    pipe = types.SimpleNamespace(
        unet=_sd_to_module({m[k]: v for k, v in sd_u.items()}, unet_cfg),
        vae=_sd_to_module(_diffusers_vae_sd(vcfg, sd_e, sd_d), vae_cfg),
        image_encoder=mgc.hf_tower(arch.CLIP_TINY, sd_c),
        scheduler=types.SimpleNamespace(config=types.SimpleNamespace(
            use_karras_sigmas=True, prediction_type="v_prediction", timestep_type="continuous", sigma_min=0.002,
            sigma_max=700.0)))
    p = B200SVDImageToVideo.from_diffusers(pipe, cuda_dev)
    assert p.unet.cfg == arch.TINY and p.conditioner.noise == "gaussian" and p.conditioner.clip.cfg == arch.CLIP_TINY
    g = np.load(GOLDEN)
    T, H, W, steps, seed = (int(v) for v in g["meta"][:5])
    z = p.sample(mg.make_image(seed), num_frames=T, num_inference_steps=steps, min_guidance_scale=1.0,
                 max_guidance_scale=3.0, fps=7, motion_bucket_id=127, noise_aug_strength=0.02,
                 generator=torch.Generator().manual_seed(seed))
    rf = _rel(p.decode(z, 8).cpu(), torch.from_numpy(g["frames"].astype(np.float32)))
    print(f"from_diffusers frames rel_l2 {rf:.3e}")
    assert rf < REL_TOL


def test_image_to_video_on_real_components(cuda_dev):
    """One image_to_video call (576 x 1024 image; reduced networks, 2 steps, 8 frames) with one autoregressive
    generation: finite frames in [0, 255] of the right shape."""
    from streamingt2v_b200 import arch
    from streamingt2v_b200.sampler import B200EulerEDMSampler
    from streamingt2v_b200.stage import B200StreamingSVDStage
    from streamingt2v_b200.vae import B200VaeDecoder
    from streamingt2v_b200.wrapper import B200StreamingWrapper
    Tg, ncond = 8, 3
    vcfg = arch.VaeConfig()
    sd_e = arch.synth_state_dict_device(arch.vae_encoder_param_shapes(vcfg), cuda_dev, 13)
    sd_d = arch.synth_state_dict_device(arch.vae_decoder_param_shapes(vcfg), cuda_dev, 14)
    first = _pipeline(cuda_dev, arch.TINY, arch.synth_state_dict_device(arch.plain_unet_param_shapes(arch.TINY), cuda_dev, 11),
                      arch.CLIP_TINY, arch.synth_state_dict_device(arch.clip_visual_param_shapes(arch.CLIP_TINY), cuda_dev, 12),
                      vcfg, sd_e, sd_d)
    cfg = dataclasses.replace(arch.TINY, num_frame_conditioning=ncond)
    wrapper = B200StreamingWrapper(cfg, arch.synth_state_dict_device(arch.unet_param_shapes(cfg), cuda_dev, 15),
                                   arch.synth_state_dict_device(arch.controlnet_param_shapes(cfg), cuda_dev, 16), cuda_dev)
    stage = B200StreamingSVDStage(wrapper, B200EulerEDMSampler(num_steps=2, num_frames=Tg), first.vae_decoder,
                                  first.conditioner, num_conditional_frames=ncond, device=cuda_dev)

    def first_chunk(image, generator=None):
        return first(image, num_frames=Tg, num_inference_steps=2, generator=generator)

    img = np.random.default_rng(3).integers(0, 256, size=(360, 640, 3), dtype=np.uint8)
    video = stage.image_to_video(img, 1, first_chunk, generator=torch.Generator().manual_seed(2))
    torch.cuda.synchronize()
    assert video.shape == (Tg + Tg - ncond, 3, 576, 1024)
    assert torch.isfinite(video).all() and float(video.min()) >= 0.0 and float(video.max()) <= 255.0
    assert torch.allclose(video[:Tg], video[:Tg].round(), atol=2e-3)    # the first chunk sits on the 8-bit grid
