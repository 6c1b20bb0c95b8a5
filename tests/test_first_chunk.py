"""CPU: the first chunk of an image-to-video request (streamingt2v_b200/first_chunk.py) and the stage's
`image_to_video`.

- The transformers CLIP and diffusers VAE weight maps of arch.py: bijections onto the grammars, shapes kept, the
  inverse of the oracle's open_clip -> transformers map, transformers' own tower on the renamed weights.
- diffusers' AlphaBlender (switch_spatial_to_temporal_mix) and SGM's VideoResBlock blend agree on the same mix_factor.
- Gaussian conditioning noise and the pipeline's draw order (image noise, then latents).
- The 8-bit round trip's arithmetic against numpy + PIL + ToTensor on edge values.
- The driver, with the CPU fakes of tests/fake_ops.py for the kernels, against the golden of
  oracle/make_golden_first_chunk.py.
- `image_to_video` resizes to 576 rows on the host and hands the first chunk to the stage."""
import os
import types

import numpy as np
import pytest
import torch

import fake_clip_ops
import fake_ops

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "first_chunk_tiny_t8_16x16.npz")


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm()).item()


def _hf_clip(cfg, sd):
    pytest.importorskip("transformers")
    from oracle import make_golden_conditioner as mgc
    return mgc.hf_tower(cfg, sd)


def _diffusers_vae_sd(vcfg, sd_e, sd_d):
    from streamingt2v_b200 import arch
    out = {}
    for m, sd in ((arch.sgm_to_diffusers_vae_encoder_keys(vcfg), sd_e), (arch.sgm_to_diffusers_vae_decoder_keys(vcfg), sd_d)):
        for k, v in sd.items():
            out[m[k]] = v.reshape(v.shape[:2]) if ".attentions." in m[k] and v.dim() == 4 else v
    return out


# ---- weight maps ---------------------------------------------------------------------------------------------------
def test_clip_map_inverts_the_oracle_map_and_runs_in_transformers():
    from oracle import clip_image_oracle as co
    from streamingt2v_b200 import arch
    cfg = arch.CLIP_TINY
    sd = arch.synth_state_dict_fast(arch.clip_visual_param_shapes(cfg), 81)
    hf = _hf_clip(cfg, sd)
    hsd = hf.state_dict()
    back = arch.from_hf_clip_vision_state_dict(hsd, hf.config)
    assert set(back) == set(sd) and all(torch.equal(back[k], sd[k]) for k in sd)       # composes to the identity
    assert arch.clip_vision_config_from_hf(hf.config) == cfg
    img = co.preprocess(torch.rand(1, 3, 96, 160, generator=torch.Generator().manual_seed(2)) * 2 - 1)
    with torch.no_grad():
        ref = hf(pixel_values=img).image_embeds
        out = co.visual(back, cfg, img)
    assert (out - ref).abs().max().item() <= 1e-4 * ref.abs().max().item()
    # every transformers tensor is used exactly once: a stray key is an error, position_ids is not
    with pytest.raises(KeyError):
        arch.from_hf_clip_vision_state_dict({**hsd, "vision_model.extra.weight": torch.zeros(1)}, hf.config)
    arch.from_hf_clip_vision_state_dict({**hsd, "vision_model.embeddings.position_ids": torch.arange(257)[None]},
                                        hf.config)


def test_clip_map_rejects_other_activations():
    from streamingt2v_b200 import arch
    hcfg = types.SimpleNamespace(hidden_act="quick_gelu", image_size=224, patch_size=14, hidden_size=160,
                                 num_hidden_layers=2, num_attention_heads=2, intermediate_size=640, projection_dim=1024,
                                 layer_norm_eps=1e-5)
    with pytest.raises(ValueError, match="gelu"):
        arch.clip_vision_config_from_hf(hcfg)
    with pytest.raises(ValueError, match="gelu"):
        arch.from_hf_clip_vision_state_dict({}, hcfg)


@pytest.mark.parametrize("vcfg", [None, (64, (1, 2), 1)])
def test_vae_maps_are_bijections_that_keep_shapes(vcfg):
    from streamingt2v_b200 import arch
    cfg = arch.VaeConfig() if vcfg is None else arch.VaeConfig(ch=vcfg[0], ch_mult=vcfg[1], num_res_blocks=vcfg[2])
    enc, dec = arch.sgm_to_diffusers_vae_encoder_keys(cfg), arch.sgm_to_diffusers_vae_decoder_keys(cfg)
    assert set(enc) == set(arch.vae_encoder_param_shapes(cfg)) and set(dec) == set(arch.vae_decoder_param_shapes(cfg))
    assert len(set(enc.values())) == len(enc) and len(set(dec.values())) == len(dec)
    assert not set(enc.values()) & set(dec.values())
    assert all(v.startswith("encoder.") or v.startswith("quant_conv.") for v in enc.values())
    assert all(v.startswith("decoder.") for v in dec.values())
    n = len(cfg.ch_mult)
    assert dec[f"up.{n - 1}.block.0.conv1.weight"] == "decoder.up_blocks.0.resnets.0.spatial_res_block.conv1.weight"
    assert dec["up.0.block.0.mix_factor"] == f"decoder.up_blocks.{n - 1}.resnets.0.time_mixer.mix_factor"
    assert dec["conv_out.time_mix_conv.weight"] == "decoder.time_conv_out.weight"
    assert dec["norm_out.weight"] == "decoder.conv_norm_out.weight"
    assert dec["mid.attn_1.proj_out.weight"] == "decoder.mid_block.attentions.0.to_out.0.weight"
    assert enc["down.0.downsample.conv.weight"] == "encoder.down_blocks.0.downsamplers.0.conv.weight"
    assert enc["quant_conv.weight"] == "quant_conv.weight"
    # round trip: renamed synthetic weights come back unchanged, every shape kept (attention: reshape only)
    sd_e = {k: torch.full(s, float(i % 5)) for i, (k, s) in enumerate(sorted(arch.vae_encoder_param_shapes(cfg).items()))}
    sd_d = {k: torch.full(s, float(i % 7)) for i, (k, s) in enumerate(sorted(arch.vae_decoder_param_shapes(cfg).items()))}
    sd = _diffusers_vae_sd(cfg, sd_e, sd_d)
    assert sd["encoder.mid_block.attentions.0.to_q.weight"].dim() == 2
    e2, d2 = arch.from_diffusers_svd_vae_state_dict(sd, cfg)
    assert all(torch.equal(e2[k], sd_e[k]) for k in sd_e) and all(torch.equal(d2[k], sd_d[k]) for k in sd_d)
    with pytest.raises(KeyError):
        arch.from_diffusers_svd_vae_state_dict({k: v for k, v in sd.items() if "time_conv_out" not in k}, cfg)
    with pytest.raises(KeyError):
        arch.from_diffusers_svd_vae_state_dict({**sd, "post_quant_conv.weight": torch.zeros(4, 4, 1, 1)}, cfg)
    bad = dict(sd)
    bad["decoder.conv_in.weight"] = torch.zeros(1, 1, 3, 3)
    with pytest.raises(ValueError):
        arch.from_diffusers_svd_vae_state_dict(bad, cfg)


def test_alpha_blender_equals_sgm_blend_for_the_same_mix_factor():
    """diffusers AlphaBlender(merge_strategy="learned", switch_spatial_to_temporal_mix=True), restated from 0.30.2:
    alpha = 1 - sigmoid(m); out = alpha * x_spatial + (1 - alpha) * x_temporal.  SGM VideoResBlock
    (temporal_ae.py:62-81, oracle/vae_decoder_oracle.py): sigmoid(m) * x_temporal + (1 - sigmoid(m)) * x_spatial.
    The same mix_factor tensor gives the same output, so the VAE map copies it unchanged."""
    g = torch.Generator().manual_seed(0)
    xs, xt = torch.randn(2, 8, 3, 4, 4, generator=g), torch.randn(2, 8, 3, 4, 4, generator=g)
    for m in (torch.tensor([-2.5]), torch.tensor([0.0]), torch.tensor([1.3])):
        a = 1.0 - torch.sigmoid(m)
        diffusers = a * xs + (1.0 - a) * xt
        s = torch.sigmoid(m)
        sgm = s * xt + (1.0 - s) * xs
        assert torch.allclose(diffusers, sgm, atol=1e-6)


# ---- the 8-bit round trip ------------------------------------------------------------------------------------------
def quantize_like_kernel(x: torch.Tensor) -> torch.Tensor:
    """b200svd_frames_quantize's operation sequence in fp32 torch (one rounding per step, rint half to even)."""
    v = (x / 2.0 + 0.5).clamp(0.0, 1.0)
    v = torch.round(v * 255.0) / 255.0
    return v * 2.0 - 1.0


def quantize_like_reference(x: torch.Tensor) -> torch.Tensor:
    """postprocess_video(output_type="pil") (numpy) -> PIL images -> ToTensor() -> * 2.0 - 1, one frame at a time."""
    from PIL import Image
    v = (x / 2 + 0.5).clamp(0, 1)
    arr = v.permute(0, 2, 3, 1).float().numpy()
    u8 = (arr * 255).round().astype("uint8")
    frames = [Image.fromarray(f) for f in u8]
    t = torch.stack([torch.from_numpy(np.array(im, np.uint8)).permute(2, 0, 1).float().div(255) for im in frames])
    return t * 2.0 - 1


def edge_frames():
    """Exact halves of the 255 grid, their fp32 neighbours, +-1, out of range, zero and random values."""
    k = torch.arange(256, dtype=torch.float64)
    halves = ((k + 0.5) / 255.0 * 2.0 - 1.0).float()             # x whose v * 255 lands on or next to k + 0.5
    vals = torch.cat([halves, torch.nextafter(halves, torch.tensor(2.0)), torch.nextafter(halves, torch.tensor(-2.0)),
                      (k / 255.0 * 2.0 - 1.0).float(),
                      torch.tensor([-1.0, 1.0, 0.0, -0.0, -1.5, 1.5, 3.0, -7.0, 1e-8, -1e-8, 0.999999, -0.999999]),
                      torch.rand(2000, generator=torch.Generator().manual_seed(3)) * 2.4 - 1.2])
    n = vals.numel()
    pad = (-n) % (3 * 8 * 8)
    vals = torch.cat([vals, torch.zeros(pad)])
    return vals.reshape(-1, 3, 8, 8).contiguous()


def test_quantize_arithmetic_matches_numpy_pil_and_to_tensor():
    x = edge_frames()
    mine, ref = quantize_like_kernel(x), quantize_like_reference(x)
    assert torch.equal(mine, ref)
    # exact halves round to even: v * 255 == 0.5 -> 0, 1.5 -> 2 (numpy semantics)
    v = torch.tensor([0.5, 1.5, 2.5, 253.5]) / 255.0
    assert torch.equal(torch.round(v * 255.0), torch.from_numpy(np.round((v * 255).numpy())))
    grid = ((mine + 1) * 127.5).round()
    assert torch.allclose((mine + 1) * 127.5, grid, atol=1e-4) and mine.min() >= -1 and mine.max() <= 1


def test_fake_frames_quantize_is_the_kernel_arithmetic():
    """The fake used by the driver test below is the same arithmetic."""
    x = edge_frames()
    assert torch.equal(frames_quantize(x), quantize_like_reference(x))


def frames_quantize(x, out=None):
    return quantize_like_kernel(x)


# ---- conditioning ------------------------------------------------------------------------------------------------
class _StubClip:
    dev = torch.device("cpu")

    def encode(self, x):
        return torch.full((x.shape[0], 1024), float(x.mean()))


class _RecordingEncoder:
    def __init__(self):
        self.seen = []

    def encode(self, x):
        self.seen.append(x.clone())
        return torch.zeros(x.shape[0], 4, x.shape[2] // 8, x.shape[3] // 8)


@pytest.fixture()
def patched(monkeypatch):
    from streamingt2v_b200 import conditioner, first_chunk, sampler, vae
    for mod in (conditioner, vae, sampler):
        monkeypatch.setattr(mod, "ops", fake_clip_ops)
    monkeypatch.setattr(first_chunk, "ops", types.SimpleNamespace(frames_quantize=frames_quantize))
    return conditioner


def test_gaussian_noise_option(patched):
    enc = _RecordingEncoder()
    cond = patched.B200SVDConditioner(_StubClip(), enc, generator=torch.Generator().manual_seed(4), noise="gaussian")
    frame = torch.rand(3, 32, 48, generator=torch.Generator().manual_seed(1)) * 2 - 1
    cond(frame, 5)
    noise = torch.randn((1, 3, 32, 48), generator=torch.Generator().manual_seed(4))
    assert torch.equal(enc.seen[0], frame[None] + 0.02 * noise)
    assert patched.B200SVDConditioner(_StubClip(), enc).noise == "uniform"          # default unchanged
    with pytest.raises(ValueError):
        patched.B200SVDConditioner(_StubClip(), enc, noise="normal")


def test_pipeline_draw_order_and_conditioning_values(patched):
    """Image noise first, then latents, from one generator; vector = [fps - 1 | motion | aug]; CLIP sees the clean
    image, the VAE the noised one; latents start at sqrt(1 + sigma_max^2) * randn."""
    from streamingt2v_b200.first_chunk import B200SVDImageToVideo
    enc = _RecordingEncoder()
    cond = patched.B200SVDConditioner(_StubClip(), enc, noise="gaussian")
    seen = {}

    def net(x, t, c, **kw):
        seen.setdefault("x0", x.clone())
        seen.setdefault("c", c)
        seen.setdefault("kw", kw)
        return torch.zeros_like(x)

    class _Dec:
        def decode(self, z, timesteps):
            seen.setdefault("groups", []).append((z.shape[0], timesteps))
            return torch.zeros(z.shape[0], 3, z.shape[2] * 8, z.shape[3] * 8)

    p = B200SVDImageToVideo(net, cond, _Dec(), device="cpu")
    img = torch.rand(3, 32, 64, generator=torch.Generator().manual_seed(0))
    T = 10
    out = p(img, num_frames=T, num_inference_steps=2, fps=9, motion_bucket_id=100, noise_aug_strength=0.05,
            decode_chunk_size=4, generator=torch.Generator().manual_seed(11))
    g = torch.Generator().manual_seed(11)
    n_img = torch.randn((1, 3, 32, 64), generator=g)
    n_lat = torch.randn((T, 4, 4, 8), generator=g)
    assert torch.equal(enc.seen[0], (img * 2.0 - 1.0)[None] + 0.05 * n_img)
    sig0 = 700.0
    c_in = 1.0 / np.sqrt(sig0 ** 2 + 1.0)
    x0 = seen["x0"]
    assert x0.shape == (2 * T, 4, 4, 8)
    assert torch.allclose(x0[:T], n_lat * float(np.sqrt(1 + sig0 ** 2)) * c_in, rtol=1e-5, atol=1e-6)
    c = seen["c"]
    assert c["crossattn"].shape == (2 * T, 1, 1024) and not c["crossattn"][:T].any()
    assert c["concat"].shape == (2 * T, 4, 4, 8)
    half = 128
    freqs = torch.exp(-np.log(10000.0) * torch.arange(half, dtype=torch.float32) / half)
    for k, v in enumerate((8.0, 100.0, 0.05)):
        ref = torch.cat([torch.cos(v * freqs), torch.sin(v * freqs)])
        assert (c["vector"][:, 256 * k:256 * (k + 1)] - ref[None]).abs().max() <= 2.0 ** -8
    assert seen["kw"]["num_video_frames"] == T and seen["kw"]["batch_size"] == 2
    assert seen["groups"] == [(4, 4), (4, 4), (2, 2)]
    assert out.shape == (T, 3, 32, 64)


def test_uint8_input_is_divided_by_255():
    from streamingt2v_b200.first_chunk import image_to_unit_tensor
    a = np.random.default_rng(0).integers(0, 256, size=(16, 24, 3), dtype=np.uint8)
    t = image_to_unit_tensor(a, "cpu")
    assert t.shape == (3, 16, 24) and torch.equal(t, torch.from_numpy(a.astype(np.float32) / 255.0).permute(2, 0, 1))
    with pytest.raises(ValueError):
        image_to_unit_tensor(np.zeros((3, 16, 24), np.uint8), "cpu")


# ---- the driver against the golden -------------------------------------------------------------------------------
def test_driver_with_fakes_matches_golden(patched):
    """B200SVDImageToVideo's host logic (conditioner on the real host code of the CLIP tower and VAE encoder, Karras
    sampler, decode groups) with the CPU fakes for the kernels and the oracle UNet for the network, against the
    golden of oracle/make_golden_first_chunk.py, before the 8-bit round trip."""
    from oracle import make_golden_first_chunk as mg
    from oracle import streaming_svd_oracle as uo
    from streamingt2v_b200 import arch, vae
    from streamingt2v_b200.conditioner import B200ClipImageEncoder
    from streamingt2v_b200.first_chunk import B200SVDImageToVideo
    g = np.load(GOLDEN)
    T, H, W, steps, seed = (int(v) for v in g["meta"][:5])
    sd_u, sd_c, sd_e, sd_d = mg.weights()
    vcfg = arch.VaeConfig()
    cond = patched.B200SVDConditioner(B200ClipImageEncoder(arch.CLIP_TINY, sd_c, "cpu"),
                                      vae.B200VaeEncoder(vcfg, sd_e, "cpu"), noise="gaussian")

    def net(x, t, c, **kw):
        return uo.unet_forward(sd_u, arch.TINY, torch.cat([x, c["concat"]], 1), t, c["crossattn"], c["vector"],
                               kw["num_video_frames"], 0)

    p = B200SVDImageToVideo(net, cond, vae.B200VaeDecoder(vcfg, sd_d, "cpu"), device="cpu")
    kw = dict(num_frames=T, num_inference_steps=steps, min_guidance_scale=1.0, max_guidance_scale=3.0, fps=7,
              motion_bucket_id=127, noise_aug_strength=0.02, generator=torch.Generator().manual_seed(seed))
    image = mg.make_image(seed)
    with torch.no_grad():
        c, _ = cond.condition(image * 2.0 - 1.0, T, fps_id=6, motion_bucket_id=127, cond_aug=0.02,
                              generator=torch.Generator().manual_seed(seed))
        z = p.sample(image, **kw)
        frames = p.decode(z, 8)
    for k in ("crossattn", "concat"):
        assert _rel(c[k], torch.from_numpy(g[k])) < 3e-2, k
    assert (c["vector"] - torch.from_numpy(g["vector"])).abs().max() <= 2.0 ** -8
    assert _rel(z, torch.from_numpy(g["latents"])) < 3e-2
    assert _rel(frames, torch.from_numpy(g["frames"].astype(np.float32))) < 3e-2


# ---- image_to_video ----------------------------------------------------------------------------------------------
def test_image_to_video_bookkeeping():
    from PIL import Image
    from streamingt2v_b200.stage import B200StreamingSVDStage, resize_and_keep
    rng = np.random.default_rng(5)
    src = rng.integers(0, 256, size=(288, 512, 3), dtype=np.uint8)
    seen = {}

    def first_chunk(image, generator=None):
        seen["image"], seen["generator"] = image, generator
        return torch.linspace(-1, 1, 4 * 3 * 576 * 1024).reshape(4, 3, 576, 1024)

    stage = B200StreamingSVDStage(None, types.SimpleNamespace(num_frames=4), None, None, device="cpu")
    gen = torch.Generator().manual_seed(1)
    video = stage.image_to_video(src, 0, first_chunk, generator=gen)
    ref = np.asarray(Image.fromarray(src).resize((1024, 576)))                         # Pillow's default filter
    assert seen["image"].dtype == np.uint8 and seen["image"].shape == (576, 1024, 3)
    assert np.array_equal(seen["image"], ref) and seen["generator"] is gen
    assert video.shape == (4, 3, 576, 1024)
    assert torch.allclose(video, (first_chunk(None) + 1) * 127.5)
    # width follows the height's scale factor, truncated (inference_utils.py:37-42)
    assert resize_and_keep(np.zeros((300, 500, 3), np.uint8)).size == (960, 576)
    with pytest.raises(AssertionError):
        stage.image_to_video(np.zeros((300, 500, 3), np.uint8), 0, first_chunk)
