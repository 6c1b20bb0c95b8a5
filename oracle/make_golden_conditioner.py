"""ORACLE tooling — build-container only.  Golden vectors for the SVD conditioner (OpenCLIP ViT-H/14 image tower,
CLIP preprocessing, SD-VAE encoder, conditioning assembly), pinned two ways:

1. The tower restatement (oracle/clip_image_oracle.py) against an independent published implementation of the same
   function, HF transformers' CLIPVisionModelWithProjection (hidden_act "gelu" = erf, eps 1e-5), with the weights
   mapped from the open_clip layout (in_proj split into q/k/v, visual_projection.weight = proj.T), at full ViT-H and at
   arch.CLIP_TINY: max error <= 1e-4 * max|ref|.
2. The assembly against the UNMODIFIED reference `GeneralConditioner` (encoders/modules.py:71-188) built from the
   literal `emb_models` of code/config.yaml:159-218 and driven as streaming_svd.py:166-193 drives it (value dict,
   get_batch_sgm, get_unconditional_conditioning).  Stand-ins, in the manner of ref_shims._Attention:
     open_clip.create_model_and_transforms  -> a module holding the open_clip `visual` key layout whose forward is
                                               clip_image_oracle.visual (checked against HF in 1.)
     kornia.geometry.resize / kornia.enhance.normalize -> clip_image_oracle.resize_224 / normalize (kornia 0.7.2
                                               restated; parity unpinned at that boundary)
     xformers.ops.memory_efficient_attention -> SDPA (the VAE encoder's attn_type "vanilla-xformers")
   The reference draws `cond_frames` noise with torch.rand_like from the global generator; torch.manual_seed(seed)
   makes that the noise of torch.rand(shape, generator=torch.Generator().manual_seed(seed)) (asserted below).

Weights come from arch.synth_state_dict; frames from numpy default_rng([seed, 77]).  Fixtures keep only outputs and
seeds (each < 1 MB); tests regenerate the frame.    python oracle/make_golden_conditioner.py"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import clip_image_oracle as co  # noqa: E402
from streamingt2v_b200 import arch  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
# name: (clip config, n images, H, W, seed)
TINY_CASES = {"clip_tiny_2_448x320": (2, 448, 320, 31),      # ks 3 on both axes
              "clip_tiny_1_128x300": (1, 128, 300, 32)}      # upsampled H axis (sigma 0.001)
FULL_CASE = ("cond_full_576x1024", 576, 1024, 25, 41)        # name, H, W, T, seed


def make_frame(n, H, W, seed):
    rng = np.random.default_rng([seed, 77])
    return torch.from_numpy(rng.uniform(-1, 1, size=(n, 3, H, W)).astype(np.float32))


def hf_tower(cfg, sd):
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    hcfg = CLIPVisionConfig(hidden_size=cfg.width, intermediate_size=cfg.mlp, num_hidden_layers=cfg.layers,
                            num_attention_heads=cfg.heads, image_size=cfg.image_size, patch_size=cfg.patch_size,
                            projection_dim=cfg.output_dim, hidden_act="gelu", layer_norm_eps=cfg.eps,
                            num_channels=3)
    m = CLIPVisionModelWithProjection(hcfg).eval()
    w = cfg.width
    hs = {"vision_model.embeddings.class_embedding": sd["class_embedding"],
          "vision_model.embeddings.patch_embedding.weight": sd["conv1.weight"],
          "vision_model.embeddings.position_embedding.weight": sd["positional_embedding"],
          "vision_model.pre_layrnorm.weight": sd["ln_pre.weight"], "vision_model.pre_layrnorm.bias": sd["ln_pre.bias"],
          "vision_model.post_layernorm.weight": sd["ln_post.weight"],
          "vision_model.post_layernorm.bias": sd["ln_post.bias"], "visual_projection.weight": sd["proj"].t()}
    for i in range(cfg.layers):
        b, h = f"transformer.resblocks.{i}", f"vision_model.encoder.layers.{i}"
        wq, wk, wv = sd[b + ".attn.in_proj_weight"].split(w, 0)
        bq, bk, bv = sd[b + ".attn.in_proj_bias"].split(w, 0)
        for nm, ww, bb in (("q_proj", wq, bq), ("k_proj", wk, bk), ("v_proj", wv, bv)):
            hs[f"{h}.self_attn.{nm}.weight"], hs[f"{h}.self_attn.{nm}.bias"] = ww, bb
        hs[f"{h}.self_attn.out_proj.weight"] = sd[b + ".attn.out_proj.weight"]
        hs[f"{h}.self_attn.out_proj.bias"] = sd[b + ".attn.out_proj.bias"]
        for a, o in (("ln_1", "layer_norm1"), ("ln_2", "layer_norm2"), ("mlp.c_fc", "mlp.fc1"), ("mlp.c_proj", "mlp.fc2")):
            hs[f"{h}.{o}.weight"], hs[f"{h}.{o}.bias"] = sd[f"{b}.{a}.weight"], sd[f"{b}.{a}.bias"]
    missing, unexpected = m.load_state_dict(hs, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    return m


def pin_tower(cfg, sd, img, label):
    m = hf_tower(cfg, sd)
    with torch.no_grad():
        ref = m(pixel_values=img).image_embeds
        out = co.visual(sd, cfg, img)
    err = (out - ref).abs().max().item()
    print(f"[tower {label}] HF CLIPVisionModelWithProjection vs oracle: max err {err:.3e} (max|ref| {ref.abs().max():.3f})")
    assert err <= 1e-4 * ref.abs().max().item(), err
    return err


# ---- the reference GeneralConditioner under stand-ins ---------------------------------------------------------------
class _Visual(nn.Module):
    """open_clip `model.visual` key layout; forward = the oracle restatement."""

    def __init__(self, cfg, sd):
        super().__init__()
        self.cfg = cfg
        self.output_tokens = False
        for k, v in sd.items():
            self.register_buffer(k.replace(".", "__"), v.clone())

    def state_dict(self, *a, **kw):
        return {k.replace("__", "."): v for k, v in self._buffers.items()}

    def forward(self, img):
        return co.visual(self.state_dict(), self.cfg, img)


def build_reference_conditioner(clip_cfg, clip_sd, vae_sd):
    from oracle import ref_shims
    ref_shims.install()
    import yaml

    class _Model(nn.Module):
        def __init__(self):
            super().__init__()
            self.visual = _Visual(clip_cfg, clip_sd)
            self.transformer = nn.Identity()

    def create_model_and_transforms(arch_name, device=None, pretrained=None):
        assert arch_name == "ViT-H-14"
        return _Model(), None, None

    def resize(x, size, interpolation, align_corners, antialias):
        assert tuple(size) == (224, 224) and interpolation == "bicubic" and align_corners and antialias
        return co.resize_224(x)

    def normalize(x, mean, std):
        return (x - mean.view(1, -1, 1, 1)) / std.view(1, -1, 1, 1)

    oc = sys.modules["open_clip"]
    oc.create_model_and_transforms = create_model_and_transforms
    kn = sys.modules["kornia"]
    kn.geometry = types.SimpleNamespace(resize=resize)
    kn.enhance = types.SimpleNamespace(normalize=normalize)

    def mea(q, k, v, attn_bias=None, op=None):
        return F.scaled_dot_product_attention(q, k, v)
    xf = types.ModuleType("xformers")
    xf.ops = types.SimpleNamespace(memory_efficient_attention=mea)
    import models.svd.sgm.modules.diffusionmodules.model as mdl
    mdl.xformers = xf
    mdl.XFORMERS_IS_AVAILABLE = True

    with open(os.path.join(ref_shims.REFERENCE_CODE, "config.yaml")) as f:
        conf = yaml.safe_load(f)

    def find(d):
        if isinstance(d, dict):
            if d.get("class_path", "").endswith("GeneralConditioner"):
                return d
            for v in d.values():
                r = find(v)
                if r is not None:
                    return r
        return None

    emb_models = find(conf)["init_args"]["emb_models"]
    from models.svd.sgm.modules.encoders.modules import GeneralConditioner
    cond = GeneralConditioner(emb_models).eval()
    ae = cond.embedders[3].encoder
    ae.encoder.load_state_dict({k: v for k, v in vae_sd.items() if not k.startswith("quant_conv.")}, strict=True)
    ae.quant_conv.load_state_dict({k[len("quant_conv."):]: v for k, v in vae_sd.items() if k.startswith("quant_conv.")})
    return cond


def run_reference(cond, frame, T, seed):
    """streaming_svd.py:166-193 on a mock of the value-dict plumbing (get_batch_sgm restated line for line)."""
    import math

    from einops import repeat
    image = frame[None]
    value_dict = {"motion_bucket_id": 127, "fps_id": 6, "cond_aug": 0.02, "cond_frames_without_noise": image}
    torch.manual_seed(seed)
    value_dict["cond_frames"] = image + 0.02 * torch.rand_like(image)
    noise = torch.rand(image.shape, generator=torch.Generator().manual_seed(seed))
    assert torch.equal(value_dict["cond_frames"], image + 0.02 * noise)
    N = [1, T]
    keys = list(set(e.input_key for e in cond.embedders))
    batch = {}
    for key in keys:
        if key in ("fps_id", "motion_bucket_id"):
            batch[key] = torch.tensor([value_dict[key]]).repeat(int(math.prod(N)))
        elif key == "cond_aug":
            batch[key] = repeat(torch.tensor([value_dict["cond_aug"]]), "1 -> b", b=math.prod(N))
        else:
            batch[key] = repeat(value_dict[key], "1 ... -> b ...", b=N[0])
    batch["num_video_frames"] = T
    batch_uc = {k: torch.clone(v) for k, v in batch.items() if isinstance(v, torch.Tensor)}
    with torch.no_grad():
        c, uc = cond.get_unconditional_conditioning(batch, batch_uc=batch_uc,
                                                    force_uc_zero_embeddings=["cond_frames", "cond_frames_without_noise"])
    return c, uc


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    full = arch.ClipVisionConfig()
    tiny = arch.CLIP_TINY
    sd_full = arch.synth_state_dict(arch.clip_visual_param_shapes(full), seed=51)
    sd_tiny = arch.synth_state_dict(arch.clip_visual_param_shapes(tiny), seed=52)
    vcfg = arch.VaeConfig()
    sd_vae = arch.synth_state_dict(arch.vae_encoder_param_shapes(vcfg), seed=53)

    # 1. tower vs HF
    for name, (n, H, W, seed) in TINY_CASES.items():
        img = co.preprocess(make_frame(n, H, W, seed))
        pin_tower(tiny, sd_tiny, img, name)
        taps = {}
        with torch.no_grad():
            out = co.encode(sd_tiny, tiny, make_frame(n, H, W, seed), taps)
        np.savez_compressed(os.path.join(GOLDEN, f"{name}.npz"), out=out.numpy(),
                            meta=np.array([n, H, W, seed, 52], np.int64),
                            **{"tap_" + k: v.numpy().astype(np.float16) for k, v in taps.items()})
    H, W = 576, 1024
    name, H, W, T, seed = FULL_CASE
    frame = make_frame(1, H, W, seed)[0]
    tower_err = pin_tower(full, sd_full, co.preprocess(frame[None]), "ViT-H")

    # 2. assembly vs the unmodified reference GeneralConditioner
    cond = build_reference_conditioner(full, sd_full, sd_vae)
    c, uc = run_reference(cond, frame, T, seed)
    assert tuple(c["crossattn"].shape) == (1, 1, 1024) and tuple(c["concat"].shape) == (1, 4, H // 8, W // 8)
    assert tuple(c["vector"].shape) == (T, 768)
    assert not uc["crossattn"].any() and not uc["concat"].any() and torch.equal(uc["vector"], c["vector"])
    with torch.no_grad():
        direct = co.encode(sd_full, full, frame[None])
    err = (direct - c["crossattn"][:, 0]).abs().max().item()
    print(f"[assembly] reference crossattn vs oracle tower: {err:.3e}; concat absmax {c['concat'].abs().max():.3f}")
    assert err == 0.0
    np.savez_compressed(os.path.join(GOLDEN, f"{name}.npz"), crossattn=c["crossattn"].numpy(),
                        concat=c["concat"].numpy(), vector=c["vector"].numpy(),
                        meta=np.array([H, W, T, seed, 51, 53], np.int64),
                        frame_sum=np.array([frame.double().sum().item()]),
                        tower_vs_hf_maxerr=np.array([tower_err]))
    print("done")


if __name__ == "__main__":
    main()
