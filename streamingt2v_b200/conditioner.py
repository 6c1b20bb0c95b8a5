"""SVD conditioner on the project's kernels — drop-in for the `conditioner(svd_input_frame, num_frames) -> (c, uc)`
callable that `B200StreamingSVDStage` takes (stage.py), i.e. for streaming_svd.py:166-193 of the reference: the value
dict, `get_batch_sgm`, and `GeneralConditioner.get_unconditional_conditioning(batch, batch_uc,
force_uc_zero_embeddings=["cond_frames", "cond_frames_without_noise"])` over the five embedders of
config.yaml:159-218 (encoders/modules.py:71-188):
    0  FrozenOpenCLIPImagePredictionEmbedder(cond_frames_without_noise)  -> crossattn [1, 1, 1024]
    1  ConcatTimestepEmbedderND(256)(fps_id)                             -> vector[:,   0:256]
    2  ConcatTimestepEmbedderND(256)(motion_bucket_id)                   -> vector[:, 256:512]
    3  VideoPredictionEmbedderWithEncoder(cond_frames), scale 1.0        -> concat [1, 4, H/8, W/8] (posterior mode)
    4  ConcatTimestepEmbedderND(256)(cond_aug)                           -> vector[:, 512:768]
`uc` has crossattn and concat zeroed and the same vector.  The reference also runs the image tower and the VAE encoder
on the unconditional batch and then multiplies by zero; this module skips that work (same output).

Same conventions as model.py / vae.py: channel-last bf16 token rows, fp32 accumulation, every tensor op one of our
kernels; torch only allocates, converts dtypes, and draws the cond_aug noise and adds it to the frame (one fp32
`image + cond_aug * noise`, written as the reference writes it)."""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch

from . import dist_utils, ops, packing
from ._lib import ACT_GELU
from .arch import ClipVisionConfig

SD = Dict[str, torch.Tensor]
CLIP_SIZE = 224


def antialias_taps(h: int, w: int) -> Tuple[List[float], List[float]]:
    """1-D Gaussian taps (y, x) of kornia 0.7.2's `resize(..., antialias=True)` to 224 x 224 (restated from its
    published source; kornia is not a dependency): blur only when downscaling, sigma_i = max((factor_i - 1)/2, 0.001),
    ks_i = int(max(4 sigma_i, 3)) made odd, taps exp(-x^2 / 2 sigma^2) normalised in fp32.  [1.0] = no blur (also for
    a 224 x 224 input, which kornia returns unchanged)."""
    factors = (h / CLIP_SIZE, w / CLIP_SIZE)
    if (h, w) == (CLIP_SIZE, CLIP_SIZE) or max(factors) <= 1:
        return [1.0], [1.0]
    out = []
    for f in factors:
        sigma = max((f - 1.0) / 2.0, 0.001)
        ks = int(max(2.0 * 2 * sigma, 3))
        ks += 1 if ks % 2 == 0 else 0
        x = torch.arange(ks, dtype=torch.float32) - ks // 2
        g = torch.exp(-x.pow(2.0) / (2 * torch.tensor(sigma, dtype=torch.float32).pow(2.0)))
        out.append((g / g.sum()).tolist())
    return out[0], out[1]


class B200ClipImageEncoder:
    """OpenCLIP ViT-H/14 image tower with FrozenOpenCLIPImageEmbedder's preprocessing (encoders/modules.py:624-636,
    697-729; open_clip 2.24 VisionTransformer, visual tower only).  `sd` is `model.visual.state_dict()` in open_clip's
    key layout (arch.clip_visual_param_shapes) — restated from open_clip's published source, not checked against a
    checkpoint offline."""

    def __init__(self, cfg: ClipVisionConfig, sd: SD, device):
        ops._lib.init(torch.device(device).index or 0)
        assert cfg.head_dim == 80 and cfg.image_size == 224 and cfg.patch_size == 14, "kernels cover ViT-*/14 @ 224, d80"
        self.cfg, self.dev = cfg, torch.device(device)
        P, d = packing, self.dev

        def ln(p):
            return (P.f32(sd[p + ".weight"], d), P.f32(sd[p + ".bias"], d))

        pos = sd["positional_embedding"]
        self.w_patch = P.pack_clip_patch(sd["conv1.weight"], d)
        self.cls_row = P.pack_clip_class_row(sd["class_embedding"], pos, d)
        self.pos_rows = P.pack_clip_patch_pos(pos, d)
        self.ln_pre, self.ln_post = ln("ln_pre"), ln("ln_post")
        self.blocks = []
        for i in range(cfg.layers):
            b = f"transformer.resblocks.{i}"
            self.blocks.append(dict(
                ln1=ln(b + ".ln_1"), ln2=ln(b + ".ln_2"),
                qkv=(P.pack_linear(sd[b + ".attn.in_proj_weight"], d), P.f32(sd[b + ".attn.in_proj_bias"], d)),
                out=(P.pack_linear(sd[b + ".attn.out_proj.weight"], d), P.f32(sd[b + ".attn.out_proj.bias"], d)),
                fc=(P.pack_linear(sd[b + ".mlp.c_fc.weight"], d), P.f32(sd[b + ".mlp.c_fc.bias"], d)),
                proj=(P.pack_linear(sd[b + ".mlp.c_proj.weight"], d), P.f32(sd[b + ".mlp.c_proj.bias"], d))))
        self.w_proj = P.pack_clip_proj(sd["proj"], d)
        self.debug_taps: Optional[dict] = None

    @torch.no_grad()
    def encode(self, image: torch.Tensor) -> torch.Tensor:
        """image: [n, 3, H, W] in [-1, 1] -> image embedding [n, output_dim] fp32."""
        n, c, h, w = image.shape
        assert c == 3
        cfg, dev = self.cfg, self.dev
        W, S = cfg.width, cfg.tokens
        x32 = image.to(dev, torch.float32).contiguous()
        ty, tx = antialias_taps(h, w)
        a = ops.clip_preprocess(x32, ty, tx)                                         # [(n 256), 592] bf16
        x = torch.empty((n * S, W), dtype=torch.bfloat16, device=dev)              # token rows (n, 257)
        ops.linear_grouped(a, self.w_patch, groups=n, out=x[1:], out_group_rows=S)  # patch tokens: rows 1..256
        ops.copy2d(self.cls_row.expand(n, W), x[0::S])                             # class token + pos[0]: row 0
        ops.add_rows(x, self.pos_rows)                                              # + pos[1..256] on patch rows
        x = ops.layer_norm(x, *self.ln_pre, cfg.eps)
        taps = self.debug_taps
        if taps is not None:
            taps["ln_pre"] = x
        for i, e in enumerate(self.blocks):
            hn = ops.layer_norm(x, *e["ln1"], cfg.eps)
            qkv = ops.linear(hn, *e["qkv"])
            att = ops.flash_attn_d80(qkv, n, S, cfg.heads)
            x = ops.linear(att, *e["out"], res1=x, s1=1.0)
            hn = ops.layer_norm(x, *e["ln2"], cfg.eps)
            f = ops.linear(hn, *e["fc"], act=ACT_GELU)
            x = ops.linear(f, *e["proj"], res1=x, s1=1.0)
            if taps is not None:
                taps[f"block.{i}"] = x
        pooled = ops.layer_norm(x[0::S], *self.ln_post, cfg.eps)                   # class rows, row stride 257*W
        if taps is not None:
            taps["pooled"] = pooled
        return ops.linear(pooled, self.w_proj, None, out_fp32=True)


class B200SVDConditioner:
    """The conditioner callable of `B200StreamingSVDStage`: `(frame [3, H, W] in [-1, 1], num_frames) -> (c, uc)` with
    `crossattn [1, 1, 1024]`, `concat [1, 4, H/8, W/8]` and `vector [num_frames, 768]`, fp32 on the device.

    cond_frames = image + cond_aug * U[0, 1) noise (streaming_svd.py:174; `torch.rand_like`, uniform).  With
    `generator` the noise is `torch.rand(image.shape, generator=generator, device=generator.device)`; without one it
    comes from torch's global generator, as in the reference.  Under torch.distributed with more than one rank, rank
    0's noise is broadcast so that every rank conditions on the same frames."""

    def __init__(self, clip: B200ClipImageEncoder, vae_encoder, *, generator: Optional[torch.Generator] = None,
                 fps_id: int = 6, motion_bucket_id: int = 127, cond_aug: float = 0.02):
        self.clip, self.vae_encoder = clip, vae_encoder
        self.generator = generator
        self.fps_id, self.motion_bucket_id, self.cond_aug = fps_id, motion_bucket_id, float(cond_aug)
        self.dev = clip.dev

    @classmethod
    def from_reference(cls, conditioner, device="cuda:0", **kw):
        """Build from the reference's instantiated `GeneralConditioner` (config.yaml:159-218): the image tower from
        `embedders[0].open_clip.model.visual.state_dict()`, the VAE encoder from `embedders[3].encoder.encoder.*` and
        `embedders[3].encoder.quant_conv.*`."""
        from .arch import VaeConfig
        from .vae import B200VaeEncoder
        sd_v = conditioner.embedders[0].open_clip.model.visual.state_dict()
        layers = sum(1 for k in sd_v if k.startswith("transformer.resblocks.") and k.endswith(".attn.in_proj_weight"))
        width = sd_v["conv1.weight"].shape[0]
        ccfg = ClipVisionConfig(image_size=int(round((sd_v["positional_embedding"].shape[0] - 1) ** 0.5))
                                * sd_v["conv1.weight"].shape[-1], patch_size=sd_v["conv1.weight"].shape[-1],
                                width=width, layers=layers, heads=width // 80,
                                mlp=sd_v["transformer.resblocks.0.mlp.c_fc.weight"].shape[0],
                                output_dim=sd_v["proj"].shape[1])
        ae = conditioner.embedders[3].encoder
        sd_e = dict(ae.encoder.state_dict())
        sd_e.update({"quant_conv." + k: v for k, v in ae.quant_conv.state_dict().items()})
        ch = sd_e["conv_in.weight"].shape[0]
        levels = sum(1 for k in sd_e if k.startswith("down.") and k.endswith(".block.0.conv1.weight"))
        vcfg = VaeConfig(ch=ch, ch_mult=tuple(sd_e[f"down.{i}.block.0.conv1.weight"].shape[0] // ch for i in range(levels)),
                         num_res_blocks=sum(1 for k in sd_e if k.startswith("down.0.block.") and k.endswith(".conv1.weight")),
                         z_channels=sd_e["quant_conv.weight"].shape[0] // 2)
        return cls(B200ClipImageEncoder(ccfg, sd_v, device), B200VaeEncoder(vcfg, sd_e, device), **kw)

    def _noise(self, image: torch.Tensor) -> torch.Tensor:
        g = self.generator
        if g is not None:
            noise = torch.rand(image.shape, generator=g, device=g.device)
        else:
            noise = torch.rand_like(image)
        noise = noise.to(self.dev, torch.float32)
        return dist_utils.broadcast_from_rank0(noise)

    @torch.no_grad()
    def __call__(self, frame: torch.Tensor, num_frames: int):
        T = int(num_frames)
        image = frame[None].to(self.dev, torch.float32).contiguous()                    # [1, 3, H, W]
        cond_frames = image + self.cond_aug * self._noise(image)
        crossattn = self.clip.encode(image)[:, None, :]                                # [1, 1, 1024]
        concat = self.vae_encoder.encode(cond_frames)                                   # [1, 4, H/8, W/8], scale 1.0
        t = torch.tensor([float(self.fps_id)] * T + [float(self.motion_bucket_id)] * T + [self.cond_aug] * T,
                         dtype=torch.float32, device=self.dev)
        emb = ops.timestep_embed(t, 256)                                                # [(3 T), 256] bf16
        vector = emb.float().view(3, T, 256).transpose(0, 1).reshape(T, 768)           # [fps | motion | cond_aug]
        c = {"crossattn": crossattn, "concat": concat, "vector": vector}
        uc = {"crossattn": torch.zeros_like(crossattn), "concat": torch.zeros_like(concat), "vector": vector.clone()}
        return c, uc
