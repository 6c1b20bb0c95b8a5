"""ORACLE — pure-torch fp32 restatement of the SVD conditioner's image branch (no reference import, usable on the GPU
machine): FrozenOpenCLIPImageEmbedder.preprocess (reference code/models/svd/sgm/modules/encoders/modules.py:624-636)
and open_clip 2.24's ViT-H/14 `model.visual` forward, in the open_clip state-dict key layout of
arch.clip_visual_param_shapes.

kornia 0.7.2 `geometry.resize(..., interpolation="bicubic", align_corners=True, antialias=True)` restated from its
published source (kornia is not installed offline — parity unpinned at that boundary):
  factors = (H/224, W/224); if max(factors) > 1: sigma_i = max((factor_i - 1)/2, 0.001),
  ks_i = int(max(4 sigma_i, 3)) (+1 if even); separable Gaussian blur, taps exp(-x^2 / 2 sigma^2) for
  x = arange(ks) - ks//2 normalised to sum 1, reflect borders; then F.interpolate(bicubic, align_corners=True).
  A 224 x 224 input is returned unchanged.
The tower is pinned against HF transformers' CLIPVisionModelWithProjection by oracle/make_golden_conditioner.py."""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
SIZE = 224


def gaussian_taps(ks: int, sigma: float) -> torch.Tensor:
    """kornia get_gaussian_kernel1d (fp32)."""
    x = torch.arange(ks, dtype=torch.float32) - ks // 2
    if ks % 2 == 0:
        x = x + 0.5
    g = torch.exp(-x.pow(2.0) / (2 * torch.tensor(sigma, dtype=torch.float32).pow(2.0)))
    return g / g.sum()


def antialias_params(h: int, w: int) -> Optional[Tuple[Tuple[int, int], Tuple[float, float]]]:
    """((ks_h, ks_w), (sigma_h, sigma_w)) of kornia's antialias blur before a resize to 224 x 224, None without blur."""
    factors = (h / SIZE, w / SIZE)
    if (h, w) == (SIZE, SIZE) or max(factors) <= 1:
        return None
    sig = (max((factors[0] - 1.0) / 2.0, 0.001), max((factors[1] - 1.0) / 2.0, 0.001))
    ks = [int(max(2.0 * 2 * sig[0], 3)), int(max(2.0 * 2 * sig[1], 3))]
    ks = [k + 1 if k % 2 == 0 else k for k in ks]
    return (ks[0], ks[1]), sig


def resize_224(x: torch.Tensor) -> torch.Tensor:
    """x: [n, 3, H, W] fp32 -> [n, 3, 224, 224] (kornia resize, bicubic, align_corners=True, antialias=True)."""
    h, w = x.shape[-2:]
    if (h, w) == (SIZE, SIZE):
        return x
    p = antialias_params(h, w)
    if p is not None:
        (ky, kx), (sy, sx) = p
        c = x.shape[1]
        gx = gaussian_taps(kx, sx).to(x)
        gy = gaussian_taps(ky, sy).to(x)
        x = F.conv2d(F.pad(x, (kx // 2, kx // 2, 0, 0), mode="reflect"), gx.view(1, 1, 1, kx).repeat(c, 1, 1, 1),
                     groups=c)
        x = F.conv2d(F.pad(x, (0, 0, ky // 2, ky // 2), mode="reflect"), gy.view(1, 1, ky, 1).repeat(c, 1, 1, 1),
                     groups=c)
    return F.interpolate(x, size=(SIZE, SIZE), mode="bicubic", align_corners=True)


def normalize(x: torch.Tensor) -> torch.Tensor:
    mean = torch.tensor(CLIP_MEAN, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
    std = torch.tensor(CLIP_STD, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
    return (x - mean) / std


def preprocess(x: torch.Tensor) -> torch.Tensor:
    """FrozenOpenCLIPImageEmbedder.preprocess: [n, 3, H, W] in [-1, 1] -> [n, 3, 224, 224] CLIP-normalised."""
    return normalize((resize_224(x.float()) + 1.0) / 2.0)


def patch_rows(img: torch.Tensor, patch: int = 14) -> torch.Tensor:
    """[n, 3, 224, 224] -> [(n g g), patch*patch*3] rows, column (kh*patch + kw)*3 + c (the patch GEMM's A operand)."""
    n, c, hh, ww = img.shape
    g = hh // patch
    t = img.reshape(n, c, g, patch, g, patch).permute(0, 2, 4, 3, 5, 1)     # n, gy, gx, kh, kw, c
    return t.reshape(n * g * g, patch * patch * c)


def _ln(x, sd, p, eps):
    return F.layer_norm(x, (x.shape[-1],), sd[p + ".weight"].float(), sd[p + ".bias"].float(), eps)


def visual(sd: Dict[str, torch.Tensor], cfg, img: torch.Tensor, taps: Optional[dict] = None,
           sdpa: bool = False) -> torch.Tensor:
    """open_clip VisionTransformer.forward on a preprocessed batch [n, 3, 224, 224] -> [n, output_dim] (fp32).
    taps (optional dict) receives "ln_pre", "block.{i}" ([n, tokens, width]) and "pooled" ([n, width], after ln_post).
    sdpa=True computes the attention with F.scaled_dot_product_attention (the eager baseline of
    scripts/bench_conditioner.py) instead of the explicit softmax."""
    sd = {k: v.float() for k, v in sd.items()}
    n = img.shape[0]
    w, heads = cfg.width, cfg.heads
    x = F.conv2d(img.float(), sd["conv1.weight"], stride=cfg.patch_size)          # [n, w, g, g]
    x = x.reshape(n, w, -1).permute(0, 2, 1)
    cls = sd["class_embedding"].view(1, 1, w).expand(n, 1, w)
    x = torch.cat([cls, x], 1) + sd["positional_embedding"][None]
    x = _ln(x, sd, "ln_pre", cfg.eps)
    if taps is not None:
        taps["ln_pre"] = x.clone()
    S = x.shape[1]
    for i in range(cfg.layers):
        b = f"transformer.resblocks.{i}"
        h = _ln(x, sd, b + ".ln_1", cfg.eps)
        qkv = h @ sd[b + ".attn.in_proj_weight"].t() + sd[b + ".attn.in_proj_bias"]
        q, k, v = (t.reshape(n, S, heads, -1).transpose(1, 2) for t in qkv.chunk(3, dim=-1))
        if sdpa:
            a = F.scaled_dot_product_attention(q, k, v)
        else:
            a = torch.softmax((q @ k.transpose(-1, -2)) / math.sqrt(q.shape[-1]), dim=-1) @ v
        a = a.transpose(1, 2).reshape(n, S, w)
        x = x + a @ sd[b + ".attn.out_proj.weight"].t() + sd[b + ".attn.out_proj.bias"]
        h = _ln(x, sd, b + ".ln_2", cfg.eps)
        h = F.gelu(h @ sd[b + ".mlp.c_fc.weight"].t() + sd[b + ".mlp.c_fc.bias"])
        x = x + h @ sd[b + ".mlp.c_proj.weight"].t() + sd[b + ".mlp.c_proj.bias"]
        if taps is not None:
            taps[f"block.{i}"] = x.clone()
    pooled = _ln(x[:, 0], sd, "ln_post", cfg.eps)
    if taps is not None:
        taps["pooled"] = pooled.clone()
    return pooled @ sd["proj"]


def encode(sd, cfg, image: torch.Tensor, taps: Optional[dict] = None, sdpa: bool = False) -> torch.Tensor:
    """FrozenOpenCLIPImageEmbedder.encode_with_vision_transformer: [n, 3, H, W] in [-1, 1] -> [n, output_dim]."""
    return visual(sd, cfg, preprocess(image), taps, sdpa)


def tap_names(cfg) -> List[str]:
    return ["ln_pre"] + [f"block.{i}" for i in range(cfg.layers)] + ["pooled"]
