"""TEST INFRASTRUCTURE — tests/fake_ops.py extended with CPU stand-ins for the conditioner's ops (head-dim-80
attention, CLIP preprocessing, the grouped patch GEMM), for the `-m "not gpu"` host-logic tests of
streamingt2v_b200/conditioner.py.  Every fake_ops function is re-exported unchanged (launch counter included); the new
ones compute in fp32 with torch CPU ops and round to bf16 where the CUDA kernels round.  The product never imports
this module."""
from __future__ import annotations

import torch
import torch.nn.functional as F

import fake_ops
from fake_ops import *  # noqa: F401,F403  (the stand-ins of every existing op)
from fake_ops import _count, _lib  # noqa: F401  (private names the host code reaches: ops._lib.init)


def launches():
    return fake_ops.launches()


def flash_attn_d80(qkv, n, s, heads, out=None):
    _count()
    Cc = heads * 80
    q, k, v = (t.float().reshape(n, s, heads, 80).permute(0, 2, 1, 3) for t in qkv[:, :3 * Cc].chunk(3, dim=1))
    o = F.scaled_dot_product_attention(q, k, v).permute(0, 2, 1, 3).reshape(n * s, Cc).to(torch.bfloat16)
    if out is not None:
        out.copy_(o)
        return out
    return o


def clip_preprocess(x, taps_y, taps_x, out=None):
    """Separable blur with the given taps (reflect borders), bicubic align_corners resize to 224, CLIP normalisation,
    patch rows [(n 256), 592] with column (kh*14 + kw)*3 + c."""
    _count()
    n, c, H, W = x.shape
    gy = torch.tensor(taps_y, dtype=torch.float32)
    gx = torch.tensor(taps_x, dtype=torch.float32)
    ky, kx = len(taps_y), len(taps_x)
    v = F.pad(x.float(), (kx // 2, kx // 2, 0, 0), mode="reflect") if kx > 1 else x.float()
    v = F.conv2d(v, gx.view(1, 1, 1, kx).repeat(c, 1, 1, 1), groups=c)
    v = F.pad(v, (0, 0, ky // 2, ky // 2), mode="reflect") if ky > 1 else v
    v = F.conv2d(v, gy.view(1, 1, ky, 1).repeat(c, 1, 1, 1), groups=c)
    if (H, W) != (224, 224):
        v = F.interpolate(v, size=(224, 224), mode="bicubic", align_corners=True)
    mean = torch.tensor((0.48145466, 0.4578275, 0.40821073)).view(1, 3, 1, 1)
    std = torch.tensor((0.26862954, 0.26130258, 0.27577711)).view(1, 3, 1, 1)
    v = ((v + 1.0) / 2.0 - mean) / std
    rows = v.reshape(n, c, 16, 14, 16, 14).permute(0, 2, 4, 3, 5, 1).reshape(n * 256, 588)
    res = torch.zeros((n * 256, 592), dtype=torch.bfloat16)
    res[:, :588] = rows.to(torch.bfloat16)
    if out is not None:
        out.copy_(res)
        return out
    return res


def linear_grouped(x, w, bias=None, *, groups, out, out_group_rows, **epi):
    rows = x.shape[0] // groups
    for g in range(groups):
        fake_ops.linear(x[g * rows:(g + 1) * rows], w, bias, out=out[g * out_group_rows:g * out_group_rows + rows],
                        **epi)
    return out
