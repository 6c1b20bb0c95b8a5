"""Weight packing: SGM/PyTorch parameter layouts -> kernel-friendly bf16 [taps][N][K] (K contiguous) buffers.

Key grammar of the state dict: SURVEY.md Appendix B (reference code/models/diffusion/video_model.py:94-495).
"""
from __future__ import annotations

import torch


def _bf16(t: torch.Tensor, device) -> torch.Tensor:
    return t.detach().to(device=device, dtype=torch.bfloat16).contiguous()


def pad_k(w: torch.Tensor, mult: int = 8) -> torch.Tensor:
    """Zero-pad the last (K) dim to a multiple of `mult` (TMA rows must be 16-byte multiples)."""
    k = w.shape[-1]
    kp = -(-k // mult) * mult
    if kp == k:
        return w
    return torch.nn.functional.pad(w, (0, kp - k))


def pack_linear(w: torch.Tensor, device) -> torch.Tensor:
    """nn.Linear weight [N, K] -> [1, N, Kp]."""
    return _bf16(pad_k(w.float())[None], device)


def pack_conv3x3(w: torch.Tensor, device) -> torch.Tensor:
    """Conv2d weight [Cout, Cin, 3, 3] -> [9, Cout, Cinp], tap = kh*3 + kw."""
    cout, cin, kh, kw = w.shape
    assert (kh, kw) == (3, 3)
    return _bf16(pad_k(w.float().permute(2, 3, 0, 1).reshape(9, cout, cin)), device)


def pack_conv1x1(w: torch.Tensor, device) -> torch.Tensor:
    """Conv2d 1x1 weight [Cout, Cin, 1, 1] -> [1, Cout, Cin]."""
    cout, cin = w.shape[:2]
    return _bf16(pad_k(w.float().reshape(1, cout, cin)), device)


def pack_tconv3(w: torch.Tensor, device) -> torch.Tensor:
    """Conv3d weight [Cout, Cin, 3, 1, 1] -> [3, Cout, Cin], tap = kt."""
    cout, cin, kt, kh, kw = w.shape
    assert (kt, kh, kw) == (3, 1, 1)
    return _bf16(pad_k(w.float()[:, :, :, 0, 0].permute(2, 0, 1)), device)


def geglu_tile(n2: int) -> int:
    """N tile of a GEGLU projection with 2F = n2 output rows: the kernel's 256-wide tile (128 value + 128 gate)."""
    if n2 % 256 != 0:
        raise ValueError(f"GEGLU width {n2} must be a multiple of 256")
    return 256


def pack_geglu(w: torch.Tensor, b: torch.Tensor, device):
    """GEGLU proj weight [2F, K] (rows [0,F) = value, [F,2F) = gate; attention.py:94-101) -> rows interleaved per
    N tile: tile j holds value rows [j*h, (j+1)*h) followed by the matching gate rows, h = bn/2.
    Returns (w_packed [1, 2F, K] bf16, bias_packed [2F] fp32, bn)."""
    n2, k = w.shape
    f = n2 // 2
    bn = geglu_tile(n2)
    h = bn // 2
    idx = []
    for j in range(n2 // bn):
        idx.extend(range(j * h, (j + 1) * h))
        idx.extend(range(f + j * h, f + (j + 1) * h))
    idx = torch.tensor(idx, dtype=torch.long)
    wp = _bf16(pad_k(w.float()[idx])[None], device)
    bp = b.detach().float()[idx].to(device).contiguous()
    return wp, bp, bn


def f32(t: torch.Tensor, device) -> torch.Tensor:
    return t.detach().to(device=device, dtype=torch.float32).contiguous()


# ---- OpenCLIP ViT-H/14 image tower (conditioner.py) -------------------------------------------------------------
def pack_clip_patch(w: torch.Tensor, device) -> torch.Tensor:
    """conv1 weight [width, 3, 14, 14] (no bias) -> [1, width, 592] in the column order of the preprocessing kernel's
    patch rows: column (kh*14 + kw)*3 + c, zero-padded from 588 to 592."""
    width, c, kh, kw = w.shape
    return _bf16(pad_k(w.float().permute(0, 2, 3, 1).reshape(width, kh * kw * c))[None], device)


def pack_clip_class_row(class_embedding: torch.Tensor, pos: torch.Tensor, device) -> torch.Tensor:
    """Token 0 of every image before ln_pre: class_embedding + positional_embedding[0], one bf16 row [1, width]."""
    return _bf16((class_embedding.float() + pos.float()[0])[None], device)


def pack_clip_patch_pos(pos: torch.Tensor, device) -> torch.Tensor:
    """positional_embedding [257, width] -> bf16 [257, width] rows [0, pos[1], ..., pos[256]]: added with add_rows to
    every image's token rows — patch tokens get their embedding, the class row (already holding pos[0]) zero."""
    p = pos.float().clone()
    p[0] = 0.0
    return _bf16(p, device)


def pack_clip_proj(proj: torch.Tensor, device) -> torch.Tensor:
    """`proj` [width, output_dim] (x @ proj) -> nn.Linear layout [1, output_dim, width]."""
    return pack_linear(proj.float().t(), device)
