"""Float64 references of the interpolation-stage kernels shared by the GPU tests."""
import torch
import torch.nn.functional as F


def ref_window_attn(q, k, v, ce, pairs, h, w, heads, shift):
    """MotionFormerBlock / InterFrameAttention arithmetic (feature_extractor.py:7-61, 146-172, 213-277) in float64 on
    token rows [2*pairs*h*w + 1, C] (q, k, v) and [h*w + 1, Cm] (ce), the last row the padding token, on any device.
    Returns (attn @ v, motion) as rows [2*pairs*h*w, C] and [2*pairs*h*w, Cm].  The masks are the reference's additive
    -100, not -inf, so a masked key still wins where its logit exceeds the others by more than 100."""
    q, k, v, ce = (t.double() for t in (q, k, v, ce))
    (qp, kp, vp, cep) = (t[-1] for t in (q, k, v, ce))
    n = 2 * pairs
    qi, ki, vi = (t[:-1].view(n, h, w, -1) for t in (q, k, v))
    cei = ce[:-1].view(1, h, w, -1).expand(n, h, w, -1)
    ws = 7
    ph, pw = -(-h // ws) * ws - h, -(-w // ws) * ws - w
    H, W = h + ph, w + pw

    def pad(t, fill):
        out = fill.view(1, 1, 1, -1).expand(t.shape[0], H, W, -1).clone()
        out[:, ph // 2:ph // 2 + h, pw // 2:pw // 2 + w] = t
        return out

    qx, kx, vx, cx = pad(qi, qp), pad(ki, kp), pad(vi, vp), pad(cei, cep)

    def part(t):
        b, _, _, c = t.shape
        return t.view(b, H // ws, ws, W // ws, ws, c).permute(0, 1, 3, 2, 4, 5).reshape(-1, ws * ws, c)

    mask = None
    if ph or pw:
        img = torch.zeros((1, H, W, 1), dtype=torch.float64, device=q.device)
        cnt = 0
        for hs in (slice(0, ph // 2), slice(ph // 2, h + ph // 2), slice(h + ph // 2, None)):
            for wsl in (slice(0, pw // 2), slice(pw // 2, w + pw // 2), slice(w + pw // 2, None)):
                img[:, hs, wsl, :] = cnt
                cnt += 1
        mw = part(img).squeeze(-1)
        mask = mw.unsqueeze(1) - mw.unsqueeze(2)
        mask = mask.masked_fill(mask != 0, -100.0).masked_fill(mask == 0, 0.0)
    if shift:
        qx, kx, vx, cx = (torch.roll(t, (-shift, -shift), (1, 2)) for t in (qx, kx, vx, cx))
        sm = torch.zeros((1, H, W, 1), dtype=torch.float64, device=q.device)
        cnt = 0
        for hs in (slice(0, -ws), slice(-ws, -shift), slice(-shift, None)):
            for wsl in (slice(0, -ws), slice(-ws, -shift), slice(-shift, None)):
                sm[:, hs, wsl, :] = cnt
                cnt += 1
        mw = part(sm).squeeze(-1)
        sm = mw.unsqueeze(1) - mw.unsqueeze(2)
        sm = sm.masked_fill(sm != 0, -100.0).masked_fill(sm == 0, 0.0)
        if mask is not None:
            sm = sm.masked_fill(mask != 0, -100.0)
        mask = sm
    Q, K, V, CE = part(qx), part(kx), part(vx), part(cx)
    nwB = Q.shape[0]
    K = torch.cat([K[nwB // 2:], K[:nwB // 2]])
    V = torch.cat([V[nwB // 2:], V[:nwB // 2]])
    N = ws * ws
    Qh = Q.view(nwB, N, heads, -1).permute(0, 2, 1, 3)
    Kh = K.view(nwB, N, heads, -1).permute(0, 2, 1, 3)
    Vh = V.view(nwB, N, heads, -1).permute(0, 2, 1, 3)
    Ch = CE.view(nwB, N, heads, -1).permute(0, 2, 1, 3)
    attn = (Qh @ Kh.transpose(-2, -1)) * 32 ** -0.5
    if mask is not None:
        nW = mask.shape[0]
        attn = (attn.view(nwB // nW, nW, heads, N, N) + mask.double().unsqueeze(1).unsqueeze(0)).view(-1, heads, N, N)
    attn = attn.softmax(-1)
    x = (attn @ Vh).transpose(1, 2).reshape(nwB, N, -1)
    m = (attn @ Ch).transpose(1, 2).reshape(nwB, N, -1) - CE

    def rev(t):
        c = t.shape[-1]
        t = t.view(n, H // ws, W // ws, ws, ws, c).permute(0, 1, 3, 2, 4, 5).reshape(n, H, W, c)
        if shift:
            t = torch.roll(t, (shift, shift), (1, 2))
        return t[:, ph // 2:ph // 2 + h, pw // 2:pw // 2 + w].reshape(n * h * w, c)

    return rev(x), rev(m)


def ref_warp(x, flow):
    """warplayer.warp in float64: grid_sample(bilinear, border, align_corners=True) at linspace grid + flow / ((size -
    1) / 2), on x's device."""
    n, c, h, w = x.shape
    gx = torch.linspace(-1.0, 1.0, w, dtype=torch.float64, device=x.device).view(1, 1, w).expand(n, h, w)
    gy = torch.linspace(-1.0, 1.0, h, dtype=torch.float64, device=x.device).view(1, h, 1).expand(n, h, w)
    g = torch.stack([gx + flow[:, 0].double() / ((w - 1.0) / 2.0), gy + flow[:, 1].double() / ((h - 1.0) / 2.0)], -1)
    return F.grid_sample(x.double(), g, mode="bilinear", padding_mode="border", align_corners=True)


def warp_bound(ref, flow, bf16_out):
    """Per-element bound on |vfi_warp - ref_warp| for input values in [0, 1], from the kernel's fp32 arithmetic.

    Coordinates.  gx = linspace(x) + f * inv with inv = 1 / ((w - 1) / 2) (each an fp32 rounding: linspace within
    2^-23, the product within 2^-23 relative), then ix = ((gx + 1) / 2) * (w - 1), two more roundings of 2^-24
    relative.  In pixels, with |gx| <= 1 + 2 |f| / (w - 1):
        |ix - ix_exact| <= 2^-24 [(w - 1) (2 + 1.5 (1 + 2 |f| / (w - 1))) + 2 |f|] <= 2^-22 (2 (w - 1) + 3 |f|)
    and the same along y.  Clamping to the border does not increase it, and the bilinear interpolant of values in
    [0, 1] changes by at most 1 per pixel along either axis, so the coordinate errors add at most dx + dy.
    Weights and sum.  The corner weights (one fp32 product each) and the four fmas add at most 8 roundings of values
    <= 1: 2^-21.  A bf16 output adds one rounding, 2^-8 |ref|."""
    n, _, h, w = flow.shape
    fx, fy = flow[:, 0].double().abs(), flow[:, 1].double().abs()
    coord = 2.0 ** -22 * (2 * (w - 1) + 3 * fx + 2 * (h - 1) + 3 * fy)
    b = (coord.unsqueeze(1) + 2.0 ** -21).expand_as(ref)
    return b + 2.0 ** -8 * ref.abs() if bf16_out else b
