"""GPU parity of the attention / normalisation / glue kernels against plain PyTorch fp32 references of the same op.
Tolerances are stated per test: inputs are the same bf16 values on both sides; outputs are bf16-rounded (2^-8
relative) and, for attention, P is rounded to bf16 before the PV product (adds ~2^-8 relative per term)."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _check(out, ref, name, rtol, atol):
    out = out.float()
    err = (out - ref).abs()
    tol = atol + rtol * ref.abs()
    bad = (err > tol).sum().item()
    print(f"{name}: max_abs_err={err.max().item():.4e} ref_absmax={ref.abs().max().item():.3e} bad={bad}/{err.numel()}")
    assert torch.isfinite(out).all(), f"{name}: non-finite output"
    assert bad == 0, f"{name}: {bad} elements out of tolerance (max err {err.max().item():.4e})"


def _rand(shape, dev, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev).to(torch.bfloat16)


@pytest.fixture(params=[3, 4, 5], ids=["two-pass", "single-pass", "16-warp"])
def fa_variant(request, cuda_dev):
    """Every FlashAttention case runs under each softmax variant the ABI accepts (the sm_90 kernel has one organisation)."""
    from streamingt2v_b200 import ops
    prev = ops.flash_attn_variant(request.param)
    yield request.param
    ops.flash_attn_variant(prev)


@pytest.mark.parametrize("n,s,heads", [(2, 256, 5), (3, 144, 2), (1, 576, 20), (2, 4, 10), (1, 1000, 5), (2, 2304, 10),
                                       (1, 9216, 5), (4, 64, 5), (3, 129, 1)])
def test_flash_attn(cuda_dev, fa_variant, n, s, heads):
    from streamingt2v_b200 import ops
    Cc = heads * 64
    qkv = _rand((n * s, 3 * Cc), cuda_dev, 1.5, seed=n * 1000 + s)
    out = ops.flash_attn(qkv, n, s, heads)
    torch.cuda.synchronize()
    q, k, v = (t.float().reshape(n, s, heads, 64).permute(0, 2, 1, 3) for t in qkv.chunk(3, dim=1))
    ref = F.scaled_dot_product_attention(q, k, v).permute(0, 2, 1, 3).reshape(n * s, Cc)
    _check(out, ref, f"flash_attn n{n} s{s} h{heads}", rtol=2 ** -6, atol=2e-2)


@pytest.mark.parametrize("s,ramp", [(1024, 6.0), (2304, 3.0), (640, 12.0)])
def test_flash_attn_rising_max(cuda_dev, fa_variant, s, ramp):
    """Key magnitudes grow along the sequence, so the row maxima keep rising by more than 2^8 between key blocks: the
    online softmax must rescale O and l by the new maximum at nearly every block and still match SDPA."""
    from streamingt2v_b200 import ops
    n, heads = 2, 3
    Cc = heads * 64
    g = torch.Generator(device="cpu").manual_seed(s)
    q = torch.randn(n * s, Cc, generator=g) * 2.0
    k = torch.randn(n * s, Cc, generator=g) * (0.1 + ramp * (torch.arange(n * s) % s)[:, None] / s)
    k = k + 0.5 * torch.sign(q)                       # correlate: the large late keys really win the softmax
    v = torch.randn(n * s, Cc, generator=g)
    qkv = torch.cat([q, k, v], 1).to(cuda_dev).to(torch.bfloat16)
    out = ops.flash_attn(qkv, n, s, heads)
    torch.cuda.synchronize()
    qf, kf, vf = (t.float().reshape(n, s, heads, 64).permute(0, 2, 1, 3) for t in qkv.chunk(3, dim=1))
    ref = F.scaled_dot_product_attention(qf, kf, vf).permute(0, 2, 1, 3).reshape(n * s, Cc)
    _check(out, ref, f"flash_attn rising max s{s} ramp{ramp}", rtol=2 ** -6, atol=2e-2)


@pytest.mark.parametrize("b,s,heads,lq,lk,pp", [(2, 64, 5, 8, 8, True), (2, 144, 10, 25, 25, True),
                                                (2, 100, 5, 25, 7, True), (1, 333, 20, 25, 17, False),
                                                (2, 4, 5, 8, 7, True)])
def test_small_attn(cuda_dev, b, s, heads, lq, lk, pp):
    from streamingt2v_b200 import ops
    Cc = heads * 64
    q = _rand((b * lq * s, Cc), cuda_dev, 1.5, seed=1)
    kv_rows = b * lk * (s if pp else 1)
    kv = _rand((kv_rows, 2 * Cc), cuda_dev, 1.5, seed=2)
    k, v = kv[:, :Cc], kv[:, Cc:]  # strided views (as produced by a fused KV projection)
    out = ops.small_attn(q, k, v, b=b, s=s, heads=heads, lq=lq, lk=lk, kv_per_pixel=pp)
    torch.cuda.synchronize()
    qf = q.float().reshape(b, lq, s, heads, 64).permute(0, 2, 3, 1, 4)           # b s h lq d
    if pp:
        kf = k.float().reshape(b, lk, s, heads, 64).permute(0, 2, 3, 1, 4)
        vf = v.float().reshape(b, lk, s, heads, 64).permute(0, 2, 3, 1, 4)
    else:
        kf = k.float().reshape(b, lk, 1, heads, 64).permute(0, 2, 3, 1, 4).expand(b, s, heads, lk, 64)
        vf = v.float().reshape(b, lk, 1, heads, 64).permute(0, 2, 3, 1, 4).expand(b, s, heads, lk, 64)
    ref = F.scaled_dot_product_attention(qf, kf, vf)                              # b s h lq d
    ref = ref.permute(0, 3, 1, 2, 4).reshape(b * lq * s, Cc)
    _check(out, ref, f"small_attn b{b} s{s} h{heads} {lq}x{lk} pp{pp}", rtol=2 ** -7, atol=1e-2)


@pytest.mark.parametrize("n,p,c,eps,silu", [(3, 64, 320, 1e-5, True), (2, 1000, 640, 1e-6, False),
                                            (50, 144, 1280, 1e-5, True), (2, 9216, 960, 1e-5, True),
                                            (2, 300, 2560, 1e-5, True), (1, 7, 1920, 1e-5, False)])
def test_group_norm(cuda_dev, n, p, c, eps, silu):
    from streamingt2v_b200 import ops
    x = (_rand((n * p, c), cuda_dev, 2.0, seed=3).float() + 0.7).to(torch.bfloat16)
    g = torch.randn(c, device=cuda_dev) * 0.2 + 1.0
    b = torch.randn(c, device=cuda_dev) * 0.2
    out = ops.group_norm(x, n, p, g, b, eps, silu=silu)
    torch.cuda.synchronize()
    ref = F.group_norm(x.float().reshape(n, p, c).permute(0, 2, 1), 32, g, b, eps)
    if silu:
        ref = F.silu(ref)
    ref = ref.permute(0, 2, 1).reshape(n * p, c)
    _check(out, ref, f"group_norm n{n} p{p} c{c}", rtol=2 ** -7, atol=1e-2)


@pytest.mark.parametrize("rows,c", [(100, 320), (1000, 640), (77, 1280), (64, 32), (64, 96), (33, 512), (10, 1024)])
def test_layer_norm(cuda_dev, rows, c):
    from streamingt2v_b200 import ops
    x = (_rand((rows, c), cuda_dev, 2.0, seed=4).float() - 0.3).to(torch.bfloat16)
    g = torch.randn(c, device=cuda_dev) * 0.2 + 1.0
    b = torch.randn(c, device=cuda_dev) * 0.2
    out = ops.layer_norm(x, g, b)
    torch.cuda.synchronize()
    ref = F.layer_norm(x.float(), (c,), g, b, 1e-5)
    _check(out, ref, f"layer_norm {rows}x{c}", rtol=2 ** -7, atol=1e-2)
    # with per-frame vector pre-add, residual-stream output and fused SiLU
    rpf = 10
    fvec = torch.randn((rows + rpf - 1) // rpf, c, device=cuda_dev)
    xs = torch.empty_like(x)
    out2 = ops.layer_norm(x, g, b, fvec=fvec, rows_per_frame=rpf, xsum=xs, silu=True)
    torch.cuda.synchronize()
    xsum_ref = x.float() + fvec.repeat_interleave(rpf, 0)[:rows]
    _check(xs, xsum_ref, "layer_norm xsum", rtol=2 ** -8, atol=1e-3)
    ref2 = F.silu(F.layer_norm(xs.float(), (c,), g, b, 1e-5))
    _check(out2, ref2, "layer_norm+fvec+silu", rtol=2 ** -7, atol=1e-2)


def test_glue(cuda_dev):
    from streamingt2v_b200 import ops
    dev = cuda_dev
    # nchw -> nhwc with channel offset, and back
    N, C1, C2, H, W = 6, 4, 4, 8, 16
    a = torch.randn(N, C1, H, W, device=dev)
    b = torch.randn(N, C2, H, W, device=dev)
    dst = torch.zeros(N * H * W, 8, dtype=torch.bfloat16, device=dev)
    ops.nchw_to_nhwc(a, dst, 0)
    ops.nchw_to_nhwc(b[1:4], dst[H * W:4 * H * W], C1)  # sliced frames
    torch.cuda.synchronize()
    ref = torch.cat([a, torch.zeros_like(b)], 1)
    ref[1:4, C1:] = b[1:4]
    ref = ref.permute(0, 2, 3, 1).reshape(N * H * W, 8)
    _check(dst, ref, "nchw_to_nhwc", rtol=2 ** -8, atol=1e-6)
    back = torch.empty(N, 8, H, W, device=dev)
    ops.nhwc_to_nchw(dst, N, 8, H * W, back)
    torch.cuda.synchronize()
    assert torch.equal(back, dst.float().reshape(N, H, W, 8).permute(0, 3, 1, 2))
    # upsample
    x = _rand((3 * 4 * 6, 64), dev, seed=5)
    y = ops.upsample2x(x, 3, 4, 6)
    torch.cuda.synchronize()
    ref = F.interpolate(x.float().reshape(3, 4, 6, 64).permute(0, 3, 1, 2), scale_factor=2, mode="nearest")
    assert torch.equal(y.float().reshape(3, 8, 12, 64), ref.permute(0, 2, 3, 1))
    # timestep embedding
    t = torch.tensor([0.0, 0.3466, -1.5, 24.0, 3.0], device=dev)
    e = ops.timestep_embed(t, 320)
    torch.cuda.synchronize()
    half = 160
    freqs = torch.exp(-math.log(10000.0) * torch.arange(half, device=dev, dtype=torch.float32) / half)
    args = t[:, None] * freqs[None]
    ref = torch.cat([torch.cos(args), torch.sin(args)], -1)
    _check(e, ref, "timestep_embed", rtol=2 ** -8, atol=4e-3)
    # add_silu
    p, q = torch.randn(50, 1280, device=dev), torch.randn(50, 1280, device=dev)
    o = ops.add_silu(p, q)
    torch.cuda.synchronize()
    _check(o, F.silu(p + q), "add_silu", rtol=2 ** -8, atol=1e-3)
    # copy2d / add_rows
    src = _rand((100, 320), dev, seed=6)
    big = torch.zeros(100, 960, dtype=torch.bfloat16, device=dev)
    ops.copy2d(src, big[:, 320:640])
    torch.cuda.synchronize()
    assert torch.equal(big[:, 320:640], src) and big[:, :320].abs().sum() == 0 and big[:, 640:].abs().sum() == 0
    d = _rand((14 * 16, 320), dev, seed=7)
    s_ = _rand((7 * 16, 320), dev, seed=8)
    ref = (d.float() + s_.float().repeat(2, 1))
    ops.add_rows(d, s_)
    torch.cuda.synchronize()
    _check(d, ref, "add_rows", rtol=2 ** -8, atol=1e-3)
    # APM mix
    ctx = torch.randn(4, 17, 1024, device=dev)
    w = torch.randn(1, 17, 3, device=dev) * 0.2
    wb = torch.randn(1, device=dev)
    lg, lb = torch.randn(1024, device=dev) * 0.1 + 1, torch.randn(1024, device=dev) * 0.1
    alpha = torch.tensor(0.6, device=dev)
    o = ops.apm_mix(ctx, w.reshape(17, 3).contiguous(), wb, lg, lb, alpha.reshape(1))
    torch.cuda.synchronize()
    mixed = F.layer_norm(F.conv1d(ctx, w, wb, padding=1), (1024,), lg, lb, 1e-5)
    ref = (ctx[:, :1] + mixed * F.silu(alpha))[:, 0]
    _check(o, ref, "apm_mix", rtol=2 ** -7, atol=1e-2)


def test_frames_to_uint8_matches_reference_torch2np(cuda_dev):
    """Bit-exact (integer output) against the expression of the reference's torch2np
    (lib/farancia/libimage/iimage.py:33-36) on values that cover the clip edges and the golden video of the stage."""
    import os

    import numpy as np
    from streamingt2v_b200 import ops
    g = torch.Generator().manual_seed(0)
    x = (torch.rand(5, 3, 37, 53, generator=g) * 300.0 - 20.0)          # below 0 and above 255 included
    x[0, 0, 0, :8] = torch.tensor([0.0, 255.0, 254.999, 0.999, 1.0, 127.5, -0.0, 255.001])
    ref = (255 * (x.clip(0, 255) - 0) / (255 - 0)).permute(0, 2, 3, 1).to(torch.uint8)
    out = ops.frames_to_uint8(x.to(cuda_dev), 0.0, 255.0)
    torch.cuda.synchronize()
    assert out.dtype == torch.uint8 and out.shape == ref.shape and torch.equal(out.cpu(), ref)
    y = torch.rand(2, 3, 16, 24, generator=g) * 2.4 - 1.2                  # [-1, 1] range variant (IImage default)
    ref2 = (255 * (y.clip(-1, 1) + 1) / 2).permute(0, 2, 3, 1).to(torch.uint8)
    assert torch.equal(ops.frames_to_uint8(y.to(cuda_dev), -1.0, 1.0).cpu(), ref2)
