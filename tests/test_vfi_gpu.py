"""GPU: the EMA-VFI kernels (csrc/vfi.cu, PReLU in the GEMM epilogue) against float64 torch references at the
network's shapes and edges, and B200VFI / interpolate_video against the goldens of the unmodified reference
(oracle/make_golden_vfi.py).

Per-element bounds: bf16 outputs are compared with a bound of one bf16 rounding of the result (2^-8 relative) plus the
fp32 accumulation error; fp32 outputs with a few fp32 ulps of the operand magnitudes.  The network tolerance is stated
relative to the reference's own bf16 discrepancy (the same module under CPU bf16 autocast against fp32, stored in each
golden): B200VFI also computes every conv and linear with bf16 operands, so its error is expected at that scale."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from vfi_refs import ref_warp as _ref_warp, ref_window_attn as _ref_window_attn, warp_bound

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


# ---------------------------------------------------------------------------------------------------------------
# window attention
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w,heads,shift", [(14, 28, 8, 0), (14, 28, 8, 3), (12, 20, 8, 0), (12, 20, 8, 3),
                                             (6, 10, 16, 0), (6, 10, 16, 3), (7, 14, 16, 3), (9, 5, 8, 3)])
def test_window_attn(cuda_dev, h, w, heads, shift):
    from streamingt2v_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(h * 100 + w + shift)
    pairs, C, Cm = 2, heads * 32, heads * 8
    T = 2 * pairs * h * w
    qkv = (torch.randn((T + 1, 3 * C), generator=g) * 1.5).to(torch.bfloat16)
    ce = torch.randn((h * w + 1, Cm), generator=g).to(torch.bfloat16)
    out = torch.full((T, C), float("nan"), dtype=torch.bfloat16, device=cuda_dev)
    mot = torch.full((T, Cm), float("nan"), dtype=torch.bfloat16, device=cuda_dev)
    ops.vfi_window_attn(qkv.to(cuda_dev), ce.to(cuda_dev), pairs=pairs, h=h, w=w, heads=heads, shift=shift, out=out,
                        motion=mot)
    torch.cuda.synchronize()
    rx, rm = _ref_window_attn(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], ce, pairs, h, w, heads, shift)
    for got, ref, name in ((out, rx, "attn@v"), (mot, rm, "motion")):
        got = got.double().cpu()
        assert torch.isfinite(got).all(), name
        bound = 2.0 ** -8 * ref.abs() + 2e-4 * (1 + ref.abs())
        err = (got - ref).abs()
        assert (err <= bound).all(), f"{name}: worst err/bound {(err / bound).max():.3f}"


# ---------------------------------------------------------------------------------------------------------------
# warp, resize
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,c,h,w,bf16", [(2, 3, 96, 160, False), (2, 32, 48, 80, True), (2, 512, 6, 10, True),
                                          (2, 3, 720, 1280, False)])
def test_warp(cuda_dev, n, c, h, w, bf16):
    """Flows up to ~1.5 image sizes, so many samples fall outside the image (border clamp); bf16 inputs are channel-last
    views written into a column slice of a wider buffer (the Unet concat)."""
    from streamingt2v_b200 import ops
    g = torch.Generator().manual_seed(c + h)
    x = torch.rand((n, c, h, w), generator=g)
    flow = (torch.rand((n, 2, h, w), generator=g) - 0.5) * torch.tensor([3.0 * w, 3.0 * h]).view(1, 2, 1, 1)
    flow[:, :, : h // 2] *= 0.01                                  # and small sub-pixel flows in the upper half
    if bf16:
        x = x.to(torch.bfloat16)
        rows = x.permute(0, 2, 3, 1).contiguous().view(-1, c).to(cuda_dev)
        xin = rows.as_strided((n, c, h, w), (h * w * c, 1, w * c, c))
        buf = torch.full((n * h * w, c + 16), float("nan"), dtype=torch.bfloat16, device=cuda_dev)
        sl = buf[:, 8:8 + c]
        out = sl.as_strided((n, c, h, w), (h * w * buf.stride(0), 1, w * buf.stride(0), buf.stride(0)))
    else:
        xin = x.to(cuda_dev)
        out = torch.full((n, c, h, w), float("nan"), device=cuda_dev)
    ops.vfi_warp(xin, flow.to(cuda_dev), out)
    torch.cuda.synchronize()
    ref = _ref_warp(x.double(), flow)
    got = out.double().cpu()
    tol = warp_bound(ref, flow, bf16)                          # derived in tests/vfi_refs.py
    err = (got - ref).abs()
    assert (err <= tol).all(), f"max err {err.max():.3g}"
    if bf16:
        assert torch.isnan(buf[:, :8]).all() and torch.isnan(buf[:, 8 + c:]).all()


@pytest.mark.parametrize("log2", [-2, -1, 1, 2])
@pytest.mark.parametrize("mode", ["fp32", "bf16", "acc"])
def test_resize(cuda_dev, log2, mode):
    from streamingt2v_b200 import ops
    g = torch.Generator().manual_seed(log2 + 10)
    n, c, h, w = 2, 5, 48, 80
    x = torch.randn((n, c, h, w), generator=g) * 10
    f = 2.0 ** log2
    mul = 0.5 * f if mode != "bf16" else 1.0
    ref = F.interpolate(x.double(), scale_factor=f, mode="bilinear", align_corners=False) * mul
    ho, wo = ref.shape[2:]
    if mode == "bf16":
        out = torch.zeros((n, ho, wo, c + 3), dtype=torch.bfloat16, device=cuda_dev)[..., :c].permute(0, 3, 1, 2)
    else:
        base = torch.randn((n, c, ho, wo), generator=g)
        out = base.clone().to(cuda_dev)
        if mode == "acc":
            ref = ref + base.double()
    ops.vfi_resize(x.to(cuda_dev), out, log2, mul, accumulate=(mode == "acc"))
    torch.cuda.synchronize()
    got = out.double().cpu()
    tol = (2.0 ** -8 * ref.abs() if mode == "bf16" else 0) + 4e-6 * (ref.abs() + 10)
    err = (got - ref).abs()
    assert (err <= tol).all(), f"max err {err.max():.3g}"


# ---------------------------------------------------------------------------------------------------------------
# depthwise conv + GELU, head gather, merge
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c,h,w", [(1024, 14, 28), (2048, 7, 14), (1024, 12, 20)])
def test_dwconv_gelu(cuda_dev, c, h, w):
    from streamingt2v_b200 import ops
    g = torch.Generator().manual_seed(c + h)
    x = torch.randn((4, h, w, c), generator=g).to(torch.bfloat16)
    wt = torch.randn((c, 1, 3, 3), generator=g) / 3
    b = torch.randn((c,), generator=g) * 0.1
    out = ops.vfi_dwconv_gelu(x.to(cuda_dev), wt.reshape(c, 9).t().contiguous().to(cuda_dev), b.to(cuda_dev))
    torch.cuda.synchronize()
    ref = F.gelu(F.conv2d(x.double().permute(0, 3, 1, 2), wt.double(), b.double(), padding=1, groups=c))
    ref = ref.permute(0, 2, 3, 1).reshape(-1, c)
    err = (out.double().cpu() - ref).abs()
    bound = 2.0 ** -8 * ref.abs() + 1e-5
    assert (err <= bound).all(), f"worst err/bound {(err / bound).max():.3f}"


@pytest.mark.parametrize("c,h,w", [(512, 7, 14), (256, 12, 20)])
def test_head_gather(cuda_dev, c, h, w):
    from streamingt2v_b200 import ops
    g = torch.Generator().manual_seed(c)
    pairs = 2
    mf = torch.randn((2 * pairs * h * w, c), generator=g).to(torch.bfloat16)
    af = torch.randn((2 * pairs * h * w, c), generator=g).to(torch.bfloat16)
    out = torch.full((pairs * 16 * h * w, c // 4 + 8), float("nan"), dtype=torch.bfloat16, device=cuda_dev)
    ops.vfi_head_gather(mf.to(cuda_dev), af.to(cuda_dev), pairs=pairs, h=h, w=w, out=out)
    torch.cuda.synchronize()
    m4 = mf.double().view(2 * pairs, h, w, c).permute(0, 3, 1, 2)
    a4 = af.double().view(2 * pairs, h, w, c).permute(0, 3, 1, 2)
    cat = torch.cat([0.5 * m4[:pairs], 0.5 * m4[pairs:], a4[:pairs], a4[pairs:]], 1)
    ref = F.pixel_shuffle(F.pixel_shuffle(cat, 2), 2).permute(0, 2, 3, 1).reshape(-1, c // 4)
    assert torch.equal(out[:, :c // 4].double().cpu(), ref)
    assert torch.isnan(out[:, c // 4:]).all()


def test_merge(cuda_dev):
    from streamingt2v_b200 import ops
    g = torch.Generator().manual_seed(7)
    H, W = 48, 80
    w0, w1 = torch.rand((2, 3, H, W), generator=g), torch.rand((2, 3, H, W), generator=g)
    fm = torch.randn((2, 5, H, W), generator=g) * 3
    res = torch.randn((2 * H * W, 3), generator=g) * 3
    pred = torch.empty((1, 3, H, W), device=cuda_dev)
    frame = torch.empty((H, W, 3), dtype=torch.uint8, device=cuda_dev)
    ops.vfi_merge(w0.to(cuda_dev), w1.to(cuda_dev), fm.to(cuda_dev), res.to(cuda_dev), pred=pred, frame=frame)
    torch.cuda.synchronize()
    m = torch.sigmoid(fm[:, 4:5].double())
    r = torch.sigmoid(res.double().view(2, H, W, 3).permute(0, 3, 1, 2)) * 2 - 1
    p = torch.clamp(w0.double() * m + w1.double() * (1 - m) + r, 0, 1)
    ref = (p[0] + p[1].flip(1).flip(2)) / 2
    assert (pred[0].double().cpu() - ref).abs().max() <= 1e-6
    ref8 = (pred[0].cpu().numpy().transpose(1, 2, 0) * 255.0).astype(np.uint8)[:, :, ::-1]
    assert np.array_equal(frame.cpu().numpy(), ref8)


# ---------------------------------------------------------------------------------------------------------------
# PReLU in the GEMM epilogue
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("schedule", [0, 1])
@pytest.mark.parametrize("M,N,K,out_fp32", [(300, 5, 128, True), (300, 72, 136, False), (1000, 136, 88, False),
                                            (129, 256, 64, False), (257, 40, 32, True)])
def test_prelu_epilogue(cuda_dev, schedule, M, N, K, out_fp32):
    from streamingt2v_b200 import ops
    from streamingt2v_b200._lib import ACT_PRELU
    g = torch.Generator().manual_seed(M + N)
    x = torch.randn((M, K), generator=g).to(torch.bfloat16)
    wt = (torch.randn((N, K), generator=g) / K ** 0.5).to(torch.bfloat16)
    b = torch.randn((N,), generator=g) * 0.1
    a = torch.rand((N,), generator=g) - 0.3                   # negative, zero-ish and positive slopes
    res = torch.randn((M, N), generator=g).to(torch.bfloat16)
    prev = ops.gemm_schedule(schedule)
    try:
        y = ops.linear(x.to(cuda_dev), wt[None].contiguous().to(cuda_dev), b.to(cuda_dev), act=ACT_PRELU,
                       slope=a.to(cuda_dev), out_fp32=out_fp32,
                       res1=None if out_fp32 else res.to(cuda_dev), s1=0.5)
        torch.cuda.synchronize()
    finally:
        ops.gemm_schedule(prev)
    v = x.double() @ wt.double().t() + b.double()
    ref = torch.where(v > 0, v, a.double() * v)
    if not out_fp32:
        ref = ref + 0.5 * res.double()
    err = (y.double().cpu() - ref).abs()
    bound = (0 if out_fp32 else 2.0 ** -8) * ref.abs() + 1e-4 * (1 + v.abs())
    assert (err <= bound).all(), f"worst err/bound {(err / bound).max():.3f}"


def test_prelu_conv_and_deconv(cuda_dev):
    """conv3x3 + PReLU and the 4-phase ConvTranspose2d(4, 2, 1) + PReLU writing into a column slice, against fp64."""
    from streamingt2v_b200 import ops
    from streamingt2v_b200._lib import ACT_PRELU
    from streamingt2v_b200.packing import pack_conv3x3
    from streamingt2v_b200.vfi import pack_deconv
    g = torch.Generator().manual_seed(3)
    n, h, w, cin, cout = 2, 12, 20, 96, 64
    x = torch.randn((n, h, w, cin), generator=g).to(torch.bfloat16)
    wc = (torch.randn((cout, cin, 3, 3), generator=g) / (9 * cin) ** 0.5).to(torch.bfloat16).float()
    wd = (torch.randn((cin, cout, 4, 4), generator=g) / (4 * cin) ** 0.5).to(torch.bfloat16).float()
    b = torch.randn((cout,), generator=g) * 0.1
    a = torch.rand((cout,), generator=g)
    xd = x.to(cuda_dev)
    y = ops.conv3x3(xd, pack_conv3x3(wc, cuda_dev), b.to(cuda_dev), act=ACT_PRELU, slope=a.to(cuda_dev))
    buf = torch.full((n * 4 * h * w, cout + 32), float("nan"), dtype=torch.bfloat16, device=cuda_dev)
    ops.conv_transpose4x4_s2(xd, pack_deconv(wd, cuda_dev), b.to(cuda_dev), act=ACT_PRELU, slope=a.to(cuda_dev),
                             out=buf[:, :cout])
    torch.cuda.synchronize()
    xc = x.double().permute(0, 3, 1, 2)
    for got, v in ((y, F.conv2d(xc, wc.double(), b.double(), padding=1)),
                   (buf[:, :cout], F.conv_transpose2d(xc, wd.double(), b.double(), stride=2, padding=1))):
        ref = torch.where(v > 0, v, a.double().view(1, -1, 1, 1) * v).permute(0, 2, 3, 1).reshape(-1, cout)
        err = (got.double().cpu() - ref).abs()
        bound = 2.0 ** -8 * ref.abs() + 1e-4 * (1 + ref.abs())
        assert (err <= bound).all(), f"worst err/bound {(err / bound).max():.3f}"
    assert torch.isnan(buf[:, cout:]).all()


def test_strided_dilated_conv(cuda_dev):
    """CrossScalePatchEmbed's stride-4 / stride-8 dilated 3x3 convs through the strided TMA view."""
    from streamingt2v_b200 import ops
    from streamingt2v_b200.packing import pack_conv3x3
    g = torch.Generator().manual_seed(5)
    for s, cin, dils in ((4, 64, (1, 2)), (8, 32, (1, 2, 3, 4))):
        x = torch.randn((4, 96, 160, cin), generator=g).to(torch.bfloat16)
        for d in dils:
            wc = (torch.randn((32, cin, 3, 3), generator=g) / (9 * cin) ** 0.5).to(torch.bfloat16).float()
            b = torch.randn((32,), generator=g) * 0.1
            y = ops.conv3x3_strided(x.to(cuda_dev), pack_conv3x3(wc, cuda_dev), b.to(cuda_dev), stride=s, dilation=d)
            torch.cuda.synchronize()
            ref = F.conv2d(x.double().permute(0, 3, 1, 2), wc.double(), b.double(), stride=s, padding=d, dilation=d)
            ref = ref.permute(0, 2, 3, 1).reshape(-1, 32)
            err = (y.double().cpu() - ref).abs()
            bound = 2.0 ** -8 * ref.abs() + 1e-4 * (1 + ref.abs())
            assert (err <= bound).all(), f"s{s} d{d}: worst err/bound {(err / bound).max():.3f}"


# ---------------------------------------------------------------------------------------------------------------
# the network against the reference's goldens
# ---------------------------------------------------------------------------------------------------------------
# Tolerance: TOL_FACTOR x the reference's own CPU bf16-autocast discrepancy of the same golden, for both the mean and
# the max absolute error of the [0, 1] prediction.
TOL_FACTOR = 4.0


def _golden(name):
    return np.load(os.path.join(GOLDEN, name))


@pytest.fixture(scope="module")
def vfi_net(cuda_dev):
    from streamingt2v_b200.vfi import B200VFI, seeded_state_dict
    d = _golden("vfi_96x160.npz")
    sd = seeded_state_dict(int(d["seed"]))
    sums = np.array([float(sd[k].double().sum()) for k in d["weight_keys"]])
    assert np.array_equal(sums, d["weight_sums"]), "the seeded weights differ from those the goldens were made with"
    return B200VFI(sd, cuda_dev)


def _bgr(frame, dev):
    return torch.from_numpy((frame / 255.)[:, :, ::-1].copy()).permute(2, 0, 1)[None].float().to(dev)


@pytest.mark.parametrize("name", ["vfi_112x224.npz", "vfi_96x160.npz"])
def test_b200vfi_inference_golden(cuda_dev, vfi_net, name):
    d = _golden(name)
    pred = vfi_net.inference(_bgr(d["frame0"], cuda_dev), _bgr(d["frame1"], cuda_dev))
    torch.cuda.synchronize()
    ref = torch.from_numpy(d["pred"]).double()
    err = (pred.double().cpu() - ref).abs()
    mean_b, max_b = float(d["bf16_mean_err"]), float(d["bf16_max_err"])
    print(f"{name}: mean err {err.mean():.4g} ({err.mean() / mean_b:.2f} x ref bf16), max err {err.max():.4g} "
          f"({err.max() / max_b:.2f} x ref bf16)")
    assert torch.isfinite(pred).all()
    assert err.mean() <= TOL_FACTOR * mean_b and err.max() <= TOL_FACTOR * max_b


@pytest.mark.parametrize("dest", [3, 4])
def test_interpolate_video_golden(cuda_dev, vfi_net, dest):
    from streamingt2v_b200.vfi import interpolate_video
    d = _golden("vfi_96x160.npz")
    frames = [d["frame0"], d["frame1"]]
    if dest == 3:
        frames.append(np.zeros_like(d["frame0"]))            # past dest // 2 + 1 frames: dropped
    video = torch.from_numpy(np.stack(frames))
    out = interpolate_video(video, dest, vfi_net)
    torch.cuda.synchronize()
    assert out.shape == (dest, 96, 160, 3) and out.device.type == "cuda" and out.dtype == torch.uint8
    o = out.cpu().numpy()
    assert np.array_equal(o[0], d["frame0"]) and np.array_equal(o[2], d["frame1"])
    if dest == 4:
        assert np.array_equal(o[3], d["frame1"])
    diff = np.abs(o[1].astype(np.int32) - d["mid"].astype(np.int32))
    print(f"dest {dest}: midpoint uint8 diff mean {diff.mean():.4f} max {diff.max()}")
    assert diff.max() <= math.ceil(255 * TOL_FACTOR * float(d["bf16_max_err"])) + 1
