"""GPU parity of the multi-tap wgmma GEMM (b200svd_gemm) against a plain PyTorch fp32 reference of the same op
(floating-point kernel: bf16 operands, fp32 accumulate).  Tolerances: inputs are identical bf16 values on both
sides, so the only differences are fp32 summation order and the final bf16 rounding of the output:
|err| <= 2^-8 * |ref| + small abs (one bf16 ulp = 2^-8 relative)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, params=[0, 1, 3], ids=["1sm", "2sm", "4cl"])
def pair_mode(request, cuda_dev):
    """Every case runs under each CTA-pair mode the ABI accepts (on sm_90 all of them launch single-CTA tiles)."""
    from streamingt2v_b200 import ops
    prev = ops.gemm_pair_mode(request.param)
    yield request.param
    ops.gemm_pair_mode(prev)


def _check(out, ref, name, rtol=2 ** -7, atol=2e-2):
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


@pytest.mark.parametrize("M,K,N,bn", [(256, 64, 32, 0), (300, 320, 320, 0), (1000, 320, 960, 0), (128, 1280, 1280, 128),
                                      (777, 640, 640, 64), (50, 768, 1280, 0), (4096, 320, 320, 160)])
def test_linear(cuda_dev, M, K, N, bn):
    from streamingt2v_b200 import ops, packing
    x = _rand((M, K), cuda_dev, seed=1)
    w = _rand((N, K), cuda_dev, K ** -0.5, seed=2)
    b = torch.randn(N, device=cuda_dev)
    out = ops.linear(x, packing.pack_linear(w, cuda_dev), b, bn=bn)
    torch.cuda.synchronize()
    ref = x.float() @ w.float().t() + b
    _check(out, ref, f"linear M{M} K{K} N{N} bn{bn}")


@pytest.mark.parametrize("M,K,N,bn", [(1357, 1280, 1280, 256), (384, 640, 640, 160), (129, 1280, 512, 256),
                                      (128 * 149 * 2 + 5, 320, 320, 160), (5000, 1280, 1000, 256)])
def test_wide_tiles_epilogue(cuda_dev, M, K, N, bn):
    """160/256-wide tiles (CTA pairs in the 2sm run): odd M-tile counts, ragged N, several tiles per CTA, all
    epilogue operands."""
    from streamingt2v_b200 import ops, packing
    rpf = 64
    x = _rand((M, K), cuda_dev, seed=1)
    w = _rand((N, K), cuda_dev, K ** -0.5, seed=2)
    b = torch.randn(N, device=cuda_dev)
    fvec = torch.randn((M + rpf - 1) // rpf, N, device=cuda_dev)
    r1 = _rand((M, N), cuda_dev, seed=3)
    r2 = _rand((M, N), cuda_dev, seed=4)
    out = ops.linear(x, packing.pack_linear(w, cuda_dev), b, act=ops.ACT_GELU, fvec=fvec, rows_per_frame=rpf,
                     s_acc=0.5, res1=r1, s1=0.7, res2=r2, s2=-0.5, bn=bn)
    torch.cuda.synchronize()
    v = x.float() @ w.float().t() + b + fvec.repeat_interleave(rpf, 0)[:M]
    ref = 0.5 * F.gelu(v) + 0.7 * r1.float() - 0.5 * r2.float()
    _check(out, ref, f"wide tile M{M} K{K} N{N} bn{bn}")


@pytest.mark.parametrize("M,K,N,bn", [(1357, 1280, 1280, 256), (384, 640, 640, 160), (2000, 1280, 640, 320),
                                      (128 * 149 * 2 + 5, 320, 320, 320), (5000, 1280, 1008, 256), (777, 640, 640, 128),
                                      (3000, 960, 960, 320), (4096, 2560, 1280, 0), (640, 320, 960, 0)])
@pytest.mark.parametrize("operands", ["all", "bias", "none", "res1"])
def test_lean_epilogue(cuda_dev, M, K, N, bn, operands):
    """Activation-free launches take the specialised packed-math epilogue (mtgemm EPI = 2): bias, per-frame vector,
    s_acc and both residuals in every combination the network uses; 128/160/256-wide tiles and the 320-wide 2-SM tile
    (two N = 160 MMAs per k step, single-buffered accumulator), ragged M / N edges, several tiles per CTA."""
    from streamingt2v_b200 import ops, packing
    rpf = 64
    x = _rand((M, K), cuda_dev, seed=1)
    w = _rand((N, K), cuda_dev, K ** -0.5, seed=2)
    b = torch.randn(N, device=cuda_dev)
    fvec = torch.randn((M + rpf - 1) // rpf, N, device=cuda_dev)
    r1 = _rand((M, N), cuda_dev, seed=3)
    r2 = _rand((M, N), cuda_dev, seed=4)
    v = x.float() @ w.float().t()
    wp = packing.pack_linear(w, cuda_dev)
    if operands == "all":
        out = ops.linear(x, wp, b, fvec=fvec, rows_per_frame=rpf, s_acc=0.5, res1=r1, s1=0.7, res2=r2, s2=-0.5, bn=bn)
        ref = 0.5 * (v + b + fvec.repeat_interleave(rpf, 0)[:M]) + 0.7 * r1.float() - 0.5 * r2.float()
    elif operands == "bias":
        out = ops.linear(x, wp, b, bn=bn)
        ref = v + b
    elif operands == "res1":
        out = ops.linear(x, wp, b, res1=r1, s1=1.0, bn=bn)
        ref = v + b + r1.float()
    else:
        out = ops.linear(x, wp, None, bn=bn)
        ref = v
    torch.cuda.synchronize()
    _check(out, ref, f"lean epilogue M{M} K{K} N{N} bn{bn} {operands}")


@pytest.mark.parametrize("Nf,H,W,Cin,Cout", [(4, 24, 64, 320, 320), (3, 18, 32, 640, 640), (2, 36, 64, 960, 320)])
def test_conv3x3_320_wide_tile(cuda_dev, monkeypatch, Nf, H, W, Cin, Cout):
    """3x3 convolutions on the 320-wide 2-SM tile (forced), bias + residual, against F.conv2d."""
    from streamingt2v_b200 import ops, packing
    x = _rand((Nf, H, W, Cin), cuda_dev, seed=1)
    wt = _rand((Cout, Cin, 3, 3), cuda_dev, (9 * Cin) ** -0.5, seed=2)
    b = torch.randn(Cout, device=cuda_dev)
    r1 = _rand((Nf * H * W, Cout), cuda_dev, seed=3)
    out = ops.conv3x3(x, packing.pack_conv3x3(wt, cuda_dev), b, res1=r1, s1=1.0, bn=320)
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), b, padding=1).permute(0, 2, 3, 1).reshape(-1, Cout)
    _check(out, ref + r1.float(), f"conv3x3 bn320 {Nf}x{H}x{W} {Cin}->{Cout}", rtol=2 ** -7, atol=3e-2)


def test_linear_epilogue(cuda_dev):
    from streamingt2v_b200 import ops, packing
    M, K, N, rpf = 640, 320, 320, 64
    x = _rand((M, K), cuda_dev, seed=1)
    w = _rand((N, K), cuda_dev, K ** -0.5, seed=2)
    b = torch.randn(N, device=cuda_dev)
    fvec = torch.randn(M // rpf, N, device=cuda_dev)
    r1 = _rand((M, N), cuda_dev, seed=3)
    r2 = _rand((M, N), cuda_dev, seed=4)
    out = ops.linear(x, packing.pack_linear(w, cuda_dev), b, act=ops.ACT_SILU, fvec=fvec, rows_per_frame=rpf,
                     s_acc=0.3, res1=r1, s1=0.7, res2=r2, s2=-0.5)
    torch.cuda.synchronize()
    v = x.float() @ w.float().t() + b + fvec.repeat_interleave(rpf, 0)
    ref = 0.3 * F.silu(v) + 0.7 * r1.float() - 0.5 * r2.float()
    _check(out, ref, "linear+epilogue")
    out32 = ops.linear(x, packing.pack_linear(w, cuda_dev), b, out_fp32=True)
    torch.cuda.synchronize()
    _check(out32, x.float() @ w.float().t() + b, "linear fp32 out", rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("K,F2", [(320, 2560), (64, 512), (128, 1024)])
def test_geglu(cuda_dev, K, F2):
    from streamingt2v_b200 import ops, packing
    M = 500
    x = _rand((M, K), cuda_dev, seed=1)
    w = _rand((F2, K), cuda_dev, K ** -0.5, seed=2)
    b = torch.randn(F2, device=cuda_dev) * 0.1
    wp, bp, bn = packing.pack_geglu(w, b, cuda_dev)
    out = ops.linear(x, wp, bp, act=ops.ACT_GEGLU, bn=bn)
    torch.cuda.synchronize()
    h = x.float() @ w.float().t() + b
    a, g = h.chunk(2, dim=-1)
    _check(out, a * F.gelu(g), f"geglu K{K} F2{F2}")


@pytest.mark.parametrize("N,H,W,Cin,Cout", [(2, 8, 8, 64, 64), (3, 9, 16, 128, 64), (2, 18, 32, 320, 320),
                                            (5, 4, 4, 64, 128), (16, 2, 2, 256, 256), (1, 72, 128, 64, 32),
                                            (2, 16, 16, 8, 64), (2, 12, 20, 96, 96)])
def test_conv3x3(cuda_dev, N, H, W, Cin, Cout):
    from streamingt2v_b200 import ops, packing
    x = _rand((N, H, W, Cin), cuda_dev, seed=1)
    w = _rand((Cout, Cin, 3, 3), cuda_dev, (9 * Cin) ** -0.5, seed=2)
    b = torch.randn(Cout, device=cuda_dev)
    out = ops.conv3x3(x, packing.pack_conv3x3(w, cuda_dev), b)
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b, padding=1).permute(0, 2, 3, 1).reshape(-1, Cout)
    _check(out, ref, f"conv3x3 N{N} {H}x{W} {Cin}->{Cout}")


@pytest.mark.parametrize("N,H,W,Cin,Cout", [(2, 8, 8, 64, 64), (3, 18, 32, 128, 128), (2, 72, 128, 32, 96),
                                            (16, 4, 4, 64, 64), (1, 36, 64, 320, 320)])
def test_conv3x3_s2(cuda_dev, N, H, W, Cin, Cout):
    from streamingt2v_b200 import ops, packing
    x = _rand((N, H, W, Cin), cuda_dev, seed=1)
    w = _rand((Cout, Cin, 3, 3), cuda_dev, (9 * Cin) ** -0.5, seed=2)
    b = torch.randn(Cout, device=cuda_dev)
    out = ops.conv3x3_s2(x, packing.pack_conv3x3(w, cuda_dev), b)
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b, padding=1, stride=2).permute(0, 2, 3, 1).reshape(-1, Cout)
    _check(out, ref, f"conv3x3_s2 N{N} {H}x{W} {Cin}->{Cout}")


@pytest.mark.parametrize("B,T,P,C", [(2, 8, 64, 64), (2, 25, 144, 128), (1, 7, 4, 256), (2, 25, 1024, 320)])
def test_tconv3(cuda_dev, B, T, P, C):
    from streamingt2v_b200 import ops, packing
    x = _rand((B, T, P, C), cuda_dev, seed=1)
    w = _rand((C, C, 3, 1, 1), cuda_dev, (3 * C) ** -0.5, seed=2)
    b = torch.randn(C, device=cuda_dev)
    r1 = _rand((B * T * P, C), cuda_dev, seed=5)
    out = ops.tconv3(x, packing.pack_tconv3(w, cuda_dev), b, res1=r1, s1=1.0, s_acc=0.4)
    torch.cuda.synchronize()
    x5 = x.float().permute(0, 3, 1, 2)[..., None]  # b c t p 1
    ref = F.conv3d(x5, w.float(), b, padding=(1, 0, 0))[..., 0].permute(0, 2, 3, 1).reshape(-1, C)
    ref = 0.4 * ref + r1.float()
    _check(out, ref, f"tconv3 B{B} T{T} P{P} C{C}")


@pytest.mark.parametrize("kind,shape,p_rows", [("conv", (6, 24, 64, 320), "frame"), ("conv", (4, 36, 64, 640), "video"),
                                                 ("tconv", (2, 5, 640, 320), "video"), ("linear", (4096, 320), 512),
                                                 ("conv", (3, 24, 40, 320), "frame")])
def test_groupnorm_statistics_from_the_gemm_epilogue(cuda_dev, monkeypatch, kind, shape, p_rows):
    """gn_rows: the GEMM epilogue leaves per-quadrant partial sums of its (bf16-rounded) output and group_norm reduces
    those instead of reading the activation.  Must agree with the statistics pass over the stored tensor."""
    from streamingt2v_b200 import ops, packing
    monkeypatch.setattr(ops, "GN_FUSE", True)                     # the runtime default leaves the fusion off
    g = torch.Generator().manual_seed(1)
    if kind == "conv":
        N, H, W, Cc = shape
        x = (torch.randn(shape, generator=g) * 1.3 + 0.2).to(cuda_dev).to(torch.bfloat16)
        wt = packing.pack_conv3x3(torch.randn(Cc, Cc, 3, 3, generator=g) * (9 * Cc) ** -0.5, cuda_dev)
        n, p = (N, H * W) if p_rows == "frame" else (1, N * H * W)
        run = lambda **kw: ops.conv3x3(x, wt, None, **kw)  # noqa: E731
    elif kind == "tconv":
        B, T, P, Cc = shape
        x = (torch.randn(shape, generator=g) * 1.3 + 0.2).to(cuda_dev).to(torch.bfloat16)
        wt = packing.pack_tconv3(torch.randn(Cc, Cc, 3, 1, 1, generator=g) * (3 * Cc) ** -0.5, cuda_dev)
        n, p = B, T * P
        run = lambda **kw: ops.tconv3(x, wt, None, **kw)  # noqa: E731
    else:
        M, Cc = shape
        x = (torch.randn(shape, generator=g) * 1.3 + 0.2).to(cuda_dev).to(torch.bfloat16)
        wt = packing.pack_linear(torch.randn(Cc, Cc, generator=g) * Cc ** -0.5, cuda_dev)
        n, p = M // p_rows, p_rows
        run = lambda **kw: ops.linear(x, wt, None, **kw)  # noqa: E731
    gamma = torch.randn(Cc, device=cuda_dev) * 0.2 + 1.0
    beta = torch.randn(Cc, device=cuda_dev) * 0.2
    y = run(gn_rows=p)
    assert getattr(y, "_b200_gn", None) is not None, "launch geometry was expected to be fusable"
    y_plain = run()
    assert torch.equal(y, y_plain)                                 # the GEMM result itself is unchanged
    sums_f = torch.empty((n, 32, 2), dtype=torch.float64, device=cuda_dev)
    sums_p = torch.empty((n, 32, 2), dtype=torch.float64, device=cuda_dev)
    out_f = ops.group_norm(y, n, p, gamma, beta, 1e-5, silu=True, sums=sums_f)
    out_p = ops.group_norm(y_plain, n, p, gamma, beta, 1e-5, silu=True, sums=sums_p)
    torch.cuda.synchronize()
    rel = ((sums_f - sums_p).abs() / sums_p.abs().clamp_min(1e-3)).max().item()
    print(f"gn partials {kind} {shape}: max rel diff of the group sums {rel:.3e}")
    assert rel < 1e-5
    assert (out_f.float() - out_p.float()).abs().max().item() <= 2e-2
    # deterministic
    y2 = run(gn_rows=p)
    s2 = torch.empty_like(sums_f)
    ops.group_norm(y2, n, p, gamma, beta, 1e-5, silu=True, sums=s2)
    assert torch.equal(s2, sums_f)
