"""Edges of the wgmma GEMM and attention kernels at the operand layouts the network uses, against float64 references.

Guard bands.  Operands and outputs live inside larger buffers filled with NaN: NaN rows before and after, and NaN
columns past the leading dimension where the API allows a stride (contiguous operands are slices of a flat NaN
buffer).  A read outside an operand multiplies a NaN (even by 0) into some output; after a launch every element of
the output view must be finite and every element outside it bitwise unchanged, which catches both unwritten and
stray writes.  All bases are 16-byte aligned, leading dims and pad widths multiples of 8 elements.

References are float64 on the exact bf16 values the kernels read; every element is bounded by the arithmetic:
  GEMM / conv, bf16 output   |out - ref| <= 2^-8 |ref| + 2^-12 rms(ref)
  GEMM / conv, fp32 output   |out - ref| <= 2^-20 |ref| + 2^-12 rms(ref)
  2^-8 is bf16's unit roundoff (round to nearest); 2^-20 leaves the fp32 epilogue (bias, fvec, scale, residuals:
  a few roundings of 2^-24) a factor of 8.  2^-12 rms(ref) covers the fp32 accumulation over K (a sum of K products
  in fp32 drifts by ~sqrt(K) 2^-24 of the terms' magnitude, far below it for every K here).  SiLU / GELU / GEGLU add
  s_acc 2^-16 |pre-activation| (times |value| for GEGLU): gelu_fast uses the Abramowitz-Stegun 7.1.25 erf with
  |error| <= 2.5e-5 < 2^-15, so |gelu error| <= 2^-16 |x|, and silu_fast (__expf, __fdividef) is within 2^-18 |x|.
  Attention                  |out - ref| <= 2^-8 |ref| + 2^-7 (softmax(Q K^T) |V|)
  P is rounded to bf16 before the P V product (2^-8 relative per term, doubled for margin); the second term is a
  second float64 attention with |V|.
Aggregate: the relative L2 error of the whole output is at most 2^-8 (GEMM / conv) or 2^-7 (attention).

Exact probes use small integers (|v| < 256, exact in bf16), so their results are compared with torch.equal or
against an exact value.  Every random case also runs its kernel twice and requires bitwise equal results."""
import math

import pytest
import torch
import torch.nn.functional as F

from guard_bands import Guarded, _check_bound

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------------
# guard bands (tests/guard_bands.py)
# ---------------------------------------------------------------------------------------------------------------------
def _out(shape, dtype, dev, **kw):
    return Guarded(shape, dtype, dev, **kw).snapshot()


def _rand(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g, dtype=torch.float64) * scale)


def _bf(t, dev):
    return t.to(dev, torch.bfloat16)


def _small_ints(t):
    assert t.abs().max().item() < 256, "probe values must stay exact in bf16"
    return t


# ---------------------------------------------------------------------------------------------------------------------
# bounds
# ---------------------------------------------------------------------------------------------------------------------
def _gemm_bound(ref, fp32, act_term=None):
    rms = ref.pow(2).mean().sqrt()
    b = (2 ** -20 if fp32 else 2 ** -8) * ref.abs() + 2 ** -12 * rms
    if act_term is not None:
        b = b + act_term
    return b


def _gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


# ---------------------------------------------------------------------------------------------------------------------
# GEMM: exact index probe
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,N,K,bn,fp32", [(333, 1000, 200, 0, False), (130, 300, 328, 128, False),
                                          (2, 777, 136, 0, True), (257, 320, 320, 160, False),
                                          (129, 96, 72, 32, True), (200, 200, 520, 64, False),
                                          (1000, 1280, 1280, 256, False)])
def test_gemm_index_probe(cuda_dev, M, N, K, bn, fp32):
    """W row n is one-hot at column f(n) = perm(n mod K): out[m, n] == A[m, f(n)] exactly, for ragged M / N, several
    N tiles and K over several 64-wide blocks (the last one ragged where K % 64 != 0).  A sits in a NaN guard band
    (columns past K, rows around M); the weights are a slice of a flat NaN buffer."""
    from streamingt2v_b200 import ops
    dev = cuda_dev
    m = torch.arange(M, dtype=torch.float64)[:, None]
    k = torch.arange(K, dtype=torch.float64)[None]
    # the k-block term keeps columns 251 apart (equal under the first two terms) distinct
    a_vals = _small_ints(torch.remainder(m * 7 + k * 13 + torch.div(k, 64, rounding_mode="floor") * (m % 5 + 3), 251)
                         - 125)
    A = Guarded((M, K), torch.bfloat16, dev).fill(a_vals.to(dev))
    perm = torch.randperm(K, generator=torch.Generator().manual_seed(K))
    f = perm[torch.arange(N) % K]
    w_vals = torch.zeros(1, N, K, dtype=torch.float64)
    w_vals[0, torch.arange(N), f] = 1.0
    W = Guarded((1, N, K), torch.bfloat16, dev, flat=True).fill(w_vals.to(dev))
    dt = torch.float32 if fp32 else torch.bfloat16
    O = _out((M, N), dt, dev)
    ops.linear(A.view, W.view, None, out=O.view, out_fp32=fp32, bn=bn)
    torch.cuda.synchronize()
    O.check("gemm index probe")
    assert torch.equal(O.view.double().cpu(), a_vals[:, f])


# ---------------------------------------------------------------------------------------------------------------------
# GEMM: random inputs at the network's layouts
# ---------------------------------------------------------------------------------------------------------------------
LINEAR_CASES = {
    # name: M, K, N, dict(options)
    "strided_a_m1_fp32": (1, 1024, 9990, dict(a_step=25, fp32=True, bias=True)),
    "strided_a_m2_fp32": (2, 1024, 4104, dict(a_step=25, fp32=True, bias=True)),
    "strided_a_m7_fp32": (7, 320, 10000, dict(a_step=3, fp32=True, bias=True)),
    "bf16_into_column_slice": (300, 640, 320, dict(out_cols=(960, 320, 8), bias=True, res1=True)),
    "fp32_n4_into_o8": (1000, 320, 4, dict(out_cols=(8, 0, 0), fp32=True, bias=True)),
    "k8_conv_in": (2053, 8, 320, dict(bias=True, act="silu")),
    "fp32_full_epilogue": (777, 640, 640, dict(fp32=True, bias=True, fvec=100, act="gelu", res1=True, res2=True,
                                               s=(0.5, 0.7, -0.5))),
    "bf16_full_epilogue_ragged": (1000, 320, 1000, dict(bias=True, fvec=64, act="silu", res1=True, res2=True,
                                                        s=(0.3, 1.0, -0.25))),
    "strided_residuals_lean": (4100, 320, 320, dict(bias=True, fvec=512, res1=True, res2=True, s=(0.8, 1.0, 0.2),
                                                    bn=160)),
}


@pytest.mark.parametrize("case", list(LINEAR_CASES))
def test_linear_layouts(cuda_dev, case):
    """Strided A with M = 1, 2, 7 (the per-batch rows ctx0[::T] of the conditioning) and N up to 10k with fp32 output;
    bf16 output into a column slice of a concat buffer; N = 4 fp32 output into o8[:, :4]; K = 8; the full epilogue
    with fp32 and bf16 output.  Residuals and the per-frame vector have leading dims != N (guard columns)."""
    from streamingt2v_b200 import ops, packing
    dev = cuda_dev
    M, K, N, o = LINEAR_CASES[case]
    step = o.get("a_step", 1)
    x = _rand((M, K), 1)
    Abuf = Guarded((M * step, K), torch.bfloat16, dev)
    Abuf.view[::step].copy_(_bf(x, dev))
    A = Abuf.view[::step]
    xb = A.double()
    w = packing.pack_linear(_rand((N, K), 2, K ** -0.5).float(), dev)
    Wg = Guarded(tuple(w.shape), torch.bfloat16, dev, flat=True).fill(w)
    wd = w[0].double()
    pre = xb @ wd.t()
    kw = dict(bn=o.get("bn", 0))
    if o.get("bias"):
        bias = torch.randn(N, generator=torch.Generator().manual_seed(3)).to(dev)
        pre = pre + bias.double()
    else:
        bias = None
    rpf = o.get("fvec")
    if rpf:
        frames = -(-M // rpf)
        Fv = Guarded((frames, N), torch.float32, dev).fill(_rand((frames, N), 4).float().to(dev))
        pre = pre + Fv.view.double().repeat_interleave(rpf, 0)[:M]
        kw.update(fvec=Fv.view, rows_per_frame=rpf)
    s_acc, s1, s2 = o.get("s", (1.0, 1.0, 1.0))
    act = o.get("act")
    act_term = None
    if act == "silu":
        kw["act"] = ops.ACT_SILU
        ref = F.silu(pre)
        act_term = abs(s_acc) * 2 ** -16 * pre.abs()
    elif act == "gelu":
        kw["act"] = ops.ACT_GELU
        ref = _gelu(pre)
        act_term = abs(s_acc) * 2 ** -16 * pre.abs()
    else:
        ref = pre
    ref = s_acc * ref
    kw["s_acc"] = s_acc
    for r, (name, s, seed) in enumerate((("res1", s1, 5), ("res2", s2, 6))):
        if o.get(name):
            R = Guarded((M, N), torch.bfloat16, dev, pad=16 * (r + 1)).fill(_bf(_rand((M, N), seed), dev))
            ref = ref + s * R.view.double()
            kw.update({name: R.view, "s" + name[-1]: s})
    fp32 = o.get("fp32", False)
    dt = torch.float32 if fp32 else torch.bfloat16
    if "out_cols" in o:
        width, c0, pad = o["out_cols"]
        O = _out((M, width), dt, dev, pad=pad)
        O.view = O.view[:, c0:c0 + N]  # the other columns of the row are outside the output and must stay untouched
    else:
        O = _out((M, N), dt, dev)
    view = O.view
    ops.linear(A, Wg.view, bias, out=view, out_fp32=fp32, **kw)
    torch.cuda.synchronize()
    O.check(case)
    first = view.clone()
    ops.linear(A, Wg.view, bias, out=view, out_fp32=fp32, **kw)
    torch.cuda.synchronize()
    assert torch.equal(first.view(torch.int16 if not fp32 else torch.int32),
                       view.view(torch.int16 if not fp32 else torch.int32)), f"{case}: not bitwise repeatable"
    _check_bound(view, ref, _gemm_bound(ref, fp32, act_term), f"linear {case}", "gemm")


@pytest.mark.parametrize("K,M", [(320, 333), (640, 77), (1280, 1001)])
def test_geglu_model_widths(cuda_dev, K, M):
    """GEGLU at the model's widths (F2 = 8 K), ragged M, bias; value * gelu(gate) in float64."""
    from streamingt2v_b200 import ops, packing
    dev = cuda_dev
    F2 = 8 * K
    x = _bf(_rand((M, K), 1), dev)
    w = _rand((F2, K), 2, K ** -0.5).float()
    b = (_rand((F2,), 3) * 0.1).float()
    wp, bp, bn = packing.pack_geglu(w, b, dev)
    A = Guarded((M, K), torch.bfloat16, dev).fill(x)
    O = _out((M, F2 // 2), torch.bfloat16, dev)
    ops.linear(A.view, wp, bp, act=ops.ACT_GEGLU, bn=bn, out=O.view)
    torch.cuda.synchronize()
    O.check(f"geglu K{K}")
    first = O.view.clone()
    ops.linear(A.view, wp, bp, act=ops.ACT_GEGLU, bn=bn, out=O.view)
    torch.cuda.synchronize()
    assert torch.equal(first.view(torch.int16), O.view.view(torch.int16))
    wb = w.to(torch.bfloat16).double().to(dev)
    h = x.double() @ wb.t() + b.double().to(dev)
    val, gate = h.chunk(2, dim=-1)
    ref = val * _gelu(gate)
    _check_bound(O.view, ref, _gemm_bound(ref, False, 2 ** -16 * val.abs() * gate.abs()), f"geglu K{K} M{M}", "gemm")


# ---------------------------------------------------------------------------------------------------------------------
# convolutions: exact tap probe
# ---------------------------------------------------------------------------------------------------------------------
def _coord_input(n, h, w):
    """[n, h, w, 8]: channels 0, 1, 2 = y + 1, x + 1, frame + 1; the rest 0."""
    x = torch.zeros(n, h, w, 8, dtype=torch.float64)
    x[..., 0] = torch.arange(h, dtype=torch.float64)[None, :, None] + 1
    x[..., 1] = torch.arange(w, dtype=torch.float64)[None, None, :] + 1
    x[..., 2] = torch.arange(n, dtype=torch.float64)[:, None, None] + 1
    return _small_ints(x)


def _tap_weights(taps):
    """[taps, 3 taps, 8]: output channel 3 t + j = input channel j through tap t."""
    w = torch.zeros(taps, 3 * taps, 8, dtype=torch.float64)
    for t in range(taps):
        for j in range(3):
            w[t, 3 * t + j, j] = 1.0
    return w


def _gather_expected(x, src_y, src_x):
    """x [n, h, w, 8] float64; src_y[t][i], src_x[t][j] source coordinates per tap (may be out of range -> 0)."""
    n, h, w, _ = x.shape
    outs = []
    for sy, sx in zip(src_y, src_x):
        sy, sx = torch.as_tensor(sy), torch.as_tensor(sx)
        ok = ((sy >= 0) & (sy < h))[:, None] & ((sx >= 0) & (sx < w))[None]
        g = x[:, sy.clamp(0, h - 1)][:, :, sx.clamp(0, w - 1)][..., :3]
        outs.append(g * ok[None, :, :, None])
    return torch.cat(outs, -1)


def _run_conv_probe(fn, x, w, expected, dev, name, **kw):
    X = Guarded(tuple(x.shape), torch.bfloat16, dev, flat=True).fill(x.to(dev))
    Wt = Guarded(tuple(w.shape), torch.bfloat16, dev, flat=True).fill(w.to(dev))
    rows, cout = expected.numel() // w.shape[1], w.shape[1]
    O = _out((rows, cout), torch.bfloat16, dev)
    fn(X.view, Wt.view, None, out=O.view, **kw)
    torch.cuda.synchronize()
    O.check(name)
    assert torch.equal(O.view.double().cpu(), expected.reshape(rows, cout)), f"{name}: wrong tap offsets or padding"


@pytest.mark.parametrize("n,h,w", [(5, 2, 2), (4, 3, 5), (2, 17, 33), (3, 7, 129), (1, 45, 3)])
def test_conv3x3_tap_probe(cuda_dev, n, h, w):
    from streamingt2v_b200 import ops
    x = _coord_input(n, h, w)
    ys = [[i + kh - 1 for i in range(h)] for kh in range(3) for kw in range(3)]
    xs = [[j + kw - 1 for j in range(w)] for kh in range(3) for kw in range(3)]
    _run_conv_probe(ops.conv3x3, x, _tap_weights(9), _gather_expected(x, ys, xs), cuda_dev, f"conv3x3 {n}x{h}x{w}")


@pytest.mark.parametrize("pad_after_only", [False, True])
@pytest.mark.parametrize("n,h,w", [(6, 2, 2), (4, 6, 10), (2, 18, 34), (3, 14, 130), (2, 4, 2)])
def test_conv3x3_s2_tap_probe(cuda_dev, n, h, w, pad_after_only):
    from streamingt2v_b200 import ops
    x = _coord_input(n, h, w)
    d = 0 if pad_after_only else -1
    ys = [[2 * i + kh + d for i in range(h // 2)] for kh in range(3) for kw in range(3)]
    xs = [[2 * j + kw + d for j in range(w // 2)] for kh in range(3) for kw in range(3)]
    _run_conv_probe(ops.conv3x3_s2, x, _tap_weights(9), _gather_expected(x, ys, xs), cuda_dev,
                    f"conv3x3_s2 {n}x{h}x{w} pad_after_only={pad_after_only}", pad_after_only=pad_after_only)


@pytest.mark.parametrize("B,T,h,w", [(3, 1, 3, 5), (4, 2, 2, 2), (2, 25, 3, 5), (1, 25, 9, 11), (2, 2, 12, 20)])
def test_tconv3_tap_probe(cuda_dev, B, T, h, w):
    """Frames are batch-major (frame = b T + t); tap dt reads frame t + dt - 1 of the same batch element, 0 outside."""
    from streamingt2v_b200 import ops
    x = _coord_input(B * T, h, w).reshape(B, T, h * w, 8)
    outs = []
    for dt in range(3):
        src = torch.arange(T) + dt - 1
        ok = ((src >= 0) & (src < T)).to(torch.float64)
        outs.append(x[:, src.clamp(0, T - 1), :, :3] * ok[None, :, None, None])
    expected = torch.cat(outs, -1)
    _run_conv_probe(ops.tconv3, x, _tap_weights(3), expected, cuda_dev, f"tconv3 B{B} T{T} {h}x{w}")


# ---------------------------------------------------------------------------------------------------------------------
# convolutions: random inputs, per-frame vector, frame-spanning boxes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,shape,cout", [("conv", (6, 3, 5, 64), 96), ("conv", (4, 12, 20, 320), 320),
                                             ("conv", (3, 2, 2, 128), 64), ("s2", (5, 6, 10, 64), 128),
                                             ("s2_after", (2, 18, 34, 128), 64), ("tconv", (2, 25, 15, 64), 64),
                                             ("tconv", (1, 3, 40, 320), 320)])
def test_conv_fvec(cuda_dev, kind, shape, cout):
    """bias + per-frame vector (rows_per_frame = H W, as the ResBlock's embedding add) + a residual with ld != N,
    on boxes that span several frames where H W < 128."""
    from streamingt2v_b200 import ops, packing
    dev = cuda_dev
    x = _bf(_rand(shape, 1), dev)
    cin = shape[-1]
    if kind == "tconv":
        B, T, P, _ = shape
        wt = _rand((cout, cin, 3, 1, 1), 2, (3 * cin) ** -0.5).float()
        wp = packing.pack_tconv3(wt, dev)
        x5 = x.double().permute(0, 3, 1, 2)[..., None]
        ref = F.conv3d(x5, wt.to(torch.bfloat16).double().to(dev), padding=(1, 0, 0))[..., 0].permute(0, 2, 3, 1)
        frames, rpf, fn, extra = B * T, P, ops.tconv3, {}
    else:
        n, h, w, _ = shape
        wt = _rand((cout, cin, 3, 3), 2, (9 * cin) ** -0.5).float()
        wp = packing.pack_conv3x3(wt, dev)
        xd = x.double().permute(0, 3, 1, 2)
        wd = wt.to(torch.bfloat16).double().to(dev)
        if kind == "conv":
            ref, fn, extra = F.conv2d(xd, wd, padding=1), ops.conv3x3, {}
        elif kind == "s2":
            ref, fn, extra = F.conv2d(xd, wd, padding=1, stride=2), ops.conv3x3_s2, {}
        else:
            ref = F.conv2d(F.pad(xd, (0, 1, 0, 1)), wd, stride=2)
            fn, extra = ops.conv3x3_s2, dict(pad_after_only=True)
        ref = ref.permute(0, 2, 3, 1)
        frames, rpf = n, ref.shape[1] * ref.shape[2]
    ref = ref.reshape(-1, cout)
    rows = ref.shape[0]
    bias = torch.randn(cout, generator=torch.Generator().manual_seed(3)).to(dev)
    Fv = Guarded((frames, cout), torch.float32, dev).fill(_rand((frames, cout), 4).float().to(dev))
    R = Guarded((rows, cout), torch.bfloat16, dev, pad=24).fill(_bf(_rand((rows, cout), 5), dev))
    ref = ref + bias.double() + Fv.view.double().repeat_interleave(rpf, 0) + R.view.double()
    X = Guarded(tuple(shape), torch.bfloat16, dev, flat=True).fill(x)
    Wg = Guarded(tuple(wp.shape), torch.bfloat16, dev, flat=True).fill(wp)
    O = _out((rows, cout), torch.bfloat16, dev)
    kw = dict(out=O.view, fvec=Fv.view, rows_per_frame=rpf, res1=R.view, s1=1.0, **extra)
    fn(X.view, Wg.view, bias, **kw)
    torch.cuda.synchronize()
    O.check(f"{kind} {shape}")
    first = O.view.clone()
    fn(X.view, Wg.view, bias, **kw)
    torch.cuda.synchronize()
    assert torch.equal(first.view(torch.int16), O.view.view(torch.int16))
    _check_bound(O.view, ref, _gemm_bound(ref, False), f"{kind} {shape}->{cout}", "conv")


# ---------------------------------------------------------------------------------------------------------------------
# attention references (float64, chunked over query rows)
# ---------------------------------------------------------------------------------------------------------------------
def _attn_ref(q, k, v, budget=1 << 28):
    """q [G, Lq, 64], k / v [G, Lk, 64] float64 -> (softmax(q k^T / 8) v, softmax(q k^T / 8) |v|), in query chunks so
    that one score block stays under `budget` bytes."""
    G, Lq, _ = q.shape
    Lk = k.shape[1]
    out = torch.empty(G, Lq, 64, dtype=torch.float64, device=q.device)
    out_abs = torch.empty_like(out)
    chunk = max(1, budget // (8 * G * Lk))
    va = v.abs()
    for i in range(0, Lq, chunk):
        s = torch.matmul(q[:, i:i + chunk], k.transpose(1, 2)) * 0.125
        p = torch.softmax(s, dim=-1)
        del s
        out[:, i:i + chunk] = torch.matmul(p, v)
        out_abs[:, i:i + chunk] = torch.matmul(p, va)
    return out, out_abs


def _attn_bound(ref, ref_abs):
    return 2 ** -8 * ref.abs() + 2 ** -7 * ref_abs


def _heads(t, n, s, heads):
    """rows (n, s) x heads*64 -> [n * heads, s, 64]"""
    return t.reshape(n, s, heads, 64).permute(0, 2, 1, 3).reshape(n * heads, s, 64)


# ---------------------------------------------------------------------------------------------------------------------
# FlashAttention
# ---------------------------------------------------------------------------------------------------------------------
FA_S = [1, 15, 127, 128, 129, 255, 257, 9216]


@pytest.mark.parametrize("s", FA_S)
def test_flash_attn_block_probe(cuda_dev, s):
    """Q = 0: every score is equal, the softmax is uniform.  V column c of head h, frame f is the indicator of key
    block (j // 128 + h + 3 f) mod 64, so output column c is (keys in those blocks) / s: pins which key blocks each
    (frame, head) covers and the mask of the ragged last block.  P = 1 exactly, so the only rounding is the output's:
    within 2^-8 (1 + 2^-14) of the exact value (the 2^-14 covers the fp32 division), exactly 0 where it is 0."""
    from streamingt2v_b200 import ops
    dev = cuda_dev
    n, heads = 2, 2
    Cc = heads * 64
    qkv = torch.zeros(n, s, 3, heads, 64, dtype=torch.float64)
    qkv[:, :, 1] = _rand((n, s, heads, 64), 1)
    blk = torch.arange(s) // 128
    expected = torch.zeros(n, heads, 64, dtype=torch.float64)
    for f in range(n):
        for h in range(heads):
            col = (blk + h + 3 * f) % 64
            qkv[f, :, 2, h] = F.one_hot(col, 64).double()
            expected[f, h] = torch.bincount(col, minlength=64).double() / s
    Q = Guarded((n * s, 3 * Cc), torch.bfloat16, dev, pad=16).fill(qkv.reshape(n * s, 3 * Cc).to(dev))
    O = _out((n * s, Cc), torch.bfloat16, dev, pad=8)
    ops.flash_attn(Q.view, n, s, heads, out=O.view)
    torch.cuda.synchronize()
    O.check(f"flash probe s{s}")
    got = O.view.double().cpu().reshape(n, s, heads, 64)
    exp = expected[:, None].expand(n, s, heads, 64)
    assert torch.equal(got == 0, exp == 0), f"s{s}: zero pattern differs (key block coverage / mask)"
    assert ((got - exp).abs() <= 2 ** -8 * (1 + 2 ** -14) * exp).all(), f"s{s}: block fractions off"


@pytest.mark.parametrize("n,s,heads,sharp", [(3, 1, 5, False), (2, 15, 10, False), (2, 127, 1, False),
                                            (1, 128, 20, False), (2, 129, 5, False), (1, 255, 10, False),
                                            (2, 257, 1, False), (1, 9216, 5, False), (2, 257, 5, True),
                                            (1, 1000, 10, True)])
def test_flash_attn_fp64(cuda_dev, n, s, heads, sharp):
    """ldqkv > 3C (NaN columns past the fused QKV), output into a strided buffer; `sharp` scales Q by 8 so the
    softmax is nearly one-hot and the running max changes between key blocks."""
    from streamingt2v_b200 import ops
    dev = cuda_dev
    Cc = heads * 64
    qkv = _rand((n * s, 3 * Cc), n * 1000 + s, 1.5)
    if sharp:
        qkv[:, :Cc] *= 8
    Q = Guarded((n * s, 3 * Cc), torch.bfloat16, dev, pad=24).fill(_bf(qkv, dev))
    O = _out((n * s, Cc), torch.bfloat16, dev, pad=40)
    ops.flash_attn(Q.view, n, s, heads, out=O.view)
    torch.cuda.synchronize()
    O.check(f"flash s{s}")
    first = O.view.clone()
    ops.flash_attn(Q.view, n, s, heads, out=O.view)
    torch.cuda.synchronize()
    assert torch.equal(first.view(torch.int16), O.view.view(torch.int16))
    qd = Q.view.double()
    q, k, v = (_heads(qd[:, i * Cc:(i + 1) * Cc], n, s, heads) for i in range(3))
    ref, ref_abs = _attn_ref(q, k, v)
    ref = ref.reshape(n, heads, s, 64).permute(0, 2, 1, 3).reshape(n * s, Cc)
    ref_abs = ref_abs.reshape(n, heads, s, 64).permute(0, 2, 1, 3).reshape(n * s, Cc)
    _check_bound(O.view, ref, _attn_bound(ref, ref_abs), f"flash n{n} s{s} h{heads} sharp{sharp}", "flash_attn",
                 l2=2 ** -7)


# ---------------------------------------------------------------------------------------------------------------------
# per-pixel attention (pixel_attn) and shared-K/V attention (small_attn)
# ---------------------------------------------------------------------------------------------------------------------
def _pixel_operands(b, s, heads, lq, lk, kv_per_pixel, q_vals, k_vals, v_vals, dev):
    """q/k/v placed as the network does: one fused QKV buffer (ld = 3C) when Lq == Lk with per-pixel K/V, else q
    alone and a fused KV buffer (ld = 2C); all inside NaN guards."""
    Cc = heads * 64
    if kv_per_pixel and lq == lk:
        G = Guarded((b * lq * s, 3 * Cc), torch.bfloat16, dev, pad=0).fill(
            torch.cat([q_vals, k_vals, v_vals], 1).to(dev))
        return G.view[:, :Cc], G.view[:, Cc:2 * Cc], G.view[:, 2 * Cc:]
    Qg = Guarded(tuple(q_vals.shape), torch.bfloat16, dev, pad=16).fill(q_vals.to(dev))
    KV = Guarded((k_vals.shape[0], 2 * Cc), torch.bfloat16, dev, pad=8).fill(torch.cat([k_vals, v_vals], 1).to(dev))
    return Qg.view, KV.view[:, :Cc], KV.view[:, Cc:]


def _pixel_ref(q, k, v, b, s, heads, lq, lk, kv_per_pixel):
    Cc = heads * 64
    qh = q.double().reshape(b, lq, s, heads, 64).permute(0, 2, 3, 1, 4).reshape(b * s * heads, lq, 64)
    if kv_per_pixel:
        kh, vh = (t.double().reshape(b, lk, s, heads, 64).permute(0, 2, 3, 1, 4).reshape(b * s * heads, lk, 64)
                  for t in (k, v))
    else:
        kh, vh = (t.double().reshape(b, lk, 1, heads, 64).permute(0, 2, 3, 1, 4).expand(b, s, heads, lk, 64)
                  .reshape(b * s * heads, lk, 64) for t in (k, v))
    ref, ref_abs = _attn_ref(qh, kh, vh)
    back = lambda t: t.reshape(b, s, heads, lq, 64).permute(0, 3, 1, 2, 4).reshape(b * lq * s, Cc)  # noqa: E731
    return back(ref), back(ref_abs)


@pytest.mark.parametrize("b,s,heads,lq,lk,pp", [(2, 15, 2, 25, 25, True), (1, 6, 1, 1, 1, True),
                                                (2, 7, 3, 32, 32, True), (1, 33, 2, 8, 25, True),
                                                (2, 5, 1, 25, 7, True), (2, 17, 2, 7, 7, True),
                                                (2, 15, 2, 25, 17, False), (1, 7, 3, 32, 17, False)])
def test_small_attention_probe(cuda_dev, b, s, heads, lq, lk, pp):
    """Q = 0: uniform softmax over the Lk frames (or tokens).  V column j < 32 is the indicator of frame j; columns
    32..35 hold the codes batch + 1, pixel // 16 + 1, pixel % 16 + 1, head + 1 (shared K/V: pixel codes 0).  So the
    output is 1/Lk on frames below Lk, exactly 0 on frames Lk..31 and on columns 36..63, and the row's own codes:
    pins the Lk mask, the zero-filled padded frames and the pixel / head gather.  pixel_attn (pp) rounds the
    normalised P to bf16 before P V and then rounds the output: two bf16 roundings, 2^-7 (1 + 2^-7) relative;
    small_attn keeps P in fp32: one rounding, 2^-8 (1 + 2^-8)."""
    from streamingt2v_b200 import ops
    dev = cuda_dev
    Cc = heads * 64
    kv_s = s if pp else 1
    v = torch.zeros(b, lk, kv_s, heads, 64, dtype=torch.float64)
    v[..., :32] = F.one_hot(torch.arange(lk), 32).double()[None, :, None, None]
    v[..., 32] = (torch.arange(b) + 1.0)[:, None, None, None]
    if pp:
        v[..., 33] = (torch.arange(s) // 16 + 1.0)[None, None, :, None]
        v[..., 34] = (torch.arange(s) % 16 + 1.0)[None, None, :, None]
    v[..., 35] = (torch.arange(heads) + 1.0)[None, None, None, :]
    v_vals = _small_ints(v).reshape(b * lk * kv_s, Cc).to(torch.bfloat16)
    k_vals = _bf(_rand((b * lk * kv_s, Cc), 2), "cpu")
    q_vals = torch.zeros(b * lq * s, Cc, dtype=torch.bfloat16)
    q, k, vv = _pixel_operands(b, s, heads, lq, lk, pp, q_vals, k_vals, v_vals, dev)
    O = _out((b * lq * s, Cc), torch.bfloat16, dev, pad=24)
    ops.small_attn(q, k, vv, b=b, s=s, heads=heads, lq=lq, lk=lk, kv_per_pixel=pp, out=O.view)
    torch.cuda.synchronize()
    name = f"probe {'pixel' if pp else 'small'} b{b} s{s} h{heads} {lq}x{lk}"
    O.check(name)
    exp = torch.zeros(b, lq, s, heads, 64, dtype=torch.float64)
    exp[..., :lk] = 1.0 / lk
    exp[..., 32] = (torch.arange(b) + 1.0)[:, None, None, None]
    if pp:
        exp[..., 33] = (torch.arange(s) // 16 + 1.0)[None, None, :, None]
        exp[..., 34] = (torch.arange(s) % 16 + 1.0)[None, None, :, None]
    exp[..., 35] = (torch.arange(heads) + 1.0)[None, None, None, :]
    exp = exp.reshape(b * lq * s, Cc)
    got = O.view.double().cpu()
    rel = 2 ** -7 * (1 + 2 ** -7) if pp else 2 ** -8 * (1 + 2 ** -8)
    assert torch.equal(got == 0, exp == 0), f"{name}: zero pattern differs (Lk mask / padded frames / gather)"
    bad = ((got - exp).abs() > rel * exp).sum().item()
    assert bad == 0, f"{name}: {bad} values beyond {rel:.3e} relative of the exact average"


@pytest.mark.parametrize("b,s,heads,lq,lk", [(2, 13, 5, 1, 1), (1, 30, 2, 32, 32), (2, 15, 10, 8, 25),
                                            (2, 7, 5, 25, 7), (1, 101, 5, 25, 25), (2, 18, 1, 7, 7)])
def test_pixel_attn_fp64(cuda_dev, b, s, heads, lq, lk):
    """S mod 4 in {1, 2, 3} (the partial last CTA of 4 pixels), Lq / Lk at the limits 1 and 32, Lq < Lk and Lq > Lk;
    q/k/v as column slices of one QKV buffer (ld = 3C) when Lq == Lk, else q alone and a KV buffer (ld = 2C); the
    output has ldo != C."""
    _pixel_case(cuda_dev, b, s, heads, lq, lk, True)


@pytest.mark.parametrize("b,s,heads,lq", [(2, 15, 5, 25), (1, 6, 2, 32), (2, 33, 10, 1)])
def test_small_attn_shared_kv_fp64(cuda_dev, b, s, heads, lq):
    """K/V shared by every pixel of a batch element: the temporal cross-attention over L = 17 context tokens."""
    _pixel_case(cuda_dev, b, s, heads, lq, 17, False)


def _pixel_case(dev, b, s, heads, lq, lk, kv_per_pixel):
    from streamingt2v_b200 import ops
    Cc = heads * 64
    kv_rows = b * lk * (s if kv_per_pixel else 1)
    q_vals = _bf(_rand((b * lq * s, Cc), 1, 1.5), "cpu")
    k_vals = _bf(_rand((kv_rows, Cc), 2, 1.5), "cpu")
    v_vals = _bf(_rand((kv_rows, Cc), 3), "cpu")
    q, k, v = _pixel_operands(b, s, heads, lq, lk, kv_per_pixel, q_vals, k_vals, v_vals, dev)
    O = _out((b * lq * s, Cc), torch.bfloat16, dev, pad=24)
    run = lambda: ops.small_attn(q, k, v, b=b, s=s, heads=heads, lq=lq, lk=lk, kv_per_pixel=kv_per_pixel,  # noqa
                                 out=O.view)
    run()
    torch.cuda.synchronize()
    name = f"{'pixel' if kv_per_pixel else 'small'} b{b} s{s} h{heads} {lq}x{lk}"
    O.check(name)
    first = O.view.clone()
    run()
    torch.cuda.synchronize()
    assert torch.equal(first.view(torch.int16), O.view.view(torch.int16))
    ref, ref_abs = _pixel_ref(q, k, v, b, s, heads, lq, lk, kv_per_pixel)
    _check_bound(O.view, ref, _attn_bound(ref, ref_abs), name, "pixel_attn" if kv_per_pixel else "small_attn",
                 l2=2 ** -7)
