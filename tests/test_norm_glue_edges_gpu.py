"""GroupNorm, LayerNorm and the glue kernels at the layouts and edges the network uses, against float64 references.

Operands and outputs sit in NaN guard bands (tests/guard_bands.py): NaN rows around them and NaN columns past the
leading dim wherever the ABI takes one.  After a launch every element of the output view is finite and every element
outside it bitwise unchanged.  References are float64 on the exact bf16 / fp32 values the kernels read.  Every random
case runs twice and must give bitwise equal results.  u = 2^-24 is the fp32 unit roundoff, 2^-8 bf16's.

GroupNorm (gn_stats + gn_apply)
  sums: each thread adds at most 256 rows in fp32 and a CTA adds at most 256 thread partials per channel in fp32
  (true at every shape below), the rest is double, so |sum - ref| <= 2^-15 sum|x| and |sumsq - ref| <= 2^-15 sumsq.
  Output: the statistics are double; rstd = rsqrtf((float)var + eps) is within 2^-22 (rsqrtf, 2 ulp) plus the
  rounding of the fp32 sums of squares, which stay within 2e-7 of exact: squares of bf16 values have 16 significant
  bits and add almost exactly in fp32, whatever the DC offset.  gn_apply then evaluates x sc + sh in fp32 with
  sc = rstd g, sh = b - mean rstd g: a few roundings of 2^-24 each of |x - mean| rstd |g|, |mean| rstd |g| and |b|.
  With a factor 8 of margin over all of it:
      |y - ref| <= 2^-8 |ref| + 2^-20 (|x - mean| rstd |g| + |mean| rstd |g| + |b|)
  SiLU (silu_fast: __expf, __fdividef; within 2^-18 |v|, slope <= 1.1) turns the second term into 1.1 times it and
  adds 2^-16 |pre-activation|.
gn_stats_partials: the partials are small integers, so every sum is exact: torch.equal.

LayerNorm (layernorm_kernel<LPR, V, VEC>: LPR lanes per row, V vectors per lane; fp32 two-pass statistics)
  mean and sum of squared deviations go through at most 8 * 8 per-lane adds and 5 shuffle levels: within 69 u
  (< 2^-17.9) of sum|v| and of the variance; rstd adds rsqrtf's 2 ulp; (v - mean) rstd g + b three roundings more.
      |y - ref| <= 2^-8 |ref| + 2^-16 (|xhat g| + rstd |g| mean|v|) + 2^-20 |b|      (xhat = (v - mean) rstd)
  plus the SiLU terms as above.  xsum = bf16(x + fvec) is one fp32 add and one rounding: torch.equal with the same
  expression in torch.  A constant row has zero deviations: the output is exactly bf16(b).

softmax_rows: e = __expf(x - max) is within (2 + 1.7 |x - max|) 2^-23 relative (__expf's documented 2 + 1.17 |x| ulp,
  and the fp32 subtraction); the fp32 row sum adds k u with k = 4 ceil(cols / 1024) + 13, its exponentials their
  p-weighted error; 1 / sum and e * inv one rounding each; then bf16.  Exponentials below 2^-126 flush to zero.
      |p - ref| <= ref (2^-8 + 2^-23 (6 + 1.7 (|x - max| + E_p|x - max|)) + k u) + 2^-126
timestep_embed: f = expf(-ln(P) c / half) in fp32 is within 2^-18.8 relative, t f one rounding more; cosf / sinf
  within 2 ulp:  |out - ref| <= 2^-8 |ref| + (1 + 2^-8) (2^-18 |t f| + 2^-22).
add_silu: a + b one rounding, silu_f = v / (1 + __expf(-v)) within (3 + 1.2 |v|) 2^-23 relative:
  |out - ref| <= 2^-8 |ref| + (3 + 1.2 |v|) 2^-23 |ref| + 1.1 u |v|.  Without SiLU the result is exact.
apm_mix: the conv over L rows is a sum of 3 L + 1 terms in fp32 (<= 52 u of its absolute sum T), the LayerNorm
  statistics a block reduction:  |out - ref| <= 2^-8 |ref| + 2^-16 (|ctx0| + |sa| (|g| rstd (T + mean|mix|
  + |xhat| (max T + mean|mix|)) + |m|)).
ddim_blend_step: at most 10 fp32 roundings along any path of the formula (coefficients included):
  |out - ref| <= 2^-20 A, A the formula evaluated on absolute values.
Layout glue (nchw_to_nhwc, nhwc_to_nchw, upsample2x, copy2d, add_rows, transpose) is exact: torch.equal."""
import math

import pytest
import torch
import torch.nn.functional as F

from guard_bands import Guarded, _check_bound

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
F64 = torch.float64


def _out(shape, dtype, dev, **kw):
    return Guarded(shape, dtype, dev, **kw).snapshot()


def _randn(shape, seed, dev, scale=1.0, shift=0.0):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randn(shape, generator=g, device=dev, dtype=torch.float32) * scale + shift


def _bits(t):
    return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _assert_same_bits(a, b, name):
    assert torch.equal(_bits(a), _bits(b)), f"{name}: not bitwise repeatable"


def _f32(v):
    """The float32 value a float argument becomes at the C ABI."""
    return torch.tensor(v, dtype=torch.float32).item()


def _raw(name, *args):
    from streamingt2v_b200 import ops
    ops._call(name, *args)


def _ptr(t):
    from streamingt2v_b200 import ops
    return ops._ptr(t)


def _stream():
    from streamingt2v_b200 import ops
    return ops._stream()


class _Rows:
    """A per-element bound check accumulated over row chunks of an output too large for one float64 copy."""

    def __init__(self):
        self.ratio, self.bad, self.n, self.e2, self.r2 = 0.0, 0, 0, 0.0, 0.0

    def add(self, out, ref, bound):
        out = out.double()
        assert torch.isfinite(out).all(), "non-finite output"
        err = (out - ref).abs()
        self.ratio = max(self.ratio, (err / bound).max().item())
        self.bad += (err > bound).sum().item()
        self.n += err.numel()
        self.e2 += err.pow(2).sum().item()
        self.r2 += ref.pow(2).sum().item()

    def finish(self, name, family, l2=2 ** -8):
        rel_l2 = math.sqrt(self.e2 / max(self.r2, 1e-300))
        print(f"[{family}] {name}: max err/bound {self.ratio:.3f}, rel L2 {rel_l2:.3e}")
        assert self.bad == 0, f"{name}: {self.bad}/{self.n} elements beyond the derived bound (worst {self.ratio:.3f})"
        assert rel_l2 <= l2, f"{name}: relative L2 error {rel_l2:.3e} > {l2:.3e}"


# ---------------------------------------------------------------------------------------------------------------------
# GroupNorm
# ---------------------------------------------------------------------------------------------------------------------
def _row_chunks(p, C):
    step = max(1, (1 << 23) // C)
    return [(r, min(p, r + step)) for r in range(0, p, step)]


def _gn_reference_stats(x, n, p):
    """float64 per (sample, group): sum, sum of squares, sum |x|, mean, variance (two-pass), in row chunks."""
    C = x.shape[1]
    cpg = C // 32
    s1, s2, sa, ss = (torch.zeros(n, 32, dtype=F64, device=x.device) for _ in range(4))
    for i in range(n):
        for r0, r1 in _row_chunks(p, C):
            xs = x[i * p + r0:i * p + r1].double().unflatten(1, (32, cpg))
            s1[i] += xs.sum((0, 2))
            s2[i] += (xs * xs).sum((0, 2))
            sa[i] += xs.abs().sum((0, 2))
    mean = s1 / (p * cpg)
    for i in range(n):
        for r0, r1 in _row_chunks(p, C):
            xs = x[i * p + r0:i * p + r1].double().unflatten(1, (32, cpg))
            ss[i] += (xs - mean[i][None, :, None]).pow(2).sum((0, 2))
    return s1, s2, sa, mean, ss / (p * cpg)


def _gn_check(X, Y, sums, n, p, gamma, beta, eps, silu, name):
    x, y = X.view, Y.view
    C = x.shape[1]
    cpg = C // 32
    s1, s2, sa, mean, var = _gn_reference_stats(x, n, p)
    got = sums.view[:n]
    d1, d2 = (got[..., 0] - s1).abs(), (got[..., 1] - s2).abs()
    assert (d1 <= 2 ** -15 * sa).all() and (d2 <= 2 ** -15 * s2).all(), \
        f"{name}: statistics off (sum {(d1 / sa).max().item():.3e}, sumsq {(d2 / s2).max().item():.3e} relative)"
    rstd = 1.0 / torch.sqrt(var + _f32(eps))
    g, b = gamma.double().view(32, cpg), beta.double().view(32, cpg)
    acc = _Rows()
    for i in range(n):
        m_, r_ = mean[i][:, None], rstd[i][:, None]
        for r0, r1 in _row_chunks(p, C):
            xs = x[i * p + r0:i * p + r1].double().unflatten(1, (32, cpg))
            dev_ = (xs - m_).abs() * r_ * g.abs() + m_.abs() * r_ * g.abs() + b.abs()
            pre = (xs - m_) * r_ * g + b
            if silu:
                ref = F.silu(pre)
                bound = 2 ** -8 * ref.abs() + 1.1 * 2 ** -20 * dev_ + 2 ** -16 * pre.abs()
            else:
                ref = pre
                bound = 2 ** -8 * ref.abs() + 2 ** -20 * dev_
            acc.add(y[i * p + r0:i * p + r1].unflatten(1, (32, cpg)), ref, bound)
    acc.finish(name, "groupnorm")


def _gn_run(X, Y, sums, n, p, gamma, beta, eps, silu):
    from streamingt2v_b200 import ops
    ops.group_norm(X.view[:n * p], n, p, gamma, beta, eps, silu=silu, out=Y.view[:n * p], sums=sums.view[:n])
    torch.cuda.synchronize()


def _gn_case(dev, n, p, C, eps, silu, name, *, x_fill, alt_n, seed=1):
    X = Guarded((n * p, C), torch.bfloat16, dev, pad=16)
    for r0, r1 in _row_chunks(n * p, C):
        X.view[r0:r1] = x_fill(r0, r1)
    gamma = _randn((C,), seed + 1, dev, 0.3, 1.0)
    beta = _randn((C,), seed + 2, dev, 0.3)
    Y = _out((n * p, C), torch.bfloat16, dev, pad=8)
    sums = _out((n, 32, 2), F64, dev, flat=True)
    _gn_run(X, Y, sums, n, p, gamma, beta, eps, silu)
    Y.check(name)
    sums.check(name + " sums")
    _gn_check(X, Y, sums, n, p, gamma, beta, eps, silu, name)
    first, first_sums = Y.view.clone(), sums.view.clone()
    _gn_run(X, Y, sums, n, p, gamma, beta, eps, silu)
    _assert_same_bits(first, Y.view, name)
    _assert_same_bits(first_sums, sums.view, name + " sums")
    # another sample count takes the same self-resetting tickets; the next launch must still see them at zero
    n2, p2 = alt_n
    _gn_run(X, Y, sums, n2, p2, gamma, beta, eps, silu)
    if (n2, p2) != (n, p) and n2 * p2 == n * p:
        _gn_check(X, Y, sums, n2, p2, gamma, beta, eps, silu, f"{name} as n{n2} p{p2}")
    _gn_run(X, Y, sums, n, p, gamma, beta, eps, silu)
    _assert_same_bits(first, Y.view, name + " after another n")
    _assert_same_bits(first_sums, sums.view, name + " sums after another n")


def _channel_fill(dev, C, seed, scale=1.0, shift=0.0):
    """Rows of randn with a per-channel scale in [0.5, 2] and per-channel mean in [-1, 1] (groups differ)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    cs = 0.5 + 1.5 * torch.rand(C, generator=g, device=dev)
    cm = 2 * torch.rand(C, generator=g, device=dev) - 1

    def fill(r0, r1):
        return _randn((r1 - r0, C), seed * 1000 + r0, dev) * cs * scale + cm + shift
    return fill


GN_NET = {
    # UNet levels of a 576x1024 video (latent 72x128), 14 frames: per-frame GroupNorm (n = frames) and the temporal
    # form (n = batch, p = T S); VAE decoder levels, n = 8 frames
    "unet_c320_s9216": (14, 9216, 320, 1e-5, True),
    "unet_c640_s2304": (14, 2304, 640, 1e-5, True),
    "unet_c1280_s576": (14, 576, 1280, 1e-5, False),
    "unet_c1280_s144": (14, 144, 1280, 1e-5, True),
    "unet_temporal_c320_s9216": (2, 14 * 9216, 320, 1e-5, False),
    "unet_temporal_c640_s2304": (2, 14 * 2304, 640, 1e-5, True),
    "unet_temporal_c1280_s576": (2, 14 * 576, 1280, 1e-5, True),
    "unet_temporal_c1280_s144": (2, 14 * 144, 1280, 1e-5, False),
    "vae_c512_p9216": (8, 9216, 512, 1e-6, True),
    "vae_c512_p36864": (8, 36864, 512, 1e-6, False),
    "vae_c256_p147456": (8, 147456, 256, 1e-6, True),
}


@pytest.mark.parametrize("case", list(GN_NET))
def test_group_norm_network_shapes(cuda_dev, case):
    n, p, C, eps, silu = GN_NET[case]
    alt = (n // 2, p) if n > 1 else (2, p // 2)
    _gn_case(cuda_dev, n, p, C, eps, silu, case, x_fill=_channel_fill(cuda_dev, C, 3), alt_n=alt)


def test_group_norm_vae_full_resolution(cuda_dev):
    """C = 128 at 576x1024, 8 frames: per frame (n = 8, P = 589824, beyond 524288 rows per sample) and the temporal
    form over the same activation (n = 1, P = 8 * 589824: 1152 chunk partials, rows per chunk capped at 4096).  The
    temporal launch is also the call with another n between the two bitwise-compared runs."""
    _gn_case(cuda_dev, 8, 589824, 128, 1e-6, True, "vae_c128_p589824", x_fill=_channel_fill(cuda_dev, 128, 5),
             alt_n=(1, 8 * 589824))


def _const_group_fill(dev, C, n, p, seed):
    """Group 5 of sample 0 and group 31 of the last sample hold one constant (zero variance)."""
    base = _channel_fill(dev, C, seed)
    cpg = C // 32

    def fill(r0, r1):
        v = base(r0, r1)
        rows = torch.arange(r0, r1, device=dev)
        v[rows < p, 5 * cpg:6 * cpg] = 3.0
        v[rows >= (n - 1) * p, 31 * cpg:] = -1.5
        return v
    return fill


GN_EDGES = {
    # name: n, p, C, eps, silu, kind
    "c32": (3, 777, 32, 1e-5, True, None),
    "c96_straddles_groups": (2, 1000, 96, 1e-6, False, None),
    "c96_p5": (4, 5, 96, 1e-5, True, None),
    "c2560": (2, 300, 2560, 1e-5, True, None),
    "c7168_dynamic_smem": (2, 70, 7168, 1e-5, False, None),
    "c7168_p1": (3, 1, 7168, 1e-6, True, None),
    "c320_p1": (3, 1, 320, 1e-6, False, None),
    "c320_p5": (2, 5, 320, 1e-5, True, None),
    "constant_group": (3, 4096, 320, 1e-5, False, "const"),
    "constant_group_silu_c96": (2, 333, 96, 1e-6, True, "const"),
    "dc_offset_256": (2, 2304, 640, 1e-6, True, "dc"),
    "dc_offset_64_c128": (2, 9216, 128, 1e-5, False, "dc64"),
}


@pytest.mark.parametrize("case", list(GN_EDGES))
def test_group_norm_edges(cuda_dev, case):
    """ldx = C + 16 and ldy = C + 8 (NaN pad columns) in every case; C = 96 puts a 16-byte vector across two groups;
    P below the rows one CTA step covers; C = 7168, the widest gn_apply launches, takes gn_stats' dynamic shared
    memory; a zero-variance group; mean / std up to 256 (bf16 at 256 is 2 apart)."""
    n, p, C, eps, silu, kind = GN_EDGES[case]
    dev = cuda_dev
    if kind == "const":
        fill = _const_group_fill(dev, C, n, p, 7)
    elif kind == "dc":
        fill = _channel_fill(dev, C, 9, scale=1.0, shift=256.0)
    elif kind == "dc64":
        fill = _channel_fill(dev, C, 9, scale=4.0, shift=256.0)
    else:
        fill = _channel_fill(dev, C, 11)
    _gn_case(dev, n, p, C, eps, silu, case, x_fill=fill, alt_n=(max(1, n - 1), p))


def test_group_norm_c8192(cuda_dev):
    """c = 8192, the ABI's widest: gn_stats (1024 threads, dynamic shared memory) meets the statistics bound; gn_apply
    needs 1024 threads per block, more than its register use allows, and must say so before writing anything."""
    from streamingt2v_b200 import _lib, ops
    dev = cuda_dev
    n, p, C = 2, 37, 8192
    X = Guarded((n * p, C), torch.bfloat16, dev, pad=16).fill(_channel_fill(dev, C, 13)(0, n * p))
    sums = _out((n, 32, 2), F64, dev, flat=True)
    scratch = torch.empty(_lib.load().b200svd_gn_scratch_doubles(n, p, C), dtype=F64, device=dev)
    counters = torch.zeros(n, dtype=torch.int32, device=dev)
    for _ in range(2):
        _raw("b200svd_gn_stats", _ptr(X.view), X.view.stride(0), n, p, C, _ptr(sums.view), _ptr(scratch),
             _ptr(counters), _stream())
        torch.cuda.synchronize()
        sums.check("gn_stats c8192")
        s1, s2, sa, _, _ = _gn_reference_stats(X.view, n, p)
        assert ((sums.view[..., 0] - s1).abs() <= 2 ** -15 * sa).all()
        assert ((sums.view[..., 1] - s2).abs() <= 2 ** -15 * s2).all()
    Y = _out((n * p, C), torch.bfloat16, dev)
    with pytest.raises(_lib.B200Error, match="threads per block"):
        ops.group_norm(X.view, n, p, torch.ones(C, device=dev), torch.zeros(C, device=dev), 1e-5, out=Y.view)
    torch.cuda.synchronize()
    assert torch.isnan(Y.buf.float()).all(), "gn_apply wrote output it then reported as failed"


# ---------------------------------------------------------------------------------------------------------------------
# GroupNorm statistics from GEMM-epilogue partials
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_slots,C,ld,n", [(1, 256, 256, 1), (63, 256, 264, 3), (65, 8192, 8192, 2),
                                            (1000, 256, 320, 5), (1000, 8192, 8200, 3)])
def test_gn_stats_partials_exact(cuda_dev, n_slots, C, ld, n):
    """Integer partials: exact sums.  Slots of the samples in shuffled order, about one in eight empty (-1); with
    n = 5 the last sample owns no slot (its sums are 0).  Pad channels past C are NaN."""
    dev = cuda_dev
    g = torch.Generator().manual_seed(n_slots * 7 + C)
    owners = n - 1 if n == 5 else n
    slot = torch.randint(0, owners, (n_slots,), generator=g, dtype=torch.int32)
    slot[torch.rand(n_slots, generator=g) < 0.125] = -1
    slot = slot.to(dev)
    vals = torch.randint(-100, 101, (n_slots, C, 2), generator=g).double()
    P = Guarded((n_slots, ld, 2), torch.float32, dev, flat=True)
    P.view[:, :C] = vals.float().to(dev)
    chunks = -(-n_slots // 64)
    scratch = torch.empty(n * chunks * 64, dtype=F64, device=dev)
    counters = torch.zeros(n, dtype=torch.int32, device=dev)
    ref = torch.zeros(n, 32, 2, dtype=F64)
    slot_cpu = slot.cpu()
    for s in range(n):
        ref[s] = vals[slot_cpu == s].sum(0).view(32, C // 32, 2).sum(1)
    S = _out((n, 32, 2), F64, dev, flat=True)

    def run(nn):
        _raw("b200svd_gn_stats_partials", _ptr(P.view), _ptr(slot), n_slots, ld, C, nn, _ptr(S.view), _ptr(scratch),
             _ptr(counters), _stream())
        torch.cuda.synchronize()

    run(n)
    S.check("gn_stats_partials")
    assert torch.equal(S.view.cpu(), ref), f"slots {n_slots} C {C}: sums differ from the exact integer sums"
    if n > 1:
        run(n - 1)              # fewer samples, same tickets
        assert torch.equal(S.view[:n - 1].cpu(), ref[:n - 1])
    run(n)
    assert torch.equal(S.view.cpu(), ref)
    assert (counters == 0).all(), "tickets not reset"


# ---------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ---------------------------------------------------------------------------------------------------------------------
LN_CASES = {
    # name: rows, C, options.  Branches, layernorm_kernel<lanes per row, vectors per lane, float4 parameters>: <8/16/32,
    # 5, vec> (C 320/640/1280), narrow <4/8/16/32, 1, vec> (C <= 256 without fvec), generic <32, 1/2/4/8, scalar>
    # (fvec, or C > 256, or misaligned gamma/beta/fvec)
    "ln5_320_fvec_xsum": (4097, 320, dict(fvec=1024, xsum=True)),
    "ln5_640_fvec_silu": (33, 640, dict(fvec=8, silu=True)),
    "ln5_1280_const": (33, 1280, dict(const=True)),
    "ln5_1280_clip_ln_post": (3, 1280, dict(stride_rows=257)),
    "ln5_1280_misaligned_fallback": (33, 1280, dict(fvec=4, xsum=True, misalign=True)),
    "narrow4_c16_const": (4097, 16, dict(const=True)),
    "narrow4_c32_silu": (3, 32, dict(silu=True)),
    "narrow8_c64": (33, 64, dict(const=True)),
    "narrow16_c96_silu": (4097, 96, dict(silu=True)),
    "narrow32_c256": (33, 256, dict(const=True)),
    "narrow32_c256_misaligned_fallback": (33, 256, dict(misalign=True, const=True)),
    "generic1_c256_fvec": (33, 256, dict(fvec=4)),
    "generic1_c256_fvec_xsum": (1, 256, dict(fvec=1, xsum=True)),
    "generic2_c512_silu": (4097, 512, dict(silu=True)),
    "generic4_c1024_fvec": (1, 1024, dict(fvec=1)),
    "generic4_c1024_const": (33, 1024, dict(const=True)),
    "generic8_c2048_fvec_xsum_silu": (33, 2048, dict(fvec=16, xsum=True, silu=True)),
    "generic8_c1288": (3, 1288, dict()),
}


def _misaligned(values, dev):
    """values (fp32, any shape) at a 4-byte offset from a 16-byte boundary, inside a NaN band."""
    G = Guarded((values.numel() + 1,), torch.float32, dev, flat=True)
    v = G.view[1:].view(values.shape)
    v.copy_(values)
    assert v.data_ptr() % 16 == 4
    return v


@pytest.mark.parametrize("case", list(LN_CASES))
def test_layer_norm_branches(cuda_dev, case):
    """ldx > C, ldy > C (NaN pad columns); rows ragged against 8 warps x rows per warp; fvec with rows_per_frame,
    with and without xsum; gamma / beta / fvec at a 4-byte offset (scalar fallback, same bound); the CLIP ln_post
    layout (3 class rows at a row stride of 257 x 1280); constant rows give exactly bf16(beta)."""
    rows, C, o = LN_CASES[case]
    _ln_case(cuda_dev, case, rows, C, o)


def _ln_case(dev, case, rows, C, o, eps=1e-5):
    """One LayerNorm launch of `rows` x C with the options of LN_CASES, run twice, against float64 in row chunks."""
    from streamingt2v_b200 import ops
    seed = rows * 7 + C
    step = o.get("stride_rows", 1)
    vals = _randn((rows, C), seed, dev, 1.5, 0.3)
    const_rows = [0, rows // 2, rows - 1] if o.get("const") and rows > 3 else []
    for r in const_rows:
        vals[r] = 2.5
    if step > 1:
        X = Guarded((rows * step, C), torch.bfloat16, dev, pad=0)
        x = X.view[::step]
        assert x.stride(0) == step * C
    else:
        X = Guarded((rows, C), torch.bfloat16, dev, pad=24)
        x = X.view
    x.copy_(vals)
    gamma = _randn((C,), seed + 1, dev, 0.3, 1.0)
    beta = _randn((C,), seed + 2, dev, 0.5)
    kw = dict(silu=o.get("silu", False))
    fv = None
    if "fvec" in o:
        rpf = o["fvec"]
        frames = -(-rows // rpf)
        fv = _randn((frames, C), seed + 3, dev, 0.7)
        if o.get("misalign"):
            kw["fvec"] = _misaligned(fv, dev)
        else:
            kw["fvec"] = Guarded((frames, C), torch.float32, dev, pad=8).fill(fv).view
        kw["rows_per_frame"] = rpf
    if o.get("misalign"):
        gamma, beta = _misaligned(gamma, dev), _misaligned(beta, dev)
    XS = None
    if o.get("xsum"):
        XS = _out((rows, C), torch.bfloat16, dev, pad=16)
        kw["xsum"] = XS.view
    Y = _out((rows, C), torch.bfloat16, dev, pad=8)
    ops.layer_norm(x, gamma, beta, eps, out=Y.view, **kw)
    torch.cuda.synchronize()
    Y.check(case)
    first = Y.view.clone()
    if XS is not None:
        XS.check(case + " xsum")
        first_xs = XS.view.clone()
    ops.layer_norm(x, gamma, beta, eps, out=Y.view, **kw)
    torch.cuda.synchronize()
    _assert_same_bits(first, Y.view, case)
    if XS is not None:
        _assert_same_bits(first_xs, XS.view, case + " xsum")
    del first
    if XS is not None:
        del first_xs

    g, b = gamma.double(), beta.double()
    acc = _Rows()
    for r0, r1 in _row_chunks(rows, C):
        xr = x[r0:r1]
        if fv is not None:
            f_rows = fv[torch.arange(r0, r1, device=dev) // kw["rows_per_frame"]]
            if XS is not None:
                xs_ref = (xr.float() + f_rows).bfloat16()
                assert torch.equal(XS.view[r0:r1], xs_ref), f"{case}: xsum != bf16(x + fvec)"
                v = xs_ref.double()
            else:
                v = xr.double() + f_rows.double()
        else:
            v = xr.double()
        mean = v.mean(1, keepdim=True)
        rstd = 1.0 / torch.sqrt((v - mean).pow(2).mean(1, keepdim=True) + _f32(eps))
        xg = (v - mean) * rstd * g
        pre = xg + b
        dev_ = xg.abs() + rstd * g.abs() * v.abs().mean(1, keepdim=True)
        if kw["silu"]:
            ref = F.silu(pre)
            bound = 2 ** -8 * ref.abs() + 1.1 * (2 ** -16 * dev_ + 2 ** -20 * b.abs()) + 2 ** -16 * pre.abs()
        else:
            ref = pre
            bound = 2 ** -8 * ref.abs() + 2 ** -16 * dev_ + 2 ** -20 * b.abs()
        acc.add(Y.view[r0:r1], ref, bound)
    if not kw["silu"]:
        for r in const_rows:
            assert torch.equal(Y.view[r], beta.bfloat16()), f"{case}: constant row {r} is not bf16(beta)"
    acc.finish(f"{case} rows{rows}", "layernorm")


# ---------------------------------------------------------------------------------------------------------------------
# exact glue
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,Cs,H,W,c_off,ld", [(6, 4, 8, 16, 4, 8), (3, 3, 5, 7, 5, 16), (14, 4, 72, 128, 0, 8)])
def test_nchw_to_nhwc_into_column_slice(cuda_dev, N, Cs, H, W, c_off, ld):
    """src frames at a stride past C H W (the extra channel is NaN: a read of it poisons the output); dst columns
    c_off .. c_off + Cs of rows of width ld, the rest of each row and the pad columns untouched."""
    from streamingt2v_b200 import ops
    dev = cuda_dev
    S = Guarded((N, Cs + 1, H, W), torch.float32, dev, flat=True)
    S.view[:, :Cs] = _randn((N, Cs, H, W), N + Cs, dev, 3.0)
    src = S.view[:, :Cs]
    D = _out((N * H * W, ld), torch.bfloat16, dev, pad=8)
    ops.nchw_to_nhwc(src, D.view, c_off)
    torch.cuda.synchronize()
    D.view = D.view[:, c_off:c_off + Cs]
    D.check("nchw_to_nhwc")
    assert torch.equal(D.view, src.bfloat16().permute(0, 2, 3, 1).reshape(N * H * W, Cs))


@pytest.mark.parametrize("fp32,c,width", [(False, 8, 8), (True, 4, 8), (True, 320, 320), (False, 4, 8)])
def test_nhwc_to_nchw(cuda_dev, fp32, c, width):
    """bf16 and fp32 rows (lds = width + pad) back to NCHW fp32; c < width reads the first c columns (the denoiser's
    o8[:, :4]); the unread columns are NaN."""
    from streamingt2v_b200 import ops
    dev = cuda_dev
    N, H, W = 3, 5, 7
    dt = torch.float32 if fp32 else torch.bfloat16
    R = Guarded((N * H * W, width), dt, dev, pad=8)
    R.view[:, :c] = _randn((N * H * W, c), c, dev)
    O = _out((N, c, H, W), torch.float32, dev, flat=True)
    ops.nhwc_to_nchw(R.view, N, c, H * W, O.view)
    torch.cuda.synchronize()
    O.check("nhwc_to_nchw")
    assert torch.equal(O.view, R.view[:, :c].float().reshape(N, H, W, c).permute(0, 3, 1, 2))


@pytest.mark.parametrize("n,h,w,C", [(2, 3, 5, 320), (3, 7, 9, 1280), (1, 1, 1, 8)])
def test_upsample2x(cuda_dev, n, h, w, C):
    dev = cuda_dev
    X = Guarded((n * h * w, C), torch.bfloat16, dev, flat=True).fill(_randn((n * h * w, C), C, dev))
    Y = _out((n * 4 * h * w, C), torch.bfloat16, dev, flat=True)
    _raw("b200svd_upsample2x", _ptr(X.view), _ptr(Y.view), n, h, w, C, _stream())
    torch.cuda.synchronize()
    Y.check("upsample2x")
    ref = X.view.view(n, h, w, C).repeat_interleave(2, 1).repeat_interleave(2, 2).reshape(-1, C)
    assert torch.equal(Y.view, ref)


@pytest.mark.parametrize("rows,cols,step", [(1000, 320, 1), (77, 640, 3), (1, 8, 5)])
def test_copy2d(cuda_dev, rows, cols, step):
    from streamingt2v_b200 import ops
    dev = cuda_dev
    S = Guarded((rows * step, cols), torch.bfloat16, dev, pad=24).fill(_randn((rows * step, cols), rows, dev))
    src = S.view[::step]
    D = _out((rows, cols), torch.bfloat16, dev, pad=16)
    ops.copy2d(src, D.view)
    torch.cuda.synchronize()
    D.check("copy2d")
    assert torch.equal(D.view, src)


@pytest.mark.parametrize("rows,cols,src_rows", [(1000, 320, 1), (1000, 320, 1000), (77, 1280, 1), (33, 64, 33)])
def test_add_rows(cuda_dev, rows, cols, src_rows):
    """One fp32 add and one rounding per element, exactly what (a.float() + b.float()).bfloat16() does."""
    from streamingt2v_b200 import ops
    dev = cuda_dev
    a = _randn((rows, cols), 1, dev, 2.0).bfloat16()
    D = Guarded((rows, cols), torch.bfloat16, dev, pad=8).fill(a).snapshot()
    S = Guarded((src_rows, cols), torch.bfloat16, dev, pad=24).fill(_randn((src_rows, cols), 2, dev))
    ops.add_rows(D.view, S.view)
    torch.cuda.synchronize()
    D.check("add_rows")
    ref = (a.float() + S.view.float().repeat(rows // src_rows, 1)).bfloat16()
    assert torch.equal(D.view, ref)


@pytest.mark.parametrize("rows,cols,pad", [(1, 1, 8), (33, 65, 8), (9216, 512, 0), (100, 64, 24)])
def test_transpose(cuda_dev, rows, cols, pad):
    dev = cuda_dev
    X = Guarded((rows, cols), torch.bfloat16, dev, pad=pad).fill(_randn((rows, cols), rows, dev))
    Y = _out((cols, rows), torch.bfloat16, dev, pad=8)
    _raw("b200svd_transpose", _ptr(X.view), X.view.stride(0), _ptr(Y.view), Y.view.stride(0), rows, cols, _stream())
    torch.cuda.synchronize()
    Y.check("transpose")
    assert torch.equal(Y.view, X.view.t())


# ---------------------------------------------------------------------------------------------------------------------
# bounded glue
# ---------------------------------------------------------------------------------------------------------------------
def _softmax_bound(s, ref, cols):
    x = (s - s.max(1, keepdim=True).values).abs()
    ex = (ref * x).sum(1, keepdim=True)
    k = 4 * -(-cols // 1024) + 13
    return ref * (2 ** -8 + 2 ** -23 * (6 + 1.7 * (x + ex)) + k * U) + 2.0 ** -126


@pytest.mark.parametrize("rows,cols", [(5, 4), (300, 1000), (37, 9216), (2, 9216)])
def test_softmax_rows(cuda_dev, rows, cols):
    """lds > cols and ldo > cols (NaN pad); logits spread over 100 below each row's maximum, so the smallest
    probabilities fall below fp32's normal range; cols = 9216 is the VAE mid-block attention width."""
    from streamingt2v_b200 import ops
    dev = cuda_dev
    g = torch.Generator(device=dev).manual_seed(cols)
    logits = -100 * torch.rand(rows, cols, generator=g, device=dev) + 40 * torch.rand(rows, 1, generator=g, device=dev)
    logits[0, :] = _randn((cols,), 3, dev, 3.0)          # one row of the usual spread
    S = Guarded((rows, cols), torch.float32, dev, pad=8).fill(logits)
    O = _out((rows, cols), torch.bfloat16, dev, pad=8)
    ops.softmax_rows(S.view, out=O.view)
    torch.cuda.synchronize()
    O.check("softmax_rows")
    first = O.view.clone()
    ops.softmax_rows(S.view, out=O.view)
    torch.cuda.synchronize()
    _assert_same_bits(first, O.view, "softmax_rows")
    s = S.view.double()
    ref = torch.softmax(s, 1)
    _check_bound(O.view, ref, _softmax_bound(s, ref, cols), f"softmax {rows}x{cols}", "softmax_rows")


@pytest.mark.parametrize("dim", [256, 320])
def test_timestep_embed(cuda_dev, dim):
    dev = cuda_dev
    t = torch.tensor([0.0, 0.5, 1.0, 24.0, 999.0, 1000.0, 500.7, 3.0], device=dev)
    t = torch.cat([t, 1000 * torch.rand(25, generator=torch.Generator(device=dev).manual_seed(dim), device=dev)])
    n, half = t.numel(), dim // 2
    T = Guarded((n,), torch.float32, dev, flat=True).fill(t)
    O = _out((n, dim), torch.bfloat16, dev, pad=8)
    _raw("b200svd_timestep_embed", _ptr(T.view), n, dim, 10000.0, _ptr(O.view), O.view.stride(0), _stream())
    torch.cuda.synchronize()
    O.check("timestep_embed")
    first = O.view.clone()
    _raw("b200svd_timestep_embed", _ptr(T.view), n, dim, 10000.0, _ptr(O.view), O.view.stride(0), _stream())
    torch.cuda.synchronize()
    _assert_same_bits(first, O.view, "timestep_embed")
    f = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=F64, device=dev) / half)
    a = T.view.double()[:, None] * f[None]
    ref = torch.cat([torch.cos(a), torch.sin(a)], 1)
    bound = 2 ** -8 * ref.abs() + (1 + 2 ** -8) * (2 ** -18 * a.abs().repeat(1, 2) + 2 ** -22)
    _check_bound(O.view, ref, bound, f"timestep_embed dim{dim}", "timestep_embed")


@pytest.mark.parametrize("silu,with_b", [(True, True), (True, False), (False, True)])
def test_add_silu(cuda_dev, silu, with_b):
    dev = cuda_dev
    shape = (50, 1280)
    A = Guarded(shape, torch.float32, dev, flat=True).fill(_randn(shape, 1, dev, 4.0))
    B = Guarded(shape, torch.float32, dev, flat=True).fill(_randn(shape, 2, dev, 4.0)) if with_b else None
    O = _out(shape, torch.bfloat16, dev, flat=True)
    _raw("b200svd_add_silu", _ptr(A.view), _ptr(B.view if B else None), _ptr(O.view), A.view.numel(), int(silu),
         _stream())
    torch.cuda.synchronize()
    O.check("add_silu")
    if not silu:
        assert torch.equal(O.view, (A.view + B.view).bfloat16())
        return
    v = A.view.double() + (B.view.double() if B else 0.0)
    ref = F.silu(v)
    bound = 2 ** -8 * ref.abs() + (3 + 1.2 * v.abs()) * 2 ** -23 * ref.abs() + 1.1 * U * v.abs()
    _check_bound(O.view, ref, bound, f"add_silu b={with_b}", "add_silu")


@pytest.mark.parametrize("N,L,D", [(3, 1, 1000), (2, 17, 1024), (5, 17, 1000)])
def test_apm_mix(cuda_dev, N, L, D):
    dev = cuda_dev
    ctx = Guarded((N, L, D), torch.float32, dev, flat=True).fill(_randn((N, L, D), L, dev))
    w = Guarded((L, 3), torch.float32, dev, flat=True).fill(_randn((L, 3), 2, dev, 0.3))
    wb = Guarded((1,), torch.float32, dev, flat=True).fill(torch.tensor([0.1]))
    lg = Guarded((D,), torch.float32, dev, flat=True).fill(_randn((D,), 3, dev, 0.2, 1.0))
    lb = Guarded((D,), torch.float32, dev, flat=True).fill(_randn((D,), 4, dev, 0.2))
    al = Guarded((1,), torch.float32, dev, flat=True).fill(torch.tensor([0.8]))
    O = _out((N, D), torch.bfloat16, dev, flat=True)
    args = [_ptr(ctx.view), N, L, D] + [_ptr(t.view) for t in (w, wb, lg, lb, al, O)] + [_stream()]
    _raw("b200svd_apm_mix", *args)
    torch.cuda.synchronize()
    O.check("apm_mix")
    first = O.view.clone()
    _raw("b200svd_apm_mix", *args)
    torch.cuda.synchronize()
    _assert_same_bits(first, O.view, "apm_mix")
    c = ctx.view.double()
    wd = w.view.double()
    pad = F.pad(c, (1, 1))
    taps = [pad[:, :, k:k + D] * wd[None, :, k, None] for k in range(3)]
    mix = wb.view.double() + sum(t.sum(1) for t in taps)
    T = wb.view.double().abs() + sum(t.abs().sum(1) for t in taps)
    mean = mix.mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt((mix - mean).pow(2).mean(1, keepdim=True) + _f32(1e-5))
    xhat = (mix - mean) * rstd
    g, b = lg.view.double(), lb.view.double()
    m = xhat * g + b
    sa = F.silu(al.view.double())
    ref = c[:, 0] + m * sa
    ma = mix.abs().mean(1, keepdim=True)
    inner = g.abs() * rstd * (T + ma + xhat.abs() * (T.max(1, keepdim=True).values + ma)) + m.abs()
    bound = 2 ** -8 * ref.abs() + 2 ** -16 * (c[:, 0].abs() + sa.abs() * inner)
    _check_bound(O.view, ref, bound, f"apm_mix N{N} L{L} D{D}", "apm_mix")


# ---------------------------------------------------------------------------------------------------------------------
# DDIM blend step
# ---------------------------------------------------------------------------------------------------------------------
DDIM_CASES = {
    # name: v_pred, guidance, offset, lat_frames, lat_start, out_frames, out_start, alpha_t, alpha_prev
    "v_cfg_offset0_world1": (True, 7.5, 0, 8, 0, 8, 0, 0.31, 0.42),
    "eps_nocfg_offset_cs_minus_1_sharded": (False, None, 7, 24, 3, 13, 5, 0.05, 0.07),
    "v_nocfg_offset_cs_writes_nothing": (True, None, 8, 16, 8, 16, 8, 0.5, 0.6),
    "eps_cfg_offset3_sharded": (False, 4.0, 3, 20, 12, 9, 1, 0.9, 0.95),
    "v_cfg_offset5_out_before_lat": (True, 1.5, 5, 30, 20, 10, 2, 0.002, 0.01),
}


@pytest.mark.parametrize("case", list(DDIM_CASES))
def test_ddim_blend_step(cuda_dev, case):
    """out_start != lat_start with out a different tensor of another frame count (the sharded enhance path); frames
    below out_start + offset and from out_start + cs on must be bitwise unchanged: blending relies on it."""
    from streamingt2v_b200 import ops
    dev = cuda_dev
    v_pred, guid, offset, lf, ls, of, os_, at, ap = DDIM_CASES[case]
    Cc, cs, H, W = 4, 8, 24, 40
    nb = 1 if guid is None else 2
    N = Guarded((nb, Cc, cs, H, W), torch.float32, dev, flat=True).fill(_randn((nb, Cc, cs, H, W), 1, dev))
    L = Guarded((1, Cc, lf, H, W), torch.float32, dev, flat=True).fill(_randn((1, Cc, lf, H, W), 2, dev))
    O = Guarded((1, Cc, of, H, W), torch.float32, dev, flat=True).fill(_randn((1, Cc, of, H, W), 3, dev)).snapshot()
    whole = O.view
    kw = dict(lat_start=ls, out_start=os_, offset=offset, guidance=guid, alpha_t=at, alpha_prev=ap,
              v_prediction=v_pred)
    ops.ddim_blend_step(N.view, L.view, whole, **kw)
    torch.cuda.synchronize()
    O.view = whole[:, :, os_ + offset:os_ + cs]
    O.check(case)
    first = O.view.clone()
    ops.ddim_blend_step(N.view, L.view, whole, **kw)
    torch.cuda.synchronize()
    O.check(case + " (second run)")
    _assert_same_bits(first, O.view, case)
    u = N.view[0].double()[:, offset:]
    e = u if guid is None else u + _f32(guid) * (N.view[1].double()[:, offset:] - u)
    E = u.abs() if guid is None else u.abs() + abs(_f32(guid)) * (N.view[1].double()[:, offset:].abs() + u.abs())
    x = L.view[0].double()[:, ls + offset:ls + cs]
    a, a_p = _f32(at), _f32(ap)
    sa, sb, sap, sdir = math.sqrt(a), math.sqrt(1 - a), math.sqrt(a_p), math.sqrt(1 - a_p)
    if v_pred:
        x0, eps = sa * x - sb * e, sa * e + sb * x
        X0, EPS = sa * x.abs() + sb * E, sa * E + sb * x.abs()
    else:
        x0, eps = (x - sb * e) / sa, e
        X0, EPS = (x.abs() + sb * E) / sa, E
    ref = sap * x0 + sdir * eps
    if ref.numel():
        _check_bound(O.view[0], ref, 2 ** -20 * (sap * X0 + sdir * EPS), case, "ddim_blend_step", l2=2 ** -20)
