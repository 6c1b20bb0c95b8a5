"""The staged bf16 epilogue of the wgmma GEMM against its register-direct fp32 epilogue.

A bf16-output launch stages each 32-column sub-tile in shared memory and writes it with a TMA store; its residuals
arrive through a TMA-fed ring.  An fp32-output launch of the same operation computes the same fp32 values and stores
them straight from the accumulator registers.  So the bf16 output must equal the fp32 output rounded to bf16,
bitwise.  The shapes have at least 4 x 132 tiles, so every persistent CTA goes round its staging and residual rings
many times.  Outputs are column slices of NaN-filled guard buffers: every element outside the view must be unchanged.
"""
import re
import shutil
import subprocess

import pytest
import torch

NAN = float("nan")
SMS = 132


class Guarded:
    """`view` = columns [c0, c0 + cols) of rows [pre, pre + rows) of a NaN-filled [pre + rows + post, ld] buffer."""

    def __init__(self, rows, cols, dtype, dev, *, c0=8, pad=16, pre=3, post=5):
        ld = c0 + -(-cols // 8) * 8 + pad
        self.buf = torch.full((pre + rows + post, ld), NAN, dtype=dtype, device=dev)
        self.view = self.buf[pre:pre + rows, c0:c0 + cols]
        assert self.view.data_ptr() % 16 == 0
        self.snap = self.buf.clone()

    def outside_unchanged(self):
        mask = torch.ones_like(self.buf, dtype=torch.bool)
        mask[3:3 + self.view.shape[0], 8:8 + self.view.shape[1]] = False
        ity = torch.int16 if self.buf.element_size() == 2 else torch.int32
        return bool((self.buf.view(ity)[mask] == self.snap.view(ity)[mask]).all())


def _rand(shape, seed, scale=1.0, dev="cpu", dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev, dtype)


def _residual(rows, cols, seed, dev):
    r = Guarded(rows, cols, torch.bfloat16, dev, c0=16, pad=8)
    r.view.copy_(_rand((rows, cols), seed, dev=dev))
    return r


def _both(run, rows, n_out, dev):
    """Run `run(out, out_fp32)` once into a bf16 and once into an fp32 guarded column slice."""
    ob = Guarded(rows, n_out, torch.bfloat16, dev)
    of = Guarded(rows, n_out, torch.float32, dev)
    run(ob.view, False)
    run(of.view, True)
    torch.cuda.synchronize()
    return ob, of


def _check(ob, of, name):
    assert torch.isfinite(of.view).all(), f"{name}: fp32 output not fully written"
    want = of.view.to(torch.bfloat16)
    got = ob.view
    n_bad = (got.view(torch.int16) != want.view(torch.int16)).sum().item()
    assert n_bad == 0, f"{name}: {n_bad}/{got.numel()} bf16 outputs differ from the rounded fp32 outputs"
    assert ob.outside_unchanged(), f"{name}: bf16 launch wrote outside its output view"
    assert of.outside_unchanged(), f"{name}: fp32 launch wrote outside its output view"


# (M, K, N, bn, act, bias, fvec rows_per_frame or 0, residuals, s_acc): M and N ragged against the tile
LINEAR_CASES = {
    "bn128_res2_fvec": (70001, 200, 120, 128, 0, True, 1000, 2, 0.75),
    "bn160_silu_res1": (38395, 320, 320, 160, 1, True, 0, 1, 1.0),
    "bn256_res2_fvec": (20000, 328, 1000, 256, 0, True, 400, 2, 0.5),
    "bn256_gelu_res1": (17001, 136, 1280, 256, 2, False, 0, 1, 1.0),
    # a width that is not a whole number of 16-byte chunks keeps the register-direct bf16 store
    "bn128_n100_res1": (67600, 64, 100, 128, 0, True, 0, 1, 1.0),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(LINEAR_CASES))
def test_linear_staged_matches_direct(cuda_dev, case):
    from streamingt2v_b200 import ops, packing
    dev = cuda_dev
    M, K, N, bn, act, has_bias, rpf, nres, s_acc = LINEAR_CASES[case]
    assert -(-M // 128) * -(-N // bn) >= 4 * SMS
    x = _rand((M, K), 1, dev=dev)
    w = packing.pack_linear(_rand((N, K), 2, K ** -0.5, dtype=torch.float32), dev)
    kw = dict(bn=bn, act=act, s_acc=s_acc)
    if has_bias:
        kw["bias"] = _rand((N,), 3, dev=dev, dtype=torch.float32)
    if rpf:
        fv = torch.zeros((-(-M // rpf), N + 24), dtype=torch.float32, device=dev)
        fv[:, :N] = _rand((fv.shape[0], N), 4, dev=dev, dtype=torch.float32)
        kw.update(fvec=fv[:, :N], rows_per_frame=rpf)
    res = [_residual(M, N, 5 + i, dev) for i in range(nres)]
    if nres >= 1:
        kw.update(res1=res[0].view, s1=0.5)
    if nres >= 2:
        kw.update(res2=res[1].view, s2=-1.25)
    ob, of = _both(lambda out, f32: ops.linear(x, w, out=out, out_fp32=f32, **kw), M, N, dev)
    _check(ob, of, case)


@pytest.mark.gpu
@pytest.mark.parametrize("K,M", [(320, 8000), (640, 4100)])
def test_geglu_staged_matches_direct(cuda_dev, K, M):
    from streamingt2v_b200 import ops, packing
    dev = cuda_dev
    F2 = 8 * K
    assert -(-M // 128) * (F2 // 256) >= 4 * SMS
    x = _rand((M, K), 1, dev=dev)
    wp, bp, bn = packing.pack_geglu(_rand((F2, K), 2, K ** -0.5, dtype=torch.float32),
                                    _rand((F2,), 3, 0.1, dtype=torch.float32), dev)
    ob, of = _both(lambda out, f32: ops.linear(x, wp, bp, act=ops.ACT_GEGLU, bn=bn, out=out, out_fp32=f32),
                   M, F2 // 2, dev)
    _check(ob, of, f"geglu K{K}")


@pytest.mark.gpu
def test_conv3x3_column_slice_ragged_frames(cuda_dev):
    """3x3 conv over 9x16 pixels x 50 frames (row box (16, 1, 8), ragged in frames) into a column slice, with a
    residual read from a column slice."""
    from streamingt2v_b200 import ops, packing
    dev = cuda_dev
    Nf, H, W, C, Co = 50, 9, 16, 64, 96
    assert ops.pick_box(W, H, Nf) == (16, 1, 8)
    x = _rand((Nf, H, W, C), 1, dev=dev)
    w = packing.pack_conv3x3(_rand((Co, C, 3, 3), 2, (9 * C) ** -0.5, dtype=torch.float32), dev)
    b = _rand((Co,), 3, dev=dev, dtype=torch.float32)
    r = _residual(Nf * H * W, Co, 4, dev)
    ob, of = _both(lambda out, f32: ops.conv3x3(x, w, b, out=out, out_fp32=f32, res1=r.view, s1=0.25),
                   Nf * H * W, Co, dev)
    _check(ob, of, "conv3x3 9x16x50")


@pytest.mark.gpu
def test_row_box_ragged_in_three_dims(cuda_dev):
    """A GEMM over a 3-D row space (13, 7, 50) tiled by the box (16, 2, 4): every box dimension is ragged, and the
    second consumer warpgroup's half of the box starts at frame 2 of it."""
    from streamingt2v_b200 import ops, packing
    dev = cuda_dev
    e1, e2, e3, K, N = 13, 7, 50, 128, 200
    b1, b2, b3 = 16, 2, 4
    rows = e1 * e2 * e3
    a = _rand((e3, e2, e1, K), 1, dev=dev)
    w = packing.pack_linear(_rand((N, K), 2, K ** -0.5, dtype=torch.float32), dev)
    r = _residual(rows, N, 3, dev)
    s = [K * 2, e1 * K * 2, e1 * e2 * K * 2, rows * K * 2]

    def run(out, f32):
        ops.gemm_raw(a=a, a_dims=(K, e1, e2, e3, 1), a_strides=s, a_box=(64, b1, b2, b3, 1), w=w, n=N, k=K, taps=1,
                     tap_off=[(0, 0, 0, 0, 0)], m_ext=(e1, e2, e3), m_box=(b1, b2, b3), m_adim=(1, 2, 3), out=out,
                     ldo=out.stride(0), out_fp32=f32, res1=r.view, ld1=r.view.stride(0), s1=1.0, bn=128)

    ob, of = _both(run, rows, N, dev)
    _check(ob, of, "row box (16, 2, 4)")
    ref = (a.reshape(rows, K).float() @ w[0].float().t() + r.view.float())
    assert (of.view - ref).abs().max().item() < 1e-2 * ref.abs().max().item()


def test_gemm_sass_has_tma_store():
    """CPU: every mtgemm instantiation issues TMA stores (UTMASTG) for its bf16 outputs."""
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    import __graft_entry__ as g
    g.build()
    from streamingt2v_b200 import _lib
    out = subprocess.run(["cuobjdump", "-sass", str(_lib.lib_path())], capture_output=True, text=True, check=True).stdout
    bodies = re.split(r"Function : ", out)
    gemm = [b for b in bodies if b.startswith("_ZN4b20013mtgemm_kernel")]
    assert len(gemm) == 5
    for b in gemm:
        assert "UTMASTG" in b, b.splitlines()[0]
