"""The alternating schedule of the wgmma GEMM against the cooperative one: bitwise the same output.

Every launch runs once with schedule 0 (both consumer warpgroups on one tile) and once with schedule 1 (whole tiles
given to the warpgroups in turn wherever that schedule exists) into NaN-filled guard buffers: the outputs must be
equal bit for bit, fully written, and nothing outside the output view may change.  The cases cover 1 and 2 tiles
(warpgroup 1 idle / one tile each), 131 / 132 / 133 / 265 tiles on 132 SMs (odd and even tile counts per CTA), one
k-block (fewer than the ring depth), 9 taps, one and two residuals with a ragged last N tile, GEGLU packed 128-wide
against the same weights packed 256-wide, a row box ragged in all three dimensions and column-slice outputs.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
NAN = float("nan")


@pytest.fixture
def schedule():
    """Sets the GEMM schedule for a block of launches and restores the previous one afterwards."""
    from streamingt2v_b200 import ops
    prev = ops.gemm_schedule(-1)

    def set_(mode):
        ops.gemm_schedule(mode)

    yield set_
    ops.gemm_schedule(prev)


class Guarded:
    """`view` = columns [8, 8 + cols) of rows [3, 3 + rows) of a NaN-filled bf16 buffer."""

    def __init__(self, rows, cols, dev, pad=16):
        self.buf = torch.full((3 + rows + 5, 8 + -(-cols // 8) * 8 + pad), NAN, dtype=torch.bfloat16, device=dev)
        self.view = self.buf[3:3 + rows, 8:8 + cols]
        self.snap = self.buf.clone()

    def outside_unchanged(self):
        mask = torch.ones_like(self.buf, dtype=torch.bool)
        mask[3:3 + self.view.shape[0], 8:8 + self.view.shape[1]] = False
        return bool((self.buf.view(torch.int16)[mask] == self.snap.view(torch.int16)[mask]).all())


def _rand(shape, seed, scale=1.0, dev="cpu", dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev, dtype)


def _compare(schedule, run, rows, n_out, dev, name):
    outs = []
    for mode in (0, 1):
        schedule(mode)
        o = Guarded(rows, n_out, dev)
        run(o.view)
        torch.cuda.synchronize()
        assert torch.isfinite(o.view.float()).all(), f"{name}: schedule {mode} left output elements unwritten"
        assert o.outside_unchanged(), f"{name}: schedule {mode} wrote outside its output view"
        outs.append(o)
    n_bad = (outs[0].view.view(torch.int16) != outs[1].view.view(torch.int16)).sum().item()
    assert n_bad == 0, f"{name}: {n_bad}/{outs[0].view.numel()} outputs differ between the schedules"
    return outs


# (M, K, N, bn, act, bias, fvec rows_per_frame or 0, residuals, s_acc)
LINEAR_CASES = {
    # the shapes of test_gemm_staged_epilogue_gpu.py that have a bf16 TMA-store epilogue
    "bn128_res2_fvec": (70001, 200, 120, 128, 0, True, 1000, 2, 0.75),
    "bn160_silu_res1": (38395, 320, 320, 160, 1, True, 0, 1, 1.0),
    "bn256_res2_fvec": (20000, 328, 1000, 256, 0, True, 400, 2, 0.5),
    "bn256_gelu_res1": (17001, 136, 1280, 256, 2, False, 0, 1, 1.0),
    # network layouts of test_kernel_edges_gpu.py
    "k8_conv_in": (2053, 8, 320, 0, 1, True, 0, 0, 1.0),
    "bf16_full_epilogue_ragged": (1000, 320, 1000, 0, 1, True, 64, 2, 0.3),
    "strided_residuals_lean": (4100, 320, 320, 160, 0, True, 512, 2, 0.8),
    # tile counts: warpgroup 1 idle, one tile each, odd and even tiles per CTA around 132 SMs
    "tiles_1": (100, 192, 128, 128, 0, True, 0, 1, 1.0),
    "tiles_2": (256, 192, 128, 128, 0, True, 0, 1, 1.0),
    "tiles_131": (131 * 128, 128, 64, 64, 0, True, 0, 0, 1.0),
    "tiles_132": (132 * 128, 128, 64, 64, 0, False, 0, 1, 1.0),
    "tiles_133": (133 * 128 - 5, 128, 32, 32, 2, True, 0, 0, 1.0),
    "tiles_265": (265 * 128, 448, 128, 128, 0, True, 0, 2, 1.0),
    # one k-block a tile: fewer fills than the ring is deep
    "k64": (40000, 64, 160, 160, 0, True, 0, 1, 1.0),
    # two residuals, last N tile ragged (200 = 128 + 72: three of its four sub-tiles)
    "ragged_n_res2": (30000, 256, 200, 128, 0, True, 0, 2, 1.0),
    "ragged_n_res1": (30000, 256, 200, 128, 1, True, 0, 1, 1.0),
}


@pytest.mark.parametrize("case", sorted(LINEAR_CASES))
def test_linear_alternating_matches_cooperative(cuda_dev, schedule, case):
    from streamingt2v_b200 import ops, packing
    dev = cuda_dev
    M, K, N, bn, act, has_bias, rpf, nres, s_acc = LINEAR_CASES[case]
    x = _rand((M, K), 1, dev=dev)
    w = packing.pack_linear(_rand((N, K), 2, K ** -0.5, dtype=torch.float32), dev)
    kw = dict(bn=bn, act=act, s_acc=s_acc)
    if has_bias:
        kw["bias"] = _rand((N,), 3, dev=dev, dtype=torch.float32)
    if rpf:
        fv = torch.zeros((-(-M // rpf), N + 24), dtype=torch.float32, device=dev)
        fv[:, :N] = _rand((fv.shape[0], N), 4, dev=dev, dtype=torch.float32)
        kw.update(fvec=fv[:, :N], rows_per_frame=rpf)
    res = [Guarded(M, N, dev, pad=8 * (i + 1)) for i in range(nres)]
    for i, r in enumerate(res):
        r.view.copy_(_rand((M, N), 5 + i, dev=dev))
    if nres >= 1:
        kw.update(res1=res[0].view, s1=0.5)
    if nres >= 2:
        kw.update(res2=res[1].view, s2=-1.25)
    outs = _compare(schedule, lambda out: ops.linear(x, w, out=out, **kw), M, N, dev, case)
    if case.startswith("tiles_") and act == 0:
        ref = x.float() @ w[0].float().t() + (kw["bias"] if has_bias else 0.0)
        for i, s in enumerate((0.5, -1.25)[:nres]):
            ref = ref + s * res[i].view.float()
        err = (outs[1].view.float() - ref).abs().max().item()
        assert err < 2 ** -6 * ref.abs().max().item(), f"{case}: max error {err}"


@pytest.mark.parametrize("K,M", [(320, 8000), (640, 4100), (1280, 1001)])
def test_geglu_128_wide_matches_256_wide(cuda_dev, schedule, K, M):
    """The same logical GEGLU weights packed for the 128- and the 256-wide tile: one output, on both schedules."""
    from streamingt2v_b200 import ops, packing
    dev = cuda_dev
    F2 = 8 * K
    x = _rand((M, K), 1, dev=dev)
    w = _rand((F2, K), 2, K ** -0.5, dtype=torch.float32)
    b = _rand((F2,), 3, 0.1, dtype=torch.float32)
    w128, b128, bn128 = packing.pack_geglu(w, b, dev, bn=128)
    w256, b256, bn256 = packing.pack_geglu(w, b, dev)
    assert (bn128, bn256) == (128, 256)
    o128 = _compare(schedule, lambda out: ops.linear(x, w128, b128, act=ops.ACT_GEGLU, bn=128, out=out),
                    M, F2 // 2, dev, f"geglu K{K} bn128")
    o256 = _compare(schedule, lambda out: ops.linear(x, w256, b256, act=ops.ACT_GEGLU, bn=256, out=out),
                    M, F2 // 2, dev, f"geglu K{K} bn256")
    assert torch.equal(o128[1].view.view(torch.int16), o256[0].view.view(torch.int16))


def test_conv3x3_nine_taps(cuda_dev, schedule):
    """3x3 conv over 9x16 pixels x 50 frames (row box (16, 1, 8), ragged in frames), residual from a column slice."""
    from streamingt2v_b200 import ops, packing
    dev = cuda_dev
    Nf, H, W, C, Co = 50, 9, 16, 64, 96
    x = _rand((Nf, H, W, C), 1, dev=dev)
    w = packing.pack_conv3x3(_rand((Co, C, 3, 3), 2, (9 * C) ** -0.5, dtype=torch.float32), dev)
    b = _rand((Co,), 3, dev=dev, dtype=torch.float32)
    r = Guarded(Nf * H * W, Co, dev)
    r.view.copy_(_rand((Nf * H * W, Co), 4, dev=dev))
    _compare(schedule, lambda out: ops.conv3x3(x, w, b, out=out, res1=r.view, s1=0.25), Nf * H * W, Co, dev, "conv3x3")


def test_row_box_ragged_in_three_dims(cuda_dev, schedule):
    """Row space (13, 7, 50) tiled by the box (16, 2, 4): the alternating schedule stores the whole box at once."""
    from streamingt2v_b200 import ops, packing
    dev = cuda_dev
    e1, e2, e3, K, N = 13, 7, 50, 128, 200
    b1, b2, b3 = 16, 2, 4
    rows = e1 * e2 * e3
    a = _rand((e3, e2, e1, K), 1, dev=dev)
    w = packing.pack_linear(_rand((N, K), 2, K ** -0.5, dtype=torch.float32), dev)
    r = Guarded(rows, N, dev)
    r.view.copy_(_rand((rows, N), 3, dev=dev))
    s = [K * 2, e1 * K * 2, e1 * e2 * K * 2, rows * K * 2]

    def run(out):
        ops.gemm_raw(a=a, a_dims=(K, e1, e2, e3, 1), a_strides=s, a_box=(64, b1, b2, b3, 1), w=w, n=N, k=K, taps=1,
                     tap_off=[(0, 0, 0, 0, 0)], m_ext=(e1, e2, e3), m_box=(b1, b2, b3), m_adim=(1, 2, 3), out=out,
                     ldo=out.stride(0), res1=r.view, ld1=r.view.stride(0), s1=1.0, bn=128)

    outs = _compare(schedule, run, rows, N, dev, "row box (16, 2, 4)")
    ref = a.reshape(rows, K).float() @ w[0].float().t() + r.view.float()
    assert (outs[1].view.float() - ref).abs().max().item() < 2 ** -6 * ref.abs().max().item()


def test_schedule_query_and_default(cuda_dev):
    from streamingt2v_b200 import ops
    assert ops.gemm_schedule(-1) == 2
    assert ops.gemm_schedule(7) == 2 and ops.gemm_schedule(-1) == 2
