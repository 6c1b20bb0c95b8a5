"""The compile-time epilogue kinds of the wgmma GEMM against the generic epilogue body: bitwise the same output.

Every specialised kind runs on both schedules at the N tiles 64, 128, 160 and 256 (GEGLU at 128 and 256, the tiles
its weights can be packed for; the 160-wide tile has no alternating form and runs cooperative on both), with rows
that do not fill the last M tile and, except for GEGLU, a ragged last N tile, once with gemm_epilogue(0) and once
with gemm_epilogue(1) into NaN-filled guard buffers.  The outputs must be equal bit for bit, fully written, and
nothing outside the output view may change.  One profiled forward of the small denoiser must have no staged bf16
launch that falls back to the generic body.
"""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu
NAN = float("nan")


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


@pytest.fixture
def modes():
    """Restores the schedule and the epilogue selector after the test."""
    from streamingt2v_b200 import ops
    sched, epi = ops.gemm_schedule(-1), ops.gemm_epilogue(-1)
    yield
    ops.gemm_schedule(sched)
    ops.gemm_epilogue(epi)


# kind -> (act, bias, per-frame vector, residuals)
KINDS = {
    "EPI_PLAIN": (0, False, False, 0),
    "EPI_BIAS": (0, True, False, 0),
    "EPI_BIAS_RES1": (0, True, False, 1),
    "EPI_BIAS_RES1_FVEC": (0, True, True, 1),
    "EPI_BIAS_FVEC": (0, True, True, 0),
    "EPI_BIAS_GEGLU": (3, True, False, 0),
    "EPI_BIAS_RES2": (0, True, False, 2),
    "EPI_BIAS_SILU": (1, True, False, 0),
    "EPI_BIAS_GELU": (2, True, False, 0),
}
M = 150 * 128 + 37   # more M tiles than SMs, so CTAs walk several tiles; the last one has 37 rows
K = 136              # two K blocks, the second ragged


@pytest.mark.parametrize("schedule", [0, 1])
@pytest.mark.parametrize("bn", [64, 128, 160, 256])
@pytest.mark.parametrize("kind", sorted(KINDS))
def test_kind_matches_generic_bitwise(cuda_dev, modes, kind, bn, schedule):
    from streamingt2v_b200 import _lib, ops, packing
    dev = cuda_dev
    act, has_bias, has_fvec, nres = KINDS[kind]
    geglu = act == ops.ACT_GEGLU
    if geglu and bn not in (128, 256):
        pytest.skip("GEGLU weights are packed for the 128- or the 256-wide tile")
    x = _rand((M, K), 1, dev=dev)
    kw = dict(bn=bn, act=act, s_acc=0.75 if nres == 2 else 1.0)
    if geglu:
        N = 2 * bn
        w, b, _ = packing.pack_geglu(_rand((N, K), 2, K ** -0.5, dtype=torch.float32),
                                     _rand((N,), 3, 0.1, dtype=torch.float32), dev, bn=bn)
        kw["bias"] = b
        n_out = N // 2
    else:
        N = n_out = bn + 40   # the last N tile holds 40 columns: two of its sub-tiles, the second half full
        w = packing.pack_linear(_rand((N, K), 2, K ** -0.5, dtype=torch.float32), dev)
        if has_bias:
            kw["bias"] = _rand((N,), 3, dev=dev, dtype=torch.float32)
    if has_fvec:
        rpf = 1000   # frame boundaries fall inside tiles and between a thread's two rows
        fv = torch.zeros((-(-M // rpf), N + 24), dtype=torch.float32, device=dev)
        fv[:, :N] = _rand((fv.shape[0], N), 4, dev=dev, dtype=torch.float32)
        kw.update(fvec=fv[:, :N], rows_per_frame=rpf)
    res = [Guarded(M, n_out, dev, pad=8 * (i + 1)) for i in range(nres)]
    for i, r in enumerate(res):
        r.view.copy_(_rand((M, n_out), 5 + i, dev=dev))
    if nres >= 1:
        kw.update(res1=res[0].view, s1=0.5)
    if nres >= 2:
        kw.update(res2=res[1].view, s2=-1.25)
    ops.gemm_schedule(schedule)
    outs = []
    for mode in (0, 1):
        ops.gemm_epilogue(mode)
        o = Guarded(M, n_out, dev)
        with ops.profile() as prof:
            ops.linear(x, w, out=o.view, **kw)
        torch.cuda.synchronize()
        want = getattr(_lib, kind) if mode == 1 else 0
        assert prof.launch_records[0][1].endswith(f"epi{want}"), prof.launch_records[0][1]
        assert torch.isfinite(o.view.float()).all(), f"{kind} bn{bn}: epilogue mode {mode} left outputs unwritten"
        assert o.outside_unchanged(), f"{kind} bn{bn}: epilogue mode {mode} wrote outside its output view"
        outs.append(o)
    n_bad = (outs[0].view.view(torch.int16) != outs[1].view.view(torch.int16)).sum().item()
    assert n_bad == 0, f"{kind} bn{bn} schedule {schedule}: {n_bad}/{outs[0].view.numel()} outputs differ"


def test_conv_with_per_frame_vector_matches_generic(cuda_dev, modes):
    """conv1 of a ResBlock: 9 taps, row box over (W, H, frames) ragged in frames, one per-frame row per image."""
    from streamingt2v_b200 import ops, packing
    dev = cuda_dev
    Nf, H, W, Cin, Co = 50, 9, 16, 64, 168
    x = _rand((Nf, H, W, Cin), 1, dev=dev)
    w = packing.pack_conv3x3(_rand((Co, Cin, 3, 3), 2, (9 * Cin) ** -0.5, dtype=torch.float32), dev)
    b = _rand((Co,), 3, dev=dev, dtype=torch.float32)
    fv = _rand((Nf, Co), 4, dev=dev, dtype=torch.float32)
    for schedule in (0, 1):
        ops.gemm_schedule(schedule)
        outs = []
        for mode in (0, 1):
            ops.gemm_epilogue(mode)
            o = Guarded(Nf * H * W, Co, dev)
            ops.conv3x3(x, w, b, out=o.view, fvec=fv, rows_per_frame=H * W)
            torch.cuda.synchronize()
            assert torch.isfinite(o.view.float()).all() and o.outside_unchanged()
            outs.append(o)
        assert torch.equal(outs[0].view.view(torch.int16), outs[1].view.view(torch.int16))


def test_denoiser_forward_has_no_generic_staged_launch(cuda_dev, modes):
    """Every bf16 GEMM of a denoiser forward whose output goes through TMA stores runs a compiled epilogue kind."""
    import re
    from streamingt2v_b200 import arch, ops, synth
    from streamingt2v_b200.wrapper import B200StreamingWrapper
    dev = cuda_dev
    cfg = arch.TINY
    sd_u = arch.synth_state_dict_fast(arch.unet_param_shapes(cfg), 11)
    sd_c = arch.synth_state_dict_fast(arch.controlnet_param_shapes(cfg), 12)
    x, t, c, kw = synth.make_inputs(cfg, T=8, h=8, w=8, seed=5)
    model = B200StreamingWrapper(cfg, sd_u, sd_c, dev)
    with ops.profile() as prof:
        model(x.to(dev), t.to(dev), {k: v.to(dev) for k, v in c.items()},
              **{k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in kw.items()})
    gemms = [d for fam, d, _, _ in prof.launch_records if fam == "mtgemm"]
    assert len(gemms) > 50
    generic = set()
    for d in gemms:
        m = re.search(r" N(\d+) .* act(\d) .* f32(\d) .* epi(\d+)$", d)
        n_out = int(m.group(1)) // (2 if m.group(2) == "3" else 1)
        if m.group(3) == "0" and n_out % 8 == 0 and m.group(4) == "0":
            generic.add(d)
    assert not generic, sorted(generic)
