"""CPU: the entry points reject operand bases their kernels cannot address, before any CUDA call.

The GEMM epilogue stores fp32 column pairs as one 8-byte float2 and loads residual pairs as 4-byte words; the
attention kernels move 16-byte chunks (cp.async, uint4) or store 4-byte words from a 16-byte aligned base.  A
misaligned base must come back as an error, never reach a launch.  The norm and glue kernels move 16-byte vectors
(softmax_rows stores 8-byte ones).  The same holds for the other argument checks of those entry points, and a call
with nothing to compute returns 0 without a launch.  The pointers below are fake host addresses, so these tests only
run where no CUDA device is visible: the checks must return before anything touches them."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="fake device pointers: host-only test")

BASE = 0x7F0000000000  # 16-byte aligned fake device address


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from streamingt2v_b200 import _lib
    return _lib.load()


def _assert_alignment_error(lib, rc):
    msg = lib.b200svd_last_error().decode()
    assert rc == 1, msg
    assert "align" in msg.lower(), msg


def _gemm_params(**kw):
    """A linear launch (M = 128, K = N = 64) that passes every check except the ones under test."""
    from streamingt2v_b200._lib import GemmParams
    p = GemmParams()
    p.a_ptr = BASE
    for i, (d, b) in enumerate(zip((64, 128, 1, 1, 1), (64, 128, 1, 1, 1))):
        p.a_dims[i], p.a_box[i] = d, b
    for i in range(4):
        p.a_strides[i] = 128
    p.w_ptr = BASE + 0x100000
    p.n, p.k, p.taps = 64, 64, 1
    for i, (e, b, a) in enumerate(zip((128, 1, 1), (128, 1, 1), (1, 2, 3))):
        p.m_ext[i], p.m_box[i], p.m_adim[i] = e, b, a
    p.out_rs[0], p.out_rs[1], p.out_rs[2] = 1, 128, 128
    p.out = BASE + 0x200000
    p.ldo = 64
    p.s_acc = p.s1 = p.s2 = 1.0
    p.rows_per_frame = 1
    for k, v in kw.items():
        setattr(p, k, v)
    return p


@pytest.mark.parametrize("kw", [
    dict(out_fp32=1, out=BASE + 0x200004),                                   # float2 stores at odd-word offsets
    dict(out_fp32=1, out=BASE + 0x200008 + 4 * 8, res1=BASE + 0x300002, ld1=64),  # residual loads, fp32 output
    dict(out_fp32=1, res2=BASE + 0x300008, ld2=64),
    dict(out_fp32=0, out=BASE + 0x200008),
], ids=["fp32_out", "fp32_out_res1", "fp32_out_res2", "bf16_out"])
def test_gemm_rejects_misaligned_bases(lib, kw):
    p = _gemm_params(**kw)
    _assert_alignment_error(lib, lib.b200svd_gemm(C.byref(p), None))


def test_flash_attn_rejects_misaligned_out(lib):
    rc = lib.b200svd_flash_attn(BASE, 3 * 64, BASE + 0x100008, 64, 1, 128, 1, 0.125, None)
    _assert_alignment_error(lib, rc)


@pytest.mark.parametrize("which", range(4), ids=["q", "k", "v", "o"])
@pytest.mark.parametrize("kernel", ["pixel", "small_pp", "small_shared"])
def test_small_attention_rejects_misaligned_operands(lib, kernel, which):
    ptrs = [BASE + i * 0x100000 for i in range(4)]
    ptrs[which] += 8
    q, k, v, o = ptrs
    if kernel == "pixel":
        rc = lib.b200svd_pixel_attn(q, 64, k, 64, v, 64, o, 64, 1, 8, 1, 8, 8, 0.125, None)
    else:
        rc = lib.b200svd_small_attn(q, 64, k, 64, v, 64, o, 64, 1, 8, 1, 8, 8, 1 if kernel == "small_pp" else 0,
                                    0.125, None)
    _assert_alignment_error(lib, rc)


def test_small_attn_routes_on_kv_per_pixel_alone(monkeypatch):
    """Per-pixel K/V always goes to the tensor-core kernel, whatever the alignment: an operand neither kernel can read
    must produce that kernel's error, not a launch of the other one."""
    from streamingt2v_b200 import ops
    calls = []
    monkeypatch.setattr(ops, "_call", lambda name, *a, **kw: calls.append(name))
    monkeypatch.setattr(ops, "_stream", lambda: None)
    flat = torch.zeros(8 * 64 + 8, dtype=torch.bfloat16)
    t = flat[1:1 + 8 * 64].view(8, 64)                      # 2-byte offset: not 16-byte aligned
    assert t.data_ptr() % 16 != 0
    ops.small_attn(t, t, t, b=1, s=1, heads=1, lq=8, lk=8, kv_per_pixel=True, out=t)
    ops.small_attn(t, t, t[:1], b=1, s=1, heads=1, lq=8, lk=1, kv_per_pixel=False, out=t)
    assert calls == ["b200svd_pixel_attn", "b200svd_small_attn"]


# ---------------------------------------------------------------------------------------------------------------------
# norm and glue entry points: 16-byte vector accesses (softmax_rows stores 8-byte groups of four bf16)
# ---------------------------------------------------------------------------------------------------------------------
X, Y, Z = BASE, BASE + 0x1000000, BASE + 0x2000000   # three aligned fake operands, far apart
GAMMA, BETA = BASE + 0x3000000, BASE + 0x3100000


def _layernorm(lib, x=X, y=Y, xsum=None, fvec=None, rows=8, c=320):
    return lib.b200svd_layernorm(x, c, y, c, rows, c, GAMMA, BETA, 1e-5, fvec, c if fvec else 0, 4, xsum,
                                 c if xsum else 0, 0, None)


MISALIGNED = {
    "gn_stats_x": lambda lib: lib.b200svd_gn_stats(X + 8, 320, 2, 64, 320, Y, Z, Z + 0x100000, None),
    "gn_apply_x": lambda lib: lib.b200svd_gn_apply(X + 8, 320, Y, 320, 2, 64, 320, Z, GAMMA, BETA, 1e-5, 0, None),
    "gn_apply_y": lambda lib: lib.b200svd_gn_apply(X, 320, Y + 2, 320, 2, 64, 320, Z, GAMMA, BETA, 1e-5, 0, None),
    "layernorm_x": lambda lib: _layernorm(lib, x=X + 8),
    "layernorm_y": lambda lib: _layernorm(lib, y=Y + 4),
    "layernorm_xsum": lambda lib: _layernorm(lib, xsum=Z + 8, fvec=GAMMA + 0x200000),
    "layernorm_y_narrow": lambda lib: _layernorm(lib, y=Y + 8, c=64),
    "copy2d_src": lambda lib: lib.b200svd_copy2d(X + 8, 320, Y, 320, 4, 320, None),
    "copy2d_dst": lambda lib: lib.b200svd_copy2d(X, 320, Y + 2, 320, 4, 320, None),
    "add_rows_dst": lambda lib: lib.b200svd_add_rows(X + 8, 320, Y, 320, 4, 1, 320, None),
    "add_rows_src": lambda lib: lib.b200svd_add_rows(X, 320, Y + 8, 320, 4, 4, 320, None),
    "upsample2x_x": lambda lib: lib.b200svd_upsample2x(X + 8, Y, 1, 3, 5, 320, None),
    "upsample2x_y": lambda lib: lib.b200svd_upsample2x(X, Y + 4, 1, 3, 5, 320, None),
    "softmax_rows_in": lambda lib: lib.b200svd_softmax_rows(X + 8, 1000, Y, 1000, 3, 1000, None),
    "softmax_rows_out": lambda lib: lib.b200svd_softmax_rows(X, 1000, Y + 4, 1000, 3, 1000, None),
}


@pytest.mark.parametrize("case", list(MISALIGNED))
def test_norm_glue_reject_misaligned_bases(lib, case):
    _assert_alignment_error(lib, MISALIGNED[case](lib))


def _assert_error(lib, rc, *words):
    msg = lib.b200svd_last_error().decode()
    assert rc == 1, msg
    for w in words:
        assert w in msg, msg


def test_layernorm_rejects_xsum_without_fvec(lib):
    """xsum is bf16(x + fvec): without fvec the kernels would leave the caller's buffer unwritten."""
    for c in (64, 320, 512):
        _assert_error(lib, _layernorm(lib, xsum=Z, c=c), "xsum", "fvec")


def test_layer_norm_wrapper_rejects_xsum_without_fvec(monkeypatch):
    from streamingt2v_b200 import ops
    monkeypatch.setattr(ops, "_call", lambda *a, **kw: pytest.fail("reached the library"))
    x = torch.zeros(4, 64, dtype=torch.bfloat16)
    with pytest.raises(AssertionError, match="fvec"):
        ops.layer_norm(x, torch.ones(64), torch.zeros(64), xsum=torch.empty_like(x))


def test_add_rows_rejects_empty_source(lib):
    for src_rows in (0, -1):
        _assert_error(lib, lib.b200svd_add_rows(X, 320, Y, 320, 4, src_rows, 320, None), "src_rows")


GN_LIMITS = {
    # p beyond the kernels' int row index, n beyond gridDim.y, c that cannot form 32 groups of whole vectors
    "p_over_int_max": (1, 2 ** 31, 320, "p <="),
    "n_over_65535": (65536, 16, 320, "n <= 65535"),
    "negative_p": (1, -5, 320, "p <="),
    "c_16": (1, 64, 16, "channel count"),
    "c_8224": (1, 64, 8224, "channel count"),
}


@pytest.mark.parametrize("case", list(GN_LIMITS))
def test_group_norm_rejects_shapes_it_cannot_index(lib, case):
    n, p, c, word = GN_LIMITS[case]
    assert lib.b200svd_gn_scratch_doubles(n, p, c) == -1
    _assert_error(lib, lib.b200svd_gn_stats(X, c, n, p, c, Y, Z, Z + 0x100000, None), "gn_stats", word)
    _assert_error(lib, lib.b200svd_gn_apply(X, c, Y, c, n, p, c, Z, GAMMA, BETA, 1e-5, 0, None), "gn_apply", word)


def test_group_norm_partials_rejects_n_over_65535(lib):
    _assert_error(lib, lib.b200svd_gn_stats_partials(X, Y, 64, 320, 320, 65536, Z, Z + 0x100000, Z + 0x200000, None),
                  "gn_stats_partials", "n <= 65535")


# zero elements: return 0 before any launch (the fake pointers are never touched)
EMPTY = {
    "layernorm_rows0": lambda lib: _layernorm(lib, rows=0),
    "layernorm_rows0_narrow": lambda lib: _layernorm(lib, rows=0, c=64),
    "layernorm_rows0_generic_fvec": lambda lib: _layernorm(lib, rows=0, c=512, xsum=Z, fvec=GAMMA + 0x200000),
    "layernorm_c0": lambda lib: _layernorm(lib, c=0),
    "softmax_rows": lambda lib: lib.b200svd_softmax_rows(X, 1000, Y, 1000, 0, 1000, None),
    "softmax_cols": lambda lib: lib.b200svd_softmax_rows(X, 1000, Y, 1000, 3, 0, None),
    "transpose_rows": lambda lib: lib.b200svd_transpose(X, 64, Y, 64, 0, 64, None),
    "transpose_cols": lambda lib: lib.b200svd_transpose(X, 64, Y, 64, 64, 0, None),
    "upsample2x": lambda lib: lib.b200svd_upsample2x(X, Y, 0, 3, 5, 320, None),
    "upsample2x_h": lambda lib: lib.b200svd_upsample2x(X, Y, 2, 0, 5, 320, None),
    "copy2d": lambda lib: lib.b200svd_copy2d(X, 320, Y, 320, 0, 320, None),
    "add_rows": lambda lib: lib.b200svd_add_rows(X, 320, Y, 320, 0, 1, 320, None),
    "add_silu": lambda lib: lib.b200svd_add_silu(X, Y, Z, 0, 1, None),
    "nchw_to_nhwc": lambda lib: lib.b200svd_nchw_to_nhwc(X, 64, 0, 4, 64, Y, 8, 0, None),
    "nchw_to_nhwc_hw": lambda lib: lib.b200svd_nchw_to_nhwc(X, 64, 3, 4, 0, Y, 8, 0, None),
    "nhwc_to_nchw": lambda lib: lib.b200svd_nhwc_to_nchw(X, 0, 8, 0, 4, 64, Y, None),
    "nhwc_to_nchw_c": lambda lib: lib.b200svd_nhwc_to_nchw(X, 1, 8, 3, 0, 64, Y, None),
    "timestep_embed": lambda lib: lib.b200svd_timestep_embed(X, 0, 320, 10000.0, Y, 320, None),
    "apm_mix": lambda lib: lib.b200svd_apm_mix(X, 0, 17, 1024, Y, Y, Y, Y, Y, Z, None),
}


@pytest.mark.parametrize("case", list(EMPTY))
def test_empty_launch_returns_zero(lib, case):
    rc = EMPTY[case](lib)
    assert rc == 0, lib.b200svd_last_error().decode()


_GN_EMPTY_SCRIPT = r"""
import sys
sys.path.insert(0, sys.argv[1])
from streamingt2v_b200 import _lib
lib = _lib.load()
X, Y, Z = 0x7F0000000000, 0x7F0001000000, 0x7F0002000000
for n, p in ((1, 0), (4, 0), (0, 100)):
    assert lib.b200svd_gn_scratch_doubles(n, p, 320) == 0, (n, p)
    assert lib.b200svd_gn_stats(X, 320, n, p, 320, Y, Z, Z + 4096, None) == 0, lib.b200svd_last_error()
    assert lib.b200svd_gn_apply(X, 320, Y, 320, n, p, 320, Z, Y, Y, 1e-5, 1, None) == 0, lib.b200svd_last_error()
for c in (0, -32):
    assert lib.b200svd_gn_scratch_doubles(1, 64, c) == -1, c
    assert lib.b200svd_gn_stats(X, 320, 1, 64, c, Y, Z, Z + 4096, None) == 1, c
print("ok")
"""


def test_group_norm_empty_and_zero_width_in_subprocess(lib):
    """p = 0 (or n = 0): nothing to normalise, return 0 without a launch.  c = 0: an error.  Both once reached an
    integer division by zero in the host-side launch geometry, which kills the process; hence the subprocess."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", _GN_EMPTY_SCRIPT, root], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.strip() == "ok", \
        f"exit {r.returncode}\nstdout: {r.stdout[-2000:]}\nstderr: {r.stderr[-2000:]}"


# ---------------------------------------------------------------------------------------------------------------------
# interpolation-stage entry points (csrc/vfi.cu)
# ---------------------------------------------------------------------------------------------------------------------
def _win(lib, qkv=X, ldq=1536, ce=Y, ldc=128, ldo=512, ldm=128, pairs=2, h=45, w=80, heads=16, shift=0):
    return lib.b200svd_vfi_window_attn(qkv, ldq, ce, ldc, Z, ldo, Z + 0x100000, ldm, pairs, h, w, heads, shift,
                                       0.17677669, None)


def _warp(lib, in_bf16=1, out_bf16=1, n=2, c=32, h=45, w=80):
    return lib.b200svd_vfi_warp(X, in_bf16, h * w * c, 1, w * c, c, Y, 2 * h * w, h * w, w, 1, Z, out_bf16,
                                h * w * c, 1, w * c, c, n, c, h, w, None)


def _resize(lib, log2=-1, out_bf16=0, accumulate=0, n=2, c=4, h=90, w=160):
    return lib.b200svd_vfi_resize(X, c * h * w, h * w, w, 1, Y, out_bf16, c * h * w, h * w, w, 1, n, c, h, w, log2,
                                  1.0, accumulate, None)


def _dwconv(lib, x=X, y=Y, n=4, h=45, w=80, c=2048):
    return lib.b200svd_vfi_dwconv_gelu(x, y, n, h, w, c, GAMMA, BETA, None)


def _gather(lib, pairs=2, h=45, w=80, c=512, ldm=512, lda=512, ldo=136):
    return lib.b200svd_vfi_head_gather(X, ldm, Y, lda, pairs, h, w, c, Z, ldo, None)


def _merge(lib, h=720, w=1280, ldr=3):
    return lib.b200svd_vfi_merge(X, Y, Z, GAMMA, ldr, h, w, BETA, BETA + 0x1000000, None)


def _pair(lib, h=720, w=1280, x8=Z):
    return lib.b200svd_vfi_pair_input(X, Y, h, w, GAMMA, x8, None)


VFI_EMPTY = {
    "window_attn_pairs0": lambda lib: _win(lib, pairs=0),
    "window_attn_h0": lambda lib: _win(lib, h=0),
    "window_attn_w0": lambda lib: _win(lib, w=0),
    "window_attn_heads0": lambda lib: _win(lib, heads=0),
    "warp_n0": lambda lib: _warp(lib, n=0),
    "warp_c0": lambda lib: _warp(lib, c=0),
    "warp_h0": lambda lib: _warp(lib, h=0),
    "warp_w0_fp32": lambda lib: _warp(lib, in_bf16=0, out_bf16=0, w=0),
    "resize_n0": lambda lib: _resize(lib, n=0),
    "resize_h0": lambda lib: _resize(lib, h=0),
    "resize_w0_up": lambda lib: _resize(lib, log2=2, w=0),
    "resize_h3_quarter": lambda lib: _resize(lib, log2=-2, h=3),          # floor(3 / 4) = 0 output rows
    "dwconv_n0": lambda lib: _dwconv(lib, n=0),
    "dwconv_c0": lambda lib: _dwconv(lib, c=0),
    "head_gather_pairs0": lambda lib: _gather(lib, pairs=0),
    "head_gather_h0": lambda lib: _gather(lib, h=0),
    "merge_h0": lambda lib: _merge(lib, h=0),
    "merge_w0": lambda lib: _merge(lib, w=0),
    "pair_input_h0": lambda lib: _pair(lib, h=0),
    "frames_to_bgr_n0": lambda lib: lib.b200svd_vfi_frames_to_bgr(X, 0, 720, 1280, Y, None),
    "frames_to_bgr_w0": lambda lib: lib.b200svd_vfi_frames_to_bgr(X, 3, 720, 0, Y, None),
}


@pytest.mark.parametrize("case", list(VFI_EMPTY))
def test_vfi_empty_output_returns_zero(lib, case):
    rc = VFI_EMPTY[case](lib)
    assert rc == 0, lib.b200svd_last_error().decode()


VFI_REJECT = {
    # (call, words the message must contain)
    "window_attn_heads_65536": (lambda lib: _win(lib, heads=65536, ldq=3 * 65536 * 32, ldc=65536 * 8,
                                                 ldo=65536 * 32, ldm=65536 * 8), ("heads=65536",)),
    "window_attn_pairs_32768": (lambda lib: _win(lib, pairs=32768), ("pairs=32768",)),
    "window_attn_negative_h": (lambda lib: _win(lib, h=-1), ("h=-1",)),
    "window_attn_shift_1": (lambda lib: _win(lib, shift=1), ("shift=1",)),
    "window_attn_shift_7": (lambda lib: _win(lib, shift=7), ("shift=7",)),
    "window_attn_qkv_misaligned": (lambda lib: _win(lib, qkv=X + 8), ("align",)),
    "window_attn_ce_misaligned": (lambda lib: _win(lib, ce=Y + 2), ("align",)),
    "window_attn_ldq_odd": (lambda lib: _win(lib, ldq=1540), ("multiples of 8",)),
    "window_attn_ldq_narrow": (lambda lib: _win(lib, ldq=1528), ("heads",)),
    "window_attn_ldc_narrow": (lambda lib: _win(lib, ldc=120), ("heads",)),
    "window_attn_ldo_narrow": (lambda lib: _win(lib, ldo=511), ("heads",)),
    "window_attn_ldm_narrow": (lambda lib: _win(lib, ldm=127), ("heads",)),
    "warp_bf16_in_fp32_out": (lambda lib: _warp(lib, in_bf16=1, out_bf16=0), ("fp32 or both bf16",)),
    "warp_fp32_in_bf16_out": (lambda lib: _warp(lib, in_bf16=0, out_bf16=1), ("fp32 or both bf16",)),
    "warp_w1": (lambda lib: _warp(lib, w=1), ("w=1",)),
    "warp_h1": (lambda lib: _warp(lib, h=1), ("h=1",)),
    "warp_negative_c": (lambda lib: _warp(lib, c=-1), ("c=-1",)),
    "resize_factor_0": (lambda lib: _resize(lib, log2=0), ("factor",)),
    "resize_factor_8": (lambda lib: _resize(lib, log2=3), ("factor",)),
    "resize_factor_1_8": (lambda lib: _resize(lib, log2=-3), ("factor",)),
    "resize_bf16_accumulate": (lambda lib: _resize(lib, out_bf16=1, accumulate=1), ("accumulate=1",)),
    "resize_negative_h": (lambda lib: _resize(lib, h=-4), ("h=-4",)),
    "dwconv_c_12": (lambda lib: _dwconv(lib, c=12), ("c=12", "multiple of 8")),
    "dwconv_x_misaligned": (lambda lib: _dwconv(lib, x=X + 8), ("align",)),
    "dwconv_y_misaligned": (lambda lib: _dwconv(lib, y=Y + 2), ("align",)),
    "head_gather_c_6": (lambda lib: _gather(lib, c=6, ldm=8, lda=8), ("c=6",)),
    "head_gather_ldo_narrow": (lambda lib: _gather(lib, ldo=127), ("leading dims",)),
    "head_gather_ldm_narrow": (lambda lib: _gather(lib, ldm=504), ("leading dims",)),
    "head_gather_lda_narrow": (lambda lib: _gather(lib, lda=504), ("leading dims",)),
    "merge_ldr_2": (lambda lib: _merge(lib, ldr=2), ("ldr=2",)),
    "pair_input_x8_misaligned": (lambda lib: _pair(lib, x8=Z + 8), ("align",)),
    "frames_to_bgr_negative_n": (lambda lib: lib.b200svd_vfi_frames_to_bgr(X, -1, 720, 1280, Y, None), ("n=-1",)),
}


@pytest.mark.parametrize("case", list(VFI_REJECT))
def test_vfi_rejects_out_of_range_arguments(lib, case):
    call, words = VFI_REJECT[case]
    _assert_error(lib, call(lib), *words)
