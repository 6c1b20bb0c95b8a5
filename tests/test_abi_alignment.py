"""CPU: the entry points reject operand bases their kernels cannot address, before any CUDA call.

The GEMM epilogue stores fp32 column pairs as one 8-byte float2 and loads residual pairs as 4-byte words; the
attention kernels move 16-byte chunks (cp.async, uint4) or store 4-byte words from a 16-byte aligned base.  A
misaligned base must come back as an error, never reach a launch.  The pointers below are fake host addresses, so
these tests only run where no CUDA device is visible: the checks must return before anything touches them."""
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
