"""Op-level host wrappers over the C ABI (ctypes): build the TMA views / tap tables and launch.

All activations are bf16, channel-last ("(b t) h w c" == token rows "(b t) (h w) c").  Nothing here computes on
the host; every function enqueues one hand-written sm_90a kernel on torch's current CUDA stream.
"""
from __future__ import annotations

import ctypes as C
import itertools
import operator
import os
from functools import lru_cache

import torch

from . import _lib
from ._lib import ACT_GEGLU, ACT_GELU, ACT_NONE, ACT_PRELU, ACT_SILU, GemmParams

_launch_count = 0
_PROFILE = None  # list of (family, flops, bytes, start_event, end_event) while profiling


def launches() -> int:
    """Number of kernel launches issued through this module (bench.py's gpu_launches)."""
    return _launch_count


def gemm_pair_mode(mode: int = -1) -> int:
    """Records a CTA-pair tile mode (0..3; kept for ABI compatibility: sm_90 runs single-CTA tiles in every mode).
    Any other value only queries.  Returns the previous mode."""
    return int(_lib.load().b200svd_gemm_pair_mode(int(mode)))


def gemm_schedule(mode: int = -1) -> int:
    """Consumer schedule of the GEMM: 0 = cooperative everywhere, 1 = alternating wherever it exists, 2 = alternating
    for launches of many short tiles (default); see b200svd_gemm_schedule.  Any other value only queries.  Returns
    the previous mode.  The output does not depend on it."""
    return int(_lib.load().b200svd_gemm_schedule(int(mode)))


def gemm_epilogue(mode: int = -1) -> int:
    """Epilogue body of the GEMM's staged bf16 outputs: 0 = the generic body everywhere, 1 = a compile-time kind
    wherever one exists (default); see b200svd_gemm_epilogue.  Any other value only queries.  Returns the previous
    mode.  The output does not depend on it."""
    return int(_lib.load().b200svd_gemm_epilogue(int(mode)))


def flash_attn_variant(v: int = -1) -> int:
    """Records a softmax variant (3..5; kept for ABI compatibility: the sm_90 kernel has one softmax organisation).
    Any other value only queries.  Returns the previous variant."""
    return int(_lib.load().b200svd_flash_attn_variant(int(v)))


class profile:
    """Context manager: brackets every launch with CUDA events on the launching stream and returns per-family
    (launches, total ms, algorithmic FLOPs, algorithmic bytes).  Used by bench.py for the live roofline numbers;
    adds two event records per launch, so it is never active inside a timed region."""

    def __enter__(self):
        global _PROFILE
        _PROFILE = []
        return self

    def __exit__(self, *exc):
        global _PROFILE
        recs, _PROFILE = _PROFILE, None
        torch.cuda.synchronize()
        self.families = {}
        self.launch_records = []  # (family, desc, ms, flops)
        for fam, flops, nbytes, e0, e1 in recs:
            desc = ""
            if isinstance(fam, tuple):
                fam, desc = fam
            self.launch_records.append((fam, desc, e0.elapsed_time(e1), flops))
            f = self.families.setdefault(fam, dict(launches=0, ms=0.0, flops=0.0, bytes=0.0))
            f["launches"] += 1
            f["ms"] += e0.elapsed_time(e1)
            f["flops"] += flops
            f["bytes"] += nbytes
        return False


def summarize_records(records, family="mtgemm", top=40):
    """Group per-launch records by descriptor: [(desc, launches, total ms, TFLOP/s)] sorted by total time."""
    agg = {}
    for fam, desc, ms, flops in records:
        if fam != family:
            continue
        a = agg.setdefault(desc, [0, 0.0, 0.0])
        a[0] += 1
        a[1] += ms
        a[2] += flops
    rows = [(d, v[0], v[1], v[2] / max(v[1], 1e-9) / 1e9) for d, v in agg.items()]
    rows.sort(key=lambda r: -r[2])
    return rows[:top]


def _prof_begin():
    if _PROFILE is None:
        return None
    e0 = torch.cuda.Event(enable_timing=True)
    e0.record()
    return e0


def _prof_end(e0, family, flops=0.0, nbytes=0.0):
    if e0 is None:
        return
    e1 = torch.cuda.Event(enable_timing=True)
    e1.record()
    _PROFILE.append((family, flops, nbytes, e0, e1))


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


@lru_cache(maxsize=None)
def pick_box(e1: int, e2: int, e3: int):
    """Power-of-two boxes (b1,b2,b3), b1*b2*b3 == 128, minimising the number of 128-row tiles over the
    output-pixel space (e1,e2,e3); ties prefer the widest innermost box (longest contiguous TMA rows)."""
    best = None
    pows = [1, 2, 4, 8, 16, 32, 64, 128]
    for b1, b2 in itertools.product(pows, pows):
        if b1 * b2 > 128:
            continue
        b3 = 128 // (b1 * b2)
        tiles = -(-e1 // b1) * -(-e2 // b2) * -(-e3 // b3)
        key = (tiles, -b1, -b2)
        if best is None or key < best[0]:
            best = (key, (b1, b2, b3))
    return best[1]


def gemm_raw(*, a, a_dims, a_strides, a_box, w, n, k, taps, tap_off, m_ext, m_box, m_adim, out, ldo, out_rs=None,
             out_fp32=False, bias=None, fvec=None, ldf=0, rows_per_frame=1, act=ACT_NONE, s_acc=1.0, res1=None,
             ld1=0, s1=1.0, res2=None, ld2=0, s2=1.0, bn=0, gn=None, slope=None):
    global _launch_count
    p = GemmParams()
    p.a_ptr = a.data_ptr()
    for i in range(5):
        p.a_dims[i] = int(a_dims[i])
        p.a_box[i] = int(a_box[i])
    for i in range(4):
        p.a_strides[i] = int(a_strides[i])
    p.w_ptr = w.data_ptr()
    p.n, p.k, p.taps = int(n), int(k), int(taps)
    for t in range(taps):
        for i in range(5):
            p.tap_off[t][i] = int(tap_off[t][i])
    if out_rs is None:
        out_rs = (1, m_ext[0], m_ext[0] * m_ext[1])
    for i in range(3):
        p.m_ext[i] = int(m_ext[i])
        p.m_box[i] = int(m_box[i])
        p.m_adim[i] = int(m_adim[i])
        p.out_rs[i] = int(out_rs[i])
    p.out = out.data_ptr()
    p.ldo = int(ldo)
    p.out_fp32 = 1 if out_fp32 else 0
    p.bias = bias.data_ptr() if bias is not None else None
    p.fvec = fvec.data_ptr() if fvec is not None else None
    p.ldf = int(ldf)
    p.rows_per_frame = int(rows_per_frame)
    p.act = int(act)
    p.s_acc = float(s_acc)
    p.res1 = res1.data_ptr() if res1 is not None else None
    p.ld1 = int(ld1)
    p.s1 = float(s1)
    p.res2 = res2.data_ptr() if res2 is not None else None
    p.ld2 = int(ld2)
    p.s2 = float(s2)
    p.bn = int(bn)
    if slope is not None:
        assert slope.dtype == torch.float32 and slope.is_contiguous() and slope.numel() >= n
        p.slope = slope.data_ptr()
    if gn is not None:
        p.gn_part = gn["part"].data_ptr()
        p.gn_slot_sample = gn["slot"].data_ptr()
        p.gn_ld = int(gn["C"])
        p.gn_rows = int(gn["p"])
    lib = _lib.load()
    e0 = _prof_begin()
    _lib.check(lib.b200svd_gemm(C.byref(p), _stream()), "b200svd_gemm")
    _launch_count += 1
    if e0 is not None:
        rows = int(m_ext[0]) * int(m_ext[1]) * int(m_ext[2])
        n_out = n // 2 if act == ACT_GEGLU else n
        nbytes = 2.0 * rows * k + 2.0 * taps * n * k + (4.0 if out_fp32 else 2.0) * rows * n_out
        nbytes += 2.0 * rows * n_out * ((res1 is not None) + (res2 is not None))
        desc = (f"M{rows} K{k} N{n} taps{taps} act{act} res{(res1 is not None) + (res2 is not None)} "
                f"fvec{int(fvec is not None)} f32{int(out_fp32)} box{tuple(int(b) for b in m_box)} "
                f"epi{int(lib.b200svd_gemm_epilogue_kind(C.byref(p)))}")
        _prof_end(e0, ("mtgemm", desc), 2.0 * rows * k * n * taps, nbytes)


# GroupNorm statistics in the producing GEMM's epilogue (activation-free bf16 launches only).  Off by default;
# B200SVD_GN_FUSE=1 turns it on.
GN_FUSE = os.environ.get("B200SVD_GN_FUSE", "0") != "0"


@lru_cache(maxsize=None)
def _gn_slots(m_ext, m_box, p):
    """Number of (M tile, quadrant) slots of a GEMM launch if every 32-row quadrant of every 128-row tile lies inside
    ONE GroupNorm sample of p consecutive output rows (then the epilogue can take the statistics), else 0."""
    import numpy as np
    (e1, e2, e3), (b1, b2, b3) = m_ext, m_box
    t1, t2, t3 = -(-e1 // b1), -(-e2 // b2), -(-e3 // b3)
    c1 = min(b1, 32)
    c2 = min(b2, 32 // c1)
    c3 = 32 // (c1 * c2)
    i1, i2, i3, q = np.meshgrid(np.arange(t1), np.arange(t2), np.arange(t3), np.arange(4), indexing="ij")
    qoff = q * 32
    a1 = i1 * b1 + qoff % b1
    a2 = i2 * b2 + (qoff // b1) % b2
    a3 = i3 * b3 + qoff // (b1 * b2)
    ok = (a1 < e1) & (a2 < e2) & (a3 < e3)                      # quadrants with at least one valid row
    z1 = np.minimum(a1 + c1, e1) - 1
    z2 = np.minimum(a2 + c2, e2) - 1
    z3 = np.minimum(a3 + c3, e3) - 1
    lo = a1 + a2 * e1 + a3 * e1 * e2
    hi = z1 + z2 * e1 + z3 * e1 * e2
    if bool(((lo // p != hi // p) & ok).any()):
        return 0
    return t1 * t2 * t3 * 4                                      # the GEMM writes every slot of every M tile


def _gn_request(gn_rows, m_ext, m_box, n_out, act, out_fp32, device):
    """Partial-statistics buffers for a launch whose output feeds a GroupNorm over samples of gn_rows rows, or None."""
    if gn_rows is None or not GN_FUSE or act != ACT_NONE or out_fp32 or n_out % 32 or n_out < 256:
        return None
    n_slots = _gn_slots(tuple(int(v) for v in m_ext), tuple(int(v) for v in m_box), int(gn_rows))
    if n_slots == 0:
        return None
    return dict(part=torch.empty((n_slots, n_out, 2), dtype=torch.float32, device=device),
                slot=torch.empty((n_slots,), dtype=torch.int32, device=device), n_slots=n_slots, p=int(gn_rows),
                C=int(n_out))


def _epi_kwargs(rows, n_out, out, bias, fvec, rows_per_frame, act, s_acc, res1, s1, res2, s2, out_fp32, slope=None):
    kw = dict(bias=bias, act=act, s_acc=s_acc, out_fp32=out_fp32)
    assert (act == ACT_PRELU) == (slope is not None), "PReLU takes a slope vector, nothing else does"
    if slope is not None:
        kw.update(slope=slope)
    if fvec is not None:
        assert fvec.dtype == torch.float32 and fvec.stride(-1) == 1
        kw.update(fvec=fvec, ldf=fvec.stride(0), rows_per_frame=rows_per_frame)
    if res1 is not None:
        assert res1.dtype == torch.bfloat16 and res1.stride(-1) == 1
        kw.update(res1=res1, ld1=res1.stride(-2), s1=s1)
    if res2 is not None:
        assert res2.dtype == torch.bfloat16 and res2.stride(-1) == 1
        kw.update(res2=res2, ld2=res2.stride(-2), s2=s2)
    return kw


def _alloc_out(rows, n_out, out, out_fp32, device):
    if out is None:
        out = torch.empty((rows, n_out), dtype=torch.float32 if out_fp32 else torch.bfloat16, device=device)
    assert out.stride(-1) == 1
    return out


def linear(x, w, bias=None, *, act=ACT_NONE, out=None, out_fp32=False, fvec=None, rows_per_frame=1, s_acc=1.0,
           res1=None, s1=1.0, res2=None, s2=1.0, bn=0, gn_rows=None, slope=None):
    """x: [M, K] bf16 (row stride arbitrary, multiple of 8); w: packed [1, N, K] bf16; returns [M, N_out]."""
    assert x.dtype == torch.bfloat16 and x.dim() == 2 and x.stride(1) == 1
    M, K = x.shape
    N = w.shape[-2]
    assert w.shape[-1] == K and w.is_contiguous()
    n_out = N // 2 if act == ACT_GEGLU else N
    out = _alloc_out(M, n_out, out, out_fp32, x.device)
    ld = x.stride(0)
    big = ld * 2 * max(M, 1)
    gn = _gn_request(gn_rows, (M, 1, 1), (128, 1, 1), n_out, act, out_fp32, x.device)
    gemm_raw(a=x, a_dims=(K, M, 1, 1, 1), a_strides=(ld * 2, big, big, big), a_box=(64, 128, 1, 1, 1),
             w=w, n=N, k=K, taps=1, tap_off=[(0, 0, 0, 0, 0)], m_ext=(M, 1, 1), m_box=(128, 1, 1),
             m_adim=(1, 2, 3), out=out, ldo=out.stride(0), bn=bn, gn=gn,
             **_epi_kwargs(M, n_out, out, bias, fvec, rows_per_frame, act, s_acc, res1, s1, res2, s2, out_fp32, slope))
    if gn is not None:
        out._b200_gn = gn          # consumed by group_norm(out, ...) instead of a statistics pass over `out`
    return out


def conv3x3(x, w, bias=None, *, out=None, **epi):
    """x: [N, H, W, C] bf16 contiguous; w: packed [9, Cout, C] (tap = kh*3+kw); stride 1, zero pad 1.
    Returns [N*H*W, Cout] rows (== [N, H, W, Cout])."""
    assert x.dtype == torch.bfloat16 and x.dim() == 4 and x.is_contiguous()
    N, H, W, Cc = x.shape
    Cout = w.shape[1]
    assert w.shape == (9, Cout, Cc) and w.is_contiguous()
    b1, b2, b3 = pick_box(W, H, N)
    taps = [(0, kw - 1, kh - 1, 0, 0) for kh in range(3) for kw in range(3)]
    return _conv_common(x, (Cc, W, H, N, 1), (Cc * 2, W * Cc * 2, H * W * Cc * 2, N * H * W * Cc * 2),
                        (64, b1, b2, b3, 1), w, Cout, Cc, taps, (W, H, N), (b1, b2, b3), (1, 2, 3), bias, out, epi)


def conv3x3_s2(x, w, bias=None, *, out=None, pad_after_only=False, **epi):
    """Stride-2 3x3 conv.  x: [N, H, W, C] with even H, W.  The input is viewed as [N, H/2, 2, W/2, 2*C] so that every
    tap is a plain shifted TMA box (out-of-range boxes are zero filled = the padding).
    pad_after_only=False: pad 1 on every side (Downsample.op of the UNet, openaimodel.py:188-195): tap k reads input
    row 2i + k - 1.  pad_after_only=True: pad (0,1,0,1) + padding-0 conv (Downsample of the autoencoder,
    diffusionmodules/model.py:73-92): tap k reads input row 2i + k."""
    assert x.dtype == torch.bfloat16 and x.dim() == 4 and x.is_contiguous()
    N, H, W, Cc = x.shape
    assert H % 2 == 0 and W % 2 == 0
    Ho, Wo = H // 2, W // 2
    Cout = w.shape[1]
    assert w.shape == (9, Cout, Cc) and w.is_contiguous()
    b1, b2, b3 = pick_box(Wo, Ho, N)
    taps = []
    # (offset in output rows, parity inside the row pair) of input row 2i + k - 1  /  2i + k
    table = ((0, 0), (0, 1), (1, 0)) if pad_after_only else ((-1, 1), (0, 0), (0, 1))
    for kh in range(3):
        dh, hp = table[kh]
        for kw in range(3):
            dw, wp = table[kw]
            taps.append((wp * Cc, dw, hp, dh, 0))
    return _conv_common(x, (2 * Cc, Wo, 2, Ho, N),
                        (2 * Cc * 2, W * Cc * 2, 2 * W * Cc * 2, H * W * Cc * 2),
                        (64, b1, 1, b2, b3), w, Cout, Cc, taps, (Wo, Ho, N), (b1, b2, b3), (1, 3, 4), bias, out, epi)


def tconv3(x, w, bias=None, *, out=None, **epi):
    """(3,1,1) temporal conv (time_stack ResBlock, video_model.py:46-59).  x: [B, T, P, C] bf16 contiguous
    (P = H*W pixels); w: packed [3, Cout, C]; zero pad 1 along T.  Returns [B*T*P, Cout] rows."""
    assert x.dtype == torch.bfloat16 and x.dim() == 4 and x.is_contiguous()
    B, T, P, Cc = x.shape
    Cout = w.shape[1]
    assert w.shape == (3, Cout, Cc) and w.is_contiguous()
    b1, b2, b3 = pick_box(P, T, B)
    taps = [(0, 0, dt - 1, 0, 0) for dt in range(3)]
    return _conv_common(x, (Cc, P, T, B, 1), (Cc * 2, P * Cc * 2, T * P * Cc * 2, B * T * P * Cc * 2),
                        (64, b1, b2, b3, 1), w, Cout, Cc, taps, (P, T, B), (b1, b2, b3), (1, 2, 3), bias, out, epi)


def _conv_common(x, a_dims, a_strides, a_box, w, Cout, K, taps, m_ext, m_box, m_adim, bias, out, epi, out_rs=None):
    rows = m_ext[0] * m_ext[1] * m_ext[2]
    act = epi.pop("act", ACT_NONE)
    out_fp32 = epi.pop("out_fp32", False)
    bn = epi.pop("bn", 0)
    n_out = Cout // 2 if act == ACT_GEGLU else Cout
    out = _alloc_out(rows, n_out, out, out_fp32, x.device)
    kw = _epi_kwargs(rows, n_out, out, bias, epi.pop("fvec", None), epi.pop("rows_per_frame", 1), act,
                     epi.pop("s_acc", 1.0), epi.pop("res1", None), epi.pop("s1", 1.0), epi.pop("res2", None),
                     epi.pop("s2", 1.0), out_fp32, epi.pop("slope", None))
    gn = _gn_request(epi.pop("gn_rows", None), m_ext, m_box, n_out, act, out_fp32, x.device)
    assert not epi, f"unknown epilogue args {list(epi)}"
    gemm_raw(a=x, a_dims=a_dims, a_strides=a_strides, a_box=a_box, w=w, n=Cout, k=K, taps=len(taps), tap_off=taps,
             m_ext=m_ext, m_box=m_box, m_adim=m_adim, out=out, ldo=out.stride(0), out_rs=out_rs, bn=bn, gn=gn, **kw)
    if gn is not None:
        out._b200_gn = gn
    return out


# ----------------------------------------------------------------------------------------------------------------
# attention
# ----------------------------------------------------------------------------------------------------------------
_FAMILY = {"b200svd_flash_attn": "flash_attn", "b200svd_flash_attn_d80": "flash_attn",
           "b200svd_clip_preprocess": "clip_preprocess", "b200svd_small_attn": "small_attn", "b200svd_pixel_attn": "pixel_attn", "b200svd_gn_stats": "groupnorm",
           "b200svd_gn_stats_partials": "groupnorm",
           "b200svd_gn_apply": "groupnorm", "b200svd_layernorm": "layernorm",
           "b200svd_resize_bicubic_u8": "resize"}


def _call(name, *args, flops=0.0, nbytes=0.0, desc=""):
    global _launch_count
    lib = _lib.load()
    e0 = _prof_begin()
    _lib.check(getattr(lib, name)(*args), name)
    _launch_count += 1
    if e0 is not None:
        fam = _FAMILY.get(name, "glue")
        _prof_end(e0, (fam, desc) if desc else fam, flops, nbytes)


def _flash_attn(entry, d, desc, qkv, n, s, heads, out):
    assert qkv.dtype == torch.bfloat16 and qkv.dim() == 2 and qkv.stride(1) == 1
    Cc = heads * d
    assert qkv.shape[0] == n * s and qkv.shape[1] >= 3 * Cc
    if out is None:
        out = torch.empty((n * s, Cc), dtype=torch.bfloat16, device=qkv.device)
    assert out.dtype == torch.bfloat16 and out.stride(1) == 1 and out.shape == (n * s, Cc)
    _call(entry, _ptr(qkv), qkv.stride(0), _ptr(out), out.stride(0), n, s, heads, d ** -0.5, _stream(),
          flops=4.0 * n * heads * float(s) * s * d, nbytes=2.0 * n * s * 4 * Cc, desc=desc)
    return out


def flash_attn(qkv, n, s, heads, out=None):
    """qkv: [(n s), >= 3*heads*64] bf16 (row stride free; columns [q | k | v] each heads*64 wide)
    -> [(n s), heads*64]."""
    return _flash_attn("b200svd_flash_attn", 64, f"n{n} s{s} h{heads}", qkv, n, s, heads, out)


def flash_attn_d80(qkv, n, s, heads, out=None):
    """Head dim 80 (CLIP ViT-H/14 tower).  qkv: [(n s), >= 3*heads*80] bf16 (row stride free; columns [q | k | v]
    each heads*80 wide) -> [(n s), heads*80]."""
    return _flash_attn("b200svd_flash_attn_d80", 80, f"d80 n{n} s{s} h{heads}", qkv, n, s, heads, out)


CLIP_PATCH_K = 14 * 14 * 3          # 588 columns of the patch-embedding A operand
CLIP_PATCH_LD = 592                 # padded to a multiple of 8 (16-byte TMA rows)


def clip_preprocess(x, taps_y, taps_x, out=None):
    """CLIP preprocessing + ViT-H/14 patch gather.  x: [n, 3, H, W] fp32 contiguous in [-1, 1]; taps_y / taps_x: the
    normalised 1-D Gaussian antialias taps (host sequences, odd lengths; [1.0] = no blur).
    Returns the patch GEMM's A operand, bf16 [(n 256), 592], column (kh*14 + kw)*3 + c, columns 588.. zero."""
    assert x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3 and x.is_contiguous()
    n, _, H, W = x.shape
    if out is None:
        out = torch.empty((n * 256, CLIP_PATCH_LD), dtype=torch.bfloat16, device=x.device)
    assert out.dtype == torch.bfloat16 and out.stride(1) == 1 and out.shape[0] == n * 256
    ty = (C.c_float * len(taps_y))(*[float(v) for v in taps_y])
    tx = (C.c_float * len(taps_x))(*[float(v) for v in taps_x])
    _call("b200svd_clip_preprocess", _ptr(x), n, H, W, _ptr(out), out.stride(0), ty, len(taps_y), tx, len(taps_x),
          _stream(), nbytes=4.0 * x.numel() + 2.0 * out.numel(), desc=f"n{n} {H}x{W} taps{len(taps_y)}x{len(taps_x)}")
    return out


def linear_grouped(x, w, bias=None, *, groups, out, out_group_rows, **epi):
    """`linear` over `groups` equal blocks of rows of x ([(groups rows), K]) whose outputs land in blocks of
    out_group_rows rows of `out`: input row r of group g -> output row g * out_group_rows + r (the GEMM's out_rs).
    Used to write the patch embedding straight into token rows 1..256 of each image."""
    assert x.dtype == torch.bfloat16 and x.dim() == 2 and x.stride(1) == 1
    M, K = x.shape
    assert M % groups == 0
    rows = M // groups
    N = w.shape[-2]
    assert w.shape[-1] == K and w.is_contiguous() and out.stride(-1) == 1
    assert out.shape[1] == N and (groups - 1) * out_group_rows + rows <= out.shape[0]
    ld = x.stride(0)
    big = ld * 2 * max(M, 1)
    act = epi.pop("act", ACT_NONE)
    out_fp32 = epi.pop("out_fp32", False)
    kw = _epi_kwargs(M, N, out, bias, epi.pop("fvec", None), epi.pop("rows_per_frame", 1), act,
                     epi.pop("s_acc", 1.0), epi.pop("res1", None), epi.pop("s1", 1.0), epi.pop("res2", None),
                     epi.pop("s2", 1.0), out_fp32)
    assert not epi, f"unknown epilogue args {list(epi)}"
    gemm_raw(a=x, a_dims=(K, rows, groups, 1, 1), a_strides=(ld * 2, rows * ld * 2, big, big),
             a_box=(64, 128, 1, 1, 1), w=w, n=N, k=K, taps=1, tap_off=[(0, 0, 0, 0, 0)], m_ext=(rows, groups, 1),
             m_box=(128, 1, 1), m_adim=(1, 2, 3), out=out, ldo=out.stride(0),
             out_rs=(1, out_group_rows, groups * out_group_rows), **kw)
    return out


def small_attn(q, k, v, *, b, s, heads, lq, lk, kv_per_pixel=True, out=None):
    """q: rows (b, i<lq, s); k, v: rows (b, j<lk, s) or (b, j) when kv_per_pixel=False; head dim 64.
    q/k/v/out need 16-byte aligned bases and leading dims that are multiples of 8 (both kernels check)."""
    for t in (q, k, v):
        assert t.dtype == torch.bfloat16 and t.dim() == 2 and t.stride(1) == 1
    Cc = heads * 64
    if out is None:
        out = torch.empty((b * lq * s, Cc), dtype=torch.bfloat16, device=q.device)
    if kv_per_pixel:
        # tensor-core path: 4 pixels x 32 padded frames per CTA, wgmma tiles
        _call("b200svd_pixel_attn", _ptr(q), q.stride(0), _ptr(k), k.stride(0), _ptr(v), v.stride(0), _ptr(out),
              out.stride(0), b, s, heads, lq, lk, 64 ** -0.5, _stream(),
              flops=4.0 * b * s * heads * lq * lk * 64, nbytes=2.0 * Cc * (2 * b * lq * s + 2 * b * lk * s),
              desc=f"b{b} s{s} h{heads} {lq}x{lk}")
        return out
    _call("b200svd_small_attn", _ptr(q), q.stride(0), _ptr(k), k.stride(0), _ptr(v), v.stride(0), _ptr(out),
          out.stride(0), b, s, heads, lq, lk, 1 if kv_per_pixel else 0, 64 ** -0.5, _stream(),
          flops=4.0 * b * s * heads * lq * lk * 64,
          nbytes=2.0 * Cc * (2 * b * lq * s + 2 * b * lk * (s if kv_per_pixel else 1)),
          desc=f"b{b} s{s} h{heads} {lq}x{lk} pp{int(kv_per_pixel)}")
    return out


# ----------------------------------------------------------------------------------------------------------------
# norms
# ----------------------------------------------------------------------------------------------------------------
_GN_SCRATCH = {}
_GN_RETIRED = []   # outgrown buffers stay allocated: a recorded CUDA graph may still point at them


def _gn_scratch(device, doubles, n):
    """Scratch of the deterministic GroupNorm reduction (chunk partials + self-resetting tickets), one per
    (device, stream): kernels on one stream run in order, kernels on different streams (two wrappers, a wrapper and
    the VAE decoder, a graph being recorded) must not share tickets.  Buffers are never freed or moved while the
    process lives — CUDA graphs bake their addresses."""
    key = (str(device), torch.cuda.current_stream().cuda_stream if device.type == "cuda" else 0)
    cur = _GN_SCRATCH.get(key)
    if cur is None or cur[0].numel() < doubles or cur[1].numel() < n:
        if cur is not None:
            _GN_RETIRED.append(cur)
        cur = (torch.empty(max(doubles, 1 << 18), dtype=torch.float64, device=device),
               torch.zeros(max(n, 1024), dtype=torch.int32, device=device))
        _GN_SCRATCH[key] = cur
    return cur


def group_norm(x, n, p, gamma, beta, eps, *, silu=False, out=None, sums=None):
    """x: [(n p), C] bf16 rows; 32 groups; statistics over (p, C/32) per sample n.  Returns bf16 [(n p), C]."""
    assert x.dtype == torch.bfloat16 and x.dim() == 2 and x.stride(1) == 1 and x.shape[0] == n * p
    Cc = x.shape[1]
    if sums is None:
        sums = torch.empty((n, 32, 2), dtype=torch.float64, device=x.device)
    if out is None:
        out = torch.empty((n * p, Cc), dtype=torch.bfloat16, device=x.device)
    gn = getattr(x, "_b200_gn", None)
    if gn is not None and gn["p"] == p and gn["C"] == Cc and x.stride(0) == Cc:
        # the producing GEMM left per-quadrant partial sums: reduce those (12.5 % of the bytes) instead of reading x
        chunks = -(-gn["n_slots"] // 64)
        scratch, counters = _gn_scratch(x.device, n * chunks * 64, n)
        _call("b200svd_gn_stats_partials", _ptr(gn["part"]), _ptr(gn["slot"]), gn["n_slots"], Cc, Cc, n, _ptr(sums),
              _ptr(scratch), _ptr(counters), _stream(), nbytes=8.0 * gn["n_slots"] * Cc,
              desc=f"stats(partials) n{n} p{p} c{Cc}")
    else:
        lib = _lib.load()
        need = lib.b200svd_gn_scratch_doubles(n, p, Cc)
        if need < 0:
            raise _lib.B200Error(f"group_norm: {lib.b200svd_last_error().decode()}")
        scratch, counters = _gn_scratch(x.device, need, n)
        _call("b200svd_gn_stats", _ptr(x), x.stride(0), n, p, Cc, _ptr(sums), _ptr(scratch), _ptr(counters), _stream(),
              nbytes=2.0 * n * p * Cc, desc=f"stats n{n} p{p} c{Cc}")
    _call("b200svd_gn_apply", _ptr(x), x.stride(0), _ptr(out), out.stride(0), n, p, Cc, _ptr(sums), _ptr(gamma),
          _ptr(beta), float(eps), 1 if silu else 0, _stream(), nbytes=4.0 * n * p * Cc, desc=f"apply n{n} p{p} c{Cc}")
    return out


def layer_norm(x, gamma, beta, eps=1e-5, *, fvec=None, rows_per_frame=1, xsum=None, silu=False, out=None):
    assert x.dtype == torch.bfloat16 and x.dim() == 2 and x.stride(1) == 1
    assert xsum is None or fvec is not None, "layer_norm: xsum = bf16(x + fvec) needs fvec"
    rows, Cc = x.shape
    if out is None:
        out = torch.empty((rows, Cc), dtype=torch.bfloat16, device=x.device)
    _call("b200svd_layernorm", _ptr(x), x.stride(0), _ptr(out), out.stride(0), rows, Cc, _ptr(gamma), _ptr(beta),
          float(eps), _ptr(fvec), fvec.stride(0) if fvec is not None else 0, rows_per_frame, _ptr(xsum),
          xsum.stride(0) if xsum is not None else 0, 1 if silu else 0, _stream(),
          nbytes=2.0 * rows * Cc * (2 + (xsum is not None)), desc=f"rows{rows} c{Cc}")
    return out


# ----------------------------------------------------------------------------------------------------------------
# glue
# ----------------------------------------------------------------------------------------------------------------
def nchw_to_nhwc(src, dst, c_off=0):
    """src [N, C, H, W] fp32 (frame stride free, CHW contiguous) -> dst rows [(N H W), ld] bf16 at column c_off."""
    assert src.dtype == torch.float32 and src.dim() == 4
    N, Cs, H, W = src.shape
    assert src.stride(3) == 1 and src.stride(2) == W and src.stride(1) == H * W
    _call("b200svd_nchw_to_nhwc", _ptr(src), src.stride(0), N, Cs, H * W, _ptr(dst), dst.stride(0), c_off, _stream())
    return dst


def nhwc_to_nchw(src, n, c, hw, out):
    assert out.dtype == torch.float32 and out.is_contiguous()
    _call("b200svd_nhwc_to_nchw", _ptr(src), 1 if src.dtype == torch.float32 else 0, src.stride(0), n, c, hw, _ptr(out),
          _stream())
    return out


def upsample2x(x, n, h, w):
    """x: [(n h w), C] bf16 contiguous -> [(n 2h 2w), C]."""
    assert x.dtype == torch.bfloat16 and x.is_contiguous()
    Cc = x.shape[-1]
    y = torch.empty((n * 4 * h * w, Cc), dtype=torch.bfloat16, device=x.device)
    _call("b200svd_upsample2x", _ptr(x), _ptr(y), n, h, w, Cc, _stream())
    return y


def timestep_embed(t, dim, max_period=10000.0):
    assert t.dtype == torch.float32 and t.is_contiguous()
    out = torch.empty((t.numel(), dim), dtype=torch.bfloat16, device=t.device)
    _call("b200svd_timestep_embed", _ptr(t), t.numel(), dim, float(max_period), _ptr(out), out.stride(0), _stream())
    return out


def add_silu(a, b=None, silu=True):
    assert a.dtype == torch.float32 and a.is_contiguous() and (b is None or (b.is_contiguous() and b.shape == a.shape))
    out = torch.empty(a.shape, dtype=torch.bfloat16, device=a.device)
    _call("b200svd_add_silu", _ptr(a), _ptr(b), _ptr(out), a.numel(), 1 if silu else 0, _stream())
    return out


def copy2d(src, dst):
    assert src.shape == dst.shape and src.dim() == 2
    _call("b200svd_copy2d", _ptr(src), src.stride(0), _ptr(dst), dst.stride(0), src.shape[0], src.shape[1], _stream())
    return dst


def add_rows(dst, src):
    """dst[r] += src[r % src_rows] (bf16, in place)."""
    _call("b200svd_add_rows", _ptr(dst), dst.stride(0), _ptr(src), src.stride(0), dst.shape[0], src.shape[0],
          dst.shape[1], _stream())
    return dst


def apm_mix(ctx, w, wb, ln_g, ln_b, alpha):
    """ctx [N, L, D] fp32 -> [N, D] bf16 (attention.py:612-620)."""
    assert ctx.dtype == torch.float32 and ctx.is_contiguous()
    N, L, D = ctx.shape
    out = torch.empty((N, D), dtype=torch.bfloat16, device=ctx.device)
    _call("b200svd_apm_mix", _ptr(ctx), N, L, D, _ptr(w), _ptr(wb), _ptr(ln_g), _ptr(ln_b), _ptr(alpha), _ptr(out),
          _stream())
    return out


def softmax_rows(scores, out=None):
    """scores: fp32 [rows, cols] (already scaled) -> bf16 probabilities."""
    assert scores.dtype == torch.float32 and scores.dim() == 2 and scores.stride(1) == 1
    rows, cols = scores.shape
    if out is None:
        out = torch.empty((rows, cols), dtype=torch.bfloat16, device=scores.device)
    _call("b200svd_softmax_rows", _ptr(scores), scores.stride(0), _ptr(out), out.stride(0), rows, cols, _stream(),
          nbytes=6.0 * rows * cols)
    return out


def transpose(x):
    """bf16 [R, C] -> contiguous [C, R]."""
    assert x.dtype == torch.bfloat16 and x.dim() == 2 and x.stride(1) == 1
    R, Cc = x.shape
    out = torch.empty((Cc, R), dtype=torch.bfloat16, device=x.device)
    _call("b200svd_transpose", _ptr(x), x.stride(0), _ptr(out), out.stride(0), R, Cc, _stream(), nbytes=4.0 * R * Cc)
    return out


def sampler_prepare(x, c_in, out=None):
    """cat([x, x]) * c_in: the doubled, input-scaled latent the denoiser network sees (guiders.py:97,
    denoiser.py:36).  x: contiguous fp32 [(b t), ...] -> [2 (b t), ...]."""
    assert x.dtype == torch.float32 and x.is_contiguous()
    rows = x.shape[0]
    chw = x.numel() // max(rows, 1)
    if out is None:
        out = torch.empty((2 * rows,) + tuple(x.shape[1:]), dtype=torch.float32, device=x.device)
    assert out.dtype == torch.float32 and out.is_contiguous() and out.numel() == 2 * x.numel()
    _call("b200svd_sampler_prepare", _ptr(x), _ptr(out), rows, chw, float(c_in), _stream(), nbytes=12.0 * x.numel())
    return out


def sampler_step(net, x, scale, *, num_frames, c_skip, c_out, sigma, next_sigma, out=None):
    """Denoiser output scaling + LinearPredictionGuider + Euler update in one kernel (denoiser.py:33-39,
    guiders.py:78-86, sampling.py:100-103).  net: fp32 [2 (b t), ...] (unconditional half first), x: fp32
    [(b t), ...], scale: fp32 [num_frames] on the device."""
    assert net.dtype == torch.float32 and net.is_contiguous() and x.dtype == torch.float32 and x.is_contiguous()
    assert net.numel() == 2 * x.numel() and scale.dtype == torch.float32 and scale.numel() == num_frames
    rows = x.shape[0]
    chw = x.numel() // max(rows, 1)
    if out is None:
        out = torch.empty_like(x)
    _call("b200svd_sampler_step", _ptr(net), _ptr(x), _ptr(out), rows, chw, int(num_frames), _ptr(scale),
          float(c_skip), float(c_out), float(sigma), float(next_sigma), _stream(), nbytes=16.0 * x.numel())
    return out


def ddim_blend_step(noise, latents, out, *, lat_start, out_start, offset, guidance, alpha_t, alpha_prev,
                    v_prediction=True):
    """One DDIM step (eta = 0) + CFG combine of one randomized-blending chunk, written into `out` from frame
    `offset` on (pipeline_i2vgen_xl.py:868-903).  noise: fp32 [2 or 1, C, cs, H, W]; latents / out: fp32 [1, C, F, H, W]
    contiguous (they may be different tensors with different F).  guidance=None: no classifier-free guidance."""
    for t_ in (noise, latents, out):
        assert t_.dtype == torch.float32 and t_.is_contiguous() and t_.dim() == 5
    nb, Cc, cs, H, W = noise.shape
    assert nb == (1 if guidance is None else 2) and latents.shape[0] == 1 and out.shape[0] == 1
    assert latents.shape[1] == Cc and out.shape[1] == Cc and latents.shape[3:] == (H, W) and out.shape[3:] == (H, W)
    _call("b200svd_ddim_blend_step", _ptr(noise), _ptr(latents), _ptr(out), Cc, cs, H * W, latents.shape[2],
          int(lat_start), out.shape[2], int(out_start), int(offset), 0 if guidance is None else 1,
          float(guidance or 0.0), float(alpha_t), float(alpha_prev), 1 if v_prediction else 0, _stream(),
          nbytes=4.0 * Cc * cs * H * W * (nb + 2))
    return out


def frames_to_uint8(x, vmin=0.0, vmax=255.0):
    """fp32 [F, C, H, W] in [vmin, vmax] -> uint8 [F, H, W, C] (the array the reference's IImage container holds,
    lib/farancia/libimage/iimage.py:21-39)."""
    assert x.dtype == torch.float32 and x.dim() == 4 and x.is_contiguous()
    Fn, Cc, H, W = x.shape
    out = torch.empty((Fn, H, W, Cc), dtype=torch.uint8, device=x.device)
    _call("b200svd_frames_to_uint8", _ptr(x), _ptr(out), Fn, Cc, H * W, float(vmin), float(vmax), _stream(),
          nbytes=5.0 * x.numel())
    return out


def frames_quantize(x, out=None):
    """fp32 frames in [-1, 1] -> fp32 on the 1/127.5 grid: the 8-bit image round trip of the first chunk
    (diffusers' postprocess_video to PIL, ToTensor(), `* 2.0 - 1`; streaming_svd.py:390-393), rounding half to even."""
    assert x.dtype == torch.float32 and x.is_contiguous()
    if out is None:
        out = torch.empty_like(x)
    assert out.dtype == torch.float32 and out.is_contiguous() and out.shape == x.shape
    _call("b200svd_frames_quantize", _ptr(x), _ptr(out), x.numel(), _stream(), nbytes=8.0 * x.numel())
    return out


def attention_single_head(q, k, v, n, s):
    """softmax(q k^T / sqrt(C)) v per frame, one head of width C (VAE AttnBlock).  q, k, v: contiguous [(n s), C] bf16.
    Built from the tensor-core GEMM (scores in fp32), a row-softmax kernel and a transpose."""
    Cc = q.shape[1]
    out = torch.empty((n * s, Cc), dtype=torch.bfloat16, device=q.device)
    scale = float(Cc) ** -0.5
    for f in range(n):
        sl = slice(f * s, (f + 1) * s)
        scores = linear(q[sl], k[sl][None], None, out_fp32=True, s_acc=scale)          # [s, s] fp32
        probs = softmax_rows(scores)
        vt = transpose(v[sl])                                                           # [C, s]
        linear(probs, vt[None], None, out=out[sl])
    return out


# ----------------------------------------------------------------------------------------------------------------
# EMA-VFI frame interpolation (csrc/vfi.cu)
# ----------------------------------------------------------------------------------------------------------------
_FAMILY.update({"b200svd_vfi_window_attn": "vfi_attn", "b200svd_vfi_warp": "vfi_warp", "b200svd_vfi_resize": "vfi_resize",
                "b200svd_vfi_dwconv_gelu": "vfi_dwconv", "b200svd_vfi_head_gather": "glue", "b200svd_vfi_merge": "glue",
                "b200svd_vfi_pair_input": "glue", "b200svd_vfi_frames_to_bgr": "glue"})


def conv3x3_strided(x, w, bias=None, *, stride, dilation, out=None, **epi):
    """3x3 conv with stride s in {2, 4, 8} and padding = dilation = d < s (CrossScalePatchEmbed,
    feature_extractor.py:352-354).  x: [N, H, W, C] bf16 contiguous, H and W multiples of s.  The input is viewed as
    [N, H/s, s, W/s, s*C]; input row s*i + d*(k-1) is output row i + q at phase r (s*q + r = d*(k-1)), so every tap
    is a shifted TMA box and the rows above / left of the image (q = -1) are the zero padding."""
    assert x.dtype == torch.bfloat16 and x.dim() == 4 and x.is_contiguous()
    N, H, W, Cc = x.shape
    s, d = int(stride), int(dilation)
    assert s in (2, 4, 8) and 1 <= d < s and H % s == 0 and W % s == 0
    Ho, Wo = H // s, W // s
    Cout = w.shape[1]
    assert w.shape == (9, Cout, Cc) and w.is_contiguous()
    b1, b2, b3 = pick_box(Wo, Ho, N)
    taps = []
    for kh in range(3):
        qh, rh = divmod(d * (kh - 1), s)
        for kw in range(3):
            qw, rw = divmod(d * (kw - 1), s)
            taps.append((rw * Cc, qw, rh, qh, 0))
    return _conv_common(x, (s * Cc, Wo, s, Ho, N),
                        (s * Cc * 2, W * Cc * 2, s * W * Cc * 2, H * W * Cc * 2),
                        (64, b1, 1, b2, b3), w, Cout, Cc, taps, (Wo, Ho, N), (b1, b2, b3), (1, 3, 4), bias, out, epi)


# ConvTranspose2d(4, stride 2, padding 1): output row 2i + a takes input rows i - 1 (kernel row 3) and i (1) for a = 0,
# i (2) and i + 1 (0) for a = 1; the same along the width.  (offset, kernel index) per output phase.
DECONV_PHASE_TAPS = (((-1, 3), (0, 1)), ((0, 2), (1, 0)))


def conv_transpose4x4_s2(x, w, bias=None, *, out, **epi):
    """ConvTranspose2d(k=4, s=2, p=1) as one 4-tap GEMM per output phase (a, b): output pixel (2i + a, 2j + b) sums
    the 2x2 input pixels DECONV_PHASE_TAPS names, so each launch is a stride-1 conv with 4 of the 9 taps and its rows
    go straight to every other pixel of the 2x output through the GEMM's output row strides.
    x: [N, H, W, C] bf16 contiguous; w: packed [4 phases (a*2+b), 4 taps, Cout, C]; out: rows [(N 2H 2W), >= Cout]
    (row stride free).  Returns out."""
    assert x.dtype == torch.bfloat16 and x.dim() == 4 and x.is_contiguous()
    N, H, W, Cc = x.shape
    Cout = w.shape[2]
    assert w.shape == (4, 4, Cout, Cc) and w.is_contiguous() and out.shape[0] == N * 4 * H * W
    b1, b2, b3 = pick_box(W, H, N)
    for a in range(2):
        for b in range(2):
            taps = [(0, dx, dy, 0, 0) for dy, _ in DECONV_PHASE_TAPS[a] for dx, _ in DECONV_PHASE_TAPS[b]]
            _conv_common(x, (Cc, W, H, N, 1), (Cc * 2, W * Cc * 2, H * W * Cc * 2, N * H * W * Cc * 2),
                         (64, b1, b2, b3, 1), w[a * 2 + b], Cout, Cc, taps, (W, H, N), (b1, b2, b3), (1, 2, 3), bias,
                         out[a * 2 * W + b:], dict(epi), out_rs=(2, 4 * W, 4 * H * W))
    return out


def vfi_window_attn(qkv, cor_embed, *, pairs, h, w, heads, shift, out, motion):
    """InterFrameAttention of one MotionFormerBlock over all windows (see b200svd_vfi_window_attn).  qkv: bf16 rows
    [2*pairs*h*w + 1, >= 3*heads*32] (last row = padding token); cor_embed: bf16 [h*w + 1, >= heads*8]; out: bf16
    [2*pairs*h*w, >= heads*32]; motion: bf16 [2*pairs*h*w, >= heads*8] (row strides free)."""
    for t in (qkv, cor_embed, out, motion):
        assert t.dtype == torch.bfloat16 and t.dim() == 2 and t.stride(1) == 1
    T = 2 * pairs * h * w
    assert qkv.shape[0] == T + 1 and cor_embed.shape[0] == h * w + 1 and out.shape[0] == T and motion.shape[0] == T
    hp, wp = -(-h // 7) * 7, -(-w // 7) * 7
    blocks = (hp // 7) * (wp // 7) * heads * 2 * pairs
    _call("b200svd_vfi_window_attn", _ptr(qkv), qkv.stride(0), _ptr(cor_embed), cor_embed.stride(0), _ptr(out),
          out.stride(0), _ptr(motion), motion.stride(0), pairs, h, w, heads, shift, 32 ** -0.5, _stream(),
          flops=blocks * 2.0 * 49 * 49 * (32 + 32 + 8), nbytes=blocks * 49 * 2.0 * (3 * 32 + 8 + 32 + 8),
          desc=f"{h}x{w} h{heads} shift{shift}")
    return out, motion


def _nchw_strides(t):
    assert t.dim() == 4
    return [int(v) for v in t.stride()]


def vfi_warp(inp, flow, out):
    """Backward warp (warplayer.warp): out = grid_sample(inp, linspace grid + flow, bilinear, border,
    align_corners=True).  inp / out: [n, c, h, w] views with any element strides (both fp32 or both bf16), flow:
    [n, 2, h, w] fp32 view (x then y)."""
    n, c, h, w = inp.shape
    assert out.shape == inp.shape and flow.shape == (n, 2, h, w) and flow.dtype == torch.float32
    ib, ob = inp.dtype == torch.bfloat16, out.dtype == torch.bfloat16
    _call("b200svd_vfi_warp", _ptr(inp), int(ib), *_nchw_strides(inp), _ptr(flow), *_nchw_strides(flow), _ptr(out),
          int(ob), *_nchw_strides(out), n, c, h, w, _stream(),
          nbytes=n * h * w * (8.0 + c * (4 * (2 if ib else 4) + (2 if ob else 4))), desc=f"{n}x{c}x{h}x{w}")
    return out


def vfi_resize(inp, out, factor_log2, mul=1.0, accumulate=False):
    """F.interpolate(inp, scale_factor=2**factor_log2, mode="bilinear", align_corners=False) * mul, written to out or,
    with accumulate, added to it.  inp: fp32 [n, c, h, w] view, out: [n, c, h*f, w*f] view (fp32, or bf16 without
    accumulate); any element strides."""
    n, c, h, w = inp.shape
    assert inp.dtype == torch.float32
    f = 2.0 ** factor_log2
    assert out.shape == (n, c, int(h * f), int(w * f))
    ob = out.dtype == torch.bfloat16
    _call("b200svd_vfi_resize", _ptr(inp), *_nchw_strides(inp), _ptr(out), int(ob), *_nchw_strides(out), n, c, h, w,
          int(factor_log2), float(mul), int(accumulate), _stream(),
          nbytes=out.numel() * (4.0 * (1 + accumulate) + (2 if ob else 4)) + 4.0 * inp.numel(),
          desc=f"{n}x{c}x{h}x{w} x2^{factor_log2}")
    return out


def vfi_dwconv_gelu(x, wt, bias, out=None):
    """x: bf16 [N, H, W, C] contiguous; wt: fp32 [9, C] (tap kh*3+kw); bias fp32 [C] -> GELU(dwconv3x3(x) + bias),
    bf16 rows [(N H W), C]."""
    assert x.dtype == torch.bfloat16 and x.dim() == 4 and x.is_contiguous()
    N, H, W, Cc = x.shape
    assert wt.shape == (9, Cc) and wt.dtype == torch.float32 and wt.is_contiguous() and bias.numel() == Cc
    if out is None:
        out = torch.empty((N * H * W, Cc), dtype=torch.bfloat16, device=x.device)
    assert out.is_contiguous() and out.shape == (N * H * W, Cc)
    _call("b200svd_vfi_dwconv_gelu", _ptr(x), _ptr(out), N, H, W, Cc, _ptr(wt), _ptr(bias), _stream(),
          flops=18.0 * x.numel(), nbytes=4.0 * x.numel(), desc=f"{N}x{H}x{W}x{Cc}")
    return out


def vfi_head_gather(mf, af, *, pairs, h, w, out):
    """Head input at timestep 0.5 (see b200svd_vfi_head_gather): mf, af bf16 rows [2*pairs*h*w, c] -> out bf16 rows
    [pairs*4h*4w, >= c/4] (columns 0..c/4-1 written)."""
    c = mf.shape[1]
    assert af.shape[1] == c and mf.shape[0] == af.shape[0] == 2 * pairs * h * w and out.shape[0] == pairs * 16 * h * w
    for t in (mf, af, out):
        assert t.dtype == torch.bfloat16 and t.stride(1) == 1
    _call("b200svd_vfi_head_gather", _ptr(mf), mf.stride(0), _ptr(af), af.stride(0), pairs, h, w, c, _ptr(out),
          out.stride(0), _stream(), nbytes=8.0 * mf.numel(), desc=f"{h}x{w} c{c}")
    return out


def vfi_merge(warped0, warped1, fm, res, *, pred=None, frame=None):
    """Final fast-TTA prediction (see b200svd_vfi_merge): warped0/1 fp32 [2, 3, H, W], fm fp32 [2, 5, H, W] (channel 4
    = mask logit), res fp32 rows [2*H*W, >= 3] (pre-sigmoid refinement).  Writes pred fp32 [1, 3, H, W] (BGR) and/or
    frame uint8 [H, W, 3] (RGB)."""
    _, _, H, W = warped0.shape
    for t in (warped0, warped1, fm):
        assert t.dtype == torch.float32 and t.is_contiguous() and t.shape[0] == 2 and t.shape[2:] == (H, W)
    assert res.dtype == torch.float32 and res.stride(1) == 1 and res.shape[0] == 2 * H * W
    assert pred is None or (pred.dtype == torch.float32 and pred.is_contiguous() and pred.numel() == 3 * H * W)
    assert frame is None or (frame.dtype == torch.uint8 and frame.is_contiguous() and frame.shape == (H, W, 3))
    _call("b200svd_vfi_merge", _ptr(warped0), _ptr(warped1), _ptr(fm), _ptr(res), res.stride(0), H, W, _ptr(pred),
          _ptr(frame), _stream(), nbytes=H * W * (4.0 * 2 * (3 + 3 + 1 + 3) + 12 + 3), desc=f"{H}x{W}")
    return pred, frame


def vfi_pair_input(img0, img1, imgs, x8):
    """img0, img1: fp32 [1, 3, H, W] contiguous -> imgs fp32 [4, 3, H, W] = [img0, flip(img0), img1, flip(img1)] and
    x8 bf16 [4, H, W, 8] (channels 3..7 zero)."""
    _, _, H, W = img0.shape
    for t in (img0, img1):
        assert t.dtype == torch.float32 and t.is_contiguous() and t.shape == (1, 3, H, W)
    assert imgs.shape == (4, 3, H, W) and imgs.is_contiguous() and x8.shape == (4, H, W, 8) and x8.is_contiguous()
    _call("b200svd_vfi_pair_input", _ptr(img0), _ptr(img1), H, W, _ptr(imgs), _ptr(x8), _stream(),
          nbytes=H * W * (24.0 + 48 + 64), desc=f"{H}x{W}")
    return imgs, x8


def vfi_frames_to_bgr(frames, out=None):
    """uint8 RGB [F, H, W, 3] contiguous -> fp32 BGR [F, 3, H, W] in [0, 1] (u / 255.0 rounded to float)."""
    assert frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3 and frames.is_contiguous()
    Fn, H, W, _ = frames.shape
    if out is None:
        out = torch.empty((Fn, 3, H, W), dtype=torch.float32, device=frames.device)
    assert out.is_contiguous() and out.shape == (Fn, 3, H, W) and out.dtype == torch.float32
    _call("b200svd_vfi_frames_to_bgr", _ptr(frames), Fn, H, W, _ptr(out), _stream(), nbytes=15.0 * frames.numel() / 3,
          desc=f"{Fn}x{H}x{W}")
    return out


# ----------------------------------------------------------------------------------------------------------------
# PIL's BICUBIC resize of uint8 frames
# ----------------------------------------------------------------------------------------------------------------
RESIZE_PRECISION_BITS = 22          # Pillow's PRECISION_BITS for 8-bit images


def _pil_bicubic(x: float) -> float:
    """Pillow's bicubic_filter (a = -0.5)."""
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1.0
    if x < 2.0:
        return (((x - 5.0) * x + 8.0) * x - 4.0) * a
    return 0.0


@lru_cache(maxsize=None)
def bicubic_taps(in_size: int, out_size: int):
    """Integer taps of Pillow's 8-bit BICUBIC resize along one axis of in_size -> out_size samples, computed in double
    precision in Pillow's order (libImaging/Resample.c, precompute_coeffs and normalize_coeffs_8bpc).  Returns CPU
    int32 tensors: bounds [out_size, 2] = (first source index, tap count) and taps [out_size, k] in 2^-22 units,
    zero past each tap count.  Cached per size pair; do not modify the result."""
    scale = in_size / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ss = 1.0 / filterscale
    one = float(1 << RESIZE_PRECISION_BITS)
    bounds, rows = [], []
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        n = min(int(center + support + 0.5), in_size) - xmin
        w = [_pil_bicubic((x + xmin - center + 0.5) * ss) for x in range(n)]
        total = 0.0
        for v in w:                     # left to right, as Pillow does (Python's sum() of floats is compensated)
            total += v
        if total != 0.0:
            w = [v / total for v in w]
        rows.append([int(v * one - 0.5) if v < 0 else int(v * one + 0.5) for v in w])
        bounds.append((xmin, n))
    k = max(len(r) for r in rows)
    taps = torch.tensor([r + [0] * (k - len(r)) for r in rows], dtype=torch.int32)
    return torch.tensor(bounds, dtype=torch.int32), taps


@lru_cache(maxsize=None)
def _bicubic_taps_on(in_size: int, out_size: int, device: torch.device):
    bounds, taps = bicubic_taps(in_size, out_size)
    return bounds.to(device), taps.to(device)


def resize_bicubic_u8(x, W, H):
    """`PIL.Image.resize((W, H))` with BICUBIC, byte for byte, for a batch of uint8 RGB frames: x uint8 [F, h, w, 3]
    on a CUDA device -> uint8 [F, H, W, 3] on the same device.  Raises ValueError for any other input."""
    if not isinstance(x, torch.Tensor) or x.dtype != torch.uint8 or x.dim() != 4 or x.shape[3] != 3 or not x.is_cuda:
        got = f"{tuple(x.shape)} {x.dtype} on {x.device}" if isinstance(x, torch.Tensor) else type(x).__name__
        raise ValueError(f"resize_bicubic_u8 takes uint8 [F, H, W, 3] frames on a CUDA device, got {got}")
    try:
        W, H = operator.index(W), operator.index(H)
    except TypeError:
        raise ValueError(f"resize_bicubic_u8: W and H must be integers, got {W!r}, {H!r}") from None
    Fn, h, w, _ = x.shape
    if W < 1 or H < 1 or h < 1 or w < 1:
        raise ValueError(f"resize_bicubic_u8: sizes must be positive, got {w}x{h} -> {W}x{H}")
    x = x.contiguous()
    dev = x.device
    out = torch.empty((Fn, H, W, 3), dtype=torch.uint8, device=dev)
    bx, tx = _bicubic_taps_on(w, W, dev) if W != w else (None, None)
    by, ty = _bicubic_taps_on(h, H, dev) if H != h else (None, None)
    ws = torch.empty((Fn, h, W, 3), dtype=torch.uint8, device=dev) if (W != w and H != h) else None
    _call("b200svd_resize_bicubic_u8", _ptr(x), Fn, h, w, _ptr(out), H, W, _ptr(bx), _ptr(tx),
          0 if tx is None else tx.shape[1], _ptr(by), _ptr(ty), 0 if ty is None else ty.shape[1], _ptr(ws), _stream(),
          nbytes=float(x.numel() + out.numel() + (2 * ws.numel() if ws is not None else 0)),
          desc=f"{Fn}x{w}x{h}->{W}x{H}")
    return out
