"""TEST INFRASTRUCTURE — the launch census of one B200VFI._predict: every op call `streamingt2v_b200.vfi` makes, with
the shapes, leading dimensions, column offsets and epilogue flags that decide its indexing.  The network runs on the
`meta` device with shape-only stand-ins for the ops, so the census needs no GPU and no memory.

GEMM records:  (op, x shape, x row stride, w shape, act, out_fp32, PReLU, res1 row stride or 0, out shape, out row
                stride, out column offset, extra)  extra = (stride, dilation) for conv3x3_strided, else ()
other records: (op, ...) as each stand-in below states; vfi_warp and vfi_resize give every operand's _layout."""
from __future__ import annotations

import types

import torch

from streamingt2v_b200 import ops as _real_ops

GEMM_OPS = ("linear", "conv3x3", "conv3x3_s2", "conv3x3_strided", "conv_transpose4x4_s2")


def _col(t):
    """Column offset of a row-major 2-D view inside its buffer."""
    return t.storage_offset() % t.stride(0) if t.dim() == 2 else 0


def _layout(t):
    """(element strides, element offset into its buffer, buffer elements) of a strided view: where a kernel that takes
    element strides reads or writes, e.g. fm[:, 2:4] as the second warp's flow or a column slice of a concat."""
    return tuple(t.stride()), t.storage_offset(), t.untyped_storage().nbytes() // t.element_size()


def _rows_ld(x):
    return x.stride(0) if x.dim() == 2 else x.shape[-1]


def _alloc(rows, n, out, out_fp32, dev):
    if out is None:
        out = torch.empty((rows, n), dtype=torch.float32 if out_fp32 else torch.bfloat16, device=dev)
    return out


class Recorder:
    def __init__(self):
        self.calls = []

    def _gemm(self, op, x, w, rows, n, out, extra=(), act=0, out_fp32=False, slope=None, res1=None, **_):
        out = _alloc(rows, n, out, out_fp32, x.device)
        self.calls.append((op, tuple(x.shape), _rows_ld(x), tuple(w.shape), int(act), bool(out_fp32),
                           slope is not None, res1.stride(0) if res1 is not None else 0, tuple(out.shape),
                           out.stride(0), _col(out), extra))
        return out

    def ops(self):
        r = self

        def linear(x, w, bias=None, *, out=None, **epi):
            return r._gemm("linear", x, w, x.shape[0], w.shape[-2], out, **epi)

        def conv3x3(x, w, bias=None, *, out=None, **epi):
            n, h, wd, _ = x.shape
            return r._gemm("conv3x3", x, w, n * h * wd, w.shape[1], out, **epi)

        def conv3x3_s2(x, w, bias=None, *, out=None, **epi):
            n, h, wd, _ = x.shape
            return r._gemm("conv3x3_s2", x, w, n * (h // 2) * (wd // 2), w.shape[1], out, **epi)

        def conv3x3_strided(x, w, bias=None, *, stride, dilation, out=None, **epi):
            n, h, wd, _ = x.shape
            return r._gemm("conv3x3_strided", x, w, n * (h // stride) * (wd // stride), w.shape[1], out,
                           extra=(stride, dilation), **epi)

        def conv_transpose4x4_s2(x, w, bias=None, *, out, **epi):
            n, h, wd, _ = x.shape
            return r._gemm("conv_transpose4x4_s2", x, w, n * 4 * h * wd, w.shape[2], out, **epi)

        def layer_norm(x, gamma, beta, eps=1e-5, *, out=None, **_):
            out = _alloc(x.shape[0], x.shape[1], out, False, x.device)
            r.calls.append(("layer_norm", tuple(x.shape), x.stride(0), out.stride(0), float(eps)))
            return out

        def copy2d(src, dst):
            r.calls.append(("copy2d", tuple(src.shape), src.stride(0), dst.stride(0), _col(dst)))
            return dst

        def nchw_to_nhwc(src, dst, c_off=0):
            r.calls.append(("nchw_to_nhwc", tuple(src.shape), tuple(src.stride()), dst.stride(0), int(c_off)))
            return dst

        def vfi_pair_input(img0, img1, imgs, x8):
            r.calls.append(("vfi_pair_input", tuple(img0.shape[2:])))
            return imgs, x8

        def vfi_window_attn(qkv, ce, *, pairs, h, w, heads, shift, out, motion):
            r.calls.append(("vfi_window_attn", pairs, h, w, heads, shift, qkv.stride(0), ce.stride(0), out.stride(0),
                            motion.stride(0), _col(motion)))
            return out, motion

        def vfi_warp(inp, flow, out):
            r.calls.append(("vfi_warp", tuple(inp.shape), str(inp.dtype)[6:], _layout(inp), _layout(flow),
                            str(out.dtype)[6:], _layout(out)))
            return out

        def vfi_resize(inp, out, factor_log2, mul=1.0, accumulate=False):
            f = 2.0 ** factor_log2
            shp = (inp.shape[0], inp.shape[1], int(inp.shape[2] * f), int(inp.shape[3] * f))
            assert tuple(out.shape) == shp
            r.calls.append(("vfi_resize", tuple(inp.shape), _layout(inp), str(out.dtype)[6:], _layout(out),
                            int(factor_log2), float(mul), bool(accumulate)))
            return out

        def vfi_dwconv_gelu(x, wt, bias, out=None):
            r.calls.append(("vfi_dwconv_gelu", tuple(x.shape)))
            n, h, w, c = x.shape
            return _alloc(n * h * w, c, out, False, x.device)

        def vfi_head_gather(mf, af, *, pairs, h, w, out):
            r.calls.append(("vfi_head_gather", tuple(mf.shape), mf.stride(0), af.stride(0), pairs, h, w,
                            out.stride(0), _col(out)))
            return out

        def vfi_merge(warped0, warped1, fm, res, *, pred=None, frame=None):
            r.calls.append(("vfi_merge", tuple(warped0.shape[2:]), res.stride(0), pred is not None, frame is not None))
            return pred, frame

        ns = {k: v for k, v in locals().items() if callable(v) and not k.startswith("_") and k != "r"}
        ns["DECONV_PHASE_TAPS"] = _real_ops.DECONV_PHASE_TAPS
        return types.SimpleNamespace(**ns)


def census(H=720, W=1280, seed=0):
    """The distinct launches of one _predict at H x W, in first-call order, and the number of calls of each."""
    from streamingt2v_b200 import vfi
    rec = Recorder()
    real = vfi.ops
    vfi.ops = rec.ops()
    try:
        net = vfi.B200VFI(vfi.seeded_state_dict(seed), "meta")
        img = torch.empty((1, 3, H, W), device="meta")
        net._predict(img, img, pred=torch.empty((1, 3, H, W), device="meta"))
    finally:
        vfi.ops = real
    counts = {}
    for c in rec.calls:
        counts[c] = counts.get(c, 0) + 1
    return list(counts), counts
