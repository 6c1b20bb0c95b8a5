"""TEST INFRASTRUCTURE — the launch census of one B200Denoiser.forward: every op call `streamingt2v_b200.model` makes,
with the shapes, leading dimensions, column offsets and epilogue flags that decide its indexing.  The network runs on
the `meta` device with shape-only stand-ins for the ops, so the census needs no GPU and no memory.

GEMM records:  (op, x shape, x row stride, w shape, act, out_fp32, bias, fvec, res1 row stride or 0, res2 row stride
                or 0, scales, bn, out shape, out row stride, out column offset)
               fvec = (rows, row stride, column offset, rows_per_frame) of the per-frame vector, or ();
               scales = (s_acc != 1, s1 != 1, s2 != 1): which blend weights the launch passes (their values come
               from the weights, so only whether they are the identity is part of the launch)
flash_attn:    (op, n, s, heads, qkv row stride, out row stride)
small_attn:    ("pixel_attn" / "small_attn", b, s, heads, lq, lk, (row stride, column offset) of q, k, v, out row
               stride); the column offsets say where q, k and v sit in their shared buffers
group_norm:    (op, x shape, x row stride, n, p, eps, silu, out row stride)
layer_norm:    (op, x shape, x row stride, out row stride, eps, fvec as above, xsum row stride or 0, silu)
glue:          (op, ...) as each stand-in below states."""
from __future__ import annotations

import dataclasses
import types

import torch

GEMM_OPS = ("linear", "conv3x3", "conv3x3_s2", "tconv3")

# the three forwards the denoiser runs: name -> (use_apm, context tokens, ControlNet)
CONFIGS = {
    "streaming": (False, 1, True),          # bench.py's step: ControlNet on 7 frames, one context token
    "apm": (True, 17, True),                # the streaming chunk with the APM context tokens
    "first_chunk": (False, 1, False),       # no ControlNet: the skips are copied into the concat buffers
}


def _col(t):
    """Column offset of a row-major 2-D view inside its buffer."""
    return t.storage_offset() % t.stride(0) if t.dim() == 2 else 0


def _rows_ld(x):
    return x.stride(0) if x.dim() == 2 else x.shape[-1]


def _fvec(f, rpf):
    return (f.shape[0], f.stride(0), _col(f), int(rpf)) if f is not None else ()


def _ld0(t):
    """Row stride of a GEMM input or residual; they all start at column 0 of their buffers (else the record would
    need their column offset)."""
    assert _col(t) == 0, "a GEMM operand at a column offset: record it"
    return _rows_ld(t)


def _alloc(rows, n, out, out_fp32, dev):
    if out is None:
        out = torch.empty((rows, n), dtype=torch.float32 if out_fp32 else torch.bfloat16, device=dev)
    return out


class Recorder:
    def __init__(self):
        self.calls = []

    def _gemm(self, op, x, w, bias, rows, n, out, act=0, out_fp32=False, fvec=None, rows_per_frame=1, s_acc=1.0,
              res1=None, s1=1.0, res2=None, s2=1.0, bn=0, gn_rows=None):
        n_out = n // 2 if act == 3 else n
        out = _alloc(rows, n_out, out, out_fp32, x.device)
        self.calls.append((op, tuple(x.shape), _ld0(x), tuple(w.shape), int(act), bool(out_fp32),
                           bias is not None, _fvec(fvec, rows_per_frame),
                           _ld0(res1) if res1 is not None else 0, _ld0(res2) if res2 is not None else 0,
                           (s_acc != 1.0, s1 != 1.0, s2 != 1.0), int(bn), tuple(out.shape), out.stride(0), _col(out)))
        return out

    def ops(self):
        r = self

        def linear(x, w, bias=None, *, out=None, **epi):
            return r._gemm("linear", x, w, bias, x.shape[0], w.shape[-2], out, **epi)

        def conv3x3(x, w, bias=None, *, out=None, **epi):
            n, h, wd, _ = x.shape
            return r._gemm("conv3x3", x, w, bias, n * h * wd, w.shape[1], out, **epi)

        def conv3x3_s2(x, w, bias=None, *, out=None, pad_after_only=False, **epi):
            # the autoencoder's padding (tests/vae_clip_census.py) is its own op name: the record layout stays
            op = "conv3x3_s2_pad_after" if pad_after_only else "conv3x3_s2"
            n, h, wd, _ = x.shape
            return r._gemm(op, x, w, bias, n * (h // 2) * (wd // 2), w.shape[1], out, **epi)

        def tconv3(x, w, bias=None, *, out=None, **epi):
            b, t, p, _ = x.shape
            return r._gemm("tconv3", x, w, bias, b * t * p, w.shape[1], out, **epi)

        def group_norm(x, n, p, gamma, beta, eps, *, silu=False, out=None):
            out = _alloc(x.shape[0], x.shape[1], out, False, x.device)
            r.calls.append(("group_norm", tuple(x.shape), x.stride(0), n, p, float(eps), bool(silu), out.stride(0)))
            return out

        def layer_norm(x, gamma, beta, eps=1e-5, *, fvec=None, rows_per_frame=1, xsum=None, silu=False, out=None):
            out = _alloc(x.shape[0], x.shape[1], out, False, x.device)
            r.calls.append(("layer_norm", tuple(x.shape), x.stride(0), out.stride(0), float(eps),
                            _fvec(fvec, rows_per_frame), xsum.stride(0) if xsum is not None else 0, bool(silu)))
            return out

        def flash_attn(qkv, n, s, heads, out=None):
            out = _alloc(n * s, heads * 64, out, False, qkv.device)
            r.calls.append(("flash_attn", n, s, heads, qkv.stride(0), out.stride(0)))
            return out

        def small_attn(q, k, v, *, b, s, heads, lq, lk, kv_per_pixel=True, out=None):
            out = _alloc(b * lq * s, heads * 64, out, False, q.device)
            r.calls.append(("pixel_attn" if kv_per_pixel else "small_attn", b, s, heads, lq, lk,
                            tuple((t.stride(0), _col(t)) for t in (q, k, v)), out.stride(0)))
            return out

        def timestep_embed(t, dim, max_period=10000.0):
            r.calls.append(("timestep_embed", t.numel(), dim, float(max_period)))
            return torch.empty((t.numel(), dim), dtype=torch.bfloat16, device=t.device)

        def add_silu(a, b=None, silu=True):
            r.calls.append(("add_silu", tuple(a.shape), b is not None, bool(silu)))
            return torch.empty(a.shape, dtype=torch.bfloat16, device=a.device)

        def apm_mix(ctx, w, wb, ln_g, ln_b, alpha):
            r.calls.append(("apm_mix", tuple(ctx.shape)))
            return torch.empty((ctx.shape[0], ctx.shape[2]), dtype=torch.bfloat16, device=ctx.device)

        def nchw_to_nhwc(src, dst, c_off=0):
            r.calls.append(("nchw_to_nhwc", tuple(src.shape), src.stride(0), tuple(dst.shape), dst.stride(0),
                            int(c_off)))
            return dst

        def nhwc_to_nchw(src, n, c, hw, out):
            r.calls.append(("nhwc_to_nchw", tuple(src.shape), str(src.dtype)[6:], src.stride(0), n, c, hw))
            return out

        def upsample2x(x, n, h, w):
            r.calls.append(("upsample2x", tuple(x.shape), n, h, w))
            return torch.empty((n * 4 * h * w, x.shape[1]), dtype=x.dtype, device=x.device)

        def copy2d(src, dst):
            r.calls.append(("copy2d", tuple(src.shape), src.stride(0), dst.stride(0), _col(dst)))
            return dst

        def add_rows(dst, src):
            r.calls.append(("add_rows", tuple(dst.shape), dst.stride(0), tuple(src.shape), src.stride(0)))
            return dst

        ns = {k: v for k, v in locals().items() if callable(v) and not k.startswith("_") and k != "r"}
        ns["_lib"] = types.SimpleNamespace(init=lambda index: None)
        return types.SimpleNamespace(**ns)


def _meta_state_dict(shapes):
    """Meta tensors, except the parameters the host reads as numbers (the blend factors): real CPU zeros."""
    return {k: torch.zeros(v) if "mix_factor" in k else torch.empty(v, device="meta") for k, v in shapes.items()}


def census(config, B=2, T=25, h=72, w=128):
    """The distinct launches of one forward of `config` (a CONFIGS key) at B x T frames of h x w latents, in first-call
    order, and the number of calls of each."""
    from streamingt2v_b200 import arch, model
    use_apm, L, ctrl = CONFIGS[config]
    cfg = dataclasses.replace(arch.UNetConfig(), use_apm=use_apm)
    rec = Recorder()
    real = model.ops
    model.ops = rec.ops()
    try:
        sd_c = _meta_state_dict(arch.controlnet_param_shapes(cfg)) if ctrl else None
        net = model.B200Denoiser(cfg, _meta_state_dict(arch.unet_param_shapes(cfg)), sd_c, "meta")
        N = B * T
        meta = lambda *s: torch.empty(s, device="meta")  # noqa: E731
        c = {"concat": meta(N, 4, h, w), "crossattn": meta(N, L, cfg.context_dim), "vector": meta(N, cfg.adm_in_channels)}
        cf = meta(1, cfg.num_frame_conditioning, 3, 8 * h, 8 * w) if ctrl else None
        net.forward(meta(N, 4, h, w), meta(N), c, batch_size=B, num_video_frames=T, ctrl_frames=cf)
    finally:
        model.ops = real
    counts = {}
    for call in rec.calls:
        counts[call] = counts.get(call, 0) + 1
    return list(counts), counts
