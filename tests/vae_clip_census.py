"""TEST INFRASTRUCTURE — the launch census of the three image stages of every chunk: the temporal VAE decoder
(B200VaeDecoder.decode), the SD-VAE encoder (B200VaeEncoder.encode) and the OpenCLIP ViT-H/14 image tower
(B200ClipImageEncoder.encode), at the sizes they run at.  The stages run on the `meta` device with the shape-only ops
of tests/denoiser_census.py (whose record layouts apply) plus the stand-ins below, so the census needs no GPU.

Extra records:
conv3x3_s2_pad_after:   a GEMM record as conv3x3_s2's, for conv3x3_s2(pad_after_only=True) (the autoencoder's
                        Downsample: pad (0, 1, 0, 1), then a padding-0 stride-2 conv)
linear_grouped:         (op, x shape, x row stride, w shape, act, out_fp32, bias, groups, out_group_rows, out shape,
                        out row stride, out row offset in its buffer)
attention_single_head:  (op, n, s, C)
flash_attn_d80:         (op, n, s, heads, qkv row stride, out row stride)
clip_preprocess:        (op, x shape, y taps, x taps)"""
from __future__ import annotations

import torch

from denoiser_census import GEMM_OPS as _DENOISER_GEMM_OPS
from denoiser_census import Recorder, _alloc, _meta_state_dict

GEMM_OPS = _DENOISER_GEMM_OPS + ("conv3x3_s2_pad_after",)

# name -> (stage, frames or images, timesteps); every configuration runs at a 576x1024 frame (latent 72x128)
CONFIGS = {
    "decode8": ("decode", 8, 8),           # the 8-frame groups of a 25-frame chunk
    "decode1": ("decode", 1, 1),           # its 25th frame
    "encode": ("encode", 1, None),         # the conditioning frame
    "clip": ("clip", 1, None),             # the conditioning image
}
H, W = 576, 1024


class StageRecorder(Recorder):
    """Recorder with the ops the image stages call beyond the denoiser's."""

    def ops(self):
        ns = super().ops()
        r = self

        def linear_grouped(x, w, bias=None, *, groups, out, out_group_rows, act=0, out_fp32=False):
            r.calls.append(("linear_grouped", tuple(x.shape), x.stride(0), tuple(w.shape), int(act), bool(out_fp32),
                            bias is not None, int(groups), int(out_group_rows), tuple(out.shape), out.stride(0),
                            out.storage_offset() // out.stride(0)))
            return out

        def attention_single_head(q, k, v, n, s):
            for t in (q, k, v):
                assert t.is_contiguous() and t.shape == (n * s, q.shape[1]), "attention operands are contiguous"
            r.calls.append(("attention_single_head", n, s, q.shape[1]))
            return torch.empty((n * s, q.shape[1]), dtype=torch.bfloat16, device=q.device)

        def flash_attn_d80(qkv, n, s, heads, out=None):
            out = _alloc(n * s, heads * 80, out, False, qkv.device)
            r.calls.append(("flash_attn_d80", n, s, heads, qkv.stride(0), out.stride(0)))
            return out

        def clip_preprocess(x, taps_y, taps_x, out=None):
            r.calls.append(("clip_preprocess", tuple(x.shape), len(taps_y), len(taps_x)))
            return _alloc(x.shape[0] * 256, 592, out, False, x.device)

        for f in (linear_grouped, attention_single_head,flash_attn_d80, clip_preprocess):
            setattr(ns, f.__name__, f)
        return ns


def _encoder_state_dict(cfg):
    """Meta tensors, except conv_out / quant_conv: the encoder folds them in float64 on the host at construction."""
    from streamingt2v_b200 import arch
    shapes = arch.vae_encoder_param_shapes(cfg)
    sd = _meta_state_dict(shapes)
    for k, v in shapes.items():
        if k.startswith(("conv_out.", "quant_conv.")):
            sd[k] = torch.zeros(v)
    return sd


def census(config):
    """The distinct launches of `config` (a CONFIGS key), in first-call order, and the number of calls of each."""
    from streamingt2v_b200 import arch, conditioner, vae
    stage, n, T = CONFIGS[config]
    meta = lambda *s: torch.empty(s, device="meta")  # noqa: E731
    rec = StageRecorder()
    mod = conditioner if stage == "clip" else vae
    real = mod.ops
    mod.ops = rec.ops()
    try:
        if stage == "decode":
            cfg = arch.VaeConfig()
            dec = vae.B200VaeDecoder(cfg, _meta_state_dict(arch.vae_decoder_param_shapes(cfg)), "meta")
            dec.decode(meta(n, cfg.z_channels, H // 8, W // 8), timesteps=T)
        elif stage == "encode":
            cfg = arch.VaeConfig()
            vae.B200VaeEncoder(cfg, _encoder_state_dict(cfg), "meta").encode(meta(n, 3, H, W))
        else:
            cfg = arch.ClipVisionConfig()
            enc = conditioner.B200ClipImageEncoder(cfg, _meta_state_dict(arch.clip_visual_param_shapes(cfg)), "meta")
            enc.encode(meta(n, 3, H, W))
    finally:
        mod.ops = real
    counts = {}
    for call in rec.calls:
        counts[call] = counts.get(call, 0) + 1
    return list(counts), counts
