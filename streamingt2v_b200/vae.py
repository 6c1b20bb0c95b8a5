"""Temporal VAE decoder on the project's kernels — drop-in for `first_stage_model.decode(z, timesteps=n)`
(reference code/models/svd/sgm/models/autoencoder.py:210-212 -> VideoDecoder, temporal_ae.py:291-347; call site
code/diffusion_trainer/streaming_svd.py:143).  Same conventions as model.py: channel-last bf16 rows, every tensor op
is one of our kernels, fp32 accumulation (the reference runs this stage in fp32; tolerance in DESIGN.md)."""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import ops, packing
from .arch import VaeConfig, vae_decoder_plan, vae_encoder_plan
from .model import _sig

SD = Dict[str, torch.Tensor]


class B200VaeDecoder:
    def __init__(self, cfg: VaeConfig, sd: SD, device):
        ops._lib.init(torch.device(device).index or 0)
        self.cfg, self.dev = cfg, torch.device(device)
        P, d = packing, self.dev
        self.plan = vae_decoder_plan(cfg)
        self.w: Dict[str, dict] = {}

        def gn(p):
            return (P.f32(sd[p + ".weight"], d), P.f32(sd[p + ".bias"], d))

        for kind, p, cin, cout in self.plan:
            if kind == "conv_in":
                self.w[p] = dict(conv=(P.pack_conv3x3(sd[p + ".weight"], d), P.f32(sd[p + ".bias"], d)))
            elif kind == "res":
                t = p + ".time_stack"
                e = dict(gn1=gn(p + ".norm1"), conv1=(P.pack_conv3x3(sd[p + ".conv1.weight"], d), P.f32(sd[p + ".conv1.bias"], d)),
                         gn2=gn(p + ".norm2"), conv2=(P.pack_conv3x3(sd[p + ".conv2.weight"], d), P.f32(sd[p + ".conv2.bias"], d)),
                         gn3=gn(t + ".in_layers.0"),
                         tconv1=(P.pack_tconv3(sd[t + ".in_layers.2.weight"], d), P.f32(sd[t + ".in_layers.2.bias"], d)),
                         gn4=gn(t + ".out_layers.0"),
                         tconv2=(P.pack_tconv3(sd[t + ".out_layers.3.weight"], d), P.f32(sd[t + ".out_layers.3.bias"], d)),
                         alpha=_sig(sd[p + ".mix_factor"]), skip=None)
                if (p + ".nin_shortcut.weight") in sd:
                    e["skip"] = (P.pack_conv1x1(sd[p + ".nin_shortcut.weight"], d), P.f32(sd[p + ".nin_shortcut.bias"], d))
                self.w[p] = e
            elif kind == "attn":
                self.w[p] = dict(norm=gn(p + ".norm"),
                                 **{n: (P.pack_conv1x1(sd[f"{p}.{n}.weight"], d), P.f32(sd[f"{p}.{n}.bias"], d))
                                    for n in ("q", "k", "v", "proj_out")})
            elif kind == "up":
                self.w[p] = dict(conv=(P.pack_conv3x3(sd[p + ".conv.weight"], d), P.f32(sd[p + ".conv.bias"], d)))
            elif kind == "out":
                self.w["out"] = dict(gn=gn("norm_out"),
                                     conv=(P.pack_conv3x3(sd["conv_out.weight"], d), P.f32(sd["conv_out.bias"], d)),
                                     tmix=(P.pack_tconv3(sd["conv_out.time_mix_conv.weight"], d),
                                           P.f32(sd["conv_out.time_mix_conv.bias"], d)))
        self.debug_taps: Optional[dict] = None

    def _res(self, p, x, n, T, h, w, cin, cout):
        """VideoResBlock (temporal_ae.py:62-81): spatial ResnetBlock (GN eps 1e-6, swish) + (3,1,1) time stack
        (GroupNorm32 eps 1e-5 over (c/32, t, h, w)) + blend  out = x_s + sigmoid(mix) * time_stack_delta."""
        e = self.w[p]
        S, B = h * w, n // T
        g1 = ops.group_norm(x, n, S, e["gn1"][0], e["gn1"][1], 1e-6, silu=True)
        h1 = ops.conv3x3(g1.view(n, h, w, cin), e["conv1"][0], e["conv1"][1], gn_rows=S)
        g2 = ops.group_norm(h1, n, S, e["gn2"][0], e["gn2"][1], 1e-6, silu=True)
        xs = x if e["skip"] is None else ops.linear(x, e["skip"][0], e["skip"][1])
        x_s = ops.conv3x3(g2.view(n, h, w, cout), e["conv2"][0], e["conv2"][1], res1=xs, s1=1.0, gn_rows=T * S)
        g3 = ops.group_norm(x_s, B, T * S, e["gn3"][0], e["gn3"][1], 1e-5, silu=True)
        h3 = ops.tconv3(g3.view(B, T, S, cout), e["tconv1"][0], e["tconv1"][1], gn_rows=T * S)
        g4 = ops.group_norm(h3, B, T * S, e["gn4"][0], e["gn4"][1], 1e-5, silu=True)
        return ops.tconv3(g4.view(B, T, S, cout), e["tconv2"][0], e["tconv2"][1], s_acc=e["alpha"], res1=x_s, s1=1.0)

    def _attn(self, p, x, n, h, w, c):
        """AttnBlock (model.py:161-201): one head of width c over the h*w tokens of each frame."""
        e = self.w[p]
        S = h * w
        xn = ops.group_norm(x, n, S, e["norm"][0], e["norm"][1], 1e-6, silu=False)
        q = ops.linear(xn, e["q"][0], e["q"][1])
        k = ops.linear(xn, e["k"][0], e["k"][1])
        v = ops.linear(xn, e["v"][0], e["v"][1])
        o = ops.attention_single_head(q, k, v, n, S)
        return ops.linear(o, e["proj_out"][0], e["proj_out"][1], res1=x, s1=1.0)

    @torch.no_grad()
    def decode(self, z: torch.Tensor, timesteps: Optional[int] = None) -> torch.Tensor:
        """z: [n, 4, h, w] (already divided by the scale factor, streaming_svd.py:125) -> [n, 3, 8h, 8w] fp32."""
        n, zc, h, w = z.shape
        T = timesteps or n
        assert n % T == 0
        dev = self.dev
        z32 = z.to(dev, torch.float32).contiguous()
        rows = torch.zeros((n * h * w, 8), dtype=torch.bfloat16, device=dev)  # z channels zero-padded to 8
        ops.nchw_to_nhwc(z32, rows, 0)
        x = None
        for kind, p, cin, cout in self.plan:
            if kind == "conv_in":
                x = ops.conv3x3(rows.view(n, h, w, 8), *self.w[p]["conv"])
            elif kind == "res":
                x = self._res(p, x, n, T, h, w, cin, cout)
            elif kind == "attn":
                x = self._attn(p, x, n, h, w, cin)
            elif kind == "up":
                xu = ops.upsample2x(x, n, h, w)
                h, w = 2 * h, 2 * w
                x = ops.conv3x3(xu.view(n, h, w, cin), *self.w[p]["conv"])
            elif kind == "out":
                e = self.w["out"]
                g = ops.group_norm(x, n, h * w, e["gn"][0], e["gn"][1], 1e-6, silu=True)
                y8 = torch.zeros((n * h * w, 8), dtype=torch.bfloat16, device=dev)   # 3 channels, padded row pitch
                ops.conv3x3(g.view(n, h, w, cin), e["conv"][0], e["conv"][1], out=y8[:, :cout])
                o8 = torch.empty((n * h * w, 8), dtype=torch.float32, device=dev)
                ops.tconv3(y8.view(n // T, T, h * w, 8), e["tmix"][0], e["tmix"][1], out=o8[:, :cout], out_fp32=True)
                out = torch.empty((n, cout, h, w), dtype=torch.float32, device=dev)
                ops.nhwc_to_nchw(o8, n, cout, h * w, out)
                return out
            if self.debug_taps is not None and kind != "out":
                self.debug_taps[p] = (x, n, h, w)
        raise AssertionError("plan has no output stage")


class B200VaeEncoder:
    """SD-VAE encoder of the conditioner on the project's kernels — drop-in for `AutoencoderKLModeOnly.encode(x)`
    (reference code/models/svd/sgm/models/autoencoder.py:468-473,602-615 -> Encoder, diffusionmodules/model.py:487-601;
    called once per chunk by VideoPredictionEmbedderWithEncoder, encoders/modules.py:697-729): returns the posterior
    MODE [n, 4, H/8, W/8] (the caller applies its scale factor, as the reference embedder does).  Same conventions as
    the decoder: channel-last bf16 rows, fp32 accumulation, every tensor op one of our kernels."""

    def __init__(self, cfg: VaeConfig, sd: SD, device):
        ops._lib.init(torch.device(device).index or 0)
        self.cfg, self.dev = cfg, torch.device(device)
        P, d = packing, self.dev
        self.plan = vae_encoder_plan(cfg)
        self.w: Dict[str, dict] = {}

        def gn(p):
            return (P.f32(sd[p + ".weight"], d), P.f32(sd[p + ".bias"], d))

        def conv(p):
            return (P.pack_conv3x3(sd[p + ".weight"], d), P.f32(sd[p + ".bias"], d))

        for kind, p, cin, cout in self.plan:
            if kind == "conv_in":
                self.w[p] = dict(conv=conv(p))
            elif kind == "res":
                e = dict(gn1=gn(p + ".norm1"), conv1=conv(p + ".conv1"), gn2=gn(p + ".norm2"), conv2=conv(p + ".conv2"),
                         skip=None)
                if (p + ".nin_shortcut.weight") in sd:
                    e["skip"] = (P.pack_conv1x1(sd[p + ".nin_shortcut.weight"], d), P.f32(sd[p + ".nin_shortcut.bias"], d))
                self.w[p] = e
            elif kind == "down":
                self.w[p] = dict(conv=conv(p + ".conv"))
            elif kind == "attn":
                self.w[p] = dict(norm=gn(p + ".norm"),
                                 **{n: (P.pack_conv1x1(sd[f"{p}.{n}.weight"], d), P.f32(sd[f"{p}.{n}.bias"], d))
                                    for n in ("q", "k", "v", "proj_out")})
            elif kind == "out":
                zc2 = 2 * cfg.z_channels
                # conv_out (C -> 2z) followed by the engine's 1x1 quant_conv (2z -> 2z): two back-to-back linear maps on
                # the channel axis, folded at pack time (W_q W_c, W_q b_c + b_q); only the z mean channels are kept
                wc = sd["conv_out.weight"].double()                                   # [2z, C, 3, 3]
                wq = sd["quant_conv.weight"].double().reshape(zc2, zc2)
                wf = torch.einsum("oz,zcij->ocij", wq, wc)[:cfg.z_channels]
                bf = (wq @ sd["conv_out.bias"].double() + sd["quant_conv.bias"].double())[:cfg.z_channels]
                wpad = torch.zeros((8,) + tuple(wf.shape[1:]), dtype=torch.float64)     # N padded to 8 output columns
                wpad[:cfg.z_channels] = wf
                bpad = torch.zeros(8, dtype=torch.float64)
                bpad[:cfg.z_channels] = bf
                self.w["out"] = dict(gn=gn("norm_out"), conv=(P.pack_conv3x3(wpad.float(), d), P.f32(bpad.float(), d)))
        self.debug_taps: Optional[dict] = None

    def _res(self, p, x, n, h, w, cin, cout):
        e = self.w[p]
        S = h * w
        g1 = ops.group_norm(x, n, S, e["gn1"][0], e["gn1"][1], 1e-6, silu=True)
        h1 = ops.conv3x3(g1.view(n, h, w, cin), e["conv1"][0], e["conv1"][1])
        g2 = ops.group_norm(h1, n, S, e["gn2"][0], e["gn2"][1], 1e-6, silu=True)
        xs = x if e["skip"] is None else ops.linear(x, e["skip"][0], e["skip"][1])
        return ops.conv3x3(g2.view(n, h, w, cout), e["conv2"][0], e["conv2"][1], res1=xs, s1=1.0)

    def _attn(self, p, x, n, h, w, c):
        e = self.w[p]
        S = h * w
        xn = ops.group_norm(x, n, S, e["norm"][0], e["norm"][1], 1e-6, silu=False)
        q = ops.linear(xn, e["q"][0], e["q"][1])
        k = ops.linear(xn, e["k"][0], e["k"][1])
        v = ops.linear(xn, e["v"][0], e["v"][1])
        o = ops.attention_single_head(q, k, v, n, S)
        return ops.linear(o, e["proj_out"][0], e["proj_out"][1], res1=x, s1=1.0)

    @torch.no_grad()
    def encode(self, x: torch.Tensor) -> torch.Tensor:
        """x: [n, 3, H, W] in [-1, 1], H and W multiples of 8 -> posterior mode [n, 4, H/8, W/8] fp32."""
        n, c_in, h, w = x.shape
        assert c_in == 3 and h % 8 == 0 and w % 8 == 0
        dev = self.dev
        x32 = x.to(dev, torch.float32).contiguous()
        rows = torch.zeros((n * h * w, 8), dtype=torch.bfloat16, device=dev)   # RGB zero-padded to 8 channels
        ops.nchw_to_nhwc(x32, rows, 0)
        cur = None
        for kind, p, cin, cout in self.plan:
            if kind == "conv_in":
                cur = ops.conv3x3(rows.view(n, h, w, 8), *self.w[p]["conv"])
            elif kind == "res":
                cur = self._res(p, cur, n, h, w, cin, cout)
            elif kind == "down":
                cur = ops.conv3x3_s2(cur.view(n, h, w, cin), *self.w[p]["conv"], pad_after_only=True)
                h, w = h // 2, w // 2
            elif kind == "attn":
                cur = self._attn(p, cur, n, h, w, cin)
            elif kind == "out":
                e = self.w["out"]
                g = ops.group_norm(cur, n, h * w, e["gn"][0], e["gn"][1], 1e-6, silu=True)
                o8 = torch.empty((n * h * w, 8), dtype=torch.float32, device=dev)
                ops.conv3x3(g.view(n, h, w, cin), e["conv"][0], e["conv"][1], out=o8, out_fp32=True)
                out = torch.empty((n, self.cfg.z_channels, h, w), dtype=torch.float32, device=dev)
                ops.nhwc_to_nchw(o8, n, self.cfg.z_channels, h * w, out)
                return out
            if self.debug_taps is not None:
                self.debug_taps[p] = (cur, n, h, w)
        raise AssertionError("plan has no output stage")
