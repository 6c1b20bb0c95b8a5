"""Host-side executor of the StreamingSVD denoiser on the project's sm_90a kernels.

Mirrors, op for op, the reference call tree under `StreamingWrapper.forward`
(code/models/diffusion/wrappers.py:23-78 -> controlnet.py:496-554 + video_model.py:540-618) but
  * keeps every activation channel-last bf16 as token rows [(b t) (h w), c] — no rearrange round trips; temporal
    ops address frames by stride,
  * folds the reference's elementwise neighbours into GEMM epilogues (bias, emb add, GEGLU, residuals,
    AlphaBlender), writes skip/concat operands in place (no torch.cat),
  * collapses the single-token cross-attentions (attn2 with context [N,1,1024], video_model.py:545-546) into
    per-frame vectors computed once per conditioning (softmax over one key == 1),
  * pre-multiplies back-to-back linear maps of the CAM merger (proj_in∘to_q, proj_out∘to_out) at pack time,
  * hoists step-invariant work (ControlNet conditioning embedding, label/time-position embeddings, cross-attention
    vectors) out of the sampler loop, keyed on the identity of the conditioning tensors.
Every tensor op below is a kernel launch through streamingt2v_b200.ops (C ABI); nothing is computed by PyTorch.
"""
from __future__ import annotations

import dataclasses
import os
from typing import Dict, List, Optional

import torch

from . import ops, packing
from .arch import Attn, Down, Plan, Res, Up, UNetConfig, build_plan
from .ops import ACT_GEGLU, ACT_SILU

SD = Dict[str, torch.Tensor]


def _sig(x: torch.Tensor) -> float:
    return float(torch.sigmoid(x.detach().float().reshape(-1)[0]))


def _same_structure(a, b) -> bool:
    """Same nesting, keys, tensor shapes/dtypes (values of non-tensor leaves must be equal)."""
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(_same_structure(a[k], b[k]) for k in a)
    if torch.is_tensor(a):
        return torch.is_tensor(b) and a.shape == b.shape and a.dtype == b.dtype and a.device == b.device
    return a == b


def _copy_structure(dst, src) -> None:
    for k, v in dst.items():
        if isinstance(v, dict):
            _copy_structure(v, src[k])
        elif torch.is_tensor(v):
            v.copy_(src[k], non_blocking=True)


class _NetWeights:
    """Packed weights of one network (VideoUNet or ControlNet encoder) in kernel layouts."""

    def __init__(self, sd: SD, cfg: UNetConfig, plan: Plan, device, root: str = ""):
        self.cfg, self.plan, self.dev = cfg, plan, device
        P = packing
        g = lambda k: sd[root + k] if root and not k.startswith(root) else sd[k]  # noqa: E731
        self.lin: Dict[str, tuple] = {}
        self.res: Dict[str, dict] = {}
        self.attn: Dict[str, dict] = {}
        self.conv: Dict[str, tuple] = {}

        def lin(p, bias=True):
            return (P.pack_linear(sd[p + ".weight"], device), P.f32(sd[p + ".bias"], device) if bias else None)

        for name in ("time_embed.0", "time_embed.2", "label_emb.0.0", "label_emb.0.2"):
            self.lin[name] = lin(root + name)

        # all ResBlock emb_layers as ONE GEMM: rows of the concatenated weight -> column slices of emb_all
        emb_w, emb_b = [], []
        self.emb_slices: Dict[str, tuple] = {}
        off = 0
        # all single-token cross-attention maps (to_out ∘ to_v) as ONE GEMM per kind
        xs_w, xs_b, xt_w, xt_b = [], [], [], []
        self.xs_slices: Dict[str, tuple] = {}
        self.xt_slices: Dict[str, tuple] = {}
        xoff = 0

        for blk in plan.input_blocks + [plan.middle] + plan.output_blocks:
            for layer in blk.layers:
                if isinstance(layer, tuple):
                    p = layer[1]
                    self.conv[p] = (P.pack_conv3x3(sd[p + ".weight"], device), P.f32(sd[p + ".bias"], device))
                elif isinstance(layer, (Down, Up)):
                    p = layer.prefix + (".op" if isinstance(layer, Down) else ".conv")
                    self.conv[p] = (P.pack_conv3x3(sd[p + ".weight"], device), P.f32(sd[p + ".bias"], device))
                elif isinstance(layer, Res):
                    p = layer.prefix
                    t = p + ".time_stack"
                    d = dict(
                        gn1=(P.f32(sd[p + ".in_layers.0.weight"], device), P.f32(sd[p + ".in_layers.0.bias"], device)),
                        conv1=(P.pack_conv3x3(sd[p + ".in_layers.2.weight"], device),
                               P.f32(sd[p + ".in_layers.2.bias"], device)),
                        gn2=(P.f32(sd[p + ".out_layers.0.weight"], device),
                             P.f32(sd[p + ".out_layers.0.bias"], device)),
                        conv2=(P.pack_conv3x3(sd[p + ".out_layers.3.weight"], device),
                               P.f32(sd[p + ".out_layers.3.bias"], device)),
                        gn3=(P.f32(sd[t + ".in_layers.0.weight"], device), P.f32(sd[t + ".in_layers.0.bias"], device)),
                        tconv1=(P.pack_tconv3(sd[t + ".in_layers.2.weight"], device),
                                P.f32(sd[t + ".in_layers.2.bias"], device)),
                        gn4=(P.f32(sd[t + ".out_layers.0.weight"], device),
                             P.f32(sd[t + ".out_layers.0.bias"], device)),
                        tconv2=(P.pack_tconv3(sd[t + ".out_layers.3.weight"], device),
                                P.f32(sd[t + ".out_layers.3.bias"], device)),
                        alpha=_sig(sd[p + ".time_mixer.mix_factor"]),
                        skip=None,
                    )
                    if (p + ".skip_connection.weight") in sd:
                        d["skip"] = (P.pack_conv1x1(sd[p + ".skip_connection.weight"], device),
                                     P.f32(sd[p + ".skip_connection.bias"], device))
                    self.res[p] = d
                    for key, pre in (("s", p), ("t", t)):
                        w, b = sd[pre + ".emb_layers.1.weight"], sd[pre + ".emb_layers.1.bias"]
                        emb_w.append(w.float())
                        emb_b.append(b.float())
                        self.emb_slices[p + "/" + key] = (off, off + w.shape[0])
                        off += w.shape[0]
                elif isinstance(layer, Attn):
                    p = layer.prefix
                    c = layer.ch
                    sb, tb = p + ".transformer_blocks.0", p + ".time_stack.0"

                    def ln(q):
                        return (P.f32(sd[q + ".weight"], device), P.f32(sd[q + ".bias"], device))

                    def qkv(q):
                        w = torch.cat([sd[q + ".to_q.weight"], sd[q + ".to_k.weight"], sd[q + ".to_v.weight"]], 0)
                        return P.pack_linear(w, device)

                    def geglu(q):
                        return P.pack_geglu(sd[q + ".weight"], sd[q + ".bias"], device)

                    d = dict(
                        ch=c, heads=layer.heads,
                        norm=ln(p + ".norm"), proj_in=lin(p + ".proj_in"), proj_out=lin(p + ".proj_out"),
                        s_norm1=ln(sb + ".norm1"), s_qkv=qkv(sb + ".attn1"), s_out=lin(sb + ".attn1.to_out.0"),
                        s_norm3=ln(sb + ".norm3"), s_ff1=geglu(sb + ".ff.net.0.proj"), s_ff2=lin(sb + ".ff.net.2"),
                        t_norm_in=ln(tb + ".norm_in"), t_ffin1=geglu(tb + ".ff_in.net.0.proj"),
                        t_ffin2=lin(tb + ".ff_in.net.2"),
                        t_norm1=ln(tb + ".norm1"), t_qkv=qkv(tb + ".attn1"), t_out=lin(tb + ".attn1.to_out.0"),
                        t_norm3=ln(tb + ".norm3"), t_ff1=geglu(tb + ".ff.net.0.proj"), t_ff2=lin(tb + ".ff.net.2"),
                        alpha=_sig(sd[p + ".time_mixer.mix_factor"]),
                        tpe0=lin(p + ".time_pos_embed.0"), tpe2=lin(p + ".time_pos_embed.2"),
                    )
                    # single-token cross attention == to_out(to_v(ctx)) + b   (softmax over one key is 1)
                    for kind, q, ws, bs, sl in (("s", sb + ".attn2", xs_w, xs_b, self.xs_slices),
                                                ("t", tb + ".attn2", xt_w, xt_b, self.xt_slices)):
                        wv = sd[q + ".to_v.weight"].double()
                        wo = sd[q + ".to_out.0.weight"].double()
                        ws.append((wo @ wv).float())
                        bs.append(sd[q + ".to_out.0.bias"].float())
                        sl[p] = (xoff, xoff + c)
                    xoff += c
                    if cfg.use_apm and root == "" and (sb + ".apm_conv.weight") in sd:
                        d["apm"] = dict(w=P.f32(sd[sb + ".apm_conv.weight"].reshape(-1, 3), device),
                                        wb=P.f32(sd[sb + ".apm_conv.bias"], device),
                                        ln=ln(sb + ".apm_ln"), alpha=P.f32(sd[sb + ".apm_alpha"].reshape(1), device))
                        # multi-token temporal cross attention (video_attention.py:150-154) needs the real maps
                        q = tb + ".attn2"
                        d["t_norm2"] = ln(tb + ".norm2")
                        d["t_x_q"] = P.pack_linear(sd[q + ".to_q.weight"], device)
                        d["t_x_kv"] = P.pack_linear(torch.cat([sd[q + ".to_k.weight"], sd[q + ".to_v.weight"]], 0),
                                                    device)
                        d["t_x_out"] = lin(q + ".to_out.0")
                    self.attn[p] = d
        self.emb_all = (P.pack_linear(torch.cat(emb_w, 0), device), P.f32(torch.cat(emb_b, 0), device))
        self.emb_total = off
        self.xs_all = (P.pack_linear(torch.cat(xs_w, 0), device), P.f32(torch.cat(xs_b, 0), device))
        self.xt_all = (P.pack_linear(torch.cat(xt_w, 0), device), P.f32(torch.cat(xt_b, 0), device))
        self.x_total = xoff


class B200Denoiser:
    """ControlNet + VideoUNet(+CAM) forward on the project's sm_90a kernels.  See module docstring."""

    def __init__(self, cfg: UNetConfig, sd_unet: SD, sd_ctrl: Optional[SD], device):
        ops._lib.init(torch.device(device).index or 0)
        self.cfg, self.dev = cfg, torch.device(device)
        if self.dev.type == "cuda" and self.dev.index is None:
            self.dev = torch.device("cuda", torch.cuda.current_device())
        self.plan_u = build_plan(cfg, "", decoder=True)
        self.wu = _NetWeights(sd_unet, cfg, self.plan_u, self.dev)
        P = packing
        d = self.dev
        self.out_gn = (P.f32(sd_unet["out.0.weight"], d), P.f32(sd_unet["out.0.bias"], d))
        self.out_conv = (P.pack_conv3x3(sd_unet["out.2.weight"], d), P.f32(sd_unet["out.2.bias"], d))
        self.cam: List[dict] = []
        self.has_ctrl = sd_ctrl is not None
        if self.has_ctrl:
            ccfg = dataclasses.replace(cfg, use_apm=False)
            self.plan_c = build_plan(ccfg, "", decoder=False)
            self.wc = _NetWeights(sd_ctrl, ccfg, self.plan_c, self.dev)
            names = [f"cross_attention_merger_input_blocks.{i}" for i in range(len(self.plan_u.skip_chans))]
            names.append("cross_attention_merger_mid_block")
            for nm in names:
                t = nm + ".temporal_transformer"
                a = t + ".attention"
                wq = sd_unet[a + ".to_q.weight"].double()
                wp, bp = sd_unet[t + ".proj_in.weight"].double(), sd_unet[t + ".proj_in.bias"].double()
                wo, bo = sd_unet[a + ".to_out.0.weight"].double(), sd_unet[a + ".to_out.0.bias"].double()
                wpo, bpo = sd_unet[t + ".proj_out.weight"].double(), sd_unet[t + ".proj_out.bias"].double()
                self.cam.append(dict(
                    norm=(P.f32(sd_unet[t + ".norm.weight"], d), P.f32(sd_unet[t + ".norm.bias"], d)),
                    q=(P.pack_linear((wq @ wp).float(), d), P.f32((wq @ bp).float(), d)),        # to_q ∘ proj_in
                    kv=P.pack_linear(torch.cat([sd_unet[a + ".to_k.weight"], sd_unet[a + ".to_v.weight"]], 0), d),
                    out=(P.pack_linear((wpo @ wo).float(), d), P.f32((wpo @ bo + bpo).float(), d)),  # proj_out ∘ to_out
                ))
            e = "controlnet_cond_embedding"
            boc = cfg.cond_embed_channels
            self.ce = dict(
                conv_in=(P.pack_conv3x3(sd_ctrl[e + ".conv_in.weight"], d), P.f32(sd_ctrl[e + ".conv_in.bias"], d)),
                blocks=[(P.pack_conv3x3(sd_ctrl[f"{e}.blocks.{i}.weight"], d), P.f32(sd_ctrl[f"{e}.blocks.{i}.bias"], d),
                         P.f32(sd_ctrl[f"{e}.norms.{i}.weight"], d), P.f32(sd_ctrl[f"{e}.norms.{i}.bias"], d))
                        for i in range(2 * (len(boc) - 1))],
                conv_out=(P.pack_conv3x3(sd_ctrl[e + ".conv_out.weight"], d), P.f32(sd_ctrl[e + ".conv_out.bias"], d)),
            )
        self._cond_key = None
        self._cond = None
        self._cond_refs = None
        self._cond_epoch = 0      # bumped whenever the conditioning is recomputed
        self._cond_struct_epoch = 0   # bumped when the conditioning BUFFERS are replaced (shape / structure change)
        self._tpe_cache: Dict[tuple, torch.Tensor] = {}
        self.debug_taps: Optional[dict] = None  # name -> bf16 rows tensor (tests only)
        # CUDA-graph replay of the forward (see _forward_graphed); B200SVD_NO_GRAPH=1 forces eager launches
        self.use_cuda_graph = self.dev.type == "cuda" and not os.environ.get("B200SVD_NO_GRAPH")
        self._graphs: Dict[tuple, dict] = {}
        self._capture_stream = torch.cuda.Stream(self.dev) if self.dev.type == "cuda" else None

    # ------------------------------------------------------------------------------------------------------------
    # building blocks
    # ------------------------------------------------------------------------------------------------------------
    def _tap(self, name, t, n, h, w):
        if self.debug_taps is not None:
            self.debug_taps[name] = (t, n, h, w)

    def _res_block(self, W: _NetWeights, layer: Res, x, n, T, h, w, emb_all, out=None):
        """VideoResBlock.forward (video_model.py:66-85 + openaimodel.py:328-354).  x: [(n h w), cin] rows."""
        d = W.res[layer.prefix]
        S = h * w
        B = n // T
        cin, cout = layer.cin, layer.cout
        a, b_ = W.emb_slices[layer.prefix + "/s"]
        e1 = emb_all[:, a:b_]
        a, b_ = W.emb_slices[layer.prefix + "/t"]
        e2 = emb_all[:, a:b_]
        g1 = ops.group_norm(x, n, S, d["gn1"][0], d["gn1"][1], 1e-5, silu=True)
        # gn_rows: the GEMM epilogue leaves the GroupNorm statistics of its output (per frame / per video) as
        # per-quadrant partial sums, so the following group_norm does not read the activation for its statistics
        h1 = ops.conv3x3(g1.view(n, h, w, cin), d["conv1"][0], d["conv1"][1], fvec=e1, rows_per_frame=S, gn_rows=S)
        g2 = ops.group_norm(h1, n, S, d["gn2"][0], d["gn2"][1], 1e-5, silu=True)
        xs = x if d["skip"] is None else ops.linear(x, d["skip"][0], d["skip"][1])
        x_s = ops.conv3x3(g2.view(n, h, w, cout), d["conv2"][0], d["conv2"][1], res1=xs, s1=1.0, gn_rows=T * S)
        # time_stack: ResBlock(dims=3) on [b, c, t, h, w]; its GroupNorm reduces over (c/32, t, h, w) per batch
        g3 = ops.group_norm(x_s, B, T * S, d["gn3"][0], d["gn3"][1], 1e-5, silu=True)
        h3 = ops.tconv3(g3.view(B, T, S, cout), d["tconv1"][0], d["tconv1"][1], fvec=e2, rows_per_frame=S,
                        gn_rows=T * S)
        g4 = ops.group_norm(h3, B, T * S, d["gn4"][0], d["gn4"][1], 1e-5, silu=True)
        # x_t = x_s + conv(..) ; blend = a*x_s + (1-a)*x_t = x_s + (1-a)*conv(..)
        return ops.tconv3(g4.view(B, T, S, cout), d["tconv2"][0], d["tconv2"][1], s_acc=1.0 - d["alpha"], res1=x_s,
                          s1=1.0, out=out)

    def _time_pos_emb(self, W: _NetWeights, layer: Attn, n, T):
        """time_pos_embed(timestep_embedding(arange(T), C)) expanded to frames (video_attention.py:298-308)."""
        key = (id(W), layer.prefix, n, T)
        if key not in self._tpe_cache:
            d = W.attn[layer.prefix]
            fr = torch.arange(T, device=self.dev, dtype=torch.float32).repeat(n // T).contiguous()
            te = ops.timestep_embed(fr, layer.ch)
            hmid = ops.linear(te, d["tpe0"][0], d["tpe0"][1], act=ACT_SILU)
            self._tpe_cache[key] = ops.linear(hmid, d["tpe2"][0], d["tpe2"][1], out_fp32=True)
        return self._tpe_cache[key]

    def _attn_block(self, W: _NetWeights, layer: Attn, x, n, T, h, w, cond, out=None):
        """SpatialVideoTransformer.forward (video_attention.py:260-333).  x: [(n h w), c] rows (may be strided)."""
        d = W.attn[layer.prefix]
        c, heads, S, B = layer.ch, layer.heads, h * w, n // T
        a, b_ = W.xs_slices[layer.prefix]
        if "xs_blocks" in cond and layer.prefix in cond["xs_blocks"]:
            xs_vec = cond["xs_blocks"][layer.prefix]
        else:
            xs_vec = cond["xs"][:, a:b_]
        xn = ops.group_norm(x, n, S, d["norm"][0], d["norm"][1], 1e-6, silu=False)
        hh = ops.linear(xn, d["proj_in"][0], d["proj_in"][1])
        # --- spatial BasicTransformerBlock (attention.py:567-593) ---
        n1 = ops.layer_norm(hh, *d["s_norm1"])
        qkv = ops.linear(n1, d["s_qkv"])
        at = ops.flash_attn(qkv, n, S, heads)
        h1 = ops.linear(at, d["s_out"][0], d["s_out"][1], res1=hh, s1=1.0, fvec=xs_vec, rows_per_frame=S)
        n3 = ops.layer_norm(h1, *d["s_norm3"])
        f1 = ops.linear(n3, d["s_ff1"][0], d["s_ff1"][1], act=ACT_GEGLU, bn=d["s_ff1"][2])
        h2 = ops.linear(f1, d["s_ff2"][0], d["s_ff2"][1], res1=h1, s1=1.0)
        # --- temporal VideoTransformerBlock (video_attention.py:125-168) on x_mix = h2 + emb_t ---
        tpe = self._time_pos_emb(W, layer, n, T)
        xmix = torch.empty_like(h2)
        nin = ops.layer_norm(h2, *d["t_norm_in"], fvec=tpe, rows_per_frame=S, xsum=xmix)
        f0 = ops.linear(nin, d["t_ffin1"][0], d["t_ffin1"][1], act=ACT_GEGLU, bn=d["t_ffin1"][2])
        xa = ops.linear(f0, d["t_ffin2"][0], d["t_ffin2"][1], res1=xmix, s1=1.0)
        n1t = ops.layer_norm(xa, *d["t_norm1"])
        qkv_t = ops.linear(n1t, d["t_qkv"])
        at_t = ops.small_attn(qkv_t[:, :c], qkv_t[:, c:2 * c], qkv_t[:, 2 * c:], b=B, s=S, heads=heads, lq=T, lk=T)
        if "t_ctx" in cond and "t_x_q" in d:
            # multi-token temporal cross attention (APM tokens): real attention, K/V shared by all pixels
            xb0 = ops.linear(at_t, d["t_out"][0], d["t_out"][1], res1=xa, s1=1.0)
            n2t = ops.layer_norm(xb0, *d["t_norm2"])
            q2 = ops.linear(n2t, d["t_x_q"])
            kv2 = ops.linear(cond["t_ctx"], d["t_x_kv"])             # [(B L), 2c]
            L = cond["t_ctx_tokens"]
            a2 = ops.small_attn(q2, kv2[:, :c], kv2[:, c:], b=B, s=S, heads=heads, lq=T, lk=L, kv_per_pixel=False)
            xb = ops.linear(a2, d["t_x_out"][0], d["t_x_out"][1], res1=xb0, s1=1.0)
        else:
            xt_vec = cond["xt"][:, a:b_]
            xb = ops.linear(at_t, d["t_out"][0], d["t_out"][1], res1=xa, s1=1.0, fvec=xt_vec, rows_per_frame=T * S)
        n3t = ops.layer_norm(xb, *d["t_norm3"])
        f2 = ops.linear(n3t, d["t_ff1"][0], d["t_ff1"][1], act=ACT_GEGLU, bn=d["t_ff1"][2])
        al = d["alpha"]
        # x_t = ff(..) + xb ; x = al*h2 + (1-al)*x_t   (AlphaBlender, util.py:358-370)
        xbl = ops.linear(f2, d["t_ff2"][0], d["t_ff2"][1], s_acc=1.0 - al, res1=xb, s1=1.0 - al, res2=h2, s2=al)
        return ops.linear(xbl, d["proj_out"][0], d["proj_out"][1], res1=x, s1=1.0, out=out)

    def _run_block(self, W, blk, x, n, T, h, w, emb_all, cond, out=None):
        """One TimestepEmbedSequential entry; returns (rows, h, w).  `out`: where the block's last op writes."""
        nl = len(blk.layers)
        for li, layer in enumerate(blk.layers):
            o = out if li == nl - 1 else None
            if isinstance(layer, tuple):
                raise AssertionError("conv_in handled by caller")
            if isinstance(layer, Res):
                x = self._res_block(W, layer, x, n, T, h, w, emb_all, out=o)
            elif isinstance(layer, Attn):
                x = self._attn_block(W, layer, x, n, T, h, w, cond, out=o)
            elif isinstance(layer, Down):
                wgt, b = W.conv[layer.prefix + ".op"]
                x = ops.conv3x3_s2(x.view(n, h, w, layer.ch), wgt, b, out=o)
                h, w = h // 2, w // 2
            elif isinstance(layer, Up):
                wgt, b = W.conv[layer.prefix + ".conv"]
                xu = ops.upsample2x(x, n, h, w)
                h, w = 2 * h, 2 * w
                x = ops.conv3x3(xu.view(n, h, w, layer.ch), wgt, b, out=o)
        return x, h, w

    def _embed(self, W: _NetWeights, t, y_bf16):
        """silu(time_embed(timestep_embedding(t)) + label_emb(y)) -> all ResBlock emb_layers in one GEMM
        (video_model.py:561-567, openaimodel.py:339-352)."""
        te = ops.timestep_embed(t, self.cfg.model_channels)
        h0 = ops.linear(te, *W.lin["time_embed.0"], act=ACT_SILU)
        e_t = ops.linear(h0, *W.lin["time_embed.2"], out_fp32=True)
        l0 = ops.linear(y_bf16, *W.lin["label_emb.0.0"], act=ACT_SILU)
        e_y = ops.linear(l0, *W.lin["label_emb.0.2"], out_fp32=True)
        emb_silu = ops.add_silu(e_t, e_y, silu=True)
        return ops.linear(emb_silu, W.emb_all[0], W.emb_all[1], out_fp32=True)

    def _cam_merge(self, i, sample, cond_feat, B, T, Fc, S, out):
        """ConditionalModel / CAM CrossAttention (cam/conditioning.py:39-81, :117-146), eval mode."""
        d = self.cam[i]
        c = sample.shape[1]
        xn = ops.group_norm(sample, B, T * S, d["norm"][0], d["norm"][1], 1e-6, silu=False)
        q = ops.linear(xn, d["q"][0], d["q"][1])
        kv = ops.linear(cond_feat, d["kv"])
        o = ops.small_attn(q, kv[:, :c], kv[:, c:], b=B, s=S, heads=c // 64, lq=T, lk=Fc)
        return ops.linear(o, d["out"][0], d["out"][1], res1=sample, s1=1.0, out=out)

    # ------------------------------------------------------------------------------------------------------------
    # step-invariant conditioning
    # ------------------------------------------------------------------------------------------------------------
    def _cond_embedding(self, ctrl_frames, h, w):
        """ControlNetConditioningEmbedding.forward (controlnet.py:104-121) on the Fc control frames."""
        Fc = ctrl_frames.shape[1]
        H, Wd = 8 * h, 8 * w
        src = ctrl_frames.reshape(Fc, ctrl_frames.shape[2], H, Wd).to(self.dev, torch.float32).contiguous()
        x = torch.zeros((Fc * H * Wd, 8), dtype=torch.bfloat16, device=self.dev)  # 3 channels zero-padded to 8
        ops.nchw_to_nhwc(src, x, 0)
        ce = self.ce
        boc = self.cfg.cond_embed_channels
        e = ops.conv3x3(x.view(Fc, H, Wd, 8), ce["conv_in"][0], ce["conv_in"][1], act=ACT_SILU)
        ch = boc[0]
        for i, (wgt, b, lg, lb) in enumerate(ce["blocks"]):
            if i % 2 == 0:
                e = ops.conv3x3(e.view(Fc, H, Wd, ch), wgt, b)
            else:
                e = ops.conv3x3_s2(e.view(Fc, H, Wd, ch), wgt, b)
                H, Wd = H // 2, Wd // 2
                ch = boc[i // 2 + 1]
            e = ops.layer_norm(e, lg, lb, 1e-5, silu=True)
        return ops.conv3x3(e.view(Fc, H, Wd, ch), ce["conv_out"][0], ce["conv_out"][1])   # [(Fc h w), 320]

    def _prepare(self, c, ctrl_frames, B, T, h, w):
        ctx, vec, concat = c["crossattn"], c["vector"], c["concat"]
        # Cache key = IDENTITY of the conditioning tensors (+ their in-place version counters).  The cache entry
        # holds strong references to the keyed tensors (self._cond_refs), so their storage cannot be freed and handed
        # to a new tensor of equal shape while the entry is alive: `is` on a live object is unambiguous, a recycled
        # data_ptr() is not.
        keyed = (ctx, vec, concat, ctrl_frames)
        key = tuple((t._version, tuple(t.shape)) if t is not None else None for t in keyed) + (B, T, h, w)
        if (self._cond_key == key and self._cond_refs is not None
                and all(a is b for a, b in zip(self._cond_refs, keyed))):
            return self._cond
        N = B * T
        Fc = self.cfg.num_frame_conditioning
        dev = self.dev
        cond = {}
        L = ctx.shape[1]
        ctx32 = ctx.to(dev, torch.float32).contiguous()
        ctx0 = ops.add_silu(ctx32[:, 0].contiguous(), None, silu=False)          # bf16 [N, 1024]
        cond["y"] = ops.add_silu(vec.to(dev, torch.float32).contiguous(), None, silu=False)
        cond["concat"] = concat.to(dev, torch.float32).contiguous().clone()   # owned: later chunks are copied into it
        W = self.wu
        if L > 1 and self.cfg.use_apm:
            # APM: the spatial context is mixed per block (attention.py:612-620); temporal blocks see all tokens
            cond["xs_blocks"] = {}
            for p, d in W.attn.items():
                a, b_ = W.xs_slices[p]
                mixed = ops.apm_mix(ctx32, d["apm"]["w"], d["apm"]["wb"], d["apm"]["ln"][0], d["apm"]["ln"][1],
                                    d["apm"]["alpha"])
                cond["xs_blocks"][p] = ops.linear(mixed, W.xs_all[0][:, a:b_].contiguous(),
                                                  W.xs_all[1][a:b_].contiguous(), out_fp32=True)
            tctx = ctx32[::T].contiguous().reshape(B * L, -1)
            cond["t_ctx"] = ops.add_silu(tctx, None, silu=False)
            cond["t_ctx_tokens"] = L
            cond["xs"] = None
        else:
            cond["xs"] = ops.linear(ctx0, W.xs_all[0], W.xs_all[1], out_fp32=True)          # [N, sumC]
            cond["xt"] = ops.linear(ctx0[::T], W.xt_all[0], W.xt_all[1], out_fp32=True)      # [B, sumC]
        if self.has_ctrl and ctrl_frames is not None:
            # ControlNet sees the first Fc frames of each batch element and only the first context token
            Wc = self.wc
            idx = (torch.arange(B, device=dev)[:, None] * T + torch.arange(Fc, device=dev)[None]).reshape(-1)
            ctx0c = ctx0[idx].contiguous()
            cc = {"y": cond["y"][idx].contiguous()}
            cc["xs"] = ops.linear(ctx0c, Wc.xs_all[0], Wc.xs_all[1], out_fp32=True)
            cc["xt"] = ops.linear(ctx0c[::Fc], Wc.xt_all[0], Wc.xt_all[1], out_fp32=True)
            ce = self._cond_embedding(ctrl_frames, h, w)                     # [(Fc S), 320]
            cc["ce"] = ce
            cond["ctrl"] = cc
        # Keep the conditioning in PERSISTENT buffers: a recorded CUDA graph points at them, so a new chunk's
        # conditioning (same shapes) is copied in place and the recording stays valid; only a structural change
        # (other shapes / APM tokens / ControlNet on-off) replaces the buffers and forces a new recording.
        if self._cond is not None and _same_structure(self._cond, cond):
            _copy_structure(self._cond, cond)
            cond = self._cond
        else:
            self._cond_struct_epoch += 1
        self._cond_key, self._cond, self._cond_refs = key, cond, keyed
        self._cond_epoch += 1
        return cond

    def reset_conditioning(self):
        """Drop the step-invariant conditioning cache (and the references it holds); the next forward recomputes it."""
        self._cond_key = self._cond_refs = None       # the buffers in self._cond stay: recorded graphs point at them

    # ------------------------------------------------------------------------------------------------------------
    # forward
    # ------------------------------------------------------------------------------------------------------------
    def _to_rows(self, x, concat, n, h, w, frames=None):
        """cat([x, concat], dim=1) (wrappers.py:33) -> channel-last bf16 rows [(n h w), 8]."""
        rows = torch.empty((n * h * w, 8), dtype=torch.bfloat16, device=self.dev)
        if frames is None:
            ops.nchw_to_nhwc(x, rows, 0)
            ops.nchw_to_nhwc(concat, rows, 4)
        else:  # (start, count) frame groups
            r = 0
            S = h * w
            for s0, cnt in frames:
                ops.nchw_to_nhwc(x[s0:s0 + cnt], rows[r * S:(r + cnt) * S], 0)
                ops.nchw_to_nhwc(concat[s0:s0 + cnt], rows[r * S:(r + cnt) * S], 4)
                r += cnt
        return rows

    def _controlnet(self, x32, t32, cond, B, T, h, w):
        """ControlNet.forward (controlnet.py:496-554) on the first Fc frames of each batch element."""
        Fc = self.cfg.num_frame_conditioning
        W = self.wc
        cc = cond["ctrl"]
        n = B * Fc
        groups = [(b * T, Fc) for b in range(B)]
        rows = self._to_rows(x32, cond["concat"], n, h, w, frames=groups)
        t_c = torch.cat([t32[b * T:b * T + Fc] for b in range(B)]).contiguous()
        emb_all = self._embed(W, t_c, cc["y"])
        S = h * w
        # conv_in, then Merger "addition" of the conditioning embedding (same Fc frames for every batch element)
        wgt, bias = W.conv[self.plan_c.input_blocks[0].layers[0][1]]
        hcur = ops.conv3x3(rows.view(n, h, w, 8), wgt, bias)
        ops.add_rows(hcur, cc["ce"])
        hs = [(hcur, h, w)]
        hh, ww = h, w
        for blk in self.plan_c.input_blocks[1:]:
            hcur, hh, ww = self._run_block(W, blk, hcur, n, Fc, hh, ww, emb_all, cc)
            hs.append((hcur, hh, ww))
        mid, hh, ww = self._run_block(W, self.plan_c.middle, hcur, n, Fc, hh, ww, emb_all, cc)
        if self.debug_taps is not None:
            for i, (t_, a, b_) in enumerate(hs):
                self._tap(f"ctrl.input_blocks.{i}", t_, n, a, b_)
            self._tap("ctrl.middle", mid, n, hh, ww)
        return hs, (mid, hh, ww)

    @torch.no_grad()
    def forward(self, x, t, c, *, batch_size, num_video_frames, ctrl_frames=None, image_only_indicator=None,
                num_conditional_frames=None, use_controlnet=True):
        """Same contract as StreamingWrapper.forward (wrappers.py:23-78): x [(B T),4,h,w], t [(B T)] (c_noise),
        c = {concat, crossattn, vector}; returns [(B T),4,h,w] fp32.  `image_only_indicator` must be all zeros
        (streaming_svd.py:208); `num_conditional_frames` is accepted and ignored, as in the reference."""
        B, T = batch_size, num_video_frames
        N, _, h, w = x.shape
        assert N == B * T
        if h % 8 or w % 8:
            raise ValueError("latent height/width must be multiples of 8 (three stride-2 levels)")
        if self.dev.type == "cuda" and torch.cuda.current_device() != self.dev.index:
            # launches go to torch's current stream OF THE CURRENT DEVICE: make that this engine's device
            with torch.cuda.device(self.dev):
                return self.forward(x, t, c, batch_size=batch_size, num_video_frames=num_video_frames,
                                    ctrl_frames=ctrl_frames, use_controlnet=use_controlnet)
        dev = self.dev
        use_ctrl = self.has_ctrl and use_controlnet and ctrl_frames is not None
        cond = self._prepare(c, ctrl_frames if use_ctrl else None, B, T, h, w)
        if self._graph_ok():
            return self._forward_graphed(x, t, cond, B, T, h, w, use_ctrl)
        x32 = x.to(dev, torch.float32).contiguous()
        t32 = t.to(dev, torch.float32).contiguous()
        return self._forward_body(x32, t32, cond, B, T, h, w, use_ctrl)

    # ------------------------------------------------------------------------------------------------------------
    # CUDA-graph replay of the step (all shapes are static over the 30 sampler steps of a chunk)
    # ------------------------------------------------------------------------------------------------------------
    def _graph_ok(self) -> bool:
        return (self.use_cuda_graph and self.debug_taps is None and ops._PROFILE is None
                and self.dev.type == "cuda")

    def _forward_graphed(self, x, t, cond, B, T, h, w, use_ctrl):
        """The ~1000 launches of one forward are recorded once per (shape, conditioning) into a CUDA graph on the
        caller's stream and replayed: one cudaGraphLaunch per sampler step instead of ~1000 ctypes calls and 7
        host-side tensor-map encodes per GEMM.  The first forward of a new shape runs eagerly (it fills the lazily
        built caches: time-position embeddings, GroupNorm scratch, kernel attributes); the conditioning tensors
        the graph points at live in persistent buffers (`_prepare` copies a new chunk's conditioning into them), so
        the recording survives across chunks; only a structural change of the conditioning records again."""
        key = (B, T, h, w, use_ctrl)
        g = self._graphs.get(key)
        N = B * T
        if g is None:
            # first visit of this shape: eager run (warms caches), static I/O buffers
            g = dict(x=torch.empty((N, 4, h, w), dtype=torch.float32, device=self.dev),
                     t=torch.empty((N,), dtype=torch.float32, device=self.dev), graph=None, epoch=-1, out=None,
                     launches=0)
            self._graphs[key] = g
            g["x"].copy_(x, non_blocking=True)
            g["t"].copy_(t, non_blocking=True)
            return self._forward_body(g["x"], g["t"], cond, B, T, h, w, use_ctrl)
        g["x"].copy_(x, non_blocking=True)
        g["t"].copy_(t, non_blocking=True)
        if g["graph"] is None or g["epoch"] != self._cond_struct_epoch:
            g["graph"] = None                      # release the previous recording (and its private memory pool)
            g["out"] = None
            graph = torch.cuda.CUDAGraph()
            l0 = ops.launches()
            torch.cuda.current_stream().synchronize()
            with torch.cuda.graph(graph, stream=self._capture_stream):
                out = self._forward_body(g["x"], g["t"], cond, B, T, h, w, use_ctrl)
            g.update(graph=graph, out=out, epoch=self._cond_struct_epoch, launches=ops.launches() - l0)
            ops._launch_count -= g["launches"]     # recording is not launching
        g["graph"].replay()
        ops._launch_count += g["launches"]
        res = torch.empty_like(g["out"])
        res.copy_(g["out"], non_blocking=True)     # D2D memcpy: the caller gets its own tensor, like the reference
        return res

    def _forward_body(self, x32, t32, cond, B, T, h, w, use_ctrl):
        N = B * T
        dev = self.dev
        Fc = self.cfg.num_frame_conditioning
        W = self.wu
        plan = self.plan_u
        hs_c = mid_c = None
        if use_ctrl:
            hs_c, mid_c = self._controlnet(x32, t32, cond, B, T, h, w)

        rows = self._to_rows(x32, cond["concat"], N, h, w)
        emb_all = self._embed(W, t32, cond["y"])
        wgt, bias = W.conv[plan.input_blocks[0].layers[0][1]]
        hcur = ops.conv3x3(rows.view(N, h, w, 8), wgt, bias)
        hs = [(hcur, h, w)]
        hh, ww = h, w
        for i, blk in enumerate(plan.input_blocks[1:], start=1):
            hcur, hh, ww = self._run_block(W, blk, hcur, N, T, hh, ww, emb_all, cond)
            hs.append((hcur, hh, ww))
            self._tap(f"unet.input_blocks.{i}", hcur, N, hh, ww)

        # concat buffers of the decoder: [h | skip] written in place (video_model.py:608 torch.cat)
        nout = len(plan.output_blocks)
        cat_bufs = []
        ch_h = plan.middle.out_ch
        for j, blk in enumerate(plan.output_blocks):
            skip_t, sh, sw = hs[nout - 1 - j]
            c_skip = skip_t.shape[1]
            buf = torch.empty((N * sh * sw, ch_h + c_skip), dtype=torch.bfloat16, device=dev)
            cat_bufs.append((buf, ch_h, c_skip, sh, sw))
            ch_h = blk.out_ch
        # CAM: fuse ControlNet features into the skips (video_model.py:582-591), straight into the concat buffers
        for i, (skip_t, sh, sw) in enumerate(hs):
            buf, chh, c_skip, _, _ = cat_bufs[nout - 1 - i]
            dst = buf[:, chh:]
            if use_ctrl:
                self._cam_merge(i, skip_t, hs_c[i][0], B, T, Fc, sh * sw, out=dst)
            else:
                ops.copy2d(skip_t, dst)
            self._tap(f"unet.merged.{i}", dst, N, sh, sw)

        # middle block (+ CAM on the mid features), written into the first concat buffer's h slot
        first = cat_bufs[0][0][:, :cat_bufs[0][1]]
        if use_ctrl:
            hmid, hh, ww = self._run_block(W, plan.middle, hcur, N, T, hh, ww, emb_all, cond)
            self._cam_merge(len(hs), hmid, mid_c[0], B, T, Fc, hh * ww, out=first)
        else:
            hmid, hh, ww = self._run_block(W, plan.middle, hcur, N, T, hh, ww, emb_all, cond, out=first)
        self._tap("unet.middle", first, N, hh, ww)

        hcur = None
        for j, blk in enumerate(plan.output_blocks):
            buf, chh, c_skip, sh, sw = cat_bufs[j]
            assert (sh, sw) == (hh, ww)
            dst = cat_bufs[j + 1][0][:, :cat_bufs[j + 1][1]] if j + 1 < nout else None
            hcur, hh, ww = self._run_block(W, blk, buf, N, T, hh, ww, emb_all, cond, out=dst)
            self._tap(f"unet.output_blocks.{j}", hcur, N, hh, ww)

        g = ops.group_norm(hcur, N, hh * ww, self.out_gn[0], self.out_gn[1], 1e-5, silu=True)
        o8 = torch.empty((N * hh * ww, 8), dtype=torch.float32, device=dev)
        ops.conv3x3(g.view(N, hh, ww, self.cfg.model_channels), self.out_conv[0], self.out_conv[1], out=o8[:, :4],
                    out_fp32=True)
        out = torch.empty((N, 4, hh, ww), dtype=torch.float32, device=dev)
        ops.nhwc_to_nchw(o8, N, 4, hh * ww, out)
        return out
