"""EMA-VFI frame interpolation on the GPU: the reference's `interpolate_video` stage.

The reference (code/i2v_enhance/i2v_enhance_interface.py:15-62, thirdparty/VFI) runs EMA-VFI in fp32 eager PyTorch,
one frame pair at a time, each with fast test-time augmentation (the pair and its H+W-flipped copy in one batch).
`B200VFI` runs the same network from the same weights on the project's kernels: the multi-tap GEMM for every conv and
linear (PReLU in its epilogue), `layer_norm`, and the kernels of csrc/vfi.cu (window attention, backward warp,
bilinear resize, depthwise conv + GELU, head input gather, merge).  GEMM operands are bf16 with fp32 accumulation;
flows, masks, warp coordinates, the flow / mask accumulation and the final merge stay fp32.

Only the configuration the reference ships is accepted (`VFI/config.py:init_model_config(F=32, W=7,
depth=[2, 2, 2, 4, 4])`, as `vfi_init` builds it); any other state dict is rejected.

Activations are channel-last bf16 rows.  The four images of a pair's batch are [img0, flip(img0), img1, flip(img1)]
(MotionFormer.forward concatenates x1 and x2 along the batch, :468-470).
"""
from __future__ import annotations

import torch

from . import ops
from ._lib import ACT_PRELU
from .packing import pack_conv3x3, pack_conv1x1, pack_linear

F_ = 32                      # base width
EMBED = [F_, 2 * F_, 4 * F_, 8 * F_, 16 * F_]
DEPTHS = [2, 2, 2, 4, 4]
MOTION = [8 * F_ // DEPTHS[3], 16 * F_ // DEPTHS[4]]   # 64, 128: 8 per head
HEADS = [8 * F_ // 32, 16 * F_ // 32]                 # 8, 16 heads of 32
HIDDEN = 4 * F_                                       # flow head width
UNET_C = 2 * F_                                       # Unet(c * 2)


def expected_shapes() -> dict:
    """Every key of MultiScaleFlow(feature_extractor(**cfg0), **cfg1).state_dict() for the shipped configuration, with
    its shape (the reference's `attn_mask` / `HW` buffers, which Model.load_model drops, excluded)."""
    s = {}

    def conv(k, cout, cin, kh=3):
        s[k + ".weight"] = (cout, cin, kh, kh)
        s[k + ".bias"] = (cout,)

    def prelu(k, c):
        s[k + ".weight"] = (c,)

    def lin(k, n, kk):
        s[k + ".weight"] = (n, kk)
        s[k + ".bias"] = (n,)

    def ln(k, c):
        s[k + ".weight"] = (c,)
        s[k + ".bias"] = (c,)

    fb = "feature_bone."
    for i in range(3):
        cin = 3 if i == 0 else EMBED[i]
        if i > 0:
            conv(fb + f"patch_embed{i + 1}.0", EMBED[i], EMBED[i - 1])
            prelu(fb + f"patch_embed{i + 1}.1", EMBED[i])
        conv(fb + f"block{i + 1}.conv.0", EMBED[i], cin)
        prelu(fb + f"block{i + 1}.conv.1", EMBED[i])
        conv(fb + f"block{i + 1}.conv.2", EMBED[i], EMBED[i])
        prelu(fb + f"block{i + 1}.conv.3", EMBED[i])
    for k in range(7):
        conv(fb + f"patch_embed4.layers.{k}", F_, EMBED[2 - (0 if k == 0 else (1 if k < 3 else 2))])
    conv(fb + "patch_embed4.proj", EMBED[3], 7 * F_, kh=1)
    ln(fb + "patch_embed4.norm", EMBED[3])
    conv(fb + "patch_embed5.proj", EMBED[4], EMBED[3])
    ln(fb + "patch_embed5.norm", EMBED[4])
    for st in (3, 4):
        C, Cm = EMBED[st], MOTION[st - 3]
        for j in range(DEPTHS[st]):
            p = fb + f"block{st + 1}.{j}."
            ln(p + "norm1", C)
            lin(p + "attn.q", C, C)
            lin(p + "attn.kv", 2 * C, C)
            lin(p + "attn.cor_embed", Cm, 2)
            lin(p + "attn.proj", C, C)
            lin(p + "attn.motion_proj", Cm, Cm)
            ln(p + "norm2", C)
            lin(p + "mlp.fc1", 4 * C, C)
            s[p + "mlp.dwconv.dwconv.weight"] = (4 * C, 1, 3, 3)
            s[p + "mlp.dwconv.dwconv.bias"] = (4 * C,)
            lin(p + "mlp.fc2", C, 4 * C)
        ln(fb + f"norm{st + 1}", C)
    for i, (st, extra) in enumerate(((4, 6), (3, 17))):
        cin = (MOTION[st - 3] * DEPTHS[st] + EMBED[st]) * 2 // 16 + extra
        for j, (ci, co) in enumerate(((cin, HIDDEN), (HIDDEN, HIDDEN), (HIDDEN, 5))):
            conv(f"block.{i}.conv.{j}.0", co, ci)
            prelu(f"block.{i}.conv.{j}.1", co)
    c = UNET_C
    for d, (ci, co) in enumerate(((17 + c, 2 * c), (4 * c, 4 * c), (8 * c, 8 * c), (16 * c, 16 * c))):
        conv(f"unet.down{d}.conv1.0", co, ci)
        prelu(f"unet.down{d}.conv1.1", co)
        conv(f"unet.down{d}.conv2.0", co, co)
        prelu(f"unet.down{d}.conv2.1", co)
    for u, (ci, co) in enumerate(((32 * c, 8 * c), (16 * c, 4 * c), (8 * c, 2 * c), (4 * c, c))):
        s[f"unet.up{u}.0.weight"] = (ci, co, 4, 4)      # ConvTranspose2d: [Cin, Cout, kh, kw]
        s[f"unet.up{u}.0.bias"] = (co,)
        prelu(f"unet.up{u}.1", co)
    conv("unet.conv", 3, c)
    return s


def check_config(state_dict) -> dict:
    """The state dict without the reference's cached mask buffers, if it is the shipped configuration; else ValueError
    naming the first difference."""
    sd = {k: v for k, v in state_dict.items() if not (k.endswith(".attn_mask") or k.endswith(".HW"))}
    want = expected_shapes()
    missing = sorted(set(want) - set(sd))
    extra = sorted(set(sd) - set(want))
    if missing or extra:
        raise ValueError("B200VFI supports only the EMA-VFI configuration of the reference (F=32, W=7, depths "
                         f"[2, 2, 2, 4, 4]); missing keys {missing[:4]}, unexpected keys {extra[:4]}")
    for k, shp in want.items():
        if tuple(sd[k].shape) != shp:
            raise ValueError(f"B200VFI supports only the reference's EMA-VFI configuration (F=32, W=7, depths "
                             f"[2, 2, 2, 4, 4]): {k} has shape {tuple(sd[k].shape)}, expected {shp}")
    return sd


def seeded_state_dict(seed: int = 0) -> dict:
    """Deterministic random weights of the shipped configuration (torch CPU generator, keys in sorted order): convs and
    linears at unit-variance fan-in scale, biases N(0, 0.05), LayerNorm gamma 1 + N(0, 0.1) and beta N(0, 0.1), PReLU
    slopes 0.25 + N(0, 0.05).  The goldens and their GPU tests build the same weights from the seed."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shp in sorted(expected_shapes().items()):
        r = torch.randn(shp, generator=g, dtype=torch.float32)
        if len(shp) > 1:
            fan_in = shp[0] * 4 if k.startswith("unet.up") else (shp[1] * shp[2] * shp[3] if len(shp) == 4 else shp[1])
            if k.endswith("dwconv.dwconv.weight"):
                fan_in = 9
            sd[k] = r / fan_in ** 0.5
        elif k.endswith(".bias"):
            sd[k] = 0.05 * r
        elif "norm" in k:
            sd[k] = 1.0 + 0.1 * r
        else:
            sd[k] = 0.25 + 0.05 * r
    return sd


def deconv_phase_weights(w: torch.Tensor) -> torch.Tensor:
    """ConvTranspose2d(4, 2, 1) weight [Cin, Cout, 4, 4] -> [4 phases (a*2+b), 4 taps, Cout, Cin] (same dtype) for
    ops.conv_transpose4x4_s2, taps in DECONV_PHASE_TAPS order, row offset major."""
    cin, cout = w.shape[:2]
    out = torch.empty((4, 4, cout, cin), dtype=w.dtype)
    for a in range(2):
        for b in range(2):
            t = 0
            for _, kh in ops.DECONV_PHASE_TAPS[a]:
                for _, kw in ops.DECONV_PHASE_TAPS[b]:
                    out[a * 2 + b, t] = w[:, :, kh, kw].t()
                    t += 1
    return out


def pack_deconv(w: torch.Tensor, device) -> torch.Tensor:
    return deconv_phase_weights(w.float()).to(device=device, dtype=torch.bfloat16).contiguous()


def _nchw(rows: torch.Tensor, n: int, h: int, w: int) -> torch.Tensor:
    """[n, c, h, w] view of channel-last rows [(n h w), ld] (first c columns of the slice)."""
    c = rows.shape[1]
    return rows.as_strided((n, c, h, w), (h * w * rows.stride(0), 1, w * rows.stride(0), rows.stride(0)))


class B200VFI:
    """EMA-VFI (the reference's `Model` with `MultiScaleFlow`) on the project's sm_90a kernels.

    state_dict: `Model.net.state_dict()` of the shipped configuration, i.e. the checkpoint's keys after
    `Model.load_model` strips `module.` (its `attn_mask` / `HW` buffers are ignored)."""

    def __init__(self, state_dict, device):
        sd = check_config(state_dict)
        self.dev = dev = torch.device(device)

        def f32(t):
            return t.detach().to(device=dev, dtype=torch.float32).contiguous()

        # pack_conv3x3 zero-pads the input channels to a multiple of 8, as the A operands are (3 -> 8, 134 -> 136,
        # 81 -> 88)
        def conv(k):
            return pack_conv3x3(sd[k + ".weight"], dev), f32(sd[k + ".bias"])

        def conv_prelu(k):
            return conv(k + ".0") + (f32(sd[k + ".1.weight"]),)

        fb = "feature_bone."
        self.stem = []
        for i in range(3):
            layers = []
            if i > 0:
                layers.append(conv_prelu(fb + f"patch_embed{i + 1}"))
            for j in (0, 2):
                layers.append(conv(fb + f"block{i + 1}.conv.{j}") + (f32(sd[fb + f"block{i + 1}.conv.{j + 1}.weight"]),))
            self.stem.append(layers)
        self.cs_layers = [conv(fb + f"patch_embed4.layers.{k}") for k in range(7)]
        self.cs_proj = (pack_conv1x1(sd[fb + "patch_embed4.proj.weight"], dev), f32(sd[fb + "patch_embed4.proj.bias"]))
        self.cs_norm = (f32(sd[fb + "patch_embed4.norm.weight"]), f32(sd[fb + "patch_embed4.norm.bias"]))
        self.pe5 = conv(fb + "patch_embed5.proj")
        self.pe5_norm = (f32(sd[fb + "patch_embed5.norm.weight"]), f32(sd[fb + "patch_embed5.norm.bias"]))
        self.blocks, self.norms = {}, {}
        for st in (3, 4):
            bl = []
            for j in range(DEPTHS[st]):
                p = fb + f"block{st + 1}.{j}."
                C = EMBED[st]
                wqkv = torch.cat([sd[p + "attn.q.weight"], sd[p + "attn.kv.weight"]], 0)
                bqkv = torch.cat([sd[p + "attn.q.bias"], sd[p + "attn.kv.bias"]], 0)
                bl.append(dict(
                    n1=(f32(sd[p + "norm1.weight"]), f32(sd[p + "norm1.bias"])),
                    qkv=(pack_linear(wqkv, dev), f32(bqkv)),
                    ce=(pack_linear(sd[p + "attn.cor_embed.weight"], dev), f32(sd[p + "attn.cor_embed.bias"])),
                    proj=(pack_linear(sd[p + "attn.proj.weight"], dev), f32(sd[p + "attn.proj.bias"])),
                    mproj=(pack_linear(sd[p + "attn.motion_proj.weight"], dev), f32(sd[p + "attn.motion_proj.bias"])),
                    n2=(f32(sd[p + "norm2.weight"]), f32(sd[p + "norm2.bias"])),
                    fc1=(pack_linear(sd[p + "mlp.fc1.weight"], dev), f32(sd[p + "mlp.fc1.bias"])),
                    dw=(f32(sd[p + "mlp.dwconv.dwconv.weight"].reshape(4 * C, 9).t()),
                        f32(sd[p + "mlp.dwconv.dwconv.bias"])),
                    fc2=(pack_linear(sd[p + "mlp.fc2.weight"], dev), f32(sd[p + "mlp.fc2.bias"])),
                    shift=0 if j % 2 == 0 else 7 // 2))
            self.blocks[st] = bl
            self.norms[st] = (f32(sd[fb + f"norm{st + 1}.weight"]), f32(sd[fb + f"norm{st + 1}.bias"]))
        self.heads = [[conv_prelu(f"block.{i}.conv.{j}") for j in range(3)] for i in range(2)]
        self.down = [(conv_prelu(f"unet.down{d}.conv1"), conv_prelu(f"unet.down{d}.conv2")) for d in range(4)]
        self.up = [(pack_deconv(sd[f"unet.up{u}.0.weight"], dev), f32(sd[f"unet.up{u}.0.bias"]),
                    f32(sd[f"unet.up{u}.1.weight"])) for u in range(4)]
        self.out_conv = conv("unet.conv")
        self._cache = {}

    @classmethod
    def from_reference(cls, vfi, device="cuda"):
        """From the reference's `Trainer.Model` (after `load_model`) or its `.net` (`MultiScaleFlow`)."""
        net = getattr(vfi, "net", vfi)
        return cls(net.state_dict(), device)

    # ---------------------------------------------------------------------------------------------------------------
    def _bufs(self, H, W):
        """Per-size buffers whose padding (zero channels, the zero padding-token row, the coordinate grid) is written
        once; every call overwrites the rest."""
        key = (H, W)
        if key in self._cache:
            return self._cache[key]
        dev = self.dev
        z = lambda *s: torch.zeros(s, dtype=torch.bfloat16, device=dev)  # noqa: E731
        b = dict(imgs=torch.empty((4, 3, H, W), dtype=torch.float32, device=dev), x8=z(4, H, W, 8))
        for st, sc in ((3, 8), (4, 16)):
            h, w = H // sc, W // sc
            T = 4 * h * w
            # MotionFormer.get_cor: channel 0 = linspace over the width, 1 = over the height; the extra zero row is
            # the padding token (cor is zero-padded before cor_embed)
            cor = torch.zeros((h * w + 1, 8), dtype=torch.float32)
            cor[:h * w, 0] = torch.linspace(-1.0, 1.0, w).repeat(h)
            cor[:h * w, 1] = torch.linspace(-1.0, 1.0, h).repeat_interleave(w)
            b[f"cor{st}"] = cor.to(device=dev, dtype=torch.bfloat16)
            b[f"xa{st}"] = z(T + 1, EMBED[st])          # last row: the padding token's zero input
        b["hin0"] = z(2 * (H // 4) * (W // 4), 136)
        b["hin1"] = z(2 * (H // 2) * (W // 2), 88)
        b["u0in"] = z(2 * H * W, 88)
        self._cache[key] = b
        return b

    def _block(self, blk, xa, mslice, cor, h, w, st):
        C, heads = EMBED[st], HEADS[st - 3]
        T = 4 * h * w
        xn = ops.layer_norm(xa, *blk["n1"], 1e-6)                       # [T + 1, C]: row T = beta
        qkv = ops.linear(xn, *blk["qkv"])
        ce = ops.linear(cor, *blk["ce"])
        att = torch.empty((T, C), dtype=torch.bfloat16, device=self.dev)
        md = torch.empty((T, MOTION[st - 3]), dtype=torch.bfloat16, device=self.dev)
        ops.vfi_window_attn(qkv, ce, pairs=2, h=h, w=w, heads=heads, shift=blk["shift"], out=att, motion=md)
        xm = ops.linear(att, *blk["proj"], res1=xn[:T])                  # x_norm + proj(attn @ v)  (:265-268)
        ops.linear(md, *blk["mproj"], out=mslice)
        hdn = ops.linear(ops.layer_norm(xm, *blk["n2"], 1e-6), *blk["fc1"])
        hdn = ops.vfi_dwconv_gelu(hdn.view(4, h, w, 4 * C), *blk["dw"])
        ops.linear(hdn, *blk["fc2"], res1=xm, out=xa[:T])

    def _features(self, b, H, W):
        """MotionFormer.forward: appearance features af[0..4] (channel-last rows) and motion features of stages 3, 4."""
        dev = self.dev
        af = []
        x = b["x8"]
        for i, layers in enumerate(self.stem):
            for li, (wt, bias, slope) in enumerate(layers):
                fn = ops.conv3x3_s2 if (i > 0 and li == 0) else ops.conv3x3
                x = fn(x, wt, bias, act=ACT_PRELU, slope=slope).view(4, H >> i, W >> i, -1)
            af.append(x)
        h, w = H // 8, W // 8
        cs = torch.empty((4 * h * w, 7 * F_), dtype=torch.bfloat16, device=dev)
        ops.conv3x3_s2(af[2], *self.cs_layers[0], out=cs[:, 0:F_])
        k = 1
        for src, s, ndil in ((af[1], 4, 2), (af[0], 8, 4)):
            for d in range(1, ndil + 1):
                ops.conv3x3_strided(src, *self.cs_layers[k], stride=s, dilation=d, out=cs[:, k * F_:(k + 1) * F_])
                k += 1
        mfs = {}
        for st, sc in ((3, 8), (4, 16)):
            h, w = H // sc, W // sc
            T = 4 * h * w
            xa = b[f"xa{st}"]
            if st == 3:
                tok = ops.linear(cs, *self.cs_proj)
                ops.layer_norm(tok, *self.cs_norm, 1e-5, out=xa[:T])
            else:
                tok = ops.conv3x3_s2(af[3].view(4, 2 * h, 2 * w, EMBED[3]), *self.pe5)
                ops.layer_norm(tok, *self.pe5_norm, 1e-5, out=xa[:T])
            Cm = MOTION[st - 3]
            mf = torch.empty((T, DEPTHS[st] * Cm), dtype=torch.bfloat16, device=dev)
            for j, blk in enumerate(self.blocks[st]):
                self._block(blk, xa, mf[:, j * Cm:(j + 1) * Cm], b[f"cor{st}"], h, w, st)
            af.append(ops.layer_norm(xa[:T], *self.norms[st], 1e-6).view(4, h, w, EMBED[st]))
            mfs[st] = mf
        return af, mfs

    def _head(self, i, hin, h, w):
        """conv + PReLU x3 of Head i on its gathered input [(2 h w), cin]; the last writes the 5 channels in fp32."""
        x = hin.view(2, h, w, -1)
        (w0, b0, s0), (w1, b1, s1), (w2, b2, s2) = self.heads[i]
        x = ops.conv3x3(x, w0, b0, act=ACT_PRELU, slope=s0).view(2, h, w, -1)
        x = ops.conv3x3(x, w1, b1, act=ACT_PRELU, slope=s1).view(2, h, w, -1)
        return ops.conv3x3(x, w2, b2, act=ACT_PRELU, slope=s2, out_fp32=True)     # [(2 h w), 5]

    def _predict(self, img0, img1, pred=None, frame=None):
        _, _, H, W = img0.shape
        if H % 16 or W % 16 or H < 16 or W < 16:
            raise ValueError(f"B200VFI: H and W must be positive multiples of 16, got {H}x{W}")
        dev = self.dev
        b = self._bufs(H, W)
        imgs = b["imgs"]
        ops.vfi_pair_input(img0.contiguous(), img1.contiguous(), imgs, b["x8"])
        i0, i1 = imgs[0:2], imgs[2:4]
        af, mfs = self._features(b, H, W)
        rows = lambda t: t.view(-1, t.shape[-1])  # noqa: E731

        # MultiScaleFlow.forward (flow_estimation.py:110-141); fm = [flow (4) | mask (1)] per TTA copy
        fm = torch.empty((2, 5, H, W), dtype=torch.float32, device=dev)
        h4, w4 = H // 4, W // 4
        hin0 = b["hin0"]
        ops.vfi_head_gather(rows(mfs[4]), rows(af[4]), pairs=2, h=H // 16, w=W // 16, out=hin0)
        ops.vfi_resize(i0, _nchw(hin0[:, 128:131], 2, h4, w4), -2)
        ops.vfi_resize(i1, _nchw(hin0[:, 131:134], 2, h4, w4), -2)
        y = _nchw(self._head(0, hin0, h4, w4), 2, h4, w4)
        ops.vfi_resize(y[:, 0:4], fm[:, 0:4], 2, 4.0)
        ops.vfi_resize(y[:, 4:5], fm[:, 4:5], 2)

        w0 = torch.empty((2, 3, H, W), dtype=torch.float32, device=dev)
        w1 = torch.empty_like(w0)
        ops.vfi_warp(i0, fm[:, 0:2], w0)
        ops.vfi_warp(i1, fm[:, 2:4], w1)
        h2, w2 = H // 2, W // 2
        hin1 = b["hin1"]
        ops.vfi_head_gather(rows(mfs[3]), rows(af[3]), pairs=2, h=H // 8, w=W // 8, out=hin1)
        for c0, src in ((64, i0), (67, i1), (70, w0), (73, w1), (76, fm[:, 4:5])):
            ops.vfi_resize(src, _nchw(hin1[:, c0:c0 + src.shape[1]], 2, h2, w2), -1)
        ops.vfi_resize(fm[:, 0:4], _nchw(hin1[:, 77:81], 2, h2, w2), -1, 0.5)
        y = _nchw(self._head(1, hin1, h2, w2), 2, h2, w2)
        ops.vfi_resize(y[:, 0:4], fm[:, 0:4], 1, 2.0, accumulate=True)
        ops.vfi_resize(y[:, 4:5], fm[:, 4:5], 1, accumulate=True)
        ops.vfi_warp(i0, fm[:, 0:2], w0)
        ops.vfi_warp(i1, fm[:, 2:4], w1)

        # Unet inputs: cat(img0, img1, warped0, warped1, mask, flow, c0[0], c1[0]) and, per level, the features
        # warped by the flow halved bilinearly (warp_features, :58-66); skip concats are column slices
        c = UNET_C
        u0in = b["u0in"]
        for c0, src in ((0, i0), (3, i1), (6, w0), (9, w1), (12, fm[:, 4:5]), (13, fm[:, 0:4])):
            ops.nchw_to_nhwc(src, u0in, c0)
        ins = [u0in]
        widths = [(17 + c, 17, 32), (4 * c, 2 * c, 64), (8 * c, 4 * c, 128), (16 * c, 8 * c, 256),
                  (32 * c, 16 * c, 512)]
        for lvl in range(1, 5):
            ins.append(torch.empty((2 * (H >> lvl) * (W >> lvl), widths[lvl][0]), dtype=torch.bfloat16, device=dev))
        flow = fm[:, 0:4]
        for lvl in range(5):
            hl, wl = H >> lvl, W >> lvl
            _, c_off, cf = widths[lvl]
            fa = rows(af[lvl])
            n_img = hl * wl
            ops.vfi_warp(_nchw(fa[:2 * n_img], 2, hl, wl), flow[:, 0:2], _nchw(ins[lvl][:, c_off:c_off + cf], 2, hl, wl))
            ops.vfi_warp(_nchw(fa[2 * n_img:], 2, hl, wl), flow[:, 2:4],
                         _nchw(ins[lvl][:, c_off + cf:c_off + 2 * cf], 2, hl, wl))
            if lvl < 4:
                nxt = torch.empty((2, 4, hl // 2, wl // 2), dtype=torch.float32, device=dev)
                flow = ops.vfi_resize(flow, nxt, -1, 0.5)
        skips = []
        for d, ((wa, ba, sa), (wb, bb, sb)) in enumerate(self.down):
            hl, wl = H >> d, W >> d
            x = ops.conv3x3_s2(ins[d].view(2, hl, wl, -1), wa, ba, act=ACT_PRELU, slope=sa).view(2, hl // 2, wl // 2, -1)
            co = x.shape[-1]
            ops.conv3x3(x, wb, bb, act=ACT_PRELU, slope=sb, out=ins[d + 1][:, 0:co])
            skips.append(ins[d + 1][:, 0:co])
        x = ins[4]
        for u, (wt, bias, slope) in enumerate(self.up):
            hl, wl = H >> (4 - u), W >> (4 - u)
            co = wt.shape[2]
            if u < 3:
                nxt = torch.empty((2 * 4 * hl * wl, 2 * co), dtype=torch.bfloat16, device=dev)
                ops.copy2d(skips[2 - u], nxt[:, co:])
            else:
                nxt = torch.empty((2 * 4 * hl * wl, co), dtype=torch.bfloat16, device=dev)
            ops.conv_transpose4x4_s2(x.view(2, hl, wl, -1), wt, bias, act=ACT_PRELU, slope=slope, out=nxt[:, 0:co])
            x = nxt
        res = ops.conv3x3(x.view(2, H, W, c), *self.out_conv, out_fp32=True)          # [(2 H W), 3], pre-sigmoid
        ops.vfi_merge(w0, w1, fm, res, pred=pred, frame=frame)

    @torch.no_grad()
    def inference(self, img0, img1):
        """Model.inference(img0, img1, TTA=True, fast_TTA=True) at timestep 0.5 (Trainer.py:85-101).
        img0, img1: BGR fp32 [1, 3, H, W] in [0, 1] on the device, H and W multiples of 16.  Returns [1, 3, H, W]."""
        for t in (img0, img1):
            if t.dim() != 4 or t.shape[:2] != (1, 3) or t.dtype != torch.float32:
                raise ValueError(f"B200VFI.inference takes fp32 [1, 3, H, W] images, got {tuple(t.shape)} {t.dtype}")
        if img0.shape != img1.shape:
            raise ValueError("B200VFI.inference: the two frames differ in size")
        pred = torch.empty((1, 3) + tuple(img0.shape[2:]), dtype=torch.float32, device=self.dev)
        self._predict(img0.to(self.dev), img1.to(self.dev), pred=pred)
        return pred


def interpolate_frame_plan(num_frames: int, dest_num_frames: int):
    """The frame order of vfi_process (i2v_enhance_interface.py:30-54): ("copy", i) for an input frame passed through,
    ("mid", i) for the midpoint of frames i and i + 1.  It keeps the first dest_num_frames // 2 + 1 input frames, and
    repeats the last one when dest_num_frames is even."""
    n = min(num_frames, dest_num_frames // 2 + 1)
    if n < 1:
        raise ValueError("interpolate_video needs at least one frame")
    plan = []
    for i in range(n - 1):
        plan += [("copy", i), ("mid", i)]
    plan.append(("copy", n - 1))
    if dest_num_frames % 2 == 0:
        plan.append(("copy", n - 1))
    return plan


@torch.no_grad()
def interpolate_video(video, dest_num_frames: int, vfi: B200VFI) -> torch.Tensor:
    """`vfi_process(video, vfi, dest_num_frames)` on the GPU: uint8 RGB [F, H, W, 3] (host or device) -> uint8 RGB
    [len(plan), H, W, 3] on the device, len(plan) = 2 n - 1 (+1 if dest_num_frames is even), n = min(F,
    dest_num_frames // 2 + 1): dest_num_frames for the (dest_num_frames + 1) // 2 frames the pipeline's first stage
    makes.  Input frames are copied bit for bit (the reference's /255 and *255 round trip is the identity on uint8);
    midpoints are B200VFI's fast-TTA prediction, truncated to uint8 as the reference's astype does.

    The reference's final `PIL.Image.resize((1280, 720))` is not applied: H and W must be multiples of 16, and on the
    reference's path the frames are already 720x1280, where that resize is the identity."""
    if video.dim() != 4 or video.shape[3] != 3 or video.dtype != torch.uint8:
        raise ValueError(f"interpolate_video takes uint8 [F, H, W, 3] frames, got {tuple(video.shape)} {video.dtype}")
    _, H, W, _ = video.shape
    if H % 16 or W % 16 or H < 16 or W < 16:
        raise ValueError(f"interpolate_video: H and W must be positive multiples of 16, got {H}x{W}")
    plan = interpolate_frame_plan(video.shape[0], dest_num_frames)
    n = plan[-1][1] + 1
    frames = video[:n].to(vfi.dev).contiguous()
    bgr = ops.vfi_frames_to_bgr(frames)
    out = torch.empty((len(plan), H, W, 3), dtype=torch.uint8, device=vfi.dev)
    for k, (kind, i) in enumerate(plan):
        if kind == "copy":
            out[k].copy_(frames[i])
        else:
            vfi._predict(bgr[i:i + 1], bgr[i + 1:i + 2], frame=out[k])
    return out
