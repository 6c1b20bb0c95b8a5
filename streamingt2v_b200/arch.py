"""Architecture plan of the StreamingSVD denoiser (VideoUNet + CAM mergers + ControlNet encoder).

A pure-Python walk of the constructor loops of the reference
(code/models/diffusion/video_model.py:94-495, code/models/control/controlnet.py:124-494) that yields
 (a) the block plan — which sub-blocks exist under which state-dict prefix, with channel counts, and
 (b) the parameter name -> shape grammar (SURVEY.md Appendix B).
The oracle (oracle/), the weight packer and the CUDA executor all consume this one description, so a mismatch
with the reference's own `state_dict()` (pinned by oracle/make_golden.py) would show up everywhere at once.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Tuple


@dataclass(frozen=True)
class UNetConfig:
    """Defaults = the shipped checkpoint config (reference code/config.yaml:69-115, :47-59)."""
    in_channels: int = 8
    model_channels: int = 320
    out_channels: int = 4
    num_res_blocks: int = 2
    attention_resolutions: Tuple[int, ...] = (4, 2, 1)
    channel_mult: Tuple[int, ...] = (1, 2, 4, 4)
    num_head_channels: int = 64
    context_dim: int = 1024
    adm_in_channels: int = 768
    use_apm: bool = False
    apm_tokens: int = 17
    # ControlNet conditioning embedding (config.yaml:54-59, use_image_encoder_normalization: true)
    cond_embed_channels: Tuple[int, ...] = (32, 96, 256, 512)
    cond_in_channels: int = 3
    num_frame_conditioning: int = 7

    @property
    def time_embed_dim(self) -> int:
        return self.model_channels * 4


TINY = UNetConfig(channel_mult=(1, 1, 2, 2))
"""Reduced same-topology config for golden fixtures / fast parity tests.  model_channels must stay 320: the
reference hard-codes the ControlNet conditioning-embedding width to 320 (controlnet.py:443-447)."""


@dataclass
class Res:
    prefix: str
    cin: int
    cout: int


@dataclass
class Attn:
    prefix: str
    ch: int

    @property
    def heads(self) -> int:
        return self.ch // 64


@dataclass
class Down:
    prefix: str  # "...N.0" ; conv at prefix + ".op"
    ch: int


@dataclass
class Up:
    prefix: str  # conv at prefix + ".conv"
    ch: int


@dataclass
class Block:
    """One TimestepEmbedSequential entry."""
    layers: list = field(default_factory=list)
    out_ch: int = 0
    ds: int = 1  # spatial downsample factor of this block's OUTPUT


@dataclass
class Plan:
    cfg: UNetConfig
    input_blocks: List[Block]
    middle: Block
    output_blocks: List[Block]  # empty for the ControlNet
    skip_chans: List[int]       # channels of hs[i] (input block outputs)


def build_plan(cfg: UNetConfig, root: str, decoder: bool = True) -> Plan:
    mc = cfg.model_channels
    inb: List[Block] = [Block(layers=[("conv_in", f"{root}input_blocks.0.0")], out_ch=mc, ds=1)]
    chans = [mc]
    ch, ds = mc, 1
    idx = 1
    nl = len(cfg.channel_mult)
    for level, mult in enumerate(cfg.channel_mult):
        for _ in range(cfg.num_res_blocks):
            layers = [Res(f"{root}input_blocks.{idx}.0", ch, mult * mc)]
            ch = mult * mc
            if ds in cfg.attention_resolutions:
                layers.append(Attn(f"{root}input_blocks.{idx}.1", ch))
            inb.append(Block(layers=layers, out_ch=ch, ds=ds))
            chans.append(ch)
            idx += 1
        if level != nl - 1:
            ds *= 2
            inb.append(Block(layers=[Down(f"{root}input_blocks.{idx}.0", ch)], out_ch=ch, ds=ds))
            chans.append(ch)
            idx += 1
    mid = Block(layers=[Res(f"{root}middle_block.0", ch, ch), Attn(f"{root}middle_block.1", ch),
                        Res(f"{root}middle_block.2", ch, ch)], out_ch=ch, ds=ds)
    outb: List[Block] = []
    if decoder:
        stack = list(chans)
        oi = 0
        for level, mult in list(enumerate(cfg.channel_mult))[::-1]:
            for i in range(cfg.num_res_blocks + 1):
                ich = stack.pop()
                layers = [Res(f"{root}output_blocks.{oi}.0", ch + ich, mc * mult)]
                ch = mc * mult
                li = 1
                if ds in cfg.attention_resolutions:
                    layers.append(Attn(f"{root}output_blocks.{oi}.{li}", ch))
                    li += 1
                if level and i == cfg.num_res_blocks:
                    ds //= 2
                    layers.append(Up(f"{root}output_blocks.{oi}.{li}", ch))
                outb.append(Block(layers=layers, out_ch=ch, ds=ds))
                oi += 1
    return Plan(cfg=cfg, input_blocks=inb, middle=mid, output_blocks=outb, skip_chans=chans)


# --------------------------------------------------------------------------------------------------------------
# parameter grammar
# --------------------------------------------------------------------------------------------------------------
def _lin(d, p, cin, cout, bias=True):
    d[p + ".weight"] = (cout, cin)
    if bias:
        d[p + ".bias"] = (cout,)


def _norm(d, p, c):
    d[p + ".weight"] = (c,)
    d[p + ".bias"] = (c,)


def _conv(d, p, cin, cout, k=3):
    d[p + ".weight"] = (cout, cin, k, k)
    d[p + ".bias"] = (cout,)


def _res_shapes(d, p, cin, cout, temb):
    _norm(d, p + ".in_layers.0", cin)
    _conv(d, p + ".in_layers.2", cin, cout)
    _lin(d, p + ".emb_layers.1", temb, cout)
    _norm(d, p + ".out_layers.0", cout)
    _conv(d, p + ".out_layers.3", cout, cout)
    if cin != cout:
        _conv(d, p + ".skip_connection", cin, cout, 1)
    t = p + ".time_stack"
    _norm(d, t + ".in_layers.0", cout)
    d[t + ".in_layers.2.weight"] = (cout, cout, 3, 1, 1)
    d[t + ".in_layers.2.bias"] = (cout,)
    _lin(d, t + ".emb_layers.1", temb, cout)
    _norm(d, t + ".out_layers.0", cout)
    d[t + ".out_layers.3.weight"] = (cout, cout, 3, 1, 1)
    d[t + ".out_layers.3.bias"] = (cout,)
    d[p + ".time_mixer.mix_factor"] = (1,)


def _xattn_shapes(d, p, c, ctx):
    _lin(d, p + ".to_q", c, c, bias=False)
    _lin(d, p + ".to_k", ctx, c, bias=False)
    _lin(d, p + ".to_v", ctx, c, bias=False)
    _lin(d, p + ".to_out.0", c, c)


def _ff_shapes(d, p, c):
    _lin(d, p + ".net.0.proj", c, 8 * c)
    _lin(d, p + ".net.2", 4 * c, c)


def _attn_shapes(d, p, c, cfg: UNetConfig):
    _norm(d, p + ".norm", c)
    _lin(d, p + ".proj_in", c, c)
    b = p + ".transformer_blocks.0"
    _xattn_shapes(d, b + ".attn1", c, c)
    _ff_shapes(d, b + ".ff", c)
    _xattn_shapes(d, b + ".attn2", c, cfg.context_dim)
    for n in ("norm1", "norm2", "norm3"):
        _norm(d, f"{b}.{n}", c)
    if cfg.use_apm:
        d[b + ".apm_conv.weight"] = (1, cfg.apm_tokens, 3)
        d[b + ".apm_conv.bias"] = (1,)
        _norm(d, b + ".apm_ln", cfg.context_dim)
        d[b + ".apm_alpha"] = ()
    _lin(d, p + ".proj_out", c, c)
    t = p + ".time_stack.0"
    _norm(d, t + ".norm_in", c)
    _ff_shapes(d, t + ".ff_in", c)
    _xattn_shapes(d, t + ".attn1", c, c)
    _ff_shapes(d, t + ".ff", c)
    _norm(d, t + ".norm2", c)
    _xattn_shapes(d, t + ".attn2", c, cfg.context_dim)
    _norm(d, t + ".norm1", c)
    _norm(d, t + ".norm3", c)
    _lin(d, p + ".time_pos_embed.0", c, 4 * c)
    _lin(d, p + ".time_pos_embed.2", 4 * c, c)
    d[p + ".time_mixer.mix_factor"] = (1,)


def _cam_shapes(d, p, c):
    t = p + ".temporal_transformer"
    _lin(d, t + ".attention.to_q", c, c, bias=False)
    _lin(d, t + ".attention.to_k", c, c, bias=False)
    _lin(d, t + ".attention.to_v", c, c, bias=False)
    _lin(d, t + ".attention.to_out.0", c, c)
    _norm(d, t + ".norm", c)
    _lin(d, t + ".proj_in", c, c)
    _lin(d, t + ".proj_out", c, c)


def _plan_shapes(d, plan: Plan, root: str):
    cfg = plan.cfg
    temb = cfg.time_embed_dim
    _lin(d, root + "time_embed.0", cfg.model_channels, temb)
    _lin(d, root + "time_embed.2", temb, temb)
    _lin(d, root + "label_emb.0.0", cfg.adm_in_channels, temb)
    _lin(d, root + "label_emb.0.2", temb, temb)
    for blk in plan.input_blocks + [plan.middle] + plan.output_blocks:
        for layer in blk.layers:
            if isinstance(layer, tuple):
                _conv(d, layer[1], cfg.in_channels, cfg.model_channels)
            elif isinstance(layer, Res):
                _res_shapes(d, layer.prefix, layer.cin, layer.cout, temb)
            elif isinstance(layer, Attn):
                _attn_shapes(d, layer.prefix, layer.ch, cfg)
            elif isinstance(layer, Down):
                _conv(d, layer.prefix + ".op", layer.ch, layer.ch)
            elif isinstance(layer, Up):
                _conv(d, layer.prefix + ".conv", layer.ch, layer.ch)


def unet_param_shapes(cfg: UNetConfig, root: str = "") -> Dict[str, tuple]:
    """Name -> shape of VideoUNet.state_dict() (controlnet_mode, attention_cross_attention merging)."""
    d: Dict[str, tuple] = {}
    plan = build_plan(cfg, root, decoder=True)
    # registration order in the reference differs; only names/shapes matter
    _plan_shapes(d, plan, root)
    for i, c in enumerate(plan.skip_chans):
        _cam_shapes(d, f"{root}cross_attention_merger_input_blocks.{i}", c)
    _cam_shapes(d, f"{root}cross_attention_merger_mid_block", plan.middle.out_ch)
    _norm(d, root + "out.0", cfg.model_channels)
    _conv(d, root + "out.2", cfg.model_channels, cfg.out_channels)
    return d


def plain_unet_param_shapes(cfg: UNetConfig, root: str = "") -> Dict[str, tuple]:
    """The UNet WITHOUT the CAM mergers: what the first chunk's plain SVD network holds (streaming_svd.py:390)."""
    d = unet_param_shapes(cfg, root)
    return {k: v for k, v in d.items() if "cross_attention_merger_" not in k}


# --------------------------------------------------------------------------------------------------------------
# diffusers weight layout of the first chunk
# --------------------------------------------------------------------------------------------------------------
_RES_MAP = (("in_layers.0", "spatial_res_block.norm1"), ("in_layers.2", "spatial_res_block.conv1"),
            ("emb_layers.1", "spatial_res_block.time_emb_proj"), ("out_layers.0", "spatial_res_block.norm2"),
            ("out_layers.3", "spatial_res_block.conv2"), ("skip_connection", "spatial_res_block.conv_shortcut"),
            ("time_stack.in_layers.0", "temporal_res_block.norm1"), ("time_stack.in_layers.2", "temporal_res_block.conv1"),
            ("time_stack.emb_layers.1", "temporal_res_block.time_emb_proj"),
            ("time_stack.out_layers.0", "temporal_res_block.norm2"), ("time_stack.out_layers.3", "temporal_res_block.conv2"),
            ("time_mixer", "time_mixer"))
_ATTN_MAP = (("time_stack.0", "temporal_transformer_blocks.0"), ("time_pos_embed.0", "time_pos_embed.linear_1"),
             ("time_pos_embed.2", "time_pos_embed.linear_2"))   # every other sub-module keeps its name


def sgm_to_diffusers_svd_keys(cfg: UNetConfig) -> Dict[str, str]:
    """SGM key -> key of diffusers' `UNetSpatioTemporalConditionModel.state_dict()` for the plain SVD UNet.

    The first chunk of a request is produced by `StableVideoDiffusionPipeline` (reference
    code/diffusion_trainer/streaming_svd.py:390, checkpoint in the diffusers layout, config.yaml:283-294): 25 of the
    175 UNet evaluations of a 200-frame request.  Same architecture as `VideoUNet` minus the CAM mergers, so the same
    kernels serve it once the names are translated.  The table restates the module correspondence of diffusers'
    public SVD conversion (block order of openaimodel.UNetModel vs down/mid/up blocks; VideoResBlock =
    SpatioTemporalResBlock{spatial_res_block, temporal_res_block, time_mixer}; SpatialVideoTransformer =
    TransformerSpatioTemporalModel{transformer_blocks, temporal_transformer_blocks, time_pos_embed, time_mixer}).
    diffusers is not installed offline: parity unpinned — `tests/test_arch.py` checks that the map is a bijection
    onto the SGM grammar; a wrong name fails loudly at load time (missing key), never silently."""
    plan = build_plan(cfg, "", decoder=True)
    nrb = cfg.num_res_blocks
    prefix: Dict[str, str] = {"time_embed.0": "time_embedding.linear_1", "time_embed.2": "time_embedding.linear_2",
                              "label_emb.0.0": "add_embedding.linear_1", "label_emb.0.2": "add_embedding.linear_2",
                              "input_blocks.0.0": "conv_in", "out.0": "conv_norm_out", "out.2": "conv_out",
                              "middle_block.0": "mid_block.resnets.0", "middle_block.1": "mid_block.attentions.0",
                              "middle_block.2": "mid_block.resnets.1"}
    idx = 1
    for level in range(len(cfg.channel_mult)):
        for j in range(nrb):
            prefix[f"input_blocks.{idx}.0"] = f"down_blocks.{level}.resnets.{j}"
            prefix[f"input_blocks.{idx}.1"] = f"down_blocks.{level}.attentions.{j}"
            idx += 1
        if level != len(cfg.channel_mult) - 1:
            prefix[f"input_blocks.{idx}.0.op"] = f"down_blocks.{level}.downsamplers.0.conv"
            idx += 1
    for oi, blk in enumerate(plan.output_blocks):
        u, j = divmod(oi, nrb + 1)
        for li, layer in enumerate(blk.layers):
            if isinstance(layer, Res):
                prefix[f"output_blocks.{oi}.{li}"] = f"up_blocks.{u}.resnets.{j}"
            elif isinstance(layer, Attn):
                prefix[f"output_blocks.{oi}.{li}"] = f"up_blocks.{u}.attentions.{j}"
            elif isinstance(layer, Up):
                prefix[f"output_blocks.{oi}.{li}.conv"] = f"up_blocks.{u}.upsamplers.0.conv"
    out: Dict[str, str] = {}
    for key in plain_unet_param_shapes(cfg):
        best = max((p for p in prefix if key == p or key.startswith(p + ".")), key=len, default=None)
        if best is None:
            raise KeyError(f"no diffusers counterpart for {key}")
        rest = key[len(best):].lstrip(".")
        is_res = ".resnets." in prefix[best]
        for a, b in (_RES_MAP if is_res else _ATTN_MAP if ".attentions." in prefix[best] else ()):
            if rest == a or rest.startswith(a + "."):
                rest = b + rest[len(a):]
                break
        out[key] = prefix[best] + ("." + rest if rest else "")
    return out


def from_diffusers_svd_state_dict(sd_diffusers: Dict[str, "torch.Tensor"], cfg: UNetConfig) -> Dict[str, "torch.Tensor"]:
    """State dict of `UNetSpatioTemporalConditionModel` -> SGM-named state dict that B200Denoiser / the oracle load."""
    m = sgm_to_diffusers_svd_keys(cfg)
    missing = [d for d in m.values() if d not in sd_diffusers]
    if missing:
        raise KeyError(f"{len(missing)} keys missing in the diffusers state dict, e.g. {missing[:4]}")
    shapes = plain_unet_param_shapes(cfg)
    out = {}
    for k, d in m.items():
        t = sd_diffusers[d]
        if tuple(t.shape) != tuple(shapes[k]):
            raise ValueError(f"{d}: shape {tuple(t.shape)} != {shapes[k]} expected for {k}")
        out[k] = t
    return out


def controlnet_param_shapes(cfg: UNetConfig, root: str = "") -> Dict[str, tuple]:
    """Name -> shape of ControlNet.state_dict() (ControlNet.from_unet, use_image_encoder_normalization)."""
    import dataclasses
    d: Dict[str, tuple] = {}
    ccfg = dataclasses.replace(cfg, use_apm=False)  # the ControlNet never uses APM (controlnet.py:176-199)
    plan = build_plan(ccfg, root, decoder=False)
    _plan_shapes(d, plan, root)
    e = root + "controlnet_cond_embedding"
    boc = cfg.cond_embed_channels
    _conv(d, e + ".conv_in", cfg.cond_in_channels, boc[0])
    bi = 0
    for i in range(len(boc) - 1):
        _conv(d, f"{e}.blocks.{bi}", boc[i], boc[i])
        _norm(d, f"{e}.norms.{bi}", boc[i])
        bi += 1
        _conv(d, f"{e}.blocks.{bi}", boc[i], boc[i + 1])
        _norm(d, f"{e}.norms.{bi}", boc[i + 1])
        bi += 1
    _conv(d, e + ".conv_out", boc[-1], 320)  # hard-coded block_out_channels[0] (controlnet.py:443-447)
    return d


def synth_state_dict(shapes: Dict[str, tuple], seed: int = 0):
    """Deterministic synthetic weights, independent of module construction order: each tensor is drawn from a
    numpy Generator seeded by (seed, crc32(name)).  Every tensor is non-zero — the reference zero-initialises
    ResBlock out convs, transformer proj_out, UNet out conv, CAM proj_out and ControlNet conv_out
    (openaimodel.py:296, attention.py:775-780, video_model.py:493, conditioning.py:113-114, controlnet.py:99-102),
    which would make parity vacuous."""
    import zlib

    import numpy as np
    import torch
    sd = {}
    for name in sorted(shapes):
        shape = shapes[name]
        rng = np.random.default_rng([seed, zlib.crc32(name.encode())])
        leaf = name.rsplit(".", 1)[-1]
        if name.endswith("mix_factor"):
            v = rng.normal(0.0, 0.7, size=shape)
        elif name.endswith("apm_alpha"):
            v = np.asarray(0.6)
        elif leaf == "weight" and len(shape) == 1:      # norm gains
            v = 1.0 + 0.1 * rng.normal(size=shape)
        elif leaf == "bias":
            v = 0.05 * rng.normal(size=shape)
        else:                                            # linear / conv weights: fan-in scaled
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            v = rng.normal(size=shape) * (fan_in ** -0.5)
        sd[name] = torch.from_numpy(np.asarray(v, dtype=np.float32).reshape(shape)).clone()
    return sd


def synth_state_dict_device(shapes: Dict[str, tuple], device, seed: int = 0):
    """Fast on-device variant of synth_state_dict for full-size benchmarks (same distribution family, values not
    reproducible across devices — use synth_state_dict wherever outputs are compared)."""
    import torch
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    sd = {}
    for name in sorted(shapes):
        shape = shapes[name]
        leaf = name.rsplit(".", 1)[-1]
        if name.endswith("mix_factor"):
            v = torch.randn(shape, generator=g, device=device) * 0.7
        elif name.endswith("apm_alpha"):
            v = torch.tensor(0.6, device=device)
        elif leaf == "weight" and len(shape) == 1:
            v = 1.0 + 0.1 * torch.randn(shape, generator=g, device=device)
        elif leaf == "bias":
            v = 0.05 * torch.randn(shape, generator=g, device=device)
        else:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            v = torch.randn(shape, generator=g, device=device) * (fan_in ** -0.5)
        sd[name] = v
    return sd


def synth_state_dict_fast(shapes: Dict[str, tuple], seed: int = 0):
    """CPU, torch-generator variant of synth_state_dict (seconds instead of ~25 s for 0.7 G parameters).
    Deterministic for a given torch build; used where both sides of a comparison run in the same process
    (smoke(), host-logic tests) — the golden fixtures use synth_state_dict."""
    import torch
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name in sorted(shapes):
        shape = shapes[name]
        leaf = name.rsplit(".", 1)[-1]
        if name.endswith("mix_factor"):
            v = torch.randn(shape, generator=g) * 0.7
        elif name.endswith("apm_alpha"):
            v = torch.tensor(0.6)
        elif leaf == "weight" and len(shape) == 1:
            v = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif leaf == "bias":
            v = 0.05 * torch.randn(shape, generator=g)
        else:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            v = torch.randn(shape, generator=g) * (fan_in ** -0.5)
        sd[name] = v
    return sd


# --------------------------------------------------------------------------------------------------------------
# temporal VAE decoder (AutoencodingEngine.decode -> VideoDecoder; reference
# code/models/svd/sgm/modules/autoencoding/temporal_ae.py:291-347, diffusionmodules/model.py:604-748)
# --------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class VaeConfig:
    """Defaults = decoder_config of the shipped checkpoint (reference code/config.yaml:242-257)."""
    ch: int = 128
    ch_mult: Tuple[int, ...] = (1, 2, 4, 4)
    num_res_blocks: int = 2
    z_channels: int = 4
    out_ch: int = 3


def vae_decoder_plan(cfg: VaeConfig):
    """[(kind, prefix, cin, cout)] in execution order (Decoder.forward, model.py:715-748)."""
    plan = []
    block_in = cfg.ch * cfg.ch_mult[-1]
    plan.append(("conv_in", "conv_in", cfg.z_channels, block_in))
    plan.append(("res", "mid.block_1", block_in, block_in))
    plan.append(("attn", "mid.attn_1", block_in, block_in))
    plan.append(("res", "mid.block_2", block_in, block_in))
    for i_level in reversed(range(len(cfg.ch_mult))):
        block_out = cfg.ch * cfg.ch_mult[i_level]
        for i_block in range(cfg.num_res_blocks + 1):
            plan.append(("res", f"up.{i_level}.block.{i_block}", block_in, block_out))
            block_in = block_out
        if i_level != 0:
            plan.append(("up", f"up.{i_level}.upsample", block_in, block_in))
    plan.append(("out", "", block_in, cfg.out_ch))
    return plan


def vae_decoder_param_shapes(cfg: VaeConfig) -> Dict[str, tuple]:
    d: Dict[str, tuple] = {}
    for kind, p, cin, cout in vae_decoder_plan(cfg):
        if kind == "conv_in":
            _conv(d, p, cin, cout)
        elif kind == "res":
            _norm(d, p + ".norm1", cin)
            _conv(d, p + ".conv1", cin, cout)
            _norm(d, p + ".norm2", cout)
            _conv(d, p + ".conv2", cout, cout)
            if cin != cout:
                _conv(d, p + ".nin_shortcut", cin, cout, 1)
            t = p + ".time_stack"
            _norm(d, t + ".in_layers.0", cout)
            d[t + ".in_layers.2.weight"] = (cout, cout, 3, 1, 1)
            d[t + ".in_layers.2.bias"] = (cout,)
            _norm(d, t + ".out_layers.0", cout)
            d[t + ".out_layers.3.weight"] = (cout, cout, 3, 1, 1)
            d[t + ".out_layers.3.bias"] = (cout,)
            d[p + ".mix_factor"] = (1,)
        elif kind == "attn":
            _norm(d, p + ".norm", cin)
            for n in ("q", "k", "v", "proj_out"):
                _conv(d, f"{p}.{n}", cin, cin, 1)
        elif kind == "up":
            _conv(d, p + ".conv", cin, cin)
        elif kind == "out":
            _norm(d, "norm_out", cin)
            _conv(d, "conv_out", cin, cout)
            d["conv_out.time_mix_conv.weight"] = (cout, cout, 3, 1, 1)
            d["conv_out.time_mix_conv.bias"] = (cout,)
    return d


# --------------------------------------------------------------------------------------------------------------
# SD-VAE encoder of the conditioner (AutoencoderKLModeOnly.encode -> Encoder + quant_conv -> mode; reference
# code/models/svd/sgm/modules/diffusionmodules/model.py:487-601, models/autoencoder.py:454-473,602-615;
# used per chunk by VideoPredictionEmbedderWithEncoder, encoders/modules.py:697-729) — SURVEY.md section 8 row f1
# --------------------------------------------------------------------------------------------------------------
def vae_encoder_plan(cfg: VaeConfig):
    """[(kind, prefix, cin, cout)] in execution order (Encoder.forward, model.py:578-601)."""
    plan = [("conv_in", "conv_in", 3, cfg.ch)]
    block_in = cfg.ch
    for i_level, mult in enumerate(cfg.ch_mult):
        block_out = cfg.ch * mult
        for i_block in range(cfg.num_res_blocks):
            plan.append(("res", f"down.{i_level}.block.{i_block}", block_in, block_out))
            block_in = block_out
        if i_level != len(cfg.ch_mult) - 1:
            plan.append(("down", f"down.{i_level}.downsample", block_in, block_in))
    plan.append(("res", "mid.block_1", block_in, block_in))
    plan.append(("attn", "mid.attn_1", block_in, block_in))
    plan.append(("res", "mid.block_2", block_in, block_in))
    plan.append(("out", "", block_in, 2 * cfg.z_channels))
    return plan


def vae_encoder_param_shapes(cfg: VaeConfig) -> Dict[str, tuple]:
    """Name -> shape of `Encoder.state_dict()` plus the engine's `quant_conv` (autoencoder.py:454-458), the latter
    under the key `quant_conv.*` as in the checkpoint (`first_stage_model.quant_conv`)."""
    d: Dict[str, tuple] = {}
    for kind, p, cin, cout in vae_encoder_plan(cfg):
        if kind == "conv_in":
            _conv(d, p, cin, cout)
        elif kind == "res":
            _norm(d, p + ".norm1", cin)
            _conv(d, p + ".conv1", cin, cout)
            _norm(d, p + ".norm2", cout)
            _conv(d, p + ".conv2", cout, cout)
            if cin != cout:
                _conv(d, p + ".nin_shortcut", cin, cout, 1)
        elif kind == "down":
            _conv(d, p + ".conv", cin, cin)
        elif kind == "attn":
            _norm(d, p + ".norm", cin)
            for n in ("q", "k", "v", "proj_out"):
                _conv(d, f"{p}.{n}", cin, cin, 1)
        elif kind == "out":
            _norm(d, "norm_out", cin)
            _conv(d, "conv_out", cin, cout)
    _conv(d, "quant_conv", 2 * cfg.z_channels, 2 * cfg.z_channels, 1)
    return d


# --------------------------------------------------------------------------------------------------------------
# OpenCLIP ViT-H/14 image tower of the conditioner (FrozenOpenCLIPImageEmbedder, reference
# code/models/svd/sgm/modules/encoders/modules.py:574-733 -> open_clip 2.24 VisionTransformer, visual tower only)
# --------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class ClipVisionConfig:
    """Defaults = open_clip's ViT-H-14 vision config (width 1280, 32 layers, head width 80, MLP ratio 4, embed 1024)."""
    image_size: int = 224
    patch_size: int = 14
    width: int = 1280
    layers: int = 32
    heads: int = 16
    mlp: int = 5120
    output_dim: int = 1024
    eps: float = 1e-5

    @property
    def head_dim(self) -> int:
        return self.width // self.heads

    @property
    def grid(self) -> int:
        return self.image_size // self.patch_size

    @property
    def tokens(self) -> int:
        return self.grid * self.grid + 1


CLIP_TINY = ClipVisionConfig(width=160, layers=2, heads=2, mlp=640)
"""Reduced same-topology tower for fast parity tests: head dim stays 80, still 224 / 14 and a 1024-wide projection."""


def clip_visual_param_shapes(cfg: ClipVisionConfig) -> Dict[str, tuple]:
    """Name -> shape of open_clip's `model.visual.state_dict()` (VisionTransformer with the default options of
    ViT-H-14: no conv bias, class token, learned positional embedding, ln_pre, pre-LN ResidualAttentionBlocks over
    nn.MultiheadAttention (fused in_proj), ln_post, `proj` [width, output_dim]).  In the SVD checkpoint these keys sit
    under `conditioner.embedders.0.open_clip.model.visual.`.  Restated from open_clip's published source: neither
    open_clip nor a checkpoint is available offline, so this layout is not checked against one."""
    w, p = cfg.width, cfg.patch_size
    d: Dict[str, tuple] = {"conv1.weight": (w, 3, p, p), "class_embedding": (w,),
                           "positional_embedding": (cfg.tokens, w)}
    _norm(d, "ln_pre", w)
    for i in range(cfg.layers):
        b = f"transformer.resblocks.{i}"
        _norm(d, b + ".ln_1", w)
        d[b + ".attn.in_proj_weight"] = (3 * w, w)
        d[b + ".attn.in_proj_bias"] = (3 * w,)
        _lin(d, b + ".attn.out_proj", w, w)
        _norm(d, b + ".ln_2", w)
        _lin(d, b + ".mlp.c_fc", w, cfg.mlp)
        _lin(d, b + ".mlp.c_proj", cfg.mlp, w)
    _norm(d, "ln_post", w)
    d["proj"] = (w, cfg.output_dim)
    return d


def clip_vision_config_from_hf(hcfg) -> ClipVisionConfig:
    """ClipVisionConfig of a transformers `CLIPVisionConfig` (the `config` of `CLIPVisionModelWithProjection`, the
    `image_encoder` of the SVD-XT checkpoint).  The tower computes erf GELU, so any other `hidden_act` is rejected."""
    if hcfg.hidden_act != "gelu":
        raise ValueError(f"hidden_act {hcfg.hidden_act!r}: the CLIP tower computes erf GELU ('gelu') only")
    return ClipVisionConfig(image_size=hcfg.image_size, patch_size=hcfg.patch_size, width=hcfg.hidden_size,
                            layers=hcfg.num_hidden_layers, heads=hcfg.num_attention_heads,
                            mlp=hcfg.intermediate_size, output_dim=hcfg.projection_dim, eps=hcfg.layer_norm_eps)


def _check_shapes(out: Dict[str, "torch.Tensor"], shapes: Dict[str, tuple], what: str):
    if set(out) != set(shapes):
        raise KeyError(f"{what}: mapped keys differ from the grammar: missing {sorted(set(shapes) - set(out))[:4]}, "
                       f"extra {sorted(set(out) - set(shapes))[:4]}")
    for k, t in out.items():
        if tuple(t.shape) != tuple(shapes[k]):
            raise ValueError(f"{what}: {k} has shape {tuple(t.shape)}, expected {shapes[k]}")


def from_hf_clip_vision_state_dict(sd: Dict[str, "torch.Tensor"], cfg) -> Dict[str, "torch.Tensor"]:
    """State dict of transformers' `CLIPVisionModelWithProjection` -> open_clip `visual` layout
    (clip_visual_param_shapes) that B200ClipImageEncoder reads.  `cfg` is the model's transformers CLIPVisionConfig.

    q/k/v_proj are concatenated into in_proj_weight / in_proj_bias (open_clip's nn.MultiheadAttention packs them in
    that order), visual_projection.weight is stored transposed as `proj`, pre_layrnorm / post_layernorm become
    ln_pre / ln_post and the embeddings are renamed.  `vision_model.embeddings.position_ids` (a buffer, not a weight)
    is ignored; any other key left over is an error.  Restated from transformers' published CLIP modelling source;
    the test suite runs transformers' own model on the renamed weights."""
    import torch
    ccfg = clip_vision_config_from_hf(cfg)
    v = "vision_model."
    out = {"conv1.weight": sd[v + "embeddings.patch_embedding.weight"],
           "class_embedding": sd[v + "embeddings.class_embedding"],
           "positional_embedding": sd[v + "embeddings.position_embedding.weight"],
           "ln_pre.weight": sd[v + "pre_layrnorm.weight"], "ln_pre.bias": sd[v + "pre_layrnorm.bias"],
           "ln_post.weight": sd[v + "post_layernorm.weight"], "ln_post.bias": sd[v + "post_layernorm.bias"],
           "proj": sd["visual_projection.weight"].t().contiguous()}
    used = {v + "embeddings.patch_embedding.weight", v + "embeddings.class_embedding",
            v + "embeddings.position_embedding.weight", v + "pre_layrnorm.weight", v + "pre_layrnorm.bias",
            v + "post_layernorm.weight", v + "post_layernorm.bias", "visual_projection.weight"}
    for i in range(ccfg.layers):
        b, h = f"transformer.resblocks.{i}", f"{v}encoder.layers.{i}"
        for leaf in ("weight", "bias"):
            qkv = [f"{h}.self_attn.{n}_proj.{leaf}" for n in "qkv"]
            out[f"{b}.attn.in_proj_{leaf}"] = torch.cat([sd[k] for k in qkv], 0)
            used.update(qkv)
            for a, o in (("attn.out_proj", "self_attn.out_proj"), ("ln_1", "layer_norm1"), ("ln_2", "layer_norm2"),
                         ("mlp.c_fc", "mlp.fc1"), ("mlp.c_proj", "mlp.fc2")):
                out[f"{b}.{a}.{leaf}"] = sd[f"{h}.{o}.{leaf}"]
                used.add(f"{h}.{o}.{leaf}")
    extra = sorted(k for k in sd if k not in used and not k.endswith("position_ids"))
    if extra:
        raise KeyError(f"{len(extra)} CLIP keys without an open_clip counterpart, e.g. {extra[:4]}")
    _check_shapes(out, clip_visual_param_shapes(ccfg), "CLIP vision")
    return out


# --------------------------------------------------------------------------------------------------------------
# diffusers weight layout of the SVD-XT VAE (AutoencoderKLTemporalDecoder: SD-VAE Encoder + quant_conv, TemporalDecoder)
# --------------------------------------------------------------------------------------------------------------
_VAE_RES_MAP = (("norm1", "norm1"), ("conv1", "conv1"), ("norm2", "norm2"), ("conv2", "conv2"),
                ("nin_shortcut", "conv_shortcut"))
# decoder resnets are SpatioTemporalResBlocks: the spatial ResnetBlock2D sits under spatial_res_block
_VAE_VIDEO_RES_MAP = tuple((a, "spatial_res_block." + b) for a, b in _VAE_RES_MAP) + (
    ("time_stack.in_layers.0", "temporal_res_block.norm1"), ("time_stack.in_layers.2", "temporal_res_block.conv1"),
    ("time_stack.out_layers.0", "temporal_res_block.norm2"), ("time_stack.out_layers.3", "temporal_res_block.conv2"),
    ("mix_factor", "time_mixer.mix_factor"))
_VAE_ATTN_MAP = (("norm", "group_norm"), ("q", "to_q"), ("k", "to_k"), ("v", "to_v"), ("proj_out", "to_out.0"))


def _vae_prefix_map(plan, n_levels: int, side: str) -> Dict[str, str]:
    """SGM module prefix -> diffusers module prefix for one side ("encoder" or "decoder") of the VAE."""
    m = {"conv_in": "conv_in", "mid.block_1": "mid_block.resnets.0", "mid.attn_1": "mid_block.attentions.0",
         "mid.block_2": "mid_block.resnets.1", "norm_out": "conv_norm_out", "conv_out": "conv_out"}
    for kind, p, _, _ in plan:
        parts = p.split(".")
        if parts[0] == "down":                       # encoder: down_blocks in SGM order
            i = int(parts[1])
            m[p] = (f"down_blocks.{i}.resnets.{parts[3]}" if kind == "res" else f"down_blocks.{i}.downsamplers.0")
        elif parts[0] == "up":                       # decoder: up_blocks.0 is the deepest level, up.{n-1}
            i = n_levels - 1 - int(parts[1])
            m[p] = (f"up_blocks.{i}.resnets.{parts[3]}" if kind == "res" else f"up_blocks.{i}.upsamplers.0")
    if side == "encoder":
        m["quant_conv"] = "quant_conv"
    else:
        m["conv_out.time_mix_conv"] = "time_conv_out"
    return m


def _sgm_to_diffusers_vae_keys(shapes: Dict[str, tuple], plan, n_levels: int, side: str) -> Dict[str, str]:
    kinds = {p: kind for kind, p, _, _ in plan}
    prefix = _vae_prefix_map(plan, n_levels, side)
    out: Dict[str, str] = {}
    for key in shapes:
        best = max((p for p in prefix if key.startswith(p + ".")), key=len)
        rest = key[len(best) + 1:]
        table = ((_VAE_VIDEO_RES_MAP if side == "decoder" else _VAE_RES_MAP) if kinds.get(best) == "res"
                 else _VAE_ATTN_MAP if kinds.get(best) == "attn" else ())
        for a, b in table:
            if rest == a or rest.startswith(a + "."):
                rest = b + rest[len(a):]
                break
        d = prefix[best] + "." + rest
        out[key] = d if best == "quant_conv" else f"{side}.{d}"
    return out


def sgm_to_diffusers_vae_encoder_keys(cfg: VaeConfig) -> Dict[str, str]:
    """vae_encoder_param_shapes key -> key of diffusers' `AutoencoderKLTemporalDecoder.state_dict()`."""
    return _sgm_to_diffusers_vae_keys(vae_encoder_param_shapes(cfg), vae_encoder_plan(cfg), len(cfg.ch_mult), "encoder")


def sgm_to_diffusers_vae_decoder_keys(cfg: VaeConfig) -> Dict[str, str]:
    """vae_decoder_param_shapes key -> key of diffusers' `AutoencoderKLTemporalDecoder.state_dict()`."""
    return _sgm_to_diffusers_vae_keys(vae_decoder_param_shapes(cfg), vae_decoder_plan(cfg), len(cfg.ch_mult), "decoder")


def from_diffusers_svd_vae_state_dict(sd: Dict[str, "torch.Tensor"], cfg: VaeConfig):
    """State dict of diffusers' `AutoencoderKLTemporalDecoder` (`svd_pipeline.vae`) -> (encoder, decoder) state dicts
    in the SGM grammar that B200VaeEncoder (`encoder.*` + `quant_conv.*`) and B200VaeDecoder (`decoder.*`) read.

    The correspondence, restated from diffusers 0.30.2's published source (diffusers is not a dependency: parity is
    unpinned, as for sgm_to_diffusers_svd_keys; a wrong name fails at load time as a missing key, never silently):
      down_blocks.i / up_blocks.i    down.i / up.{n-1-i}: the decoder's up_blocks run deepest level first
      resnets.j.spatial_res_block.*  block.j.*  (conv_shortcut -> nin_shortcut)
      resnets.j.temporal_res_block   block.j.time_stack  (norm1 / conv1 / norm2 / conv2 -> in_layers.0 / .2,
                                     out_layers.0 / .3)
      resnets.j.time_mixer.mix_factor  block.j.mix_factor, unchanged: diffusers' AlphaBlender(merge_strategy="learned",
                                     switch_spatial_to_temporal_mix=True) takes a = 1 - sigmoid(m) and returns
                                     a * x_spatial + (1 - a) * x_temporal = (1 - sigmoid(m)) x_s + sigmoid(m) x_t, which
                                     is SGM VideoResBlock's sigmoid(m) x_t + (1 - sigmoid(m)) x_s for the same m
      mid_block.attentions.0         mid.attn_1: group_norm -> norm, to_q/k/v -> q/k/v, to_out.0 -> proj_out; the
                                     diffusers Linear [C, C] is the SGM 1x1 conv [C, C, 1, 1] (a reshape only)
      conv_norm_out                  norm_out
      time_conv_out                  conv_out.time_mix_conv
      downsamplers.0 / upsamplers.0  downsample / upsample
    Missing keys, keys left over and shape mismatches other than the attention reshape raise."""
    out = []
    used = set()
    for m, shapes in ((sgm_to_diffusers_vae_encoder_keys(cfg), vae_encoder_param_shapes(cfg)),
                      (sgm_to_diffusers_vae_decoder_keys(cfg), vae_decoder_param_shapes(cfg))):
        missing = [d for d in m.values() if d not in sd]
        if missing:
            raise KeyError(f"{len(missing)} keys missing in the diffusers VAE state dict, e.g. {missing[:4]}")
        part = {}
        for k, d in m.items():
            t = sd[d]
            if t.dim() == 2 and len(shapes[k]) == 4:       # attention Linear -> 1x1 conv
                t = t.reshape(shapes[k])
            part[k] = t
        _check_shapes(part, shapes, "VAE")
        used.update(m.values())
        out.append(part)
    extra = sorted(k for k in sd if k not in used)
    if extra:
        raise KeyError(f"{len(extra)} VAE keys without an SGM counterpart, e.g. {extra[:4]}")
    return out[0], out[1]
