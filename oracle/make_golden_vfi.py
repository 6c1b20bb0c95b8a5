"""ORACLE tooling — build-container only (needs /root/reference).  Goldens of the EMA-VFI interpolation stage from the
UNMODIFIED reference modules (code/i2v_enhance/thirdparty/VFI/model) run on the CPU in fp32:

    tests/golden/vfi_112x224.npz   the /8 and /16 maps (14x28, 7x14) are multiples of the 7x7 window
    tests/golden/vfi_96x160.npz    they are not (12x20, 6x10): centre padding and the padding mask
    tests/golden/vfi_720x1280.npz  the size the stage runs at (90x160, 45x80: bottom / right and centre padding)

The weights are `streamingt2v_b200.vfi.seeded_state_dict(SEED)` (torch's CPU generator), so the GPU tests rebuild them
from the seed instead of storing ~60M parameters; each file keeps a per-key checksum to catch a generator change.
Each file holds two uint8 RGB frames, the reference's `Model.inference(I0, I2, TTA=True, fast_TTA=True)` on their
/255 BGR tensors, the uint8 midpoint vfi_process makes from it, and the reference's own bf16 discrepancy: the same
module under CPU bf16 autocast against fp32.

The 720x1280 file stays small: its frames are `streamingt2v_b200.synth.test_frames` of the seed (only their crc32 is
stored), and the prediction, the midpoint and the signed bf16 discrepancy are kept on REGIONS only (`synth.crop_regions`:
the four 64x64 corners, a 64x64 centre tile, the first, middle and last row and column).  Its bf16_max_err /
bf16_mean_err are taken over those regions.

The reference imports `timm.models.layers` (DropPath, to_2tuple, trunc_normal_; absent here, used only at
construction) and hard-codes `.cuda()` (flow_estimation.py:76,122): a stand-in module and an identity `Tensor.cuda`
cover both while the reference runs.  A fresh module is built per size: MotionFormerBlock caches its shifted-window
mask keyed by H_p*W_p only (feature_extractor.py:223), which both sizes share at /16 (7x14).

    python oracle/make_golden_vfi.py [--out tests/golden] [--sizes all|small|full]
"""
from __future__ import annotations

import argparse
import os
import sys
import time
import types

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
VFI_CODE = "/root/reference/code/i2v_enhance/thirdparty/VFI"
SEED = 1234
SIZES = ((112, 224), (96, 160))
FULL = (720, 1280)          # stored on regions only


def _install_timm():
    if "timm.models.layers" in sys.modules:
        return

    def to_2tuple(x):
        return tuple(x) if isinstance(x, (tuple, list)) else (x, x)

    def trunc_normal_(t, std=1.0, **_):
        with torch.no_grad():
            return nn.init.trunc_normal_(t, std=std)

    class DropPath(nn.Identity):
        def __init__(self, *_a, **_k):
            super().__init__()

    timm = types.ModuleType("timm")
    models = types.ModuleType("timm.models")
    layers = types.ModuleType("timm.models.layers")
    layers.DropPath, layers.to_2tuple, layers.trunc_normal_ = DropPath, to_2tuple, trunc_normal_
    timm.models, models.layers = models, layers
    sys.modules.update({"timm": timm, "timm.models": models, "timm.models.layers": layers})


def build_reference_net():
    """MultiScaleFlow(feature_extractor(**cfg0), **cfg1) of VFI/config.py's shipped configuration (F=32, W=7,
    depths [2, 2, 2, 4, 4]) as vfi_init builds it, with LayerNorm eps 1e-6 in the blocks."""
    from functools import partial
    _install_timm()
    if VFI_CODE not in sys.path:
        sys.path.insert(0, VFI_CODE)
    from model import feature_extractor, flow_estimation
    F, W, depth = 32, 7, [2, 2, 2, 4, 4]
    cfg0 = {'embed_dims': [F, 2 * F, 4 * F, 8 * F, 16 * F], 'motion_dims': [0, 0, 0, 8 * F // depth[-2], 16 * F // depth[-1]],
            'num_heads': [8 * F // 32, 16 * F // 32], 'mlp_ratios': [4, 4], 'qkv_bias': True,
            'norm_layer': partial(nn.LayerNorm, eps=1e-6), 'depths': depth, 'window_sizes': [W, W]}
    cfg1 = {'embed_dims': [F, 2 * F, 4 * F, 8 * F, 16 * F], 'motion_dims': [0, 0, 0, 8 * F // depth[-2], 16 * F // depth[-1]],
            'depths': depth, 'num_heads': [8 * F // 32, 16 * F // 32], 'window_sizes': [W, W], 'scales': [4, 8, 16],
            'hidden_dims': [4 * F, 4 * F], 'c': F}
    return flow_estimation(feature_extractor(**cfg0), **cfg1).eval()


def reference_inference(net, img0, img1):
    """Trainer.Model.inference(img0, img1, TTA=True, fast_TTA=True), timestep 0.5 (Trainer.py:85-96)."""
    imgs = torch.cat((img0, img1), 1)
    inp = torch.cat((imgs, imgs.flip(2).flip(3)), 0)
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        _, _, _, preds = net(inp, timestep=0.5)
    finally:
        torch.Tensor.cuda = cuda
    return (preds[0] + preds[1].flip(1).flip(2)).unsqueeze(0) / 2.


def golden(h, w):
    from streamingt2v_b200.synth import test_frames
    from streamingt2v_b200.vfi import seeded_state_dict
    torch.manual_seed(0)
    net = build_reference_net()
    sd = seeded_state_dict(SEED)
    net.load_state_dict(sd)
    fr0, fr1 = test_frames(h, w, SEED + h)
    # vfi_process: uint8 RGB / 255. (float64) -> BGR -> float32
    bgr = [torch.from_numpy((f[:, :, :3] / 255.)[:, :, ::-1].copy()).permute(2, 0, 1)[None].float() for f in (fr0, fr1)]
    with torch.no_grad():
        t0 = time.perf_counter()
        pred = reference_inference(net, *bgr)
        t1 = time.perf_counter()
        with torch.autocast("cpu", dtype=torch.bfloat16):
            pred_bf16 = reference_inference(build_fresh(sd), *bgr).float()
        t2 = time.perf_counter()
    print(f"{h}x{w}: reference fp32 {t1 - t0:.1f} s, bf16 autocast {t2 - t1:.1f} s", file=sys.stderr)
    mid = (pred[0].numpy().transpose(1, 2, 0) * 255.0).astype(np.uint8)[:, :, ::-1]
    d = (pred_bf16 - pred).abs()
    extra = {"bf16_diff": (pred_bf16 - pred).numpy()} if (h, w) == FULL else {}
    return dict(**extra, seed=np.int64(SEED), frame0=fr0, frame1=fr1, pred=pred.numpy(), mid=np.ascontiguousarray(mid),
                bf16_max_err=np.float64(d.max()), bf16_mean_err=np.float64(d.mean()),
                weight_keys=np.array(sorted(sd)), weight_sums=np.array([float(sd[k].double().sum()) for k in sorted(sd)]))


def golden_regions(h, w):
    """The full-size golden: golden(h, w) cut to synth.crop_regions, frames replaced by their crc32."""
    from streamingt2v_b200.synth import crop_regions, frames_checksum, region_spec
    g = golden(h, w)
    spec = region_spec(h, w)
    pred = g["pred"][0]                                                   # [3, h, w]
    disc = g.pop("bf16_diff")[0]
    mid = np.ascontiguousarray(g["mid"].transpose(2, 0, 1))               # [3, h, w] (RGB)
    out = dict(seed=g["seed"], height=np.int64(h), width=np.int64(w),
               frames_crc32=np.int64(frames_checksum(g["frame0"], g["frame1"])),
               pred_regions=crop_regions(pred, **spec), mid_regions=crop_regions(mid, **spec),
               bf16_diff_regions=crop_regions(disc, **spec), weight_keys=g["weight_keys"], weight_sums=g["weight_sums"],
               **{k: np.asarray(v) for k, v in spec.items()})
    d = np.abs(out["bf16_diff_regions"].astype(np.float64))
    out.update(bf16_max_err=np.float64(d.max()), bf16_mean_err=np.float64(d.mean()))
    return out


def build_fresh(sd):
    net = build_reference_net()
    net.load_state_dict(sd)
    return net


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden"))
    ap.add_argument("--sizes", default="all", choices=["all", "small", "full"],
                    help="small: 112x224 and 96x160; full: 720x1280 (regions only)")
    args = ap.parse_args()
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    sizes = (SIZES if args.sizes != "full" else ()) + ((FULL,) if args.sizes != "small" else ())
    for h, w in sizes:
        t0 = time.perf_counter()
        g = golden_regions(h, w) if (h, w) == FULL else golden(h, w)
        path = os.path.join(args.out, f"vfi_{h}x{w}.npz")
        np.savez_compressed(path, **g)
        print(f"{path}: bf16-autocast discrepancy max {g['bf16_max_err']:.4g} mean {g['bf16_mean_err']:.4g}; "
              f"{time.perf_counter() - t0:.0f} s, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
