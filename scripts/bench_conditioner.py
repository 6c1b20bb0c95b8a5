"""Benchmark of the SVD conditioner (B200SVDConditioner: CLIP preprocessing + ViT-H/14 image tower + SD-VAE encoder +
conditioning assembly) at the StreamingSVD chunk shape: one 576x1024 anchor frame, T = 25, full-size synthetic weights.

Prints one JSON line: median ms per conditioner call over >= 20 warmed calls (CUDA events), the per-family split from
ops.profile(), launches per call, the GPU name and power limit (read-only nvidia-smi query), and the same computation
as eager PyTorch under fp16 autocast (oracle restatements, SDPA attention) on the same GPU as a baseline.
Needs a CUDA device; writes nothing.    python scripts/bench_conditioner.py [--calls 20] [--warmup 3]"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
        return name, power
    except Exception as e:  # noqa: BLE001
        return torch.cuda.get_device_name(0), f"unknown ({e.__class__.__name__})"


def _time(fn, calls, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(calls):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return statistics.median(ms), min(ms), max(ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--H", type=int, default=576)
    ap.add_argument("--W", type=int, default=1024)
    ap.add_argument("--T", type=int, default=25)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_conditioner.py needs a CUDA device (H100)")
    from oracle import clip_image_oracle as co
    from oracle import vae_encoder_oracle as vo
    from streamingt2v_b200 import _lib, arch, ops
    from streamingt2v_b200.conditioner import B200ClipImageEncoder, B200SVDConditioner
    from streamingt2v_b200.vae import B200VaeEncoder
    dev = torch.device("cuda:0")
    _lib.init(0)
    ccfg, vcfg = arch.ClipVisionConfig(), arch.VaeConfig()
    sd_c = arch.synth_state_dict_device(arch.clip_visual_param_shapes(ccfg), dev, seed=1)
    sd_v = arch.synth_state_dict_device(arch.vae_encoder_param_shapes(vcfg), dev, seed=2)
    cond = B200SVDConditioner(B200ClipImageEncoder(ccfg, sd_c, dev), B200VaeEncoder(vcfg, sd_v, dev),
                              generator=torch.Generator(device=dev).manual_seed(3))
    frame = torch.rand(3, args.H, args.W, generator=torch.Generator().manual_seed(4)).to(dev) * 2 - 1
    T = args.T

    med, lo, hi = _time(lambda: cond(frame, T), max(args.calls, 20), args.warmup)
    l0 = ops.launches()
    cond(frame, T)
    launches = ops.launches() - l0
    with ops.profile() as prof:
        cond(frame, T)
    families = {k: dict(launches=v["launches"], ms=round(v["ms"], 3)) for k, v in sorted(prof.families.items())}

    def eager():
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            image = frame[None]
            cond_frames = image + 0.02 * torch.rand_like(image)
            co.encode(sd_c, ccfg, image, sdpa=True)
            vo.encode(sd_v, vcfg, cond_frames)
    e_med, e_lo, e_hi = _time(eager, max(args.calls, 20), args.warmup)
    name, power = _gpu_info()
    print(json.dumps(dict(
        metric="conditioner_ms_per_call", shape=f"1x3x{args.H}x{args.W}", num_frames=T, weights="synthetic full-size",
        ms_median=round(med, 3), ms_min=round(lo, 3), ms_max=round(hi, 3), calls=max(args.calls, 20),
        launches_per_call=launches, families=families,
        eager_fp16_autocast_ms_median=round(e_med, 3), eager_fp16_autocast_ms_min=round(e_lo, 3),
        speedup_vs_eager=round(e_med / med, 3), gpu=name, power_limit=power)))


if __name__ == "__main__":
    main()
