"""Benchmark of a whole image-to-video request (pipeline.B200StreamingPipeline) and of its PIL-exact resize kernel.

  * resize: 100 frames 1024x576 -> 1280x720 (every first-stage frame before enhance), ops.resize_bicubic_u8 (median
    of --calls warmed calls, CUDA events) against Pillow's Image.resize frame by frame on one host core, as the
    reference runs it (inference_i2v.py:197-199); the two outputs are compared byte for byte;
  * request: one request of --num-frames frames from a 576x1024 image with full-size synthetic weights (plain SVD UNet,
    StreamingSVD UNet with ControlNet, ViT-H/14 CLIP tower, SD-VAE encoder, temporal VAE decoder, seeded EMA-VFI) and
    an identity enhance, timed per stage (image_to_video, enhance_video = the two resizes + the identity,
    interpolate_video) after a warm-up request that has one autoregressive chunk;
  * the card's name, power limit and max SM clock (read-only nvidia-smi query) in the same process.
Prints one JSON line.  Needs a CUDA device; writes nothing.
    python scripts/bench_request.py [--num-frames 200] [--resize-only]"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return name, power, clock
    except Exception as e:  # noqa: BLE001
        return torch.cuda.get_device_name(0), f"unknown ({e.__class__.__name__})", "unknown"


def bench_resize(dev, calls):
    from PIL import Image

    from streamingt2v_b200 import ops
    frames = np.random.default_rng(0).integers(0, 256, size=(100, 576, 1024, 3), dtype=np.uint8)
    x = torch.from_numpy(frames).to(dev)
    for _ in range(3):
        ops.resize_bicubic_u8(x, 1280, 720)
    torch.cuda.synchronize()
    ms = []
    for _ in range(calls):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = ops.resize_bicubic_u8(x, 1280, 720)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    t0 = time.perf_counter()
    pil = np.stack([np.asarray(Image.fromarray(f).resize((1280, 720))) for f in frames])
    pil_ms = (time.perf_counter() - t0) * 1e3
    moved = frames.nbytes + 100 * 576 * 1280 * 3 * 2 + out.numel()     # input, intermediate written + read, output
    med = statistics.median(ms)
    return dict(frames=100, size="1024x576->1280x720", kernel_ms_median=round(med, 3), kernel_ms_min=round(min(ms), 3),
                kernel_ms_max=round(max(ms), 3), kernel_gb_per_s=round(moved / med / 1e6, 1),
                pil_host_ms=round(pil_ms, 1), host_cores=os.cpu_count(),
                bit_exact=bool(np.array_equal(out.cpu().numpy(), pil)))


def build_pipeline(dev, steps, stage_steps):
    from streamingt2v_b200 import arch
    from streamingt2v_b200.conditioner import B200ClipImageEncoder, B200SVDConditioner
    from streamingt2v_b200.first_chunk import B200SVDImageToVideo
    from streamingt2v_b200.pipeline import B200StreamingPipeline
    from streamingt2v_b200.sampler import B200EulerEDMSampler
    from streamingt2v_b200.stage import B200StreamingSVDStage
    from streamingt2v_b200.vae import B200VaeDecoder, B200VaeEncoder
    from streamingt2v_b200.vfi import B200VFI, seeded_state_dict
    from streamingt2v_b200.wrapper import B200StreamingWrapper
    T = 25
    ucfg, ccfg, vcfg = arch.UNetConfig(), arch.ClipVisionConfig(), arch.VaeConfig()
    syn = arch.synth_state_dict_device
    clip = B200ClipImageEncoder(ccfg, syn(arch.clip_visual_param_shapes(ccfg), dev, 1), dev)
    enc = B200VaeEncoder(vcfg, syn(arch.vae_encoder_param_shapes(vcfg), dev, 2), dev)
    dec = B200VaeDecoder(vcfg, syn(arch.vae_decoder_param_shapes(vcfg), dev, 3), dev)
    plain = B200StreamingWrapper(ucfg, syn(arch.plain_unet_param_shapes(ucfg), dev, 4), None, dev)
    first = B200SVDImageToVideo(plain, B200SVDConditioner(clip, enc, noise="gaussian"), dec, device=dev)
    streaming = B200StreamingWrapper(ucfg, syn(arch.unet_param_shapes(ucfg), dev, 5),
                                     syn(arch.controlnet_param_shapes(ucfg), dev, 6), dev)
    stage = B200StreamingSVDStage(streaming, B200EulerEDMSampler(num_steps=stage_steps, num_frames=T), dec,
                                  B200SVDConditioner(clip, enc), device=dev)

    def first_chunk(img, generator=None):
        return first(img, num_frames=T, num_inference_steps=steps, generator=generator)

    def identity_enhance(image, video, **_):
        return video

    return B200StreamingPipeline(stage, first_chunk, B200VFI(seeded_state_dict(0), dev), identity_enhance)


def bench_request(dev, num_frames, steps, stage_steps):
    pipe = build_pipeline(dev, steps, stage_steps)
    image = np.random.default_rng(7).integers(0, 256, size=(576, 1024, 3), dtype=np.uint8)

    def request(n, seed):
        """pipe(image, n) stage by stage, each stage timed up to a device synchronise."""
        ms = {}

        def timed(name, fn):
            t0 = time.perf_counter()
            out = fn()
            torch.cuda.synchronize()
            ms[name] = (time.perf_counter() - t0) * 1e3
            return out

        g = torch.Generator().manual_seed(seed)
        video = timed("image_to_video", lambda: pipe.image_to_video(image, (n + 1) // 2, generator=g))
        enh = timed("enhance_video", lambda: pipe.enhance_video(image, video, chunk_size=(n + 1) // 2, overlap_size=0))
        out = timed("interpolate_video", lambda: pipe.interpolate_video(enh, n))
        return out, ms

    request(2 * (25 + 1), 0)                     # warm-up: first chunk, one autoregressive chunk, resizes, VFI
    out, ms = request(num_frames, 1)
    total = sum(ms.values())
    return dict(num_frames=num_frames, frames_out=int(out.shape[0]), first_chunk_steps=steps, stage_steps=stage_steps,
                stage_ms={k: round(v, 1) for k, v in ms.items()}, total_s=round(total / 1e3, 2),
                frames_per_s=round(int(out.shape[0]) / (total / 1e3), 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20, help="timed resize calls")
    ap.add_argument("--num-frames", type=int, default=200, help="frames of the request (the reference's default)")
    ap.add_argument("--steps", type=int, default=25, help="first-chunk sampler steps")
    ap.add_argument("--stage-steps", type=int, default=30, help="sampler steps of the autoregressive chunks")
    ap.add_argument("--resize-only", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_request.py needs a CUDA device (H100)")
    from streamingt2v_b200 import _lib
    _lib.init(0)
    dev = torch.device("cuda:0")
    res = dict(metric="request", resize=bench_resize(dev, args.calls))
    if not args.resize_only:
        res["request"] = bench_request(dev, args.num_frames, args.steps, args.stage_steps)
    name, power, clock = _gpu_info()
    res.update(gpu=name, power_limit=power, max_sm_clock=clock, weights="synthetic full-size", enhance="identity")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
