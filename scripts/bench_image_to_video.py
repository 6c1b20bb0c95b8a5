"""Benchmark of image -> video on the kernels, at the reference's request shape: one 576x1024 image, full-size
synthetic weights (plain SVD UNet + StreamingSVD UNet with ControlNet, ViT-H/14 CLIP tower, SD-VAE encoder, temporal
VAE decoder).

  * first chunk (B200SVDImageToVideo, 25 frames, 25 Karras steps, decode groups of 8) split into conditioning,
    sampling, decode and the 8-bit round trip, each timed with CUDA events around its own stage;
  * a 100-frame StreamingSVD video from the image: B200StreamingSVDStage.image_to_video with the first chunk plus 5
    autoregressive chunks (25 frames, 30 AlignYourSteps steps, 7 conditioning frames each), frames/s;
  * the card's name, power limit and max SM clock, read (read-only nvidia-smi query) in the same process.
Prints one JSON line.  Needs a CUDA device; writes nothing.    python scripts/bench_image_to_video.py [--runs 3]"""
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


class _Timer:
    def __init__(self):
        self.ms = {}

    def __call__(self, name, fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        self.ms.setdefault(name, []).append(e0.elapsed_time(e1))
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=25, help="first-chunk sampler steps")
    ap.add_argument("--stage-steps", type=int, default=30, help="sampler steps of the autoregressive chunks")
    ap.add_argument("--chunks", type=int, default=5, help="autoregressive chunks after the first")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_image_to_video.py needs a CUDA device (H100)")
    from streamingt2v_b200 import _lib, arch, ops
    from streamingt2v_b200.conditioner import B200ClipImageEncoder, B200SVDConditioner
    from streamingt2v_b200.first_chunk import B200SVDImageToVideo
    from streamingt2v_b200.sampler import B200EulerEDMSampler
    from streamingt2v_b200.stage import B200StreamingSVDStage
    from streamingt2v_b200.vae import B200VaeDecoder, B200VaeEncoder
    from streamingt2v_b200.wrapper import B200StreamingWrapper
    dev = torch.device("cuda:0")
    _lib.init(0)
    T, H, W = 25, 576, 1024
    ucfg, ccfg, vcfg = arch.UNetConfig(), arch.ClipVisionConfig(), arch.VaeConfig()
    syn = arch.synth_state_dict_device
    clip = B200ClipImageEncoder(ccfg, syn(arch.clip_visual_param_shapes(ccfg), dev, 1), dev)
    enc = B200VaeEncoder(vcfg, syn(arch.vae_encoder_param_shapes(vcfg), dev, 2), dev)
    dec = B200VaeDecoder(vcfg, syn(arch.vae_decoder_param_shapes(vcfg), dev, 3), dev)
    plain = B200StreamingWrapper(ucfg, syn(arch.plain_unet_param_shapes(ucfg), dev, 4), None, dev)
    first = B200SVDImageToVideo(plain, B200SVDConditioner(clip, enc, noise="gaussian"), dec, device=dev)
    streaming = B200StreamingWrapper(ucfg, syn(arch.unet_param_shapes(ucfg), dev, 5),
                                     syn(arch.controlnet_param_shapes(ucfg), dev, 6), dev)
    stage = B200StreamingSVDStage(streaming, B200EulerEDMSampler(num_steps=args.stage_steps, num_frames=T), dec,
                                  B200SVDConditioner(clip, enc), device=dev)
    image = np.random.default_rng(7).integers(0, 256, size=(H, W, 3), dtype=np.uint8)
    kw = dict(num_frames=T, num_inference_steps=args.steps, min_guidance_scale=1.0, max_guidance_scale=3.0, fps=7,
              motion_bucket_id=127, noise_aug_strength=0.02)

    tm = _Timer()

    def split_first_chunk(seed):
        g = torch.Generator().manual_seed(seed)
        img = tm("image_upload", lambda: torch.from_numpy(image).to(dev).permute(2, 0, 1).float().div(255.0))
        tm("conditioning", lambda: first.conditioner.condition(img * 2.0 - 1.0, T, fps_id=6, motion_bucket_id=127,
                                                               cond_aug=0.02, generator=g))
        z = tm("sampling", lambda: first.sample(img, generator=torch.Generator().manual_seed(seed), **kw))
        frames = tm("decode", lambda: first.decode(z, 8))
        tm("quantize", lambda: ops.frames_quantize(frames))

    split_first_chunk(0)                                        # warm-up: every shape of the timed window
    tm.ms.clear()
    for r in range(args.runs):
        split_first_chunk(r + 1)
    # the sampling leg above re-runs the conditioning inside sample(); report it without that share
    med = {k: statistics.median(v) for k, v in tm.ms.items()}
    med["sampling_only"] = med["sampling"] - med["conditioning"]

    def first_chunk(img, generator=None):
        return first(img, generator=generator, **kw)

    def video():
        return stage.image_to_video(image, args.chunks, first_chunk, generator=torch.Generator().manual_seed(11))

    v = video()                                                 # warm-up of the autoregressive shapes
    torch.cuda.synchronize()
    wall = []
    for _ in range(max(1, args.runs - 1)):
        t0 = time.perf_counter()
        v = video()
        torch.cuda.synchronize()
        wall.append(time.perf_counter() - t0)
    n_frames = int(v.shape[0])
    assert bool(torch.isfinite(v).all())
    name, power, clock = _gpu_info()
    print(json.dumps(dict(
        metric="image_to_video", image=f"{H}x{W}", weights="synthetic full-size", runs=args.runs,
        first_chunk_ms=dict(conditioning=round(med["conditioning"], 2),
                            sampling=round(med["sampling_only"], 2), steps=args.steps,
                            decode=round(med["decode"], 2), quantize=round(med["quantize"], 3),
                            total=round(med["sampling"] + med["decode"] + med["quantize"], 2)),
        video_frames=n_frames, video_s=round(statistics.median(wall), 3),
        video_frames_per_s=round(n_frames / statistics.median(wall), 3), autoregressive_chunks=args.chunks,
        stage_steps=args.stage_steps, gpu=name, power_limit=power, max_sm_clock=clock)))


if __name__ == "__main__":
    main()
