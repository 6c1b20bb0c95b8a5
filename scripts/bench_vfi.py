"""Benchmark of the EMA-VFI interpolation stage (B200VFI, streamingt2v_b200/vfi.py) at the reference's 720x1280 frames,
with the shipped configuration and seeded synthetic weights (vfi.seeded_state_dict).

Prints one JSON line: the median ms of one fast-TTA pair (`B200VFI.inference`) over >= 10 warmed calls (CUDA events),
the time of one 100 -> 200-frame `interpolate_video` (99 pairs, device-resident uint8 frames), the per-family split of
one pair from ops.profile() with its FLOP count computed from the launch shapes, and the GPU name and power limit
(read-only nvidia-smi query).  Needs a CUDA device; writes nothing.
    python scripts/bench_vfi.py [--calls 10] [--warmup 3] [--frames 100]"""
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
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return name, power, clock
    except Exception as e:  # noqa: BLE001
        return torch.cuda.get_device_name(0), f"unknown ({e.__class__.__name__})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--H", type=int, default=720)
    ap.add_argument("--W", type=int, default=1280)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vfi.py needs a CUDA device (H100)")
    from streamingt2v_b200 import _lib, ops
    from streamingt2v_b200.vfi import B200VFI, interpolate_video, seeded_state_dict
    _lib.init(0)
    dev = torch.device("cuda:0")
    net = B200VFI(seeded_state_dict(0), dev)
    g = torch.Generator(device="cpu").manual_seed(0)
    img0 = torch.rand((1, 3, args.H, args.W), generator=g).to(dev)
    img1 = torch.roll(img0, shifts=(4, -6), dims=(2, 3))

    for _ in range(args.warmup):
        net.inference(img0, img1)
    torch.cuda.synchronize()
    ms = []
    for _ in range(args.calls):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        net.inference(img0, img1)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    with ops.profile() as prof:
        net.inference(img0, img1)
    fams = {k: dict(launches=v["launches"], ms=round(v["ms"], 3), gflop=round(v["flops"] / 1e9, 2))
            for k, v in sorted(prof.families.items(), key=lambda kv: -kv[1]["ms"])}
    flops = sum(v["flops"] for v in prof.families.values())

    video = (torch.rand((args.frames, args.H, args.W, 3), generator=g) * 255).to(torch.uint8).to(dev)
    dest = 2 * args.frames
    interpolate_video(video[:2], 2, net)                                      # warm the frame-conversion path
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = interpolate_video(video, dest, net)
    e1.record()
    torch.cuda.synchronize()
    name, power, clock = _gpu_info()
    print(json.dumps(dict(
        workload=f"EMA-VFI fast-TTA pair {args.H}x{args.W}", gpu=name, power_limit=power, max_sm_clock=clock,
        pair_ms_median=round(statistics.median(ms), 3), pair_ms_min=round(min(ms), 3), pair_ms_max=round(max(ms), 3),
        pair_gflop=round(flops / 1e9, 1), pair_tflops=round(flops / statistics.median(ms) / 1e9, 1),
        video_frames_in=args.frames, video_frames_out=int(out.shape[0]),
        video_ms=round(e0.elapsed_time(e1), 1), families=fams)))


if __name__ == "__main__":
    main()
