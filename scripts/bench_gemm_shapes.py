#!/usr/bin/env python
"""The heaviest GEMM launches of one denoise step (2 x 25 frames, latent 72 x 128), standalone, on both schedules.

    python scripts/bench_gemm_shapes.py [--out FILE] [--no-phases]

For each shape, schedule (0 = cooperative, 2 = the default rule) and epilogue body (0 = generic, 1 = the compile-time
kind, ops.gemm_epilogue): warm-up, CUDA events over enough launches for
at least 0.2 s, achieved TFLOP/s and GB/s from the shape (the formulas of ops.gemm_raw), and the bound that applies
against the H100 SXM data sheet (989 TFLOP/s dense bf16, 3.35 TB/s) -- data-sheet figures, not reached ones.  The
card's name and power limit are read in the same run.

Unless --no-phases: mtgemm.cu is also built with -DMTGEMM_PHASE_CLOCKS into a second library in a temporary directory
(never loaded by the package), in which the A/B producer thread and the leader of each consumer warpgroup add up
clock64() differences per phase; one launch per shape and schedule is run through it and the phases are printed as
shares of the thread's lifetime, averaged over the CTAs.  Needs an sm_90 GPU.
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_TFLOPS, PEAK_GBS = 989.0, 3350.0
PHASES = ["ring wait", "mma", "res wait", "store wait", "epilogue", "other"]
FRAMES = 50


def shapes():
    """(name, kind, rows or image dims, K, N) of one launch each; how often a step runs it is not modelled."""
    out = []
    for (h, w), c in (((72, 128), 320), ((36, 64), 640), ((18, 32), 1280)):
        m = FRAMES * h * w
        out += [(f"geglu {h}x{w} K{c}", "geglu", m, c, 8 * c),
                (f"qkv {h}x{w} K{c}", "linear", m, c, 3 * c),
                (f"residual linear {h}x{w} K{c}", "linear_res", m, c, c),
                (f"fvec + res1 linear {h}x{w} K{c}", "linear_res_fvec", m, c, c),
                (f"ff-out 2 residuals, s_acc {h}x{w} K{4 * c}", "linear_res2", m, 4 * c, c),
                (f"conv3x3 + fvec {h}x{w} C{c}", "conv3x3_fvec", (FRAMES, h, w), c, c),
                (f"ff-out {h}x{w} K{4 * c}", "linear_res", m, 4 * c, c),
                (f"conv3x3 {h}x{w} C{c}", "conv3x3", (FRAMES, h, w), c, c),
                (f"tconv(3,1,1) {h}x{w} C{c}", "tconv3", (2, 25, h * w), c, c)]
    out.append(("conv3x3 9x16 C1280", "conv3x3", (FRAMES, 9, 16), 1280, 1280))
    return out


def build_phase_lib(tmp):
    from streamingt2v_b200 import build
    objs = []
    for src in sorted(build.CSRC.glob("*.cu")):
        o = os.path.join(tmp, src.stem + ".o")
        extra = ["-DMTGEMM_PHASE_CLOCKS"] if src.stem == "mtgemm" else []
        subprocess.check_call([build._nvcc(), *build.NVCC_FLAGS, *extra, "-c", str(src), "-o", o])
        objs.append(o)
    lib = os.path.join(tmp, "libb200svd_phase.so")
    subprocess.check_call([build._nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", lib, *objs])
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-phases", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm_shapes.py measures on the GPU: no CUDA device")
    from streamingt2v_b200 import _lib, ops, packing
    dev = torch.device("cuda:0")
    _lib.init(0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    lines = [f"card: {card}"]
    g = torch.Generator().manual_seed(0)

    def rnd(shape, scale=1.0, dtype=torch.bfloat16):
        return (torch.randn(shape, generator=g) * scale).to(dev, dtype)

    cases = []
    for name, kind, m, k, n in shapes():
        bias = rnd((n,), 0.1, torch.float32)
        if kind == "geglu":
            x = rnd((m, k))
            w = torch.randn((n, k), generator=g) * k ** -0.5
            packs = {0: packing.pack_geglu(w, bias.cpu(), dev), 2: packing.pack_geglu(w, bias.cpu(), dev, bn=128)}
            run = lambda s, x=x, packs=packs: ops.linear(x, packs[s][0], packs[s][1], act=ops.ACT_GEGLU, bn=packs[s][2])
            rows, taps, n_out, nres = m, 1, n // 2, 0
        elif kind.startswith("linear"):
            x = rnd((m, k))
            w = packing.pack_linear(torch.randn((n, k), generator=g) * k ** -0.5, dev)
            kw = {}
            if kind != "linear":
                kw.update(res1=rnd((m, n)))
            if kind == "linear_res2":
                kw.update(res2=rnd((m, n)), s2=0.5, s_acc=0.7)
            if kind == "linear_res_fvec":
                kw.update(fvec=rnd((FRAMES, n), 1.0, torch.float32), rows_per_frame=m // FRAMES)
            run = lambda s, x=x, w=w, bias=bias, kw=kw: ops.linear(x, w, bias, **kw)
            rows, taps, n_out, nres = m, 1, n, ("res1" in kw) + ("res2" in kw)
        elif kind in ("conv3x3", "conv3x3_fvec"):
            x = rnd((*m, k))
            w = packing.pack_conv3x3(torch.randn((n, k, 3, 3), generator=g) * (9 * k) ** -0.5, dev)
            kw = {}
            if kind == "conv3x3_fvec":
                kw.update(fvec=rnd((m[0], n), 1.0, torch.float32), rows_per_frame=m[1] * m[2])
            run = lambda s, x=x, w=w, bias=bias, kw=kw: ops.conv3x3(x, w, bias, **kw)
            rows, taps, n_out, nres = m[0] * m[1] * m[2], 9, n, 0
        else:
            x = rnd((*m, k))
            w = packing.pack_tconv3(torch.randn((n, k, 3, 1, 1), generator=g) * (3 * k) ** -0.5, dev)
            res = rnd((m[0] * m[1] * m[2], n))
            run = lambda s, x=x, w=w, bias=bias, res=res: ops.tconv3(x, w, bias, res1=res)
            rows, taps, n_out, nres = m[0] * m[1] * m[2], 3, n, 1
        flops = 2.0 * rows * k * n * taps
        nbytes = 2.0 * rows * k + 2.0 * taps * n * k + 2.0 * rows * n_out * (1 + nres)
        cases.append((name, run, flops, nbytes))

    prev, prev_epi = ops.gemm_schedule(-1), ops.gemm_epilogue(-1)
    lines.append(f"{'shape':44s} {'sched':5s} {'epi':3s} {'ms':>8s} {'TFLOP/s':>8s} {'GB/s':>7s}  bound (data sheet)      share")
    for name, run, flops, nbytes in cases:
        for sched, epi in ((0, 0), (0, 1), (2, 0), (2, 1)):
            ops.gemm_schedule(sched)
            ops.gemm_epilogue(epi)
            for _ in range(3):
                run(sched)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps, ms = 4, 0.0
            while ms < 200.0:
                reps *= 2
                e0.record()
                for _ in range(reps):
                    run(sched)
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1)
            t = ms / reps
            t_ops, t_bytes = flops / PEAK_TFLOPS / 1e9, nbytes / PEAK_GBS / 1e6
            bound = "operations" if t_ops >= t_bytes else "bytes"
            lines.append(f"{name:44s} {sched:5d} {epi:3d} {t:8.3f} {flops / t / 1e9:8.1f} {nbytes / t / 1e6:7.0f}  "
                         f"{bound:10s} {max(t_ops, t_bytes):7.3f} ms  {max(t_ops, t_bytes) / t:5.1%}")
    ops.gemm_schedule(prev)
    ops.gemm_epilogue(prev_epi)

    if not args.no_phases:
        with tempfile.TemporaryDirectory() as tmp:
            os.environ["B200SVD_LIB"] = build_phase_lib(tmp)
            _lib._LIB = None
            _lib._inited.clear()
            lib = _lib.load()
            _lib.init(0)
            sms = torch.cuda.get_device_properties(0).multi_processor_count
            buf = torch.zeros((sms, 3, 8), dtype=torch.int64, device=dev)
            lib.b200svd_gemm_phase_buffer.argtypes = [C.c_void_p]
            lib.b200svd_gemm_phase_buffer(C.c_void_p(buf.data_ptr()))
            lines.append("")
            lines.append("phase shares of the thread's lifetime (clock64, one launch, mean over CTAs)")
            lines.append(f"{'shape':44s} {'sched':5s} {'epi':3s} role      " + " ".join(f"{p:>10s}" for p in PHASES))
            for name, run, _, _ in cases:
                for sched, epi in ((0, 0), (0, 1), (2, 0), (2, 1)):
                    ops.gemm_schedule(sched)
                    ops.gemm_epilogue(epi)
                    run(sched)
                    torch.cuda.synchronize()
                    buf.zero_()
                    run(sched)
                    torch.cuda.synchronize()
                    b = buf.double().cpu()
                    for role, rname in ((0, "producer"), (1, "consumer0"), (2, "consumer1")):
                        tot = b[:, role, 7].sum().item()
                        if tot == 0:
                            continue
                        sh = [b[:, role, i].sum().item() / tot for i in range(6)]
                        lines.append(f"{name:44s} {sched:5d} {epi:3d} {rname:9s} " + " ".join(f"{v:10.1%}" for v in sh))
            lib.b200svd_gemm_phase_buffer(C.c_void_p(0))
            ops.gemm_schedule(prev)
            ops.gemm_epilogue(prev_epi)
    text = "\n".join(lines)
    print(text)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
