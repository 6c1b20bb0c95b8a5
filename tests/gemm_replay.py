"""TEST INFRASTRUCTURE — replaying a census GEMM launch against float64: the reference op, the launch, the bound, the
rerun / schedule / epilogue-body comparison.  Shared by tests/test_vfi_launches_gpu.py,
tests/test_denoiser_launches_gpu.py and tests/test_vae_clip_launches_gpu.py.

Bound.  Operands are bf16, so every product x*w is exact in fp32; the kernel sums n = K * taps of them (plus the
bias) in fp32.  Each addition rounds by at most 2^-24 relative, so the sum is within gamma_n S, gamma_n = n 2^-24 /
(1 - n 2^-24) <= n 2^-23, of the exact one, S = sum |x| |w| + |bias| (a second float64 op on |x|, |w|).  The epilogue
adds a few roundings more (`terms` extra terms of 2^-23 S, every addend's magnitude included in S); an activation
slope a scales the result by |a|.  The bf16 store rounds to nearest, 2^-8 relative (fp32 stores: 2^-23 with the
epilogue's rounding):
    |out - ref| <= 2^-8 |ref| + (K taps + terms) 2^-23 amp S        (bf16 outputs; 2^-23 |ref| for fp32)"""
import torch
import torch.nn.functional as F


def free():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def bits(t):
    return t.view({2: torch.int16, 4: torch.int32}[t.element_size()])


def ref_gemm(op, x, wt, extra=()):
    """float64 op on x ([rows, K], NHWC, or [B, T, P, C] for tconv3) with wt in torch layout -> rows [M, N]."""
    if op == "linear":
        return x @ wt.t()
    if op == "tconv3":
        # (3, 1, 1) conv over the frames of each video: frame 0 and frame T-1 see zeros, never the other video
        y = F.conv2d(x.permute(0, 3, 1, 2), wt[..., None], padding=(1, 0))       # [B, N, T, P]
        return y.permute(0, 2, 3, 1).reshape(-1, y.shape[1])
    xc = x.permute(0, 3, 1, 2)
    if op == "conv3x3":
        y = F.conv2d(xc, wt, padding=1)
    elif op == "conv3x3_s2":
        y = F.conv2d(xc, wt, stride=2, padding=1)
    elif op == "conv3x3_s2_pad_after":
        # the autoencoder's Downsample: zero pad after (bottom and right) only, then a padding-0 stride-2 conv
        y = F.conv2d(F.pad(xc, (0, 1, 0, 1)), wt, stride=2)
    elif op == "conv3x3_strided":
        s, d = extra
        y = F.conv2d(xc, wt, stride=s, padding=d, dilation=d)
    else:
        y = F.conv_transpose2d(xc, wt, stride=2, padding=1)
    return y.permute(0, 2, 3, 1).reshape(-1, y.shape[1])


def launch(op, x, w, b, out, extra, epi):
    from streamingt2v_b200 import ops
    if op == "conv3x3_strided":
        ops.conv3x3_strided(x, w, b, stride=extra[0], dilation=extra[1], out=out, **epi)
    elif op == "conv3x3_s2_pad_after":
        ops.conv3x3_s2(x, w, b, out=out, pad_after_only=True, **epi)
    else:
        getattr(ops, op)(x, w, b, out=out, **epi)


def gemm_bound(ref, s_abs, k_taps, fp32, amp=1.0, terms=4):
    return (2.0 ** -23 if fp32 else 2.0 ** -8) * ref.abs() + (k_taps + terms) * 2.0 ** -23 * amp * s_abs


def replay(run, O, name, schedules=(None,), epilogues=(None,)):
    """run() twice under every forced consumer schedule (None: the default) and epilogue body (None: the default),
    checking O's guard bands after each; every output must equal the first bitwise.  Returns the first output."""
    from streamingt2v_b200 import ops
    first = None
    for epi in epilogues:
        for sched in schedules:
            prev_s = ops.gemm_schedule(sched) if sched is not None else None
            prev_e = ops.gemm_epilogue(epi) if epi is not None else None
            try:
                for _ in range(2):
                    run()
                    torch.cuda.synchronize()
                    where = f"{name} schedule {sched} epilogue {epi}"
                    O.check(where)
                    if first is None:
                        first = O.view.clone()
                    else:
                        assert torch.equal(bits(O.view), bits(first)), f"{where}: differs bitwise from the first run"
            finally:
                if prev_s is not None:
                    ops.gemm_schedule(prev_s)
                if prev_e is not None:
                    ops.gemm_epilogue(prev_e)
    return first
