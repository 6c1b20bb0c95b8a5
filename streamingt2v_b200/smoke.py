"""smoke(): one small invocation of the hot path on cuda:0, checked against the oracle (test infrastructure)."""
from __future__ import annotations

import time

import torch


def run_smoke():
    if not torch.cuda.is_available():
        raise RuntimeError("smoke() needs a CUDA device (H100)")
    from oracle import streaming_svd_oracle as orc  # checker only
    from . import arch, ops, synth
    from .wrapper import B200StreamingWrapper
    dev = torch.device("cuda:0")
    cfg = arch.TINY
    T, h, w = 8, 8, 8
    t0 = time.time()
    sd_u = arch.synth_state_dict_fast(arch.unet_param_shapes(cfg), 11)
    sd_c = arch.synth_state_dict_fast(arch.controlnet_param_shapes(cfg), 12)
    x, t, c, kw = synth.make_inputs(cfg, T=T, h=h, w=w, seed=5)
    model = B200StreamingWrapper(cfg, sd_u, sd_c, dev)
    l0 = ops.launches()
    out = model(x.to(dev), t.to(dev), {k: v.to(dev) for k, v in c.items()},
                **{k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in kw.items()})
    torch.cuda.synchronize()
    n_launch = ops.launches() - l0
    with torch.no_grad():
        ref = orc.streaming_wrapper_forward(sd_u, sd_c, cfg, x, t, c, **kw)
    out = out.float().cpu()
    rel = ((out - ref).norm() / ref.norm()).item()
    print(f"[smoke] StreamingWrapper.forward on cuda:0: {n_launch} kernel launches, out {tuple(out.shape)}, "
          f"rel_l2 vs oracle {rel:.3e} (tolerance 3e-2), {time.time() - t0:.1f}s")
    if not (torch.isfinite(out).all() and rel < 3e-2):
        raise AssertionError(f"smoke parity failed: rel_l2={rel}")
