"""Drop-in for the reference's denoiser seam.

`B200StreamingWrapper.forward(x, t, c, **kwargs)` has the exact signature, argument meaning and return value of
`StreamingWrapper.forward` (reference code/models/diffusion/wrappers.py:23-78) — the single callable that
`Denoiser.forward` invokes per sampler step (denoiser.py:37) and that `StreamingSVD.on_inference_epoch_start`
constructs (streaming_svd.py:50-56).  Install point: `trainer.inference_model = B200StreamingWrapper.from_reference(
trainer.model.diffusion_model, trainer.controlnet)` (see INTEGRATION.md).
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn as nn

from .arch import UNetConfig
from .model import B200Denoiser


class B200StreamingWrapper(nn.Module):
    def __init__(self, cfg: UNetConfig, sd_unet: Dict[str, torch.Tensor], sd_ctrl: Optional[Dict[str, torch.Tensor]],
                 device="cuda:0"):
        super().__init__()
        if not torch.cuda.is_available():
            raise RuntimeError("B200StreamingWrapper needs a CUDA device (sm_90a); there is no CPU fallback")
        self.cfg = cfg
        self.num_frame_conditioning = cfg.num_frame_conditioning
        self.engine = B200Denoiser(cfg, sd_unet, sd_ctrl, device)

    @classmethod
    def from_reference(cls, diffusion_model: nn.Module, controlnet: Optional[nn.Module], device="cuda:0",
                       num_frame_conditioning: int = 7):
        """Build from the reference's own instantiated modules (VideoUNet, ControlNet): reads their constructor
        attributes for the config and their state_dict() (SGM key names) for the weights."""
        cfg = UNetConfig(
            in_channels=diffusion_model.in_channels, model_channels=diffusion_model.model_channels,
            out_channels=diffusion_model.out_channels, num_res_blocks=diffusion_model.num_res_blocks,
            attention_resolutions=tuple(diffusion_model.attention_resolutions),
            channel_mult=tuple(diffusion_model.channel_mult), num_head_channels=diffusion_model.num_head_channels,
            context_dim=diffusion_model.context_dim, adm_in_channels=diffusion_model.adm_in_channels,
            use_apm=any(k.endswith("apm_alpha") for k in diffusion_model.state_dict()),
            num_frame_conditioning=num_frame_conditioning)
        sd_c = controlnet.state_dict() if controlnet is not None else None
        if sd_c is not None:
            e = "controlnet_cond_embedding"
            n_pairs = sum(1 for k in sd_c if k.startswith(e + ".blocks.") and k.endswith(".weight")) // 2
            chans = [sd_c[f"{e}.conv_in.weight"].shape[0]] + [sd_c[f"{e}.blocks.{2 * i + 1}.weight"].shape[0]
                                                               for i in range(n_pairs)]
            import dataclasses
            cfg = dataclasses.replace(cfg, cond_embed_channels=tuple(chans))
        return cls(cfg, diffusion_model.state_dict(), sd_c, device)

    @classmethod
    def from_diffusers_svd(cls, unet: nn.Module, device="cuda:0", cfg: Optional[UNetConfig] = None):
        """Build the plain SVD denoiser of the FIRST chunk from diffusers' `UNetSpatioTemporalConditionModel`
        (`svd_pipeline.unet`, streaming_svd.py:62,390): its state dict is renamed to the SGM grammar
        (arch.sgm_to_diffusers_svd_keys) and runs on the same kernels, without ControlNet / CAM.  Calls then pass
        `ctrl_frames=None`."""
        from . import arch
        cfg = cfg or UNetConfig()
        return cls(cfg, arch.from_diffusers_svd_state_dict(unet.state_dict(), cfg), None, device)

    def forward(self, x: torch.Tensor, t: torch.Tensor, c: dict, **kwargs):
        batch_size = kwargs.pop("batch_size")
        num_video_frames = kwargs.pop("num_video_frames")
        image_only_indicator = kwargs.pop("image_only_indicator", None)
        if image_only_indicator is not None and bool(torch.as_tensor(image_only_indicator).any()):
            raise NotImplementedError("image_only_indicator != 0 is not on the StreamingSVD path (streaming_svd.py:208)")
        ctrl_frames = kwargs.pop("ctrl_frames", None)
        kwargs.pop("num_conditional_frames", None)  # accepted and ignored, exactly like the reference
        out = self.engine.forward(x, t, c, batch_size=batch_size, num_video_frames=num_video_frames,
                                  ctrl_frames=ctrl_frames)
        return out.to(x.dtype) if out.dtype != x.dtype else out

    # memory-optimisation hooks of the reference CLI (inference_i2v.py:143-154): chunking is meaningless here
    def enable_forward_chunking(self, *_, **__):
        return None

    def disable_forward_chunking(self, *_, **__):
        return None

    def set_chunk_feed_forward(self, *_, **__):
        return None
