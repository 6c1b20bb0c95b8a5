"""The first chunk of an image-to-video request on the project's kernels: drop-in for
`svd_pipeline(image, decode_chunk_size=8).frames[0]` followed by `ToTensor()` and `* 2.0 - 1`
(code/diffusion_trainer/streaming_svd.py:388-393), i.e. diffusers' `StableVideoDiffusionPipeline.__call__` with the
SVD-XT checkpoint, restated from diffusers 0.30.2's published source (diffusers is not a dependency: parity unpinned).

Every network is one the later chunks already run: the plain SVD UNet (`B200StreamingWrapper.from_diffusers_svd`), the
conditioner (`B200SVDConditioner.from_diffusers_svd`: CLIP tower + VAE encoder), the Karras Euler sampler and the
temporal VAE decoder.  The pipeline's 8-bit PIL round trip is one kernel (`ops.frames_quantize`)."""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from . import dist_utils, ops
from .arch import UNetConfig
from .sampler import B200EulerEDMSampler

SPATIAL_COMPRESSION = 8


def unet_config_from_diffusers_svd(config) -> UNetConfig:
    """UNetConfig of a `UNetSpatioTemporalConditionModel.config`.  SVD's down blocks are three
    CrossAttnDownBlockSpatioTemporal and one DownBlockSpatioTemporal (attention at downsample factors 1, 2, 4) with
    64-channel heads; other layouts are rejected rather than run with the wrong plan."""
    boc = tuple(config.block_out_channels)
    heads = tuple(config.num_attention_heads) if not isinstance(config.num_attention_heads, int) else \
        (config.num_attention_heads,) * len(boc)
    n = len(boc)
    if tuple(config.down_block_types) != ("CrossAttnDownBlockSpatioTemporal",) * (n - 1) + ("DownBlockSpatioTemporal",):
        raise ValueError(f"unsupported down_block_types {config.down_block_types}")
    if any(c != 64 * h for c, h in zip(boc, heads)):
        raise ValueError(f"the kernels expect 64-channel heads: block_out_channels {boc}, heads {heads}")
    return UNetConfig(in_channels=int(config.in_channels), model_channels=boc[0], out_channels=int(config.out_channels),
                      num_res_blocks=int(config.layers_per_block),
                      attention_resolutions=tuple(2 ** i for i in range(n - 1))[::-1],
                      channel_mult=tuple(c // boc[0] for c in boc), num_head_channels=64,
                      context_dim=int(config.cross_attention_dim),
                      adm_in_channels=int(config.projection_class_embeddings_input_dim))


def image_to_unit_tensor(image, device) -> torch.Tensor:
    """[3, H, W] float tensor in [0, 1], or uint8 [H, W, 3] array / tensor -> fp32 [3, H, W] in [0, 1] on `device`.
    uint8 is divided by 255 in fp32, as diffusers' `pil_to_numpy` does."""
    if isinstance(image, np.ndarray):
        image = torch.from_numpy(np.array(image))                  # a copy: the array may be read-only
    if image.dtype == torch.uint8:
        if image.dim() != 3 or image.shape[-1] != 3:
            raise ValueError(f"uint8 images are [H, W, 3], got {tuple(image.shape)}")
        return image.to(device).permute(2, 0, 1).float().div(255.0).contiguous()
    if image.dim() != 3 or image.shape[0] != 3:
        raise ValueError(f"float images are [3, H, W] in [0, 1], got {tuple(image.shape)}")
    return image.to(device, torch.float32).contiguous()


class B200SVDImageToVideo:
    """`first_chunk(image, ...) -> [num_frames, 3, H, W]` fp32 on the device, in [-1, 1] on the 1/127.5 grid: the
    tensor the reference holds after streaming_svd.py:393."""

    def __init__(self, unet, conditioner, vae_decoder, *, sigma_min: float = 0.002, sigma_max: float = 700.0,
                 scale_factor: float = 0.18215, device="cuda:0"):
        self.unet = unet                        # B200StreamingWrapper of the plain SVD UNet (no ControlNet)
        self.conditioner = conditioner          # B200SVDConditioner(noise="gaussian")
        self.vae_decoder = vae_decoder          # B200VaeDecoder
        self.sigma_min, self.sigma_max = float(sigma_min), float(sigma_max)
        self.scale_factor = float(scale_factor)
        self.device = torch.device(device)

    @classmethod
    def from_diffusers(cls, pipeline, device="cuda:0"):
        """Build from a `StableVideoDiffusionPipeline`, or any object exposing `unet`, `vae`, `image_encoder` (modules
        with `config` and `state_dict()`) and `scheduler.config`.  The scheduler must be SVD's EulerDiscreteScheduler:
        Karras sigmas, v-prediction, continuous timesteps."""
        from .arch import from_diffusers_svd_vae_state_dict
        from .conditioner import B200SVDConditioner, vae_config_from_diffusers
        from .vae import B200VaeDecoder
        from .wrapper import B200StreamingWrapper
        sc = pipeline.scheduler.config
        if not (getattr(sc, "use_karras_sigmas", False) and getattr(sc, "prediction_type", None) == "v_prediction"
                and getattr(sc, "timestep_type", None) == "continuous"):
            raise ValueError("the first chunk needs SVD's scheduler: Karras sigmas, v-prediction, continuous timesteps")
        unet = B200StreamingWrapper.from_diffusers_svd(pipeline.unet, device,
                                                       unet_config_from_diffusers_svd(pipeline.unet.config))
        cond = B200SVDConditioner.from_diffusers_svd(pipeline, device)
        vcfg = vae_config_from_diffusers(pipeline.vae.config)
        _, sd_d = from_diffusers_svd_vae_state_dict(pipeline.vae.state_dict(), vcfg)
        dec = B200VaeDecoder(vcfg, sd_d, device)
        return cls(unet, cond, dec, sigma_min=sc.sigma_min, sigma_max=sc.sigma_max,
                   scale_factor=pipeline.vae.config.scaling_factor, device=device)

    def _randn(self, shape, generator: Optional[torch.Generator]) -> torch.Tensor:
        """diffusers' randn_tensor: drawn on the generator's device (the execution device without one)."""
        dev = generator.device if generator is not None else self.device
        x = torch.randn(shape, generator=generator, device=dev).to(self.device, torch.float32)
        return dist_utils.broadcast_from_rank0(x)

    @torch.no_grad()
    def __call__(self, image, *, num_frames: int = 25, num_inference_steps: int = 25, min_guidance_scale: float = 1.0,
                 max_guidance_scale: float = 3.0, fps: int = 7, motion_bucket_id: int = 127,
                 noise_aug_strength: float = 0.02, decode_chunk_size: int = 8,
                 generator: Optional[torch.Generator] = None) -> torch.Tensor:
        z = self.sample(image, num_frames=num_frames, num_inference_steps=num_inference_steps,
                        min_guidance_scale=min_guidance_scale, max_guidance_scale=max_guidance_scale, fps=fps,
                        motion_bucket_id=motion_bucket_id, noise_aug_strength=noise_aug_strength, generator=generator)
        # decode_latents, then postprocess_video(output_type="pil") -> ToTensor() -> * 2.0 - 1
        return ops.frames_quantize(self.decode(z, decode_chunk_size))

    @torch.no_grad()
    def sample(self, image, *, num_frames: int, num_inference_steps: int, min_guidance_scale: float,
               max_guidance_scale: float, fps: int, motion_bucket_id: int, noise_aug_strength: float,
               generator: Optional[torch.Generator]) -> torch.Tensor:
        """The pipeline up to the denoised latents [num_frames, 4, H/8, W/8] (output_type="latent")."""
        T = int(num_frames)
        img = image_to_unit_tensor(image, self.device)
        H, W = img.shape[-2:]
        # conditioning (draws the image noise first), then the initial latents
        c, uc = self.conditioner.condition(img * 2.0 - 1.0, T, fps_id=fps - 1, motion_bucket_id=motion_bucket_id,
                                           cond_aug=noise_aug_strength, generator=generator)
        c, uc = dict(c), dict(uc)
        for k in ("crossattn", "concat"):                 # the UNet repeats the image embedding / latent per frame
            c[k] = c[k].repeat_interleave(T, dim=0)
            uc[k] = uc[k].repeat_interleave(T, dim=0)
        randn = self._randn((T, 4, H // SPATIAL_COMPRESSION, W // SPATIAL_COMPRESSION), generator)
        # EulerDiscreteScheduler (Karras, v-prediction) with the per-frame linear guidance of the pipeline
        sampler = B200EulerEDMSampler(num_steps=num_inference_steps, num_frames=T, min_scale=min_guidance_scale,
                                      max_scale=max_guidance_scale, schedule="karras", sigma_min=self.sigma_min,
                                      sigma_max=self.sigma_max)
        return sampler(self.unet, randn, c, uc, image_only_indicator=torch.zeros(2, T, device=self.device),
                       num_video_frames=T, batch_size=2)

    def decode(self, z: torch.Tensor, decode_chunk_size: int = 8) -> torch.Tensor:
        """decode_latents: z / scaling_factor decoded in groups of `decode_chunk_size` frames, each group its own
        temporal window.  Returns the frames before the 8-bit round trip, fp32 [F, 3, H, W]."""
        z = 1.0 / self.scale_factor * z
        outs = []
        for i in range(0, z.shape[0], int(decode_chunk_size)):
            part = z[i:i + int(decode_chunk_size)]
            outs.append(self.vae_decoder.decode(part, timesteps=len(part)))
        return torch.cat(outs, dim=0)
