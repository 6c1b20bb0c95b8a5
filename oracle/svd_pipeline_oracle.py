"""ORACLE — test infrastructure only.  fp32 PyTorch restatement of diffusers' `StableVideoDiffusionPipeline.__call__`
(the first chunk of an image-to-video request, code/diffusion_trainer/streaming_svd.py:388-393), built from parts that
are pinned elsewhere:
  * the plain SVD UNet: streaming_svd_oracle.unet_forward without ControlNet (pinned against the reference's own
    VideoUNet by oracle/make_golden.py);
  * the VAE encoder / temporal decoder: vae_encoder_oracle / vae_decoder_oracle (pinned against the reference's
    Encoder and VideoDecoder);
  * the CLIP tower: clip_image_oracle (pinned against transformers' CLIPVisionModelWithProjection);
  * the flow between them — noise order, conditioning, Karras Euler loop, decode groups, 8-bit round trip — restated
    from diffusers 0.30.2's published source.  diffusers is not installed: that part is unpinned.
It takes SGM / open_clip named state dicts (the arch maps rename the diffusers / transformers ones) and runs on any
device the inputs live on."""
from __future__ import annotations

import numpy as np
import torch

from oracle import clip_image_oracle as co
from oracle import sampler_oracle as so
from oracle import streaming_svd_oracle as uo
from oracle import vae_decoder_oracle as vdo
from oracle import vae_encoder_oracle as veo


def karras_sigmas(n: int, sigma_min: float = 0.002, sigma_max: float = 700.0, rho: float = 7.0) -> np.ndarray:
    """EulerDiscreteScheduler._convert_to_karras, then the appended 0."""
    ramp = np.linspace(0, 1, n)
    lo, hi = sigma_min ** (1 / rho), sigma_max ** (1 / rho)
    return np.concatenate([(hi + ramp * (lo - hi)) ** rho, [0.0]])


def conditioning(sd_clip, clip_cfg, sd_enc, vae_cfg, image01, noise, T, *, fps=7, motion_bucket_id=127,
                 noise_aug_strength=0.02):
    """_encode_image, the noised VAE encode, _get_add_time_ids.  image01 [3, H, W] in [0, 1]; noise [1, 3, H, W].
    Returns (crossattn [1, 1, D], concat [1, 4, H/8, W/8], vector [T, 768]) of the conditional half; the negative
    half has zero crossattn / concat and the same vector."""
    x = image01[None].float() * 2.0 - 1.0
    crossattn = co.encode(sd_clip, clip_cfg, x)[:, None]
    concat = veo.encode(sd_enc, vae_cfg, x + noise_aug_strength * noise)
    ids = torch.tensor([fps - 1, motion_bucket_id, noise_aug_strength], dtype=torch.float32, device=x.device)
    vector = uo.timestep_embedding(ids, 256).reshape(1, 768).expand(T, 768).contiguous()
    return crossattn, concat, vector


def sample(sd_unet, unet_cfg, crossattn, concat, vector, latents_noise, *, num_inference_steps=25,
           min_guidance_scale=1.0, max_guidance_scale=3.0):
    """Karras Euler loop with classifier-free guidance; latents_noise [T, 4, h, w] ~ N(0, 1)."""
    T = latents_noise.shape[0]
    sig = karras_sigmas(num_inference_steps)
    ctx = torch.cat([torch.zeros_like(crossattn), crossattn]).repeat_interleave(T, 0)
    cat = torch.cat([torch.zeros_like(concat), concat]).repeat_interleave(T, 0)
    y = torch.cat([vector, vector])

    def net(xin, c_noise):
        return uo.unet_forward(sd_unet, unet_cfg, torch.cat([xin, cat], 1), c_noise, ctx, y, T, 0)

    x = latents_noise * float(np.sqrt(1.0 + sig[0] ** 2))          # init_noise_sigma ("leading" spacing)
    for i in range(num_inference_steps):
        x = so.sampler_step(net, x, float(sig[i]), float(sig[i + 1]), T, min_guidance_scale, max_guidance_scale)
    return x


def decode(sd_dec, vae_cfg, z, decode_chunk_size=8, scaling_factor=0.18215):
    z = 1.0 / scaling_factor * z
    return torch.cat([vdo.decode(sd_dec, vae_cfg, z[i:i + decode_chunk_size], len(z[i:i + decode_chunk_size]))
                      for i in range(0, z.shape[0], decode_chunk_size)])


def quantize(frames: torch.Tensor) -> torch.Tensor:
    """postprocess_video(output_type="pil") -> ToTensor() -> * 2.0 - 1, in numpy / torch fp32 as the pipeline does."""
    v = (frames.float() / 2 + 0.5).clamp(0, 1).cpu().numpy()
    u8 = (v * 255).round().astype(np.uint8)
    return torch.from_numpy(u8).float().div(255) * 2.0 - 1


def pipeline(sd_unet, unet_cfg, sd_clip, clip_cfg, sd_enc, sd_dec, vae_cfg, image01, seed, *, num_frames,
             num_inference_steps=25, fps=7, motion_bucket_id=127, noise_aug_strength=0.02, decode_chunk_size=8):
    """The whole call with a CPU torch.Generator seeded `seed`: image noise, then the latents.  Returns a dict of the
    conditioning, the decoded frames before the 8-bit round trip and after it."""
    H, W = image01.shape[-2:]
    g = torch.Generator().manual_seed(seed)
    noise = torch.randn((1, 3, H, W), generator=g).to(image01.device)
    lat = torch.randn((num_frames, 4, H // 8, W // 8), generator=g).to(image01.device)
    crossattn, concat, vector = conditioning(sd_clip, clip_cfg, sd_enc, vae_cfg, image01, noise, num_frames, fps=fps,
                                             motion_bucket_id=motion_bucket_id, noise_aug_strength=noise_aug_strength)
    z = sample(sd_unet, unet_cfg, crossattn, concat, vector, lat, num_inference_steps=num_inference_steps)
    frames = decode(sd_dec, vae_cfg, z, decode_chunk_size)
    return {"crossattn": crossattn, "concat": concat, "vector": vector, "latents": z, "frames": frames,
            "frames_q": quantize(frames)}
