"""Stage driver of the autoregressive StreamingSVD stage (SURVEY.md section 8 row a22) on top of the project's pieces:
denoiser seam (`B200StreamingWrapper`), sampler (`B200EulerEDMSampler`) and temporal VAE decoder (`B200VaeDecoder`).

Mirrors, method for method, the reference's `StreamingSVD` LightningModule
(code/diffusion_trainer/streaming_svd.py):
    decode_first_stage            :124-151   scale, decode in groups of <= 8 frames, concatenate
    _generate_conditional_output  :155-221   conditioning, noise, 30-step sampler, decode, clamp
    extract_ctrl_frames           :263-290   last `num_conditional_frames` frames of the previous chunk
    _autoregressive_generation    :293-356   chunk loop: condition on the previous chunk, keep frames after the first
                                             `num_conditional_frames`, concatenate, convert to [0, 255]
It is host logic: frame bookkeeping on whole tensors (slicing, concatenation, range conversion — the reference's
`result_processor.convert_range`, utils/result_processor.py:4-14).  The conditioner is injected as a callable
`conditioner(svd_input_frame, num_frames) -> (c, uc)` with `crossattn [1,L,1024]`, `concat [1,4,h,w]`,
`vector [num_frames,768]`, exactly what `conditioner.get_unconditional_conditioning` returns at
streaming_svd.py:181-188; `conditioner.B200SVDConditioner` is that callable on the project's kernels (OpenCLIP ViT-H/14
image tower with CLIP preprocessing, SD-VAE encoder, fps / motion / cond_aug embeddings).  The heavy components raise without the CUDA library; nothing here falls back to a CPU
implementation."""
from __future__ import annotations

import math
from typing import Callable, List, Optional, Sequence, Union

import numpy as np
import torch

from . import dist_utils

SCALE_FACTOR = 0.18215      # config.yaml scale_factor (diff_trainer_params.scale_factor)
MAX_DECODE_CHUNK = 8        # streaming_svd.py:127 (4 with use_memopt)
SPATIAL_COMPRESSION = 8     # streaming_svd.py:157
IMAGE_HEIGHT, IMAGE_WIDTH = 576, 1024   # streaming_svd.py:384-385


def convert_range(video: torch.Tensor, output_range: Sequence[float], input_range: Sequence[float]) -> torch.Tensor:
    """utils/result_processor.py:4-14 with an explicit input range."""
    video = (video - input_range[0]) / (input_range[1] - input_range[0])
    return video * (output_range[1] - output_range[0]) + output_range[0]


def resize_and_keep(image):
    """utils/inference_utils.py:37-42: PIL resize to height 576, width scaled by the same factor (truncated), with
    Pillow's default filter.  `image` is a PIL image or a uint8 [H, W, 3] array; returns a PIL image."""
    from PIL import Image
    if not isinstance(image, Image.Image):
        image = Image.fromarray(np.asarray(image, dtype=np.uint8))
    hpercent = IMAGE_HEIGHT / float(image.size[1])
    return image.resize((int(float(image.size[0]) * float(hpercent)), IMAGE_HEIGHT))


def _to_fchw(video: torch.Tensor) -> torch.Tensor:
    """Accept [F,C,H,W] or [F,H,W,C] like the reference's rearranges (streaming_svd.py:245-250, :314-315)."""
    if video.dim() == 4 and video.shape[1] == 3:
        return video
    if video.dim() == 4 and video.shape[-1] == 3:
        return video.permute(0, 3, 1, 2)
    raise NotImplementedError(f"Unexpected video input format: {tuple(video.shape)}")


class B200StreamingSVDStage:
    def __init__(self, inference_model, sampler, vae_decoder, conditioner: Callable, *, num_conditional_frames: int = 7,
                 anchor_frame: int = 6, scale_factor: float = SCALE_FACTOR, max_decode_chunk: int = MAX_DECODE_CHUNK,
                 device="cuda:0", shard_decode: bool = False):
        self.inference_model = inference_model      # B200StreamingWrapper        (streaming_svd.py:50-56)
        self.sampler = sampler                      # B200EulerEDMSampler         (config.yaml:139-157)
        self.vae_decoder = vae_decoder              # B200VaeDecoder              (first_stage_model.decode)
        self.conditioner = conditioner
        self.num_conditional_frames = int(num_conditional_frames)
        self.anchor_frame = int(anchor_frame)           # inference_params.anchor_frames: '6' (config.yaml:316)
        self.scale_factor = float(scale_factor)
        self.max_decode_chunk = int(max_decode_chunk)
        self.device = torch.device(device)
        # opt-in: spread the groups of <= 8 frames of decode_first_stage over the ranks of the process group
        # (SURVEY.md section 8(e): "VAE decode: embarrassingly, frame groups of 8, gather at the end")
        self.shard_decode = bool(shard_decode)

    # -- streaming_svd.py:124-151 ----------------------------------------------------------------------------------
    def decode_first_stage(self, z: torch.Tensor) -> torch.Tensor:
        z = 1.0 / self.scale_factor * z
        n_samples = min(z.shape[0], self.max_decode_chunk)
        n_rounds = math.ceil(z.shape[0] / n_samples)
        rank, world = dist_utils.rank_world() if self.shard_decode else (0, 1)
        if world == 1:
            outs = []
            for n in range(n_rounds):
                part = z[n * n_samples:(n + 1) * n_samples]
                outs.append(self.vae_decoder.decode(part, timesteps=len(part)))
            return torch.cat(outs, dim=0)
        # group g is decoded by rank g % world into slot g // world of that rank's contribution
        slots = math.ceil(n_rounds / world)
        mine = None
        for g in range(rank, n_rounds, world):
            part = z[g * n_samples:(g + 1) * n_samples]
            out = self.vae_decoder.decode(part, timesteps=len(part))
            if mine is None:
                mine = out.new_zeros((slots * n_samples,) + tuple(out.shape[1:]))
            mine[(g // world) * n_samples:(g // world) * n_samples + len(part)] = out
        if mine is None:   # more ranks than groups: contribute zeros of the right shape
            mine = torch.zeros((slots * n_samples, 3, z.shape[-2] * SPATIAL_COMPRESSION,
                                z.shape[-1] * SPATIAL_COMPRESSION), dtype=torch.float32, device=z.device)
        allp = dist_utils.all_gather_cat(mine)
        per_rank = slots * n_samples
        outs = []
        for g in range(n_rounds):
            n_g = min(n_samples, z.shape[0] - g * n_samples)
            o = (g % world) * per_rank + (g // world) * n_samples
            outs.append(allp[o:o + n_g])
        return torch.cat(outs, dim=0)

    # -- streaming_svd.py:263-290 ----------------------------------------------------------------------------------
    def extract_ctrl_frames(self, video: torch.Tensor) -> torch.Tensor:
        video = _to_fchw(video)[None]                                   # "F C W H -> 1 F C W H", range already [-1,1]
        return video[:, -self.num_conditional_frames:]

    # -- streaming_svd.py:155-221 ----------------------------------------------------------------------------------
    def generate_conditional_output(self, svd_input_frame: torch.Tensor, ctrl_frames: torch.Tensor,
                                    generator: Optional[torch.Generator] = None) -> torch.Tensor:
        T = self.sampler.num_frames
        H, W = svd_input_frame.shape[-2], svd_input_frame.shape[-1]
        shape = (T, 4, H // SPATIAL_COMPRESSION, W // SPATIAL_COMPRESSION)
        batch_size = 1
        c, uc = self.conditioner(svd_input_frame, T)
        c, uc = dict(c), dict(uc)
        for k in ("crossattn", "concat"):                               # :190-194 repeat "b ... -> (b t) ..."
            uc[k] = uc[k].repeat_interleave(T, dim=0)
            c[k] = c[k].repeat_interleave(T, dim=0)
        randn = torch.randn(shape, generator=generator, device=generator.device if generator is not None else "cpu")
        randn = randn.to(self.device)
        if self.shard_decode or getattr(self.sampler, "cfg_parallel", False):
            # every rank of a sharded step / decode must integrate the SAME latent: rank 0's noise wins (the ranks'
            # generators are not assumed to be seeded alike).  The conditioner's cond_aug noise (streaming_svd.py:174)
            # is drawn inside the injected callable; B200SVDConditioner broadcasts rank 0's the same way.
            randn = dist_utils.broadcast_from_rank0(randn)
        extra = dict(image_only_indicator=torch.zeros(2 * batch_size, T, device=self.device), num_video_frames=T,
                     batch_size=2 * batch_size, num_conditional_frames=self.num_conditional_frames,
                     ctrl_frames=ctrl_frames)
        samples_z = self.sampler(self.inference_model, randn, c, uc, **extra)     # :216 sampler(denoiser, randn, c, uc)
        samples_x = self.decode_first_stage(samples_z)
        return torch.clamp(samples_x, min=-1.0, max=1.0)

    # -- streaming_svd.py:293-356 ----------------------------------------------------------------------------------
    def autoregressive_generation(self, initial_generation: Union[torch.Tensor, List[torch.Tensor]],
                                  n_autoregressive_generations: int,
                                  generator: Optional[torch.Generator] = None) -> torch.Tensor:
        """initial_generation: the first chunk, float in [-1, 1], [F,C,H,W] or [F,H,W,C].  Returns the whole video
        [F_total,C,H,W] in [0, 255] (the reference wraps the same tensor in its IImage container)."""
        chunks = initial_generation if isinstance(initial_generation, list) else [initial_generation]
        chunks = [_to_fchw(chunks[0])] + list(chunks[1:])
        for _ in range(int(n_autoregressive_generations)):
            ctrl_frames = self.extract_ctrl_frames(chunks[-1])
            svd_input_frame = chunks[0][self.anchor_frame]
            result = self.generate_conditional_output(svd_input_frame, ctrl_frames, generator)
            chunks.append(result[self.num_conditional_frames:])         # :347 keep all but the conditioning frames
        chunks = [convert_range(ch.to(torch.float32), [0, 255], [-1, 1]) for ch in chunks]
        return torch.cat([ch.to(chunks[0].device) for ch in chunks], dim=0)

    # -- streaming_svd.py:359-399 ----------------------------------------------------------------------------------
    def image_to_video(self, image, n_autoregressive_generations: int, first_chunk: Callable,
                       generator: Optional[torch.Generator] = None) -> torch.Tensor:
        """image (PIL image or uint8 [H, W, 3]) -> the whole video [F_total, C, H, W] in [0, 255].  The image is resized
        to height 576 on the host (one image per request) and must then be 1024 x 576; `first_chunk` (normally a
        `first_chunk.B200SVDImageToVideo`) makes the first chunk from it with the same `generator`, and
        `autoregressive_generation` continues from there."""
        img = resize_and_keep(image)
        assert img.width == IMAGE_WIDTH and img.height == IMAGE_HEIGHT, f"image resized to {img.size}, need 1024x576"
        video_chunks = first_chunk(np.asarray(img.convert("RGB")), generator=generator)
        return self.autoregressive_generation(video_chunks.to(self.device), n_autoregressive_generations, generator)

    def to_uint8_frames(self, video: torch.Tensor) -> torch.Tensor:
        """[F,C,H,W] float in [0, 255] -> uint8 [F,H,W,C] ON THE DEVICE: the array the reference's IImage container
        ends up holding after `result_processor.concat_chunks` (utils/result_processor.py:17-31,
        lib/farancia/libimage/iimage.py:21-39), ready for a 1-byte-per-sample device->host copy."""
        from . import ops
        return ops.frames_to_uint8(video.to(self.device, torch.float32).contiguous(), 0.0, 255.0)
