"""Randomized-blending denoising loop of the enhance stage (SURVEY.md section 8 row a24, loop part; north_star:
"chunk_size/overlap_size/randomized-blending args", "the i2v_enhance randomized-blending chunks ... shard across the
8 GPUs of one box with NCCL over NVLink only for the overlap-region allgather").

Mirrors the loop body of `I2VGenXLPipeline.__call__` (reference code/i2v_enhance/pipeline_i2vgen_xl.py:841-909):
for every scheduler timestep, every chunk of `chunk_size` frames (stride `chunk_size - overlap_size`) is denoised
independently from the SAME `latents` — UNet with its own first-frame conditioning, classifier-free guidance, one
DDIM step — and written into `latents_denoised` from a random offset inside the overlap on (offset 0 for the first
chunk), later chunks overwriting earlier ones.  The UNet is injected: `unet(sample[2,C,cs,H,W], t, **per_chunk) ->
[2,C,cs,H,W]` (the reference's `self.unet(...)[0]`, pipeline_i2vgen_xl.py:857-867; this project's I2VGen-XL UNet itself is
not built yet — DESIGN.md).  The guidance combine + DDIM step + blended write are ONE CUDA kernel
(`b200svd_ddim_blend_step`); there is no CPU fallback.

Multi-GPU (`shard=True`, one process per GPU): within a timestep the chunks are independent, so chunk i is denoised
by rank i % world into a per-rank slot buffer; ONE all-gather of the slot buffers per timestep (<= 4.4 MB per chunk at
90x160) and every rank assembles the identical blended latent.  The random offsets are drawn on rank 0 in the
reference's order (one `randint(0, overlap_size - 1)` per non-first chunk per timestep, python `random`) and broadcast,
so a sharded run reproduces the single-process run bit for bit."""
from __future__ import annotations

import random
from typing import Callable, List, Optional, Sequence

import torch

from . import dist_utils, ops


def chunk_starts(num_frames: int, chunk_size: int, overlap_size: int, n_chunks: int) -> List[int]:
    """CHUNK_START of every chunk (pipeline_i2vgen_xl.py:845,904) and the reference's divisibility check (:908-910)."""
    starts = [i * (chunk_size - overlap_size) for i in range(n_chunks)]
    end = n_chunks * (chunk_size - overlap_size)
    if end + overlap_size > num_frames:
        raise NotImplementedError(f"Video of size={num_frames} is not dividable into chunks with size={chunk_size} "
                                  f"and overlap={overlap_size}")
    return starts


def draw_offsets(n_steps: int, n_chunks: int, overlap_size: int, rng=None) -> List[List[int]]:
    """The random offsets in the order the reference draws them (:891-898): per timestep, per chunk; chunk 0 -> 0."""
    rng = random if rng is None else rng
    out = []
    for _ in range(n_steps):
        row = []
        for idx in range(n_chunks):
            row.append(0 if idx == 0 or overlap_size == 0 else rng.randint(0, overlap_size - 1))
        out.append(row)
    return out


class B200RandomizedBlending:
    def __init__(self, unet: Callable, alphas_cumprod: Sequence[float], *, chunk_size: int = 38, overlap_size: int = 12,
                 guidance_scale: Optional[float] = 9.0, prediction_type: str = "v_prediction",
                 num_train_timesteps: int = 1000, final_alpha_cumprod: float = 1.0, rng=None, shard: bool = False):
        if prediction_type not in ("v_prediction", "epsilon"):
            raise NotImplementedError(prediction_type)
        self.unet = unet
        self.alphas_cumprod = [float(a) for a in alphas_cumprod]
        self.chunk_size, self.overlap_size = int(chunk_size), int(overlap_size)
        self.guidance_scale = None if guidance_scale is None or guidance_scale <= 1.0 else float(guidance_scale)
        self.v_prediction = prediction_type == "v_prediction"
        self.num_train_timesteps = int(num_train_timesteps)
        self.final_alpha_cumprod = float(final_alpha_cumprod)
        self.rng = rng
        self.shard = bool(shard)

    def _alphas(self, t: int, step_ratio: int):
        """DDIMScheduler.step: alpha_prod_t, alpha_prod_t_prev (prev_timestep = t - train_steps // inference_steps)."""
        prev = t - step_ratio
        return self.alphas_cumprod[t], (self.alphas_cumprod[prev] if prev >= 0 else self.final_alpha_cumprod)

    @torch.no_grad()
    def __call__(self, latents: torch.Tensor, timesteps: Sequence[int], per_chunk_kwargs: Sequence[dict],
                 num_inference_steps: Optional[int] = None, **unet_kwargs) -> torch.Tensor:
        """latents: fp32 [1, C, F, H, W]; timesteps: the (SDEdit-truncated) scheduler timesteps in order;
        per_chunk_kwargs[i]: the keyword arguments that differ per chunk (`image_latents`, `image_embeddings`,
        pipeline_i2vgen_xl.py:861-862).  Returns the denoised latents [1, C, F, H, W]."""
        assert latents.dim() == 5 and latents.shape[0] == 1, "batch 1 (one video), as in the reference's enhance call"
        latents = latents.to(torch.float32).contiguous()
        _, Cc, F, H, W = latents.shape
        n_chunks = len(per_chunk_kwargs)
        cs = self.chunk_size
        starts = chunk_starts(F, cs, self.overlap_size, n_chunks)
        n_inf = int(num_inference_steps) if num_inference_steps is not None else len(timesteps)
        step_ratio = self.num_train_timesteps // n_inf
        rank, world = dist_utils.rank_world() if self.shard else (0, 1)
        offsets = draw_offsets(len(timesteps), n_chunks, self.overlap_size, self.rng) if rank == 0 else None
        if world > 1:
            offsets = dist_utils.broadcast_object(offsets)
        slots = -(-n_chunks // world)
        for si, t in enumerate(timesteps):
            t = int(t)
            a_t, a_prev = self._alphas(t, step_ratio)
            if world == 1:
                denoised = torch.empty_like(latents)
            else:
                mine = torch.zeros((slots, Cc, cs, H, W), dtype=torch.float32, device=latents.device)
            for idx in range(rank, n_chunks, world):
                chunk = latents[:, :, starts[idx]:starts[idx] + cs]
                xin = torch.cat([chunk] * 2) if self.guidance_scale is not None else chunk   # scale_model_input == id
                noise = self.unet(xin.contiguous(), t, **per_chunk_kwargs[idx], **unet_kwargs)
                noise = noise.to(torch.float32).contiguous()
                if world == 1:
                    ops.ddim_blend_step(noise, latents, denoised, lat_start=starts[idx], out_start=starts[idx],
                                        offset=offsets[si][idx], guidance=self.guidance_scale, alpha_t=a_t,
                                        alpha_prev=a_prev, v_prediction=self.v_prediction)
                else:
                    ops.ddim_blend_step(noise, latents, mine[idx // world][None], lat_start=starts[idx], out_start=0,
                                        offset=0, guidance=self.guidance_scale, alpha_t=a_t, alpha_prev=a_prev,
                                        v_prediction=self.v_prediction)
            if world > 1:
                allp = dist_utils.all_gather_cat(mine)                     # [world * slots, C, cs, H, W], rank-major
                denoised = torch.empty_like(latents)
                for idx in range(n_chunks):                                 # ascending: later chunks overwrite earlier
                    off = offsets[si][idx]
                    src = allp[(idx % world) * slots + idx // world]
                    denoised[0, :, starts[idx] + off:starts[idx] + cs] = src[:, off:]
            latents = denoised
        return latents
