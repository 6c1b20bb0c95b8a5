"""Deterministic synthetic inputs for the denoiser seam and the interpolation stage (no datasets / checkpoints are
available offline).

Shapes follow the call made by the reference stage driver (code/diffusion_trainer/streaming_svd.py:186-216):
x [(B T),4,h,w], t = c_noise [(B T)], c = {concat [(B T),4,h,w], crossattn [(B T),L,1024], vector [(B T),768]},
ctrl_frames [1,7,3,8h,8w] in [-1,1].  Values come from numpy Generators seeded by (seed, crc32(name)) so that the
build container (golden generation) and the GPU box (tests, bench) see identical tensors.
"""
from __future__ import annotations

import math
import zlib

import numpy as np
import torch


def _rng(seed: int, name: str):
    return np.random.default_rng([seed, zlib.crc32(name.encode())])


def make_inputs(cfg, *, T: int, h: int, w: int, B: int = 2, seed: int = 1, sigma: float = 4.0, ctx_tokens: int = 1):
    n = B * T

    def normal(name, shape, scale=1.0):
        return torch.from_numpy((_rng(seed, name).normal(size=shape) * scale).astype(np.float32))

    c_in = 1.0 / math.sqrt(sigma * sigma + 1.0)                      # denoiser_scaling.py:51-59
    x = normal("x", (n, 4, h, w), sigma * c_in)
    t = torch.full((n,), 0.25 * math.log(sigma), dtype=torch.float32)  # c_noise
    concat = normal("concat", (n, 4, h, w), 1.0)
    cross = normal("crossattn", (n, ctx_tokens, cfg.context_dim), 1.0)
    # vector = concat of three sinusoidal scalar embeddings in the reference; any bounded vector serves
    vec = torch.from_numpy(np.cos(_rng(seed, "vector").uniform(0, 2 * math.pi, size=(n, cfg.adm_in_channels))
                                  ).astype(np.float32))
    ctrl = torch.from_numpy(_rng(seed, "ctrl_frames").uniform(-1, 1, size=(1, cfg.num_frame_conditioning, 3, 8 * h,
                                                                           8 * w)).astype(np.float32))
    c = {"concat": concat, "crossattn": cross, "vector": vec}
    kwargs = dict(batch_size=B, num_video_frames=T, image_only_indicator=torch.zeros(B, T), ctrl_frames=ctrl,
                  num_conditional_frames=cfg.num_frame_conditioning)
    return x, t, c, kwargs


def test_frames(h, w, seed):
    """Two smooth uint8 RGB frames [h, w, 3] (numpy) for the interpolation stage, the second the first shifted by a
    few pixels with a moving bright square.  torch's CPU generator and bicubic resize, so the goldens and their GPU
    tests make the same frames from the seed."""
    g = torch.Generator().manual_seed(seed)
    base = torch.nn.functional.interpolate(torch.rand((1, 3, h // 8, w // 8), generator=g), size=(h, w),
                                           mode="bicubic", align_corners=False)[0]
    f0 = base.clone()
    f1 = torch.roll(base, shifts=(3, -5), dims=(1, 2))
    f0[:, h // 4:h // 4 + 12, w // 4:w // 4 + 12] = 0.95
    f1[:, h // 4 + 4:h // 4 + 16, w // 4 + 6:w // 4 + 18] = 0.95
    to8 = lambda t: (t.clamp(0, 1) * 255).round().to(torch.uint8).permute(1, 2, 0).numpy()  # noqa: E731
    return to8(f0), to8(f1)


def frames_checksum(*frames) -> int:
    """crc32 over the frames' bytes: a golden made from seeded frames records it to catch a generator change."""
    c = 0
    for f in frames:
        c = zlib.crc32(np.ascontiguousarray(f).tobytes(), c)
    return c


def region_spec(h, w, tile=64):
    """Where a full-size interpolation golden keeps its values: 64x64 tiles at the four corners and the centre
    (tile_origins, [5, 2] (y, x)), and whole rows / columns at the first, middle and last index."""
    origins = [(0, 0), (0, w - tile), (h - tile, 0), (h - tile, w - tile), (h // 2 - tile // 2, w // 2 - tile // 2)]
    return dict(tile_origins=np.array(origins, np.int64), tile=tile, rows=np.array([0, h // 2 - 1, h - 1], np.int64),
                cols=np.array([0, w // 2 - 1, w - 1], np.int64))


def crop_regions(t, *, tile_origins, tile, rows, cols):
    """[C, h, w] (numpy or torch) -> [C, L]: the tiles, rows and columns of region_spec flattened and concatenated."""
    cat = np.concatenate if isinstance(t, np.ndarray) else torch.cat
    c = t.shape[0]
    parts = [t[:, y:y + tile, x:x + tile].reshape(c, -1) for y, x in np.asarray(tile_origins).tolist()]
    parts += [t[:, int(r), :] for r in rows] + [t[:, :, int(k)] for k in cols]
    return cat(parts, 1)
