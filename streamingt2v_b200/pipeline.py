"""A whole image-to-video request from one call: the reference's `StreamingPipeline` (code/inference_i2v.py:51-260)
on the project's pieces.

    image_to_video     :175-191   first chunk + ceil((F - T) / (T - n_cond)) autoregressive chunks, video[:F]
    enhance_video      :193-209   PIL BICUBIC resizes of the image and of every frame to 1280x720, then the enhance
                                  stage (i2v_enhance_interface.i2v_enhance_process)
    interpolate_video  :211-224   EMA-VFI midpoints (i2v_enhance_interface.vfi_process) up to the requested length
    __call__           :227-258   the `__main__` request: (num_frames + 1) // 2 frames from the first stage, enhance,
                                  interpolate back to num_frames; without randomized blending enhance runs one chunk
                                  of all frames with no overlap (:237-239)

The frames stay on the device from the first chunk to VFI's output as long as the enhance callable keeps them there:
the float frames become uint8 with `frames_to_uint8` (the reference's IImage container) and the resizes run in
`ops.resize_bicubic_u8`, which equals Pillow byte for byte.

Enhance is a callable, so that any implementation of the I2VGen-XL stage plugs in:

    enhance(image_u8 [720, 1280, 3], video_u8 [F, 720, 1280, 3], *, chunk_size, overlap_size,
            use_randomized_blending, generator) -> uint8 [F', 720, 1280, 3]

with F' < F when randomized blending drops the frames that do not fill a last chunk (i2v_enhance_interface.py:115-118).
INTEGRATION.md shows the adapter that wraps the reference's own `i2v_enhance_process`."""
from __future__ import annotations

import math
import operator
from typing import Callable, Optional

import numpy as np
import torch

from . import ops
from . import vfi as vfi_stage

ENHANCE_HEIGHT, ENHANCE_WIDTH = 720, 1280      # i2v_enhance_interface.py:99-100, inference_i2v.py:195,198


def _image_u8(image) -> np.ndarray:
    """The request image (PIL image or array) as uint8 [H, W, 3]."""
    arr = np.asarray(image)
    if arr.dtype != np.uint8 or arr.ndim != 3 or arr.shape[2] != 3 or arr.shape[0] < 1 or arr.shape[1] < 1:
        raise ValueError(f"the request image must be uint8 RGB [H, W, 3], got {arr.shape} {arr.dtype}")
    return arr


class B200StreamingPipeline:
    """stage: a `stage.B200StreamingSVDStage`; first_chunk: the first-chunk callable `stage.image_to_video` takes
    (normally a `first_chunk.B200SVDImageToVideo`); vfi: a `vfi.B200VFI`; enhance: the enhance callable above."""

    def __init__(self, stage, first_chunk: Callable, vfi, enhance: Callable):
        self.stage = stage
        self.first_chunk = first_chunk
        self.vfi = vfi
        self.enhance = enhance

    # -- inference_i2v.py:175-191 ------------------------------------------------------------------------------------
    def _n_autoregressive_generations(self, num_frames: int) -> int:
        """Chunks after the first for a video of num_frames frames (:179-184); none when the first chunk suffices."""
        n_cond = self.stage.num_conditional_frames
        n_frames_per_gen = self.stage.sampler.num_frames
        return max(0, math.ceil((num_frames - n_frames_per_gen) / (n_frames_per_gen - n_cond)))

    def image_to_video(self, image, num_frames: int, *, generator: Optional[torch.Generator] = None) -> torch.Tensor:
        """image (PIL image or uint8 [H, W, 3]) -> uint8 [num_frames, 576, 1024, 3] on the device (fewer frames if the
        chunks make fewer)."""
        image = _image_u8(image)
        video = self.stage.image_to_video(image, self._n_autoregressive_generations(num_frames), self.first_chunk,
                                          generator=generator)
        return self.stage.to_uint8_frames(video[:num_frames])

    # -- inference_i2v.py:193-209 ------------------------------------------------------------------------------------
    def enhance_video(self, image, video: torch.Tensor, *, chunk_size: int = 38, overlap_size: int = 12,
                      use_randomized_blending: bool = False,
                      generator: Optional[torch.Generator] = None) -> torch.Tensor:
        """The request image and the first stage's uint8 [F, h, w, 3] frames, both resized to 1280x720 with PIL's
        BICUBIC filter on the device, through the enhance callable -> uint8 [F', 720, 1280, 3]."""
        dev = self.stage.device
        img = torch.from_numpy(np.ascontiguousarray(_image_u8(image)))[None].to(dev)
        img = ops.resize_bicubic_u8(img, ENHANCE_WIDTH, ENHANCE_HEIGHT)[0]
        frames = ops.resize_bicubic_u8(video.to(dev), ENHANCE_WIDTH, ENHANCE_HEIGHT)
        out = self.enhance(img, frames, chunk_size=chunk_size, overlap_size=overlap_size,
                           use_randomized_blending=use_randomized_blending, generator=generator)
        if not (isinstance(out, torch.Tensor) and out.dtype == torch.uint8 and out.dim() == 4
                and tuple(out.shape[1:]) == (ENHANCE_HEIGHT, ENHANCE_WIDTH, 3) and 1 <= out.shape[0] <= frames.shape[0]):
            got = f"{tuple(out.shape)} {out.dtype}" if isinstance(out, torch.Tensor) else type(out).__name__
            raise ValueError(f"enhance must return uint8 [F', {ENHANCE_HEIGHT}, {ENHANCE_WIDTH}, 3] with 1 <= F' <= "
                             f"{frames.shape[0]}, got {got}")
        return out

    # -- inference_i2v.py:211-224 ------------------------------------------------------------------------------------
    def interpolate_video(self, video: torch.Tensor, dest_num_frames: int) -> torch.Tensor:
        """uint8 [F, 720, 1280, 3] -> uint8 [dest_num_frames, 720, 1280, 3] on the device (fewer when F is short)."""
        return vfi_stage.interpolate_video(video, dest_num_frames, self.vfi)

    # -- inference_i2v.py:227-258 ------------------------------------------------------------------------------------
    @torch.no_grad()
    def __call__(self, image, num_frames: int, *, use_randomized_blending: bool = False, chunk_size: int = 38,
                 overlap_size: int = 12, generator: Optional[torch.Generator] = None) -> torch.Tensor:
        """One request: image -> uint8 [num_frames', 720, 1280, 3] on the device, the array the reference saves as its
        video.  num_frames' = num_frames unless randomized blending drops frames in the enhance stage."""
        try:
            num_frames = operator.index(num_frames)
        except TypeError:
            raise ValueError(f"num_frames must be an integer, got {num_frames!r}") from None
        if num_frames < 1:
            raise ValueError(f"num_frames must be positive, got {num_frames}")
        if not use_randomized_blending:
            chunk_size = (num_frames + 1) // 2
            overlap_size = 0
        video = self.image_to_video(image, (num_frames + 1) // 2, generator=generator)
        video_enh = self.enhance_video(image, video, use_randomized_blending=use_randomized_blending,
                                       chunk_size=chunk_size, overlap_size=overlap_size, generator=generator)
        return self.interpolate_video(video_enh, num_frames)
