"""CPU: the frame arithmetic of `pipeline.B200StreamingPipeline` against the reference's request
(code/inference_i2v.py `__main__` and `StreamingPipeline`, code/i2v_enhance/i2v_enhance_interface.py), with stand-ins
that record what they are given: a stage that makes identifiable frames, an enhance that truncates as the reference's
randomized blending does, a VFI network that marks its midpoints, and Pillow in place of the resize kernel (whose
parity with Pillow tests/test_resize*.py check)."""
import math
import types

import numpy as np
import pytest
import torch
from PIL import Image

import fake_ops
from streamingt2v_b200 import pipeline as pl
from streamingt2v_b200 import vfi

TG, NCOND = 8, 3            # frames per generation and conditioning frames of the stand-in stage
FRAME_H, FRAME_W = 18, 32   # the stand-in stage's frame size (the real one makes 576x1024)


def reference_request(num_frames, use_randomized_blending, chunk_size, overlap_size):
    """The numbers of one request, restated from the reference."""
    if not use_randomized_blending:                                           # inference_i2v.py:237-239
        chunk_size, overlap_size = (num_frames + 1) // 2, 0
    first_stage = (num_frames + 1) // 2                                       # :249
    n_gen = math.ceil((first_stage - TG) / (TG - NCOND))                      # :179-184; range(n) of n <= 0 is empty
    generated = TG + max(n_gen, 0) * (TG - NCOND)                             # streaming_svd.py:318-354
    kept = min(first_stage, generated)                                        # inference_i2v.py:190
    enhanced = kept
    if use_randomized_blending:                                               # i2v_enhance_interface.py:90-118
        starts = [i for i in range(0, kept, chunk_size - overlap_size)
                  if len(range(i, min(i + chunk_size, kept))) == chunk_size]
        enhanced = (chunk_size - overlap_size) * (len(starts) - 1) + chunk_size
    n = min(enhanced, num_frames // 2 + 1)                                    # vfi_process, :31
    out = 2 * n - 1 + (1 if num_frames % 2 == 0 else 0)                       # :40-54
    return dict(n_gen=n_gen, kept=kept, chunk_size=chunk_size, overlap_size=overlap_size, enhanced=enhanced, out=out,
                midpoints=list(range(n - 1)))


def _stage_video(n_frames):
    """[n, 3, h, w] float in [0, 255]; frame f has f in its pixel (0, 0) red channel."""
    v = torch.rand((n_frames, 3, FRAME_H, FRAME_W), generator=torch.Generator().manual_seed(n_frames)) * 255.0
    v[:, 0, 0, 0] = torch.arange(n_frames, dtype=torch.float32)
    return v


class FakeStage:
    num_conditional_frames = NCOND
    sampler = types.SimpleNamespace(num_frames=TG)
    device = torch.device("cpu")

    def __init__(self):
        self.calls = []

    def image_to_video(self, image, n_autoregressive_generations, first_chunk, generator=None):
        self.calls.append(dict(image=image, n_gen=n_autoregressive_generations, first_chunk=first_chunk,
                               generator=generator))
        return _stage_video(TG + n_autoregressive_generations * (TG - NCOND))

    def to_uint8_frames(self, video):
        return fake_ops.frames_to_uint8(video.contiguous(), 0.0, 255.0)


class FakeEnhance:
    """Records its inputs; returns the video, truncated as randomized blending does (i2v_enhance_interface.py:90-118)."""

    def __init__(self):
        self.calls = []

    def __call__(self, image, video, *, chunk_size, overlap_size, use_randomized_blending, generator):
        self.calls.append(dict(image=image.clone(), video=video.clone(), chunk_size=chunk_size,
                               overlap_size=overlap_size, use_randomized_blending=use_randomized_blending,
                               generator=generator))
        if use_randomized_blending:
            chunks = [video[i:i + chunk_size] for i in range(0, len(video), chunk_size - overlap_size)
                      if len(video[i:i + chunk_size]) == chunk_size]
            video = video[:(chunk_size - overlap_size) * (len(chunks) - 1) + chunk_size]
        out = video.clone()
        out[:, 0, 0, 0] = torch.arange(len(out), dtype=torch.uint8)         # frame index, for the VFI stand-in
        return out


class FakeVFI:
    dev = torch.device("cpu")

    def __init__(self):
        self.midpoints = []

    def _predict(self, b0, b1, frame):
        i = int(round(float(b0[0, 2, 0, 0]) * 255))                        # R of pixel (0, 0) (BGR input)
        assert int(round(float(b1[0, 2, 0, 0]) * 255)) == i + 1
        self.midpoints.append(i)
        frame.fill_(200)


def pil_resize(x, W, H):
    return torch.from_numpy(np.stack([np.asarray(Image.fromarray(f).resize((W, H))) for f in x.numpy()]))


@pytest.fixture
def host_ops(monkeypatch):
    monkeypatch.setattr(pl, "ops", types.SimpleNamespace(resize_bicubic_u8=pil_resize))
    monkeypatch.setattr(vfi, "ops", types.SimpleNamespace(
        vfi_frames_to_bgr=lambda fr: (fr[..., [2, 1, 0]].double() / 255.0).float().permute(0, 3, 1, 2).contiguous()))


def _request_image():
    return np.random.default_rng(5).integers(0, 256, size=(45, 70, 3), dtype=np.uint8)


@pytest.mark.parametrize("num_frames,blend,chunk_size,overlap_size", [
    (1, False, 38, 12), (2, False, 38, 12), (9, False, 38, 12), (16, False, 38, 12), (17, False, 38, 12),
    (30, False, 38, 12), (41, False, 38, 12),
    (30, True, 6, 2), (31, True, 6, 2), (41, True, 8, 3), (36, True, 5, 1), (16, True, 8, 0),
])
def test_request_frame_arithmetic(host_ops, num_frames, blend, chunk_size, overlap_size):
    ref = reference_request(num_frames, blend, chunk_size, overlap_size)
    stage, enhance, net = FakeStage(), FakeEnhance(), FakeVFI()
    first_chunk = object()
    gen = torch.Generator().manual_seed(1)
    image = _request_image()
    p = pl.B200StreamingPipeline(stage, first_chunk, net, enhance)
    out = p(image, num_frames, use_randomized_blending=blend, chunk_size=chunk_size, overlap_size=overlap_size,
            generator=gen)

    # first stage: generation count, the request image and generator handed on
    (sc,) = stage.calls
    assert sc["n_gen"] == max(ref["n_gen"], 0)
    assert np.array_equal(sc["image"], image) and sc["first_chunk"] is first_chunk and sc["generator"] is gen
    # enhance: the image and the first `kept` frames, as uint8, resized to 1280x720; chunk parameters
    (ec,) = enhance.calls
    u8 = fake_ops.frames_to_uint8(_stage_video(TG + sc["n_gen"] * (TG - NCOND)), 0.0, 255.0)[:ref["kept"]]
    assert ec["video"].shape == (ref["kept"], 720, 1280, 3)
    assert torch.equal(ec["video"], pil_resize(u8, 1280, 720))
    assert torch.equal(ec["image"], pil_resize(torch.from_numpy(image)[None], 1280, 720)[0])
    assert (ec["chunk_size"], ec["overlap_size"]) == (ref["chunk_size"], ref["overlap_size"])
    assert ec["use_randomized_blending"] is blend and ec["generator"] is gen
    # VFI: interpolates the enhanced frames up to num_frames
    assert out.shape == (ref["out"], 720, 1280, 3) and out.dtype == torch.uint8
    assert net.midpoints == ref["midpoints"]
    if not blend:
        assert out.shape[0] == num_frames


def test_no_autoregressive_chunk_when_the_first_suffices(host_ops):
    stage = FakeStage()
    p = pl.B200StreamingPipeline(stage, None, FakeVFI(), FakeEnhance())
    for half, want in ((1, 0), (TG, 0), (TG + 1, 1), (TG + TG - NCOND, 1), (TG + TG - NCOND + 1, 2)):
        p.image_to_video(_request_image(), half)
        assert stage.calls[-1]["n_gen"] == want


def test_rejects_bad_requests(host_ops):
    p = pl.B200StreamingPipeline(FakeStage(), None, FakeVFI(), FakeEnhance())
    with pytest.raises(ValueError, match="positive"):
        p(_request_image(), 0)
    with pytest.raises(ValueError, match="integer"):
        p(_request_image(), 8.0)
    with pytest.raises(ValueError, match="uint8 RGB"):
        p(np.zeros((45, 70, 4), np.uint8), 8)
    with pytest.raises(ValueError, match="uint8 RGB"):
        p(np.zeros((45, 70, 3), np.float32), 8)

    def wrong_size(image, video, **kw):
        return video[:, :576]

    with pytest.raises(ValueError, match="enhance must return"):
        pl.B200StreamingPipeline(FakeStage(), None, FakeVFI(), wrong_size)(_request_image(), 8)
