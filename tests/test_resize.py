"""CPU: the host taps of the PIL-exact BICUBIC resize (`ops.bicubic_taps`), run through a numpy restatement of the two
passes of csrc/resize.cu, equal `PIL.Image.resize` byte for byte.  The size table covers both of the reference's
resizes (inference_i2v.py:194-199), up- and downscales including large ratios, one axis unchanged, identity, and tiny
and odd sizes; tests/test_resize_gpu.py runs the kernel on the same table."""
import numpy as np
import pytest
from PIL import Image

from streamingt2v_b200 import ops

# (w_in, h_in, w_out, h_out)
SIZES = [
    (1024, 576, 1280, 720),     # every first-stage frame before enhance (inference_i2v.py:198)
    (1920, 1080, 1280, 720),    # a 1080p request image (:195)
    (640, 360, 1280, 720),
    (1000, 563, 1280, 720),
    (37, 23, 1280, 720),
    (2000, 1500, 1024, 576),
    (1023, 577, 1024, 576),
    (1280, 576, 1280, 720),     # width unchanged: vertical pass only
    (1024, 720, 1280, 720),     # height unchanged: horizontal pass only
    (1280, 720, 1280, 720),     # identity
    (3000, 40, 7, 3),           # downscale by 430 and 13
    (333, 777, 250, 100),
    (1, 1, 5, 9),
    (3, 2, 1, 1),
    (7, 5, 64, 2),
]


def _pass(x, bounds, taps, axis):
    """One pass of the kernel along `axis` of uint8 [..., 3]: out[i] = clip((2^21 + sum_j taps[i, j] *
    x[bounds[i, 0] + j]) >> 22, 0, 255) over j < bounds[i, 1], in int32."""
    x = np.moveaxis(x, axis, -2)
    k = taps.shape[1]
    j = np.arange(k)[None]
    valid = j < bounds[:, 1:2]
    idx = np.where(valid, bounds[:, :1] + j, 0)
    g = x[..., idx, :].astype(np.int32)                                      # [..., n_out, k, 3]
    acc = (1 << 21) + (g * np.where(valid, taps, 0)[..., None]).sum(-2, dtype=np.int32)
    return np.moveaxis(np.clip(acc >> 22, 0, 255).astype(np.uint8), -2, axis)


def resize_like_kernel(frames, W, H):
    """uint8 [F, h, w, 3] -> [F, H, W, 3]: horizontal pass, then vertical, each skipped when its axis keeps its size."""
    _, h, w, _ = frames.shape
    out = frames
    if W != w:
        b, t = ops.bicubic_taps(w, W)
        out = _pass(out, b.numpy(), t.numpy(), 2)
    if H != h:
        b, t = ops.bicubic_taps(h, H)
        out = _pass(out, b.numpy(), t.numpy(), 1)
    return out


def pil_resize(frames, W, H):
    return np.stack([np.asarray(Image.fromarray(f).resize((W, H), Image.BICUBIC)) for f in frames])


def random_frames(n, h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, size=(n, h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize("w,h,W,H", SIZES)
def test_host_taps_reproduce_pil(w, h, W, H):
    x = random_frames(2, h, w, seed=w * 7 + h)
    x[1] = np.where(x[1] > 127, 255, 0)                 # hard edges: the negative lobes push sums past 0 and 255
    got = resize_like_kernel(x, W, H)
    want = pil_resize(x, W, H)
    assert got.shape == want.shape == (2, H, W, 3)
    assert np.array_equal(got, want), int(np.abs(got.astype(int) - want.astype(int)).max())


def test_taps_layout():
    """bounds hold (first source index, tap count) inside the source, taps are zero past each count and every row
    sums to 2^22 up to the rounding of its taps."""
    for n_in, n_out in ((1024, 1280), (576, 720), (3000, 7), (1, 5)):
        b, t = ops.bicubic_taps(n_in, n_out)
        b, t = b.numpy(), t.numpy()
        assert b.shape == (n_out, 2) and t.shape[0] == n_out and t.shape[1] == b[:, 1].max()
        assert (b[:, 0] >= 0).all() and (b[:, 1] >= 1).all() and (b.sum(1) <= n_in).all()
        assert all((t[i, b[i, 1]:] == 0).all() for i in range(n_out))
        assert (np.abs(t.sum(1).astype(np.int64) - (1 << 22)) <= b[:, 1]).all()
