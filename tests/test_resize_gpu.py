"""GPU: `ops.resize_bicubic_u8` (csrc/resize.cu) equals `PIL.Image.resize` with BICUBIC byte for byte on the size
table of tests/test_resize.py and on a 100-frame batch at the reference's 1024x576 -> 1280x720; malformed input
raises ValueError before anything is launched."""
import numpy as np
import pytest
import torch

from test_resize import SIZES, pil_resize, random_frames

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("w,h,W,H", SIZES)
def test_resize_matches_pil(cuda_dev, w, h, W, H):
    from streamingt2v_b200 import ops
    x = random_frames(3, h, w, seed=w * 11 + h)
    x[2] = np.where(x[2] > 127, 255, 0)
    got = ops.resize_bicubic_u8(torch.from_numpy(x).to(cuda_dev), W, H)
    torch.cuda.synchronize()
    want = pil_resize(x, W, H)
    assert got.shape == (3, H, W, 3) and got.dtype == torch.uint8 and got.device == cuda_dev
    g = got.cpu().numpy()
    assert np.array_equal(g, want), int(np.abs(g.astype(int) - want.astype(int)).max())


def test_resize_100_frames_matches_pil(cuda_dev):
    from streamingt2v_b200 import ops
    x = random_frames(100, 576, 1024, seed=100)
    x[::7] = np.where(x[::7] > 127, 255, 0)
    got = ops.resize_bicubic_u8(torch.from_numpy(x).to(cuda_dev), 1280, 720).cpu().numpy()
    want = pil_resize(x, 1280, 720)
    assert np.array_equal(got, want), int(np.abs(got.astype(int) - want.astype(int)).max())


def test_resize_non_contiguous_and_empty(cuda_dev):
    from streamingt2v_b200 import ops
    x = random_frames(4, 23, 37, seed=4)
    xd = torch.from_numpy(x).to(cuda_dev)
    got = ops.resize_bicubic_u8(xd[::2], 64, 48).cpu().numpy()
    assert np.array_equal(got, pil_resize(x[::2], 64, 48))
    assert ops.resize_bicubic_u8(xd[:0], 64, 48).shape == (0, 48, 64, 3)


def test_resize_rejects_malformed_input(cuda_dev):
    from streamingt2v_b200 import ops
    good = torch.zeros((2, 8, 8, 3), dtype=torch.uint8, device=cuda_dev)
    bad_inputs = [
        good.float(),                                          # not uint8
        good[..., :1].contiguous(),                            # one channel
        torch.zeros((2, 8, 8, 4), dtype=torch.uint8, device=cuda_dev),
        good[0],                                               # [H, W, 3] without the frame axis
        good.cpu(),                                            # host tensor
        good.cpu().numpy(),                                    # not a tensor
        torch.zeros((2, 0, 8, 3), dtype=torch.uint8, device=cuda_dev),
    ]
    for x in bad_inputs:
        with pytest.raises(ValueError):
            ops.resize_bicubic_u8(x, 16, 16)
    for W, H in ((0, 16), (16, -1), (16.0, 16), ("16", 16), (None, 16)):
        with pytest.raises(ValueError):
            ops.resize_bicubic_u8(good, W, H)
