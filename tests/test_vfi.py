"""CPU: host logic of the EMA-VFI stage (streamingt2v_b200/vfi.py): the configuration check, the ConvTranspose2d
phase decomposition, the window / shift / padding mask rule the window-attention kernel implements, the frame
bookkeeping of interpolate_video, and (with the reference checkout) that the goldens regenerate bit for bit."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from streamingt2v_b200 import ops, vfi

REFERENCE_VFI = "/root/reference/code/i2v_enhance/thirdparty/VFI"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_config_check_accepts_shipped_and_rejects_others():
    sd = vfi.seeded_state_dict(0)
    sd2 = dict(sd)
    sd2["feature_bone.block4.1.attn_mask"] = torch.zeros(1)      # the reference's cached buffers are ignored
    assert set(vfi.check_config(sd2)) == set(sd)
    bad = dict(sd)
    bad["feature_bone.block5.0.mlp.fc1.weight"] = torch.zeros(1024, 512)   # mlp ratio 2
    with pytest.raises(ValueError, match="fc1.weight"):
        vfi.check_config(bad)
    small = {k: v for k, v in sd.items() if not k.startswith("feature_bone.block5.3.")}   # depth 3
    with pytest.raises(ValueError, match="missing keys"):
        vfi.check_config(small)


def test_deconv_phase_identity_fp64():
    """ConvTranspose2d(4, stride 2, padding 1) == per output phase (a, b) the 4-tap stride-1 conv of
    ops.conv_transpose4x4_s2 with deconv_phase_weights, in float64."""
    g = torch.Generator().manual_seed(0)
    n, cin, cout, h, w = 2, 5, 3, 6, 7
    x = torch.randn((n, cin, h, w), generator=g, dtype=torch.float64)
    wt = torch.randn((cin, cout, 4, 4), generator=g, dtype=torch.float64)
    ref = F.conv_transpose2d(x, wt, stride=2, padding=1)
    ph = vfi.deconv_phase_weights(wt)                                      # [4, 4, cout, cin]
    xp = F.pad(x, (1, 1, 1, 1))
    out = torch.zeros_like(ref)
    for a in range(2):
        for b in range(2):
            taps = [(dy, dx) for dy, _ in ops.DECONV_PHASE_TAPS[a] for dx, _ in ops.DECONV_PHASE_TAPS[b]]
            acc = torch.zeros((n, cout, h, w), dtype=torch.float64)
            for t, (dy, dx) in enumerate(taps):
                acc += torch.einsum("nchw,oc->nohw", xp[:, :, 1 + dy:1 + dy + h, 1 + dx:1 + dx + w], ph[a * 2 + b, t])
            out[:, :, a::2, b::2] = acc
    assert torch.allclose(out, ref, rtol=0, atol=1e-12)


def _kernel_tokens(h, w, shift):
    """The window-attention kernel's per-(window, position) rule (csrc/vfi.cu vfi_win_token), restated: the source
    token (or -1 for padding) and the mask label; two positions are masked iff their labels differ."""
    hp, wp = -(-h // 7) * 7, -(-w // 7) * 7
    pt, pl = (hp - h) // 2, (wp - w) // 2
    r3 = lambda v, a, b: 0 if v < a else (1 if v < b else 2)  # noqa: E731
    nwx = wp // 7
    src = np.zeros((hp // 7 * nwx, 49), np.int64)
    lab = np.zeros_like(src)
    for win in range(src.shape[0]):
        for pos in range(49):
            Y, X = (win // nwx) * 7 + pos // 7, (win % nwx) * 7 + pos % 7
            sl, ys, xs = 0, Y, X
            if shift:
                sl = r3(Y, hp - 7, hp - shift) * 3 + r3(X, wp - 7, wp - shift)
                ys, xs = (Y + shift) % hp, (X + shift) % wp
            pad = r3(Y, pt, pt + h) * 3 + r3(X, pl, pl + w) if (hp, wp) != (h, w) else 0
            lab[win, pos] = sl * 9 + pad
            y, x = ys - pt, xs - pl
            src[win, pos] = y * w + x if 0 <= y < h and 0 <= x < w else -1
    return src, lab


def _reference_block():
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from oracle.make_golden_vfi import _install_timm
    _install_timm()
    if REFERENCE_VFI not in sys.path:
        sys.path.insert(0, REFERENCE_VFI)
    import importlib
    return importlib.import_module("model.feature_extractor")


@pytest.mark.skipif(not os.path.isdir(REFERENCE_VFI), reason="needs the reference checkout")
@pytest.mark.parametrize("h,w", [(14, 28), (12, 20), (6, 10), (7, 14), (9, 5), (90, 160), (45, 80)])
@pytest.mark.parametrize("shift", [0, 3])
def test_window_masks_match_reference(h, w, shift):
    """The kernel's token map and labels reproduce the reference's pad_if_needed + roll + window_partition and its
    -100 masks (pad mask, shift mask, and the pad mask applied unrolled in shifted blocks)."""
    fe = _reference_block()
    blk = fe.MotionFormerBlock(dim=32, motion_dim=8, num_heads=1, window_size=7, shift_size=shift).eval()
    src, lab = _kernel_tokens(h, w, shift)
    idx = torch.arange(h * w, dtype=torch.float64).view(1, h, w, 1) + 1      # 0 = padding
    x_pad, mask = fe.pad_if_needed(idx, idx.size(), (7, 7))
    if shift:
        x_pad = torch.roll(x_pad, shifts=(-shift, -shift), dims=(1, 2))
    tok = fe.window_partition(x_pad, (7, 7)).squeeze(-1).long() - 1
    assert np.array_equal(tok.numpy(), src)
    # the attention mask the block builds: run its mask code through a stub attention that records it
    seen = {}
    blk.attn.forward = lambda x1, x2, cor, H, W, mask=None: (seen.setdefault("m", mask), (torch.zeros_like(x1),) * 2)[1]
    blk.mlp.forward = lambda x, H, W: torch.zeros_like(x)
    x = torch.zeros((2, h * w, 32))
    cor = torch.zeros((2, h, w, 2))
    blk(x, cor, h, w, 1)
    m = seen["m"]
    want = (lab[:, :, None] != lab[:, None, :])
    if m is None:
        assert not want.any()
    else:
        assert np.array_equal((m != 0).numpy(), want) and set(np.unique(m.numpy())) <= {0.0, -100.0}


def test_interpolate_frame_plan():
    P = vfi.interpolate_frame_plan
    assert P(100, 200) == [x for i in range(99) for x in (("copy", i), ("mid", i))] + [("copy", 99), ("copy", 99)]
    assert len(P(100, 199)) == 199 and P(100, 199)[-1] == ("copy", 99)
    assert len(P(100, 200)) == 200
    # vfi_process keeps video[:dest // 2 + 1]
    assert P(10, 5) == [("copy", 0), ("mid", 0), ("copy", 1), ("mid", 1), ("copy", 2)]
    assert P(10, 6) == [("copy", 0), ("mid", 0), ("copy", 1), ("mid", 1), ("copy", 2), ("mid", 2), ("copy", 3),
                        ("copy", 3)]
    assert P(1, 2) == [("copy", 0), ("copy", 0)]
    with pytest.raises(ValueError):
        P(0, 4)


@pytest.mark.parametrize("frames,dest", [(5, 7), (5, 8), (9, 7), (4, 6)])
def test_interpolate_video_bookkeeping(monkeypatch, frames, dest):
    """interpolate_video with a stand-in network: pass-through frames are the inputs bit for bit, midpoint k is
    predicted from input frames (k, k + 1) (their BGR /255 tensors), in the reference's order."""
    import types
    fake_ops = types.SimpleNamespace(
        vfi_frames_to_bgr=lambda fr: (fr[..., [2, 1, 0]].double() / 255.0).float().permute(0, 3, 1, 2).contiguous())
    monkeypatch.setattr(vfi, "ops", fake_ops)

    class FakeVFI:
        dev = torch.device("cpu")

        def _predict(self, b0, b1, frame):
            # midpoint marker: 100 + index of the first frame, recovered from its pixel value
            frame.fill_(100 + int(round(float(b0[0, 0, 0, 0]) * 255)))

    g = torch.Generator().manual_seed(frames)
    video = torch.randint(0, 30, (frames, 16, 32, 3), generator=g, dtype=torch.uint8)
    video[:, 0, 0, 2] = torch.arange(frames, dtype=torch.uint8)   # R of pixel (0, 0) = frame index (B after the flip)
    out = vfi.interpolate_video(video, dest, FakeVFI())
    plan = vfi.interpolate_frame_plan(frames, dest)
    assert out.shape[0] == len(plan)
    for k, (kind, i) in enumerate(plan):
        if kind == "copy":
            assert torch.equal(out[k], video[i])
        else:
            assert int(out[k, 0, 0, 0]) == 100 + i


def test_interpolate_video_rejects_bad_sizes():
    with pytest.raises(ValueError, match="multiples of 16"):
        vfi.interpolate_video(torch.zeros((3, 100, 160, 3), dtype=torch.uint8), 5, None)


@pytest.mark.skipif(not os.path.isdir(REFERENCE_VFI), reason="needs the reference checkout")
def test_golden_regeneration_is_deterministic():
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from oracle import make_golden_vfi as m
    g = m.golden(96, 160)
    d = np.load(os.path.join(GOLDEN, "vfi_96x160.npz"))
    for k in d.files:
        assert np.array_equal(np.asarray(g[k]), d[k]), k
