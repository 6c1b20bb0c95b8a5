"""The interpolation stage at the 720x1280 geometry it runs at: a census of the launches one B200VFI._predict makes,
every GEMM launch of that census replayed at its real shape against float64, and the csrc/vfi.cu kernels at the
network's shapes and edges, all in NaN guard bands; plus B200VFI and interpolate_video against the 720x1280 golden.

Census.  CENSUS is the literal list of distinct launches (tests/vfi_census.py states the record layouts);
test_census_matches_vfi_py recomputes it on the CPU (the network on the `meta` device with shape-only ops), so a
launch shape added to vfi.py fails here until it is added to the table, and with it to the replays below.

GEMM bound (tests/gemm_replay.py, which the denoiser's replays share).  Operands are bf16, so every product x*w is
exact in fp32; the kernel sums n = K * taps of them (plus the bias) in fp32.  Each addition rounds by at most 2^-24 relative, so the sum is within gamma_n S, gamma_n = n 2^-24 /
(1 - n 2^-24) <= n 2^-23, of the exact one, S = sum |x| |w| + |bias| (a second float64 launch on |x|, |w|).  The
epilogue adds a few roundings more (bias, PReLU multiply, residual add: 4 more terms of 2^-23 S, the residual's
magnitude added to S), and a PReLU slope a scales the negative side by |a|.  The bf16 store rounds to nearest, 2^-8
relative (fp32 stores: 2^-23 with the epilogue's rounding):
    |out - ref| <= 2^-8 |ref| + (K taps + 4) 2^-23 max(1, |a|) S        (bf16 outputs; 2^-23 |ref| for fp32)
and, as guard_bands._check_bound requires, relative L2 <= 2^-8.  The float64 references run on the device
(torch conv2d / conv_transpose2d / matmul): a CPU im2col of these sizes would not fit in memory.

Every GEMM replay runs twice (and the staged, activation-free ones once per forced consumer schedule and once at the
default) and requires bitwise-equal outputs.  Each case frees its tensors before the next: the GPU is shared."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gemm_replay import bits, free, gemm_bound, launch, ref_gemm, replay
from guard_bands import Guarded, _check_bound
from vfi_census import GEMM_OPS, census
from vfi_refs import ref_warp, ref_window_attn

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL_FACTOR = 4.0          # as tests/test_vfi_gpu.py: x the reference's own bf16-autocast discrepancy

# fmt: off
CENSUS = [
    ('vfi_pair_input', (720, 1280)),
    ('conv3x3', (4, 720, 1280, 8), 8, (9, 32, 8), 4, False, True, 0, (3686400, 32), 32, 0, ()),
    ('conv3x3', (4, 720, 1280, 32), 32, (9, 32, 32), 4, False, True, 0, (3686400, 32), 32, 0, ()),
    ('conv3x3_s2', (4, 720, 1280, 32), 32, (9, 64, 32), 4, False, True, 0, (921600, 64), 64, 0, ()),
    ('conv3x3', (4, 360, 640, 64), 64, (9, 64, 64), 4, False, True, 0, (921600, 64), 64, 0, ()),
    ('conv3x3_s2', (4, 360, 640, 64), 64, (9, 128, 64), 4, False, True, 0, (230400, 128), 128, 0, ()),
    ('conv3x3', (4, 180, 320, 128), 128, (9, 128, 128), 4, False, True, 0, (230400, 128), 128, 0, ()),
    ('conv3x3_s2', (4, 180, 320, 128), 128, (9, 32, 128), 0, False, False, 0, (57600, 32), 224, 0, ()),
    ('conv3x3_strided', (4, 360, 640, 64), 64, (9, 32, 64), 0, False, False, 0, (57600, 32), 224, 32, (4, 1)),
    ('conv3x3_strided', (4, 360, 640, 64), 64, (9, 32, 64), 0, False, False, 0, (57600, 32), 224, 64, (4, 2)),
    ('conv3x3_strided', (4, 720, 1280, 32), 32, (9, 32, 32), 0, False, False, 0, (57600, 32), 224, 96, (8, 1)),
    ('conv3x3_strided', (4, 720, 1280, 32), 32, (9, 32, 32), 0, False, False, 0, (57600, 32), 224, 128, (8, 2)),
    ('conv3x3_strided', (4, 720, 1280, 32), 32, (9, 32, 32), 0, False, False, 0, (57600, 32), 224, 160, (8, 3)),
    ('conv3x3_strided', (4, 720, 1280, 32), 32, (9, 32, 32), 0, False, False, 0, (57600, 32), 224, 192, (8, 4)),
    ('linear', (57600, 224), 224, (1, 256, 224), 0, False, False, 0, (57600, 256), 256, 0, ()),
    ('layer_norm', (57600, 256), 256, 256, 1e-05),
    ('layer_norm', (57601, 256), 256, 256, 1e-06),
    ('linear', (57601, 256), 256, (1, 768, 256), 0, False, False, 0, (57601, 768), 768, 0, ()),
    ('linear', (14401, 8), 8, (1, 64, 8), 0, False, False, 0, (14401, 64), 64, 0, ()),
    ('vfi_window_attn', 2, 90, 160, 8, 0, 768, 64, 256, 64, 0),
    ('linear', (57600, 256), 256, (1, 256, 256), 0, False, False, 256, (57600, 256), 256, 0, ()),
    ('linear', (57600, 64), 64, (1, 64, 64), 0, False, False, 0, (57600, 64), 256, 0, ()),
    ('layer_norm', (57600, 256), 256, 256, 1e-06),
    ('linear', (57600, 256), 256, (1, 1024, 256), 0, False, False, 0, (57600, 1024), 1024, 0, ()),
    ('vfi_dwconv_gelu', (4, 90, 160, 1024)),
    ('linear', (57600, 1024), 1024, (1, 256, 1024), 0, False, False, 256, (57600, 256), 256, 0, ()),
    ('vfi_window_attn', 2, 90, 160, 8, 3, 768, 64, 256, 64, 0),
    ('linear', (57600, 64), 64, (1, 64, 64), 0, False, False, 0, (57600, 64), 256, 64, ()),
    ('linear', (57600, 64), 64, (1, 64, 64), 0, False, False, 0, (57600, 64), 256, 128, ()),
    ('linear', (57600, 64), 64, (1, 64, 64), 0, False, False, 0, (57600, 64), 256, 192, ()),
    ('conv3x3_s2', (4, 90, 160, 256), 256, (9, 512, 256), 0, False, False, 0, (14400, 512), 512, 0, ()),
    ('layer_norm', (14400, 512), 512, 512, 1e-05),
    ('layer_norm', (14401, 512), 512, 512, 1e-06),
    ('linear', (14401, 512), 512, (1, 1536, 512), 0, False, False, 0, (14401, 1536), 1536, 0, ()),
    ('linear', (3601, 8), 8, (1, 128, 8), 0, False, False, 0, (3601, 128), 128, 0, ()),
    ('vfi_window_attn', 2, 45, 80, 16, 0, 1536, 128, 512, 128, 0),
    ('linear', (14400, 512), 512, (1, 512, 512), 0, False, False, 512, (14400, 512), 512, 0, ()),
    ('linear', (14400, 128), 128, (1, 128, 128), 0, False, False, 0, (14400, 128), 512, 0, ()),
    ('layer_norm', (14400, 512), 512, 512, 1e-06),
    ('linear', (14400, 512), 512, (1, 2048, 512), 0, False, False, 0, (14400, 2048), 2048, 0, ()),
    ('vfi_dwconv_gelu', (4, 45, 80, 2048)),
    ('linear', (14400, 2048), 2048, (1, 512, 2048), 0, False, False, 512, (14400, 512), 512, 0, ()),
    ('vfi_window_attn', 2, 45, 80, 16, 3, 1536, 128, 512, 128, 0),
    ('linear', (14400, 128), 128, (1, 128, 128), 0, False, False, 0, (14400, 128), 512, 128, ()),
    ('linear', (14400, 128), 128, (1, 128, 128), 0, False, False, 0, (14400, 128), 512, 256, ()),
    ('linear', (14400, 128), 128, (1, 128, 128), 0, False, False, 0, (14400, 128), 512, 384, ()),
    ('vfi_head_gather', (14400, 512), 512, 512, 2, 45, 80, 136, 0),
    ('vfi_resize', (2, 3, 720, 1280), ((2764800, 921600, 1280, 1), 0, 11059200), 'bfloat16', ((7833600, 1, 43520, 136), 128, 15667200), -2, 1.0, False),
    ('vfi_resize', (2, 3, 720, 1280), ((2764800, 921600, 1280, 1), 5529600, 11059200), 'bfloat16', ((7833600, 1, 43520, 136), 131, 15667200), -2, 1.0, False),
    ('conv3x3', (2, 180, 320, 136), 136, (9, 128, 136), 4, False, True, 0, (115200, 128), 128, 0, ()),
    ('conv3x3', (2, 180, 320, 128), 128, (9, 128, 128), 4, False, True, 0, (115200, 128), 128, 0, ()),
    ('conv3x3', (2, 180, 320, 128), 128, (9, 5, 128), 4, True, True, 0, (115200, 5), 5, 0, ()),
    ('vfi_resize', (2, 4, 180, 320), ((288000, 1, 1600, 5), 0, 576000), 'float32', ((4608000, 921600, 1280, 1), 0, 9216000), 2, 4.0, False),
    ('vfi_resize', (2, 1, 180, 320), ((288000, 1, 1600, 5), 4, 576000), 'float32', ((4608000, 921600, 1280, 1), 3686400, 9216000), 2, 1.0, False),
    ('vfi_warp', (2, 3, 720, 1280), 'float32', ((2764800, 921600, 1280, 1), 0, 11059200), ((4608000, 921600, 1280, 1), 0, 9216000), 'float32', ((2764800, 921600, 1280, 1), 0, 5529600)),
    ('vfi_warp', (2, 3, 720, 1280), 'float32', ((2764800, 921600, 1280, 1), 5529600, 11059200), ((4608000, 921600, 1280, 1), 1843200, 9216000), 'float32', ((2764800, 921600, 1280, 1), 0, 5529600)),
    ('vfi_head_gather', (57600, 256), 256, 256, 2, 90, 160, 88, 0),
    ('vfi_resize', (2, 3, 720, 1280), ((2764800, 921600, 1280, 1), 0, 11059200), 'bfloat16', ((20275200, 1, 56320, 88), 64, 40550400), -1, 1.0, False),
    ('vfi_resize', (2, 3, 720, 1280), ((2764800, 921600, 1280, 1), 5529600, 11059200), 'bfloat16', ((20275200, 1, 56320, 88), 67, 40550400), -1, 1.0, False),
    ('vfi_resize', (2, 3, 720, 1280), ((2764800, 921600, 1280, 1), 0, 5529600), 'bfloat16', ((20275200, 1, 56320, 88), 70, 40550400), -1, 1.0, False),
    ('vfi_resize', (2, 3, 720, 1280), ((2764800, 921600, 1280, 1), 0, 5529600), 'bfloat16', ((20275200, 1, 56320, 88), 73, 40550400), -1, 1.0, False),
    ('vfi_resize', (2, 1, 720, 1280), ((4608000, 921600, 1280, 1), 3686400, 9216000), 'bfloat16', ((20275200, 1, 56320, 88), 76, 40550400), -1, 1.0, False),
    ('vfi_resize', (2, 4, 720, 1280), ((4608000, 921600, 1280, 1), 0, 9216000), 'bfloat16', ((20275200, 1, 56320, 88), 77, 40550400), -1, 0.5, False),
    ('conv3x3', (2, 360, 640, 88), 88, (9, 128, 88), 4, False, True, 0, (460800, 128), 128, 0, ()),
    ('conv3x3', (2, 360, 640, 128), 128, (9, 128, 128), 4, False, True, 0, (460800, 128), 128, 0, ()),
    ('conv3x3', (2, 360, 640, 128), 128, (9, 5, 128), 4, True, True, 0, (460800, 5), 5, 0, ()),
    ('vfi_resize', (2, 4, 360, 640), ((1152000, 1, 3200, 5), 0, 2304000), 'float32', ((4608000, 921600, 1280, 1), 0, 9216000), 1, 2.0, True),
    ('vfi_resize', (2, 1, 360, 640), ((1152000, 1, 3200, 5), 4, 2304000), 'float32', ((4608000, 921600, 1280, 1), 3686400, 9216000), 1, 1.0, True),
    ('nchw_to_nhwc', (2, 3, 720, 1280), (2764800, 921600, 1280, 1), 88, 0),
    ('nchw_to_nhwc', (2, 3, 720, 1280), (2764800, 921600, 1280, 1), 88, 3),
    ('nchw_to_nhwc', (2, 3, 720, 1280), (2764800, 921600, 1280, 1), 88, 6),
    ('nchw_to_nhwc', (2, 3, 720, 1280), (2764800, 921600, 1280, 1), 88, 9),
    ('nchw_to_nhwc', (2, 1, 720, 1280), (4608000, 921600, 1280, 1), 88, 12),
    ('nchw_to_nhwc', (2, 4, 720, 1280), (4608000, 921600, 1280, 1), 88, 13),
    ('vfi_warp', (2, 32, 720, 1280), 'bfloat16', ((29491200, 1, 40960, 32), 0, 117964800), ((4608000, 921600, 1280, 1), 0, 9216000), 'bfloat16', ((81100800, 1, 112640, 88), 17, 162201600)),
    ('vfi_warp', (2, 32, 720, 1280), 'bfloat16', ((29491200, 1, 40960, 32), 58982400, 117964800), ((4608000, 921600, 1280, 1), 1843200, 9216000), 'bfloat16', ((81100800, 1, 112640, 88), 49, 162201600)),
    ('vfi_resize', (2, 4, 720, 1280), ((4608000, 921600, 1280, 1), 0, 9216000), 'float32', ((921600, 230400, 640, 1), 0, 1843200), -1, 0.5, False),
    ('vfi_warp', (2, 64, 360, 640), 'bfloat16', ((14745600, 1, 40960, 64), 0, 58982400), ((921600, 230400, 640, 1), 0, 1843200), 'bfloat16', ((58982400, 1, 163840, 256), 128, 117964800)),
    ('vfi_warp', (2, 64, 360, 640), 'bfloat16', ((14745600, 1, 40960, 64), 29491200, 58982400), ((921600, 230400, 640, 1), 460800, 1843200), 'bfloat16', ((58982400, 1, 163840, 256), 192, 117964800)),
    ('vfi_resize', (2, 4, 360, 640), ((921600, 230400, 640, 1), 0, 1843200), 'float32', ((230400, 57600, 320, 1), 0, 460800), -1, 0.5, False),
    ('vfi_warp', (2, 128, 180, 320), 'bfloat16', ((7372800, 1, 40960, 128), 0, 29491200), ((230400, 57600, 320, 1), 0, 460800), 'bfloat16', ((29491200, 1, 163840, 512), 256, 58982400)),
    ('vfi_warp', (2, 128, 180, 320), 'bfloat16', ((7372800, 1, 40960, 128), 14745600, 29491200), ((230400, 57600, 320, 1), 115200, 460800), 'bfloat16', ((29491200, 1, 163840, 512), 384, 58982400)),
    ('vfi_resize', (2, 4, 180, 320), ((230400, 57600, 320, 1), 0, 460800), 'float32', ((57600, 14400, 160, 1), 0, 115200), -1, 0.5, False),
    ('vfi_warp', (2, 256, 90, 160), 'bfloat16', ((3686400, 1, 40960, 256), 0, 14745600), ((57600, 14400, 160, 1), 0, 115200), 'bfloat16', ((14745600, 1, 163840, 1024), 512, 29491200)),
    ('vfi_warp', (2, 256, 90, 160), 'bfloat16', ((3686400, 1, 40960, 256), 7372800, 14745600), ((57600, 14400, 160, 1), 28800, 115200), 'bfloat16', ((14745600, 1, 163840, 1024), 768, 29491200)),
    ('vfi_resize', (2, 4, 90, 160), ((57600, 14400, 160, 1), 0, 115200), 'float32', ((14400, 3600, 80, 1), 0, 28800), -1, 0.5, False),
    ('vfi_warp', (2, 512, 45, 80), 'bfloat16', ((1843200, 1, 40960, 512), 0, 7372800), ((14400, 3600, 80, 1), 0, 28800), 'bfloat16', ((7372800, 1, 163840, 2048), 1024, 14745600)),
    ('vfi_warp', (2, 512, 45, 80), 'bfloat16', ((1843200, 1, 40960, 512), 3686400, 7372800), ((14400, 3600, 80, 1), 7200, 28800), 'bfloat16', ((7372800, 1, 163840, 2048), 1536, 14745600)),
    ('conv3x3_s2', (2, 720, 1280, 88), 88, (9, 128, 88), 4, False, True, 0, (460800, 128), 128, 0, ()),
    ('conv3x3', (2, 360, 640, 128), 128, (9, 128, 128), 4, False, True, 0, (460800, 128), 256, 0, ()),
    ('conv3x3_s2', (2, 360, 640, 256), 256, (9, 256, 256), 4, False, True, 0, (115200, 256), 256, 0, ()),
    ('conv3x3', (2, 180, 320, 256), 256, (9, 256, 256), 4, False, True, 0, (115200, 256), 512, 0, ()),
    ('conv3x3_s2', (2, 180, 320, 512), 512, (9, 512, 512), 4, False, True, 0, (28800, 512), 512, 0, ()),
    ('conv3x3', (2, 90, 160, 512), 512, (9, 512, 512), 4, False, True, 0, (28800, 512), 1024, 0, ()),
    ('conv3x3_s2', (2, 90, 160, 1024), 1024, (9, 1024, 1024), 4, False, True, 0, (7200, 1024), 1024, 0, ()),
    ('conv3x3', (2, 45, 80, 1024), 1024, (9, 1024, 1024), 4, False, True, 0, (7200, 1024), 2048, 0, ()),
    ('copy2d', (28800, 512), 1024, 1024, 512),
    ('conv_transpose4x4_s2', (2, 45, 80, 2048), 2048, (4, 4, 512, 2048), 4, False, True, 0, (28800, 512), 1024, 0, ()),
    ('copy2d', (115200, 256), 512, 512, 256),
    ('conv_transpose4x4_s2', (2, 90, 160, 1024), 1024, (4, 4, 256, 1024), 4, False, True, 0, (115200, 256), 512, 0, ()),
    ('copy2d', (460800, 128), 256, 256, 128),
    ('conv_transpose4x4_s2', (2, 180, 320, 512), 512, (4, 4, 128, 512), 4, False, True, 0, (460800, 128), 256, 0, ()),
    ('conv_transpose4x4_s2', (2, 360, 640, 256), 256, (4, 4, 64, 256), 4, False, True, 0, (1843200, 64), 64, 0, ()),
    ('conv3x3', (2, 720, 1280, 64), 64, (9, 3, 64), 0, True, False, 0, (1843200, 3), 3, 0, ()),
    ('vfi_merge', (720, 1280), 3, True, False),
]
# fmt: on


def test_census_matches_vfi_py():
    """CPU: the distinct launches of one 720x1280 _predict are exactly CENSUS, in call order."""
    distinct, counts = census(720, 1280)
    assert distinct == CENSUS, "vfi.py's launches changed: update CENSUS (and its replays) from tests/vfi_census.py"
    assert sum(1 for c in distinct if c[0] in GEMM_OPS) == len(GEMM)
    assert sum(counts.values()) == 163


GEMM = [c for c in CENSUS if c[0] in GEMM_OPS]


# ---------------------------------------------------------------------------------------------------------------------
# every GEMM launch of the census
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(len(GEMM)), ids=[f"{i:02d}-{c[0]}-{'x'.join(map(str, c[1]))}-n{c[8][1]}"
                                                       f"-ld{c[9]}-col{c[10]}" for i, c in enumerate(GEMM)])
def test_gemm_launch_fp64(cuda_dev, idx):
    from streamingt2v_b200._lib import ACT_PRELU
    from streamingt2v_b200.vfi import pack_deconv
    op, xs, xld, ws, act, f32, prelu, res_ld, os_, old, col, extra = GEMM[idx]
    assert xld == xs[-1], "census inputs are contiguous"
    dev = cuda_dev
    g = torch.Generator(device=dev).manual_seed(1000 + idx)
    rows, n = os_
    taps = 1 if op == "linear" else (4 if op == "conv_transpose4x4_s2" else 9)
    K = xs[-1]
    X = Guarded(xs, torch.bfloat16, dev, flat=True).fill(torch.randn(xs, generator=g, device=dev))
    if op == "conv_transpose4x4_s2":
        wt = (torch.randn((K, n, 4, 4), generator=g, device=dev) / (4 * K) ** 0.5).to(torch.bfloat16).double()
        w = pack_deconv(wt.cpu(), dev)
    else:
        w = (torch.randn(ws, generator=g, device=dev) / (taps * K) ** 0.5).to(torch.bfloat16).contiguous()
        wt = w[0].double() if op == "linear" else w.double().view(3, 3, n, K).permute(2, 3, 0, 1)
    b = torch.randn((n,), generator=g, device=dev) * 0.1
    epi = dict(out_fp32=f32)
    if prelu:
        assert act == ACT_PRELU
        a = torch.randn((n,), generator=g, device=dev) * 0.5        # negative and positive slopes ...
        a[::3] = 0.0                                                # ... and zero ones
        epi.update(act=ACT_PRELU, slope=a.contiguous())
    if res_ld:
        assert res_ld == n
        res = torch.randn((rows, n), generator=g, device=dev).to(torch.bfloat16)
        epi.update(res1=res)
    O = Guarded(os_, torch.float32 if f32 else torch.bfloat16, dev, pre=16, post=16, ld=old, col=col)
    if op == "conv_transpose4x4_s2" and old > n:
        # the skip half of the concat, written before the deconv by copy2d, must come through bitwise
        O.buf[16:16 + rows, n:2 * n] = torch.randn((rows, n), generator=g, device=dev).to(O.dtype)
    O.snapshot()
    out = replay(lambda: launch(op, X.view, w, b, O.view, extra, epi), O, f"{op} {xs}",
                 schedules=(None,) if prelu else (0, 1, None))
    x64 = X.view.double()
    v = ref_gemm(op, x64, wt, extra) + b.double()
    s_abs = ref_gemm(op, x64.abs(), wt.abs(), extra) + b.double().abs()
    del x64
    amp = 1.0
    if prelu:
        a64 = a.double()
        ref = torch.where(v > 0, v, a64 * v)
        amp = a64.abs().clamp_min(1.0)
    else:
        ref = v
    if res_ld:
        ref = ref + res.double()
        s_abs = s_abs + res.double().abs()
    bound = gemm_bound(ref, s_abs, K * taps, f32, amp)
    _check_bound(out, ref, bound, f"{op} {xs}->{n} ld{old} col{col}", f"gemm {op}{' prelu' if prelu else ''}")
    del v, s_abs, ref, bound, out, X, O
    free()


# ---------------------------------------------------------------------------------------------------------------------
# window attention
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("h,w,heads,shift,pad,sharp", [
    (45, 80, 16, 0, 0, False), (45, 80, 16, 3, 0, False), (90, 160, 8, 0, 0, False), (90, 160, 8, 3, 0, False),
    (45, 80, 16, 3, 8, False), (90, 160, 8, 0, 16, False), (45, 80, 16, 3, 0, True), (90, 160, 8, 3, 0, True)])
def test_window_attn_production(cuda_dev, h, w, heads, shift, pad, sharp):
    """The network's grids (45x80 padded by 4 and 4 with centre offset 2; 90x160 padded by 1 at the bottom / right),
    its row strides or wider ones (`pad` extra columns on every leading dim), out and motion in NaN guard bands:
    padding tokens are never written.  sharp: q, k scaled so logits reach about +-150, where a key behind the
    additive -100 mask can still win."""
    from streamingt2v_b200 import ops
    dev = cuda_dev
    g = torch.Generator(device=dev).manual_seed(h * 10 + shift + pad + sharp)
    pairs, C, Cm = 2, heads * 32, heads * 8
    T = 2 * pairs * h * w
    qkv_buf = torch.full((T + 1, 3 * C + pad), float("nan"), dtype=torch.bfloat16, device=dev)
    qkv = qkv_buf[:, :3 * C]
    vals = torch.randn((T + 1, 3 * C), generator=g, device=dev)
    if sharp:
        vals[:, :2 * C] *= 6.0
    qkv.copy_(vals)
    ce_buf = torch.full((h * w + 1, Cm + pad), float("nan"), dtype=torch.bfloat16, device=dev)
    ce = ce_buf[:, :Cm]
    ce.copy_(torch.randn((h * w + 1, Cm), generator=g, device=dev))
    O = Guarded((T, C), torch.bfloat16, dev, ld=C + pad).snapshot()
    M = Guarded((T, Cm), torch.bfloat16, dev, ld=Cm + pad).snapshot()
    outs = []
    for _ in range(2):
        ops.vfi_window_attn(qkv, ce, pairs=pairs, h=h, w=w, heads=heads, shift=shift, out=O.view, motion=M.view)
        torch.cuda.synchronize()
        O.check("attn@v")
        M.check("motion")
        outs.append((O.view.clone(), M.view.clone()))
    assert all(torch.equal(bits(a), bits(b)) for a, b in zip(outs[0], outs[1])), "reruns differ bitwise"
    rx, rm = ref_window_attn(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], ce, pairs, h, w, heads, shift)
    # fp32 logits: 32 products summed, |error| <= 32 2^-23 sum|q||k| scale + one rounding; a logit error e moves
    # softmax-weighted sums of v by at most 2 e max|v|
    q, k = qkv[:, :C].double().abs(), qkv[:, C:2 * C].double().abs()
    e = (34 * 2.0 ** -23) * 32 * q.max().item() * k.max().item() * 32 ** -0.5
    for got, ref, vmax, name in ((outs[0][0], rx, qkv[:, 2 * C:].double().abs().max().item(), "attn@v"),
                                 (outs[0][1], rm, ce.double().abs().max().item(), "motion")):
        bound = 2.0 ** -8 * ref.abs() + 2e-4 * (1 + ref.abs()) + 2 * e * vmax
        _check_bound(got, ref, bound, f"{h}x{w} heads{heads} shift{shift} pad{pad} sharp{sharp} {name}",
                     "window_attn", l2=2 ** -7)
    free()


# ---------------------------------------------------------------------------------------------------------------------
# warp
# ---------------------------------------------------------------------------------------------------------------------
WARPS = [c for c in CENSUS if c[0] == "vfi_warp"]
GUARD = 64          # NaN elements before and after every strided buffer


def _strided(layout, shape, dtype, dev, values=None):
    """A view with the census layout (strides, offset, buffer elements) in a NaN buffer with GUARD elements on each
    side, optionally filled.  Returns (buffer, view)."""
    stride, off, numel = layout
    buf = torch.full((numel + 2 * GUARD,), float("nan"), dtype=dtype, device=dev)
    view = buf.as_strided(shape, stride, off + GUARD)
    if values is not None:
        view.copy_(values)
    return buf, view


def _check_strided(buf, snap, view, name):
    """Inside the view: finite.  Everywhere else in the buffer: bitwise what it was at the snapshot."""
    assert torch.isfinite(view).all(), f"{name}: unwritten or non-finite output elements"
    inside = torch.zeros(buf.shape, dtype=torch.bool, device=buf.device)
    inside.as_strided(view.shape, view.stride(), view.storage_offset()).fill_(True)
    n_bad = (bits(buf)[~inside] != bits(snap)[~inside]).sum().item()
    assert n_bad == 0, f"{name}: {n_bad} elements outside the output view were written"


def _edge_flows(n, h, w, dev, g):
    """Flows in five bands of rows: random up to 1.5 image sizes (sub-pixel in its first rows); landing exactly on
    x = w - 1 and y = h - 1; whole-pixel shifts; -0.0; far outside the image (+-1e4 pixels)."""
    f = torch.empty((n, 2, h, w), dtype=torch.float32, device=dev)
    band = (torch.arange(h, device=dev) * 5 // h).view(1, h, 1).expand(n, h, w)
    xs = torch.arange(w, device=dev, dtype=torch.float32).view(1, 1, w).expand(n, h, w)
    ys = torch.arange(h, device=dev, dtype=torch.float32).view(1, h, 1).expand(n, h, w)
    rnd = (torch.rand((n, 2, h, w), generator=g, device=dev) - 0.5) * torch.tensor([3.0 * w, 3.0 * h], device=dev
                                                                                     ).view(1, 2, 1, 1)
    rnd[:, :, :max(1, h // 20)] *= 0.001
    ints = torch.randint(-3, 4, (n, 2, h, w), generator=g, device=dev).float()
    far = torch.where(torch.rand((n, 2, h, w), generator=g, device=dev) < 0.5, -1e4, 1e4)
    for c, edge in ((0, (w - 1) - xs), (1, (h - 1) - ys)):
        f[:, c] = torch.where(band == 0, rnd[:, c], torch.where(band == 1, edge, torch.where(
            band == 2, ints[:, c], torch.where(band == 3, torch.full_like(xs, -0.0), far[:, c]))))
    return f


@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(len(WARPS)), ids=[f"{c[2]}-c{c[1][1]}-{c[1][2]}x{c[1][3]}-in{c[3][1]}-flow{c[4][1]}"
                                                        f"-out{c[6][1]}" for c in WARPS])
def test_warp_production(cuda_dev, idx):
    """Every warp of the census with its operands where the network has them: fp32 frames at 720x1280 (the second
    pair's images at their offset in the TTA batch) and bf16 channel-last features at every UNet level (c = 32 ...
    512, down to 45x80, the second image pair's rows) written into their column slices of the skip concat; the flow
    a channel slice of the flow / mask buffer (x1's flow at channel 2), holding the edge flows of _edge_flows."""
    from streamingt2v_b200 import ops
    from vfi_refs import warp_bound
    _, (n, c, h, w), idt, il, fl, odt, ol = WARPS[idx]
    dev = cuda_dev
    g = torch.Generator(device=dev).manual_seed(77 + idx)
    dt = {"bfloat16": torch.bfloat16, "float32": torch.float32}
    _, flow = _strided(fl, (n, 2, h, w), torch.float32, dev, _edge_flows(n, h, w, dev, g))
    _, xin = _strided(il, (n, c, h, w), dt[idt], dev, torch.rand((n, c, h, w), generator=g, device=dev))
    obuf, out = _strided(ol, (n, c, h, w), dt[odt], dev)
    snap = obuf.clone()
    outs = []
    for _ in range(2):
        ops.vfi_warp(xin, flow, out)
        torch.cuda.synchronize()
        _check_strided(obuf, snap, out, "warp")
        outs.append(out.clone())
    assert torch.equal(bits(outs[0]), bits(outs[1]))
    ref = ref_warp(xin, flow)
    _check_bound(outs[0], ref, warp_bound(ref, flow, odt == "bfloat16"),
                 f"{n}x{c}x{h}x{w} {odt} in+{il[1]} flow+{fl[1]} out+{ol[1]}", "warp")
    del outs, ref, obuf, snap
    free()


# ---------------------------------------------------------------------------------------------------------------------
# resize
# ---------------------------------------------------------------------------------------------------------------------
RESIZES = [c for c in CENSUS if c[0] == "vfi_resize"]
ODD_RESIZES = [((2, 4, 45, 80), 1), ((2, 4, 45, 80), 2), ((2, 1, 45, 81), -1), ((2, 3, 47, 83), -2),
               ((2, 4, 45, 80), -1), ((1, 5, 1, 3), 2)]


def _resize_case(dev, shape, il, odt, ol, log2, mul, acc, seed):
    from streamingt2v_b200 import ops
    n, c, h, w = shape
    f = 2.0 ** log2
    oshape = (n, c, int(h * f), int(w * f))
    g = torch.Generator(device=dev).manual_seed(seed)
    _, xin = _strided(il, shape, torch.float32, dev, torch.randn(shape, generator=g, device=dev) * 10)
    obuf, out = _strided(ol, oshape, torch.bfloat16 if odt == "bfloat16" else torch.float32, dev)
    base = torch.randn(oshape, generator=g, device=dev)
    if acc:
        out.copy_(base)
    snap = obuf.clone()
    ops.vfi_resize(xin, out, log2, mul, accumulate=acc)
    torch.cuda.synchronize()
    _check_strided(obuf, snap, out, "resize")
    ref = F.interpolate(xin.double(), scale_factor=f, mode="bilinear", align_corners=False) * mul
    if acc:
        ref = ref + base.double()
    bound = (2.0 ** -8 * ref.abs() if odt == "bfloat16" else 0) + 4e-6 * (ref.abs() + 10 * abs(mul))
    _check_bound(out, ref, bound, f"{shape} x2^{log2} mul{mul} acc{acc} {odt} in+{il[1]} out+{ol[1]}", "resize")
    del obuf, snap, ref
    free()


@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(len(RESIZES)),
                         ids=[f"{'x'.join(map(str, c[1]))}-x2^{c[5]}-{c[3]}-in{c[2][1]}-out{c[4][1]}"
                              f"{'-acc' if c[7] else ''}" for c in RESIZES])
def test_resize_production(cuda_dev, idx):
    """Every resize of the census with its operands where the network has them: 1/4 of the frames into the bf16
    columns 128..133 of the first head's input (ld 136), the 1/2 resizes into the second's (ld 88), x4 and x2
    (accumulating) of the heads' channel-last outputs (the mask channel at its offset 4) into the flow / mask
    buffer (the mask at channel 4), and the flow halving 720 -> 360 -> 180 -> 90 -> 45."""
    _, shape, il, odt, ol, log2, mul, acc = RESIZES[idx]
    _resize_case(cuda_dev, shape, il, odt, ol, log2, mul, acc, 300 + idx)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,log2", ODD_RESIZES, ids=[f"{'x'.join(map(str, s))}-x2^{k}" for s, k in ODD_RESIZES])
@pytest.mark.parametrize("acc", [False, True])
def test_resize_odd_sizes(cuda_dev, shape, log2, acc):
    """Odd inputs: the 45-row end of the flow chain scaled up by 2 and 4, and 1/2, 1/4 of sizes that are not multiples
    of the factor (the output is floor(size * factor), as F.interpolate sizes it)."""
    n, c, h, w = shape
    f = 2.0 ** log2
    ho, wo = int(h * f), int(w * f)
    il = ((c * h * w, h * w, w, 1), 0, n * c * h * w)
    ol = ((c * ho * wo, ho * wo, wo, 1), 0, n * c * ho * wo)
    _resize_case(cuda_dev, shape, il, "float32", ol, log2, 0.5 * f, acc, 400 + h + log2)


# ---------------------------------------------------------------------------------------------------------------------
# depthwise conv + GELU, head gather
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("h,w,c", [(90, 160, 1024), (45, 80, 2048)])
def test_dwconv_gelu_production(cuda_dev, h, w, c):
    from streamingt2v_b200 import ops
    dev = cuda_dev
    g = torch.Generator(device=dev).manual_seed(c + h)
    X = Guarded((4, h, w, c), torch.bfloat16, dev, flat=True).fill(torch.randn((4, h, w, c), generator=g, device=dev))
    wt = torch.randn((c, 1, 3, 3), generator=g, device=dev) / 3
    b = torch.randn((c,), generator=g, device=dev) * 0.1
    O = Guarded((4 * h * w, c), torch.bfloat16, dev, flat=True).snapshot()
    outs = []
    for _ in range(2):
        ops.vfi_dwconv_gelu(X.view, wt.reshape(c, 9).t().contiguous(), b, out=O.view)
        torch.cuda.synchronize()
        O.check("dwconv_gelu")
        outs.append(O.view.clone())
    assert torch.equal(bits(outs[0]), bits(outs[1]))
    ref = F.gelu(F.conv2d(X.view.double().permute(0, 3, 1, 2), wt.double(), b.double(), padding=1, groups=c))
    ref = ref.permute(0, 2, 3, 1).reshape(-1, c)
    # 9 fp32 fmas and the bias (a few 2^-24 of sum |x w| <= 3 max|x|), erff within 2 ulp; then one bf16 rounding
    _check_bound(outs[0], ref, 2.0 ** -8 * ref.abs() + 1e-5, f"{h}x{w}x{c}", "dwconv")
    free()


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,c,ld", [(45, 80, 512, 136), (90, 160, 256, 88)])
def test_head_gather_production(cuda_dev, h, w, c, ld):
    """pairs = 2 into the heads' inputs (ld 136 / 88); the columns after c/4 belong to the resizes and must come
    through bitwise."""
    from streamingt2v_b200 import ops
    dev = cuda_dev
    g = torch.Generator(device=dev).manual_seed(c)
    pairs = 2
    mf = torch.randn((2 * pairs * h * w, c), generator=g, device=dev).to(torch.bfloat16)
    af = torch.randn((2 * pairs * h * w, c), generator=g, device=dev).to(torch.bfloat16)
    rows = pairs * 16 * h * w
    O = Guarded((rows, c // 4), torch.bfloat16, dev, pre=16, post=16, ld=ld, col=0)
    O.buf[16:16 + rows, c // 4:] = torch.randn((rows, ld - c // 4), generator=g, device=dev).to(torch.bfloat16)
    O.snapshot()
    ops.vfi_head_gather(mf, af, pairs=pairs, h=h, w=w, out=O.view)
    torch.cuda.synchronize()
    O.check("head_gather")
    m4 = mf.double().view(2 * pairs, h, w, c).permute(0, 3, 1, 2)
    a4 = af.double().view(2 * pairs, h, w, c).permute(0, 3, 1, 2)
    cat = torch.cat([0.5 * m4[:pairs], 0.5 * m4[pairs:], a4[:pairs], a4[pairs:]], 1)
    ref = F.pixel_shuffle(F.pixel_shuffle(cat, 2), 2).permute(0, 2, 3, 1).reshape(-1, c // 4)
    assert torch.equal(O.view.double(), ref)
    free()


# ---------------------------------------------------------------------------------------------------------------------
# merge, pair input, frames to BGR
# ---------------------------------------------------------------------------------------------------------------------
def _ref_merge(w0, w1, fm, res, H, W):
    m = torch.sigmoid(fm[:, 4:5].double())
    r = torch.sigmoid(res.double().view(2, H, W, 3).permute(0, 3, 1, 2)) * 2 - 1
    p = torch.clamp(w0.double() * m + w1.double() * (1 - m) + r, 0, 1)
    return (p[0] + p[1].flip(1).flip(2)) / 2


@pytest.mark.gpu
def test_merge_720x1280(cuda_dev):
    from streamingt2v_b200 import ops
    dev = cuda_dev
    H, W = 720, 1280
    g = torch.Generator(device=dev).manual_seed(11)
    w0, w1 = (torch.rand((2, 3, H, W), generator=g, device=dev) for _ in range(2))
    fm = torch.randn((2, 5, H, W), generator=g, device=dev) * 3
    res = torch.randn((2 * H * W, 3), generator=g, device=dev) * 3
    P = Guarded((1, 3, H, W), torch.float32, dev, flat=True).snapshot()
    Fr = torch.full((H * W * 3 + 64,), 7, dtype=torch.uint8, device=dev)
    frame = Fr[16:16 + H * W * 3].view(H, W, 3)
    ops.vfi_merge(w0, w1, fm, res, pred=P.view, frame=frame)
    torch.cuda.synchronize()
    P.check("merge pred")
    assert (Fr[:16] == 7).all() and (Fr[16 + H * W * 3:] == 7).all()
    ref = _ref_merge(w0, w1, fm, res, H, W)
    # sigmoid (expf within 2 ulp) and ~8 fp32 roundings of values <= 2
    _check_bound(P.view[0], ref, torch.full_like(ref, 1e-6), "720x1280", "merge")
    ref8 = (P.view[0].cpu().numpy().transpose(1, 2, 0) * 255.0).astype(np.uint8)[:, :, ::-1]
    assert np.array_equal(frame.cpu().numpy(), ref8)
    free()


@pytest.mark.gpu
def test_merge_uint8_truncation_exact(cuda_dev):
    """pred values whose float32 product with 255 is exactly an integer k and the float32 just below it: the uint8
    frame is numpy's (pred * 255.0).astype(uint8) bit for bit.  mask logit 100 (sigmoid == 1 in fp32) and refinement
    0 (2 sigmoid(0) - 1 == 0) make pred == warped0 exactly, the flipped copy holds the same values mirrored."""
    from streamingt2v_b200 import ops
    dev = cuda_dev
    vals = []
    for k in range(256):
        t = np.float32(k / 255.0)
        vals += [t, np.nextafter(t, np.float32(-1)), np.nextafter(t, np.float32(2))]
    v = np.clip(np.array(vals, np.float32), 0, 1)
    prod = v * np.float32(255.0)
    on = prod == np.round(prod)
    below = (np.nextafter(np.ceil(prod), np.float32(0)) == prod) & ~on
    assert on.sum() >= 200 and below.sum() >= 100, (on.sum(), below.sum())
    H, W = 16, 3 * 16 * 3
    n = H * W
    grid = np.resize(v, 3 * n).reshape(3, H, W)
    w0 = torch.from_numpy(np.stack([grid, grid[:, ::-1, ::-1]])).to(dev).contiguous()
    w1 = torch.rand((2, 3, H, W), device=dev)
    fm = torch.zeros((2, 5, H, W), device=dev)
    fm[:, 4] = 100.0
    res = torch.zeros((2 * n, 3), device=dev)
    pred = torch.empty((1, 3, H, W), device=dev)
    frame = torch.empty((H, W, 3), dtype=torch.uint8, device=dev)
    ops.vfi_merge(w0, w1, fm, res, pred=pred, frame=frame)
    torch.cuda.synchronize()
    p = pred[0].cpu().numpy()
    assert np.array_equal(p.view(np.int32), grid.view(np.int32)), "pred != warped0 on the constructed inputs"
    ref8 = (p.transpose(1, 2, 0) * 255.0).astype(np.uint8)[:, :, ::-1]
    assert np.array_equal(frame.cpu().numpy(), ref8)


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(720, 1280), (16, 48)])
def test_pair_input_exact(cuda_dev, H, W):
    """imgs = [img0, flip(img0), img1, flip(img1)] bit for bit; x8 = bf16 (round to nearest even) of the three
    channels, channels 3..7 zero."""
    from streamingt2v_b200 import ops
    dev = cuda_dev
    g = torch.Generator(device=dev).manual_seed(H)
    i0, i1 = (torch.rand((1, 3, H, W), generator=g, device=dev) for _ in range(2))
    imgs = torch.full((4, 3, H, W), float("nan"), device=dev)
    X8 = Guarded((4, H, W, 8), torch.bfloat16, dev, flat=True).snapshot()
    ops.vfi_pair_input(i0, i1, imgs, X8.view)
    torch.cuda.synchronize()
    X8.check("x8")
    want = torch.cat([i0, i0.flip(2).flip(3), i1, i1.flip(2).flip(3)])
    assert torch.equal(imgs.view(torch.int32), want.view(torch.int32))
    x8 = torch.zeros((4, H, W, 8), dtype=torch.bfloat16, device=dev)
    x8[..., :3] = want.permute(0, 2, 3, 1).to(torch.bfloat16)
    assert torch.equal(X8.view.view(torch.int16), x8.view(torch.int16))


@pytest.mark.gpu
@pytest.mark.parametrize("F_,H,W", [(1, 16, 16), (3, 720, 1280)])
def test_frames_to_bgr_exact(cuda_dev, F_, H, W):
    """(float)(u / 255.0) with the channel order reversed, bit for bit: every byte value in every channel (first
    case), and a multi-frame 720x1280 batch."""
    from streamingt2v_b200 import ops
    dev = cuda_dev
    if F_ == 1:
        u = np.arange(256, dtype=np.uint8).reshape(1, 16, 16)
        fr = np.stack([u, 255 - u, (u.astype(np.int32) * 7 % 256).astype(np.uint8)], -1)
    else:
        fr = np.random.default_rng(5).integers(0, 256, (F_, H, W, 3), dtype=np.uint8)
    O = Guarded((F_, 3, H, W), torch.float32, dev, flat=True).snapshot()
    ops.vfi_frames_to_bgr(torch.from_numpy(fr).to(dev), out=O.view)
    torch.cuda.synchronize()
    O.check("frames_to_bgr")
    want = (fr / 255.0).astype(np.float32)[..., ::-1].transpose(0, 3, 1, 2)
    assert np.array_equal(O.view.cpu().numpy().view(np.int32), np.ascontiguousarray(want).view(np.int32))


# ---------------------------------------------------------------------------------------------------------------------
# the network at 720x1280 against the reference's golden (regions)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden720():
    from streamingt2v_b200 import synth
    d = dict(np.load(os.path.join(GOLDEN, "vfi_720x1280.npz")))
    h, w = int(d["height"]), int(d["width"])
    f0, f1 = synth.test_frames(h, w, int(d["seed"]) + h)
    assert synth.frames_checksum(f0, f1) == int(d["frames_crc32"]), "the seeded frames differ from the golden's"
    d["frame0"], d["frame1"] = f0, f1
    d["spec"] = dict(tile_origins=d["tile_origins"], tile=int(d["tile"]), rows=d["rows"], cols=d["cols"])
    return d


@pytest.fixture(scope="module")
def vfi_net720(cuda_dev, golden720):
    from streamingt2v_b200.vfi import B200VFI, seeded_state_dict
    sd = seeded_state_dict(int(golden720["seed"]))
    sums = np.array([float(sd[k].double().sum()) for k in golden720["weight_keys"]])
    assert np.array_equal(sums, golden720["weight_sums"]), "the seeded weights differ from the golden's"
    return B200VFI(sd, cuda_dev)


def _bgr(frame, dev):
    return torch.from_numpy((frame / 255.)[:, :, ::-1].copy()).permute(2, 0, 1)[None].float().to(dev)


@pytest.mark.gpu
def test_b200vfi_inference_golden_720x1280(cuda_dev, golden720, vfi_net720):
    from streamingt2v_b200 import synth
    d = golden720
    pred = vfi_net720.inference(_bgr(d["frame0"], cuda_dev), _bgr(d["frame1"], cuda_dev))
    torch.cuda.synchronize()
    assert torch.isfinite(pred).all()
    got = synth.crop_regions(pred[0].double().cpu().numpy(), **d["spec"])
    err = np.abs(got - d["pred_regions"].astype(np.float64))
    mean_b, max_b = float(d["bf16_mean_err"]), float(d["bf16_max_err"])
    print(f"720x1280: mean err {err.mean():.4g} ({err.mean() / mean_b:.2f} x ref bf16), max err {err.max():.4g} "
          f"({err.max() / max_b:.2f} x ref bf16)")
    assert err.mean() <= TOL_FACTOR * mean_b and err.max() <= TOL_FACTOR * max_b


@pytest.mark.gpu
def test_interpolate_video_golden_720x1280(cuda_dev, golden720, vfi_net720):
    from streamingt2v_b200 import synth
    from streamingt2v_b200.vfi import interpolate_video
    d = golden720
    video = torch.from_numpy(np.stack([d["frame0"], d["frame1"]]))
    out = interpolate_video(video, 3, vfi_net720)
    torch.cuda.synchronize()
    assert out.shape == (3, 720, 1280, 3) and out.dtype == torch.uint8
    o = out.cpu().numpy()
    assert np.array_equal(o[0], d["frame0"]) and np.array_equal(o[2], d["frame1"])
    mid = synth.crop_regions(np.ascontiguousarray(o[1].transpose(2, 0, 1)), **d["spec"])
    diff = np.abs(mid.astype(np.int32) - d["mid_regions"].astype(np.int32))
    print(f"720x1280 midpoint uint8 diff mean {diff.mean():.4f} max {diff.max()}")
    assert diff.max() <= math.ceil(255 * TOL_FACTOR * float(d["bf16_max_err"])) + 1
