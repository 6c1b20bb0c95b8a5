"""The image stages of every chunk at the geometry they run at: a census of the launches of the temporal VAE decoder
(an 8-frame group and the 1-frame tail group of a 25-frame chunk, 72x128 latents to 576x1024), the SD-VAE encoder
(one 576x1024 frame) and the OpenCLIP ViT-H/14 image tower (one image from 576x1024: 257 tokens, width 1280, 32
blocks); every GEMM launch of that census replayed at its real shape against float64, and the attention, norm and glue
launches at their census shapes, all in NaN guard bands.

Census.  CENSUS is the literal union of the four censuses (tests/vae_clip_census.py and tests/denoiser_census.py
state the record layouts), each record with its number of calls in each configuration; test_census_matches_stages
recomputes them on the CPU, so a launch added to vae.py or conditioner.py fails here until it is added to the table,
and test_every_record_is_replayed maps every record to the test that replays it.

GEMM bound (tests/gemm_replay.py, as tests/test_denoiser_launches_gpu.py states it).  gamma = (K taps + 6) 2^-23; the
accumulator is within gamma S of the exact one, S = sum |x| |w| + |bias|; then
    none   |out - ref| <= c |ref| + gamma (|s_acc| S + |s1| |res1|)
    GELU   the CLIP MLP's c_fc (ACT_GELU, no blend).  The kernel evaluates gelu_fast(pre') on the accumulator pre' =
           pre + e, |e| <= gamma S.  |gelu'| <= 1.13 everywhere (its maximum is 1.1289), so |gelu(pre') - gelu(pre)|
           <= 1.13 gamma S.  gelu_fast is x/2 + |x|/2 erf(|x|/sqrt2) with Abramowitz-Stegun 7.1.25's erf, whose
           absolute error is at most 2.5e-5 (ptx.cuh; ex2.approx and rcp.approx add about 2^-22 relative to terms
           below 1): within 1.25e-5 |pre'| < 2^-16 |pre'| of gelu(pre'); the 2^-16 gamma S of |pre'| - |pre| fits in
           the 0.001 between 1.1289 and 1.13.  So  c |ref| + 1.13 gamma S + 2^-16 |pre|
with c = 2^-8 for bf16 stores and 2^-23 for fp32 ones; relative L2 within 2^-8.  The blend weights are sigmoid(1) and
1 - sigmoid(1), not 1/2.  Every replay runs twice under consumer schedules 0, 1 and the default and under both
epilogue bodies; all twelve outputs are equal bit for bit.  Partial-width outputs (conv_out into columns 0..2 of the
8-wide y8, time_mix_conv into columns 0..2 of the fp32 o8) find the other columns of their rows filled and must
leave them bitwise unchanged.  float64 references run on the device in bands: rows of a linear, (frame, output image
rows) of a conv with its one-row halo (the pad-after stride-2 conv reads rows 2i .. 2i + 2), (video, pixel range) of a
tconv3, which pads each video separately; no band holds more than a few hundred MB, whatever algorithm torch picks.

linear_grouped (the patch embedding: K = 592, rows 1..256 of every 257-row image through out_rs) runs at the census
n = 1 and at n = 2, where the group stride 257 is used; the class-token rows 0 and 257 hold data and stay bitwise.

attention_single_head (the VAE mid-block AttnBlock, S = 9216, C = 512) at every census shape, one frame's 9216^2
score block alive at a time.  Its four launches are checked one by one: the Q K^T linear (fp32 out, s_acc = C^-1/2)
and the P V linear (K = 9216) by the GEMM replay and bound; softmax_rows against float64 on the fp32 scores it read,
with test_norm_glue_edges_gpu.py's bound (its relative part r <= 2^-8 + 2^-23 (6 + 1.7 (|x - max| + E|x - max|)) + k u,
plus 2^-126 flushed); transpose exactly.  The composite is then equal bit for bit to those parts and, against
float64 attention p = softmax(sa q k^T) (sa the fp32 scale the kernel receives), within
    |out - ref| <= 2^-8 |ref| + (1 + 2^-7) ((m - 1) + m r + m (1 + r) gamma_PV) A,   A = sum_j p_ij |v_j|
where m = exp(2 Delta_i), Delta_i = max_j of the score bound of row i (a logit error d shifts p by a factor within
exp(+-2 max d)), r the softmax's relative bound of row i, and gamma_PV = (9216 + 6) 2^-23 the P V accumulation.  The
dominant term is r's 2^-8: the bf16 rounding of P.  Relative L2 within 2^-7.  The sharp variant scales Q by 8.

Norms use test_norm_glue_edges_gpu.py's cases and bounds at every census shape not already run there (GN_NET's shapes
and test_group_norm_vae_full_resolution's two launches are).  Layout glue is exact.  flash_attn_d80 runs at the
census qkv leading dim 3 C (no pad column), with test_conditioner_gpu.py's bound; clip_preprocess's census shape is
one test_conditioner_gpu.py::test_clip_preprocess runs.  Each case frees its tensors before the next: the GPU is
shared."""
import pytest
import torch

from gemm_replay import bits, free, launch, ref_gemm, replay
from guard_bands import Guarded
from test_conditioner_gpu import _attn64
from test_denoiser_launches_gpu import AL, _chunks, _f32, _glue_case
from test_kernel_edges_gpu import _gelu
from test_norm_glue_edges_gpu import GN_NET, U, _channel_fill, _gn_case, _ln_case, _Rows, _softmax_bound
from vae_clip_census import CONFIGS, GEMM_OPS, census

# calls per run of each configuration: decode8, decode1, encode, clip
CALLS = {"decode8": 132, "decode1": 132, "encode": 56, "clip": 231}

# fmt: off
CENSUS = [
    (('nchw_to_nhwc', (8, 4, 72, 128), 36864, (73728, 8), 8, 0), (1, 0, 0, 0)),
    (('conv3x3', (8, 72, 128, 8), 8, (9, 512, 8), 0, False, True, (), 0, 0, (False, False, False), 0, (73728, 512), 512, 0), (1, 0, 0, 0)),
    (('group_norm', (73728, 512), 512, 8, 9216, 1e-06, True, 512), (10, 0, 0, 0)),
    (('conv3x3', (8, 72, 128, 512), 512, (9, 512, 512), 0, False, True, (), 0, 0, (False, False, False), 0, (73728, 512), 512, 0), (5, 0, 0, 0)),
    (('conv3x3', (8, 72, 128, 512), 512, (9, 512, 512), 0, False, True, (), 512, 0, (False, False, False), 0, (73728, 512), 512, 0), (5, 0, 0, 0)),
    (('group_norm', (73728, 512), 512, 1, 73728, 1e-05, True, 512), (10, 0, 0, 0)),
    (('tconv3', (1, 8, 9216, 512), 512, (3, 512, 512), 0, False, True, (), 0, 0, (False, False, False), 0, (73728, 512), 512, 0), (5, 0, 0, 0)),
    (('tconv3', (1, 8, 9216, 512), 512, (3, 512, 512), 0, False, True, (), 512, 0, (True, False, False), 0, (73728, 512), 512, 0), (5, 0, 0, 0)),
    (('group_norm', (73728, 512), 512, 8, 9216, 1e-06, False, 512), (1, 0, 0, 0)),
    (('linear', (73728, 512), 512, (1, 512, 512), 0, False, True, (), 0, 0, (False, False, False), 0, (73728, 512), 512, 0), (3, 0, 0, 0)),
    (('attention_single_head', 8, 9216, 512), (1, 0, 0, 0)),
    (('linear', (73728, 512), 512, (1, 512, 512), 0, False, True, (), 512, 0, (False, False, False), 0, (73728, 512), 512, 0), (1, 0, 0, 0)),
    (('upsample2x', (73728, 512), 8, 72, 128), (1, 0, 0, 0)),
    (('conv3x3', (8, 144, 256, 512), 512, (9, 512, 512), 0, False, True, (), 0, 0, (False, False, False), 0, (294912, 512), 512, 0), (4, 0, 0, 0)),
    (('group_norm', (294912, 512), 512, 8, 36864, 1e-06, True, 512), (6, 0, 0, 0)),
    (('conv3x3', (8, 144, 256, 512), 512, (9, 512, 512), 0, False, True, (), 512, 0, (False, False, False), 0, (294912, 512), 512, 0), (3, 0, 0, 0)),
    (('group_norm', (294912, 512), 512, 1, 294912, 1e-05, True, 512), (6, 0, 0, 0)),
    (('tconv3', (1, 8, 36864, 512), 512, (3, 512, 512), 0, False, True, (), 0, 0, (False, False, False), 0, (294912, 512), 512, 0), (3, 0, 0, 0)),
    (('tconv3', (1, 8, 36864, 512), 512, (3, 512, 512), 0, False, True, (), 512, 0, (True, False, False), 0, (294912, 512), 512, 0), (3, 0, 0, 0)),
    (('upsample2x', (294912, 512), 8, 144, 256), (1, 0, 0, 0)),
    (('conv3x3', (8, 288, 512, 512), 512, (9, 512, 512), 0, False, True, (), 0, 0, (False, False, False), 0, (1179648, 512), 512, 0), (1, 0, 0, 0)),
    (('group_norm', (1179648, 512), 512, 8, 147456, 1e-06, True, 512), (1, 0, 0, 0)),
    (('conv3x3', (8, 288, 512, 512), 512, (9, 256, 512), 0, False, True, (), 0, 0, (False, False, False), 0, (1179648, 256), 256, 0), (1, 0, 0, 0)),
    (('group_norm', (1179648, 256), 256, 8, 147456, 1e-06, True, 256), (5, 0, 0, 0)),
    (('linear', (1179648, 512), 512, (1, 256, 512), 0, False, True, (), 0, 0, (False, False, False), 0, (1179648, 256), 256, 0), (1, 0, 0, 0)),
    (('conv3x3', (8, 288, 512, 256), 256, (9, 256, 256), 0, False, True, (), 256, 0, (False, False, False), 0, (1179648, 256), 256, 0), (3, 0, 0, 0)),
    (('group_norm', (1179648, 256), 256, 1, 1179648, 1e-05, True, 256), (6, 0, 0, 0)),
    (('tconv3', (1, 8, 147456, 256), 256, (3, 256, 256), 0, False, True, (), 0, 0, (False, False, False), 0, (1179648, 256), 256, 0), (3, 0, 0, 0)),
    (('tconv3', (1, 8, 147456, 256), 256, (3, 256, 256), 0, False, True, (), 256, 0, (True, False, False), 0, (1179648, 256), 256, 0), (3, 0, 0, 0)),
    (('conv3x3', (8, 288, 512, 256), 256, (9, 256, 256), 0, False, True, (), 0, 0, (False, False, False), 0, (1179648, 256), 256, 0), (2, 0, 0, 0)),
    (('upsample2x', (1179648, 256), 8, 288, 512), (1, 0, 0, 0)),
    (('conv3x3', (8, 576, 1024, 256), 256, (9, 256, 256), 0, False, True, (), 0, 0, (False, False, False), 0, (4718592, 256), 256, 0), (1, 0, 0, 0)),
    (('group_norm', (4718592, 256), 256, 8, 589824, 1e-06, True, 256), (1, 0, 0, 0)),
    (('conv3x3', (8, 576, 1024, 256), 256, (9, 128, 256), 0, False, True, (), 0, 0, (False, False, False), 0, (4718592, 128), 128, 0), (1, 0, 0, 0)),
    (('group_norm', (4718592, 128), 128, 8, 589824, 1e-06, True, 128), (6, 0, 0, 0)),
    (('linear', (4718592, 256), 256, (1, 128, 256), 0, False, True, (), 0, 0, (False, False, False), 0, (4718592, 128), 128, 0), (1, 0, 0, 0)),
    (('conv3x3', (8, 576, 1024, 128), 128, (9, 128, 128), 0, False, True, (), 128, 0, (False, False, False), 0, (4718592, 128), 128, 0), (3, 0, 0, 0)),
    (('group_norm', (4718592, 128), 128, 1, 4718592, 1e-05, True, 128), (6, 0, 0, 0)),
    (('tconv3', (1, 8, 589824, 128), 128, (3, 128, 128), 0, False, True, (), 0, 0, (False, False, False), 0, (4718592, 128), 128, 0), (3, 0, 0, 0)),
    (('tconv3', (1, 8, 589824, 128), 128, (3, 128, 128), 0, False, True, (), 128, 0, (True, False, False), 0, (4718592, 128), 128, 0), (3, 0, 0, 0)),
    (('conv3x3', (8, 576, 1024, 128), 128, (9, 128, 128), 0, False, True, (), 0, 0, (False, False, False), 0, (4718592, 128), 128, 0), (2, 0, 0, 0)),
    (('conv3x3', (8, 576, 1024, 128), 128, (9, 3, 128), 0, False, True, (), 0, 0, (False, False, False), 0, (4718592, 3), 8, 0), (1, 0, 0, 0)),
    (('tconv3', (1, 8, 589824, 8), 8, (3, 3, 8), 0, True, True, (), 0, 0, (False, False, False), 0, (4718592, 3), 8, 0), (1, 0, 0, 0)),
    (('nhwc_to_nchw', (4718592, 8), 'float32', 8, 8, 3, 589824), (1, 0, 0, 0)),
    (('nchw_to_nhwc', (1, 4, 72, 128), 36864, (9216, 8), 8, 0), (0, 1, 0, 0)),
    (('conv3x3', (1, 72, 128, 8), 8, (9, 512, 8), 0, False, True, (), 0, 0, (False, False, False), 0, (9216, 512), 512, 0), (0, 1, 0, 0)),
    (('group_norm', (9216, 512), 512, 1, 9216, 1e-06, True, 512), (0, 10, 9, 0)),
    (('conv3x3', (1, 72, 128, 512), 512, (9, 512, 512), 0, False, True, (), 0, 0, (False, False, False), 0, (9216, 512), 512, 0), (0, 5, 4, 0)),
    (('conv3x3', (1, 72, 128, 512), 512, (9, 512, 512), 0, False, True, (), 512, 0, (False, False, False), 0, (9216, 512), 512, 0), (0, 5, 4, 0)),
    (('group_norm', (9216, 512), 512, 1, 9216, 1e-05, True, 512), (0, 10, 0, 0)),
    (('tconv3', (1, 1, 9216, 512), 512, (3, 512, 512), 0, False, True, (), 0, 0, (False, False, False), 0, (9216, 512), 512, 0), (0, 5, 0, 0)),
    (('tconv3', (1, 1, 9216, 512), 512, (3, 512, 512), 0, False, True, (), 512, 0, (True, False, False), 0, (9216, 512), 512, 0), (0, 5, 0, 0)),
    (('group_norm', (9216, 512), 512, 1, 9216, 1e-06, False, 512), (0, 1, 1, 0)),
    (('linear', (9216, 512), 512, (1, 512, 512), 0, False, True, (), 0, 0, (False, False, False), 0, (9216, 512), 512, 0), (0, 3, 3, 0)),
    (('attention_single_head', 1, 9216, 512), (0, 1, 1, 0)),
    (('linear', (9216, 512), 512, (1, 512, 512), 0, False, True, (), 512, 0, (False, False, False), 0, (9216, 512), 512, 0), (0, 1, 1, 0)),
    (('upsample2x', (9216, 512), 1, 72, 128), (0, 1, 0, 0)),
    (('conv3x3', (1, 144, 256, 512), 512, (9, 512, 512), 0, False, True, (), 0, 0, (False, False, False), 0, (36864, 512), 512, 0), (0, 4, 1, 0)),
    (('group_norm', (36864, 512), 512, 1, 36864, 1e-06, True, 512), (0, 6, 3, 0)),
    (('conv3x3', (1, 144, 256, 512), 512, (9, 512, 512), 0, False, True, (), 512, 0, (False, False, False), 0, (36864, 512), 512, 0), (0, 3, 2, 0)),
    (('group_norm', (36864, 512), 512, 1, 36864, 1e-05, True, 512), (0, 6, 0, 0)),
    (('tconv3', (1, 1, 36864, 512), 512, (3, 512, 512), 0, False, True, (), 0, 0, (False, False, False), 0, (36864, 512), 512, 0), (0, 3, 0, 0)),
    (('tconv3', (1, 1, 36864, 512), 512, (3, 512, 512), 0, False, True, (), 512, 0, (True, False, False), 0, (36864, 512), 512, 0), (0, 3, 0, 0)),
    (('upsample2x', (36864, 512), 1, 144, 256), (0, 1, 0, 0)),
    (('conv3x3', (1, 288, 512, 512), 512, (9, 512, 512), 0, False, True, (), 0, 0, (False, False, False), 0, (147456, 512), 512, 0), (0, 1, 0, 0)),
    (('group_norm', (147456, 512), 512, 1, 147456, 1e-06, True, 512), (0, 1, 0, 0)),
    (('conv3x3', (1, 288, 512, 512), 512, (9, 256, 512), 0, False, True, (), 0, 0, (False, False, False), 0, (147456, 256), 256, 0), (0, 1, 0, 0)),
    (('group_norm', (147456, 256), 256, 1, 147456, 1e-06, True, 256), (0, 5, 3, 0)),
    (('linear', (147456, 512), 512, (1, 256, 512), 0, False, True, (), 0, 0, (False, False, False), 0, (147456, 256), 256, 0), (0, 1, 0, 0)),
    (('conv3x3', (1, 288, 512, 256), 256, (9, 256, 256), 0, False, True, (), 256, 0, (False, False, False), 0, (147456, 256), 256, 0), (0, 3, 2, 0)),
    (('group_norm', (147456, 256), 256, 1, 147456, 1e-05, True, 256), (0, 6, 0, 0)),
    (('tconv3', (1, 1, 147456, 256), 256, (3, 256, 256), 0, False, True, (), 0, 0, (False, False, False), 0, (147456, 256), 256, 0), (0, 3, 0, 0)),
    (('tconv3', (1, 1, 147456, 256), 256, (3, 256, 256), 0, False, True, (), 256, 0, (True, False, False), 0, (147456, 256), 256, 0), (0, 3, 0, 0)),
    (('conv3x3', (1, 288, 512, 256), 256, (9, 256, 256), 0, False, True, (), 0, 0, (False, False, False), 0, (147456, 256), 256, 0), (0, 2, 1, 0)),
    (('upsample2x', (147456, 256), 1, 288, 512), (0, 1, 0, 0)),
    (('conv3x3', (1, 576, 1024, 256), 256, (9, 256, 256), 0, False, True, (), 0, 0, (False, False, False), 0, (589824, 256), 256, 0), (0, 1, 0, 0)),
    (('group_norm', (589824, 256), 256, 1, 589824, 1e-06, True, 256), (0, 1, 0, 0)),
    (('conv3x3', (1, 576, 1024, 256), 256, (9, 128, 256), 0, False, True, (), 0, 0, (False, False, False), 0, (589824, 128), 128, 0), (0, 1, 0, 0)),
    (('group_norm', (589824, 128), 128, 1, 589824, 1e-06, True, 128), (0, 6, 4, 0)),
    (('linear', (589824, 256), 256, (1, 128, 256), 0, False, True, (), 0, 0, (False, False, False), 0, (589824, 128), 128, 0), (0, 1, 0, 0)),
    (('conv3x3', (1, 576, 1024, 128), 128, (9, 128, 128), 0, False, True, (), 128, 0, (False, False, False), 0, (589824, 128), 128, 0), (0, 3, 2, 0)),
    (('group_norm', (589824, 128), 128, 1, 589824, 1e-05, True, 128), (0, 6, 0, 0)),
    (('tconv3', (1, 1, 589824, 128), 128, (3, 128, 128), 0, False, True, (), 0, 0, (False, False, False), 0, (589824, 128), 128, 0), (0, 3, 0, 0)),
    (('tconv3', (1, 1, 589824, 128), 128, (3, 128, 128), 0, False, True, (), 128, 0, (True, False, False), 0, (589824, 128), 128, 0), (0, 3, 0, 0)),
    (('conv3x3', (1, 576, 1024, 128), 128, (9, 128, 128), 0, False, True, (), 0, 0, (False, False, False), 0, (589824, 128), 128, 0), (0, 2, 2, 0)),
    (('conv3x3', (1, 576, 1024, 128), 128, (9, 3, 128), 0, False, True, (), 0, 0, (False, False, False), 0, (589824, 3), 8, 0), (0, 1, 0, 0)),
    (('tconv3', (1, 1, 589824, 8), 8, (3, 3, 8), 0, True, True, (), 0, 0, (False, False, False), 0, (589824, 3), 8, 0), (0, 1, 0, 0)),
    (('nhwc_to_nchw', (589824, 8), 'float32', 8, 1, 3, 589824), (0, 1, 0, 0)),
    (('nchw_to_nhwc', (1, 3, 576, 1024), 1769472, (589824, 8), 8, 0), (0, 0, 1, 0)),
    (('conv3x3', (1, 576, 1024, 8), 8, (9, 128, 8), 0, False, True, (), 0, 0, (False, False, False), 0, (589824, 128), 128, 0), (0, 0, 1, 0)),
    (('conv3x3_s2_pad_after', (1, 576, 1024, 128), 128, (9, 128, 128), 0, False, True, (), 0, 0, (False, False, False), 0, (147456, 128), 128, 0), (0, 0, 1, 0)),
    (('group_norm', (147456, 128), 128, 1, 147456, 1e-06, True, 128), (0, 0, 1, 0)),
    (('conv3x3', (1, 288, 512, 128), 128, (9, 256, 128), 0, False, True, (), 0, 0, (False, False, False), 0, (147456, 256), 256, 0), (0, 0, 1, 0)),
    (('linear', (147456, 128), 128, (1, 256, 128), 0, False, True, (), 0, 0, (False, False, False), 0, (147456, 256), 256, 0), (0, 0, 1, 0)),
    (('conv3x3_s2_pad_after', (1, 288, 512, 256), 256, (9, 256, 256), 0, False, True, (), 0, 0, (False, False, False), 0, (36864, 256), 256, 0), (0, 0, 1, 0)),
    (('group_norm', (36864, 256), 256, 1, 36864, 1e-06, True, 256), (0, 0, 1, 0)),
    (('conv3x3', (1, 144, 256, 256), 256, (9, 512, 256), 0, False, True, (), 0, 0, (False, False, False), 0, (36864, 512), 512, 0), (0, 0, 1, 0)),
    (('linear', (36864, 256), 256, (1, 512, 256), 0, False, True, (), 0, 0, (False, False, False), 0, (36864, 512), 512, 0), (0, 0, 1, 0)),
    (('conv3x3_s2_pad_after', (1, 144, 256, 512), 512, (9, 512, 512), 0, False, True, (), 0, 0, (False, False, False), 0, (9216, 512), 512, 0), (0, 0, 1, 0)),
    (('conv3x3', (1, 72, 128, 512), 512, (9, 8, 512), 0, True, True, (), 0, 0, (False, False, False), 0, (9216, 8), 8, 0), (0, 0, 1, 0)),
    (('nhwc_to_nchw', (9216, 8), 'float32', 8, 1, 4, 9216), (0, 0, 1, 0)),
    (('clip_preprocess', (1, 3, 576, 1024), 3, 7), (0, 0, 0, 1)),
    (('linear_grouped', (256, 592), 592, (1, 1280, 592), 0, False, False, 1, 257, (256, 1280), 1280, 1), (0, 0, 0, 1)),
    (('copy2d', (1, 1280), 1280, 328960, 0), (0, 0, 0, 1)),
    (('add_rows', (257, 1280), 1280, (257, 1280), 1280), (0, 0, 0, 1)),
    (('layer_norm', (257, 1280), 1280, 1280, 1e-05, (), 0, False), (0, 0, 0, 65)),
    (('linear', (257, 1280), 1280, (1, 3840, 1280), 0, False, True, (), 0, 0, (False, False, False), 0, (257, 3840), 3840, 0), (0, 0, 0, 32)),
    (('flash_attn_d80', 1, 257, 16, 3840, 1280), (0, 0, 0, 32)),
    (('linear', (257, 1280), 1280, (1, 1280, 1280), 0, False, True, (), 1280, 0, (False, False, False), 0, (257, 1280), 1280, 0), (0, 0, 0, 32)),
    (('linear', (257, 1280), 1280, (1, 5120, 1280), 2, False, True, (), 0, 0, (False, False, False), 0, (257, 5120), 5120, 0), (0, 0, 0, 32)),
    (('linear', (257, 5120), 5120, (1, 1280, 5120), 0, False, True, (), 1280, 0, (False, False, False), 0, (257, 1280), 1280, 0), (0, 0, 0, 32)),
    (('layer_norm', (1, 1280), 328960, 1280, 1e-05, (), 0, False), (0, 0, 0, 1)),
    (('linear', (1, 1280), 1280, (1, 1024, 1280), 0, True, False, (), 0, 0, (False, False, False), 0, (1, 1024), 1024, 0), (0, 0, 0, 1)),
]
# fmt: on


def test_census_matches_stages():
    """CPU: the launches of each configuration, with their call counts, are exactly its part of CENSUS."""
    for i, config in enumerate(CONFIGS):
        _, counts = census(config)
        want = {rec: n[i] for rec, n in CENSUS if n[i]}
        assert counts == want, f"vae.py / conditioner.py launches changed ({config}): update CENSUS (and its " \
                               "replays) from tests/vae_clip_census.py"
        assert sum(counts.values()) == CALLS[config]
    assert len(CENSUS) == len({rec for rec, _ in CENSUS})


RECORDS = [rec for rec, _ in CENSUS]
GEMM = [r for r in RECORDS if r[0] in GEMM_OPS]
GROUPED = [r for r in RECORDS if r[0] == "linear_grouped"]
ATTN = [r for r in RECORDS if r[0] == "attention_single_head"]
FLASH80 = [r for r in RECORDS if r[0] == "flash_attn_d80"]
GLUE = [r for r in RECORDS if r[0] in ("nchw_to_nhwc", "nhwc_to_nchw", "add_rows", "copy2d", "upsample2x")]
GN_ELSEWHERE = set(GN_NET.values()) | {(8, 589824, 128, 1e-6, True), (1, 8 * 589824, 128, 1e-6, True)}
GN_ALL = sorted({(r[3], r[4], r[1][1], r[5], r[6]) for r in RECORDS if r[0] == "group_norm"})
GN = [c for c in GN_ALL if c not in GN_ELSEWHERE]
LN = sorted({(r[1][0], r[1][1], r[2] // r[1][1], r[4]) for r in RECORDS if r[0] == "layer_norm"})


def test_census_reaches_the_stage_launches():
    """CPU: the census reaches the launches only these stages make: the GELU epilogue, an fp32 output 3 columns wide,
    the pad-after stride-2 conv, tconv3 over a single frame, the grouped patch GEMM and the single-head attention."""
    from streamingt2v_b200._lib import ACT_GELU
    assert any(r[0] == "linear" and r[4] == ACT_GELU for r in GEMM)
    assert any(r[5] and r[12][1] == 3 and r[13] == 8 for r in GEMM)
    assert any(not r[5] and r[12][1] == 3 and r[13] == 8 for r in GEMM)
    assert any(r[0] == "conv3x3_s2_pad_after" for r in GEMM)
    assert any(r[0] == "tconv3" and r[1][1] == 1 and r[10][0] and r[8] for r in GEMM)
    assert GROUPED and (1, 9216, 512) in [r[1:] for r in ATTN] and (8, 9216, 512) in [r[1:] for r in ATTN]


def _clip_preprocess_params():
    import test_conditioner_gpu as tc
    p = {m.args[0]: m.args[1] for m in tc.test_clip_preprocess.pytestmark if m.name == "parametrize"}
    return p["hw"], p["n"]


def test_every_record_is_replayed():
    """CPU: every CENSUS record belongs to exactly one replay below, or is a shape another file runs."""
    hws, ns = _clip_preprocess_params()
    for rec in RECORDS:
        op = rec[0]
        if op == "group_norm":
            key = (rec[3], rec[4], rec[1][1], rec[5], rec[6])
            where = [key in GN, key in GN_ELSEWHERE]
        elif op == "layer_norm":
            where = [(rec[1][0], rec[1][1], rec[2] // rec[1][1], rec[4]) in LN]
        elif op == "clip_preprocess":
            n, _, h, w = rec[1]
            where = [(h, w) in hws and n in ns]
        else:
            where = [rec in GEMM, rec in GROUPED, rec in ATTN, rec in FLASH80, rec in GLUE]
        assert sum(where) == 1, f"{rec}: replayed by {sum(where)} tests"


# ---------------------------------------------------------------------------------------------------------------------
# every GEMM launch of the census
# ---------------------------------------------------------------------------------------------------------------------
def _randn_fill(view, g, scale=1.0):
    """randn * scale into `view` a slab of rows at a time: no fp32 copy of a multi-GB operand."""
    v2 = view if view.dim() == 2 else view.view(-1, view.shape[-1])
    step = max(1, (1 << 26) // v2.shape[1])
    for r0 in range(0, v2.shape[0], step):
        part = v2[r0:r0 + step]
        part.copy_(torch.randn(part.shape, generator=g, device=view.device) * scale)
    return view


def _bands(op, xs, N):
    """(input band, output rows) of one launch for the float64 reference: the row chunks of a linear and (video,
    pixel range) chunks of a tconv3 as in the denoiser file (about 2^25 elements each); (frame, output image rows
    y0..y1) of a conv, about 2^24 elements."""
    if op in ("linear", "tconv3"):
        yield from _chunks(op, xs, N)
        return
    n, h, w, K = xs
    ho, wo = (h, w) if op == "conv3x3" else (h // 2, w // 2)
    step = max(1, (1 << 24) // (w * max(N, K)))       # torch's float64 conv may unfold a band 9 times over
    for f in range(n):
        for y0 in range(0, ho, step):
            y1 = min(ho, y0 + step)
            yield (f, y0, y1), slice((f * ho + y0) * wo, (f * ho + y1) * wo)


def _band_ref(op, x, band, wt, wabs):
    """float64 op(x) and op(|x|) with |w| on one band.  A conv band reads its output rows' taps: one input row more
    on each side for conv3x3 (zero padding at the image edges only), rows 2 y0 .. 2 y1 for the pad-after stride-2
    conv (the zero row below the image only in the last band)."""
    if op in ("linear", "tconv3"):
        x64 = x[band].double()
        return ref_gemm(op, x64, wt), ref_gemm(op, x64.abs(), wabs)
    f, y0, y1 = band
    h, w = x.shape[1:3]
    a, b = (max(0, y0 - 1), min(h, y1 + 1)) if op == "conv3x3" else (2 * y0, min(h, 2 * y1 + 1))
    x64 = x[f:f + 1, a:b].double()
    out = []
    for xv, wv in ((x64, wt), (x64.abs(), wabs)):
        y = ref_gemm(op, xv, wv)
        if op == "conv3x3":
            y = y.view(b - a, w, -1)[y0 - a:y1 - a].reshape(-1, y.shape[-1])
        out.append(y)
    return out


def _gemm_id(i, r):
    op, xs, xld, ws, act, f32, bias, fvec, r1, r2, scales, bn, os_, old, col = r
    tags = [f"{i:02d}", op, "x".join(map(str, xs)), f"n{os_[1]}"]
    tags += [t for t, on in (("gelu", act == 2), ("f32", f32), ("res1", r1), ("sacc", scales[0])) if on]
    if old != os_[1] or col:
        tags.append(f"ld{old}-col{col}")
    return "-".join(tags)


@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(len(GEMM)), ids=[_gemm_id(i, r) for i, r in enumerate(GEMM)])
def test_gemm_launch_fp64(cuda_dev, idx):
    from streamingt2v_b200._lib import ACT_GELU, ACT_NONE
    op, xs, xld, ws, act, f32, has_bias, fvec, r1_ld, r2_ld, scales, bn, os_, old, col = GEMM[idx]
    assert act in (ACT_NONE, ACT_GELU) and not (fvec or r2_ld or bn or scales[1] or scales[2]), "extend the replay"
    assert act == ACT_NONE or not (r1_ld or scales[0]), "an activation before a blend: extend the bound"
    dev = cuda_dev
    g = torch.Generator(device=dev).manual_seed(6000 + idx)
    taps, N, K = ws
    rows, n_out = os_
    if op == "linear":
        X = Guarded(xs, torch.bfloat16, dev, ld=xld)
    else:
        assert xld == K, "conv inputs are contiguous"
        X = Guarded(xs, torch.bfloat16, dev, flat=True)
    _randn_fill(X.view, g)
    w = (torch.randn(ws, generator=g, device=dev) / (taps * K) ** 0.5).to(torch.bfloat16).contiguous()
    wt = (w[0] if op == "linear" else w.permute(1, 2, 0) if op == "tconv3"
          else w.view(3, 3, N, K).permute(2, 3, 0, 1)).double()
    b = torch.randn((N,), generator=g, device=dev) * 0.1 if has_bias else None
    b64 = b.double() if has_bias else torch.zeros(N, dtype=torch.float64, device=dev)
    s_acc = 1.0 - AL if scales[0] else 1.0             # the time stack's sigmoid(mix) blend
    epi = dict(act=act, out_fp32=f32, s_acc=s_acc)
    R1 = None
    if r1_ld:
        R1 = Guarded((rows, n_out), torch.bfloat16, dev, ld=r1_ld)
        _randn_fill(R1.view, g)
        epi.update(res1=R1.view, s1=1.0)
    O = Guarded(os_, torch.float32 if f32 else torch.bfloat16, dev, pre=16, post=16, ld=old, col=col)
    if old > n_out:
        # y8 / o8: the other columns of each row hold data that must come through bitwise
        O.buf[16:16 + rows] = torch.randn((rows, old), generator=g, device=dev).to(O.dtype)
        O.view.fill_(float("nan"))
    O.snapshot()
    name = _gemm_id(idx, GEMM[idx])
    out = replay(lambda: launch(op, X.view, w, b, O.view, (), epi), O, name, schedules=(0, 1, None),
                 epilogues=(0, 1))
    del O

    gamma = (K * taps + 6) * 2.0 ** -23
    c = 2.0 ** -23 if f32 else 2.0 ** -8
    sa = _f32(s_acc)
    wabs = wt.abs()
    acc = _Rows()
    for band, ridx in _bands(op, xs, N):
        if torch.is_tensor(ridx):
            ridx = ridx.to(dev)
        v, s = _band_ref(op, X.view, band, wt, wabs)
        v, s = v + b64, s + b64.abs()
        if act == ACT_GELU:
            ref = _gelu(v)
            bound = 1.13 * gamma * s + 2.0 ** -16 * v.abs()
        else:
            ref = sa * v
            bound = gamma * abs(sa) * s
        if R1 is not None:
            r = R1.view[ridx].double()
            ref = ref + r
            bound = bound + gamma * r.abs()
        bound = bound + c * ref.abs()          # the store's rounding, of the final value
        acc.add(out[ridx], ref, bound)
        del v, s, ref, bound
    acc.finish(name, f"gemm {op} act{act}{' f32' if f32 else ''}")
    del out, X, R1
    free()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2])
def test_linear_grouped_launch(cuda_dev, n):
    """The patch embedding into token rows 1..256 of each image: census n = 1, and n = 2, where out_rs's group
    stride of 257 rows is used.  The class-token rows between the groups hold data and must stay bitwise."""
    from streamingt2v_b200 import ops
    (rec,) = GROUPED
    _, (rows, K), xld, ws, act, f32, has_bias, groups, S, (orows, W), old, row0 = rec
    assert (groups, act, f32, has_bias, row0, orows, old) == (1, 0, False, False, 1, S - 1, W)
    dev = cuda_dev
    g = torch.Generator(device=dev).manual_seed(7000 + n)
    X = _randn_fill(Guarded((n * rows, K), torch.bfloat16, dev, ld=xld).view, g)
    w = (torch.randn(ws, generator=g, device=dev) / K ** 0.5).to(torch.bfloat16).contiguous()
    O = Guarded((n * S, W), torch.bfloat16, dev, pre=16, post=16, ld=old)
    O.view.fill_(float("nan"))
    cls = torch.randn((n, W), generator=g, device=dev).to(torch.bfloat16)
    O.view[0::S] = cls
    O.snapshot()
    out = replay(lambda: ops.linear_grouped(X, w, None, groups=n, out=O.view[row0:], out_group_rows=S), O,
                 f"linear_grouped n{n}", schedules=(0, 1, None), epilogues=(0, 1))
    assert torch.equal(bits(out[0::S]), bits(cls)), "class-token rows written"
    gamma = (K + 6) * 2.0 ** -23
    wt = w[0].double()
    acc = _Rows()
    for i in range(n):
        x64 = X[i * rows:(i + 1) * rows].double()
        ref = x64 @ wt.t()
        bound = 2.0 ** -8 * ref.abs() + gamma * (x64.abs() @ wt.abs().t())
        acc.add(out[i * S + row0:i * S + row0 + rows], ref, bound)
    acc.finish(f"linear_grouped n{n} K{K}", "gemm linear_grouped")
    del X, O, out
    free()


# ---------------------------------------------------------------------------------------------------------------------
# the VAE mid-block attention: its four launches, then the composite
# ---------------------------------------------------------------------------------------------------------------------
ATTN_CASES = [(r[1], False) for r in ATTN] + [(1, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,sharp", ATTN_CASES, ids=[f"n{n}{'-sharp' if sh else ''}" for n, sh in ATTN_CASES])
def test_attention_single_head_launch(cuda_dev, n, sharp):
    from streamingt2v_b200 import ops
    _, _, s, C = next(r for r in ATTN if r[1] == n)
    dev = cuda_dev
    g = torch.Generator(device=dev).manual_seed(8000 + 10 * n + sharp)
    q, k, v = (_randn_fill(Guarded((n * s, C), torch.bfloat16, dev, flat=True).view, g,
                           12.0 if sharp and i == 0 else 1.5) for i in range(3))
    comp = ops.attention_single_head(q, k, v, n, s)
    torch.cuda.synchronize()
    scale = float(C) ** -0.5
    sa = _f32(scale)
    g_qk, g_pv = (C + 6) * 2.0 ** -23, (s + 6) * 2.0 ** -23
    k_sm = 4 * -(-s // 1024) + 13
    accs = {part: _Rows() for part in ("qk", "softmax", "pv", "composite")}
    name = f"attention n{n} s{s} C{C}{' sharp' if sharp else ''}"
    for f in range(n):
        sl = slice(f * s, (f + 1) * s)
        Sg = Guarded((s, s), torch.float32, dev, pre=16, post=16, ld=s).snapshot()
        scores = replay(lambda: ops.linear(q[sl], k[sl][None], None, out=Sg.view, out_fp32=True, s_acc=scale), Sg,
                        f"{name} q k^T frame {f}", schedules=(0, 1, None), epilogues=(0, 1))
        del Sg
        P = Guarded((s, s), torch.bfloat16, dev, ld=s).snapshot()
        ops.softmax_rows(scores, out=P.view)
        torch.cuda.synchronize()
        P.check(f"{name} softmax frame {f}")
        first = P.view.clone()
        ops.softmax_rows(scores, out=P.view)
        torch.cuda.synchronize()
        assert torch.equal(bits(first), bits(P.view)), "softmax reruns differ bitwise"
        del first
        vt = ops.transpose(v[sl])
        torch.cuda.synchronize()
        assert torch.equal(bits(vt), bits(v[sl].t().contiguous())), "transpose not exact"
        Og = Guarded((s, C), torch.bfloat16, dev, pre=16, post=16, ld=C).snapshot()
        pv = replay(lambda: ops.linear(P.view, vt[None], None, out=Og.view), Og, f"{name} P V frame {f}",
                    schedules=(0, 1, None), epilogues=(0, 1))
        del Og, vt
        assert torch.equal(bits(comp[sl]), bits(pv)), "the composite differs from its four launches"

        k64, v64 = k[sl].double(), v[sl].double()
        kabs, vabs = k64.abs(), v64.abs()
        for r0 in range(0, s, s // 4):
            r1 = min(s, r0 + s // 4)
            q64 = q[sl][r0:r1].double()
            s64 = sa * (q64 @ k64.t())
            e = 2.0 ** -23 * s64.abs() + g_qk * sa * (q64.abs() @ kabs.t())       # the fp32 scores' bound
            del q64
            accs["qk"].add(scores[r0:r1], s64, e)
            delta = e.max(1, keepdim=True).values
            del e
            x = scores[r0:r1].double()
            pk = torch.softmax(x, 1)
            accs["softmax"].add(P.view[r0:r1], pk, _softmax_bound(x, pk, s))
            xm = (x - x.max(1, keepdim=True).values).abs()
            r = 2.0 ** -8 + 2.0 ** -23 * (6 + 1.7 * (xm.max(1, keepdim=True).values
                                                     + (pk * xm).sum(1, keepdim=True))) + k_sm * U
            del x, pk, xm
            ph = P.view[r0:r1].double()
            ref = ph @ v64
            accs["pv"].add(pv[r0:r1], ref, 2.0 ** -8 * ref.abs() + g_pv * (ph @ vabs))
            del ph
            p = torch.softmax(s64, 1)
            del s64
            ref, A = p @ v64, p @ vabs
            del p
            m = torch.exp(2 * delta)
            bound = 2.0 ** -8 * ref.abs() + (1 + 2.0 ** -7) * ((m - 1) + m * r + m * (1 + r) * g_pv) * A \
                + s * 2.0 ** -126 * vabs.max()
            accs["composite"].add(comp[sl][r0:r1], ref, bound)
            del ref, A, bound
        del scores, P, pv
        free()
    accs["qk"].finish(name + " q k^T", "attention q k^T linear")
    accs["softmax"].finish(name + " softmax", "attention softmax_rows")
    accs["pv"].finish(name + " P V", "attention P V linear")
    accs["composite"].finish(name, "attention composite", l2=2 ** -7)
    del q, k, v, comp
    free()


# ---------------------------------------------------------------------------------------------------------------------
# CLIP's head-dim-80 FlashAttention at the census leading dims
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(len(FLASH80)), ids=[f"n{r[1]}-s{r[2]}-h{r[3]}-ld{r[4]}" for r in FLASH80])
def test_flash_attn_d80_launch(cuda_dev, idx):
    """The fused QKV buffer at ld = 3 C exactly (no pad column after v), in NaN guard rows."""
    from streamingt2v_b200 import ops
    _, n, s, heads, qld, old = FLASH80[idx]
    C = heads * 80
    assert qld == 3 * C and old == C
    dev = cuda_dev
    g = torch.Generator(device=dev).manual_seed(9000 + idx)
    Q = Guarded((n * s, 3 * C), torch.bfloat16, dev, ld=qld)
    _randn_fill(Q.view, g, 1.5)
    O = Guarded((n * s, C), torch.bfloat16, dev, ld=old).snapshot()
    outs = []
    for _ in range(2):
        ops.flash_attn_d80(Q.view, n, s, heads, out=O.view)
        torch.cuda.synchronize()
        O.check(f"flash_attn_d80 n{n} s{s}")
        outs.append(bits(O.view).clone())
    assert torch.equal(outs[0], outs[1]), "reruns differ bitwise"
    ref, ref_abs = _attn64(Q.view, n, s, heads)
    acc = _Rows()
    acc.add(O.view, ref, 2.0 ** -8 * ref.abs() + 2.0 ** -7 * ref_abs)
    acc.finish(f"flash_attn_d80 n{n} s{s} h{heads}", "flash_attn_d80", l2=2 ** -7)
    del Q, O
    free()


# ---------------------------------------------------------------------------------------------------------------------
# norms at every census shape not run elsewhere (test_norm_glue_edges_gpu.py's cases and bounds)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n,p,c,eps,silu", GN, ids=[f"n{n}-p{p}-c{c}-eps{eps:g}{'-silu' if si else ''}"
                                                    for n, p, c, eps, si in GN])
def test_group_norm_launch(cuda_dev, n, p, c, eps, silu):
    """Per frame (n = 8 or 1, eps 1e-6) and the time stack's norm over all frames of a group (n = 1, eps 1e-5), up to
    8 x 589 824 rows of 256 channels.  Between the two bitwise-compared runs another launch takes the same tickets:
    half the samples, or for n = 1 (the statistics buffer holds one sample) half the rows."""
    alt = (n // 2, p) if n > 1 else (1, p // 2)
    _gn_case(cuda_dev, n, p, c, eps, silu, f"n{n} p{p} c{c}", x_fill=_channel_fill(cuda_dev, c, 3), alt_n=alt)
    free()


@pytest.mark.gpu
@pytest.mark.parametrize("rows,c,step,eps", LN, ids=[f"{r}x{c}-stride{st}" for r, c, st, _ in LN])
def test_layer_norm_launch(cuda_dev, rows, c, step, eps):
    """The tower's pre-LN norms over the 257 token rows, and ln_post over the class row alone at a row stride of
    257 x 1280."""
    recs = [r for r in RECORDS if r[0] == "layer_norm" and (r[1], r[2] // r[1][1]) == ((rows, c), step)]
    assert recs and all(r[5:] == ((), 0, False) for r in recs), "fvec / xsum / SiLU: extend the case"
    _ln_case(cuda_dev, f"{rows}x{c}-stride{step}", rows, c, dict(stride_rows=step) if step > 1 else {}, eps=eps)
    free()


# ---------------------------------------------------------------------------------------------------------------------
# layout glue at every census shape: exact
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(len(GLUE)), ids=[f"{r[0]}-{'x'.join(map(str, r[1]))}-{i}"
                                                       for i, r in enumerate(GLUE)])
def test_glue_launch_exact(cuda_dev, idx):
    """nchw_to_nhwc of the latents (4 channels) and the frame (3) into 8-wide rows; upsample2x up to its 2.4 GB output;
    nhwc_to_nchw of the 3 (decoder) or 4 (encoder) channels of the fp32 o8; the class row into the token buffer at a
    row stride of 257 x 1280; the positional rows over the 257 tokens.  Outputs in NaN guards, the rest of their rows
    bitwise unchanged."""
    _glue_case(cuda_dev, GLUE[idx], 9500 + idx)
