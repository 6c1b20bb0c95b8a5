"""CPU: host side of the SVD conditioner (streamingt2v_b200/conditioner.py).

- The ViT-H/14 host pipeline (weight packing, patch rows written into token rows 1..256, class row, positional rows,
  ln_post over the class rows at row stride 257 * width) with tests/fake_clip_ops.py (tests/fake_ops.py plus the
  conditioner's ops) standing in for the kernels, against the fp32 oracle (oracle/clip_image_oracle.py) at CLIP_TINY.
- The SASS of the head-dim-80 attention kernel (wgmma, TMA, ex2; no mma.sync).
- The new entry points reject bad operands before any launch (fake device pointers: host only).
- `B200SVDConditioner.from_reference` on the reference's own GeneralConditioner (stand-ins of
  oracle/make_golden_conditioner.py), run end to end with the CPU fakes.
- Rank 0's cond_aug noise is what every rank conditions on."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import fake_clip_ops

BASE = 0x7F0000000000


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm()).item()


@pytest.fixture()
def patched(monkeypatch):
    from streamingt2v_b200 import conditioner, vae
    monkeypatch.setattr(conditioner, "ops", fake_clip_ops)
    monkeypatch.setattr(vae, "ops", fake_clip_ops)
    return conditioner


def test_clip_param_grammar():
    from streamingt2v_b200 import arch
    full = arch.clip_visual_param_shapes(arch.ClipVisionConfig())
    assert full["conv1.weight"] == (1280, 3, 14, 14) and full["positional_embedding"] == (257, 1280)
    assert full["transformer.resblocks.31.attn.in_proj_weight"] == (3840, 1280) and full["proj"] == (1280, 1024)
    assert len(full) == 3 + 2 + 32 * 12 + 2 + 1                                 # conv1, cls, pos, ln_pre, blocks, ln_post, proj
    assert 630e6 < sum(int(np.prod(s)) for s in full.values()) < 635e6           # ViT-H/14 visual: 632 M parameters
    tiny = arch.CLIP_TINY
    assert tiny.head_dim == 80 and tiny.tokens == 257 and tiny.output_dim == 1024


def test_patch_packing_matches_conv():
    """pack_clip_patch + the preprocessing kernel's column order reproduce conv1 (14x14, stride 14, no bias)."""
    from oracle import clip_image_oracle as co
    from streamingt2v_b200 import packing
    g = torch.Generator().manual_seed(0)
    w = torch.randn(32, 3, 14, 14, generator=g)
    img = torch.randn(2, 3, 224, 224, generator=g)
    wp = packing.pack_clip_patch(w, "cpu")
    assert wp.shape == (1, 32, 592) and not wp[0, :, 588:].any()
    rows = co.patch_rows(img)                                                  # [(2 256), 588]
    got = rows @ wp[0, :, :588].float().t()
    ref = torch.nn.functional.conv2d(img, w.to(torch.bfloat16).float(), stride=14).reshape(2, 32, 256).permute(0, 2, 1)
    assert torch.allclose(got.reshape(2, 256, 32), ref, atol=1e-3, rtol=1e-4)


@pytest.mark.parametrize("n,H,W", [(2, 448, 320), (1, 128, 300), (3, 224, 224)])
def test_clip_host_pipeline_matches_oracle(patched, n, H, W):
    from oracle import clip_image_oracle as co
    from streamingt2v_b200 import arch
    cfg = arch.CLIP_TINY
    sd = arch.synth_state_dict_fast(arch.clip_visual_param_shapes(cfg), 7)
    x = torch.rand(n, 3, H, W, generator=torch.Generator().manual_seed(H + W + n)) * 2 - 1
    enc = patched.B200ClipImageEncoder(cfg, sd, "cpu")
    enc.debug_taps = {}
    out = enc.encode(x)
    taps = {}
    with torch.no_grad():
        ref = co.encode(sd, cfg, x, taps)
    assert out.shape == (n, 1024) and out.dtype == torch.float32
    for k in co.tap_names(cfg):
        got = enc.debug_taps[k].float()
        assert _rel(got.reshape(taps[k].shape), taps[k]) < 2e-2, k
    assert _rel(out, ref) < 2e-2
    # each image is encoded independently of its batch neighbours (row plumbing of the class / patch rows)
    one = enc.encode(x[-1:])
    assert _rel(one, ref[-1:]) < 2e-2


def test_antialias_taps_follow_kornia_formulas():
    from oracle import clip_image_oracle as co
    from streamingt2v_b200.conditioner import antialias_taps
    for hw in [(576, 1024), (448, 320), (128, 300), (1080, 1920), (224, 224), (100, 200)]:
        ty, tx = antialias_taps(*hw)
        p = co.antialias_params(*hw)
        if p is None:
            assert (ty, tx) == ([1.0], [1.0])
            continue
        (ky, kx), (sy, sx) = p
        assert torch.equal(torch.tensor(ty), co.gaussian_taps(ky, sy)) and torch.equal(torch.tensor(tx), co.gaussian_taps(kx, sx))
    assert [len(t) for t in antialias_taps(576, 1024)] == [3, 7]
    assert antialias_taps(128, 300)[0] == [0.0, 1.0, 0.0]                    # sigma 0.001 on the upsampled axis


# ---------------------------------------------------------------------------------------------------------------------
# library: SASS and argument checks
# ---------------------------------------------------------------------------------------------------------------------
def test_d80_attention_sass():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    import __graft_entry__ as g
    g.build()
    from streamingt2v_b200 import _lib
    out = subprocess.run(["cuobjdump", "-sass", str(_lib.lib_path())], capture_output=True, text=True, check=True).stdout
    bodies, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            bodies[cur] = []
        elif cur is not None:
            bodies[cur].append(line)
    sel = {k: "\n".join(v) for k, v in bodies.items() if "flash_attn_d80_kernel" in k}
    assert len(sel) == 1
    body = next(iter(sel.values()))
    assert "HGMMA" in body and "UTMALDG" in body and "MUFU.EX2" in body
    assert not re.search(r"(?<![A-Z])HMMA\b", body)
    assert len([k for k in bodies if "mtgemm_kernel" in k]) == 5


@pytest.fixture(scope="module")
def lib():
    if torch.cuda.is_available():
        pytest.skip("fake device pointers: host-only test")
    import __graft_entry__ as g
    g.build()
    from streamingt2v_b200 import _lib
    return _lib.load()


def _err(lib, rc, word):
    msg = lib.b200svd_last_error().decode()
    assert rc == 1, msg
    assert word in msg.lower(), msg


def _flash_entry(lib, d):
    return lib.b200svd_flash_attn if d == 64 else lib.b200svd_flash_attn_d80


@pytest.mark.parametrize("d", [64, 80])
@pytest.mark.parametrize("which", ["qkv", "out"])
def test_flash_attn_d80_rejects_misaligned(lib, which, d):
    qkv, out = BASE, BASE + 0x100000
    if which == "qkv":
        qkv += 8
    else:
        out += 8
    C2 = 2 * d  # two heads
    _err(lib, _flash_entry(lib, d)(qkv, 3 * C2, out, C2, 1, 257, 2, d ** -0.5, None), "align")


@pytest.mark.parametrize("d", [64, 80])
@pytest.mark.parametrize("args,word", [
    (lambda C2: dict(ldqkv=3 * C2 + 4), "multiples of 8"),
    (lambda C2: dict(ldqkv=3 * C2 - 8), "ldqkv"),
    (lambda C2: dict(ldo=C2 - 8), "ldo"),
    (lambda C2: dict(s=0), "need n, s, heads"),
], ids=["ld_not_8", "ldqkv_short", "ldo_short", "empty"])
def test_flash_attn_d80_rejects_bad_sizes(lib, args, word, d):
    C2 = 2 * d  # two heads
    a = dict(ldqkv=3 * C2, ldo=C2, n=1, s=257, heads=2)
    a.update(args(C2))
    rc = _flash_entry(lib, d)(BASE, a["ldqkv"], BASE + 0x100000, a["ldo"], a["n"], a["s"], a["heads"], 0.1, None)
    _err(lib, rc, word)


def test_clip_preprocess_rejects_bad_input(lib):
    taps = (C.c_float * 3)(0.25, 0.5, 0.25)
    one = (C.c_float * 1)(1.0)
    good = dict(x=BASE, n=1, h=576, w=1024, out=BASE + 0x1000000, ldp=592, ty=taps, ky=3, tx=taps, kx=3)

    def call(**kw):
        a = dict(good, **kw)
        return lib.b200svd_clip_preprocess(a["x"], a["n"], a["h"], a["w"], a["out"], a["ldp"], a["ty"], a["ky"],
                                           a["tx"], a["kx"], None)
    _err(lib, call(out=BASE + 0x1000008), "align")
    _err(lib, call(x=BASE + 2), "align")
    _err(lib, call(ldp=588), "ldp")
    _err(lib, call(ldp=584), "ldp")
    _err(lib, call(ky=2), "taps")
    _err(lib, call(ty=one, ky=1, h=1, tx=taps, kx=3, w=1), "reflect")
    _err(lib, call(n=0), "need n")


# ---------------------------------------------------------------------------------------------------------------------
# conditioner assembly
# ---------------------------------------------------------------------------------------------------------------------
class _RecordingEncoder:
    def __init__(self):
        self.seen = []
        self.dev = torch.device("cpu")

    def encode(self, x):
        self.seen.append(x.clone())
        return torch.ones(x.shape[0], 4, x.shape[2] // 8, x.shape[3] // 8)


class _StubClip:
    dev = torch.device("cpu")

    def encode(self, x):
        return torch.full((x.shape[0], 1024), float(x.mean()))


def test_conditioner_noise_and_vector(patched):
    from oracle import ref_shims  # noqa: F401  (importable without the reference checkout)
    enc = _RecordingEncoder()
    cond = patched.B200SVDConditioner(_StubClip(), enc, generator=torch.Generator().manual_seed(4))
    frame = torch.rand(3, 32, 48, generator=torch.Generator().manual_seed(1)) * 2 - 1
    c, uc = cond(frame, 5)
    noise = torch.rand((1, 3, 32, 48), generator=torch.Generator().manual_seed(4))
    assert torch.equal(enc.seen[0], frame[None] + 0.02 * noise)               # uniform noise, scaled by cond_aug
    assert c["crossattn"].shape == (1, 1, 1024) and c["concat"].shape == (1, 4, 4, 6) and c["vector"].shape == (5, 768)
    # vector = [emb(fps_id) | emb(motion_bucket_id) | emb(cond_aug)], sgm timestep_embedding (util.py:207-231)
    half = 128
    freqs = torch.exp(-np.log(10000.0) * torch.arange(half, dtype=torch.float32) / half)
    for k, v in enumerate((6.0, 127.0, 0.02)):
        a = v * freqs
        ref = torch.cat([torch.cos(a), torch.sin(a)])
        assert (c["vector"][:, 256 * k:256 * (k + 1)] - ref[None]).abs().max() <= 2.0 ** -8
    assert not uc["crossattn"].any() and not uc["concat"].any() and torch.equal(uc["vector"], c["vector"])


def test_conditioner_broadcasts_rank0_noise(patched, monkeypatch):
    """With a process group of more than one rank, every rank conditions on rank 0's noise (the ranks' generators are
    not assumed to be seeded alike)."""
    rank0 = torch.full((1, 3, 16, 16), 0.5)
    calls = []

    def fake_broadcast(t):
        calls.append(t.shape)
        return rank0.clone()
    monkeypatch.setattr(patched.dist_utils, "broadcast_from_rank0", fake_broadcast)
    enc = _RecordingEncoder()
    cond = patched.B200SVDConditioner(_StubClip(), enc, generator=torch.Generator().manual_seed(123))
    frame = torch.zeros(3, 16, 16)
    cond(frame, 3)
    assert calls == [torch.Size([1, 3, 16, 16])]
    assert torch.equal(enc.seen[0], torch.full((1, 3, 16, 16), 0.02 * 0.5))


def test_from_reference_extracts_weights(patched):
    """from_reference on the reference's own GeneralConditioner (literal config.yaml emb_models, stand-ins of
    oracle/make_golden_conditioner.py) reads the open_clip visual tower and the AutoencoderKL encoder + quant_conv, and
    with the CPU fakes reproduces the reference's (c, uc) for a small frame."""
    if not os.path.isdir("/root/reference/code"):
        pytest.skip("reference checkout not available")
    from oracle import make_golden_conditioner as mg
    from streamingt2v_b200 import arch
    cfg = arch.CLIP_TINY
    sd_c = arch.synth_state_dict_fast(arch.clip_visual_param_shapes(cfg), 61)
    sd_v = arch.synth_state_dict_fast(arch.vae_encoder_param_shapes(arch.VaeConfig()), 62)
    ref_cond = mg.build_reference_conditioner(cfg, sd_c, sd_v)
    frame = torch.rand(3, 64, 96, generator=torch.Generator().manual_seed(3)) * 2 - 1
    T, seed = 4, 17
    c_ref, uc_ref = mg.run_reference(ref_cond, frame, T, seed)
    cond = patched.B200SVDConditioner.from_reference(ref_cond, "cpu", generator=torch.Generator().manual_seed(seed))
    assert cond.clip.cfg == cfg
    assert cond.vae_encoder.cfg == arch.VaeConfig()
    c, uc = cond(frame, T)
    for k in ("crossattn", "concat"):
        assert c[k].shape == c_ref[k].shape and _rel(c[k], c_ref[k]) < 3e-2, k
        assert not uc[k].any() and not uc_ref[k].any()
    assert (c["vector"] - c_ref["vector"]).abs().max() <= 2.0 ** -8
