"""CPU: which compile-time epilogue kind a GEMM launch takes (b200svd_gemm_epilogue_kind), the selector
(b200svd_gemm_epilogue), and the compiled bodies themselves: in the library's SASS every GEMM kernel that has
specialised bodies holds runs of staging stores with neither a branch nor a global load between them, which the
generic body, with its per-element tests of activation, bias, per-frame vector and residuals, never produces.
"""
import ctypes as C
import re
import shutil
import subprocess

import pytest


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from streamingt2v_b200 import _lib
    return _lib.load()


def _params(n=320, act=0, bias=False, fvec=False, res1=False, res2=False, out_fp32=False, gn=False):
    """Only the fields the epilogue kind depends on; pointers are dummies, nothing is launched."""
    from streamingt2v_b200._lib import GemmParams
    p = GemmParams()
    p.n, p.k, p.taps = n, 64, 1
    p.act, p.out_fp32, p.s_acc = act, int(out_fp32), 1.0
    p.bias = 0x1000 if bias else None
    p.fvec = 0x2000 if fvec else None
    p.res1 = 0x3000 if res1 else None
    p.res2 = 0x4000 if res2 else None
    p.gn_part = 0x5000 if gn else None
    return p


# the launches of model.py, vae.py and conditioner.py
TABLE = [
    ("fused QKV, CAM q/k/v (no bias)", dict(), "EPI_PLAIN"),
    ("convolutions and linears without a residual", dict(bias=True), "EPI_BIAS"),
    ("s_ff2, t_ffin2, t_out, proj_out, conv2, VAE", dict(bias=True, res1=True), "EPI_BIAS_RES1"),
    ("s_out, t_out with xt_vec", dict(bias=True, res1=True, fvec=True), "EPI_BIAS_RES1_FVEC"),
    ("conv1, tconv1", dict(bias=True, fvec=True), "EPI_BIAS_FVEC"),
    ("s_ff1, t_ffin1, t_ff1", dict(bias=True, act=3, n=2560), "EPI_BIAS_GEGLU"),
    ("t_ff2", dict(bias=True, res1=True, res2=True), "EPI_BIAS_RES2"),
    ("conv_in of the ControlNet conditioning, embeddings", dict(bias=True, act=1), "EPI_BIAS_SILU"),
    ("image tower fc", dict(bias=True, act=2), "EPI_BIAS_GELU"),
]

GENERIC = [
    ("residual without a bias", dict(res1=True)),
    ("per-frame vector without a bias", dict(fvec=True)),
    ("res2 alone", dict(bias=True, res2=True)),
    ("two residuals and a per-frame vector", dict(bias=True, res1=True, res2=True, fvec=True)),
    ("SiLU with a residual", dict(bias=True, act=1, res1=True)),
    ("GELU without a bias", dict(act=2)),
    ("GEGLU without a bias", dict(act=3, n=2560)),
    ("GroupNorm partials", dict(bias=True, gn=True)),
    ("fp32 output", dict(bias=True, out_fp32=True)),
    ("output width not a multiple of 8", dict(bias=True, n=12)),
    ("GEGLU output width not a multiple of 8", dict(bias=True, act=3, n=24)),
]


@pytest.mark.parametrize("where,kw,kind", TABLE, ids=[t[2] for t in TABLE])
def test_network_launches_have_a_kind(lib, where, kw, kind):
    from streamingt2v_b200 import _lib
    assert lib.b200svd_gemm_epilogue_kind(C.byref(_params(**kw))) == getattr(_lib, kind), where


@pytest.mark.parametrize("what,kw", GENERIC, ids=[g[0] for g in GENERIC])
def test_everything_else_is_generic(lib, what, kw):
    assert lib.b200svd_gemm_epilogue_kind(C.byref(_params(**kw))) == 0, what


def test_kind_ids_match_the_header():
    import os
    from streamingt2v_b200 import _lib
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "b200svd.h")).read()
    ids = dict(re.findall(r"B200SVD_(EPI_[A-Z0-9_]+) = (\d+)", src))
    assert len(ids) == 10
    for name, v in ids.items():
        assert getattr(_lib, name) == int(v)


def test_selector_round_trips(lib):
    from streamingt2v_b200 import ops
    assert ops.gemm_epilogue(-1) == 1                         # default: specialised where one exists
    try:
        assert ops.gemm_epilogue(0) == 1 and ops.gemm_epilogue(-1) == 0
        assert lib.b200svd_gemm_epilogue_kind(C.byref(_params(bias=True))) == 0   # forced generic
        assert ops.gemm_epilogue(7) == 0 and ops.gemm_epilogue(-1) == 0           # other values only query
    finally:
        ops.gemm_epilogue(1)
    assert ops.gemm_epilogue(-1) == 1
    assert lib.b200svd_gemm_epilogue_kind(C.byref(_params(bias=True))) != 0


def _clean_store_runs(body, min_len=8):
    """Number of runs of at least min_len shared-memory stores (STS / STSM) with no branch and no global load between
    consecutive ones."""
    ops = re.findall(r"^\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_.]+)", body, flags=re.M)
    runs, cur, clean = 0, 0, True
    for o in ops:
        if o.startswith("STS"):
            if cur and clean:
                cur += 1
            else:
                runs += cur >= min_len
                cur = 1
            clean = True
        elif o.startswith(("BRA", "BRX", "LDG")):
            clean = False
    return runs + (cur >= min_len)


def test_every_gemm_kernel_stages_branch_free_in_sass(lib):
    """Each of the eight GEMM kernels (both schedules) holds specialised bodies.  A thread stages 8 column pairs per 64 rows of a sub-tile.  A specialised body writes them back to back; in the
    generic body every pair is separated from the next by the activation branch chain."""
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    from streamingt2v_b200 import _lib
    out = subprocess.run(["cuobjdump", "-sass", str(_lib.lib_path())], capture_output=True, text=True, check=True).stdout
    seen = 0
    for b in re.split(r"Function : ", out)[1:]:
        name = b.splitlines()[0]
        if "mtgemm_kernel" not in name and "mtgemm_alt_kernel" not in name:
            continue
        seen += 1
        runs = _clean_store_runs(b)
        assert runs > 1, (name, runs)
    assert seen == 8
