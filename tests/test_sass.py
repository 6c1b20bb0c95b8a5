"""CPU: the built sm_90a library really contains what DESIGN.md says it does — checked on the SASS of
streamingt2v_b200/libb200svd.so with cuobjdump (wgmma -> HGMMA, TMA load -> UTMALDG, setmaxnreg -> USETMAXREG).
Skipped when cuobjdump is not on the PATH."""
import re
import shutil
import subprocess

import pytest


@pytest.fixture(scope="module")
def sass():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    import __graft_entry__ as g
    g.build()
    from streamingt2v_b200 import _lib
    out = subprocess.run(["cuobjdump", "-sass", str(_lib.lib_path())], capture_output=True, text=True, check=True).stdout
    kernels = {}
    cur = None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            kernels[cur] = []
        elif cur is not None:
            kernels[cur].append(line)
    return {k: "\n".join(v) for k, v in kernels.items()}


def _of(sass, needle):
    sel = {k: v for k, v in sass.items() if needle in k}
    assert sel, f"no kernel matching {needle}"
    return sel


def test_arch_is_sm90a(sass):
    from streamingt2v_b200 import _lib
    out = subprocess.run(["cuobjdump", "-lelf", str(_lib.lib_path())], capture_output=True, text=True).stdout
    assert "sm_90a" in out


def test_gemm_uses_wgmma_and_tma(sass):
    g = _of(sass, "mtgemm_kernel")
    assert len(g) == 5, sorted(g)                                          # N tiles 32, 64, 128, 160, 256
    for name, body in g.items():
        assert "HGMMA" in body, f"{name}: no wgmma"
        assert "UTMALDG" in body, f"{name}: TMA load missing"
        assert "USETMAXREG" in body, f"{name}: producer / consumer register split missing"
        assert not re.search(r"(?<![A-Z])HMMA\b", body), f"{name}: legacy mma.sync path"


def test_attention_kernels_use_wgmma(sass):
    for needle in ("flash_attn_kernel", "pixel_attn_kernel"):
        for name, body in _of(sass, needle).items():
            assert "HGMMA" in body and "UTMALDG" in body, f"{name}: not on wgmma + TMA"
            assert "MUFU.EX2" in body
            assert not re.search(r"(?<![A-Z])HMMA\b", body), f"{name}: legacy mma.sync path"
