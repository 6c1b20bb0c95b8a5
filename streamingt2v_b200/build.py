"""In-tree build of libb200svd.so (hand-written sm_90a CUDA, C ABI) and of the C oracle helpers.

nvcc cross-compiles without a GPU.  Objects are cached by mtime under build/ and linked into
streamingt2v_b200/libb200svd.so, which is loaded from the source tree.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "streamingt2v_b200" / "csrc"
OBJ_DIR = ROOT / "build" / "obj"
LIB_PATH = ROOT / "streamingt2v_b200" / "libb200svd.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _newest_header_mtime() -> float:
    hs = list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) + list((ROOT / "include").glob("*.h"))
    return max(h.stat().st_mtime for h in hs)


def _compile_one(src: Path, obj: Path, verbose: bool) -> None:
    cmd = [_nvcc(), *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
    if verbose:
        print(" ".join(cmd), flush=True)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")


def build_lib(force: bool = False, verbose: bool = False) -> Path:
    """Compile every csrc/*.cu for sm_90a and link libb200svd.so. Returns the library path."""
    OBJ_DIR.mkdir(parents=True, exist_ok=True)
    srcs = sorted(CSRC.glob("*.cu"))
    if not srcs:
        raise RuntimeError("no CUDA sources found")
    hdr_m = _newest_header_mtime()
    jobs = []
    objs = []
    for s in srcs:
        o = OBJ_DIR / (s.stem + ".o")
        objs.append(o)
        if force or not o.exists() or o.stat().st_mtime < max(s.stat().st_mtime, hdr_m):
            jobs.append((s, o))
    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(lambda so: _compile_one(so[0], so[1], verbose), jobs))
    need_link = force or bool(jobs) or not LIB_PATH.exists() or any(
        o.stat().st_mtime > LIB_PATH.stat().st_mtime for o in objs)
    if need_link:
        cmd = [_nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(LIB_PATH),
               *[str(o) for o in objs]]
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB_PATH


if __name__ == "__main__":
    p = build_lib(force="--force" in sys.argv, verbose=True)
    print("built", p)
