"""ctypes binding of libb200svd.so (the C-ABI boundary, include/b200svd.h).

No torch types cross this boundary: tensors are passed as raw device pointers + sizes, the CUDA stream as a
void*.  The library is mandatory — there is no CPU or eager-PyTorch fallback; a missing/unloadable library or a
device other than sm_90 raises.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_LIB = None
LIB_PATH = Path(__file__).resolve().parent / "libb200svd.so"

MAX_TAPS = 12
ACT_NONE, ACT_SILU, ACT_GELU, ACT_GEGLU, ACT_PRELU = 0, 1, 2, 3, 4
# B200SVD_EPI_*: compile-time epilogue kinds of the GEMM, 0 = the generic body
(EPI_GENERIC, EPI_PLAIN, EPI_BIAS, EPI_BIAS_RES1, EPI_BIAS_RES1_FVEC, EPI_BIAS_FVEC, EPI_BIAS_GEGLU, EPI_BIAS_RES2,
 EPI_BIAS_SILU, EPI_BIAS_GELU) = range(10)


class GemmParams(C.Structure):
    _fields_ = [
        ("a_ptr", C.c_void_p),
        ("a_dims", C.c_uint64 * 5),
        ("a_strides", C.c_uint64 * 4),
        ("a_box", C.c_uint32 * 5),
        ("w_ptr", C.c_void_p),
        ("n", C.c_uint32),
        ("k", C.c_uint32),
        ("taps", C.c_uint32),
        ("tap_off", (C.c_int32 * 5) * MAX_TAPS),
        ("m_ext", C.c_uint32 * 3),
        ("m_box", C.c_uint32 * 3),
        ("m_adim", C.c_uint32 * 3),
        ("out_rs", C.c_int64 * 3),
        ("out", C.c_void_p),
        ("ldo", C.c_int64),
        ("out_fp32", C.c_int32),
        ("bias", C.c_void_p),
        ("fvec", C.c_void_p),
        ("ldf", C.c_int64),
        ("rows_per_frame", C.c_uint32),
        ("act", C.c_int32),
        ("s_acc", C.c_float),
        ("res1", C.c_void_p),
        ("ld1", C.c_int64),
        ("s1", C.c_float),
        ("res2", C.c_void_p),
        ("ld2", C.c_int64),
        ("s2", C.c_float),
        ("bn", C.c_int32),
        ("gn_part", C.c_void_p),
        ("gn_slot_sample", C.c_void_p),
        ("gn_ld", C.c_int64),
        ("gn_rows", C.c_uint32),
        ("slope", C.c_void_p),
    ]


class B200Error(RuntimeError):
    pass


def lib_path() -> Path:
    return Path(os.environ.get("B200SVD_LIB", str(LIB_PATH)))


def load():
    """Load libb200svd.so (once) and declare the prototypes."""
    global _LIB
    if _LIB is not None:
        return _LIB
    p = lib_path()
    if not p.exists():
        raise B200Error(
            f"{p} not found — build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no fallback path)")
    lib = C.CDLL(str(p))
    lib.b200svd_last_error.restype = C.c_char_p
    lib.b200svd_last_error.argtypes = []
    lib.b200svd_version.restype = C.c_int
    lib.b200svd_init.restype = C.c_int
    lib.b200svd_init.argtypes = [C.c_int]
    _declare(lib)
    lib.b200svd_gemm_pair_mode.restype = C.c_int
    lib.b200svd_gemm_pair_mode.argtypes = [C.c_int]
    lib.b200svd_flash_attn_variant.restype = C.c_int
    lib.b200svd_flash_attn_variant.argtypes = [C.c_int]
    lib.b200svd_gn_scratch_doubles.restype = C.c_int64
    lib.b200svd_gn_scratch_doubles.argtypes = [C.c_int64, C.c_int64, C.c_int]
    _LIB = lib
    return lib


# name -> argtypes; every entry returns int (0 = ok).  Kept in one table so the symbol-export test can walk it.
_P, _I64, _I, _F = C.c_void_p, C.c_int64, C.c_int, C.c_float
PROTOTYPES = {
    "b200svd_gemm": [C.POINTER(GemmParams), _P],
    "b200svd_gemm_schedule": [_I],                      # returns the previous schedule, not a status
    "b200svd_gemm_epilogue": [_I],                      # returns the previous mode
    "b200svd_gemm_epilogue_kind": [C.POINTER(GemmParams)],  # returns a B200SVD_EPI_* id
    "b200svd_flash_attn": [_P, _I64, _P, _I64, _I, _I, _I, _F, _P],
    "b200svd_flash_attn_d80": [_P, _I64, _P, _I64, _I, _I, _I, _F, _P],
    "b200svd_clip_preprocess": [_P, _I, _I, _I, _P, _I64, _P, _I, _P, _I, _P],
    "b200svd_small_attn": [_P, _I64, _P, _I64, _P, _I64, _P, _I64, _I, _I, _I, _I, _I, _I, _F, _P],
    "b200svd_pixel_attn": [_P, _I64, _P, _I64, _P, _I64, _P, _I64, _I, _I, _I, _I, _I, _F, _P],
    "b200svd_gn_stats": [_P, _I64, _I64, _I64, _I, _P, _P, _P, _P],
    "b200svd_gn_apply": [_P, _I64, _P, _I64, _I64, _I64, _I, _P, _P, _P, _F, _I, _P],
    "b200svd_layernorm": [_P, _I64, _P, _I64, _I64, _I, _P, _P, _F, _P, _I64, _I, _P, _I64, _I, _P],
    "b200svd_nchw_to_nhwc": [_P, _I64, _I, _I, _I64, _P, _I64, _I, _P],
    "b200svd_nhwc_to_nchw": [_P, _I, _I64, _I, _I, _I64, _P, _P],
    "b200svd_upsample2x": [_P, _P, _I, _I, _I, _I, _P],
    "b200svd_timestep_embed": [_P, _I, _I, _F, _P, _I64, _P],
    "b200svd_add_silu": [_P, _P, _P, _I64, _I, _P],
    "b200svd_copy2d": [_P, _I64, _P, _I64, _I64, _I, _P],
    "b200svd_add_rows": [_P, _I64, _P, _I64, _I64, _I64, _I, _P],
    "b200svd_softmax_rows": [_P, _I64, _P, _I64, _I64, _I, _P],
    "b200svd_transpose": [_P, _I64, _P, _I64, _I, _I, _P],
    "b200svd_apm_mix": [_P, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P],
    "b200svd_sampler_prepare": [_P, _P, _I64, _I64, _F, _P],
    "b200svd_sampler_step": [_P, _P, _P, _I64, _I64, _I, _P, _F, _F, _F, _F, _P],
    "b200svd_gn_stats_partials": [_P, _P, _I64, _I64, _I, _I64, _P, _P, _P, _P],
    "b200svd_frames_to_uint8": [_P, _P, _I64, _I, _I64, _F, _F, _P],
    "b200svd_frames_quantize": [_P, _P, _I64, _P],
    "b200svd_ddim_blend_step": [_P, _P, _P, _I, _I, _I64, _I, _I, _I, _I, _I, _I, _F, _F, _F, _I, _P],
    "b200svd_vfi_window_attn": [_P, _I64, _P, _I64, _P, _I64, _P, _I64, _I, _I, _I, _I, _I, _F, _P],
    "b200svd_vfi_warp": [_P, _I, _I64, _I64, _I64, _I64, _P, _I64, _I64, _I64, _I64, _P, _I, _I64, _I64, _I64, _I64,
                         _I, _I, _I, _I, _P],
    "b200svd_vfi_resize": [_P, _I64, _I64, _I64, _I64, _P, _I, _I64, _I64, _I64, _I64, _I, _I, _I, _I, _I, _F, _I, _P],
    "b200svd_vfi_dwconv_gelu": [_P, _P, _I, _I, _I, _I, _P, _P, _P],
    "b200svd_vfi_head_gather": [_P, _I64, _P, _I64, _I, _I, _I, _I, _P, _I64, _P],
    "b200svd_vfi_merge": [_P, _P, _P, _P, _I64, _I, _I, _P, _P, _P],
    "b200svd_vfi_pair_input": [_P, _P, _I, _I, _P, _P, _P],
    "b200svd_vfi_frames_to_bgr": [_P, _I64, _I, _I, _P, _P],
    "b200svd_resize_bicubic_u8": [_P, _I64, _I, _I, _P, _I, _I, _P, _P, _I, _P, _P, _I, _P, _P],
}


def _declare(lib):
    for name, argtypes in PROTOTYPES.items():
        fn = getattr(lib, name)
        fn.restype = C.c_int
        fn.argtypes = argtypes


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = load().b200svd_last_error().decode("utf-8", "replace")
        raise B200Error(f"{what}: {msg}" if what else msg)


_inited = set()


def init(device: int = 0):
    if device in _inited:
        return
    lib = load()
    check(lib.b200svd_init(int(device)), "b200svd_init")
    _inited.add(device)
