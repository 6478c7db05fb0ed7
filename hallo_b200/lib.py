"""ctypes binding of the C-ABI library (include/hallo_b200.h).

The product path has no CPU or PyTorch fallback: if ``libhallo_b200.so`` is missing or a call
fails, a ``RuntimeError`` is raised (north_star: "no CPU fallback").
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
# HALLO_B200_LIB: load another build of the same sources
LIB_PATH = os.environ.get("HALLO_B200_LIB") or os.path.join(_HERE, "libhallo_b200.so")

HB_F16, HB_BF16 = 0, 1
HB_EPI_GEGLU = 1
HB_EPI_SILU = 2
HB_EPI_RELU = 4


class GemmParams(C.Structure):
    _fields_ = [
        ("dtype", C.c_int32),
        ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
        ("A", C.c_void_p), ("lda", C.c_int64),
        ("A2", C.c_void_p), ("lda2", C.c_int64), ("K1", C.c_int32),
        ("W", C.c_void_p), ("ldw", C.c_int64),
        ("C", C.c_void_p), ("ldc", C.c_int64),
        ("bias", C.c_void_p),
        ("group_bias", C.c_void_p), ("ld_group_bias", C.c_int64), ("rows_per_group", C.c_int32),
        ("row_scale", C.c_void_p),
        ("residual", C.c_void_p), ("ldr", C.c_int64),
        ("alpha", C.c_float),
        ("flags", C.c_int32),
        ("conv3x3", C.c_int32),
        ("img_n", C.c_int32), ("img_h", C.c_int32), ("img_w", C.c_int32),
        ("ln_stats", C.c_void_p), ("ln_colsum", C.c_void_p), ("ln_eps", C.c_float),
        ("stats_out", C.c_void_p),
        ("scatter", C.c_void_p),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_int64),
    ]


class RowScatter(C.Structure):
    """hb_row_scatter (include/hallo_b200.h): output rows of a GEMM stored into per-destination (peer-mapped) buffers."""
    _fields_ = [("base", C.c_void_p * 16), ("seg", C.c_int32), ("segs_per_dest", C.c_int32),
                ("seg_stride", C.c_int64), ("row0", C.c_int64)]


class AttentionParams(C.Structure):
    _fields_ = [
        ("dtype", C.c_int32), ("head_dim", C.c_int32), ("heads", C.c_int32),
        ("L", C.c_int32), ("frames", C.c_int32),
        ("Q", C.c_void_p), ("ldq", C.c_int64),
        ("K", C.c_void_p), ("ldk", C.c_int64),
        ("V", C.c_void_p), ("ldv", C.c_int64),
        ("Kref", C.c_void_p), ("ldkref", C.c_int64),
        ("Vref", C.c_void_p), ("ldvref", C.c_int64),
        ("ref_frames", C.c_int32),
        ("ref_index", C.c_void_p),
        ("O", C.c_void_p), ("ldo", C.c_int64),
    ]


_lib: Optional[C.CDLL] = None


def load() -> C.CDLL:
    """Load the shared library; raises if it has not been built (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'`. "
            "hallo_b200 has no CPU / PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    lib.hallo_b200_abi_version.restype = C.c_int
    lib.hallo_b200_last_error.restype = C.c_char_p
    lib.hallo_b200_launch_count.restype = C.c_int64
    lib.hallo_b200_launch_count.argtypes = [C.c_int]
    lib.hallo_b200_device_error.argtypes = [C.POINTER(C.c_uint)]
    lib.hallo_b200_set_option.argtypes = [C.c_char_p, C.c_int]
    lib.hallo_b200_get_option.argtypes = [C.c_char_p]
    lib.hallo_b200_gemm_workspace_bytes.restype = C.c_int64
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().hallo_b200_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"hallo_b200 {what} failed (status {rc}): {msg}")


def dtype_code(torch_dtype) -> int:
    import torch
    if torch_dtype == torch.float16:
        return HB_F16
    if torch_dtype == torch.bfloat16:
        return HB_BF16
    raise RuntimeError(f"hallo_b200 supports fp16/bf16 storage only, got {torch_dtype}")


def ptr(t) -> Optional[int]:
    return None if t is None else t.data_ptr()


def current_stream() -> C.c_void_p:
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def launch_count(reset: bool = False) -> int:
    return int(load().hallo_b200_launch_count(1 if reset else 0))


def set_option(name: str, value: int) -> None:
    """Kernel-selection switch (include/hallo_b200.h: hallo_b200_set_option); read at launch / graph-capture time."""
    check(load().hallo_b200_set_option(name.encode(), int(value)), f"set_option({name})")


def get_option(name: str) -> int:
    v = int(load().hallo_b200_get_option(name.encode()))
    if v < 0:
        raise KeyError(name)
    return v


def device_error() -> int:
    code = C.c_uint(0)
    load().hallo_b200_device_error(C.byref(code))
    return int(code.value)
