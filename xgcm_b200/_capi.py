"""ctypes binding of ``include/xgcm_b200.h`` — the only way numerics are reached.

There is deliberately NO fallback: if ``libxgcm_b200.so`` is missing or a call
fails, an exception is raised.  Status codes map onto the exception classes the
reference raises for the same conditions (SURVEY §8-b error conventions).
"""

from __future__ import annotations

import ctypes as C
from pathlib import Path
from typing import Optional, Sequence

LIB_PATH = Path(__file__).resolve().parent / "libxgcm_b200.so"

# enums of include/xgcm_b200.h
XG_F32, XG_F64 = 0, 1
OPS = {"diff": 0, "interp": 1, "min": 2, "max": 3}
BCS = {None: 0, "periodic": 1, "fill": 2, "extend": 3, "extrapolate": 4}
TRIMS = {"none": 0, "drop_last": 1, "drop_first": 2}
REDUCE = {"sum": 0, "mean": 1, "wvalid": 2}
BINOPS = {"mul": 0, "div": 1, "add": 2, "sub": 3, "divnz": 4}
XG_MAX_NDIM = 8
XG_HOST_GROUP_BASE = 1048576  # handles of xg_host_group: XG_HOST_GROUP_BASE + k

_EXC = {-1: ValueError, -2: NotImplementedError, -3: RuntimeError, -4: RuntimeError}

_i64p = C.POINTER(C.c_int64)
_i32p = C.POINTER(C.c_int)
_f64p = C.POINTER(C.c_double)
_vp = C.c_void_p
_vpp = C.POINTER(C.c_void_p)

# name -> (restype, argtypes); mirrors the header declaration by declaration
SIGNATURES = {
    "xg_version": (C.c_int, []),
    "xg_last_error": (C.c_char_p, []),
    "xg_launch_count": (C.c_longlong, []),
    "xg_last_launch": (C.c_char_p, []),
    "xg_device_info": (C.c_int, [C.c_int, C.POINTER(C.c_int), _i64p, _i64p]),
    "xg_stencil2": (
        C.c_int,
        [C.c_int, C.c_int, _vp, _vp, C.c_int, _i64p, C.c_int, C.c_int, C.c_int, C.c_int,
         C.c_double, _vp, _i64p, _vp, _i64p, _vp, _vp, _vp],
    ),
    "xg_stencil_multi": (
        C.c_int,
        [C.c_int, _vp, _vp, C.c_int, _i64p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int),
         C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_double), _vp],
    ),
    "xg_cumscan": (
        C.c_int,
        [C.c_int, _vp, _vp, C.c_int, _i64p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
         C.c_int, C.c_double, _vp, _i64p, _vp, _i64p, C.c_int, _vp],
    ),
    "xg_wreduce": (
        C.c_int,
        [C.c_int, _vp, _vp, _i64p, _vp, C.c_int, _i64p, C.c_int, C.c_int, C.c_int, _vp],
    ),
    "xg_vinterp_linear": (
        C.c_int,
        [C.c_int, _vp, _vp, _i64p, _vp, _i64p, C.c_int64, _vp, C.c_int, _i64p, C.c_int, C.c_int,
         C.c_int, C.c_int, _vp],
    ),
    "xg_vinterp_conservative": (
        C.c_int,
        [C.c_int, _vp, _vp, _i64p, _vp, C.c_int64, C.c_int, _vp, C.c_int, _i64p, C.c_int, _vp],
    ),
    "xg_pad": (
        C.c_int,
        [C.c_int, _vp, _vp, C.c_int, _i64p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, _vp],
    ),
    "xg_strided_copy": (C.c_int, [C.c_int, _vp, _i64p, _vp, _i64p, C.c_int, _i64p, C.c_int, _vp]),
    "xg_strided_copy_batch": (
        C.c_int,
        [C.c_int, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_int, _i64p, _i64p, _i64p,
         C.POINTER(C.c_int), _vp],
    ),
    "xg_fold_rows": (
        C.c_int,
        [C.c_int, _vp, _vp, C.c_int, _i64p, C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_int, C.c_int,
         C.c_int64, C.c_int64, C.c_int, _vp, _i64p, _vp],
    ),
    "xg_binary": (C.c_int, [C.c_int, C.c_int, _vp, _vp, _i64p, _vp, C.c_int, _i64p, _vp]),
    "xg_fill_uniform": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_uint64, C.c_uint64, _vp]),
    "xg_fill_uniform_host": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_uint64, C.c_uint64]),
    "xg_stencil2_host": (
        C.c_int,
        [C.c_int, C.c_int, _vp, _vp, C.c_int, _i64p, C.c_int, C.c_int, C.c_int, C.c_int,
         C.c_double, _vp, _i64p, _vp, _i64p, C.c_int],
    ),
    "xg_stencil2_host_fold": (
        C.c_int,
        [C.c_int, C.c_int, _vp, _vp, C.c_int, _i64p, C.c_int, C.c_int, C.c_int, C.c_int,
         C.c_double, _vp, _i64p, _vp, _i64p, C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_int, C.c_int],
    ),
    "xg_stencil2_host_connected": (
        C.c_int,
        [C.c_int, C.c_int, _vp, _vp, _i64p, _vp, C.c_int, _i64p, C.c_int, C.c_int, C.c_int, C.c_double,
         _vp, _i64p, C.c_int, C.c_int, _i32p, _i32p, _i64p, _i64p, _i64p, _i64p, _i64p, _i32p, C.c_int],
    ),
    "xg_host_workspace_bytes": (C.c_int, [C.c_int, _i64p]),
    "xg_host_group": (C.c_int, [C.c_int, _i32p, _i32p]),
    "xg_stencil2_host_multi": (
        C.c_int,
        [C.c_int, _i32p, C.c_int, _vp, _vpp, C.c_int, _i64p, _i32p, _i32p, _i32p, _i32p, _f64p, C.c_int],
    ),
    "xg_cumscan_host": (
        C.c_int,
        [C.c_int, _vp, _vp, C.c_int, _i64p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
         C.c_double, _vp, _i64p, _vp, _i64p, C.c_int, C.c_int],
    ),
    "xg_wreduce_host": (
        C.c_int,
        [C.c_int, _vp, _vp, _i64p, _vp, C.c_int, _i64p, C.c_int, C.c_int, C.c_int, C.c_int],
    ),
    "xg_vinterp_linear_host": (
        C.c_int,
        [C.c_int, _vp, _vp, _i64p, _vp, _i64p, C.c_int64, _vp, C.c_int, _i64p, C.c_int, C.c_int, C.c_int,
         C.c_int, C.c_int],
    ),
    "xg_vinterp_conservative_host": (
        C.c_int,
        [C.c_int, _vp, _vp, _i64p, C.c_int, _vp, C.c_int64, C.c_int, _vp, C.c_int, _i64p, C.c_int, C.c_int],
    ),
    "xg_stencil_multi_host": (
        C.c_int,
        [C.c_int, _vp, _vp, C.c_int, _i64p, C.c_int, _i32p, _i32p, _i32p, _i32p, _i32p, _f64p, C.c_int],
    ),
    "xg_wreduce_host_multi": (
        C.c_int,
        [C.c_int, _vp, _vp, _i64p, _vp, C.c_int, _i64p, C.c_int, _i32p, C.c_int, C.c_int, C.c_int],
    ),
    "xg_host_pipe_workspace_bytes": (C.c_int, [C.c_int, _i64p]),
    "xg_host_workspace_release": (C.c_int, []),
    "xg_stencil_pair": (
        C.c_int,
        [C.c_int, _vp, _vp, _vp, C.c_int, _i64p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, _vp, _i64p,
         C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, _vp, _i64p, C.c_int, _vp, _i64p, _vp],
    ),
    "xg_stencil_pair_halo": (
        C.c_int,
        [C.c_int, _vp, _vp, _vp, C.c_int, _i64p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, _vp, _i64p,
         C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, _vp, _i64p, C.c_int, _vp, _i64p, _vp, _vp, _vp],
    ),
    "xg_stencil_pair_host": (
        C.c_int,
        [C.c_int, _vp, _vp, _vp, C.c_int, _i64p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, _vp, _i64p,
         C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, _vp, _i64p, C.c_int, _vp, _i64p, C.c_int],
    ),
    "xg_stencil_pair_host_fold": (
        C.c_int,
        [C.c_int, _vp, _vp, _vp, C.c_int, _i64p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, _vp, _i64p,
         C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, _vp, _i64p, C.c_int, _vp, _i64p,
         C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_int, C.c_int],
    ),
    "xg_nccl_load": (C.c_int, [C.c_char_p]),
    "xg_comm_unique_id": (C.c_int, [_vp]),
    "xg_comm_init": (C.c_int, [_vp, C.c_int, C.c_int, _vpp]),
    "xg_comm_destroy": (C.c_int, [_vp]),
    "xg_halo_exchange": (C.c_int, [_vp, _vp, _vp, _vp, _vp, C.c_size_t, C.c_int, _vp]),
    "xg_stencil2_sharded": (
        C.c_int,
        [_vp, C.c_int, C.c_int, _vp, _vp, C.c_int, _i64p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double,
         _vp, _i64p, _vp, _i64p, _vp, C.c_size_t, _vp],
    ),
}

_lib: Optional[C.CDLL] = None


class LibraryMissingError(ImportError):
    pass


def load() -> C.CDLL:
    """Load the shared library (once) and attach the prototypes."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise LibraryMissingError(
            f"{LIB_PATH} not found. Build it with `python -m xgcm_b200._build` "
            "(needs nvcc). xgcm_b200 has no CPU fallback."
        )
    lib = C.CDLL(str(LIB_PATH))
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export it
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = lib
    return lib


def last_error() -> str:
    return load().xg_last_error().decode("utf-8", "replace")


def check(status: int) -> None:
    if status != 0:
        raise _EXC.get(status, RuntimeError)(last_error() or f"xgcm_b200 error {status}")


def i64_array(values: Optional[Sequence[int]]):
    if values is None:
        return None
    return (C.c_int64 * len(values))(*[int(v) for v in values])


def dtype_code(np_dtype) -> int:
    import numpy as np

    dt = np.dtype(np_dtype)
    if dt == np.float32:
        return XG_F32
    if dt == np.float64:
        return XG_F64
    raise TypeError(f"xgcm_b200 kernels support float32/float64 fields, got {dt}")


def last_launch() -> str:
    """Label of the kernel this thread launched last (xg_last_launch)."""
    return load().xg_last_launch().decode("utf-8", "replace")
