"""ctypes binding of libtsb200.so (the C-ABI declared in include/tsb200.h).

The library is the ONLY compute backend of this package: if it cannot be loaded the import fails
loudly (there is no CPU or PyTorch fallback for the hot path).
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_int, c_int64, c_size_t, c_void_p
from pathlib import Path

_PKG = Path(__file__).resolve().parent
LIB_PATH = Path(os.environ.get("TSB200_LIB", _PKG / "libtsb200.so"))

# (name, restype, argtypes) — must list every symbol declared in include/tsb200.h
SIGNATURES = {
    "tsb200_version": (c_int, []),
    "tsb200_strerror": (c_char_p, [c_int]),
    "tsb200_device_ok": (c_int, []),
    "tsb200_cuda_version": (c_int, []),
    "tsb200_sm_count": (c_int, []),
    "tsb200_spmm_fw_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int64, c_int64, c_int, c_int]),
    "tsb200_spmm_fw": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                               c_int64, c_int64, c_int64, c_int64, c_int64, c_int, c_int,
                               c_void_p, c_size_t, c_void_p]),
    "tsb200_spmm_plan_bytes": (c_size_t, [c_int64, c_int64]),
    "tsb200_spmm_plan": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_size_t, c_void_p, c_void_p]),
    "tsb200_spmm_fw_planned_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int64, c_int]),
    "tsb200_spmm_fw_planned": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                       c_int64, c_int64, c_int64, c_int64, c_int, c_int, c_void_p, c_size_t,
                                       c_int64, c_int64, c_int64, c_void_p, c_size_t, c_void_p]),
    "tsb200_spmm_fw_acc": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                   c_int64, c_int64, c_int64, c_int64, c_int64, c_int, c_void_p, c_size_t, c_void_p]),
    "tsb200_spmm_value_bw_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int64, c_int64, c_int]),
    "tsb200_spmm_value_bw": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_int64, c_int64, c_int64, c_int64, c_int64, c_int, c_int,
                                     c_void_p, c_size_t, c_void_p]),
    "tsb200_spmm_minmax_bw": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_int64, c_int64, c_int64, c_int64, c_int64, c_int, c_void_p]),
    "tsb200_ind2ptr": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_void_p]),
    "tsb200_ptr2ind": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_void_p]),
    "tsb200_csr2csc_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int64]),
    "tsb200_csr2csc": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_void_p,
                               c_void_p, c_size_t, c_void_p]),
    "tsb200_coalesce_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int64]),
    "tsb200_coalesce_sort": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_size_t,
                                     c_void_p, c_void_p]),
    "tsb200_coalesce_emit": (c_int, [c_int64, c_int64, c_int64, c_void_p, c_int64, c_int, c_int,
                                     c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_void_p]),
    "tsb200_coalesce_perm": (c_int, [c_int64, c_void_p, c_void_p, c_void_p]),
    "tsb200_segment_reduce": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int, c_int,
                                      c_void_p]),
    "tsb200_segment_reduce_bw": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64,
                                         c_int, c_int, c_void_p]),
    "tsb200_spspmm_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int64, c_int64, c_int64]),
    "tsb200_spspmm_symbolic": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64,
                                       c_int64, c_int64, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    "tsb200_spspmm_numeric": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p,
                                      c_void_p, c_void_p, c_int, c_void_p, c_size_t, c_void_p]),
    "tsb200_spspmm_bound": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_size_t, c_void_p, c_void_p]),
    "tsb200_spspmm_fused": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_int64, c_int, c_void_p, c_size_t, c_void_p, c_void_p]),
    "tsb200_spmm_fw_host": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_int64, c_int64, c_int64, c_int64, c_int64, c_int, c_int]),
}


class Tsb200Error(RuntimeError):
    pass


def _load() -> ctypes.CDLL:
    if not LIB_PATH.exists():
        raise ImportError(
            f"pytorch_sparse_b200: {LIB_PATH} is missing. Build it with "
            f"`python build_native.py` (needs nvcc, sm_90a). There is no fallback path.")
    try:
        lib = ctypes.CDLL(str(LIB_PATH), mode=ctypes.RTLD_GLOBAL)
    except OSError as e:  # pragma: no cover
        raise ImportError(f"pytorch_sparse_b200: cannot load {LIB_PATH}: {e}") from e
    for name, (restype, argtypes) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:
            raise ImportError(f"pytorch_sparse_b200: {LIB_PATH} does not export {name}") from e
        fn.restype = restype
        fn.argtypes = argtypes
    return lib


lib = _load()


def strerror(code: int) -> str:
    return lib.tsb200_strerror(code).decode()


def check(code: int, what: str) -> None:
    if code != 0:
        raise Tsb200Error(f"{what} failed: {strerror(code)} (code {code})")
