"""Registers the hot-path operators with PyTorch's dispatcher under the reference's own schemas
(csrc/spmm.cpp:305-348, csrc/convert.cpp:46-48):

    torch.ops.tsb200.{spmm_sum, spmm_mean, spmm_min, spmm_max, ind2ptr, ptr2ind, cuda_version}
    torch.ops.tsb200.{coalesce, sort_perm, csr2csc, segment_reduce, spspmm, spmm_res, spmm_fp8, spmm_fp8_quant,
                      quantize_fp8, sddmm, sddmm_fp8, spmm_heads, sddmm_heads, spmm_multi, spmm_softmax_aggr,
                      segment_softmax}  (own)

and — unless a `torch_sparse` package is importable in this environment or TSB200_REGISTER_TORCH_SPARSE=0 —
the same operators as `torch.ops.torch_sparse.*`, so code that calls the reference's ops by name
(including TorchScript code: `torch.jit.script` functions can call these ops) keeps working on top of this package.
"""
from __future__ import annotations

import importlib.util
import logging
import os

import torch

from . import ops

_SCHEMAS = {
    "spmm_sum": "(Tensor? row, Tensor rowptr, Tensor col, Tensor? value, Tensor? colptr, Tensor? csr2csc, "
                "Tensor mat) -> Tensor",
    "spmm_mean": "(Tensor? row, Tensor rowptr, Tensor col, Tensor? value, Tensor? rowcount, Tensor? colptr, "
                 "Tensor? csr2csc, Tensor mat) -> Tensor",
    "spmm_min": "(Tensor rowptr, Tensor col, Tensor? value, Tensor mat) -> (Tensor, Tensor)",
    "spmm_max": "(Tensor rowptr, Tensor col, Tensor? value, Tensor mat) -> (Tensor, Tensor)",
    "ind2ptr": "(Tensor ind, int M) -> Tensor",
    "ptr2ind": "(Tensor ptr, int E) -> Tensor",
    "cuda_version": "() -> int",
}
# the rest of the native surface (no counterpart among the reference's registered ops, whose Python layer builds these
# from torch_scatter / torch.sparse.mm): registered under `tsb200` only, so TorchScript code can reach every kernel
_EXTRA_SCHEMAS = {
    # the reference's spmm_sum / spmm_mean plus the structure-only `row[csr2csc]` a caller may keep (SparseStorage.row_csc)
    "spmm_sum_csc": "(Tensor? row, Tensor rowptr, Tensor col, Tensor? value, Tensor? colptr, Tensor? csr2csc, "
                    "Tensor mat, Tensor? row_csc) -> Tensor",
    "spmm_mean_csc": "(Tensor? row, Tensor rowptr, Tensor col, Tensor? value, Tensor? rowcount, Tensor? colptr, "
                     "Tensor? csr2csc, Tensor mat, Tensor? row_csc) -> Tensor",
    "coalesce": "(Tensor row, Tensor col, Tensor? value, int M, int N, str reduce) -> (Tensor, Tensor, Tensor?)",
    "sort_perm": "(Tensor row, Tensor col, int M, int N) -> Tensor?",
    "csr2csc": "(Tensor row, Tensor col, int M, int N) -> (Tensor, Tensor, Tensor)",
    "segment_reduce": "(Tensor ptr, Tensor value, str reduce, Tensor? perm, Tensor? seg) -> Tensor",
    "spspmm": "(Tensor rowptrA, Tensor colA, Tensor? valueA, Tensor rowptrB, Tensor colB, Tensor? valueB, "
              "int M, int K, int N, bool want_value) -> (Tensor, Tensor, Tensor, Tensor?)",
    # residual / residual_scale: an e4m3 residual added to every row (sum / mean; tsb200_spmm_fw_fp8_res)
    "spmm_fp8": "(Tensor rowptr, Tensor col, Tensor? value, Tensor x8, Tensor scale, str reduce, "
                "ScalarType out_dtype, Tensor? residual=None, Tensor? residual_scale=None) -> (Tensor, Tensor?)",
    "spmm_fp8_quant": "(Tensor rowptr, Tensor col, Tensor? value, Tensor x8, Tensor scale, str reduce, "
                      "Tensor? residual=None, Tensor? residual_scale=None) -> (Tensor, Tensor, Tensor?)",
    "quantize_fp8": "(Tensor x, bool per_row) -> (Tensor, Tensor)",
    # per-entry dot products <a[row_e], b[col_e]>; colptr / csr2csc / row_csc (the CSC view) only for a gradient to b
    "sddmm": "(Tensor row, Tensor rowptr, Tensor col, Tensor? colptr, Tensor? csr2csc, Tensor? row_csc, Tensor a, "
             "Tensor b) -> Tensor",
    "sddmm_fp8": "(Tensor rowptr, Tensor col, Tensor a8, Tensor a_scale, Tensor b8, Tensor b_scale, "
                 "ScalarType out_dtype) -> Tensor",
    # spmm_sum_csc / spmm_mean_csc (reduce sum, add or mean) plus residual_scale * residual on every row, in one pass
    "spmm_res": "(Tensor? row, Tensor rowptr, Tensor col, Tensor? value, Tensor? rowcount, Tensor? colptr, "
                "Tensor? csr2csc, Tensor mat, Tensor? row_csc, Tensor residual, Tensor? residual_scale, str reduce) "
                "-> Tensor",
    # several aggregations (sum / add, mean, min, max, var, std) of every row's messages: [M, len(aggrs), K]
    "spmm_multi": "(Tensor? row, Tensor rowptr, Tensor col, Tensor? value, Tensor? colptr, Tensor? csr2csc, "
                  "Tensor mat, Tensor? row_csc, str[] aggrs) -> Tensor",
    # the softmax-weighted sum of every row's messages per column, with temperature t ([], [1] or [K]; None: 1)
    "spmm_softmax_aggr": "(Tensor rowptr, Tensor col, Tensor? value, Tensor? colptr, Tensor? csr2csc, Tensor mat, "
                         "Tensor? row_csc, Tensor? t) -> Tensor",
    # multi-head: value [E, H] over x [N, H, D]; scores [E, H] of a [M, H, D] and b [N, H, D]
    "spmm_heads": "(Tensor? row, Tensor rowptr, Tensor col, Tensor? value, Tensor? colptr, Tensor? csr2csc, "
                  "Tensor x, Tensor? row_csc) -> Tensor",
    "sddmm_heads": "(Tensor row, Tensor rowptr, Tensor col, Tensor? colptr, Tensor? csr2csc, Tensor? row_csc, "
                   "Tensor a, Tensor b) -> Tensor",
    # softmax of value [E, *] over each segment of ptr (rowptr, or colptr with perm = csr2csc), per trailing column
    "segment_softmax": "(Tensor ptr, Tensor value, Tensor? perm) -> Tensor",
}


def _csr2csc(row, col, M: int, N: int):
    perm, colptr, row_csc = ops.csr2csc(row, col, M, N, want_colptr=True, want_row_csc=True)
    return perm, colptr, row_csc


_EXTRA_IMPLS = {
    "spmm_sum_csc": ops.spmm_sum, "spmm_mean_csc": ops.spmm_mean, "spmm_res": ops.spmm_res, "spmm_multi": ops.spmm_multi,
    "spmm_softmax_aggr": ops.spmm_softmax_aggr,
    "coalesce": ops.coalesce, "sort_perm": ops.sort_perm, "csr2csc": _csr2csc,
    "segment_reduce": lambda ptr, value, reduce, perm, seg: ops.segment_reduce(ptr, value, reduce, perm, seg),
    "spspmm": ops.spspmm,
    "spmm_fp8": lambda rowptr, col, value, x8, scale, reduce, out_dtype, residual=None, residual_scale=None:
        ops.spmm_fw_fp8(rowptr, col, value, x8, scale, reduce, out_dtype, residual=residual,
                        residual_scale=residual_scale),
    "spmm_fp8_quant": lambda rowptr, col, value, x8, scale, reduce, residual=None, residual_scale=None:
        ops.spmm_fw_fp8_quant(rowptr, col, value, x8, scale, reduce, residual=residual, residual_scale=residual_scale),
    "quantize_fp8": ops.quantize_fp8,
    "sddmm": ops.sddmm, "sddmm_fp8": ops.sddmm_fp8,
    "spmm_heads": ops.spmm_heads, "sddmm_heads": ops.sddmm_heads,
    "segment_softmax": ops.segment_softmax,
}
_IMPLS = {
    "spmm_sum": ops.spmm_sum, "spmm_mean": ops.spmm_mean, "spmm_min": ops.spmm_min, "spmm_max": ops.spmm_max,
    "ind2ptr": ops.ind2ptr, "ptr2ind": ops.ptr2ind, "cuda_version": ops.cuda_version,
}
_LIBS = []  # keep Library objects alive
log = logging.getLogger(__name__)


def _register(ns: str, extra: bool = False) -> bool:
    """All-or-nothing: if any definition collides (a compiled torch_sparse already owns the namespace) the partial
    fragment is destroyed again, so the namespace is never left half registered."""
    lib = torch.library.Library(ns, "FRAGMENT")
    schemas, impls = dict(_SCHEMAS), dict(_IMPLS)
    if extra:
        schemas.update(_EXTRA_SCHEMAS)
        impls.update(_EXTRA_IMPLS)
    try:
        for name, schema in schemas.items():
            lib.define(name + schema)
            # the Python implementations wrap autograd.Functions, i.e. they are "composite implicit"
            lib.impl(name, impls[name], "CompositeImplicitAutograd")
    except Exception as e:
        lib._destroy()
        log.warning("pytorch_sparse_b200: torch.ops.%s.* not registered (%s)", ns, e)
        return False
    _LIBS.append(lib)
    return True


def _real_torch_sparse_present() -> bool:
    try:
        spec = importlib.util.find_spec("torch_sparse")
    except (ImportError, ValueError):
        return False
    return spec is not None


REGISTERED = {"tsb200": _register("tsb200", extra=True)}
# Aliasing into the reference's own namespace: on by default only when no `torch_sparse` package is importable
# (importing a compiled torch_sparse afterwards would collide with these definitions). TSB200_REGISTER_TORCH_SPARSE=1
# forces it (the reference-suite shim does), =0 forbids it.
_want = os.environ.get("TSB200_REGISTER_TORCH_SPARSE")
if _want == "1" or (_want is None and not _real_torch_sparse_present()):
    REGISTERED["torch_sparse"] = _register("torch_sparse")
else:
    REGISTERED["torch_sparse"] = False
