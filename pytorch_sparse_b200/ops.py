"""Tensor-level operators over the libtsb200 C-ABI.

This module is the Python mirror of the reference's native operator layer
(`torch.ops.torch_sparse.*`, csrc/spmm.cpp:305-348, csrc/convert.cpp:22-48): same names, argument
meaning, optional-argument rules and error behaviour, with every computation done by the CUDA
library. All functions require CUDA tensors and raise a RuntimeError for CPU tensors (like the
reference's CHECK_CUDA, csrc/cuda/utils.cuh:5-6) — there is no CPU path.
"""
from __future__ import annotations

import collections
import ctypes
import os
from typing import List, Optional, Tuple

import torch
from torch import Tensor

from . import _lib
from ._lib import check, lib

_DTYPES = {
    torch.float32: 0, torch.float64: 1, torch.float16: 2, torch.bfloat16: 3,
    torch.int32: 4, torch.int64: 5, torch.int16: 6, torch.int8: 7, torch.uint8: 8,
}
_REDUCE = {"sum": 0, "add": 0, "mean": 1, "min": 2, "max": 3}


def _dtype_code(dtype: torch.dtype) -> int:
    try:
        return _DTYPES[dtype]
    except KeyError:
        raise RuntimeError(f'"spmm" not implemented for \'{dtype}\'') from None


def _reduce_code(reduce: str) -> int:
    try:
        return _REDUCE[reduce]
    except KeyError:
        raise ValueError(f"unknown reduce '{reduce}'") from None


def _p(t: Optional[Tensor]):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _stream(device: torch.device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _check_cuda(t: Tensor, name: str) -> None:
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be CUDA tensor")


def _check_input(cond: bool) -> None:
    if not cond:
        raise RuntimeError("Input mismatch")


class _on_device:
    """`with torch.cuda.device(dev)` costs several microseconds per call; skip it when `dev` is current."""
    __slots__ = ("ctx",)

    def __init__(self, dev: torch.device):
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        self.ctx = None if torch.cuda.current_device() == idx else torch.cuda.device(idx)

    def __enter__(self):
        if self.ctx is not None:
            self.ctx.__enter__()

    def __exit__(self, *exc):
        if self.ctx is not None:
            self.ctx.__exit__(*exc)
        return False


def _workspace(nbytes: int, device: torch.device) -> Optional[Tensor]:
    if nbytes <= 0:
        return None
    return torch.empty(nbytes, dtype=torch.uint8, device=device)


def _i64(t: Tensor, name: str) -> Tensor:
    if t.dtype != torch.int64:
        raise RuntimeError(f"{name} must be int64")
    return t.contiguous()


# --------------------------------------------------------------------------------------------------
# SpMM forward / value gradient / fused min-max backward
# --------------------------------------------------------------------------------------------------
class SpmmPlan:
    """The segment structure of one CSR matrix (tsb200_spmm_plan): which rows are cut into segments, the segment list
    and the multi-segment rows. Depends on `rowptr` only — build it once per matrix and pass it to `spmm_fw`."""
    __slots__ = ("data", "M", "E", "n_seg", "n_long", "n_slot")

    def __init__(self, rowptr: Tensor, E: int):
        _check_cuda(rowptr, "rowptr")
        rowptr = _i64(rowptr, "rowptr")
        self.M, self.E = rowptr.numel() - 1, int(E)
        dev = rowptr.device
        with _on_device(dev):
            nbytes = lib.tsb200_spmm_plan_bytes(self.M, self.E)
            self.data = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            counts = (ctypes.c_int64 * 3)()
            check(lib.tsb200_spmm_plan(_p(rowptr), self.M, self.E, _p(self.data), nbytes, counts, _stream(dev)),
                  "tsb200_spmm_plan")
        self.n_seg, self.n_long, self.n_slot = int(counts[0]), int(counts[1]), int(counts[2])


def spmm_plan(rowptr: Tensor, E: int) -> SpmmPlan:
    return SpmmPlan(rowptr, E)


# Plans are structure-only, so they are kept per `rowptr` tensor like the reference keeps csr2csc / colptr per storage:
# the second product with the same rowptr builds the plan (0.2 ms + one stream synchronisation, like the first csr2csc),
# every later one uses it. The key is the tensor's storage, offset, extent and version counter; the entry holds a
# reference to the storage, so its address cannot be recycled for another tensor while the entry lives.
_PLAN_CACHE: "collections.OrderedDict" = collections.OrderedDict()
_PLAN_CACHE_MAX = 16


def _auto_plan(rowptr: Tensor, E: int) -> Optional[SpmmPlan]:
    if os.environ.get("TSB200_AUTO_PLAN", "1") == "0":
        return None
    try:
        st = rowptr.untyped_storage()
        key = (st._cdata, rowptr.storage_offset(), rowptr.numel(), rowptr._version, int(E), rowptr.device.index)
    except RuntimeError:      # e.g. inference tensors keep no version counter
        return None
    ent = _PLAN_CACHE.get(key)
    if ent is None:
        _PLAN_CACHE[key] = [st, None]
        while len(_PLAN_CACHE) > _PLAN_CACHE_MAX:
            _PLAN_CACHE.popitem(last=False)
        return None
    _PLAN_CACHE.move_to_end(key)
    if ent[1] is None:
        if torch.cuda.is_current_stream_capturing():   # building a plan synchronises the stream
            return None
        ent[1] = SpmmPlan(rowptr, E)
    return ent[1]


def spmm_fw(rowptr: Tensor, col: Tensor, value: Optional[Tensor], mat: Tensor,
            reduce: str, plan: Optional[SpmmPlan] = None) -> Tuple[Tensor, Optional[Tensor]]:
    """`spmm_fw(rowptr, col, optional_value, mat, reduce) -> (out, arg_out?)`
    (csrc/spmm.cpp:22-35; checks follow csrc/cuda/spmm_cuda.cu:97-110). With a `plan` (spmm_plan(rowptr, E)) the
    product is one memset + one kernel (tsb200_spmm_fw_planned). min/max results and arg_out are the same as without
    a plan, and so are sums over dense rows wider than 128 bytes. For narrower rows a sum can differ in the last bits
    (within the same rounding bound) on rows the plan defers for the nnz budget of their 32-row group, when the
    unplanned call uses smaller work items (matrices of fewer than about 500k rows): such a row is summed by several
    lane groups instead of one."""
    _check_cuda(rowptr, "rowptr")
    _check_cuda(col, "col")
    if value is not None:
        _check_cuda(value, "optional_value.value()")
    _check_cuda(mat, "mat")
    _check_input(rowptr.dim() == 1)
    _check_input(col.dim() == 1)
    if value is not None:
        _check_input(value.dim() == 1)
        _check_input(value.size(0) == col.size(0))
        if value.dtype != mat.dtype:
            raise RuntimeError(f"expected value of dtype {mat.dtype} but got {value.dtype}")
        value = value.contiguous()
    _check_input(mat.dim() >= 2)
    red = _reduce_code(reduce)
    rowptr = _i64(rowptr, "rowptr")
    col = _i64(col, "col")
    mat = mat.contiguous()
    dt = _dtype_code(mat.dtype)

    M = rowptr.numel() - 1
    N, K = mat.size(-2), mat.size(-1)
    B = mat.numel() // (N * K) if N * K > 0 else int(torch.Size(mat.shape[:-2]).numel())
    E = col.numel()
    sizes = list(mat.shape)
    sizes[-2] = M
    dev = mat.device
    out = torch.empty(sizes, dtype=mat.dtype, device=dev)
    arg_out = torch.empty(sizes, dtype=torch.int64, device=dev) if red >= 2 else None
    if out.numel() == 0:
        return out, arg_out
    if E == 0:
        out.zero_()
        if arg_out is not None:
            arg_out.fill_(0)
        return out, arg_out
    with _on_device(dev):
        plannable = B == 1 and dt in (0, 2, 3) and (K * mat.element_size()) % 16 == 0
        pl, ws, nws = _plan_workspace(plan, plannable, rowptr, B, M, K, E, dt, red, dev)
        if pl[0] is not None:
            rc = lib.tsb200_spmm_fw_planned(_p(rowptr), _p(col), _p(value), _p(mat), _p(out), _p(arg_out), M, N, K, E,
                                            dt, red, *pl, _p(ws), nws, _stream(dev))
            if rc != -2:   # TSB200_ERR_UNSUPPORTED (alignment): fall through to the unplanned call
                check(rc, "tsb200_spmm_fw_planned")
                return out, arg_out
            pl, ws, nws = _plan_workspace(None, False, rowptr, B, M, K, E, dt, red, dev)
        check(lib.tsb200_spmm_fw(_p(rowptr), _p(col), _p(value), _p(mat), _p(out), _p(arg_out),
                                 B, M, N, K, E, dt, red, _p(ws), nws, _stream(dev)), "tsb200_spmm_fw")
    return out, arg_out


def _plan_workspace(plan: Optional[SpmmPlan], plannable: bool, rowptr: Tensor, B: int, M: int, K: int, E: int,
                    dt: int, red: int, dev: torch.device):
    """The plan and the workspace of one SpMM forward. A plannable product uses the given plan, else the one cached
    for `rowptr`, and only if it was built for these M and E. Returns (plan arguments, workspace, workspace bytes);
    the plan arguments are (plan, plan_bytes, n_seg, n_long, n_slot), with plan None for an unplanned call."""
    if plannable and plan is None:
        plan = _auto_plan(rowptr, E)
    if plannable and plan is not None and plan.M == M and plan.E == E:
        nws = lib.tsb200_spmm_fw_planned_workspace_bytes(K, plan.n_long, plan.n_slot, red)
        pl = (_p(plan.data), plan.data.numel(), plan.n_seg, plan.n_long, plan.n_slot)
    else:
        nws = lib.tsb200_spmm_fw_workspace_bytes(B, M, K, E, dt, red)
        pl = (None, 0, 0, 0, 0)
    return pl, _workspace(nws, dev), nws


_ONE = {}  # a scalar 1 per (device, dtype): the scale of a residual passed without one


def _res_args(what: str, residual: Tensor, residual_scale: Optional[Tensor], mat: Tensor, M: int, red: int):
    """The checks of the residual of spmm_fw_res; returns (residual_scale, residual_scale_stride)."""
    _check_cuda(residual, "residual")
    if red >= 2:
        raise RuntimeError(f"{what}: a residual is only added to reduce='sum' / 'mean' results, not min / max")
    if mat.dim() != 2:
        raise RuntimeError(f"{what}: a residual needs a 2-D dense operand [N, K], got {mat.dim()}-D")
    if residual.device != mat.device:
        raise RuntimeError(f"{what}: residual must be on the device of the dense operand ({mat.device})")
    if residual.dtype != mat.dtype:
        raise RuntimeError(f"{what}: residual must have the dense operand's dtype {mat.dtype}, got {residual.dtype}")
    K = mat.size(1)
    if residual.dim() != 2 or residual.size(0) != M or residual.size(1) != K:
        raise RuntimeError(f"{what}: residual must have the result's shape [M, K] = [{M}, {K}], "
                           f"got {list(residual.shape)}")
    if not residual.is_contiguous():
        raise RuntimeError(f"{what}: residual must be contiguous")
    sdt = torch.float64 if mat.dtype == torch.float64 else torch.float32
    if residual_scale is None:
        key = (mat.device, sdt)
        one = _ONE.get(key)
        if one is None:
            one = _ONE[key] = torch.ones((), dtype=sdt, device=mat.device)
        return one, 0
    _check_cuda(residual_scale, "residual_scale")
    if residual_scale.device != mat.device:
        raise RuntimeError(f"{what}: residual_scale must be on the device of the dense operand ({mat.device})")
    if residual_scale.dtype != sdt:
        raise RuntimeError(f"{what}: residual_scale must be {sdt} for a {mat.dtype} operand, got {residual_scale.dtype}")
    if residual_scale.dim() == 0:
        stride = 0
    elif residual_scale.dim() == 1 and residual_scale.size(0) == M:
        stride = 1
    else:
        raise RuntimeError(f"{what}: residual_scale must have shape [] or [M] = [{M}], "
                           f"got {list(residual_scale.shape)}")
    return residual_scale.contiguous(), stride


def spmm_fw_res(rowptr: Tensor, col: Tensor, value: Optional[Tensor], mat: Tensor, residual: Tensor,
                residual_scale: Optional[Tensor] = None, reduce: str = "sum",
                plan: Optional[SpmmPlan] = None) -> Tensor:
    """`spmm_fw(rowptr, col, value, mat, reduce)` plus `residual_scale[m] * residual[m]` on every row m, added in the
    kernels' store epilogue (tsb200_spmm_fw_res): out = round(fl(y + fl(s * r))) with y the fp32 (fp64) row result
    `spmm_fw` computes on the same path, one IEEE product and one IEEE add. `mat` is 2-D [N, K] (bf16, f16, f32, f64),
    `residual` [M, K] contiguous in its dtype, `residual_scale` None (1) or float32 (float64 for f64) of shape [] or
    [M]; reduce sum / add / mean. Planned like `spmm_fw` (the same per-rowptr plan cache). Forward only: see SPMMRes."""
    _check_cuda(rowptr, "rowptr")
    _check_cuda(col, "col")
    if value is not None:
        _check_cuda(value, "optional_value.value()")
    _check_cuda(mat, "mat")
    red = _reduce_code(reduce)
    M = rowptr.numel() - 1
    scale, stride = _res_args("spmm_res", residual, residual_scale, mat, M, red)
    _check_input(rowptr.dim() == 1)
    _check_input(col.dim() == 1)
    if value is not None:
        _check_input(value.dim() == 1)
        _check_input(value.size(0) == col.size(0))
        if value.dtype != mat.dtype:
            raise RuntimeError(f"expected value of dtype {mat.dtype} but got {value.dtype}")
        value = value.contiguous()
    rowptr = _i64(rowptr, "rowptr")
    col = _i64(col, "col")
    mat = mat.contiguous()
    dt = _dtype_code(mat.dtype)
    N, K = mat.shape
    E = col.numel()
    dev = mat.device
    out = torch.empty(M, K, dtype=mat.dtype, device=dev)
    if out.numel() == 0:
        return out
    with _on_device(dev):
        plannable = E > 0 and dt in (0, 2, 3) and (K * mat.element_size()) % 16 == 0
        pl, ws, nws = _plan_workspace(plan, plannable, rowptr, 1, M, K, E, dt, red, dev)
        check(lib.tsb200_spmm_fw_res(_p(rowptr), _p(col), _p(value), _p(mat), _p(residual), _p(scale), stride,
                                     _p(out), M, N, K, E, dt, red, *pl, _p(ws), nws, _stream(dev)),
              "tsb200_spmm_fw_res")
    return out


# aggregator codes of tsb200_spmm_fw_multi: the reduce codes plus TSB200_VAR / TSB200_STD
_AGGR = {"sum": 0, "add": 0, "mean": 1, "min": 2, "max": 3, "var": 4, "std": 5}


def _aggr_codes(aggrs: List[str]) -> List[int]:
    if len(aggrs) == 0:
        raise ValueError("spmm_multi: aggrs must name at least one aggregator")
    codes: List[int] = []
    for a in aggrs:
        c = _AGGR.get(a)
        if c is None:
            raise ValueError(f"spmm_multi: unknown aggregator '{a}' (expected sum, add, mean, min, max, var or std)")
        if c in codes:
            raise ValueError(f"spmm_multi: aggregator '{a}' is given more than once")
        codes.append(c)
    return codes


def _spmm_fw_multi(rowptr: Tensor, col: Tensor, value: Optional[Tensor], mat: Tensor, codes: List[int],
                   want_args: bool, plan: Optional[SpmmPlan] = None):
    _check_cuda(rowptr, "rowptr")
    _check_cuda(col, "col")
    if value is not None:
        _check_cuda(value, "optional_value.value()")
    _check_cuda(mat, "mat")
    if mat.dim() != 2:
        raise RuntimeError(f"spmm_multi: the dense operand must be 2-D [N, K], got {mat.dim()}-D")
    _check_input(rowptr.dim() == 1)
    _check_input(col.dim() == 1)
    if value is not None:
        _check_input(value.dim() == 1)
        _check_input(value.size(0) == col.size(0))
        if value.dtype != mat.dtype:
            raise RuntimeError(f"expected value of dtype {mat.dtype} but got {value.dtype}")
        value = value.contiguous()
    rowptr = _i64(rowptr, "rowptr")
    col = _i64(col, "col")
    mat = mat.contiguous()
    dt = _dtype_code(mat.dtype)
    M = rowptr.numel() - 1
    N, K = mat.shape
    E = col.numel()
    dev = mat.device
    out = torch.empty(M, len(codes), K, dtype=mat.dtype, device=dev)
    arg_min = torch.empty(M, K, dtype=torch.int64, device=dev) if want_args and 2 in codes else None
    arg_max = torch.empty(M, K, dtype=torch.int64, device=dev) if want_args and 3 in codes else None
    if out.numel() == 0:
        return out, arg_min, arg_max
    with _on_device(dev):
        plannable = E > 0 and dt in (0, 2, 3) and (K * mat.element_size()) % 16 == 0
        if plannable and plan is None:
            plan = _auto_plan(rowptr, E)
        if plannable and plan is not None and plan.M == M and plan.E == E:
            nws = lib.tsb200_spmm_fw_multi_workspace_bytes(K, E, 1, plan.n_long, plan.n_slot)
            pl = (_p(plan.data), plan.data.numel(), plan.n_seg, plan.n_long, plan.n_slot)
        else:
            nws = lib.tsb200_spmm_fw_multi_workspace_bytes(K, E, 0, 0, 0)
            pl = (None, 0, 0, 0, 0)
        ws = _workspace(nws, dev)
        check(lib.tsb200_spmm_fw_multi(_p(rowptr), _p(col), _p(value), _p(mat), (ctypes.c_int * len(codes))(*codes),
                                       len(codes), _p(out), _p(arg_min), _p(arg_max), M, N, K, E, dt, *pl, _p(ws), nws,
                                       _stream(dev)), "tsb200_spmm_fw_multi")
    return out, arg_min, arg_max


def spmm_fw_multi(rowptr: Tensor, col: Tensor, value: Optional[Tensor], mat: Tensor, aggrs: List[str],
                  want_args: bool = False,
                  plan: Optional[SpmmPlan] = None) -> Tuple[Tensor, Optional[Tensor], Optional[Tensor]]:
    """`out [M, A, K]`: aggregator aggrs[a] (sum / add, mean, min, max, var, std) of every row's messages
    value[e] * mat[col[e]] in out[:, a], from one gather pass (tsb200_spmm_fw_multi). The sum, mean, min and max
    slices are bit for bit `spmm_fw`'s on the same path. var = max(Q / n - mean^2, 0) with Q the fp32 (fp64) sum of
    squared messages and n = max(degree, 1); std = sqrt(var) where var > 1e-5, else 0. `mat` is 2-D [N, K] (bf16,
    f16, f32, f64). want_args: also return arg_min / arg_max [M, K] (None for an aggregator not requested), as
    `spmm_fw` returns arg_out. Planned like `spmm_fw` (the same per-rowptr plan cache). Forward only: see SPMMMulti."""
    return _spmm_fw_multi(rowptr, col, value, mat, _aggr_codes(aggrs), want_args, plan)


def _smx_t(t: Tensor, mat: Tensor) -> int:
    """The checks of a softmax aggregation's temperature; returns its stride (0: one scalar, 1: one per column)."""
    _check_cuda(t, "t")
    acc = torch.float64 if mat.dtype == torch.float64 else torch.float32
    if t.device != mat.device:
        raise RuntimeError(f"spmm_softmax_aggr: t must be on the device of the dense operand ({mat.device})")
    if t.dtype != acc:
        raise RuntimeError(f"spmm_softmax_aggr: t must be {acc} for a {mat.dtype} operand, got {t.dtype}")
    K = mat.size(-1)
    if t.dim() == 0 or (t.dim() == 1 and t.size(0) == 1):
        return 0
    if t.dim() == 1 and t.size(0) == K:
        return 1
    raise RuntimeError(f"spmm_softmax_aggr: t must have shape [], [1] or [K] = [{K}], got {list(t.shape)}")


def _smx_operands(rowptr: Tensor, col: Tensor, value: Optional[Tensor], mat: Tensor):
    _check_cuda(rowptr, "rowptr")
    _check_cuda(col, "col")
    if value is not None:
        _check_cuda(value, "optional_value.value()")
    _check_cuda(mat, "mat")
    if mat.dim() != 2:
        raise RuntimeError(f"spmm_softmax_aggr: the dense operand must be 2-D [N, K], got {mat.dim()}-D")
    _check_input(rowptr.dim() == 1)
    _check_input(col.dim() == 1)
    if value is not None:
        _check_input(value.dim() == 1)
        _check_input(value.size(0) == col.size(0))
        if value.dtype != mat.dtype:
            raise RuntimeError(f"expected value of dtype {mat.dtype} but got {value.dtype}")
        value = value.contiguous()
    return _i64(rowptr, "rowptr"), _i64(col, "col"), value, mat.contiguous()


def spmm_fw_softmax_aggr(rowptr: Tensor, col: Tensor, value: Optional[Tensor], mat: Tensor, t: Tensor,
                         want_lse: bool = False,
                         plan: Optional[SpmmPlan] = None) -> Tuple[Tensor, Optional[Tensor]]:
    """`(out [M, K], lse [M, K]?)`: per row m and column k the messages p_e = value[e] * mat[col[e], k] summed with
    the weights softmax_e(t_k p_e) over the row's entries (tsb200_spmm_fw_softmax_aggr), and lse = max_e t_k p_e +
    log(sum_e exp(t_k p_e - max)) in fp32 (fp64 for f64) when want_lse. `mat` is 2-D [N, K] (bf16, f16, f32, f64); `t`
    has the accumulator dtype (float32, float64 for f64) and shape [] or [1] (one temperature) or [K] (one per column).
    An empty row gives 0 (lse -inf). With t = 0 the result is bit for bit `spmm_fw(..., "mean")` on the same path for
    bf16 / f16, and for f32 without values. Planned like `spmm_fw` (the same per-rowptr plan cache). Forward only: see
    SPMMSoftmaxAggr."""
    rowptr, col, value, mat = _smx_operands(rowptr, col, value, mat)
    stride = _smx_t(t, mat)
    t = t.contiguous()
    dt = _dtype_code(mat.dtype)
    M = rowptr.numel() - 1
    N, K = mat.shape
    E = col.numel()
    dev = mat.device
    out = torch.empty(M, K, dtype=mat.dtype, device=dev)
    lse = torch.empty(M, K, dtype=t.dtype, device=dev) if want_lse else None
    if out.numel() == 0:
        return out, lse
    with _on_device(dev):
        plannable = E > 0 and dt in (0, 2, 3) and (K * mat.element_size()) % 16 == 0
        if plannable and plan is None:
            plan = _auto_plan(rowptr, E)
        if plannable and plan is not None and plan.M == M and plan.E == E:
            nws = lib.tsb200_spmm_fw_softmax_aggr_workspace_bytes(K, E, 1, plan.n_long, plan.n_slot)
            pl = (_p(plan.data), plan.data.numel(), plan.n_seg, plan.n_long, plan.n_slot)
        else:
            nws = lib.tsb200_spmm_fw_softmax_aggr_workspace_bytes(K, E, 0, 0, 0)
            pl = (None, 0, 0, 0, 0)
        ws = _workspace(nws, dev)
        check(lib.tsb200_spmm_fw_softmax_aggr(_p(rowptr), _p(col), _p(value), _p(mat), _p(t), stride, _p(out),
                                              _p(lse), M, N, K, E, dt, *pl, _p(ws), nws, _stream(dev)),
              "tsb200_spmm_fw_softmax_aggr")
    return out, lse


def spmm_softmax_aggr_bw_rows(rowptr: Tensor, col: Tensor, value: Optional[Tensor], mat: Tensor, t: Tensor,
                              grad_out: Tensor, out: Tensor, lse: Tensor, want_value: bool,
                              want_t: bool) -> Tuple[Optional[Tensor], Optional[Tensor]]:
    """The row-wise backward of `spmm_fw_softmax_aggr` (tsb200_spmm_softmax_aggr_bw_rows): `(grad_value [E]?, U
    [M, K]?)` with U[r, k] = g[r, k] sum_e alpha_e (p_e - out[r, k])^2 in t's dtype, whose column sums are the
    temperature's gradient."""
    rowptr, col, value, mat = _smx_operands(rowptr, col, value, mat)
    stride = _smx_t(t, mat)
    M = rowptr.numel() - 1
    N, K = mat.shape
    E = col.numel()
    dev = mat.device
    gv = torch.empty(E, dtype=mat.dtype, device=dev) if want_value and value is not None else None
    U = torch.empty(M, K, dtype=t.dtype, device=dev) if want_t else None
    with _on_device(dev):
        nws = lib.tsb200_spmm_softmax_aggr_bw_workspace_bytes(K, E)
        ws = _workspace(nws, dev)
        check(lib.tsb200_spmm_softmax_aggr_bw_rows(_p(rowptr), _p(col), _p(value), _p(mat), _p(t.contiguous()),
                                                   stride, _p(grad_out.contiguous()), _p(out), _p(lse), _p(gv), _p(U),
                                                   M, N, K, E, _dtype_code(mat.dtype), _p(ws), nws, _stream(dev)),
              "tsb200_spmm_softmax_aggr_bw_rows")
    return gv, U


def spmm_softmax_aggr_bw_cols(colptr: Tensor, row_csc: Tensor, value_csc: Optional[Tensor], mat: Tensor, t: Tensor,
                              grad_out: Tensor, out: Tensor, lse: Tensor) -> Tensor:
    """The column-wise backward of `spmm_fw_softmax_aggr` (tsb200_spmm_softmax_aggr_bw_cols) on the CSC view:
    grad_mat [N, K]."""
    colptr, row_csc, value_csc, mat = _smx_operands(colptr, row_csc, value_csc, mat)
    stride = _smx_t(t, mat)
    N, K = mat.shape
    M = out.size(0)
    E = row_csc.numel()
    dev = mat.device
    grad_mat = torch.empty_like(mat)
    with _on_device(dev):
        nws = lib.tsb200_spmm_softmax_aggr_bw_workspace_bytes(K, E)
        ws = _workspace(nws, dev)
        check(lib.tsb200_spmm_softmax_aggr_bw_cols(_p(colptr), _p(row_csc), _p(value_csc), _p(mat),
                                                   _p(t.contiguous()), stride, _p(grad_out.contiguous()), _p(out),
                                                   _p(lse), _p(grad_mat), M, N, K, E, _dtype_code(mat.dtype), _p(ws),
                                                   nws, _stream(dev)),
              "tsb200_spmm_softmax_aggr_bw_cols")
    return grad_mat


_FP8_OUT = {torch.float32: 0, torch.float16: 2, torch.bfloat16: 3}


def _fp8_args(what: str, rowptr: Tensor, col: Tensor, value: Optional[Tensor], x8: Tensor, scale: Tensor,
              out_dtype: Optional[torch.dtype]):
    """The checks shared by spmm_fw_fp8 (out_dtype given) and spmm_fw_fp8_quant (None: float32 values);
    returns (rowptr, col, value, scale, scale_stride)."""
    _check_cuda(rowptr, "rowptr")
    _check_cuda(col, "col")
    if value is not None:
        _check_cuda(value, "optional_value.value()")
    _check_cuda(x8, "x8")
    _check_cuda(scale, "scale")
    if torch.is_grad_enabled() and (scale.requires_grad or (value is not None and value.requires_grad)):
        raise RuntimeError(f"{what} is forward only: value and scale must not require grad "
                           "(call it under torch.no_grad() or detach them)")
    if x8.dtype != torch.float8_e4m3fn:
        raise RuntimeError(f"{what}: x8 must be torch.float8_e4m3fn, got {x8.dtype}")
    if x8.dim() != 2:
        raise RuntimeError(f"{what}: x8 must be 2-D [N, K], got {x8.dim()}-D")
    N, K = x8.shape
    if K % 16 != 0:
        raise RuntimeError(f"{what}: the number of columns K = {K} must be a multiple of 16")
    if not x8.is_contiguous() or x8.data_ptr() % 16 != 0:
        raise RuntimeError(f"{what}: x8 must be contiguous and 16-byte aligned")
    if out_dtype is not None and out_dtype not in _FP8_OUT:
        raise RuntimeError(f"{what}: out_dtype must be torch.bfloat16, torch.float16 or torch.float32, got {out_dtype}")
    value_dtype = torch.float32 if out_dtype is None else out_dtype
    if scale.dtype != torch.float32:
        raise RuntimeError(f"{what}: scale must be float32, got {scale.dtype}")
    if scale.dim() == 0:
        stride = 0
    elif scale.dim() == 1 and scale.size(0) == N:
        stride = 1
    else:
        raise RuntimeError(f"{what}: scale must have shape [] or [N] = [{N}], got {list(scale.shape)}")
    scale = scale.contiguous()
    _check_input(rowptr.dim() == 1)
    _check_input(col.dim() == 1)
    if value is not None:
        _check_input(value.dim() == 1)
        _check_input(value.size(0) == col.size(0))
        if value.dtype != value_dtype:
            raise RuntimeError(f"expected value of dtype {value_dtype} but got {value.dtype}")
        value = value.contiguous()
    return _i64(rowptr, "rowptr"), _i64(col, "col"), value, scale, stride


def _fp8_residual(what: str, residual: Optional[Tensor], residual_scale: Optional[Tensor], x8: Tensor, M: int,
                  red: int):
    """The checks of the optional residual of spmm_fw_fp8 / spmm_fw_fp8_quant: None without one, otherwise
    (residual, residual_scale, residual_scale_stride)."""
    if residual is None and residual_scale is None:
        return None
    if residual is None or residual_scale is None:
        raise RuntimeError(f"{what}: residual and residual_scale go together: pass both or neither")
    _check_cuda(residual, "residual")
    _check_cuda(residual_scale, "residual_scale")
    if red >= 2:
        raise RuntimeError(f"{what}: a residual is only added to reduce='sum' / 'mean' results, not min / max")
    if torch.is_grad_enabled() and residual_scale.requires_grad:
        raise RuntimeError(f"{what} is forward only: residual_scale must not require grad "
                           "(call it under torch.no_grad() or detach it)")
    if residual.device != x8.device or residual_scale.device != x8.device:
        raise RuntimeError(f"{what}: residual and residual_scale must be on the device of x8 ({x8.device})")
    if residual.dtype != torch.float8_e4m3fn:
        raise RuntimeError(f"{what}: residual must be torch.float8_e4m3fn, got {residual.dtype}")
    K = x8.size(1)
    if residual.dim() != 2 or residual.size(0) != M or residual.size(1) != K:
        raise RuntimeError(f"{what}: residual must have the result's shape [M, K] = [{M}, {K}], "
                           f"got {list(residual.shape)}")
    if not residual.is_contiguous() or residual.data_ptr() % 16 != 0:
        raise RuntimeError(f"{what}: residual must be contiguous and 16-byte aligned")
    if residual_scale.dtype != torch.float32:
        raise RuntimeError(f"{what}: residual_scale must be float32, got {residual_scale.dtype}")
    if residual_scale.dim() == 0:
        stride = 0
    elif residual_scale.dim() == 1 and residual_scale.size(0) == M:
        stride = 1
    else:
        raise RuntimeError(f"{what}: residual_scale must have shape [] or [M] = [{M}], "
                           f"got {list(residual_scale.shape)}")
    return residual, residual_scale.contiguous(), stride


def _fp8_call(rowptr: Tensor, col: Tensor, value: Optional[Tensor], x8: Tensor, scale: Tensor, stride: int, res,
              out: Tensor, out_scale: Optional[Tensor], arg_out: Optional[Tensor], dt: int, red: int,
              plan: Optional[SpmmPlan]) -> None:
    """tsb200_spmm_fw_fp8_res: out_dtype code `dt` result, or an e4m3 result when out_scale is given (dt = float32).
    Without a residual (res None) it is tsb200_spmm_fw_fp8 / tsb200_spmm_fw_fp8_quant."""
    residual, residual_scale, rstride = res if res is not None else (None, None, 0)
    N, K = x8.shape
    M, E = rowptr.numel() - 1, col.numel()
    dev = x8.device
    with _on_device(dev):
        pl, ws, nws = _plan_workspace(plan, E > 0, rowptr, 1, M, K, E, dt, red, dev)
        check(lib.tsb200_spmm_fw_fp8_res(_p(rowptr), _p(col), _p(value), _p(x8), _p(scale), stride, _p(residual),
                                         _p(residual_scale), rstride, _p(out), _p(out_scale), _p(arg_out), M, N, K, E,
                                         dt, red, *pl, _p(ws), nws, _stream(dev)), "tsb200_spmm_fw_fp8_res")


def spmm_fw_fp8(rowptr: Tensor, col: Tensor, value: Optional[Tensor], x8: Tensor, scale: Tensor,
                reduce: str = "sum", out_dtype: torch.dtype = torch.bfloat16,
                plan: Optional[SpmmPlan] = None, residual: Optional[Tensor] = None,
                residual_scale: Optional[Tensor] = None) -> Tuple[Tensor, Optional[Tensor]]:
    """`spmm_fw_fp8(rowptr, col, optional_value, x8, scale, reduce, out_dtype) -> (out, arg_out?)`
    (tsb200_spmm_fw_fp8): the SpMM forward over an e4m3 dense operand `x8` [N, K] (K % 16 == 0) whose row c stands for
    `x8[c].float() * scale[c]` (`scale` float32 of shape [N]) or `x8[c].float() * scale` (shape []). `value` has
    `out_dtype` (bf16, f16 or f32), as `spmm_fw`'s value has the dense dtype. Entry e weighs fl32(value[e] * scale[c]);
    sums accumulate weight * x8 in fp32 and round once, min/max compare the product rounded to `out_dtype`. Forward
    only. Planned like `spmm_fw` (the same per-rowptr plan cache).
    `residual` (e4m3 [M, K]) with `residual_scale` (float32 [] or [M]), sum / mean only (tsb200_spmm_fw_fp8_res): the
    result is round_out(fl32(y + fl32(residual_scale[m] * residual[m]))) with y the float32 result."""
    rowptr, col, value, scale, stride = _fp8_args("spmm_fp8", rowptr, col, value, x8, scale, out_dtype)
    red = _reduce_code(reduce)
    K = x8.size(1)
    M, E = rowptr.numel() - 1, col.numel()
    res = _fp8_residual("spmm_fp8", residual, residual_scale, x8, M, red)
    dev = x8.device
    out = torch.empty(M, K, dtype=out_dtype, device=dev)
    arg_out = torch.empty(M, K, dtype=torch.int64, device=dev) if red >= 2 else None
    if out.numel() == 0:
        return out, arg_out
    if res is None and E == 0:
        out.zero_()
        if arg_out is not None:
            arg_out.fill_(0)
        return out, arg_out
    _fp8_call(rowptr, col, value, x8, scale, stride, res, out, None, arg_out, _FP8_OUT[out_dtype], red, plan)
    return out, arg_out


FP8_QUANT_MAX_K = 2048


def spmm_fw_fp8_quant(rowptr: Tensor, col: Tensor, value: Optional[Tensor], x8: Tensor, scale: Tensor,
                      reduce: str = "sum", plan: Optional[SpmmPlan] = None, residual: Optional[Tensor] = None,
                      residual_scale: Optional[Tensor] = None) -> Tuple[Tensor, Tensor, Optional[Tensor]]:
    """`spmm_fw_fp8_quant(rowptr, col, optional_value, x8, scale, reduce) -> (y8, y_scale, arg_out?)`
    (tsb200_spmm_fw_fp8_quant): `spmm_fw_fp8` with a float32 result y, written as e4m3 with one scale per row by the
    kernel itself: y_scale[m] = amax|y[m]| / 448 (1 when that is not > 0, NaN rows included) and y8 = e4m3(y / y_scale),
    bit for bit `quantize_fp8(y, per_row=True)` on the CPU. `value` is float32. (y8, y_scale) are the `x8` and `scale`
    of the next hop. K <= 2048. Forward only; planned like `spmm_fw` (the same per-rowptr plan cache).
    `residual` (e4m3 [M, K]) with `residual_scale` (float32 [] or [M]), sum / mean only (tsb200_spmm_fw_fp8_res):
    the rows quantised are z = fl32(y + fl32(residual_scale[m] * residual[m])) instead of y."""
    rowptr, col, value, scale, stride = _fp8_args("spmm_fp8_quant", rowptr, col, value, x8, scale, None)
    K = x8.size(1)
    if K > FP8_QUANT_MAX_K:
        raise RuntimeError(f"spmm_fp8_quant: the number of columns K = {K} must be at most {FP8_QUANT_MAX_K}")
    red = _reduce_code(reduce)
    M, E = rowptr.numel() - 1, col.numel()
    res = _fp8_residual("spmm_fp8_quant", residual, residual_scale, x8, M, red)
    dev = x8.device
    y8 = torch.empty(M, K, dtype=torch.float8_e4m3fn, device=dev)
    y_scale = torch.empty(M, dtype=torch.float32, device=dev)
    arg_out = torch.empty(M, K, dtype=torch.int64, device=dev) if red >= 2 else None
    if M == 0:
        return y8, y_scale, arg_out
    if K == 0 or (res is None and E == 0):
        y8.zero_()
        y_scale.fill_(1.0)
        if arg_out is not None:
            arg_out.fill_(0)
        return y8, y_scale, arg_out
    _fp8_call(rowptr, col, value, x8, scale, stride, res, y8, y_scale, arg_out, _FP8_OUT[torch.float32], red, plan)
    return y8, y_scale, arg_out


_QUANT_IN = {torch.float32: 0, torch.float16: 2, torch.bfloat16: 3}
# torch's own messages for the amax of no elements, which the CPU quantize_fp8 raises
_AMAX_EMPTY_DIM = "amax(): Expected reduction dim 1 to have non-zero size."
_AMAX_EMPTY = ("amax(): Expected reduction dim to be specified for input.numel() == 0. "
               "Specify the reduction dim with the 'dim' argument.")


def quantize_fp8(x: Tensor, per_row: bool = True) -> Tuple[Tensor, Tensor]:
    """`quantize_fp8(x, per_row) -> (x8, scale)` (tsb200_quantize_fp8): a bf16 / f16 / f32 CUDA matrix [N, K] as e4m3
    with a float32 scale per row ([N]) or for the whole tensor ([]), bit for bit `matmul.quantize_fp8(x.cpu())`:
    scale = amax|x| / 448 (IEEE division), 1 when that amax is not > 0 (NaN included), x8 = e4m3(x / scale). One
    streaming kernel (two for a per-tensor scale) and no float temporaries; rows may be strided (`x[:, a:b]` of a
    wider matrix is read in place), a last dimension that is not contiguous is copied first. x8 is contiguous and
    16-byte aligned, a valid `spmm_fp8` operand. No host synchronisation, so the call can be captured in a CUDA graph.
    Forward only: the outputs carry no autograd history."""
    _check_cuda(x, "x")
    if x.dim() != 2:
        raise ValueError("quantize_fp8 expects a 2-D tensor [N, K]")
    if x.dtype not in _QUANT_IN:
        raise RuntimeError(f"quantize_fp8: x must be torch.bfloat16, torch.float16 or torch.float32, got {x.dtype}")
    N, K = x.shape
    if K == 0:
        raise IndexError(_AMAX_EMPTY_DIM) if per_row else RuntimeError(_AMAX_EMPTY)
    if N == 0 and not per_row:
        raise RuntimeError(_AMAX_EMPTY)
    if (K > 1 and x.stride(1) != 1) or (N > 1 and x.stride(0) < K):
        x = x.contiguous()
    ld = x.stride(0) if N > 1 else K
    dev = x.device
    x8 = torch.empty(N, K, dtype=torch.float8_e4m3fn, device=dev)
    scale = torch.empty((N,) if per_row else (), dtype=torch.float32, device=dev)
    if N == 0:
        return x8, scale
    ws = None if per_row else torch.empty(4, dtype=torch.uint8, device=dev)   # the per-tensor amax word
    with _on_device(dev):
        check(lib.tsb200_quantize_fp8(_p(x), N, K, ld, _QUANT_IN[x.dtype], int(per_row), _p(x8), _p(scale), _p(ws),
                                      0 if ws is None else ws.numel(), _stream(dev)), "tsb200_quantize_fp8")
    return x8, scale


def spmm_fw_acc(rowptr: Tensor, col: Tensor, value: Optional[Tensor], mat: Tensor, partial: Tensor,
                out: Optional[Tensor], acc_mode: int) -> None:
    """One column block of a SUM SpMM whose blocks are launched separately (tsb200_spmm_fw_acc): `partial` is the
    fp32 [.., M, K] accumulator shared by the blocks; acc_mode 1 = first block, 2 = middle, 3 = last (writes `out`)."""
    for t, n in ((rowptr, "rowptr"), (col, "col"), (mat, "mat"), (partial, "partial")):
        _check_cuda(t, n)
    _check_input(acc_mode in (1, 2, 3) and partial.dtype == torch.float32 and partial.is_contiguous())
    _check_input(mat.is_contiguous() and (value is None or (value.dtype == mat.dtype and value.is_contiguous())))
    rowptr, col = _i64(rowptr, "rowptr"), _i64(col, "col")
    M = rowptr.numel() - 1
    N, K = mat.size(-2), mat.size(-1)
    B = mat.numel() // (N * K) if N * K > 0 else 0
    E = col.numel()
    _check_input(partial.numel() == B * M * K)
    if acc_mode == 3:
        _check_input(out is not None and out.dtype == mat.dtype and out.is_contiguous() and out.numel() == B * M * K)
    if B * M * K == 0:
        return
    if E == 0:  # an empty column block contributes nothing
        if acc_mode == 1:
            partial.zero_()
        elif acc_mode == 3:
            out.copy_(partial.view(out.shape))
        return
    dev = mat.device
    dt = _dtype_code(mat.dtype)
    with _on_device(dev):
        nws = lib.tsb200_spmm_fw_workspace_bytes(B, M, K, E, dt, 0)
        ws = _workspace(nws, dev)
        check(lib.tsb200_spmm_fw_acc(_p(rowptr), _p(col), _p(value), _p(mat), _p(out), _p(partial), acc_mode,
                                     B, M, N, K, E, dt, _p(ws), nws, _stream(dev)), "tsb200_spmm_fw_acc")


def spmm_value_bw(row: Tensor, rowptr: Tensor, col: Tensor, mat: Tensor, grad: Tensor,
                  reduce: str) -> Tensor:
    """`spmm_value_bw(row, rowptr, col, mat, grad, reduce)` (csrc/spmm.cpp:37-49)."""
    for t, n in ((row, "row"), (rowptr, "rowptr"), (col, "col"), (mat, "mat"), (grad, "grad")):
        _check_cuda(t, n)
    red = _reduce_code(reduce)
    mat = mat.contiguous()
    grad = grad.contiguous()
    if grad.dtype != mat.dtype:
        grad = grad.to(mat.dtype)
    row, rowptr, col = _i64(row, "row"), _i64(rowptr, "rowptr"), _i64(col, "col")
    M, N, K = grad.size(-2), mat.size(-2), mat.size(-1)
    E = row.numel()
    B = mat.numel() // (N * K) if N * K > 0 else 0
    dev = mat.device
    out = torch.zeros(E, dtype=grad.dtype, device=dev)
    if E == 0 or B * K == 0:
        return out
    with _on_device(dev):
        dt = _dtype_code(mat.dtype)
        nws = lib.tsb200_spmm_value_bw_workspace_bytes(B, M, K, E, dt)
        ws = _workspace(nws, dev)
        check(lib.tsb200_spmm_value_bw(_p(row), _p(rowptr), _p(col), _p(mat), _p(grad), _p(out),
                                       B, M, N, K, E, dt, red, _p(ws), nws, _stream(dev)),
              "tsb200_spmm_value_bw")
    return out


def spmm_minmax_bw(col: Tensor, value: Optional[Tensor], mat: Tensor, grad_out: Tensor, arg_out: Tensor,
                   need_value: bool, need_mat: bool) -> Tuple[Optional[Tensor], Optional[Tensor]]:
    """Fused backward of spmm_min / spmm_max (replaces csrc/spmm.cpp:204-242, 264-302)."""
    for t, n in ((col, "col"), (mat, "mat"), (grad_out, "grad_out"), (arg_out, "arg_out")):
        _check_cuda(t, n)
    if not mat.dtype.is_floating_point:
        raise RuntimeError("spmm_min/max backward needs a floating point dtype")
    mat = mat.contiguous()
    grad_out = grad_out.contiguous().to(mat.dtype)
    arg_out = arg_out.contiguous()
    col = _i64(col, "col")
    if value is not None:
        value = value.contiguous()
    N, K = mat.size(-2), mat.size(-1)
    M = grad_out.size(-2)
    E = col.numel()
    B = mat.numel() // (N * K) if N * K > 0 else 0
    dev = mat.device
    acc = torch.float64 if mat.dtype == torch.float64 else torch.float32
    gv = torch.zeros(E, dtype=acc, device=dev) if need_value else None
    gm = torch.zeros(mat.shape, dtype=acc, device=dev) if need_mat else None
    if E > 0 and B * M * K > 0 and (need_value or need_mat):
        with _on_device(dev):
            check(lib.tsb200_spmm_minmax_bw(_p(col), _p(value), _p(mat), _p(grad_out), _p(arg_out), _p(gv),
                                            _p(gm), B, M, N, K, E, _dtype_code(mat.dtype), _stream(dev)),
                  "tsb200_spmm_minmax_bw")
    if gv is not None and gv.dtype != mat.dtype:
        gv = gv.to(mat.dtype)
    if gm is not None and gm.dtype != mat.dtype:
        gm = gm.to(mat.dtype)
    return gv, gm


# --------------------------------------------------------------------------------------------------
# format kernels
# --------------------------------------------------------------------------------------------------
def ind2ptr(ind: Tensor, M: int) -> Tensor:
    """`torch.ops.torch_sparse.ind2ptr(ind, M)` (csrc/convert.cpp:22-33)."""
    _check_cuda(ind, "ind")
    ind = _i64(ind, "ind")
    out = torch.empty(M + 1, dtype=torch.int64, device=ind.device)
    with _on_device(ind.device):
        check(lib.tsb200_ind2ptr(_p(ind), ind.numel(), M, _p(out), _stream(ind.device)), "tsb200_ind2ptr")
    return out


def ptr2ind(ptr: Tensor, E: int) -> Tensor:
    """`torch.ops.torch_sparse.ptr2ind(ptr, E)` (csrc/convert.cpp:35-45)."""
    _check_cuda(ptr, "ptr")
    ptr = _i64(ptr, "ptr")
    out = torch.empty(E, dtype=torch.int64, device=ptr.device)
    with _on_device(ptr.device):
        check(lib.tsb200_ptr2ind(_p(ptr), ptr.numel() - 1, E, _p(out), _stream(ptr.device)), "tsb200_ptr2ind")
    return out


def csr2csc(row: Tensor, col: Tensor, M: int, N: int, want_colptr: bool = True,
            want_row_csc: bool = False) -> Tuple[Tensor, Optional[Tensor], Optional[Tensor]]:
    """csr2csc permutation (+ colptr, + row[csr2csc]) of a row-major sorted COO
    (torch_sparse/storage.py:369-385, 407-416)."""
    _check_cuda(row, "row")
    _check_cuda(col, "col")
    row, col = _i64(row, "row"), _i64(col, "col")
    E, dev = col.numel(), col.device
    perm = torch.empty(E, dtype=torch.int64, device=dev)
    colptr = torch.empty(N + 1, dtype=torch.int64, device=dev) if want_colptr else None
    row_csc = torch.empty(E, dtype=torch.int64, device=dev) if want_row_csc else None
    with _on_device(dev):
        nws = lib.tsb200_csr2csc_workspace_bytes(E, M, N)
        ws = _workspace(nws, dev)
        check(lib.tsb200_csr2csc(_p(row), _p(col), E, M, N, _p(perm), _p(colptr), _p(row_csc), _p(ws), nws,
                                 _stream(dev)), "tsb200_csr2csc")
    return perm, colptr, row_csc


def _segment_reduce_raw(ptr: Tensor, value: Tensor, reduce: str, perm: Optional[Tensor],
                        want_arg: bool) -> Tuple[Tensor, Optional[Tensor]]:
    _check_cuda(ptr, "ptr")
    _check_cuda(value, "value")
    ptr = _i64(ptr, "ptr")
    value = value.contiguous()
    red = _reduce_code(reduce)
    S = ptr.numel() - 1
    E = value.size(0)
    D = value.numel() // E if E > 0 else int(torch.Size(value.shape[1:]).numel())
    out = torch.zeros((S,) + tuple(value.shape[1:]), dtype=value.dtype, device=value.device)
    arg = None
    if want_arg and red >= 2:
        arg = torch.full(out.shape, -1, dtype=torch.int64, device=value.device)
    if S == 0 or D == 0 or E == 0:
        return out, arg
    if perm is not None:
        perm = _i64(perm, "perm")
    with _on_device(value.device):
        check(lib.tsb200_segment_reduce(_p(ptr), _p(perm), _p(value), _p(out), _p(arg), S, D,
                                        _dtype_code(value.dtype), red, _stream(value.device)),
              "tsb200_segment_reduce")
    return out, arg


def segment_reduce_bw(seg: Tensor, count: Optional[Tensor], arg: Optional[Tensor], grad_out: Tensor, E: int,
                      reduce: str) -> Tensor:
    """Gradient of a segment / duplicate-run reduction w.r.t. its E input entries (tsb200_segment_reduce_bw):
    the autograd of torch_scatter.segment_csr / scatter that torch_sparse/storage.py:451 and
    torch_sparse/reduce.py:36-54 rely on, as one gather kernel."""
    _check_cuda(grad_out, "grad_out")
    grad_out = grad_out.contiguous()
    S = grad_out.size(0)
    D = grad_out.numel() // S if S > 0 else int(torch.Size(grad_out.shape[1:]).numel())
    grad_in = torch.empty((E,) + tuple(grad_out.shape[1:]), dtype=grad_out.dtype, device=grad_out.device)
    if E == 0 or D == 0:
        return grad_in
    if not grad_out.dtype.is_floating_point:
        raise RuntimeError("segment_reduce backward needs a floating point dtype")
    with _on_device(grad_out.device):
        check(lib.tsb200_segment_reduce_bw(_p(seg), _p(count), _p(arg), _p(grad_out), _p(grad_in), E, S, D,
                                           _dtype_code(grad_out.dtype), _reduce_code(reduce),
                                           _stream(grad_out.device)), "tsb200_segment_reduce_bw")
    return grad_in


class _SegmentReduce(torch.autograd.Function):
    @staticmethod
    def forward(ctx, value, ptr, reduce, perm, seg):
        out, arg = _segment_reduce_raw(ptr, value, reduce, perm, want_arg=True)
        ctx.reduce = reduce
        ctx.E = value.size(0)
        if seg is None:  # segment id of every input entry
            seg = ptr2ind(ptr, ctx.E)
            if perm is not None:
                seg = torch.empty_like(seg).scatter_(0, perm, seg)
        count = (ptr[1:] - ptr[:-1]) if _reduce_code(reduce) == 1 else None
        ctx.save_for_backward(seg, count, arg)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        seg, count, arg = ctx.saved_tensors
        return segment_reduce_bw(seg, count, arg, grad_out, ctx.E, ctx.reduce), None, None, None, None


def segment_reduce(ptr: Tensor, value: Tensor, reduce: str = "sum", perm: Optional[Tensor] = None,
                   seg: Optional[Tensor] = None) -> Tensor:
    """out[s] = reduce(value[perm?][ptr[s]:ptr[s+1]]) along dim 0, empty segments -> 0
    (torch_scatter.segment_csr as used by torch_sparse/reduce.py:36-54). Differentiable in `value`
    like the reference's; `seg` (segment id of every entry of `value`, e.g. the COO row / col vector)
    is an optional hint that saves rebuilding it for the backward."""
    if value.requires_grad and torch.is_grad_enabled():
        return _SegmentReduce.apply(value, ptr, reduce, perm, seg)
    return _segment_reduce_raw(ptr, value, reduce, perm, want_arg=False)[0]


def _segment_softmax_check(ptr: Tensor, value: Tensor, perm: Optional[Tensor]) -> None:
    _check_cuda(ptr, "ptr")
    _check_cuda(value, "value")
    if perm is not None:
        _check_cuda(perm, "perm")
    if not value.dtype.is_floating_point or value.dtype not in _DTYPES:
        raise RuntimeError(f'"softmax" not implemented for \'{value.dtype}\'')
    if value.dim() == 0:
        raise RuntimeError("softmax: value must be [E] or [E, *], got a 0-D tensor")
    if perm is not None and perm.numel() != value.size(0):
        raise RuntimeError(f"softmax: value must have {perm.numel()} rows (the nnz), got {value.size(0)}")


def _segment_softmax_raw(ptr: Tensor, value: Tensor, perm: Optional[Tensor]) -> Tensor:
    ptr, value = _i64(ptr, "ptr"), value.contiguous()
    if perm is not None:
        perm = _i64(perm, "perm")
    out = torch.empty_like(value)
    S, E = ptr.numel() - 1, value.size(0)
    if S <= 0 or out.numel() == 0:
        return out
    with _on_device(value.device):
        check(lib.tsb200_segment_softmax(_p(ptr), _p(perm), _p(value), _p(out), S, E, value.numel() // E,
                                         _dtype_code(value.dtype), _stream(value.device)), "tsb200_segment_softmax")
    return out


def segment_softmax_bw(ptr: Tensor, out: Tensor, grad_out: Tensor, perm: Optional[Tensor]) -> Tensor:
    """grad_in = out * (grad_out - sum over the segment of out * grad_out), per column (tsb200_segment_softmax_bw)."""
    ptr, out, grad_out = _i64(ptr, "ptr"), out.contiguous(), grad_out.contiguous()
    if perm is not None:
        perm = _i64(perm, "perm")
    grad_in = torch.empty_like(out)
    S, E = ptr.numel() - 1, out.size(0)
    if S <= 0 or out.numel() == 0:
        return grad_in
    with _on_device(out.device):
        check(lib.tsb200_segment_softmax_bw(_p(ptr), _p(perm), _p(out), _p(grad_out), _p(grad_in), S, E,
                                            out.numel() // E, _dtype_code(out.dtype), _stream(out.device)),
              "tsb200_segment_softmax_bw")
    return grad_in


class _SegmentSoftmax(torch.autograd.Function):
    @staticmethod
    def forward(ctx, value, ptr, perm):
        ptr = _i64(ptr, "ptr")
        perm = None if perm is None else _i64(perm, "perm")
        out = _segment_softmax_raw(ptr, value, perm)
        ctx.save_for_backward(out, ptr, perm)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        out, ptr, perm = ctx.saved_tensors
        return segment_softmax_bw(ptr, out, grad_out, perm), None, None


def segment_softmax(ptr: Tensor, value: Tensor, perm: Optional[Tensor] = None) -> Tensor:
    """Softmax of `value` [E] or [E, *] over each segment [ptr[s], ptr[s+1]), one per trailing column; with `perm`
    (csr2csc, ptr = colptr) segment entry j is value[perm[j]], and the result is written back in `value`'s order.
    bf16 / f16 / f32 / f64, fp32 arithmetic (fp64 for fp64); see tsb200_segment_softmax. Differentiable in `value`
    once: the backward is one kernel over the saved result."""
    _segment_softmax_check(ptr, value, perm)
    if value.requires_grad and torch.is_grad_enabled():
        return _SegmentSoftmax.apply(value, ptr, perm)
    return _segment_softmax_raw(ptr, value, perm)


class _PinnedScalar:
    """One pinned int64 per device-side count read back from the GPU (E', nnz(C)). The buffers are pooled:
    `read()` returns the value (after the caller synchronised the stream) and hands the buffer back."""
    _pool: list = []

    def __init__(self):
        self.t = self._pool.pop() if self._pool else torch.zeros(1, dtype=torch.int64, device="cpu").pin_memory()

    def ptr(self):
        return ctypes.c_void_p(self.t.data_ptr())

    def read(self) -> int:
        v = int(self.t.item())
        if len(self._pool) < 16:
            self._pool.append(self.t)
        return v


def sort_perm(row: Tensor, col: Tensor, M: int, N: int) -> Optional[Tensor]:
    """Stable permutation that sorts (row, col) row-major — the sort-on-construct of
    SparseStorage (torch_sparse/storage.py:149-162). Returns None when the input is already
    sorted (the reference skips the sort in that case too, storage.py:154)."""
    _check_cuda(row, "row")
    _check_cuda(col, "col")
    row, col = _i64(row, "row"), _i64(col, "col")
    E, dev = col.numel(), col.device
    if E < 2:
        return None
    with _on_device(dev):
        nws = lib.tsb200_coalesce_workspace_bytes(E, M, N)
        ws = _workspace(nws, dev)
        st = _stream(dev)
        check(lib.tsb200_coalesce_sort(_p(row), _p(col), E, M, N, _p(ws), nws, None, st), "tsb200_coalesce_sort")
        if int(ws[:4].view(torch.int32).item()) == 0:  # device flag "input was unsorted"
            return None
        perm = torch.empty(E, dtype=torch.int64, device=dev)
        check(lib.tsb200_coalesce_perm(E, _p(perm), _p(ws), st), "tsb200_coalesce_perm")
    return perm


def _coalesce_raw(row: Tensor, col: Tensor, value: Optional[Tensor], M: int, N: int, reduce: str,
                  want_bw: bool):
    """-> (row', col', value', (seg, count, arg) or None). `want_bw` also emits what the backward of the value
    reduction reads: the run id of every input entry, the run lengths (mean) and the arg entry (min/max)."""
    _check_cuda(row, "row")
    _check_cuda(col, "col")
    row, col = _i64(row, "row"), _i64(col, "col")
    red = _reduce_code(reduce)
    E, dev = col.numel(), col.device
    if value is not None:
        _check_cuda(value, "value")
        _check_input(value.size(0) == E)
        value = value.contiguous()
    if E == 0:
        return row, col, value, None
    with _on_device(dev):
        nws = lib.tsb200_coalesce_workspace_bytes(E, M, N)
        ws = _workspace(nws, dev)
        st = _stream(dev)
        pin = _PinnedScalar()
        check(lib.tsb200_coalesce_sort(_p(row), _p(col), E, M, N, _p(ws), nws, pin.ptr(), st),
              "tsb200_coalesce_sort")
        torch.cuda.current_stream(dev).synchronize()
        n_unique = pin.read()
        row_out = torch.empty(n_unique, dtype=torch.int64, device=dev)
        col_out = torch.empty(n_unique, dtype=torch.int64, device=dev)
        value_out = None
        D, dt = 1, 0
        if value is not None:
            D = value.numel() // E
            dt = _dtype_code(value.dtype)
            value_out = torch.empty((n_unique,) + tuple(value.shape[1:]), dtype=value.dtype, device=dev)
        seg = count = arg = None
        if want_bw and value is not None:
            seg = torch.empty(E, dtype=torch.int64, device=dev)
            if red == 1:
                count = torch.empty(n_unique, dtype=torch.int64, device=dev)
            if red >= 2:
                arg = torch.empty(value_out.shape, dtype=torch.int64, device=dev)
        check(lib.tsb200_coalesce_emit(E, N, n_unique, _p(value), D, dt, red, _p(row_out), _p(col_out),
                                       _p(value_out), None, _p(seg), _p(count), _p(arg), _p(ws), st),
              "tsb200_coalesce_emit")
    return row_out, col_out, value_out, ((seg, count, arg) if seg is not None else None)


class _Coalesce(torch.autograd.Function):
    @staticmethod
    def forward(ctx, value, row, col, M, N, reduce):
        row_out, col_out, value_out, bw = _coalesce_raw(row, col, value, M, N, reduce, want_bw=True)
        ctx.reduce = reduce
        ctx.E = value.size(0)
        ctx.identity = bw is None          # E == 0: value passes through
        if bw is not None:
            ctx.save_for_backward(*bw)
        ctx.mark_non_differentiable(row_out, col_out)
        return row_out, col_out, value_out

    @staticmethod
    def backward(ctx, _g_row, _g_col, grad_value):
        if ctx.identity:
            return grad_value, None, None, None, None, None
        seg, count, arg = ctx.saved_tensors
        return segment_reduce_bw(seg, count, arg, grad_value, ctx.E, ctx.reduce), None, None, None, None, None


def coalesce(row: Tensor, col: Tensor, value: Optional[Tensor], M: int, N: int,
             reduce: str = "add") -> Tuple[Tensor, Tensor, Optional[Tensor]]:
    """Sort by (row, col), merge duplicate entries, reduce their values
    (torch_sparse/coalesce.py:5-25 -> torch_sparse/storage.py:149-162, 436-466). Differentiable in `value`
    (the reference's value reduction is torch_scatter.segment_csr, storage.py:451)."""
    if value is not None and value.requires_grad and torch.is_grad_enabled():
        return _Coalesce.apply(value, row, col, M, N, reduce)
    return _coalesce_raw(row, col, value, M, N, reduce, want_bw=False)[:3]


def spspmm(rowptr_a: Tensor, col_a: Tensor, val_a: Optional[Tensor], rowptr_b: Tensor, col_b: Tensor,
           val_b: Optional[Tensor], M: int, Kd: int, N: int,
           want_value: bool) -> Tuple[Tensor, Tensor, Tensor, Optional[Tensor]]:
    """C = A @ B for CSR operands -> (rowptr_c, row_c, col_c, val_c?) sorted, unique, structural
    (replaces torch.sparse.mm at torch_sparse/matmul.py:94-111)."""
    for t, n in ((rowptr_a, "rowptrA"), (col_a, "colA"), (rowptr_b, "rowptrB"), (col_b, "colB")):
        _check_cuda(t, n)
    rowptr_a, col_a = _i64(rowptr_a, "rowptrA"), _i64(col_a, "colA")
    rowptr_b, col_b = _i64(rowptr_b, "rowptrB"), _i64(col_b, "colB")
    dev = col_a.device
    dtype = None
    if want_value:
        dtype = val_a.dtype if val_a is not None else (val_b.dtype if val_b is not None else torch.float32)
        if val_a is not None and val_b is not None and val_a.dtype != val_b.dtype:
            raise RuntimeError("spspmm: value dtypes of both operands must match")
        if dtype not in (torch.float32, torch.float64):
            # torch.sparse.mm: '"sparse_matmul" not implemented' for Half/BFloat16/integers
            raise RuntimeError(f'"sparse_matmul" not implemented for \'{dtype}\'')
        val_a = None if val_a is None else val_a.contiguous()
        val_b = None if val_b is None else val_b.contiguous()
    else:
        val_a = val_b = None
    nnz_a, nnz_b = col_a.numel(), col_b.numel()
    rowptr_c = torch.empty(M + 1, dtype=torch.int64, device=dev)
    esize = 0 if not want_value else (8 if dtype == torch.float64 else 4)
    # two_phase (symbolic + numeric kernels) is the default. "fused" selects the single-pass kernel (rows placed by
    # a decoupled look-back, outputs sized by the product bound): bit-identical structure, one kernel instead of two,
    # kept as an option. "auto" takes the single pass when the product bound fits comfortably into the memory still
    # available, otherwise it counts first (two phases).
    mode = os.environ.get("TSB200_SPSPMM", "two_phase")
    dt = _dtype_code(dtype) if want_value else 0

    def single_pass():
        """The product bound, then the single pass into arrays of that size; None when auto declines."""
        pin = _PinnedScalar()
        check(lib.tsb200_spspmm_bound(_p(col_a), _p(rowptr_b), nnz_a, _p(ws), nws, pin.ptr(), st),
              "tsb200_spspmm_bound")
        torch.cuda.current_stream(dev).synchronize()
        bound = pin.read()
        if mode == "auto" and bound * (16 + esize) > 0.45 * _available_bytes(dev):
            return None
        row_c = torch.empty(bound, dtype=torch.int64, device=dev)
        col_c = torch.empty(bound, dtype=torch.int64, device=dev)
        val_c = torch.empty(bound, dtype=dtype, device=dev) if want_value else None
        pin = _PinnedScalar()
        check(lib.tsb200_spspmm_fused(_p(rowptr_a), _p(col_a), _p(val_a), _p(rowptr_b), _p(col_b), _p(val_b), M, Kd,
                                      N, nnz_a, nnz_b, _p(rowptr_c), _p(row_c), _p(col_c), _p(val_c), bound, dt, _p(ws),
                                      nws, pin.ptr(), st), "tsb200_spspmm_fused")
        torch.cuda.current_stream(dev).synchronize()
        nnz_c = pin.read()
        if nnz_c < 0:  # cannot happen with capacity = number of products
            raise _lib.Tsb200Error("tsb200_spspmm_fused: output capacity exceeded")
        row_c, col_c = row_c[:nnz_c], col_c[:nnz_c]
        val_c = None if val_c is None else val_c[:nnz_c]
        if nnz_c < 0.75 * bound:  # many merged products: do not keep the oversized allocations alive
            row_c, col_c = row_c.clone(), col_c.clone()
            val_c = None if val_c is None else val_c.clone()
        return rowptr_c, row_c, col_c, val_c

    def two_phase():
        pin = _PinnedScalar()
        check(lib.tsb200_spspmm_symbolic(_p(rowptr_a), _p(col_a), _p(rowptr_b), _p(col_b), M, Kd, N, nnz_a,
                                         nnz_b, _p(rowptr_c), _p(ws), nws, pin.ptr(), st),
              "tsb200_spspmm_symbolic")
        torch.cuda.current_stream(dev).synchronize()
        nnz_c = pin.read()
        row_c = torch.empty(nnz_c, dtype=torch.int64, device=dev)
        col_c = torch.empty(nnz_c, dtype=torch.int64, device=dev)
        val_c = torch.empty(nnz_c, dtype=dtype, device=dev) if want_value else None
        if nnz_c > 0:
            check(lib.tsb200_spspmm_numeric(_p(rowptr_a), _p(col_a), _p(val_a), _p(rowptr_b), _p(col_b),
                                            _p(val_b), M, Kd, N, nnz_a, nnz_b, _p(rowptr_c), _p(row_c),
                                            _p(col_c), _p(val_c), dt, _p(ws), nws, st), "tsb200_spspmm_numeric")
        return rowptr_c, row_c, col_c, val_c

    with _on_device(dev):
        nws = lib.tsb200_spspmm_workspace_bytes(M, Kd, N, nnz_a, nnz_b)
        ws = _workspace(nws, dev)
        st = _stream(dev)
        out = single_pass() if mode in ("fused", "auto") else None
        return out if out is not None else two_phase()


def _available_bytes(dev: torch.device) -> int:
    """Device memory a new allocation can draw on: free on the device plus what PyTorch's allocator holds unused."""
    free, _total = torch.cuda.mem_get_info(dev)
    return int(free) + int(torch.cuda.memory_reserved(dev)) - int(torch.cuda.memory_allocated(dev))


_PINNED_POOL: dict = {}   # nbytes -> list of (pinned uint8 tensor, idle use-count); cudaHostAlloc of 256 MB costs ~30 ms


def _storage_uses(t: Tensor) -> int:
    return torch._C._storage_Use_Count(t.untyped_storage()._cdata)


def _pinned_empty(shape, dtype: torch.dtype, pin: bool = True) -> Tensor:
    """A pinned host tensor from a small pool. A pooled buffer is handed out again only when no tensor other
    than the pool's own handle references its storage any more (every view a caller derived from an earlier
    result holds a storage reference, so the C++ use-count tells)."""
    esize = torch.empty(0, dtype=dtype, device="cpu").element_size()
    numel = int(torch.Size(shape).numel())
    nbytes = max(1, numel * esize)
    bucket = _PINNED_POOL.setdefault((nbytes, pin), [])
    base = None
    for cand, idle in bucket:
        if _storage_uses(cand) <= idle:
            base = cand
            break
    if base is None:
        base = torch.empty(nbytes, dtype=torch.uint8, device="cpu", pin_memory=pin)
        if len(bucket) < 4:
            bucket.append((base, _storage_uses(base)))
    return base[:numel * esize].view(dtype).view(shape)


def spmm_fw_host(rowptr: Tensor, col: Tensor, value: Optional[Tensor], mat: Tensor, reduce: str = "sum",
                 out: Optional[Tensor] = None, arg_out: Optional[Tensor] = None) -> Tuple[Tensor, Optional[Tensor]]:
    """Host-buffer SpMM: CPU tensors in, CPU tensors out, H2D/D2H inside (tsb200_spmm_fw_host). Pass pinned
    tensors for full PCIe speed; `out` / `arg_out` may be supplied (pinned, right shape/dtype), otherwise
    they come from a pinned pool when `mat` is pinned."""
    for t, n in ((rowptr, "rowptr"), (col, "col"), (mat, "mat")):
        if t.is_cuda:
            raise RuntimeError(f"{n} must be CPU tensor")
    red = _reduce_code(reduce)
    rowptr, col, mat = _i64(rowptr, "rowptr"), _i64(col, "col"), mat.contiguous()
    if value is not None:
        value = value.to(mat.dtype).contiguous()
    M = rowptr.numel() - 1
    N, K = mat.size(-2), mat.size(-1)
    B = mat.numel() // (N * K) if N * K > 0 else 0
    sizes = list(mat.shape)
    sizes[-2] = M
    alloc = _pinned_empty if mat.is_pinned() else (lambda shape, dtype: torch.empty(shape, dtype=dtype, device="cpu"))
    if out is None:
        out = alloc(sizes, mat.dtype)
    else:
        _check_input(list(out.shape) == sizes and out.dtype == mat.dtype and out.is_contiguous() and not out.is_cuda)
    if red >= 2:
        if arg_out is None:
            arg_out = alloc(sizes, torch.int64)
        else:
            _check_input(list(arg_out.shape) == sizes and arg_out.dtype == torch.int64 and arg_out.is_contiguous())
    else:
        arg_out = None
    check(lib.tsb200_spmm_fw_host(_p(rowptr), _p(col), _p(value), _p(mat), _p(out), _p(arg_out), B, M, N, K,
                                  col.numel(), _dtype_code(mat.dtype), red), "tsb200_spmm_fw_host")
    return out, arg_out


# --------------------------------------------------------------------------------------------------
# autograd Functions mirroring SPMMSum / SPMMMean / SPMMMin / SPMMMax (csrc/spmm.cpp:55-303)
# --------------------------------------------------------------------------------------------------
def _assert_present(t: Optional[Tensor], name: str) -> None:
    if t is None:
        raise RuntimeError(f"Argument `{name}` is missing")


class SPMMSum(torch.autograd.Function):
    @staticmethod
    def forward(ctx, row, rowptr, col, value, colptr, csr2csc, mat, row_csc=None):
        # row_csc (= row[csr2csc]) is an optional extra over the reference's signature: structure-only, so a
        # caller that keeps it (SparseStorage.row_csc) saves one E-sized gather per backward (csrc/spmm.cpp:104)
        has_value = value is not None
        need_value = has_value and ctx.needs_input_grad[3]
        need_mat = ctx.needs_input_grad[6]
        if need_value:
            _assert_present(row, "row")
        if need_mat:
            _assert_present(row, "row")
            _assert_present(colptr, "colptr")
            _assert_present(csr2csc, "csr2csc")
        out, _ = spmm_fw(rowptr, col, value, mat, "sum")
        ctx.has_value = has_value
        ctx.save_for_backward(row, rowptr, col, value, colptr, csr2csc, mat, row_csc if need_mat else None)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        row, rowptr, col, value, colptr, csr2csc, mat, row_csc = ctx.saved_tensors
        grad_value, grad_mat = _sum_grads(ctx.has_value and ctx.needs_input_grad[3], ctx.needs_input_grad[6], row,
                                          rowptr, col, value, colptr, csr2csc, mat, row_csc, grad_out)
        return None, None, None, grad_value, None, None, grad_mat, None


def _sum_grads(need_value: bool, need_mat: bool, row, rowptr, col, value, colptr, csr2csc, mat, row_csc, grad_out):
    """(grad_value, grad_mat) of a sum SpMM: SPMMSum's backward, shared with SPMMRes."""
    grad_value = grad_mat = None
    if need_value:
        grad_value = spmm_value_bw(row, rowptr, col, mat, grad_out, "sum")
    if need_mat:
        # grad_mat = A^T @ grad_out as a CSR SpMM on the CSC view (csrc/spmm.cpp:100-108)
        v = value.index_select(0, csr2csc) if value is not None else None
        if row_csc is None:
            row_csc = row.index_select(0, csr2csc)
        grad_mat, _ = spmm_fw(colptr, row_csc, v, grad_out, "sum")
    return grad_value, grad_mat


class SPMMMean(torch.autograd.Function):
    @staticmethod
    def forward(ctx, row, rowptr, col, value, rowcount, colptr, csr2csc, mat, row_csc=None):
        has_value = value is not None
        if has_value and ctx.needs_input_grad[3]:
            _assert_present(row, "row")
        if ctx.needs_input_grad[7]:
            _assert_present(row, "row")
            _assert_present(rowcount, "rowcount")
            _assert_present(colptr, "colptr")
            _assert_present(csr2csc, "csr2csc")
        out, _ = spmm_fw(rowptr, col, value, mat, "mean")
        ctx.has_value = has_value
        ctx.save_for_backward(row, rowptr, col, value, rowcount, colptr, csr2csc, mat,
                              row_csc if ctx.needs_input_grad[7] else None)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        row, rowptr, col, value, rowcount, colptr, csr2csc, mat, row_csc = ctx.saved_tensors
        grad_value, grad_mat = _mean_grads(ctx.has_value and ctx.needs_input_grad[3], ctx.needs_input_grad[7], row,
                                           rowptr, col, value, rowcount, colptr, csr2csc, mat, row_csc, grad_out)
        return None, None, None, grad_value, None, None, None, grad_mat, None


def _mean_grads(need_value: bool, need_mat: bool, row, rowptr, col, value, rowcount, colptr, csr2csc, mat, row_csc,
                grad_out):
    """(grad_value, grad_mat) of a mean SpMM: SPMMMean's backward, shared with SPMMRes."""
    grad_value = grad_mat = None
    if need_value:
        grad_value = spmm_value_bw(row, rowptr, col, mat, grad_out, "mean")
    if need_mat:
        # per-nnz weight value/count(row) (or 1/count) in CSC order (csrc/spmm.cpp:166-177), divided in the
        # accumulator type and rounded once to mat's dtype: the forward and grad_value divide by the exact count,
        # which bf16 (above 256) and f16 (above 2048) cannot always hold (DESIGN §3.2)
        if row_csc is None:
            row_csc = row.index_select(0, csr2csc)
        acc = torch.float64 if mat.dtype == torch.float64 else torch.float32
        cnt = rowcount.index_select(0, row_csc).to(acc).clamp_(min=1)
        w = value.index_select(0, csr2csc).to(acc).div_(cnt) if value is not None else cnt.reciprocal_()
        grad_mat, _ = spmm_fw(colptr, row_csc, w.to(mat.dtype), grad_out, "sum")
    return grad_value, grad_mat


_ZERO_PTR = {}  # per device: a zero row pointer, the empty pattern of _scale_rows


def _scale_rows(g: Tensor, scale: Tensor) -> Tensor:
    """s[m] * g[m] in fp32 (fp64), rounded once to g's dtype, in one pass over g (a zero product gives +0): the
    residual-only SpMM over an empty pattern, tsb200_spmm_fw_res with E = 0 and residual g."""
    M, K = g.shape
    z = _ZERO_PTR.get(g.device)
    if z is None or z.numel() < M + 1:
        z = _ZERO_PTR[g.device] = torch.zeros(M + 1, dtype=torch.int64, device=g.device)
    return spmm_fw_res(z[:M + 1], z[:0], None, g.new_empty(0, K), g.contiguous(), scale)


class SPMMRes(torch.autograd.Function):
    """`spmm_fw_res`, sum or mean. grad_value and grad_mat are those of SPMMSum / SPMMMean; grad_residual is
    s * g formed in fp32 (fp64) and rounded once, in one pass (_scale_rows); grad_residual_scale is sum_k g * r per row
    ([M]) or over all ([])."""
    @staticmethod
    def forward(ctx, row, rowptr, col, value, rowcount, colptr, csr2csc, mat, row_csc, residual, residual_scale,
                reduce):
        mean = _reduce_code(reduce) == 1
        need_value = value is not None and ctx.needs_input_grad[3]
        need_mat = ctx.needs_input_grad[7]
        if need_value or need_mat:
            _assert_present(row, "row")
        if need_mat:
            if mean:
                _assert_present(rowcount, "rowcount")
            _assert_present(colptr, "colptr")
            _assert_present(csr2csc, "csr2csc")
        out = spmm_fw_res(rowptr, col, value, mat, residual, residual_scale, reduce)
        ctx.mean, ctx.need_value = mean, need_value
        ctx.save_for_backward(row, rowptr, col, value, rowcount, colptr, csr2csc, mat,
                              row_csc if need_mat else None, residual if ctx.needs_input_grad[10] else None,
                              residual_scale)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        row, rowptr, col, value, rowcount, colptr, csr2csc, mat, row_csc, residual, scale = ctx.saved_tensors
        need_mat = ctx.needs_input_grad[7]
        grad_value = grad_mat = grad_res = grad_scale = None
        if ctx.need_value or need_mat:
            if ctx.mean:
                grad_value, grad_mat = _mean_grads(ctx.need_value, need_mat, row, rowptr, col, value, rowcount, colptr,
                                                   csr2csc, mat, row_csc, grad_out)
            else:
                grad_value, grad_mat = _sum_grads(ctx.need_value, need_mat, row, rowptr, col, value, colptr, csr2csc,
                                                  mat, row_csc, grad_out)
        acc = torch.float64 if mat.dtype == torch.float64 else torch.float32
        if ctx.needs_input_grad[9]:
            grad_res = grad_out if scale is None else _scale_rows(grad_out, scale)
        if ctx.needs_input_grad[10]:
            gr = grad_out.to(acc) * residual.to(acc)
            grad_scale = gr.sum(1) if scale.dim() == 1 else gr.sum()
        return (None, None, None, grad_value, None, None, None, grad_mat, None, grad_res, grad_scale, None)


class SPMMMulti(torch.autograd.Function):
    """`spmm_fw_multi`, differentiable in the values and `mat` with no kernel of its own. With g_c the gradient of
    slice c, n = max(degree, 1), mu the mean and g_v = g_var [var > 0] + g_std / (2 std) [std > 0] (the clamps of var
    and std pass no gradient), per row a = g_sum + g_mean / n - 2 mu g_v / n and b = 2 g_v / n, so that the gradient of
    every message p_e = v_e x[col_e] is a + b p_e:
        grad_x = A^T a + x * (A_{v^2}^T b)          (two SpMMs on the CSC view; A_{v^2} has the values v^2)
        grad_v[e] = <a_row, x_col> + v_e <b_row, x_col^2>   (two SDDMMs)
    plus the min / max gradients of spmm_minmax_bw. Terms without a gradient are skipped. The mean is computed as an
    extra slice when var / std need a gradient and it is not requested."""
    @staticmethod
    def forward(ctx, row, rowptr, col, value, colptr, csr2csc, mat, row_csc, aggrs):
        codes = _aggr_codes(aggrs)
        need_value = value is not None and ctx.needs_input_grad[3]
        need_mat = ctx.needs_input_grad[6]
        if need_value or need_mat:
            _assert_present(row, "row")
        if need_mat:
            _assert_present(colptr, "colptr")
            _assert_present(csr2csc, "csr2csc")
        need = need_value or need_mat
        kcodes = list(codes)
        if need and (4 in codes or 5 in codes) and 1 not in codes:
            kcodes.append(1)
        full, arg_min, arg_max = _spmm_fw_multi(rowptr, col, value, mat, kcodes, need)
        out = full if len(kcodes) == len(codes) else full[:, :len(codes)].clone()
        ctx.codes, ctx.need_value = kcodes, need_value
        ctx.save_for_backward(row, rowptr, col, value, colptr, csr2csc, mat, row_csc if need_mat else None,
                              full if need else None, arg_min, arg_max)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        row, rowptr, col, value, colptr, csr2csc, mat, row_csc, full, arg_min, arg_max = ctx.saved_tensors
        need_value, need_mat = ctx.need_value, ctx.needs_input_grad[6]
        if not (need_value or need_mat):
            return None, None, None, None, None, None, None, None, None
        codes = ctx.codes
        acc = torch.float64 if mat.dtype == torch.float64 else torch.float32

        def grad_of(c: int) -> Optional[Tensor]:
            return grad_out[:, codes.index(c)] if c in codes and codes.index(c) < grad_out.size(1) else None

        # the row coefficients a and b are formed in fp32 (fp64) and rounded once to the dtype; the products and the
        # sum of the gradient's terms run in the dtype, as autograd sums the terms of the unfused composition
        dt = mat.dtype
        g_sum, g_mean, g_var, g_std = grad_of(0), grad_of(1), grad_of(4), grad_of(5)
        a = b = None
        if g_mean is None and g_var is None and g_std is None:
            a = g_sum
        else:
            inv_n = (rowptr[1:] - rowptr[:-1]).clamp(min=1).to(acc).reciprocal_().unsqueeze(1)
            if g_mean is not None:
                a = g_mean * inv_n
            if g_sum is not None:
                a = g_sum.to(acc, copy=True) if a is None else a.add_(g_sum)
            gv = None   # g_v / n
            if g_var is not None:
                gv = (g_var * inv_n).masked_fill_(~(full[:, codes.index(4)] > 0), 0)
            if g_std is not None:
                std = full[:, codes.index(5)]
                t = (g_std * inv_n).div_(std).mul_(0.5).masked_fill_(~(std > 0), 0)
                gv = t if gv is None else gv.add_(t)
            if gv is not None:
                b = gv.mul_(2)
                mb = b * full[:, codes.index(1)]
                a = mb.neg_() if a is None else a.sub_(mb)
                b = b.to(dt)
            a = a.to(dt) if a is not None else None

        grad_value = grad_mat = None
        if need_mat:
            if row_csc is None:
                row_csc = row.index_select(0, csr2csc)
            v_csc = value.index_select(0, csr2csc) if value is not None else None
            if a is not None:
                grad_mat = spmm_fw(colptr, row_csc, v_csc, a, "sum")[0]
            if b is not None:
                t = spmm_fw(colptr, row_csc, v_csc * v_csc if v_csc is not None else None, b, "sum")[0].mul_(mat)
                grad_mat = t if grad_mat is None else grad_mat.add_(t)
        if need_value:
            if a is not None:
                grad_value = spmm_value_bw(row, rowptr, col, mat, a, "sum")
            if b is not None:
                t = spmm_value_bw(row, rowptr, col, mat * mat, b, "sum").mul_(value)
                grad_value = t if grad_value is None else grad_value.add_(t)
        for c, arg in ((2, arg_min), (3, arg_max)):
            g = grad_of(c)
            if g is None:
                continue
            gvm, gmm = spmm_minmax_bw(col, value, mat, g, arg, need_value, need_mat)
            if gvm is not None:
                grad_value = gvm if grad_value is None else grad_value.add_(gvm)
            if gmm is not None:
                grad_mat = gmm if grad_mat is None else grad_mat.add_(gmm)
        if need_mat and grad_mat is None:
            grad_mat = torch.zeros_like(mat)
        if need_value and grad_value is None:
            grad_value = torch.zeros_like(value)
        return None, None, None, grad_value, None, None, grad_mat, None, None


def spmm_multi(row: Optional[Tensor], rowptr: Tensor, col: Tensor, value: Optional[Tensor], colptr: Optional[Tensor],
               csr2csc: Optional[Tensor], mat: Tensor, row_csc: Optional[Tensor], aggrs: List[str]) -> Tensor:
    return SPMMMulti.apply(row, rowptr, col, value, colptr, csr2csc, mat, row_csc, aggrs)


class SPMMSoftmaxAggr(torch.autograd.Function):
    """`spmm_fw_softmax_aggr`, differentiable in the values, `mat` and `t`. With g = grad_out, o = out and
    alpha_e = exp(t p_e - lse), the gradient of message e is d_e = g alpha_e (1 + t (p_e - o)), per column:
        grad_value[e] = <x[col_e], d_e>,  grad_t = sum_r g[r] sum_{e in r} alpha_e (p_e - o[r])^2   (row-wise kernel)
        grad_mat[n] = sum_{e in column n} v_e d_e                                             (column-wise kernel)
    out and lse are saved only when a gradient is wanted, only the kernels whose gradients are wanted run, and only
    grad_mat reads the CSC view (colptr, csr2csc, row_csc). grad_t is U.sum(0) (U.sum() for one temperature) of the
    kernel's per-row plane, with no atomics anywhere, so it is the same bit for bit from run to run."""
    @staticmethod
    def forward(ctx, rowptr, col, value, colptr, csr2csc, mat, row_csc, t):
        need_value = value is not None and ctx.needs_input_grad[2]
        need_mat = ctx.needs_input_grad[5]
        need_t = t is not None and ctx.needs_input_grad[7]
        if need_mat:
            _assert_present(colptr, "colptr")
            _assert_present(csr2csc, "csr2csc")
        if t is None:   # t = 1, not learnable
            key = (mat.device, torch.float64 if mat.dtype == torch.float64 else torch.float32)
            t = _ONE.get(key)
            if t is None:
                t = _ONE[key] = torch.ones((), dtype=key[1], device=mat.device)
        need = need_value or need_mat or need_t
        out, lse = spmm_fw_softmax_aggr(rowptr, col, value, mat, t, want_lse=need)
        ctx.need = (need_value, need_mat, need_t)
        ctx.save_for_backward(rowptr, col, value, colptr, csr2csc, mat, row_csc if need_mat else None, t,
                              out if need else None, lse)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        rowptr, col, value, colptr, csr2csc, mat, row_csc, t, out, lse = ctx.saved_tensors
        need_value, need_mat, need_t = ctx.need
        grad_value = grad_mat = grad_t = None
        grad_out = grad_out.contiguous()
        if need_value or need_t:
            grad_value, U = spmm_softmax_aggr_bw_rows(rowptr, col, value, mat, t, grad_out, out, lse, need_value,
                                                      need_t)
            if U is not None:
                grad_t = (U.sum(0) if t.dim() == 1 and t.numel() > 1 else U.sum()).reshape(t.shape)
        if need_mat:
            if row_csc is None:
                row_csc = ptr2ind(rowptr, col.numel()).index_select(0, csr2csc)
            v_csc = value.index_select(0, csr2csc) if value is not None else None
            grad_mat = spmm_softmax_aggr_bw_cols(colptr, row_csc, v_csc, mat, t, grad_out, out, lse)
        return None, None, grad_value, None, None, grad_mat, None, grad_t


def spmm_softmax_aggr(rowptr: Tensor, col: Tensor, value: Optional[Tensor], colptr: Optional[Tensor],
                      csr2csc: Optional[Tensor], mat: Tensor, row_csc: Optional[Tensor],
                      t: Optional[Tensor]) -> Tensor:
    return SPMMSoftmaxAggr.apply(rowptr, col, value, colptr, csr2csc, mat, row_csc, t)


def _minmax_forward(ctx, reduce, rowptr, col, value, mat):
    out, arg_out = spmm_fw(rowptr, col, value, mat, reduce)
    ctx.has_value = value is not None
    ctx.save_for_backward(col, value, mat, arg_out)
    ctx.mark_non_differentiable(arg_out)
    return out, arg_out


def _minmax_backward(ctx, grad_out):
    col, value, mat, arg_out = ctx.saved_tensors
    need_value = ctx.has_value and ctx.needs_input_grad[2]
    need_mat = ctx.needs_input_grad[3]
    grad_value, grad_mat = spmm_minmax_bw(col, value, mat, grad_out, arg_out, need_value, need_mat)
    return None, None, grad_value, grad_mat


class SPMMMin(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rowptr, col, value, mat):
        return _minmax_forward(ctx, "min", rowptr, col, value, mat)

    @staticmethod
    def backward(ctx, grad_out, _grad_arg):
        return _minmax_backward(ctx, grad_out)


class SPMMMax(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rowptr, col, value, mat):
        return _minmax_forward(ctx, "max", rowptr, col, value, mat)

    @staticmethod
    def backward(ctx, grad_out, _grad_arg):
        return _minmax_backward(ctx, grad_out)


# Exported operators: same signatures as torch.ops.torch_sparse.spmm_{sum,mean,min,max}
# (csrc/spmm.cpp:305-342).
def spmm_sum(row: Optional[Tensor], rowptr: Tensor, col: Tensor, value: Optional[Tensor],
             colptr: Optional[Tensor], csr2csc: Optional[Tensor], mat: Tensor,
             row_csc: Optional[Tensor] = None) -> Tensor:
    return SPMMSum.apply(row, rowptr, col, value, colptr, csr2csc, mat, row_csc)


def spmm_mean(row: Optional[Tensor], rowptr: Tensor, col: Tensor, value: Optional[Tensor],
              rowcount: Optional[Tensor], colptr: Optional[Tensor], csr2csc: Optional[Tensor],
              mat: Tensor, row_csc: Optional[Tensor] = None) -> Tensor:
    return SPMMMean.apply(row, rowptr, col, value, rowcount, colptr, csr2csc, mat, row_csc)


def spmm_res(row: Optional[Tensor], rowptr: Tensor, col: Tensor, value: Optional[Tensor], rowcount: Optional[Tensor],
             colptr: Optional[Tensor], csr2csc: Optional[Tensor], mat: Tensor, row_csc: Optional[Tensor],
             residual: Tensor, residual_scale: Optional[Tensor], reduce: str) -> Tensor:
    return SPMMRes.apply(row, rowptr, col, value, rowcount, colptr, csr2csc, mat, row_csc, residual, residual_scale,
                         reduce)


def spmm_min(rowptr: Tensor, col: Tensor, value: Optional[Tensor], mat: Tensor) -> Tuple[Tensor, Tensor]:
    return SPMMMin.apply(rowptr, col, value, mat)


def spmm_max(rowptr: Tensor, col: Tensor, value: Optional[Tensor], mat: Tensor) -> Tuple[Tensor, Tensor]:
    return SPMMMax.apply(rowptr, col, value, mat)


# --------------------------------------------------------------------------------------------------
# SDDMM: per-entry dot products of two dense operands
# --------------------------------------------------------------------------------------------------
def _sddmm_check(rowptr: Tensor, col: Tensor, a: Tensor, b: Tensor, colptr: Optional[Tensor]) -> None:
    for t, n in ((rowptr, "rowptr"), (col, "col"), (a, "a"), (b, "b")):
        _check_cuda(t, n)
    for t, n in ((a, "a"), (b, "b")):
        if t.dim() != 2:
            raise RuntimeError(f"sddmm: {n} must be 2-D, got {t.dim()}-D")
    if not a.dtype.is_floating_point or a.dtype not in _DTYPES:
        raise RuntimeError(f'"sddmm" not implemented for \'{a.dtype}\'')
    if b.dtype != a.dtype:
        raise RuntimeError(f"sddmm: a and b must have the same dtype, got {a.dtype} and {b.dtype}")
    M = rowptr.numel() - 1
    if a.size(0) != M or a.size(1) != b.size(1):
        raise RuntimeError(f"sddmm: a must be [M, K] = [{M}, {b.size(1)}] for b of shape {list(b.shape)}, "
                           f"got {list(a.shape)}")
    if colptr is not None and colptr.numel() - 1 != b.size(0):
        raise RuntimeError(f"sddmm: b must have {colptr.numel() - 1} rows (the matrix's columns), got {b.size(0)}")


class SDDMM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, row, rowptr, col, colptr, csr2csc, row_csc, a, b):
        need_a, need_b = ctx.needs_input_grad[6], ctx.needs_input_grad[7]
        if need_b:
            _assert_present(colptr, "colptr")
            _assert_present(csr2csc, "csr2csc")
        # the SpMM value gradient with grad := a, mat := b (tsb200_spmm_value_bw, reduce = sum)
        out = spmm_value_bw(row, rowptr, col, b, a, "sum")
        ctx.save_for_backward(row if need_b else None, rowptr if need_a else None, col if need_a else None,
                              colptr if need_b else None, csr2csc if need_b else None,
                              row_csc if need_b else None, a if need_b else None, b if need_a else None)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        row, rowptr, col, colptr, csr2csc, row_csc, a, b = ctx.saved_tensors
        grad_a = grad_b = None
        if ctx.needs_input_grad[6]:     # grad_a = A(g) @ b on the CSR view
            grad_a, _ = spmm_fw(rowptr, col, grad_out, b, "sum")
        if ctx.needs_input_grad[7]:     # grad_b = A(g)^T @ a on the CSC view
            if row_csc is None:
                row_csc = row.index_select(0, csr2csc)
            grad_b, _ = spmm_fw(colptr, row_csc, grad_out.index_select(0, csr2csc), a, "sum")
        return None, None, None, None, None, None, grad_a, grad_b


def sddmm(row: Tensor, rowptr: Tensor, col: Tensor, colptr: Optional[Tensor], csr2csc: Optional[Tensor],
          row_csc: Optional[Tensor], a: Tensor, b: Tensor) -> Tensor:
    """`out[e] = <a[row[e]], b[col[e]]>` for every entry of the CSR structure (rowptr, col), in CSR order, with `row`
    its COO row. `a` [M, K] and `b` [N, K] share a floating dtype; fp32 accumulation (fp64 for fp64), one rounding to
    the dtype. Differentiable in `a` (an SpMM on the CSR view) and `b` (an SpMM on the CSC view, which needs `colptr`,
    `csr2csc` and optionally the cached `row_csc = row[csr2csc]`)."""
    _sddmm_check(rowptr, col, a, b, colptr)
    return SDDMM.apply(row, rowptr, col, colptr, csr2csc, row_csc, a, b)


# --------------------------------------------------------------------------------------------------
# Multi-head SpMM / SDDMM: one weight per entry and head over [rows, H, D] operands
# --------------------------------------------------------------------------------------------------
def _heads_dtype(what: str, t: Tensor) -> None:
    if not t.dtype.is_floating_point or t.dtype not in _DTYPES:
        raise RuntimeError(f'"{what}" not implemented for \'{t.dtype}\'')


def _spmm_heads_check(rowptr: Tensor, col: Tensor, value: Optional[Tensor], x: Tensor,
                      colptr: Optional[Tensor]) -> None:
    for t, n in ((rowptr, "rowptr"), (col, "col"), (x, "x")):
        _check_cuda(t, n)
    if value is not None:
        _check_cuda(value, "value")
    if x.dim() != 3:
        raise RuntimeError(f"spmm_heads: x must be 3-D [N, H, D], got {x.dim()}-D")
    _heads_dtype("spmm_heads", x)
    E, H = col.numel(), x.size(1)
    if value is not None:
        if value.dim() != 2 or value.size(0) != E or value.size(1) != H:
            raise RuntimeError(f"spmm_heads: value must be [E, H] = [{E}, {H}], got {list(value.shape)}")
        if value.dtype != x.dtype:
            raise RuntimeError(f"spmm_heads: value and x must have the same dtype, got {value.dtype} and {x.dtype}")
    if colptr is not None and colptr.numel() - 1 != x.size(0):
        raise RuntimeError(f"spmm_heads: x must have {colptr.numel() - 1} rows (the matrix's columns), got {x.size(0)}")


def _sddmm_heads_check(rowptr: Tensor, col: Tensor, a: Tensor, b: Tensor, colptr: Optional[Tensor]) -> None:
    for t, n in ((rowptr, "rowptr"), (col, "col"), (a, "a"), (b, "b")):
        _check_cuda(t, n)
    for t, n in ((a, "a"), (b, "b")):
        if t.dim() != 3:
            raise RuntimeError(f"sddmm_heads: {n} must be 3-D [rows, H, D], got {t.dim()}-D")
    _heads_dtype("sddmm_heads", a)
    if b.dtype != a.dtype:
        raise RuntimeError(f"sddmm_heads: a and b must have the same dtype, got {a.dtype} and {b.dtype}")
    M = rowptr.numel() - 1
    if a.size(0) != M or a.shape[1:] != b.shape[1:]:
        raise RuntimeError(f"sddmm_heads: a must be [M, H, D] = [{M}, {b.size(1)}, {b.size(2)}] for b of shape "
                           f"{list(b.shape)}, got {list(a.shape)}")
    if colptr is not None and colptr.numel() - 1 != b.size(0):
        raise RuntimeError(f"sddmm_heads: b must have {colptr.numel() - 1} rows (the matrix's columns), got {b.size(0)}")


def _spmm_heads_fw(rowptr: Tensor, col: Tensor, value: Optional[Tensor], x: Tensor) -> Tensor:
    """out [M, H, D] = per head h, sum over row m's entries of value[e, h] * x[col_e, h] (tsb200_spmm_heads); a
    plannable product uses the plan cached for `rowptr`, like `spmm_fw`."""
    rowptr, col, x = _i64(rowptr, "rowptr"), _i64(col, "col"), x.contiguous()
    if value is not None:
        value = value.contiguous()
    M, (N, H, D), E = rowptr.numel() - 1, x.shape, col.numel()
    dev = x.device
    out = torch.empty((M, H, D), dtype=x.dtype, device=dev)
    if out.numel() == 0:
        return out
    dt = _dtype_code(x.dtype)
    with _on_device(dev):
        plannable = E > 0 and dt in (0, 2, 3) and (D * x.element_size()) % 16 == 0
        pl, ws, nws = _plan_workspace(None, plannable, rowptr, 1, M, H * D, E, dt, 0, dev)
        check(lib.tsb200_spmm_heads(_p(rowptr), _p(col), _p(value), _p(x), _p(out), M, N, H, D, E, dt, *pl,
                                    _p(ws), nws, _stream(dev)), "tsb200_spmm_heads")
    return out


def _sddmm_heads_fw(rowptr: Tensor, col: Tensor, a: Tensor, b: Tensor) -> Tensor:
    """s [E, H] = per head h, <a[row_e, h], b[col_e, h]> in CSR order (tsb200_sddmm_heads)."""
    rowptr, col, a, b = _i64(rowptr, "rowptr"), _i64(col, "col"), a.contiguous(), b.contiguous()
    M, (N, H, D), E = rowptr.numel() - 1, b.shape, col.numel()
    dev = a.device
    out = torch.empty((E, H), dtype=a.dtype, device=dev)
    if out.numel() == 0:
        return out
    dt = _dtype_code(a.dtype)
    with _on_device(dev):
        nws = lib.tsb200_spmm_value_bw_workspace_bytes(1, M, H * D, E, dt)
        ws = _workspace(nws, dev)
        check(lib.tsb200_sddmm_heads(_p(rowptr), _p(col), _p(a), _p(b), _p(out), M, N, H, D, E, dt, _p(ws), nws,
                                     _stream(dev)), "tsb200_sddmm_heads")
    return out


class SPMMHeads(torch.autograd.Function):
    @staticmethod
    def forward(ctx, row, rowptr, col, value, colptr, csr2csc, x, row_csc=None):
        has_value = value is not None
        need_x = ctx.needs_input_grad[6]
        if need_x:
            _assert_present(colptr, "colptr")
            _assert_present(csr2csc, "csr2csc")
            if row_csc is None:
                _assert_present(row, "row")
        out = _spmm_heads_fw(rowptr, col, value, x)
        ctx.has_value = has_value
        ctx.save_for_backward(row if need_x else None, rowptr, col, value, colptr if need_x else None,
                              csr2csc if need_x else None, x if has_value and ctx.needs_input_grad[3] else None,
                              row_csc if need_x else None)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        row, rowptr, col, value, colptr, csr2csc, x, row_csc = ctx.saved_tensors
        grad_value = grad_x = None
        if ctx.has_value and ctx.needs_input_grad[3]:     # d value[e, h] = <g[row_e, h], x[col_e, h]>
            grad_value = _sddmm_heads_fw(rowptr, col, grad_out, x)
        if ctx.needs_input_grad[6]:     # d x = A^T(value) @ g per head, on the CSC view
            if row_csc is None:
                row_csc = row.index_select(0, csr2csc)
            v = value.index_select(0, csr2csc) if ctx.has_value else None
            grad_x = _spmm_heads_fw(colptr, row_csc, v, grad_out)
        return None, None, None, grad_value, None, None, grad_x, None


class SDDMMHeads(torch.autograd.Function):
    @staticmethod
    def forward(ctx, row, rowptr, col, colptr, csr2csc, row_csc, a, b):
        need_a, need_b = ctx.needs_input_grad[6], ctx.needs_input_grad[7]
        if need_b:
            _assert_present(colptr, "colptr")
            _assert_present(csr2csc, "csr2csc")
        out = _sddmm_heads_fw(rowptr, col, a, b)
        ctx.save_for_backward(row if need_b else None, rowptr if need_a else None, col if need_a else None,
                              colptr if need_b else None, csr2csc if need_b else None,
                              row_csc if need_b else None, a if need_b else None, b if need_a else None)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        row, rowptr, col, colptr, csr2csc, row_csc, a, b = ctx.saved_tensors
        grad_a = grad_b = None
        if ctx.needs_input_grad[6]:     # grad_a = A(g) @ b per head, on the CSR view
            grad_a = _spmm_heads_fw(rowptr, col, grad_out, b)
        if ctx.needs_input_grad[7]:     # grad_b = A(g)^T @ a per head, on the CSC view
            if row_csc is None:
                row_csc = row.index_select(0, csr2csc)
            grad_b = _spmm_heads_fw(colptr, row_csc, grad_out.index_select(0, csr2csc), a)
        return None, None, None, None, None, None, grad_a, grad_b


def spmm_heads(row: Optional[Tensor], rowptr: Tensor, col: Tensor, value: Optional[Tensor], colptr: Optional[Tensor],
               csr2csc: Optional[Tensor], x: Tensor, row_csc: Optional[Tensor] = None) -> Tensor:
    """`out[m, h] = sum_{e in row m} value[e, h] * x[col_e, h]` for `x` [N, H, D] and `value` [E, H] (None: all ones),
    `out` [M, H, D]; bf16 / f16 / f32 / f64 with fp32 accumulation (fp64 for fp64) and one rounding. Differentiable in
    `value` (`sddmm_heads(g, x)`) and `x` (an `spmm_heads` on the CSC view, which needs `colptr`, `csr2csc` and `row`
    or the cached `row_csc = row[csr2csc]`)."""
    _spmm_heads_check(rowptr, col, value, x, colptr)
    return SPMMHeads.apply(row, rowptr, col, value, colptr, csr2csc, x, row_csc)


def sddmm_heads(row: Tensor, rowptr: Tensor, col: Tensor, colptr: Optional[Tensor], csr2csc: Optional[Tensor],
                row_csc: Optional[Tensor], a: Tensor, b: Tensor) -> Tensor:
    """`s[e, h] = <a[row_e, h], b[col_e, h]>` for `a` [M, H, D] and `b` [N, H, D], `s` [E, H] in CSR order; dtypes and
    accumulation as `sddmm`. Differentiable in `a` (an `spmm_heads` with values g on the CSR view) and `b` (one on the
    CSC view, which needs `colptr`, `csr2csc` and optionally the cached `row_csc`)."""
    _sddmm_heads_check(rowptr, col, a, b, colptr)
    return SDDMMHeads.apply(row, rowptr, col, colptr, csr2csc, row_csc, a, b)


FP8_SDDMM_MAX_K = 2048


def _fp8_scale(what: str, name: str, scale: Tensor, rows: int) -> int:
    if scale.dtype != torch.float32:
        raise RuntimeError(f"{what}: {name} must be float32, got {scale.dtype}")
    if scale.dim() == 0:
        return 0
    if scale.dim() == 1 and scale.size(0) == rows:
        return 1
    raise RuntimeError(f"{what}: {name} must have shape [] or [{rows}], got {list(scale.shape)}")


def sddmm_fp8(rowptr: Tensor, col: Tensor, a8: Tensor, a_scale: Tensor, b8: Tensor, b_scale: Tensor,
              out_dtype: torch.dtype = torch.float32) -> Tensor:
    """`sddmm_fp8(rowptr, col, a8, a_scale, b8, b_scale, out_dtype) -> out[E]` (tsb200_sddmm_fp8): per entry e (row r,
    column c) the dot product of two e4m3 rows, out[e] = round_out(fl32(fl32(a_scale[r] * b_scale[c]) * d_e)) with
    d_e = sum_k a8[r, k] * b8[c, k] accumulated in fp32 (every product exact). `a8` [M, K] and `b8` [N, K] are
    contiguous, 16-byte aligned e4m3 (as `quantize_fp8` makes them), K % 16 == 0 and K <= 2048; scales are float32 of
    shape [] or [rows]; out_dtype bf16, f16 or f32. Forward only."""
    what = "sddmm_fp8"
    for t, n in ((rowptr, "rowptr"), (col, "col"), (a8, "a8"), (a_scale, "a_scale"), (b8, "b8"), (b_scale, "b_scale")):
        _check_cuda(t, n)
    if torch.is_grad_enabled() and (a_scale.requires_grad or b_scale.requires_grad):
        raise RuntimeError(f"{what} is forward only: a_scale and b_scale must not require grad "
                           "(call it under torch.no_grad() or detach them)")
    for t, n in ((a8, "a8"), (b8, "b8")):
        if t.dtype != torch.float8_e4m3fn:
            raise RuntimeError(f"{what}: {n} must be torch.float8_e4m3fn, got {t.dtype}")
        if t.dim() != 2:
            raise RuntimeError(f"{what}: {n} must be 2-D, got {t.dim()}-D")
    M = rowptr.numel() - 1
    K = b8.size(1)
    if a8.size(0) != M or a8.size(1) != K:
        raise RuntimeError(f"{what}: a8 must be [M, K] = [{M}, {K}] for b8 of shape {list(b8.shape)}, "
                           f"got {list(a8.shape)}")
    if K % 16 != 0:
        raise ValueError(f"{what}: the number of columns K = {K} must be a multiple of 16")
    if K > FP8_SDDMM_MAX_K:
        raise ValueError(f"{what}: the number of columns K = {K} must be at most {FP8_SDDMM_MAX_K}")
    for t, n in ((a8, "a8"), (b8, "b8")):
        if not t.is_contiguous() or t.data_ptr() % 16 != 0:
            raise RuntimeError(f"{what}: {n} must be contiguous and 16-byte aligned")
    if out_dtype not in _FP8_OUT:
        raise RuntimeError(f"{what}: out_dtype must be torch.bfloat16, torch.float16 or torch.float32, got {out_dtype}")
    sa = _fp8_scale(what, "a_scale", a_scale, M)
    sb = _fp8_scale(what, "b_scale", b_scale, b8.size(0))
    _check_input(rowptr.dim() == 1 and col.dim() == 1)
    rowptr, col = _i64(rowptr, "rowptr"), _i64(col, "col")
    a_scale, b_scale = a_scale.contiguous(), b_scale.contiguous()
    E, N = col.numel(), b8.size(0)
    dev = b8.device
    if E == 0 or M == 0 or K == 0:     # nothing to launch; an empty dot product is +0
        return torch.zeros(E, dtype=out_dtype, device=dev)
    out = torch.empty(E, dtype=out_dtype, device=dev)
    with _on_device(dev):
        nws = lib.tsb200_sddmm_fp8_workspace_bytes(M, K, E)
        ws = _workspace(nws, dev)
        check(lib.tsb200_sddmm_fp8(_p(rowptr), _p(col), _p(a8), _p(a_scale), sa, _p(b8), _p(b_scale), sb, _p(out),
                                   M, N, K, E, _FP8_OUT[out_dtype], _p(ws), nws, _stream(dev)), "tsb200_sddmm_fp8")
    return out


def cuda_version() -> int:
    """CUDA toolkit version of the native library in CUDA_VERSION encoding, like
    torch.ops.torch_sparse.cuda_version() (csrc/version.cpp:27-41)."""
    return _lib.lib.tsb200_cuda_version()
