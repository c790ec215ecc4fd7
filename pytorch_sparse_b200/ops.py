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
from typing import Optional, Tuple

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
        if plan is None and plannable:
            plan = _auto_plan(rowptr, E)
        if plan is not None and plannable and plan.M == M and plan.E == E:
            nws = lib.tsb200_spmm_fw_planned_workspace_bytes(K, plan.n_long, plan.n_slot, red)
            ws = _workspace(nws, dev)
            rc = lib.tsb200_spmm_fw_planned(_p(rowptr), _p(col), _p(value), _p(mat), _p(out), _p(arg_out), M, N, K, E,
                                            dt, red, _p(plan.data), plan.data.numel(), plan.n_seg, plan.n_long,
                                            plan.n_slot, _p(ws), nws, _stream(dev))
            if rc != -2:   # TSB200_ERR_UNSUPPORTED (alignment): fall through to the unplanned call
                check(rc, "tsb200_spmm_fw_planned")
                return out, arg_out
        nws = lib.tsb200_spmm_fw_workspace_bytes(B, M, K, E, dt, red)
        ws = _workspace(nws, dev)
        check(lib.tsb200_spmm_fw(_p(rowptr), _p(col), _p(value), _p(mat), _p(out), _p(arg_out),
                                 B, M, N, K, E, dt, red, _p(ws), nws, _stream(dev)), "tsb200_spmm_fw")
    return out, arg_out


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
    # kept as an option.
    mode = os.environ.get("TSB200_SPSPMM", "two_phase")
    with _on_device(dev):
        nws = lib.tsb200_spspmm_workspace_bytes(M, Kd, N, nnz_a, nnz_b)
        ws = _workspace(nws, dev)
        st = _stream(dev)
        pin = _PinnedScalar()
        if mode in ("fused", "auto"):
            # single pass: output arrays sized by the number of products (an upper bound of nnz(C)); taken when that
            # bound fits comfortably into the memory still available, otherwise count first (two phases)
            check(lib.tsb200_spspmm_bound(_p(col_a), _p(rowptr_b), nnz_a, _p(ws), nws, pin.ptr(), st),
                  "tsb200_spspmm_bound")
            torch.cuda.current_stream(dev).synchronize()
            bound = pin.read()
            pin = _PinnedScalar()
            if mode == "fused" or bound * (16 + esize) <= 0.45 * _available_bytes(dev):
                row_c = torch.empty(bound, dtype=torch.int64, device=dev)
                col_c = torch.empty(bound, dtype=torch.int64, device=dev)
                val_c = torch.empty(bound, dtype=dtype, device=dev) if want_value else None
                check(lib.tsb200_spspmm_fused(_p(rowptr_a), _p(col_a), _p(val_a), _p(rowptr_b), _p(col_b), _p(val_b),
                                              M, Kd, N, nnz_a, nnz_b, _p(rowptr_c), _p(row_c), _p(col_c), _p(val_c),
                                              bound, _dtype_code(dtype) if want_value else 0, _p(ws), nws, pin.ptr(),
                                              st), "tsb200_spspmm_fused")
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
                                            _p(col_c), _p(val_c), _dtype_code(dtype) if want_value else 0,
                                            _p(ws), nws, st), "tsb200_spspmm_numeric")
    return rowptr_c, row_c, col_c, val_c


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
        grad_value = grad_mat = None
        if ctx.has_value and ctx.needs_input_grad[3]:
            grad_value = spmm_value_bw(row, rowptr, col, mat, grad_out, "sum")
        if ctx.needs_input_grad[6]:
            # grad_mat = A^T @ grad_out as a CSR SpMM on the CSC view (csrc/spmm.cpp:100-108)
            v = value.index_select(0, csr2csc) if ctx.has_value else None
            if row_csc is None:
                row_csc = row.index_select(0, csr2csc)
            grad_mat, _ = spmm_fw(colptr, row_csc, v, grad_out, "sum")
        return None, None, None, grad_value, None, None, grad_mat, None


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
        grad_value = grad_mat = None
        if ctx.has_value and ctx.needs_input_grad[3]:
            grad_value = spmm_value_bw(row, rowptr, col, mat, grad_out, "mean")
        if ctx.needs_input_grad[7]:
            # per-nnz weight value/count(row) (or 1/count) in CSC order (csrc/spmm.cpp:166-177)
            if row_csc is None:
                row_csc = row.index_select(0, csr2csc)
            cnt = rowcount.index_select(0, row_csc).to(mat.dtype).clamp_(min=1)
            w = value.index_select(0, csr2csc).div(cnt) if ctx.has_value else cnt.reciprocal_()
            grad_mat, _ = spmm_fw(colptr, row_csc, w, grad_out, "sum")
        return None, None, None, grad_value, None, None, None, grad_mat, None


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


def spmm_min(rowptr: Tensor, col: Tensor, value: Optional[Tensor], mat: Tensor) -> Tuple[Tensor, Tensor]:
    return SPMMMin.apply(rowptr, col, value, mat)


def spmm_max(rowptr: Tensor, col: Tensor, value: Optional[Tensor], mat: Tensor) -> Tuple[Tensor, Tensor]:
    return SPMMMax.apply(rowptr, col, value, mat)


def cuda_version() -> int:
    """CUDA toolkit version of the native library in CUDA_VERSION encoding, like
    torch.ops.torch_sparse.cuda_version() (csrc/version.cpp:27-41)."""
    return _lib.lib.tsb200_cuda_version()
