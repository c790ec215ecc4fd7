"""Return codes of the 17 C entry points of `csrc/spmm_fw.cu` and `csrc/spmm_bw.cu`, without a GPU: the workspace and
plan sizes, every early exit (negative extents and counts, bad enums and strides, required NULLs, extent limits at and
just past their boundary, pointer alignments, workspace and plan faults, nothing to do), and which calls pass
validation on the vector path and on the generic or fallback path.

Pointers are fake (`P` = 256, 256-byte aligned) and never dereferenced. The table runs in a child interpreter that sees
no CUDA device (CUDA_VISIBLE_DEVICES=""), so a call that passes validation fails at its first CUDA call with a positive
CUDA error: those rows expect `CUDA`, never a particular code. Where both paths of an entry point end that way, a short
workspace tells them apart: the row-split path reports it (-3), the generic path never reads the workspace."""
import json
import os
import subprocess
import sys
from pathlib import Path

import pytest

F32, F64, F16, BF16, I32 = 0, 1, 2, 3, 4
SUM, MEAN, MIN, MAX = 0, 1, 2, 3
INVALID, UNSUPPORTED, WORKSPACE = -1, -2, -3
CUDA = "cuda"  # passed validation: the first CUDA call fails with a positive code

P = 256               # a 256-byte aligned fake pointer
W = 1 << 20           # a 256-byte aligned fake workspace or plan
MIS = W | 128         # a misaligned one
BIG = 1 << 62         # a byte count no layout reaches
E_MAX = (1 << 31) - 65  # the most entries the row-split kernels take
N_MAX = (1 << 32) - 1   # the most dense rows (and rows M of a second operand gathered by row index)

# argument names and defaults of each entry point, in signature order; the defaults pass validation on the vector path
BASE = {
    "spmm_fw_workspace_bytes": dict(B=1, M=100, K=64, E=1000, dtype=F32, reduce=SUM),
    "spmm_fw": dict(rowptr=P, col=P, value=P, mat=P, out=P, arg_out=P, B=1, M=64, N=64, K=64, E=1000, dtype=BF16,
                    reduce=SUM, ws=W, wsb=BIG, stream=None),
    "spmm_fw_acc": dict(rowptr=P, col=P, value=P, mat=P, out=P, partial=P, acc_mode=3, B=1, M=64, N=64, K=64, E=1000,
                        dtype=BF16, ws=W, wsb=BIG, stream=None),
    "spmm_plan_bytes": dict(M=100, E=1000),
    "spmm_plan": dict(rowptr=P, M=100, E=1000, plan=W, pb=BIG, counts=None, stream=None),
    "spmm_fw_planned_workspace_bytes": dict(K=64, n_long=3, n_slot=10, reduce=SUM),
    "spmm_fw_planned": dict(rowptr=P, col=P, value=P, mat=P, out=P, arg_out=P, M=64, N=64, K=64, E=1000, dtype=BF16,
                            reduce=SUM, plan=W, pb=BIG, ns=5, nl=2, nsl=8, ws=W, wsb=BIG, stream=None),
    "spmm_fw_fp8": dict(rowptr=P, col=P, value=P, mat=P, scale=P, scale_stride=1, out=P, arg_out=P, M=64, N=64, K=64,
                        E=1000, out_dtype=BF16, reduce=SUM, plan=None, pb=0, ns=0, nl=0, nsl=0, ws=W, wsb=BIG,
                        stream=None),
    "spmm_fw_fp8_quant": dict(rowptr=P, col=P, value=P, mat=P, scale=P, scale_stride=1, out=P, out_scale=P, arg_out=P,
                              M=64, N=64, K=64, E=1000, reduce=SUM, plan=None, pb=0, ns=0, nl=0, nsl=0, ws=W, wsb=BIG,
                              stream=None),
    "spmm_fw_fp8_res": dict(rowptr=P, col=P, value=P, mat=P, scale=P, scale_stride=1, res8=P, res_scale=P,
                            res_stride=1, out=P, out_scale=None, arg_out=P, M=64, N=64, K=64, E=1000, out_dtype=BF16,
                            reduce=SUM, plan=None, pb=0, ns=0, nl=0, nsl=0, ws=W, wsb=BIG, stream=None),
    "spmm_heads": dict(rowptr=P, col=P, value=P, x=P, out=P, M=64, N=64, H=2, D=16, E=1000, dtype=BF16, plan=None,
                       pb=0, ns=0, nl=0, nsl=0, ws=W, wsb=BIG, stream=None),
    "spmm_value_bw_workspace_bytes": dict(B=1, M=100, K=64, E=1000, dtype=F32),
    "spmm_value_bw": dict(row=P, rowptr=P, col=P, mat=P, grad=P, out=P, B=1, M=64, N=64, K=64, E=1000, dtype=BF16,
                          reduce=SUM, ws=W, wsb=BIG, stream=None),
    "sddmm_fp8_workspace_bytes": dict(M=100, K=64, E=1000),
    "sddmm_fp8": dict(rowptr=P, col=P, a8=P, a_scale=P, a_stride=1, b8=P, b_scale=P, b_stride=1, out=P, M=64, N=64,
                      K=64, E=1000, out_dtype=BF16, ws=W, wsb=BIG, stream=None),
    "spmm_minmax_bw": dict(col=P, value=P, mat=P, grad_out=P, arg_out=P, grad_value=P, grad_mat=P, B=1, M=64, N=64,
                           K=64, E=1000, dtype=BF16, stream=None),
    "sddmm_heads": dict(rowptr=P, col=P, a=P, b=P, out=P, M=64, N=64, H=2, D=16, E=1000, dtype=BF16, ws=W, wsb=BIG,
                        stream=None),
}


def negatives(fn, *names):
    return [(fn, {n: -1}, INVALID) for n in names]


def workspace_faults(fn, missing=WORKSPACE, misaligned=INVALID, both=WORKSPACE, **kw):
    """NULL, short, misaligned, and short and misaligned together (which fault is reported first)."""
    return [(fn, dict(kw, ws=None), missing), (fn, dict(kw, wsb=1), WORKSPACE), (fn, dict(kw, ws=MIS), misaligned),
            (fn, dict(kw, ws=MIS, wsb=1), both)]


def plan_faults(fn, missing_ws=WORKSPACE, **kw):
    """Short plan, misaligned plan, both (the size is checked first), segment and long-row counts at and past the
    capacity of a plan of 64 rows and 1000 entries (102 segments, 67 long rows), and the planned workspace."""
    return [(fn, dict(kw, pb=1), WORKSPACE), (fn, dict(kw, plan=W | 128), INVALID), (fn, dict(kw, plan=W | 128, pb=1),
                                                                                       WORKSPACE),
            (fn, dict(kw, ns=102), CUDA), (fn, dict(kw, ns=103), INVALID),
            (fn, dict(kw, nl=67), CUDA), (fn, dict(kw, nl=68), INVALID),
            (fn, dict(kw, wsb=1), WORKSPACE), (fn, dict(kw, ws=MIS), INVALID), (fn, dict(kw, ws=None), missing_ws)]


PLANNED = dict(plan=W, pb=BIG, ns=5, nl=2, nsl=8)

TABLE = [
    # ---- sizes
    ("spmm_fw_workspace_bytes", {}, 23552),
    ("spmm_fw_workspace_bytes", dict(reduce=MAX), 59904),
    ("spmm_fw_workspace_bytes", dict(B=3, dtype=BF16, reduce=MEAN), 30464),
    ("spmm_fw_workspace_bytes", dict(M=-1), 23552),
    ("spmm_fw_workspace_bytes", dict(dtype=F64), 0),
    ("spmm_fw_workspace_bytes", dict(dtype=I32), 0),
    ("spmm_fw_workspace_bytes", dict(B=0), 0),
    ("spmm_fw_workspace_bytes", dict(K=0), 0),
    ("spmm_fw_workspace_bytes", dict(E=0), 0),
    ("spmm_plan_bytes", {}, 6144),
    ("spmm_plan_bytes", dict(M=0, E=0), 4352),
    ("spmm_plan_bytes", dict(M=-1), 0),
    ("spmm_plan_bytes", dict(E=-1), 0),
    ("spmm_fw_planned_workspace_bytes", {}, 3072),
    ("spmm_fw_planned_workspace_bytes", dict(reduce=MIN), 8192),
    ("spmm_fw_planned_workspace_bytes", dict(K=0, n_long=0, n_slot=0), 512),
    ("spmm_fw_planned_workspace_bytes", dict(K=-1), 0),
    ("spmm_fw_planned_workspace_bytes", dict(n_long=-1), 0),
    ("spmm_fw_planned_workspace_bytes", dict(n_slot=-1), 0),
    ("spmm_value_bw_workspace_bytes", {}, 5376),
    ("spmm_value_bw_workspace_bytes", dict(M=-1, dtype=F16), 5376),
    ("spmm_value_bw_workspace_bytes", dict(B=2), 0),
    ("spmm_value_bw_workspace_bytes", dict(K=0), 0),
    ("spmm_value_bw_workspace_bytes", dict(E=0), 0),
    ("spmm_value_bw_workspace_bytes", dict(dtype=F64), 0),
    ("sddmm_fp8_workspace_bytes", {}, 5376),
    ("sddmm_fp8_workspace_bytes", dict(M=-1), 5376),
    ("sddmm_fp8_workspace_bytes", dict(K=0), 0),
    ("sddmm_fp8_workspace_bytes", dict(E=0), 0),

    # ---- tsb200_spmm_fw: row-split path, else the generic kernel
    ("spmm_fw", {}, CUDA),
    ("spmm_fw", dict(reduce=MAX), CUDA),
    ("spmm_fw", dict(dtype=F64, wsb=1), CUDA),            # generic: no workspace read
    ("spmm_fw", dict(dtype=I32, wsb=1), CUDA),
    ("spmm_fw", dict(K=12, wsb=1), CUDA),                 # 24-byte rows
    *negatives("spmm_fw", "B", "M", "N", "K", "E"),
    ("spmm_fw", dict(reduce=-1), INVALID), ("spmm_fw", dict(reduce=4), INVALID),
    ("spmm_fw", dict(dtype=9), INVALID), ("spmm_fw", dict(dtype=-1), INVALID),
    ("spmm_fw", dict(M=0), 0), ("spmm_fw", dict(K=0), 0), ("spmm_fw", dict(B=0), 0),
    ("spmm_fw", dict(rowptr=None), INVALID), ("spmm_fw", dict(out=None), INVALID),
    ("spmm_fw", dict(reduce=MAX, arg_out=None), INVALID), ("spmm_fw", dict(arg_out=None), CUDA),
    ("spmm_fw", dict(col=None), INVALID), ("spmm_fw", dict(mat=None), INVALID),
    ("spmm_fw", dict(E=0, col=None, mat=None), CUDA),
    ("spmm_fw", dict(value=None, wsb=1), WORKSPACE),
    *workspace_faults("spmm_fw"),
    ("spmm_fw", dict(E=E_MAX, wsb=1), WORKSPACE), ("spmm_fw", dict(E=E_MAX + 1, wsb=1), CUDA),
    ("spmm_fw", dict(N=N_MAX, wsb=1), WORKSPACE), ("spmm_fw", dict(N=N_MAX + 1, wsb=1), CUDA),
    ("spmm_fw", dict(dtype=F32, K=(1 << 29) - 4, wsb=1), WORKSPACE), ("spmm_fw", dict(dtype=F32, K=1 << 29, wsb=1), CUDA),
    ("spmm_fw", dict(mat=P + 8, wsb=1), CUDA), ("spmm_fw", dict(mat=P + 16, wsb=1), WORKSPACE),
    ("spmm_fw", dict(out=P + 8, wsb=1), CUDA),
    ("spmm_fw", dict(col=P + 4, wsb=1), CUDA), ("spmm_fw", dict(col=P + 8, wsb=1), WORKSPACE),
    ("spmm_fw", dict(value=P + 2, wsb=1), CUDA), ("spmm_fw", dict(value=P + 4, wsb=1), WORKSPACE),
    ("spmm_fw", dict(reduce=MAX, arg_out=P + 8, wsb=1), CUDA), ("spmm_fw", dict(reduce=MAX, wsb=1), WORKSPACE),

    # ---- tsb200_spmm_fw_acc: row-split path or -2
    ("spmm_fw_acc", {}, CUDA),
    ("spmm_fw_acc", dict(acc_mode=1, out=None), CUDA),
    ("spmm_fw_acc", dict(dtype=F64), UNSUPPORTED), ("spmm_fw_acc", dict(dtype=9), UNSUPPORTED),
    *negatives("spmm_fw_acc", "B", "M", "N", "K", "E"),
    ("spmm_fw_acc", dict(E=0), INVALID),
    ("spmm_fw_acc", dict(acc_mode=0), INVALID), ("spmm_fw_acc", dict(acc_mode=4), INVALID),
    ("spmm_fw_acc", dict(partial=None), INVALID), ("spmm_fw_acc", dict(rowptr=None), INVALID),
    ("spmm_fw_acc", dict(col=None), INVALID), ("spmm_fw_acc", dict(mat=None), INVALID),
    ("spmm_fw_acc", dict(out=None), INVALID),
    ("spmm_fw_acc", dict(M=0), 0), ("spmm_fw_acc", dict(K=0), 0), ("spmm_fw_acc", dict(B=0), 0),
    ("spmm_fw_acc", dict(partial=P + 8), UNSUPPORTED), ("spmm_fw_acc", dict(dtype=F32, K=6), UNSUPPORTED),
    ("spmm_fw_acc", dict(K=12), UNSUPPORTED),
    *workspace_faults("spmm_fw_acc"),
    ("spmm_fw_acc", dict(E=E_MAX), CUDA), ("spmm_fw_acc", dict(E=E_MAX + 1), UNSUPPORTED),
    ("spmm_fw_acc", dict(N=N_MAX), CUDA), ("spmm_fw_acc", dict(N=N_MAX + 1), UNSUPPORTED),
    ("spmm_fw_acc", dict(dtype=F32, K=(1 << 29) - 4), CUDA), ("spmm_fw_acc", dict(dtype=F32, K=1 << 29), UNSUPPORTED),
    ("spmm_fw_acc", dict(mat=P + 8), UNSUPPORTED), ("spmm_fw_acc", dict(out=P + 8), UNSUPPORTED),
    ("spmm_fw_acc", dict(acc_mode=2, out=P + 8), CUDA),  # `out` is only written by the last block
    ("spmm_fw_acc", dict(col=P + 4), UNSUPPORTED), ("spmm_fw_acc", dict(value=P + 2), UNSUPPORTED),
    ("spmm_fw_acc", dict(value=None), CUDA),

    # ---- tsb200_spmm_plan
    ("spmm_plan", {}, CUDA), ("spmm_plan", dict(M=0, E=0), CUDA),
    *negatives("spmm_plan", "M", "E"),
    ("spmm_plan", dict(rowptr=None), INVALID), ("spmm_plan", dict(plan=None), INVALID),
    ("spmm_plan", dict(pb=6144), CUDA), ("spmm_plan", dict(pb=6143), WORKSPACE),
    ("spmm_plan", dict(plan=W | 128), INVALID), ("spmm_plan", dict(plan=W | 128, pb=1), WORKSPACE),

    # ---- tsb200_spmm_fw_planned: row-split path or -2
    ("spmm_fw_planned", {}, CUDA), ("spmm_fw_planned", dict(reduce=MIN), CUDA),
    ("spmm_fw_planned", dict(dtype=F64), UNSUPPORTED), ("spmm_fw_planned", dict(dtype=9), UNSUPPORTED),
    *negatives("spmm_fw_planned", "M", "N", "K", "E", "ns", "nl", "nsl"),
    ("spmm_fw_planned", dict(E=0), INVALID),
    ("spmm_fw_planned", dict(reduce=-1), INVALID), ("spmm_fw_planned", dict(reduce=4), INVALID),
    ("spmm_fw_planned", dict(M=0), 0), ("spmm_fw_planned", dict(K=0), 0),
    *[("spmm_fw_planned", {n: None}, INVALID) for n in ("rowptr", "col", "mat", "out", "plan")],
    ("spmm_fw_planned", dict(reduce=MAX, arg_out=None), INVALID), ("spmm_fw_planned", dict(arg_out=None), CUDA),
    ("spmm_fw_planned", dict(value=None), CUDA),
    *plan_faults("spmm_fw_planned"),
    ("spmm_fw_planned", dict(ws=MIS, wsb=1), WORKSPACE),
    ("spmm_fw_planned", dict(E=E_MAX), CUDA), ("spmm_fw_planned", dict(E=E_MAX + 1), UNSUPPORTED),
    ("spmm_fw_planned", dict(N=N_MAX), CUDA), ("spmm_fw_planned", dict(N=N_MAX + 1), UNSUPPORTED),
    ("spmm_fw_planned", dict(dtype=F32, K=(1 << 29) - 4), CUDA),
    ("spmm_fw_planned", dict(dtype=F32, K=1 << 29), UNSUPPORTED),
    ("spmm_fw_planned", dict(mat=P + 8), UNSUPPORTED), ("spmm_fw_planned", dict(out=P + 8), UNSUPPORTED),
    ("spmm_fw_planned", dict(col=P + 4), UNSUPPORTED), ("spmm_fw_planned", dict(value=P + 2), UNSUPPORTED),
    ("spmm_fw_planned", dict(value=P + 4), CUDA),
    ("spmm_fw_planned", dict(reduce=MAX, arg_out=P + 8), UNSUPPORTED),

    # ---- tsb200_spmm_fw_fp8: row-split path (planned or not) or -2
    ("spmm_fw_fp8", {}, CUDA), ("spmm_fw_fp8", dict(PLANNED), CUDA), ("spmm_fw_fp8", dict(reduce=MAX), CUDA),
    ("spmm_fw_fp8", dict(out_dtype=F32, scale_stride=0, value=None), CUDA),
    *negatives("spmm_fw_fp8", "M", "N", "K", "E", "ns", "nl", "nsl"),
    ("spmm_fw_fp8", dict(reduce=-1), INVALID), ("spmm_fw_fp8", dict(reduce=4), INVALID),
    ("spmm_fw_fp8", dict(scale_stride=2), INVALID), ("spmm_fw_fp8", dict(scale_stride=-1), INVALID),
    ("spmm_fw_fp8", dict(out_dtype=F64), UNSUPPORTED), ("spmm_fw_fp8", dict(out_dtype=I32), UNSUPPORTED),
    ("spmm_fw_fp8", dict(K=24), UNSUPPORTED), ("spmm_fw_fp8", dict(K=4096), CUDA),
    ("spmm_fw_fp8", dict(M=0), 0), ("spmm_fw_fp8", dict(K=0), 0),
    ("spmm_fw_fp8", dict(rowptr=None), INVALID), ("spmm_fw_fp8", dict(out=None), INVALID),
    ("spmm_fw_fp8", dict(reduce=MAX, arg_out=None), INVALID),
    ("spmm_fw_fp8", dict(E=0, col=None, mat=None, scale=None, ws=None), CUDA),  # every row empty: memsets
    ("spmm_fw_fp8", dict(col=None), INVALID), ("spmm_fw_fp8", dict(mat=None), INVALID),
    ("spmm_fw_fp8", dict(scale=None), INVALID),
    ("spmm_fw_fp8", dict(E=E_MAX), CUDA), ("spmm_fw_fp8", dict(E=E_MAX + 1), UNSUPPORTED),
    ("spmm_fw_fp8", dict(N=N_MAX), CUDA), ("spmm_fw_fp8", dict(N=N_MAX + 1), UNSUPPORTED),
    ("spmm_fw_fp8", dict(K=(1 << 31) - 16), CUDA), ("spmm_fw_fp8", dict(K=1 << 31), UNSUPPORTED),
    ("spmm_fw_fp8", dict(mat=P + 8), UNSUPPORTED), ("spmm_fw_fp8", dict(out=P + 8), UNSUPPORTED),
    ("spmm_fw_fp8", dict(col=P + 4), UNSUPPORTED), ("spmm_fw_fp8", dict(scale=P + 2), UNSUPPORTED),
    ("spmm_fw_fp8", dict(scale=P + 4), CUDA), ("spmm_fw_fp8", dict(value=P + 2), UNSUPPORTED),
    ("spmm_fw_fp8", dict(value=P + 4), CUDA),
    ("spmm_fw_fp8", dict(reduce=MAX, arg_out=P + 8), UNSUPPORTED),
    *workspace_faults("spmm_fw_fp8", missing=INVALID, both=INVALID),
    *plan_faults("spmm_fw_fp8", missing_ws=INVALID, **PLANNED),

    # ---- tsb200_spmm_fw_fp8_quant
    ("spmm_fw_fp8_quant", {}, CUDA), ("spmm_fw_fp8_quant", dict(PLANNED), CUDA),
    ("spmm_fw_fp8_quant", dict(reduce=MIN), CUDA),
    *negatives("spmm_fw_fp8_quant", "M", "N", "K", "E", "ns", "nl", "nsl"),
    ("spmm_fw_fp8_quant", dict(reduce=4), INVALID), ("spmm_fw_fp8_quant", dict(scale_stride=2), INVALID),
    ("spmm_fw_fp8_quant", dict(K=24), UNSUPPORTED),
    ("spmm_fw_fp8_quant", dict(K=2048), CUDA), ("spmm_fw_fp8_quant", dict(K=2064), UNSUPPORTED),
    ("spmm_fw_fp8_quant", dict(M=0), 0), ("spmm_fw_fp8_quant", dict(M=0, out_scale=None), 0),
    ("spmm_fw_fp8_quant", dict(K=0), CUDA),  # every scale is 1
    ("spmm_fw_fp8_quant", dict(out_scale=None), INVALID), ("spmm_fw_fp8_quant", dict(K=0, out_scale=None), INVALID),
    ("spmm_fw_fp8_quant", dict(out_scale=P + 2), UNSUPPORTED),
    ("spmm_fw_fp8_quant", dict(E=0), CUDA),
    ("spmm_fw_fp8_quant", dict(scale=None), INVALID),
    ("spmm_fw_fp8_quant", dict(E=E_MAX), CUDA), ("spmm_fw_fp8_quant", dict(E=E_MAX + 1), UNSUPPORTED),
    ("spmm_fw_fp8_quant", dict(out=P + 8), UNSUPPORTED),
    *workspace_faults("spmm_fw_fp8_quant", missing=INVALID, both=INVALID),
    ("spmm_fw_fp8_quant", dict(PLANNED, pb=1), WORKSPACE),

    # ---- tsb200_spmm_fw_fp8_res
    ("spmm_fw_fp8_res", {}, CUDA), ("spmm_fw_fp8_res", dict(PLANNED), CUDA),
    ("spmm_fw_fp8_res", dict(reduce=MEAN, res_stride=0), CUDA),
    ("spmm_fw_fp8_res", dict(out_scale=P, out_dtype=F32), CUDA),
    ("spmm_fw_fp8_res", dict(out_scale=P), INVALID),      # an e4m3 result takes float32 values
    ("spmm_fw_fp8_res", dict(out_scale=P, out_dtype=F32, K=2064), UNSUPPORTED),
    ("spmm_fw_fp8_res", dict(res8=None, reduce=MAX), CUDA),
    *negatives("spmm_fw_fp8_res", "M", "N", "K", "E", "ns", "nl", "nsl"),
    ("spmm_fw_fp8_res", dict(reduce=4), INVALID), ("spmm_fw_fp8_res", dict(scale_stride=2), INVALID),
    ("spmm_fw_fp8_res", dict(res_scale=None), INVALID), ("spmm_fw_fp8_res", dict(res_stride=2), INVALID),
    ("spmm_fw_fp8_res", dict(reduce=MAX), UNSUPPORTED), ("spmm_fw_fp8_res", dict(reduce=MIN), UNSUPPORTED),
    ("spmm_fw_fp8_res", dict(res8=P + 8), UNSUPPORTED), ("spmm_fw_fp8_res", dict(res_scale=P + 2), UNSUPPORTED),
    ("spmm_fw_fp8_res", dict(M=0), 0), ("spmm_fw_fp8_res", dict(K=0), 0),
    ("spmm_fw_fp8_res", dict(E=0, col=None, ws=None), CUDA),  # every row empty: the residual alone
    ("spmm_fw_fp8_res", dict(E=0, out=P + 8), UNSUPPORTED),
    ("spmm_fw_fp8_res", dict(E=0, out_scale=P, out_dtype=F32), CUDA),
    ("spmm_fw_fp8_res", dict(N=N_MAX + 1), UNSUPPORTED), ("spmm_fw_fp8_res", dict(col=P + 4), UNSUPPORTED),
    *workspace_faults("spmm_fw_fp8_res", missing=INVALID, both=INVALID),
    ("spmm_fw_fp8_res", dict(PLANNED, ns=103), INVALID),

    # ---- tsb200_spmm_heads: row-split path (planned or not), else the generic kernel
    ("spmm_heads", {}, CUDA), ("spmm_heads", dict(PLANNED), CUDA),
    ("spmm_heads", dict(dtype=F64, wsb=1), CUDA), ("spmm_heads", dict(dtype=F32, D=12, wsb=1), WORKSPACE),
    ("spmm_heads", dict(D=12, wsb=1), CUDA),               # 24-byte heads
    ("spmm_heads", dict(H=4, D=4, wsb=1), CUDA),           # 8-byte heads in 32-byte rows
    *negatives("spmm_heads", "M", "N", "H", "D", "E", "ns", "nl", "nsl"),
    ("spmm_heads", dict(dtype=I32), UNSUPPORTED), ("spmm_heads", dict(dtype=9), UNSUPPORTED),
    ("spmm_heads", dict(H=1 << 20, D=1 << 20), CUDA), ("spmm_heads", dict(H=1 << 20, D=(1 << 20) + 1), UNSUPPORTED),
    ("spmm_heads", dict(M=0), 0), ("spmm_heads", dict(H=0), 0), ("spmm_heads", dict(D=0), 0),
    ("spmm_heads", dict(rowptr=None), INVALID), ("spmm_heads", dict(out=None), INVALID),
    ("spmm_heads", dict(E=0, col=None, x=None), CUDA),     # every row empty: a memset
    ("spmm_heads", dict(col=None), INVALID), ("spmm_heads", dict(x=None), INVALID),
    # no weights: the plain sum of tsb200_spmm_fw / tsb200_spmm_fw_planned
    ("spmm_heads", dict(value=None), CUDA), ("spmm_heads", dict(value=None, wsb=1), WORKSPACE),
    ("spmm_heads", dict(value=None, dtype=F64, wsb=1), CUDA),
    ("spmm_heads", dict(PLANNED, value=None), CUDA), ("spmm_heads", dict(PLANNED, value=None, dtype=F64), UNSUPPORTED),
    ("spmm_heads", dict(PLANNED, value=None, pb=1), WORKSPACE),
    *workspace_faults("spmm_heads"),
    *plan_faults("spmm_heads", **PLANNED),
    ("spmm_heads", dict(E=(1 << 30) - 1, wsb=1), WORKSPACE), ("spmm_heads", dict(E=1 << 30, wsb=1), CUDA),  # H * E
    ("spmm_heads", dict(H=1, E=E_MAX, wsb=1), WORKSPACE), ("spmm_heads", dict(H=1, E=E_MAX + 1, wsb=1), CUDA),
    ("spmm_heads", dict(N=N_MAX, wsb=1), WORKSPACE), ("spmm_heads", dict(N=N_MAX + 1, wsb=1), CUDA),
    ("spmm_heads", dict(H=1, D=(1 << 30) - 8, wsb=1), WORKSPACE), ("spmm_heads", dict(H=1, D=1 << 30, wsb=1), CUDA),
    ("spmm_heads", dict(x=P + 8, wsb=1), CUDA), ("spmm_heads", dict(out=P + 8, wsb=1), CUDA),
    ("spmm_heads", dict(col=P + 4, wsb=1), CUDA), ("spmm_heads", dict(value=P + 2, wsb=1), CUDA),
    ("spmm_heads", dict(value=P + 4, wsb=1), WORKSPACE),

    # ---- tsb200_spmm_value_bw: row-wise SDDMM, nnz-parallel vector or generic kernel; all three end in CUDA here
    ("spmm_value_bw", {}, CUDA), ("spmm_value_bw", dict(reduce=MEAN), CUDA),
    ("spmm_value_bw", dict(B=2), CUDA), ("spmm_value_bw", dict(dtype=F64), CUDA), ("spmm_value_bw", dict(dtype=I32), CUDA),
    ("spmm_value_bw", dict(ws=None), CUDA), ("spmm_value_bw", dict(wsb=1), CUDA), ("spmm_value_bw", dict(ws=MIS), CUDA),
    ("spmm_value_bw", dict(E=E_MAX + 1), CUDA), ("spmm_value_bw", dict(M=N_MAX + 1), CUDA),
    ("spmm_value_bw", dict(col=P + 4), CUDA), ("spmm_value_bw", dict(mat=P + 8), CUDA),
    *negatives("spmm_value_bw", "B", "M", "N", "K", "E"),
    ("spmm_value_bw", dict(reduce=MIN), INVALID), ("spmm_value_bw", dict(reduce=MAX), INVALID),
    ("spmm_value_bw", dict(reduce=-1), INVALID), ("spmm_value_bw", dict(dtype=9), INVALID),
    ("spmm_value_bw", dict(E=0), 0), ("spmm_value_bw", dict(E=0, row=None, out=None), 0),
    *[("spmm_value_bw", {n: None}, INVALID) for n in ("row", "rowptr", "col", "out", "mat", "grad")],
    ("spmm_value_bw", dict(K=0, mat=None, grad=None), CUDA), ("spmm_value_bw", dict(B=0, mat=None, grad=None), CUDA),

    # ---- tsb200_sddmm_fp8: row-wise path or -2
    ("sddmm_fp8", {}, CUDA), ("sddmm_fp8", dict(out_dtype=F32, a_stride=0, b_stride=0), CUDA),
    *negatives("sddmm_fp8", "M", "N", "K", "E"),
    ("sddmm_fp8", dict(a_stride=2), INVALID), ("sddmm_fp8", dict(b_stride=-1), INVALID),
    ("sddmm_fp8", dict(out_dtype=F64), UNSUPPORTED), ("sddmm_fp8", dict(out_dtype=I32), UNSUPPORTED),
    ("sddmm_fp8", dict(K=24), UNSUPPORTED), ("sddmm_fp8", dict(K=2048), CUDA), ("sddmm_fp8", dict(K=2064), UNSUPPORTED),
    ("sddmm_fp8", dict(E=0), 0), ("sddmm_fp8", dict(E=0, out=None), 0),
    ("sddmm_fp8", dict(out=None), INVALID),
    ("sddmm_fp8", dict(out=P + 1), UNSUPPORTED), ("sddmm_fp8", dict(out=P + 2), CUDA),
    ("sddmm_fp8", dict(out_dtype=F32, out=P + 2), UNSUPPORTED),
    ("sddmm_fp8", dict(K=0, rowptr=None, col=None, a8=None, b8=None, ws=None), CUDA),  # empty dot products: a memset
    *[("sddmm_fp8", {n: None}, INVALID) for n in ("rowptr", "col", "a8", "a_scale", "b8", "b_scale")],
    ("sddmm_fp8", dict(E=E_MAX), CUDA), ("sddmm_fp8", dict(E=E_MAX + 1), UNSUPPORTED),
    ("sddmm_fp8", dict(N=N_MAX), CUDA), ("sddmm_fp8", dict(N=N_MAX + 1), UNSUPPORTED),
    ("sddmm_fp8", dict(M=N_MAX), CUDA), ("sddmm_fp8", dict(M=N_MAX + 1), UNSUPPORTED),
    ("sddmm_fp8", dict(a8=P + 8), UNSUPPORTED), ("sddmm_fp8", dict(b8=P + 8), UNSUPPORTED),
    ("sddmm_fp8", dict(col=P + 4), UNSUPPORTED),
    ("sddmm_fp8", dict(a_scale=P + 2), UNSUPPORTED), ("sddmm_fp8", dict(b_scale=P + 2), UNSUPPORTED),
    ("sddmm_fp8", dict(a_scale=P + 4, b_scale=P + 4), CUDA),
    *workspace_faults("sddmm_fp8", missing=INVALID, both=INVALID),

    # ---- tsb200_spmm_minmax_bw: one kernel
    ("spmm_minmax_bw", {}, CUDA), ("spmm_minmax_bw", dict(dtype=F64), CUDA),
    ("spmm_minmax_bw", dict(grad_value=None, mat=None), CUDA), ("spmm_minmax_bw", dict(grad_mat=None, value=None), CUDA),
    *negatives("spmm_minmax_bw", "B", "M", "N", "K", "E"),
    ("spmm_minmax_bw", dict(B=0), 0), ("spmm_minmax_bw", dict(M=0), 0), ("spmm_minmax_bw", dict(K=0), 0),
    ("spmm_minmax_bw", dict(E=0), 0),
    ("spmm_minmax_bw", dict(grad_value=None, grad_mat=None), 0),
    *[("spmm_minmax_bw", {n: None}, INVALID) for n in ("col", "grad_out", "arg_out", "mat")],
    ("spmm_minmax_bw", dict(dtype=I32), UNSUPPORTED),

    # ---- tsb200_sddmm_heads: row-wise path, else the generic kernel
    ("sddmm_heads", {}, CUDA), ("sddmm_heads", dict(dtype=F64, wsb=1), CUDA), ("sddmm_heads", dict(ws=None), CUDA),
    ("sddmm_heads", dict(ws=MIS), CUDA), ("sddmm_heads", dict(wsb=1), WORKSPACE),
    *negatives("sddmm_heads", "M", "N", "H", "D", "E"),
    ("sddmm_heads", dict(dtype=I32), UNSUPPORTED), ("sddmm_heads", dict(dtype=9), UNSUPPORTED),
    ("sddmm_heads", dict(H=1 << 20, D=1 << 20), CUDA), ("sddmm_heads", dict(H=1 << 20, D=(1 << 20) + 1), UNSUPPORTED),
    ("sddmm_heads", dict(E=0), 0), ("sddmm_heads", dict(H=0), 0), ("sddmm_heads", dict(E=0, out=None), 0),
    ("sddmm_heads", dict(out=None), INVALID),
    ("sddmm_heads", dict(D=0, rowptr=None, col=None, a=None, b=None), CUDA),  # empty dot products: a memset
    *[("sddmm_heads", {n: None}, INVALID) for n in ("rowptr", "col", "a", "b")],
    ("sddmm_heads", dict(D=24, wsb=1), CUDA),              # 3 vectors per head
    ("sddmm_heads", dict(H=2, D=256, wsb=1), WORKSPACE),   # 32 per head, 64 per row
    ("sddmm_heads", dict(H=1, D=512, wsb=1), CUDA),        # 64 per head
    ("sddmm_heads", dict(H=4, D=256, wsb=1), CUDA),        # 128 per row
    ("sddmm_heads", dict(H=1, E=E_MAX, wsb=1), WORKSPACE), ("sddmm_heads", dict(H=1, E=E_MAX + 1, wsb=1), CUDA),
    ("sddmm_heads", dict(M=N_MAX, wsb=1), WORKSPACE), ("sddmm_heads", dict(M=N_MAX + 1, wsb=1), CUDA),
    ("sddmm_heads", dict(N=N_MAX, wsb=1), WORKSPACE), ("sddmm_heads", dict(N=N_MAX + 1, wsb=1), CUDA),
    ("sddmm_heads", dict(a=P + 8, wsb=1), CUDA), ("sddmm_heads", dict(b=P + 8, wsb=1), CUDA),
    ("sddmm_heads", dict(col=P + 4, wsb=1), CUDA),
    ("sddmm_heads", dict(out=P + 1, wsb=1), CUDA), ("sddmm_heads", dict(out=P + 2, wsb=1), WORKSPACE),
]


def _label(i, row):
    fn, over, _ = row
    return f"{i:03d}-{fn}(" + ",".join(f"{k}={v}" for k, v in over.items()) + ")"


def _run():
    """In the child: refuse to call anything if a CUDA device is visible, else print every row's result as JSON."""
    import torch
    assert torch.cuda.device_count() == 0, "a CUDA device is visible: no entry point is called"
    from pytorch_sparse_b200 import _lib
    codes = []
    for fn, over, _ in TABLE:
        args = dict(BASE[fn])
        assert set(over) <= set(args), (fn, over)
        args.update(over)
        codes.append(getattr(_lib.lib, "tsb200_" + fn)(*args.values()))
    print(json.dumps(codes))


@pytest.fixture(scope="module")
def codes():
    here = Path(__file__).resolve().parent
    code = f"import sys; sys.path[:0] = [{str(here.parent)!r}, {str(here)!r}]; import {Path(__file__).stem} as t; t._run()"
    flags = ["-s"] if sys.flags.no_user_site else []
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, *flags, "-c", code], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, f"the table failed to run:\n{r.stdout[-4000:]}\n{r.stderr[-4000:]}"
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_covers_every_entry_point():
    from pytorch_sparse_b200 import _lib
    csrc = Path(__file__).resolve().parent.parent / "pytorch_sparse_b200" / "csrc"
    names = set()
    for src in ("spmm_fw.cu", "spmm_bw.cu"):
        for line in (csrc / src).read_text().splitlines():
            if line.startswith('extern "C"'):
                names.add(line.split("(")[0].split()[-1])
    assert len(names) == 17 and names == {"tsb200_" + fn for fn in BASE}
    for fn, args in BASE.items():
        assert len(args) == len(_lib.SIGNATURES["tsb200_" + fn][1]), fn
    assert {fn for fn, _, _ in TABLE} == set(BASE)


@pytest.mark.parametrize("i", range(len(TABLE)), ids=[_label(i, row) for i, row in enumerate(TABLE)])
def test_return_code(codes, i):
    fn, over, want = TABLE[i]
    got = codes[i]
    if want == CUDA:
        assert got > 0, f"tsb200_{fn}({over}): {got}, want a CUDA error (validation passed)"
    else:
        assert got == want, f"tsb200_{fn}({over}): {got}, want {want}"
