"""SpMM forward (16-bit / fp32 and FP8, with its e4m3 result and residual) and row-wise SDDMM at every work-item size.

The row kernels hand out work in items of 1 << item_shift consecutive rows; the host picks the size from the matrix
height and the occupancy, so a test matrix of a few thousand rows only ever runs one-row items and one of 600k rows
only 32-row items. TSB200_SPMM_ITEM_SHIFT (0..5, read on every call) sets the size, and this file runs every kernel
family at every size: multi-row items that do not start on a 32-row boundary (the plan mask read at r0 & 31), items
shorter than the lane groups of the group-per-row kernel, lane groups other than group 0 owning a row (the e4m3
per-group amax, the per-row output scale, residual row and residual scale at r0 + rl), the unplanned nnz budget of
a 2^s-row item, and the batch index of a multi-row item. The tests without the override check that it takes effect
(the main kernel's grid), that the automatic choice is one of the sizes tested here, and FP8 at 32-row items.

Checks are those of test_spmm_kernels_gpu, test_spmm_fp8_gpu, test_spmm_fp8_quant_gpu, test_spmm_fp8_residual_gpu
and test_spmm_backward_kernels_gpu: outputs prefilled with NaN (arg_out -1, e4m3 0x7f), sums within the rounding bound
of the fp64 oracle, min / max and arg_out bit for bit. One oracle or replay per operand serves all six sizes.

Planned and unplanned results are bit-identical, except in the group-per-row families for the rows that one side
defers for the 1024-nnz item budget and the other does not: the plan applies the budget to 32-row groups, an unplanned
call to its 2^s-row items. A deferred row is summed by the segment kernel's lane groups, in another order. The e4m3
result and the residual are defined on the float32 result of the same path at the same item size, so they are
bit-exact there, unplanned included.
"""
import json
import re

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import ops
from test_spmm_backward_kernels_gpu import ROWWISE, _operands, call_value_bw, check_value_bw
from test_spmm_fp8_gpu import KS, KS_PARTIAL, OUTS, Replay, call_fp8, make_scale, make_values, make_x8, mat  # noqa: F401
from test_spmm_fp8_quant_gpu import assert_q_equal, call_quant
from test_spmm_fp8_residual_gpu import E4M3, assert_out_equal, call_res, finish, make_residual, rho_of
from test_spmm_kernels_gpu import (DEV, FAMILIES, FLOATS, TABLE, Ref, _dev, _id, assert_bits_equal,  # noqa: F401
                                   assert_sum_bound, call_acc_blocks, call_fw, call_planned, dense, family_of, large,
                                   plan_budget_rows, small, sub_csr, values)

pytestmark = pytest.mark.gpu
ENV = "TSB200_SPMM_ITEM_SHIFT"
SHIFTS = range(6)
ACC_FAMILIES = ("gpr8", "vec32ch2")     # the P = 3 column-block accumulate: one group-per-row, one vector family


def budget_diff(rowptr_c, shift):
    """Rows deferred for the item budget by exactly one of a planned call (32-row groups) and an unplanned call with
    2^shift-row items."""
    return plan_budget_rows(rowptr_c) ^ plan_budget_rows(rowptr_c, 1 << shift)


def assert_same_path_result(out_p, out_u, arg_p, arg_u, gpr, rowptr_c, shift, what):
    """Planned against unplanned at one item size: bit for bit, except the budget rows of the group-per-row kernel's
    sums that only one side defers."""
    if arg_u is not None:
        assert_bits_equal(out_p, out_u, what + " planned vs unplanned")
        assert torch.equal(arg_p, arg_u), what + ": planned vs unplanned arg_out"
    elif gpr:
        keep = ~budget_diff(rowptr_c, shift).to(DEV)
        assert_bits_equal(out_p[keep], out_u[keep], what + " planned vs unplanned")
    else:
        assert_bits_equal(out_p, out_u, what + " planned vs unplanned")


def test_budget_rows_differ_by_item_size(small):
    """The structured matrix's budget block (32 rows of 48 nnz) is deferred in part by 32-row items only: the
    exclusion above is empty at shift 5 and not empty below it."""
    rowptr_c = small["rowptr"]
    assert not bool(budget_diff(rowptr_c, 5).any())
    for s in range(5):
        assert bool(budget_diff(rowptr_c, s).any()), s


# ---- 1. 16-bit / fp32 forward: every family, every item size ---------------------------------------------------------
@pytest.mark.parametrize("has_value", [True, False], ids=["value", "novalue"])
@pytest.mark.parametrize("dtype,K", TABLE, ids=_id)
def test_family_every_item_size(oracle, small, monkeypatch, dtype, K, has_value):
    rowptr_c, col_c = small["rowptr"], small["col"]
    E, N = col_c.numel(), small["N"]
    fam = family_of(dtype, K)
    rowptr, col = _dev(rowptr_c, col_c)
    plan = ops.spmm_plan(rowptr, E)
    for quantized, reduces in ((False, ("sum", "mean")), (True, ("min", "max"))):
        mat_c = dense(N, K, dtype, K, quantized)
        val_c = values(E, dtype, K + 1, quantized) if has_value else None
        mat, val = _dev(mat_c, val_c)
        ref = Ref(oracle, rowptr_c, col_c, val_c, mat_c)
        for s in SHIFTS:
            monkeypatch.setenv(ENV, str(s))
            what = f"{fam} {dtype} K={K} value={has_value} shift={s}"
            for reduce in reduces:
                out_u, arg_u = call_fw(rowptr, col, val, mat, reduce)
                ref.check(reduce, out_u, arg_u, what + " unplanned")
                out_p, arg_p = call_planned(plan, rowptr, col, val, mat, reduce)
                ref.check(reduce, out_p, arg_p, what + " planned")
                assert_same_path_result(out_p, out_u, arg_p, arg_u, fam.startswith("gpr"), rowptr_c, s,
                                        f"{what} {reduce}")
            if has_value and not quantized and fam in ACC_FAMILIES:
                out_a = call_acc_blocks(rowptr, col, val, mat, 3)
                assert_sum_bound(out_a, ref.sum64(), ref.S(), ref.deg + 3, dtype, what=f"{what} acc P=3")


@pytest.mark.parametrize("fam", [f for f in FAMILIES if f != "tiled"])
def test_family_batched_every_item_size(oracle, small, monkeypatch, fam):
    """B = 3, a different dense operand per batch (unplanned): item index / blocks per batch over multi-row items."""
    rowptr_c, col_c = small["rowptr"], small["col"]
    E, N = col_c.numel(), small["N"]
    rowptr, col = _dev(rowptr_c, col_c)
    for dtype in FLOATS:
        K = FAMILIES[fam][0 if dtype == torch.float32 else 1][-1]
        for quantized, reduces in ((False, ("sum", "mean")), (True, ("min", "max"))):
            mat_c = dense(N, K, dtype, 40 + K, quantized, B=3)
            val_c = values(E, dtype, 41, quantized)
            mat, val = _dev(mat_c, val_c)
            ref = Ref(oracle, rowptr_c, col_c, val_c, mat_c)
            for s in SHIFTS:
                monkeypatch.setenv(ENV, str(s))
                for reduce in reduces:
                    out, arg = call_fw(rowptr, col, val, mat, reduce)
                    ref.check(reduce, out, arg, f"{fam} {dtype} K={K} B=3 shift={s}")


# ---- 2. FP8 forward, e4m3 result and residual: every shape, every item size -------------------------------------------
class CachedReplay(Replay):
    """Replay with the min/max replay kept per (reduction, output dtype): one replay serves every item size."""

    def __init__(self, *args):
        super().__init__(*args)
        self._mm = {}

    def minmax(self, reduce, out_dtype):
        if (reduce, out_dtype) not in self._mm:
            self._mm[reduce, out_dtype] = super().minmax(reduce, out_dtype)
        return self._mm[reduce, out_dtype]


def check_quant(y, arg_y, rowptr, col, v, x8, sc, reduce, plan, what):
    """tsb200_spmm_fw_fp8_quant against CPU quantize_fp8 of the float32 result y of the same path and item size."""
    ref8, refs = ts.quantize_fp8(y.cpu(), per_row=True)
    y8, ys, arg = call_quant(rowptr, col, v, x8, sc, reduce, plan=plan)
    assert_q_equal(y8, ys, ref8, refs, what + " e4m3 result")
    if arg is not None:
        assert torch.equal(arg, arg_y), what + ": e4m3 result arg_out differs"


# (per-row scales, entry values): per-row scales with values, a per-tensor scale without
FP8_CASES = [(True, True), (False, False)]


@pytest.mark.parametrize("per_row,has_value", FP8_CASES, ids=["rowscale-value", "tensorscale-novalue"])
@pytest.mark.parametrize("K", KS + KS_PARTIAL)
def test_fp8_every_item_size(mat, monkeypatch, K, per_row, has_value):
    rowptr_c, col_c, M, N = mat["rowptr"], mat["col"], mat["M"], mat["N"]
    E = col_c.numel()
    rowptr, col = _dev(rowptr_c, col_c)
    plan = ops.spmm_plan(rowptr, E)
    gpr = K <= 128          # 16-byte vectors of 16 e4m3 values: up to 8 per dense row run the group-per-row kernel
    q8 = K <= 2048          # an e4m3 result is one column tile wide
    for ties, reduces in ((False, ("sum", "mean")), (True, ("min", "max"))):
        x8_c = make_x8(N, K, K + ties, ties)
        sc_c = make_scale(N, K + 2, per_row)
        v_c = make_values(E, K + 3, ties) if has_value else None
        rep = CachedReplay(rowptr_c, col_c, v_c, x8_c, sc_c)
        x8, sc, v = _dev(x8_c, sc_c, v_c)
        if not ties:
            r8_c, rsc_c = make_residual(M, K, K + 4, per_row)
            rho = rho_of(r8_c, rsc_c)
            r8, rsc = _dev(r8_c, rsc_c)
        for s in SHIFTS:
            monkeypatch.setenv(ENV, str(s))
            for reduce in reduces:
                got = {}
                for plan_, path in ((None, "unplanned"), (plan, "planned")):
                    what = f"K={K} per_row={per_row} value={has_value} shift={s} {path}"
                    for out_dtype in OUTS:
                        vo = None if v is None else v.to(out_dtype)
                        out, arg = call_fp8(rowptr, col, vo, x8, sc, reduce, out_dtype, plan=plan_)
                        rep.check(reduce, out, arg, out_dtype, f"{what} {_id(out_dtype)}")
                        got[path, out_dtype] = out, arg
                    y, arg_y = got[path, torch.float32]
                    if q8:
                        check_quant(y, arg_y, rowptr, col, v, x8, sc, reduce, plan_, f"{what} {reduce}")
                    if not ties:
                        for out_dtype in (torch.float32, E4M3) if q8 else (torch.float32,):
                            out, ys, _ = call_res(rowptr, col, v, x8, sc, r8, rsc, reduce, out_dtype, plan=plan_)
                            assert_out_equal(out, ys, finish(y.cpu() + rho, out_dtype),
                                             f"{what} {reduce} residual {_id(out_dtype)}")
                for out_dtype in OUTS:
                    (out_u, arg_u), (out_p, arg_p) = got["unplanned", out_dtype], got["planned", out_dtype]
                    assert_same_path_result(out_p, out_u, arg_p, arg_u, gpr, rowptr_c, s,
                                            f"K={K} per_row={per_row} shift={s} {reduce} {_id(out_dtype)}")


# ---- 3. row-wise SDDMM: every family, every item size ------------------------------------------------------------------
@pytest.mark.parametrize("dtype,K,B", ROWWISE, ids=_id)
def test_sddmm_every_item_size(oracle, small, monkeypatch, dtype, K, B):
    rowptr_c, col_c, N, M = small["rowptr"], small["col"], small["N"], small["M"]
    mat_c, grad_c = _operands(N, M, K, B, dtype, K + B)
    row = torch.repeat_interleave(torch.arange(M), rowptr_c[1:] - rowptr_c[:-1])
    args = _dev(row, rowptr_c, col_c, mat_c, grad_c)
    for s in SHIFTS:
        monkeypatch.setenv(ENV, str(s))
        for reduce in ("sum", "mean"):
            out = call_value_bw(*args, reduce)
            check_value_bw(oracle, rowptr_c, col_c, mat_c, grad_c, reduce, out,
                           f"value_bw {dtype} K={K} shift={s} {reduce}")


# ---- 4. the override takes effect ---------------------------------------------------------------------------------------
def kernel_grids(fn, pattern, tmp_path):
    """The grids of the kernels whose names match `pattern` that `fn` launches, from a profiler trace (`args.grid` of
    the kernel events). Repeated when the profiler drops the record, as in util.launched_kernels."""
    for attempt in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        path = tmp_path / f"trace{attempt}.json"
        prof.export_chrome_trace(str(path))
        events = [e for e in json.loads(path.read_text())["traceEvents"]
                  if e.get("cat") == "kernel" and re.search(pattern, e.get("name", ""))]
        if events:
            assert all("grid" in e.get("args", {}) for e in events), events[0]
            return [tuple(e["args"]["grid"]) for e in events]
    raise AssertionError(f"the profiler recorded no kernel matching {pattern}")


def _cdiv(a, b):
    return -(-a // b)


def test_override_sets_item_size(small, monkeypatch, tmp_path):
    """The unplanned main kernel of a vector family runs ceil(ceil(M / 2^s) / 8) CTAs of 8 warps, one item per warp:
    71, 36, 18 and 9 for M = 2253 at shifts 2 ... 5, fewer than any persistent grid on the device."""
    rowptr, col = _dev(small["rowptr"], small["col"])
    M, N = small["M"], small["N"]
    mat = dense(N, 128, torch.bfloat16, 0, False).to(DEV)
    assert family_of(torch.bfloat16, 128) == "vec16"
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    for s in range(2, 6):
        monkeypatch.setenv(ENV, str(s))
        want = _cdiv(_cdiv(M, 1 << s), 8)
        assert want < sms
        grids = kernel_grids(lambda: call_fw(rowptr, col, None, mat, "sum"), r"spmm_vec_kernel<", tmp_path)
        assert grids == [(want, 1, 1)], (s, grids)
    assert [_cdiv(_cdiv(M, 1 << s), 8) for s in range(2, 6)] == [71, 36, 18, 9]


# ---- 5. the automatic choice is what was tested -----------------------------------------------------------------------
def _auto_vs(monkeypatch, shift, fn):
    """fn() without the override and at `shift`."""
    monkeypatch.delenv(ENV, raising=False)
    a = fn()
    monkeypatch.setenv(ENV, str(shift))
    b = fn()
    monkeypatch.delenv(ENV, raising=False)
    return a, b


def assert_results_equal(a, b, what):
    assert_bits_equal(a[0], b[0], what)
    if a[1] is not None:
        assert torch.equal(a[1], b[1]), what + ": arg_out differs"


# one group-per-row and one vector family: 16-bit (dtype, K) and e4m3 K
AUTO_16 = [(torch.bfloat16, 16), (torch.bfloat16, 128)]
AUTO_FP8 = (64, 256)


@pytest.mark.parametrize("which,shift", [("small", 0), ("large", 5)])
def test_automatic_item_size(request, monkeypatch, which, shift):
    """Without the override, small matrices run one-row items and ~600k-row ones 32-row items (for any occupancy of
    at most 8 CTAs per SM): bit-identical to the result at that shift, planned and unplanned."""
    m = request.getfixturevalue(which)
    rowptr_c, col_c, N = m["rowptr"], m["col"], m["N"]
    E = col_c.numel()
    rowptr, col = _dev(rowptr_c, col_c)
    plan = ops.spmm_plan(rowptr, E)
    assert {family_of(dt, K)[:3] for dt, K in AUTO_16} == {"gpr", "vec"}
    for dtype, K in AUTO_16:
        for quantized, reduce in ((False, "sum"), (True, "max")):
            mat, val = _dev(dense(N, K, dtype, 5, quantized), values(E, dtype, 6, quantized))
            for p in (None, plan):
                fn = (lambda: call_fw(rowptr, col, val, mat, reduce)) if p is None else \
                     (lambda: call_planned(plan, rowptr, col, val, mat, reduce))
                a, b = _auto_vs(monkeypatch, shift, fn)
                assert_results_equal(a, b, f"{which} {dtype} K={K} {reduce} planned={p is not None} auto vs {shift}")
    for K in AUTO_FP8:
        for ties, reduce, out_dtype in ((False, "sum", torch.float32), (True, "max", torch.bfloat16)):
            x8, sc = _dev(make_x8(N, K, 9, ties), make_scale(N, 10, True))
            v = make_values(E, 11, ties).to(out_dtype).to(DEV)
            for p in (None, plan):
                a, b = _auto_vs(monkeypatch, shift, lambda: call_fp8(rowptr, col, v, x8, sc, reduce, out_dtype, plan=p))
                assert_results_equal(a, b, f"{which} fp8 K={K} {reduce} planned={p is not None} auto vs {shift}")


def sample_arg(arg_rows, idx, E):
    """arg_out of the sampled rows (global nnz numbers, E for none) in the sample's own nnz numbering."""
    a = arg_rows.cpu()
    glob = torch.cat([idx, torch.tensor([E])])
    s = torch.searchsorted(glob, a)
    s = torch.where(glob[s.clamp(max=idx.numel())] == a, s, -1)
    return torch.where(a == E, idx.numel(), s)


@pytest.mark.parametrize("K", (16, 128, 256, 512))
def test_fp8_full_size_items(large, monkeypatch, K):
    """FP8 forward with 32-row items (no override): every element written, a sample of whole 32-row groups against
    the replay, and bit-identical to the result at shift 5, planned and unplanned. Min / max only up to K = 256, so
    that no output (arg_out included) exceeds 1.2 GB."""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    assert large["M"] >= 32 * 16 * 8 * sms
    rowptr_c, col_c, rows, N = large["rowptr"], large["col"], large["rows"], large["N"]
    E = col_c.numel()
    rowptr, col = _dev(rowptr_c, col_c)
    plan = ops.spmm_plan(rowptr, E)
    sp, scol, idx = sub_csr(rowptr_c, col_c, rows)
    rows_d = rows.to(DEV)
    cases = [(False, "sum", torch.float32), (False, "mean", torch.bfloat16)]
    if K <= 256:
        cases += [(True, "max", torch.float16), (True, "min", torch.bfloat16)]
    for ties, reduce, out_dtype in cases:
        x8_c, sc_c = make_x8(N, K, 12 + ties, ties), make_scale(N, 13, True)
        v_c = make_values(E, 14, ties)
        x8, sc, v = _dev(x8_c, sc_c, v_c.to(out_dtype))
        rep = Replay(sp, scol, v_c[idx].to(out_dtype), x8_c, sc_c)
        for p in (None, plan):
            what = f"fp8 K={K} {reduce} {_id(out_dtype)} M={large['M']} planned={p is not None}"
            a, b = _auto_vs(monkeypatch, 5, lambda: call_fp8(rowptr, col, v, x8, sc, reduce, out_dtype, plan=p))
            assert_results_equal(a, b, what + " auto vs 5")
            del b
            out, arg = a
            if arg is None:
                assert not bool(out.isnan().any()), what + ": output element not written"
            else:
                assert bool((arg >= 0).all()), what + ": arg_out element not written"
            rep.check(reduce, out[rows_d], None if arg is None else sample_arg(arg[rows_d], idx, E), out_dtype, what)
            del a, out, arg
