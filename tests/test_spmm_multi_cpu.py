"""Multi-aggregation SpMM without a GPU: the return codes of tsb200_spmm_fw_multi and its workspace size, the operator
schema, TorchScript and exports, the argument checks of `ops.spmm_fw_multi` / `spmm_multi`, and the backward of
SPMMMulti against fp64 autograd of the definition, with its CUDA calls restated in torch on CPU tensors.

The return-code table runs in a child interpreter that sees no CUDA device, as tests/test_rowsplit_abi_cpu.py does: a
call that passes validation fails at its first CUDA call with a positive CUDA error (`CUDA`). A short workspace tells the
vector path (which reports it, -3) from the generic kernel (which reads no workspace)."""
import ctypes
import importlib
import json
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import ops
from test_rowsplit_abi_cpu import (BF16, BIG, CUDA, E_MAX, F16, F32, F64, I32, INVALID, MIS, N_MAX, P, PLANNED,
                                   UNSUPPORTED, W, WORKSPACE, negatives, plan_faults, workspace_faults)

tsm = importlib.import_module("pytorch_sparse_b200.matmul")
FN = "spmm_fw_multi"
SUM, MEAN, MIN, MAX, VAR, STD = range(6)


def AG(*codes):
    return (ctypes.c_int * max(len(codes), 1))(*codes)


PNA = AG(MEAN, MIN, MAX, STD)
BASE = dict(rowptr=P, col=P, value=P, mat=P, aggrs=PNA, n=4, out=P, amin=P, amax=P, M=64, N=64, K=64, E=1000,
            dtype=BF16, plan=None, pb=0, ns=0, nl=0, nsl=0, ws=W, wsb=BIG, stream=None)

TABLE = [
    (FN, {}, CUDA), (FN, dict(PLANNED), CUDA), (FN, dict(amin=None, amax=None), CUDA),
    (FN, dict(dtype=F32, value=None), CUDA), (FN, dict(dtype=F16), CUDA),
    (FN, dict(aggrs=AG(SUM, MEAN, MIN, MAX, VAR, STD), n=6), CUDA), (FN, dict(aggrs=AG(VAR), n=1, amin=None,
                                                                              amax=None), CUDA),
    # the generic kernel: fp64, partial widths, E == 0; it reads no workspace and no plan
    (FN, dict(dtype=F64, wsb=1), CUDA), (FN, dict(PLANNED, dtype=F64, pb=1), CUDA),
    (FN, dict(K=12, wsb=1), CUDA), (FN, dict(dtype=F32, K=3, wsb=1), CUDA),
    (FN, dict(E=0, col=None, mat=None, ws=None), CUDA),
    *negatives(FN, "M", "N", "K", "E", "ns", "nl", "nsl"),
    # the aggregator list: empty, too long, out of range, repeated; an arg pointer without its aggregator
    (FN, dict(n=0), INVALID), (FN, dict(aggrs=AG(*range(6), 0), n=7), INVALID), (FN, dict(aggrs=None), INVALID),
    (FN, dict(aggrs=AG(MEAN, 6), n=2), INVALID), (FN, dict(aggrs=AG(-1), n=1), INVALID),
    (FN, dict(aggrs=AG(MEAN, MEAN), n=2), INVALID), (FN, dict(aggrs=AG(MIN, MAX, MIN), n=3), INVALID),
    (FN, dict(aggrs=AG(MEAN, MAX), n=2), INVALID), (FN, dict(aggrs=AG(MEAN, MIN), n=2), INVALID),
    (FN, dict(aggrs=AG(MEAN, MAX), n=2, amin=None), CUDA),
    (FN, dict(dtype=9), INVALID), (FN, dict(dtype=-1), INVALID), (FN, dict(dtype=I32), UNSUPPORTED),
    (FN, dict(M=0), 0), (FN, dict(K=0), 0), (FN, dict(M=0, out=None), 0),
    *[(FN, {n: None}, INVALID) for n in ("rowptr", "out", "col", "mat")],
    # alignments of the vector path; anything else runs the generic kernel
    (FN, dict(mat=P + 8, wsb=1), CUDA), (FN, dict(mat=P + 16, wsb=1), WORKSPACE),
    (FN, dict(out=P + 8, wsb=1), CUDA), (FN, dict(amin=P + 8, wsb=1), CUDA), (FN, dict(amax=P + 8, wsb=1), CUDA),
    (FN, dict(col=P + 4, wsb=1), CUDA), (FN, dict(col=P + 8, wsb=1), WORKSPACE),
    (FN, dict(value=P + 2, wsb=1), CUDA), (FN, dict(value=P + 4, wsb=1), WORKSPACE),
    *workspace_faults(FN),
    *plan_faults(FN, **PLANNED),
    (FN, dict(PLANNED, ws=MIS, wsb=1), WORKSPACE),
    (FN, dict(E=E_MAX, wsb=1), WORKSPACE), (FN, dict(E=E_MAX + 1, wsb=1), CUDA),
    (FN, dict(N=N_MAX, wsb=1), WORKSPACE), (FN, dict(N=N_MAX + 1, wsb=1), CUDA),
]


def _run():
    """In the child: refuse to call anything if a CUDA device is visible, else print every row's result as JSON."""
    assert torch.cuda.device_count() == 0, "a CUDA device is visible: no entry point is called"
    from pytorch_sparse_b200 import _lib
    codes = []
    for fn, over, _ in TABLE:
        args = dict(BASE)
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


def test_signature():
    from pytorch_sparse_b200 import _lib
    assert len(BASE) == len(_lib.SIGNATURES["tsb200_" + FN][1])
    header = (Path(__file__).resolve().parent.parent / "include" / "tsb200.h").read_text()
    assert "TSB200_API int tsb200_spmm_fw_multi(" in header
    assert "#define TSB200_VAR 4" in header and "#define TSB200_STD 5" in header


@pytest.mark.parametrize("i", range(len(TABLE)),
                         ids=[f"{i:03d}-" + ",".join(f"{k}={v if not isinstance(v, ctypes.Array) else list(v)}"
                                                     for k, v in o.items()) for i, (_, o, _) in enumerate(TABLE)])
def test_return_code(codes, i):
    fn, over, want = TABLE[i]
    got = codes[i]
    if want == CUDA:
        assert got > 0, f"tsb200_{fn}({over}): {got}, want a CUDA error (validation passed)"
    else:
        assert got == want, f"tsb200_{fn}({over}): {got}, want {want}"


# ---- workspace layout -------------------------------------------------------------------------------------------------
def _up(n):
    return (n + 255) // 256 * 256


def _layout(K, E, planned, n_long, n_slot):
    """The layout restated: counters, segments (32 B), long rows (24 B) or the planned completion counters, then
    4 fp32 partial columns and 2 int64 arg columns per column and slot."""
    if planned:
        slots = max(n_slot, 1)
        head = 256 + _up(max(n_long, 1) * 4)
    else:
        slots = E // 128 + 64
        head = 256 + _up((E // 32 + E // 128 + 64) * 32) + _up((E // 256 + 64) * 24)
    return head + _up(slots * 4 * K * 4) + _up(slots * 2 * K * 8)


@pytest.mark.parametrize("K,E", [(1, 1), (8, 1000), (64, 1000), (128, 1 << 20), (3, 777), (2048, 123457)])
def test_workspace_bytes(K, E):
    f = ts._lib.lib.tsb200_spmm_fw_multi_workspace_bytes
    assert f(K, E, 0, 0, 0) == _layout(K, E, False, 0, 0)
    for nl, ns in ((0, 0), (1, 2), (7, 40)):
        assert f(K, E, 1, nl, ns) == _layout(K, E, True, nl, ns)
    assert f(0, E, 0, 0, 0) == 0 and f(K, 0, 0, 0, 0) == 0 and f(-1, E, 0, 0, 0) == 0
    assert f(K, E, 1, -1, 0) == 0 and f(K, E, 1, 0, -1) == 0


# ---- Python surface ---------------------------------------------------------------------------------------------------
def test_schema_and_exports():
    schema = str(torch.ops.tsb200.spmm_multi.default._schema)
    assert "Tensor mat, Tensor? row_csc, str[] aggrs" in schema
    assert ts.spmm_multi is tsm.spmm_multi and "spmm_multi" in ts.__all__
    assert callable(ops.spmm_fw_multi) and ops.SPMMMulti is not None and ts.SparseTensor.spmm_multi is not None


def test_torchscript():
    def f(src: ts.SparseTensor, x: torch.Tensor) -> torch.Tensor:
        return tsm.spmm_multi(src, x, ["mean", "min", "max", "std"])

    g = torch.jit.script(f)
    assert "tsb200::spmm_multi" in str(g.inlined_graph)


def test_cpu_tensors_refused():
    with pytest.raises(RuntimeError, match="rowptr must be CUDA tensor"):
        ops.spmm_fw_multi(torch.zeros(3, dtype=torch.long), torch.zeros(0, dtype=torch.long), None, torch.ones(3, 4),
                          ["sum"])


@pytest.mark.parametrize("aggrs,msg", [
    ([], "aggrs must name at least one aggregator"),
    (["mean", "median"], "unknown aggregator 'median'"),
    (["softmax"], "unknown aggregator 'softmax'"),
    (["max", "max"], "aggregator 'max' is given more than once"),
    (["sum", "add"], "aggregator 'add' is given more than once"),
])
def test_aggregator_errors(aggrs, msg):
    with pytest.raises(ValueError, match=msg):
        ops._aggr_codes(aggrs)
    A = ts.SparseTensor(row=torch.tensor([0]), col=torch.tensor([0]), sparse_sizes=(1, 1))
    with pytest.raises((ValueError, RuntimeError), match=msg):
        tsm.spmm_multi(A, torch.ones(1, 4), aggrs)


def test_shape_errors(monkeypatch):
    A = ts.SparseTensor(row=torch.tensor([0, 1]), col=torch.tensor([0, 2]), sparse_sizes=(2, 3))
    with pytest.raises(RuntimeError, match="other must be 2-D \\[N, K\\], got 3-D"):
        tsm.spmm_multi(A, torch.ones(3, 2, 4), ["sum"])
    with pytest.raises(RuntimeError, match="other must have 3 rows \\(the sparse sizes\\), got 4"):
        tsm.spmm_multi(A, torch.ones(4, 4), ["sum"])
    monkeypatch.setattr(ops, "_check_cuda", lambda t, name: None)
    with pytest.raises(RuntimeError, match="the dense operand must be 2-D \\[N, K\\], got 1-D"):
        ops.spmm_fw_multi(torch.zeros(3, dtype=torch.long), torch.zeros(0, dtype=torch.long), None, torch.ones(3),
                          ["sum"])
    with pytest.raises(RuntimeError, match="expected value of dtype torch.float32 but got torch.float64"):
        ops.spmm_fw_multi(torch.zeros(3, dtype=torch.long), torch.zeros(1, dtype=torch.long),
                          torch.ones(1, dtype=torch.float64), torch.ones(3, 4), ["sum"])


# ---- the backward, on CPU tensors ------------------------------------------------------------------------------------
NAMES = ["sum", "mean", "min", "max", "var", "std"]


def definition(rowptr, col, value, x, aggrs):
    """out [M, A, K] by the definition, differentiable by torch: the messages of each row, their sum, mean, min / max
    (the smallest entry wins ties), var = max(Q / n - mu^2, 0) with its gradient 0 where the clamp is active, and
    std = sqrt(var) where var > 1e-5, else 0."""
    M, K = rowptr.numel() - 1, x.size(1)
    rows = []
    for m in range(M):
        s, e = int(rowptr[m]), int(rowptr[m + 1])
        p = x[col[s:e]] * (value[s:e, None] if value is not None else 1)
        n = max(e - s, 1)
        S = p.sum(0) if e > s else x.new_zeros(K)
        mu = S / n
        d = (p * p).sum(0) / n - mu * mu if e > s else x.new_zeros(K)
        var = torch.where(d > 0, d, torch.zeros_like(d))
        std = torch.where(var > 1e-5, var.clamp(min=1e-300).sqrt(), torch.zeros_like(var))
        stats = {"sum": S, "add": S, "mean": mu, "var": var, "std": std}
        if e > s:
            stats["min"] = torch.stack([p[int(p[:, k].detach().argmin()), k] for k in range(K)])
            stats["max"] = torch.stack([p[int(p[:, k].detach().argmax()), k] for k in range(K)])
        else:
            stats["min"] = stats["max"] = x.new_zeros(K)
        rows.append(torch.stack([stats[a] for a in aggrs]))
    return torch.stack(rows)


@pytest.fixture
def cpu_kernels(monkeypatch):
    """SPMMMulti's CUDA calls restated in fp64 torch on CPU tensors: the multi forward (with its args), the CSR sum
    SpMM (the CSC-view products), the SDDMM and the min / max backward."""
    monkeypatch.setattr(ops, "_check_cuda", lambda t, name: None)

    def fw_multi(rowptr, col, value, mat, codes, want_args, plan=None):
        out = definition(rowptr, col, value, mat, [NAMES[c] for c in codes])
        amin = amax = None
        if want_args:
            E = col.numel()
            M, K = rowptr.numel() - 1, mat.size(1)
            amin = torch.full((M, K), E, dtype=torch.long)
            amax = torch.full((M, K), E, dtype=torch.long)
            for m in range(M):
                s, e = int(rowptr[m]), int(rowptr[m + 1])
                if e > s:
                    p = mat[col[s:e]] * (value[s:e, None] if value is not None else 1)
                    amin[m] = s + p.argmin(0)
                    amax[m] = s + p.argmax(0)
        return out, amin, amax

    def spmm_sum(rowptr, col, value, mat, reduce, plan=None):
        assert reduce == "sum"
        M = rowptr.numel() - 1
        row = torch.repeat_interleave(torch.arange(M), rowptr[1:] - rowptr[:-1])
        w = value if value is not None else mat.new_ones(col.numel())
        return mat.new_zeros(M, mat.size(1)).index_add_(0, row, mat[col] * w[:, None]), None

    def sddmm(row, rowptr, col, mat, grad, reduce):
        return (grad[row] * mat[col]).sum(1)

    def minmax_bw(col, value, mat, g, arg, need_value, need_mat):
        E = col.numel()
        m, k = torch.nonzero(arg < E, as_tuple=True)
        e = arg[m, k]
        gv = mat.new_zeros(E).index_put_((e,), g[m, k] * mat[col[e], k], accumulate=True) if need_value else None
        w = value[e] if value is not None else 1
        gm = torch.zeros_like(mat).index_put_((col[e], k), g[m, k] * w, accumulate=True) if need_mat else None
        return gv, gm

    monkeypatch.setattr(ops, "_spmm_fw_multi", fw_multi)
    monkeypatch.setattr(ops, "spmm_fw", spmm_sum)
    monkeypatch.setattr(ops, "spmm_value_bw", sddmm)
    monkeypatch.setattr(ops, "spmm_minmax_bw", minmax_bw)


def _matrix(seed, with_value):
    g = torch.Generator().manual_seed(seed)
    M, N, K = 9, 7, 5
    deg = torch.tensor([0, 1, 3, 6, 2, 1, 0, 4, 5])
    rowptr = torch.cat([torch.zeros(1, dtype=torch.long), deg.cumsum(0)])
    E = int(rowptr[-1])
    col = torch.cat([torch.randperm(N, generator=g)[:int(d)] for d in deg])
    value = torch.randn(E, generator=g, dtype=torch.float64) if with_value else None
    x = torch.randn(N, K, generator=g, dtype=torch.float64)
    x[3] = 0.25           # a constant dense row: rows gathering only it have var 0
    return rowptr, col, value, x


@pytest.mark.parametrize("aggrs", [["mean", "min", "max", "std"], ["sum", "max"], ["var"], ["std"], ["var", "std"],
                                   ["add", "mean", "min", "max", "var", "std"], ["std", "sum", "min"]])
@pytest.mark.parametrize("with_value", [True, False])
def test_backward_matches_definition(cpu_kernels, aggrs, with_value):
    rowptr, col, value, x = _matrix(len(aggrs), with_value)
    M = rowptr.numel() - 1
    row = torch.repeat_interleave(torch.arange(M), rowptr[1:] - rowptr[:-1])
    perm = torch.argsort(col * M + row)
    colptr = torch.cat([torch.zeros(1, dtype=torch.long), torch.bincount(col, minlength=x.size(0)).cumsum(0)])
    x1 = x.clone().requires_grad_()
    v1 = value.clone().requires_grad_() if value is not None else None
    out = ops.SPMMMulti.apply(row, rowptr, col, v1, colptr, perm, x1, None, aggrs)
    x2 = x.clone().requires_grad_()
    v2 = value.clone().requires_grad_() if value is not None else None
    ref = definition(rowptr, col, v2, x2, aggrs)
    torch.testing.assert_close(out, ref.detach(), rtol=1e-12, atol=1e-12)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    got = torch.autograd.grad(out, [x1] + ([v1] if v1 is not None else []), g)
    want = torch.autograd.grad(ref, [x2] + ([v2] if v2 is not None else []), g)
    for a, b in zip(got, want):
        torch.testing.assert_close(a, b, rtol=1e-10, atol=1e-10)
