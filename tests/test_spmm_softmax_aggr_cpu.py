"""Softmax-aggregation SpMM without a GPU: the return codes of tsb200_spmm_fw_softmax_aggr and its two backward entry
points, the forward's workspace size, the operator schema, TorchScript and exports, the argument checks of
`ops.spmm_fw_softmax_aggr` / `spmm_softmax_aggr`, and SPMMSoftmaxAggr's wiring against fp64 autograd of the
definition, with its CUDA calls restated in torch on CPU tensors.

The return-code table runs in a child interpreter that sees no CUDA device, as tests/test_rowsplit_abi_cpu.py does: a
call that passes validation fails at its first CUDA call with a positive CUDA error (`CUDA`). A short workspace tells the
forward's vector path (which reports it, -3) from its generic kernel (which reads no workspace)."""
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
FW, ROWS, COLS = "spmm_fw_softmax_aggr", "spmm_softmax_aggr_bw_rows", "spmm_softmax_aggr_bw_cols"
BASES = {
    FW: dict(rowptr=P, col=P, value=P, mat=P, t=P, ts=1, out=P, lse=P, M=64, N=64, K=64, E=1000, dtype=BF16,
             plan=None, pb=0, ns=0, nl=0, nsl=0, ws=W, wsb=BIG, stream=None),
    ROWS: dict(rowptr=P, col=P, value=P, mat=P, t=P, ts=1, g=P, out=P, lse=P, gv=P, U=P, M=64, N=64, K=64, E=1000,
               dtype=BF16, ws=W, wsb=BIG, stream=None),
    COLS: dict(colptr=P, row_csc=P, value=P, mat=P, t=P, ts=1, g=P, out=P, lse=P, gm=P, M=64, N=64, K=64, E=1000,
               dtype=BF16, ws=W, wsb=BIG, stream=None),
}

TABLE = [
    (FW, {}, CUDA), (FW, dict(PLANNED), CUDA), (FW, dict(lse=None), CUDA), (FW, dict(ts=0), CUDA),
    (FW, dict(dtype=F32, value=None), CUDA), (FW, dict(dtype=F16), CUDA),
    # the generic kernel: fp64, partial widths, E == 0; it reads no workspace and no plan
    (FW, dict(dtype=F64, wsb=1), CUDA), (FW, dict(PLANNED, dtype=F64, pb=1), CUDA),
    (FW, dict(K=12, wsb=1), CUDA), (FW, dict(dtype=F32, K=3, wsb=1), CUDA),
    (FW, dict(E=0, col=None, mat=None, ws=None), CUDA),
    *negatives(FW, "M", "N", "K", "E", "ns", "nl", "nsl"),
    (FW, dict(ts=2), INVALID), (FW, dict(ts=-1), INVALID),
    (FW, dict(dtype=9), INVALID), (FW, dict(dtype=-1), INVALID), (FW, dict(dtype=I32), UNSUPPORTED),
    (FW, dict(t=P + 2), UNSUPPORTED), (FW, dict(dtype=F64, t=P + 4, wsb=1), UNSUPPORTED),
    (FW, dict(M=0), 0), (FW, dict(K=0), 0), (FW, dict(M=0, out=None, t=None), 0),
    *[(FW, {n: None}, INVALID) for n in ("rowptr", "out", "col", "mat", "t")],
    # alignments of the vector path; anything else runs the generic kernel
    (FW, dict(mat=P + 8, wsb=1), CUDA), (FW, dict(mat=P + 16, wsb=1), WORKSPACE),
    (FW, dict(out=P + 8, wsb=1), CUDA), (FW, dict(lse=P + 8, wsb=1), CUDA), (FW, dict(lse=P + 16, wsb=1), WORKSPACE),
    (FW, dict(col=P + 4, wsb=1), CUDA), (FW, dict(value=P + 2, wsb=1), CUDA), (FW, dict(value=P + 4, wsb=1), WORKSPACE),
    *workspace_faults(FW),
    *plan_faults(FW, **PLANNED),
    (FW, dict(PLANNED, ws=MIS, wsb=1), WORKSPACE),
    (FW, dict(E=E_MAX, wsb=1), WORKSPACE), (FW, dict(E=E_MAX + 1, wsb=1), CUDA),
    (FW, dict(N=N_MAX, wsb=1), WORKSPACE), (FW, dict(N=N_MAX + 1, wsb=1), CUDA),
    # the row-wise backward: either output may be NULL, grad_value needs the values
    (ROWS, {}, CUDA), (ROWS, dict(gv=None), CUDA), (ROWS, dict(U=None), CUDA), (ROWS, dict(gv=None, U=None), 0),
    (ROWS, dict(value=None, gv=None), CUDA), (ROWS, dict(value=None), INVALID), (ROWS, dict(dtype=F64), CUDA),
    (ROWS, dict(ts=0, dtype=F32, K=3), CUDA), (ROWS, dict(E=0, col=None, mat=None), CUDA),
    *negatives(ROWS, "M", "N", "K", "E"), (ROWS, dict(ts=2), INVALID), (ROWS, dict(dtype=I32), UNSUPPORTED),
    (ROWS, dict(dtype=9), INVALID), (ROWS, dict(t=P + 2), UNSUPPORTED), (ROWS, dict(M=0), 0),
    *[(ROWS, {n: None}, INVALID) for n in ("rowptr", "col", "mat", "t", "g", "out", "lse")],
    # the row-split path of the backward reads its workspace; the generic kernel (fp64, partial or > 1024-byte rows,
    # unaligned operands, E == 0) reads none
    *workspace_faults(ROWS), *workspace_faults(COLS),
    (ROWS, dict(dtype=F64, wsb=1), CUDA), (ROWS, dict(K=12, wsb=1), CUDA), (ROWS, dict(K=520, wsb=1), CUDA),
    (ROWS, dict(K=512, wsb=1), WORKSPACE), (ROWS, dict(mat=P + 8, wsb=1), CUDA), (ROWS, dict(lse=P + 8, wsb=1), CUDA),
    (ROWS, dict(g=P + 8, wsb=1), CUDA), (ROWS, dict(out=P + 8, wsb=1), CUDA), (ROWS, dict(gv=P + 2, wsb=1), WORKSPACE),
    (COLS, dict(dtype=F64, wsb=1), CUDA), (COLS, dict(dtype=F32, K=3, wsb=1), CUDA), (COLS, dict(gm=P + 8, wsb=1), CUDA),
    (COLS, dict(lse=P + 8, wsb=1), CUDA), (COLS, dict(value=P + 2, wsb=1), CUDA), (COLS, dict(dtype=F32, K=256, wsb=1),
                                                                                   WORKSPACE),
    (COLS, dict(E=E_MAX + 1, wsb=1), CUDA), (COLS, dict(M=N_MAX + 1, wsb=1), CUDA), (COLS, dict(M=N_MAX, wsb=1), WORKSPACE),
    # the column-wise backward: nothing is launched without grad_mat
    (COLS, {}, CUDA), (COLS, dict(value=None), CUDA), (COLS, dict(dtype=F64), CUDA), (COLS, dict(gm=None), 0),
    (COLS, dict(E=0, row_csc=None, g=None, out=None, lse=None), CUDA), (COLS, dict(N=0), 0), (COLS, dict(K=0), 0),
    *negatives(COLS, "M", "N", "K", "E"), (COLS, dict(ts=3), INVALID), (COLS, dict(dtype=I32), UNSUPPORTED),
    (COLS, dict(dtype=F64, t=P + 4), UNSUPPORTED),
    *[(COLS, {n: None}, INVALID) for n in ("colptr", "row_csc", "mat", "t", "g", "out", "lse")],
]


def _run():
    """In the child: refuse to call anything if a CUDA device is visible, else print every row's result as JSON."""
    assert torch.cuda.device_count() == 0, "a CUDA device is visible: no entry point is called"
    from pytorch_sparse_b200 import _lib
    codes = []
    for fn, over, _ in TABLE:
        args = dict(BASES[fn])
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


def test_signatures():
    from pytorch_sparse_b200 import _lib
    header = (Path(__file__).resolve().parent.parent / "include" / "tsb200.h").read_text()
    for fn, base in BASES.items():
        assert len(base) == len(_lib.SIGNATURES["tsb200_" + fn][1]), fn
        assert f"TSB200_API int tsb200_{fn}(" in header
    assert "TSB200_API size_t tsb200_spmm_fw_softmax_aggr_workspace_bytes(" in header


@pytest.mark.parametrize("i", range(len(TABLE)),
                         ids=[f"{i:03d}-{fn[-4:]}-" + ",".join(f"{k}={v}" for k, v in o.items())
                              for i, (fn, o, _) in enumerate(TABLE)])
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
    """The layout restated: counters, segments (32 B), long rows (24 B) or the planned completion counters, then 3 fp32
    partial columns (mu, s, a) per column and slot."""
    if planned:
        slots = max(n_slot, 1)
        head = 256 + _up(max(n_long, 1) * 4)
    else:
        slots = E // 128 + 64
        head = 256 + _up((E // 32 + E // 128 + 64) * 32) + _up((E // 256 + 64) * 24)
    return head + _up(slots * 3 * K * 4)


@pytest.mark.parametrize("K,E", [(1, 1), (8, 1000), (64, 1000), (128, 1 << 20), (3, 777), (2048, 123457)])
def test_workspace_bytes(K, E):
    f = ts._lib.lib.tsb200_spmm_fw_softmax_aggr_workspace_bytes
    assert f(K, E, 0, 0, 0) == _layout(K, E, False, 0, 0)
    for nl, ns in ((0, 0), (1, 2), (7, 40)):
        assert f(K, E, 1, nl, ns) == _layout(K, E, True, nl, ns)
    assert f(0, E, 0, 0, 0) == 0 and f(K, 0, 0, 0, 0) == 0 and f(-1, E, 0, 0, 0) == 0
    assert f(K, E, 1, -1, 0) == 0 and f(K, E, 1, 0, -1) == 0


@pytest.mark.parametrize("K,E", [(1, 1), (64, 1000), (3, 777), (512, 123457)])
def test_backward_workspace_bytes(K, E):
    """The backward's workspace: the unplanned forward layout over K fp32 partial columns per slot."""
    f = ts._lib.lib.tsb200_spmm_softmax_aggr_bw_workspace_bytes
    head = 256 + _up((E // 32 + E // 128 + 64) * 32) + _up((E // 256 + 64) * 24)
    assert f(K, E) == head + _up((E // 128 + 64) * K * 4)
    assert f(0, E) == 0 and f(K, 0) == 0 and f(-1, E) == 0


# ---- Python surface ---------------------------------------------------------------------------------------------------
def test_schema_and_exports():
    schema = str(torch.ops.tsb200.spmm_softmax_aggr.default._schema)
    assert "Tensor mat, Tensor? row_csc, Tensor? t) -> Tensor" in schema
    assert ts.spmm_softmax_aggr is tsm.spmm_softmax_aggr and "spmm_softmax_aggr" in ts.__all__
    assert ops.SPMMSoftmaxAggr is not None and ts.SparseTensor.spmm_softmax_aggr is not None


def test_torchscript():
    def f(src: ts.SparseTensor, x: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
        return tsm.spmm_softmax_aggr(src, x, t) + tsm.spmm_softmax_aggr(src, x)

    g = torch.jit.script(f)
    assert "tsb200::spmm_softmax_aggr" in str(g.inlined_graph)


def test_cpu_tensors_refused():
    with pytest.raises(RuntimeError, match="rowptr must be CUDA tensor"):
        ops.spmm_fw_softmax_aggr(torch.zeros(3, dtype=torch.long), torch.zeros(0, dtype=torch.long), None,
                                 torch.ones(3, 4), torch.ones(()))


def test_argument_errors(monkeypatch):
    A = ts.SparseTensor(row=torch.tensor([0, 1]), col=torch.tensor([0, 2]), sparse_sizes=(2, 3))
    with pytest.raises(RuntimeError, match="other must be 2-D \\[N, K\\], got 3-D"):
        tsm.spmm_softmax_aggr(A, torch.ones(3, 2, 4))
    with pytest.raises(RuntimeError, match="other must have 3 rows \\(the sparse sizes\\), got 4"):
        tsm.spmm_softmax_aggr(A, torch.ones(4, 4))
    monkeypatch.setattr(ops, "_check_cuda", lambda t, name: None)
    rp, c1 = torch.zeros(3, dtype=torch.long), torch.zeros(1, dtype=torch.long)
    with pytest.raises(RuntimeError, match="the dense operand must be 2-D \\[N, K\\], got 1-D"):
        ops.spmm_fw_softmax_aggr(rp, c1, None, torch.ones(3), torch.ones(()))
    with pytest.raises(RuntimeError, match="expected value of dtype torch.float32 but got torch.float64"):
        ops.spmm_fw_softmax_aggr(rp, c1, torch.ones(1, dtype=torch.float64), torch.ones(3, 4), torch.ones(()))
    for t in (torch.ones(3), torch.ones(2, 4), torch.ones(5)):
        with pytest.raises(RuntimeError, match="t must have shape \\[\\], \\[1\\] or \\[K\\] = \\[4\\]"):
            ops.spmm_fw_softmax_aggr(rp, c1, None, torch.ones(3, 4), t)
    with pytest.raises(RuntimeError, match="t must be torch.float32 for a torch.bfloat16 operand"):
        ops.spmm_fw_softmax_aggr(rp, c1, None, torch.ones(3, 4, dtype=torch.bfloat16), torch.ones((), dtype=torch.bfloat16))
    with pytest.raises(RuntimeError, match="t must be torch.float64 for a torch.float64 operand"):
        ops.spmm_fw_softmax_aggr(rp, c1, None, torch.ones(3, 4, dtype=torch.float64), torch.ones(4))


# ---- the autograd Function, on CPU tensors ----------------------------------------------------------------------------
def definition(rowptr, col, value, x, t):
    """(out, lse) [M, K] by the definition, differentiable by torch: per row, the messages p = v x[col], their softmax
    over the row's entries of t p per column, and the weighted sum; an empty row gives 0 and lse -inf."""
    M, K = rowptr.numel() - 1, x.size(1)
    outs, lses = [], []
    for m in range(M):
        s, e = int(rowptr[m]), int(rowptr[m + 1])
        if e == s:
            outs.append(x.new_zeros(K))
            lses.append(x.new_full((K,), float("-inf")))
            continue
        p = x[col[s:e]] * (value[s:e, None] if value is not None else 1)
        y = t * p
        outs.append((torch.softmax(y, 0) * p).sum(0))
        lses.append(torch.logsumexp(y, 0))
    return torch.stack(outs), torch.stack(lses)


def _messages(ptr, idx, value, mat, t, out, lse, other):
    """p, alpha and d of every entry of a CSR (other = col) or CSC (other = the row of each entry) walk."""
    n = ptr.numel() - 1
    own = torch.repeat_interleave(torch.arange(n), ptr[1:] - ptr[:-1])
    r, c = (own, idx) if other == "col" else (idx, own)
    p = mat[c] * (value[:, None] if value is not None else 1)
    alpha = torch.exp(t * p - lse[r])
    return r, c, p, alpha


@pytest.fixture
def cpu_kernels(monkeypatch):
    """SPMMSoftmaxAggr's CUDA calls restated in fp64 torch on CPU tensors: the forward by the definition, and the two
    backward kernels by their formulas. Records which kernels ran."""
    monkeypatch.setattr(ops, "_check_cuda", lambda t, name: None)
    calls = []

    def fw(rowptr, col, value, mat, t, want_lse=False, plan=None):
        calls.append("fw" + ("+lse" if want_lse else ""))
        with torch.no_grad():
            out, lse = definition(rowptr, col, value, mat, t)
        return out, lse if want_lse else None

    def bw_rows(rowptr, col, value, mat, t, grad_out, out, lse, want_value, want_t):
        calls.append("rows")
        r, c, p, alpha = _messages(rowptr, col, value, mat, t, out, lse, "col")
        d = grad_out[r] * alpha * (1 + t * (p - out[r]))
        gv = (mat[c] * d).sum(1) if want_value and value is not None else None
        U = (torch.zeros_like(out).index_add_(0, r, alpha * (p - out[r]) ** 2) * grad_out) if want_t else None
        return gv, U

    def bw_cols(colptr, row_csc, value_csc, mat, t, grad_out, out, lse):
        calls.append("cols")
        r, c, p, alpha = _messages(colptr, row_csc, value_csc, mat, t, out, lse, "row")
        d = grad_out[r] * alpha * (1 + t * (p - out[r]))
        return torch.zeros_like(mat).index_add_(0, c, d * (value_csc[:, None] if value_csc is not None else 1))

    monkeypatch.setattr(ops, "spmm_fw_softmax_aggr", fw)
    monkeypatch.setattr(ops, "spmm_softmax_aggr_bw_rows", bw_rows)
    monkeypatch.setattr(ops, "spmm_softmax_aggr_bw_cols", bw_cols)
    return calls


def _matrix(seed, with_value):
    g = torch.Generator().manual_seed(seed)
    M, N, K = 9, 7, 5
    deg = torch.tensor([0, 1, 3, 6, 2, 1, 0, 4, 5])
    rowptr = torch.cat([torch.zeros(1, dtype=torch.long), deg.cumsum(0)])
    E = int(rowptr[-1])
    col = torch.cat([torch.randperm(N, generator=g)[:int(d)] for d in deg])
    col[4] = col[5] = 2   # a duplicate entry: both count
    value = torch.randn(E, generator=g, dtype=torch.float64) if with_value else None
    x = torch.randn(N, K, generator=g, dtype=torch.float64)
    return rowptr, col, value, x


@pytest.mark.parametrize("t_kind", ["scalar", "one", "channel", "negative"])
@pytest.mark.parametrize("wrt", [("x",), ("v",), ("t",), ("x", "v", "t"), ("v", "t")])
@pytest.mark.parametrize("with_value", [True, False])
def test_backward_matches_definition(cpu_kernels, t_kind, wrt, with_value):
    if "v" in wrt and not with_value:
        pytest.skip("no values to differentiate")
    rowptr, col, value, x = _matrix(3, with_value)
    M, N, K = rowptr.numel() - 1, x.size(0), x.size(1)
    t0 = {"scalar": torch.tensor(0.7, dtype=torch.float64), "one": torch.tensor([1.3], dtype=torch.float64),
          "channel": torch.linspace(-1, 2, K, dtype=torch.float64),
          "negative": torch.tensor(-2.0, dtype=torch.float64)}[t_kind]
    row = torch.repeat_interleave(torch.arange(M), rowptr[1:] - rowptr[:-1])
    perm = torch.argsort(col * M + row)
    colptr = torch.cat([torch.zeros(1, dtype=torch.long), torch.bincount(col, minlength=N).cumsum(0)])
    leaves1 = dict(x=x.clone(), v=value.clone() if value is not None else None, t=t0.clone())
    leaves2 = {k: (v.clone() if v is not None else None) for k, v in leaves1.items()}
    for k in wrt:
        leaves1[k].requires_grad_()
        leaves2[k].requires_grad_()
    out = ops.SPMMSoftmaxAggr.apply(rowptr, col, leaves1["v"], colptr if "x" in wrt else None,
                                    perm if "x" in wrt else None, leaves1["x"], row[perm] if "x" in wrt else None,
                                    leaves1["t"])
    ref, _ = definition(rowptr, col, leaves2["v"], leaves2["x"], leaves2["t"])
    torch.testing.assert_close(out, ref.detach(), rtol=1e-12, atol=1e-12)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    got = torch.autograd.grad(out, [leaves1[k] for k in wrt], g)
    want = torch.autograd.grad(ref, [leaves2[k] for k in wrt], g)
    for k, a, b in zip(wrt, got, want):
        assert a.shape == b.shape and a.dtype == b.dtype, k
        torch.testing.assert_close(a, b, rtol=1e-10, atol=1e-10, msg=k)
    # only the kernels whose gradients are wanted ran, and the forward kept lse only for a backward
    assert cpu_kernels[0] == "fw+lse"
    assert ("rows" in cpu_kernels) == ("v" in wrt or "t" in wrt)
    assert ("cols" in cpu_kernels) == ("x" in wrt)


def test_no_gradient_keeps_no_lse(cpu_kernels):
    rowptr, col, value, x = _matrix(4, True)
    out = ops.SPMMSoftmaxAggr.apply(rowptr, col, value, None, None, x, None, torch.tensor(0.5, dtype=torch.float64))
    assert cpu_kernels == ["fw"] and not out.requires_grad


@pytest.mark.parametrize("wrt", ["v", "t"])
def test_value_or_temperature_gradient_builds_no_csc_view(cpu_kernels, wrt):
    rowptr, col, value, x = _matrix(5, True)
    M, N = rowptr.numel() - 1, x.size(0)
    v = value.clone().requires_grad_(wrt == "v")
    A = ts.SparseTensor(rowptr=rowptr, col=col, value=v, sparse_sizes=(M, N))
    t = torch.tensor(0.9, dtype=torch.float64, requires_grad=wrt == "t")
    out = tsm.spmm_softmax_aggr(A, x, t)
    out.sum().backward()
    st = A.storage
    assert st._csr2csc is None and st._colptr is None
    assert cpu_kernels == ["fw+lse", "rows"]
    assert (v.grad if wrt == "v" else t.grad) is not None
