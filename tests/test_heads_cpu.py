"""`spmm_heads` / `sddmm_heads` without a GPU: the registered op schemas, TorchScript of a function calling both, the
exported names, the C-ABI symbols and their argument checks, CPU tensors being refused, and the argument errors."""
import ctypes

import pytest
import torch
from torch import Tensor

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import SparseTensor, _lib, ops

SCHEMAS = {
    "spmm_heads": "tsb200::spmm_heads(Tensor? row, Tensor rowptr, Tensor col, Tensor? value, Tensor? colptr, "
                  "Tensor? csr2csc, Tensor x, Tensor? row_csc) -> Tensor",
    "sddmm_heads": "tsb200::sddmm_heads(Tensor row, Tensor rowptr, Tensor col, Tensor? colptr, Tensor? csr2csc, "
                   "Tensor? row_csc, Tensor a, Tensor b) -> Tensor",
}


def test_op_schemas():
    for name, want in SCHEMAS.items():
        assert str(getattr(torch.ops.tsb200, name).default._schema) == want


def attend(src: SparseTensor, q: Tensor, k: Tensor, v: Tensor) -> Tensor:
    s = ts.sddmm_heads(src, q, k)
    return ts.spmm_heads(src.set_value(s, layout="csr"), v)


def test_scripts_to_the_ops():
    graph = str(torch.jit.script(attend).inlined_graph)
    assert "tsb200::sddmm_heads(" in graph and "tsb200::spmm_heads(" in graph
    assert "tsb200::spmm_heads(" in str(torch.jit.script(ts.spmm_heads).graph)
    assert "tsb200::sddmm_heads(" in str(torch.jit.script(ts.sddmm_heads).graph)


def test_exported_names():
    assert "spmm_heads" in ts.__all__ and "sddmm_heads" in ts.__all__
    assert hasattr(SparseTensor, "spmm_heads") and hasattr(SparseTensor, "sddmm_heads")


def test_c_abi_symbols_and_argument_errors():
    lib = _lib.lib
    for name in ("tsb200_spmm_heads", "tsb200_sddmm_heads"):
        assert name in _lib.SIGNATURES and hasattr(lib, name)
    p = ctypes.c_void_p(256)      # never dereferenced: every call below returns before any launch
    ws = ctypes.c_void_p(1 << 20)

    def spmm(M=8, N=8, H=2, D=16, E=40, dt=3, x=p, out=p, col=p, rowptr=p, work=ws, nws=1 << 30, plan=None, pb=0,
             ns=0, nl=0, nsl=0):
        return lib.tsb200_spmm_heads(rowptr, col, p, x, out, M, N, H, D, E, dt, plan, pb, ns, nl, nsl, work, nws, None)

    def sddmm(M=8, N=8, H=2, D=16, E=40, dt=3, a=p, b=p, out=p, col=p, rowptr=p, work=ws, nws=1 << 30):
        return lib.tsb200_sddmm_heads(rowptr, col, a, b, out, M, N, H, D, E, dt, work, nws, None)

    for call in (spmm, sddmm):
        assert call(M=-1) == -1 and call(N=-1) == -1 and call(H=-1) == -1 and call(D=-1) == -1 and call(E=-1) == -1
        assert call(dt=4) == -2 and call(dt=8) == -2          # integer dtypes
        assert call(H=1 << 21, D=1 << 20) == -2               # H * D >= 2^40
        assert call(out=None) == -1
        assert call(rowptr=None) == -1 and call(col=None) == -1
        assert call(H=0) == 0                                 # nothing to write
    assert spmm(M=0) == 0 and spmm(D=0) == 0
    assert spmm(x=None) == -1
    assert spmm(nws=1) == -3                                  # short workspace on the vector path
    assert spmm(work=ctypes.c_void_p(1 << 20 | 128)) == -1    # misaligned workspace
    assert spmm(plan=ctypes.c_void_p(1 << 21), pb=1) == -3    # short plan
    assert spmm(ns=-1) == -1
    assert sddmm(E=0) == 0
    assert sddmm(a=None) == -1 and sddmm(b=None) == -1
    assert sddmm(nws=1) == -3


def test_cpu_tensors_refused():
    row = torch.tensor([0, 1, 1])
    col = torch.tensor([1, 0, 1])
    rowptr = torch.tensor([0, 1, 3])
    x = torch.randn(2, 2, 8)
    v = torch.randn(3, 2)
    for fn in (lambda: ops.spmm_heads(row, rowptr, col, v, None, None, x),
               lambda: torch.ops.tsb200.spmm_heads(row, rowptr, col, v, None, None, x, None),
               lambda: ops.sddmm_heads(row, rowptr, col, None, None, None, x, x),
               lambda: torch.ops.tsb200.sddmm_heads(row, rowptr, col, None, None, None, x, x)):
        with pytest.raises(RuntimeError, match="must be CUDA tensor"):
            fn()
    src = SparseTensor(row=row, col=col, value=v, sparse_sizes=(2, 2))
    with pytest.raises(RuntimeError, match="must be CUDA tensor"):
        src.spmm_heads(x)
    with pytest.raises(RuntimeError, match="must be CUDA tensor"):
        src.sddmm_heads(x, x.requires_grad_())


def test_argument_errors(monkeypatch):
    monkeypatch.setattr(ops, "_check_cuda", lambda t, n: None)     # the checks below run before any data is touched
    rowptr = torch.tensor([0, 1, 3])
    col = torch.tensor([1, 0, 1])
    x = torch.randn(2, 2, 8)
    cases = [
        (lambda: ops._spmm_heads_check(rowptr, col, None, x[0], None), r"spmm_heads: x must be 3-D \[N, H, D\], got 2-D"),
        (lambda: ops._spmm_heads_check(rowptr, col, None, x.long(), None),
         "\"spmm_heads\" not implemented for 'torch.int64'"),
        (lambda: ops._spmm_heads_check(rowptr, col, torch.randn(3, 3), x, None),
         r"spmm_heads: value must be \[E, H\] = \[3, 2\], got \[3, 3\]"),
        (lambda: ops._spmm_heads_check(rowptr, col, torch.randn(3), x, None),
         r"spmm_heads: value must be \[E, H\] = \[3, 2\], got \[3\]"),
        (lambda: ops._spmm_heads_check(rowptr, col, torch.randn(3, 2).double(), x, None),
         "spmm_heads: value and x must have the same dtype, got torch.float64 and torch.float32"),
        (lambda: ops._spmm_heads_check(rowptr, col, None, x, torch.tensor([0, 1, 2, 3])),
         r"spmm_heads: x must have 3 rows \(the matrix's columns\), got 2"),
        (lambda: ops._sddmm_heads_check(rowptr, col, x[0], x, None), r"sddmm_heads: a must be 3-D \[rows, H, D\], got 2-D"),
        (lambda: ops._sddmm_heads_check(rowptr, col, x, x[0], None), r"sddmm_heads: b must be 3-D \[rows, H, D\], got 2-D"),
        (lambda: ops._sddmm_heads_check(rowptr, col, x.int(), x.int(), None),
         "\"sddmm_heads\" not implemented for 'torch.int32'"),
        (lambda: ops._sddmm_heads_check(rowptr, col, x, x.half(), None),
         "sddmm_heads: a and b must have the same dtype, got torch.float32 and torch.float16"),
        (lambda: ops._sddmm_heads_check(rowptr, col, torch.randn(2, 2, 4), x, None),
         r"sddmm_heads: a must be \[M, H, D\] = \[2, 2, 8\] for b of shape \[2, 2, 8\], got \[2, 2, 4\]"),
        (lambda: ops._sddmm_heads_check(rowptr, col, x, x, torch.tensor([0, 1, 2, 3])),
         r"sddmm_heads: b must have 3 rows \(the matrix's columns\), got 2"),
    ]
    for fn, msg in cases:
        with pytest.raises(RuntimeError, match=msg):
            fn()
    src = SparseTensor(row=torch.tensor([0, 1, 1]), col=col, sparse_sizes=(2, 3))
    with pytest.raises(RuntimeError, match=r"spmm_heads: x must have 3 rows \(the sparse sizes\), got 2"):
        ts.spmm_heads(src, x)
    with pytest.raises(RuntimeError, match=r"sddmm_heads: a must have 2 rows and b 3 rows \(the sparse sizes\), got 2 "
                                           r"and 2"):
        ts.sddmm_heads(src, x, x)
