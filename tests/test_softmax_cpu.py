"""Sparse softmax without a GPU: the registered op schema, TorchScript of `softmax` and of an attention function, the
exported names, the C-ABI symbols and their argument checks, CPU tensors being refused, and the argument errors."""
import ctypes

import pytest
import torch
from torch import Tensor

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import SparseTensor, _lib, ops


def test_op_schema():
    assert str(torch.ops.tsb200.segment_softmax.default._schema) == \
        "tsb200::segment_softmax(Tensor ptr, Tensor value, Tensor? perm) -> Tensor"


def attend(src: SparseTensor, q: Tensor, k: Tensor, v: Tensor) -> Tensor:
    s = ts.sddmm_heads(src, q, k)
    return ts.spmm_heads(ts.softmax(src.set_value(s, layout="csr"), 1), v)


def test_scripts_to_the_op():
    assert "tsb200::segment_softmax(" in str(torch.jit.script(ts.softmax).graph)
    graph = str(torch.jit.script(attend).inlined_graph)
    assert "tsb200::segment_softmax(" in graph and "tsb200::spmm_heads(" in graph


def test_exported_names():
    assert "softmax" in ts.__all__ and callable(ts.softmax)
    assert hasattr(SparseTensor, "softmax")


def test_c_abi_symbols_and_argument_errors():
    lib = _lib.lib
    for name in ("tsb200_segment_softmax", "tsb200_segment_softmax_bw"):
        assert name in _lib.SIGNATURES and hasattr(lib, name)
    p = ctypes.c_void_p(256)      # never dereferenced: every call below returns before any launch

    def fw(S=4, E=40, D=8, dt=3, ptr=p, perm=None, value=p, out=p):
        return lib.tsb200_segment_softmax(ptr, perm, value, out, S, E, D, dt, None)

    def bw(S=4, E=40, D=8, dt=3, ptr=p, perm=None, value=p, out=p, g=p):
        return lib.tsb200_segment_softmax_bw(ptr, perm, value, g, out, S, E, D, dt, None)

    for call in (fw, bw):
        assert call(S=-1) == -1 and call(E=-1) == -1 and call(D=-1) == -1
        assert call(S=0) == 0 and call(E=0) == 0 and call(D=0) == 0       # nothing to do: no launch
        assert call(ptr=None) == -1 and call(value=None) == -1 and call(out=None) == -1
        for dt in (4, 5, 6, 7, 8):                                         # integer dtypes
            assert call(dt=dt) == -2
    assert bw(g=None) == -1


def test_cpu_tensors_refused():
    row = torch.tensor([0, 1, 1])
    col = torch.tensor([1, 0, 1])
    rowptr = torch.tensor([0, 1, 3])
    v = torch.randn(3, 2)
    for fn in (lambda: ops.segment_softmax(rowptr, v),
               lambda: torch.ops.tsb200.segment_softmax(rowptr, v, None)):
        with pytest.raises(RuntimeError, match="must be CUDA tensor"):
            fn()
    src = SparseTensor(row=row, col=col, value=v, sparse_sizes=(2, 2))
    for dim in (0, 1):
        with pytest.raises(RuntimeError, match="must be CUDA tensor"):
            src.softmax(dim)


def test_argument_errors(monkeypatch):
    monkeypatch.setattr(ops, "_check_cuda", lambda t, n: None)     # the checks below run before any data is touched
    row = torch.tensor([0, 1, 1])
    col = torch.tensor([1, 0, 1])
    src = SparseTensor(row=row, col=col, sparse_sizes=(2, 2))
    with pytest.raises(ValueError, match="softmax: the sparse tensor has no values"):
        ts.softmax(src, 1)
    two = src.set_value(torch.randn(3), layout="csr")
    heads = src.set_value(torch.randn(3, 4), layout="csr")
    for s, dim in ((two, 2), (two, -3), (heads, -1), (heads, -2), (heads, 2)):
        with pytest.raises(ValueError, match=f"softmax: dim must be 0 or 1 .* got {dim} for a {s.dim()}-D"):
            ts.softmax(s, dim)
    with pytest.raises(RuntimeError, match="\"softmax\" not implemented for 'torch.int64'"):
        ts.softmax(src.set_value(torch.arange(3), layout="csr"), 1)
    with pytest.raises(RuntimeError, match="\"softmax\" not implemented for 'torch.int32'"):
        ops.segment_softmax(torch.tensor([0, 1, 3]), torch.arange(3, dtype=torch.int32))
    bad = src.set_value(torch.randn(3), layout="csr")
    bad.storage._value = torch.randn(4)
    with pytest.raises(RuntimeError, match=r"softmax: value must have 3 rows \(the nnz\), got 4"):
        ts.softmax(bad, 1)
    with pytest.raises(RuntimeError, match=r"softmax: value must have 3 rows \(the nnz\), got 4"):
        ops.segment_softmax(torch.tensor([0, 1, 3]), torch.randn(4), torch.tensor([1, 0, 2]))
    with pytest.raises(RuntimeError, match="softmax: value must be \\[E\\] or \\[E, \\*\\], got a 0-D tensor"):
        ops.segment_softmax(torch.tensor([0, 1, 3]), torch.tensor(1.0))
