"""`sddmm` / `sddmm_fp8` without a GPU: the registered op schemas, TorchScript of a function calling both, the exported
names, the C-ABI symbols and their argument checks, and CPU tensors being refused."""
import ctypes
from typing import Tuple

import pytest
import torch
from torch import Tensor

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import SparseTensor, _lib, ops

SCHEMAS = {
    "sddmm": "tsb200::sddmm(Tensor row, Tensor rowptr, Tensor col, Tensor? colptr, Tensor? csr2csc, Tensor? row_csc, "
             "Tensor a, Tensor b) -> Tensor",
    "sddmm_fp8": "tsb200::sddmm_fp8(Tensor rowptr, Tensor col, Tensor a8, Tensor a_scale, Tensor b8, Tensor b_scale, "
                 "ScalarType out_dtype) -> Tensor",
}


def test_op_schemas():
    for name, want in SCHEMAS.items():
        assert str(getattr(torch.ops.tsb200, name).default._schema) == want


def score_edges(src: SparseTensor, z: Tensor, z8: Tensor, s: Tensor) -> Tuple[Tensor, Tensor]:
    return ts.sddmm(src, z, z), ts.sddmm_fp8(src, z8, s, z8, s, torch.bfloat16)


def test_scripts_to_the_ops():
    graph = str(torch.jit.script(score_edges).inlined_graph)
    assert "tsb200::sddmm(" in graph and "tsb200::sddmm_fp8(" in graph
    assert "tsb200::sddmm(" in str(torch.jit.script(ts.sddmm).graph)
    assert "tsb200::sddmm_fp8(" in str(torch.jit.script(ts.sddmm_fp8).graph)


def test_exported_names():
    assert "sddmm" in ts.__all__ and "sddmm_fp8" in ts.__all__
    assert hasattr(SparseTensor, "sddmm") and hasattr(SparseTensor, "sddmm_fp8")


def test_c_abi_symbols_and_argument_errors():
    for name in ("tsb200_sddmm_fp8", "tsb200_sddmm_fp8_workspace_bytes"):
        assert name in _lib.SIGNATURES and hasattr(_lib.lib, name)
    lib = _lib.lib
    wsb = lib.tsb200_sddmm_fp8_workspace_bytes
    assert wsb(100, 0, 1000) == 0 and wsb(100, 16, 0) == 0
    assert wsb(100, 128, 1000) == lib.tsb200_spmm_value_bw_workspace_bytes(1, 100, 128, 1000, 0) > 0
    p = ctypes.c_void_p(256)      # never dereferenced: every call below returns before any launch
    ws = ctypes.c_void_p(1 << 20)

    def call(M=8, N=8, K=32, E=40, dt=3, a8=p, b8=p, out=p, sa=0, sb=1, col=p, work=ws, nws=1 << 30):
        return lib.tsb200_sddmm_fp8(p, col, a8, p, sa, b8, p, sb, out, M, N, K, E, dt, work, nws, None)

    assert call(M=-1) == -1                       # negative extent
    assert call(E=-1) == -1
    assert call(sa=2) == -1 and call(sb=-1) == -1  # scale strides 0 / 1 only
    assert call(dt=1) == -2 and call(dt=8) == -2  # f64, u8 results
    assert call(K=24) == -2                       # K % 16
    assert call(K=2064) == -2                     # K > 2048
    assert call(E=0) == 0                         # nothing to do
    assert call(out=None) == -1
    assert call(a8=None) == -1 and call(b8=None) == -1
    assert call(a8=ctypes.c_void_p(264)) == -2    # operands 16 B aligned
    assert call(b8=ctypes.c_void_p(264)) == -2
    assert call(col=ctypes.c_void_p(260)) == -2   # col 8 B
    assert call(out=ctypes.c_void_p(258), dt=0) == -2   # out aligned to its element
    assert call(E=(1 << 31) - 64) == -2
    assert call(N=1 << 32) == -2
    assert call(work=None) == -1 and call(work=ctypes.c_void_p(1 << 20 | 128)) == -1
    assert call(nws=1) == -3                      # short workspace


def test_cpu_tensors_refused():
    row = torch.tensor([0, 1, 1])
    col = torch.tensor([1, 0, 1])
    rowptr = torch.tensor([0, 1, 3])
    a = torch.randn(2, 16)
    with pytest.raises(RuntimeError, match="must be CUDA tensor"):
        ops.sddmm(row, rowptr, col, None, None, None, a, a)
    with pytest.raises(RuntimeError, match="must be CUDA tensor"):
        torch.ops.tsb200.sddmm(row, rowptr, col, None, None, None, a, a)
    src = SparseTensor(row=row, col=col, sparse_sizes=(2, 2))
    with pytest.raises(RuntimeError, match="must be CUDA tensor"):
        ts.sddmm(src, a, a)
    with pytest.raises(RuntimeError, match="must be CUDA tensor"):
        src.sddmm(a, a.requires_grad_())
    a8, s = ts.quantize_fp8(a.detach())
    with pytest.raises(RuntimeError, match="must be CUDA tensor"):
        ops.sddmm_fp8(rowptr, col, a8, s, a8, s)
    with pytest.raises(RuntimeError, match="must be CUDA tensor"):
        torch.ops.tsb200.sddmm_fp8(rowptr, col, a8, s, a8, s, torch.float32)
    with pytest.raises(RuntimeError, match="must be CUDA tensor"):
        src.sddmm_fp8(a8, s, a8, s)
