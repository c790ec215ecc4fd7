"""`quantize_fp8` without a GPU: the registered op, the TorchScript form, the C-ABI symbol and its argument checks, and
the CPU path (the definition the native quantiser is tested against) computing exactly what it computed before."""
import ctypes

import pytest
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import _lib, ops


def torch_quantize_fp8(x, per_row):
    """The CPU expression as it stands, restated."""
    xf = x.float()
    amax = xf.abs().amax(dim=1) if per_row else xf.abs().amax()
    scale = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    x8 = (xf / (scale.unsqueeze(1) if per_row else scale)).to(torch.float8_e4m3fn)
    return x8, scale


def test_op_schema():
    schema = str(torch.ops.tsb200.quantize_fp8.default._schema)
    assert schema == "tsb200::quantize_fp8(Tensor x, bool per_row) -> (Tensor, Tensor)", schema


def test_quantize_fp8_scripts_to_the_op():
    scripted = torch.jit.script(ts.quantize_fp8)
    assert "tsb200::quantize_fp8" in str(scripted.graph)
    x = torch.randn(6, 20)
    for per_row in (True, False):
        a8, a = scripted(x, per_row)
        b8, b = torch_quantize_fp8(x, per_row)
        assert torch.equal(a8.view(torch.uint8), b8.view(torch.uint8)) and torch.equal(a, b)


def test_bindings_and_c_abi():
    assert "quantize_fp8" in ts.__all__
    assert "tsb200_quantize_fp8" in _lib.SIGNATURES and hasattr(_lib.lib, "tsb200_quantize_fp8")
    q = _lib.lib.tsb200_quantize_fp8
    p = ctypes.c_void_p(256)      # never dereferenced: every call below returns before any launch
    assert q(p, -1, 16, 16, 3, 1, p, p, None, 0, None) == -1          # negative N
    assert q(p, 4, 16, 8, 3, 1, p, p, None, 0, None) == -1            # ld < K
    assert q(p, 4, 16, 16, 3, 2, p, p, None, 0, None) == -1           # per_row not 0 / 1
    assert q(p, 4, 0, 16, 3, 1, p, p, None, 0, None) == -1            # K == 0: the amax of nothing
    assert q(p, 0, 16, 16, 3, 0, p, p, p, 4, None) == -1              # per tensor, N == 0
    assert q(None, 4, 16, 16, 3, 1, p, p, None, 0, None) == -1        # NULL x
    assert q(p, 4, 16, 16, 1, 1, p, p, None, 0, None) == -2           # f64
    assert q(p, 4, 16, 16, 3, 1, p, ctypes.c_void_p(258), None, 0, None) == -2   # misaligned scale
    assert q(p, 4, 16, 16, 3, 0, p, p, None, 0, None) == -3           # per tensor without a workspace
    assert q(p, 4, 16, 16, 3, 0, p, p, p, 2, None) == -3              # short workspace
    assert q(p, 0, 16, 16, 3, 1, p, p, None, 0, None) == 0            # N == 0 per row: nothing to do


def test_ops_reject_cpu_tensors():
    with pytest.raises(RuntimeError, match="must be CUDA tensor"):
        ops.quantize_fp8(torch.ones(2, 16))
    with pytest.raises(RuntimeError, match="must be CUDA tensor"):
        torch.ops.tsb200.quantize_fp8(torch.ones(2, 16), True)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16, torch.float64, torch.int32])
@pytest.mark.parametrize("per_row", [True, False], ids=["rowscale", "tensorscale"])
def test_cpu_path_unchanged(dtype, per_row):
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(37, 33, generator=g, dtype=torch.float64) * 50).to(dtype)
    if dtype.is_floating_point:
        x[3] = 0.0
        x[4, 2] = float("nan")
        x[5, 7] = float("inf")
    for inp in (x, x[:, 1:30], x.t()):
        a8, a = ts.quantize_fp8(inp, per_row)
        b8, b = torch_quantize_fp8(inp, per_row)
        assert torch.equal(a8.view(torch.uint8), b8.view(torch.uint8))
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_cpu_path_keeps_autograd_history():
    x = torch.randn(5, 16, requires_grad=True)
    for per_row in (True, False):
        _, s = ts.quantize_fp8(x, per_row)
        assert s.grad_fn is not None
        s.sum().backward()
    assert x.grad is not None


def test_cpu_error_cases_unchanged():
    with pytest.raises(ValueError):
        ts.quantize_fp8(torch.ones(2, 3, 4))
    with pytest.raises(IndexError):
        ts.quantize_fp8(torch.ones(3, 0), True)
    with pytest.raises(RuntimeError):
        ts.quantize_fp8(torch.ones(3, 0), False)
    with pytest.raises(RuntimeError):
        ts.quantize_fp8(torch.ones(0, 4), False)
    x8, s = ts.quantize_fp8(torch.ones(0, 4), True)
    assert x8.shape == (0, 4) and s.shape == (0,)
