"""FP8 helpers that need no GPU: `quantize_fp8` and the TorchScript form of `spmm_fp8`."""
import pytest
import torch

import pytorch_sparse_b200 as ts


def e4m3_half_ulp(y):
    """1/2 ulp of e4m3 at |y| (3 fraction bits; normals from 2^-6, subnormal spacing 2^-9)."""
    _, e = torch.frexp(y.abs())
    e = torch.clamp(e - 1, min=-6)          # exponent of the binade (subnormals share the smallest)
    return torch.ldexp(torch.full_like(y, 0.5), (e - 3).to(torch.int32))


@pytest.mark.parametrize("per_row", [True, False], ids=["rowscale", "tensorscale"])
def test_quantize_fp8_round_trip(per_row):
    g = torch.Generator().manual_seed(0)
    x = torch.randn(200, 48, generator=g) * torch.logspace(-4, 3, 200).view(-1, 1)
    x[[3, 77]] = 0.0                                         # all-zero rows
    x[5, :7] = -0.0
    x8, scale = ts.quantize_fp8(x, per_row)
    assert x8.dtype == torch.float8_e4m3fn and x8.shape == x.shape
    assert scale.dtype == torch.float32 and scale.shape == ((200,) if per_row else ())
    s = scale.view(-1, 1) if per_row else scale
    amax = x.abs().amax(dim=1) if per_row else x.abs().amax()
    assert torch.equal(scale, torch.where(amax > 0, amax / 448.0, torch.ones_like(amax)))
    if per_row:
        assert bool((scale[[3, 77]] == 1).all()) and bool((x8[[3, 77]].float() == 0).all())
    assert not bool(x8.float().isnan().any())
    # x / s is rounded once to e4m3: error <= 1/2 ulp there (plus the fp32 roundings of the division and of the
    # product back, relative 2^-24 each)
    y = x / s
    err = (x8.float() * s - x).abs()
    bound = e4m3_half_ulp(y) * s * (1 + 2.0 ** -22) + x.abs() * 2.0 ** -22
    assert bool((err <= bound).all()), float((err - bound).max())
    assert bool((x8.float().abs() <= 448).all())


def test_quantize_fp8_rejects_non_2d():
    with pytest.raises(ValueError):
        ts.quantize_fp8(torch.ones(3))


def test_spmm_fp8_scripts():
    scripted = torch.jit.script(ts.spmm_fp8)
    assert "tsb200::spmm_fp8" in str(scripted.graph)
    torch.jit.script(ts.quantize_fp8)
