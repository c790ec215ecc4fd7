"""The FP8-result SpMM without a GPU: its TorchScript form and its public bindings."""
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import ops


def test_spmm_fp8_quant_scripts():
    scripted = torch.jit.script(ts.spmm_fp8_quant)
    assert "tsb200::spmm_fp8_quant" in str(scripted.graph)


def test_spmm_fp8_quant_bindings():
    assert "spmm_fp8_quant" in ts.__all__
    assert callable(ts.SparseTensor.spmm_fp8_quant)
    assert ops.FP8_QUANT_MAX_K == 2048
