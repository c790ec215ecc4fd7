"""pytorch_sparse_b200 — a from-scratch, Hopper-native (sm_90a) implementation of the
torch_sparse sparse-matmul hot path (CSR SpMM fwd/bwd, COO coalesce, SpSpMM) behind the
reference's own `SparseTensor` / `(index, value)` API.

    import pytorch_sparse_b200 as torch_sparse      # drop-in for the hot path

All arithmetic runs in libtsb200.so (hand-written CUDA behind the C-ABI in include/tsb200.h);
importing this package fails if that library is missing — there is no CPU fallback.
"""
from . import _lib  # noqa: F401  (loads libtsb200.so, raises ImportError when absent)
from . import ops  # noqa: F401
from .storage import SparseStorage  # noqa: F401
from .tensor import SparseTensor  # noqa: F401
from .matmul import matmul, spmm_sum, spmm_add, spmm_mean, spmm_min, spmm_max, spspmm_sum  # noqa: F401
from .matmul import spmm_fp8, spmm_fp8_quant, quantize_fp8, sddmm, sddmm_fp8, spmm_heads, sddmm_heads  # noqa: F401
from .matmul import spmm_multi, spmm_softmax_aggr  # noqa: F401
from .softmax import softmax  # noqa: F401
from .transpose import t, transpose  # noqa: F401
from .functional import coalesce, spmm, spspmm  # noqa: F401
from .add import add, add_, add_nnz, add_nnz_, spadd, narrow, mul, mul_, mul_nnz, mul_nnz_  # noqa: F401
from .reduce import sum, mean, min, max  # noqa: F401,A004
from .index_select import index_select, index_select_nnz, masked_select, select, to_symmetric  # noqa: F401
from . import torch_ops  # noqa: F401  (registers torch.ops.tsb200.* / torch.ops.torch_sparse.*)

__version__ = "0.1.0"

__all__ = ["SparseStorage", "SparseTensor", "t", "matmul", "coalesce", "transpose", "spmm", "spspmm", "spmm_fp8",
           "spmm_fp8_quant", "quantize_fp8", "sddmm", "sddmm_fp8", "spmm_heads", "sddmm_heads", "spmm_multi",
           "spmm_softmax_aggr", "softmax",
           "spadd",
           "add",
           "add_", "add_nnz", "add_nnz_",
           "narrow", "mul", "mul_", "mul_nnz", "mul_nnz_", "masked_select", "select", "sum", "mean", "min", "max", "index_select", "index_select_nnz", "to_symmetric", "__version__"]
