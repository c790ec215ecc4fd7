"""Softmax of a SparseTensor's stored values over each row (`dim=1`) or column (`dim=0`), one softmax per trailing
value column (per head for [E, H] scores), like `torch.sparse.softmax`. TorchScript-callable: the work is the
registered `torch.ops.tsb200.segment_softmax`."""
from __future__ import annotations

import torch

from .tensor import SparseTensor


def softmax(src: SparseTensor, dim: int) -> SparseTensor:
    """`src` with each row's (dim=1) or column's (dim=0) stored values replaced by their softmax, per trailing value
    column; same structure and cached views, values in CSR order with the value's dtype and shape. Every stored entry
    counts, duplicates included; an empty row or column has nothing to write. dim=-1 / -2 only for a 2-D tensor.
    bf16 / f16 / f32 / f64 values, fp32 arithmetic (fp64 for fp64). Differentiable in the values (once). A row
    softmax builds no CSC view."""
    value = src.storage.value()
    if value is None:
        raise ValueError("softmax: the sparse tensor has no values")
    d = dim + 2 if dim < 0 and src.dim() == 2 else dim
    if d != 0 and d != 1:
        raise ValueError("softmax: dim must be 0 or 1 (-2 or -1 for a 2-D sparse tensor), got " + str(dim)
                         + " for a " + str(src.dim()) + "-D sparse tensor")
    if value.size(0) != src.nnz():
        raise RuntimeError("softmax: value must have " + str(src.nnz()) + " rows (the nnz), got "
                           + str(value.size(0)))
    st = src.storage
    if d == 1:
        out = torch.ops.tsb200.segment_softmax(st.rowptr(), value, None)
    else:
        out = torch.ops.tsb200.segment_softmax(st.colptr(), value, st.csr2csc())
    return src.set_value(out, layout="csr")


SparseTensor.softmax = lambda self, dim: softmax(self, dim)
