"""Sparse @ dense (SpMM) and sparse @ sparse (SpSpMM) entry points.

Public names and behaviour follow torch_sparse/matmul.py (`spmm_sum/add/mean/min/max` :9-76, `spmm` :79-91,
`spspmm_sum` :94-111, `spspmm` :118-126, `matmul` :141-163, `SparseTensor` bindings :166-171), and like the
reference's these functions are TorchScript-compatible (`torch.jit.script(spspmm)`, test/test_matmul.py:79): every
native step is a registered operator. A reduction materialises only the cached CSR/CSC views a requested gradient
will read (the reference's rule, :19-25, :46-53).
"""
from typing import List, Optional, Tuple

import torch
from torch import Tensor

from .tensor import SparseTensor


def spmm_sum(src: SparseTensor, other: Tensor) -> Tensor:
    rowptr, col, value = src.csr()
    st = src.storage
    row, colptr, csr2csc = st._row, st._colptr, st._csr2csc
    row_csc: Optional[Tensor] = None
    if value is not None:
        value = value.to(other.dtype)
        if value.requires_grad:
            row = st.row()
    if other.requires_grad:     # A^T @ grad_out runs on the CSC view
        row = st.row()
        csr2csc = st.csr2csc()
        colptr = st.colptr()
        row_csc = st.row_csc()  # structure-only: gathered once per matrix instead of once per backward
    return torch.ops.tsb200.spmm_sum_csc(row, rowptr, col, value, colptr, csr2csc, other, row_csc)


def spmm_add(src: SparseTensor, other: Tensor) -> Tensor:
    return spmm_sum(src, other)


def spmm_mean(src: SparseTensor, other: Tensor) -> Tensor:
    rowptr, col, value = src.csr()
    st = src.storage
    row, rowcount, colptr, csr2csc = st._row, st._rowcount, st._colptr, st._csr2csc
    row_csc: Optional[Tensor] = None
    if value is not None:
        value = value.to(other.dtype)
        if value.requires_grad:
            row = st.row()
    if other.requires_grad:
        row = st.row()
        rowcount = st.rowcount()
        csr2csc = st.csr2csc()
        colptr = st.colptr()
        row_csc = st.row_csc()
    return torch.ops.tsb200.spmm_mean_csc(row, rowptr, col, value, rowcount, colptr, csr2csc, other, row_csc)


def spmm_min(src: SparseTensor, other: Tensor) -> Tuple[Tensor, Tensor]:
    rowptr, col, value = src.csr()
    if value is not None:
        value = value.to(other.dtype)
    return torch.ops.tsb200.spmm_min(rowptr, col, value, other)


def spmm_max(src: SparseTensor, other: Tensor) -> Tuple[Tensor, Tensor]:
    rowptr, col, value = src.csr()
    if value is not None:
        value = value.to(other.dtype)
    return torch.ops.tsb200.spmm_max(rowptr, col, value, other)


def spmm_res(src: SparseTensor, other: Tensor, residual: Tensor, residual_scale: Optional[Tensor] = None,
             reduce: str = "sum") -> Tensor:
    """`src @ other + residual_scale * residual` in one pass: the residual ([M, K], other's dtype) is added to every row
    in the kernels' store epilogue, out = round(fl(y + fl(s * r))) with y the fp32 (fp64) sum or mean. `other` is 2-D
    (bf16, f16, f32, f64); `residual_scale` is None (1) or float32 (float64 for f64) of shape [] or [M]. Differentiable
    in the values, `other`, `residual` and `residual_scale`; only the caches a requested gradient reads are built."""
    rowptr, col, value = src.csr()
    st = src.storage
    row, rowcount, colptr, csr2csc = st._row, st._rowcount, st._colptr, st._csr2csc
    row_csc: Optional[Tensor] = None
    if value is not None:
        value = value.to(other.dtype)
        if value.requires_grad:
            row = st.row()
    if other.requires_grad:     # A^T @ grad_out runs on the CSC view
        row = st.row()
        if reduce == "mean":
            rowcount = st.rowcount()
        csr2csc = st.csr2csc()
        colptr = st.colptr()
        row_csc = st.row_csc()
    return torch.ops.tsb200.spmm_res(row, rowptr, col, value, rowcount, colptr, csr2csc, other, row_csc, residual,
                                     residual_scale, reduce)


def spmm(src: SparseTensor, other: Tensor, reduce: str = "sum", residual: Optional[Tensor] = None,
         residual_scale: Optional[Tensor] = None) -> Tensor:
    """`src @ other` reduced per row (sum / add / mean / min / max). With `residual` (sum / add / mean, 2-D `other`):
    `src @ other + residual_scale * residual` in one pass (see `spmm_res`)."""
    if residual is not None:
        return spmm_res(src, other, residual, residual_scale, reduce)
    if residual_scale is not None:
        raise ValueError("spmm: residual_scale needs a residual")
    if reduce == "sum" or reduce == "add":
        return spmm_sum(src, other)
    elif reduce == "mean":
        return spmm_mean(src, other)
    elif reduce == "min":
        return spmm_min(src, other)[0]     # values only; arg_out stays internal
    elif reduce == "max":
        return spmm_max(src, other)[0]
    else:
        raise ValueError("unknown reduce '" + reduce + "'")


def spmm_multi(src: SparseTensor, other: Tensor, aggrs: List[str]) -> Tensor:
    """Several aggregations of every row's messages value[e] * other[col[e]] from one gather pass: out [M, A, K] holds
    aggregator aggrs[a] in out[:, a] (sum / add, mean, min, max, var, std; each at most once), and `out.flatten(1)` is
    their feature-dim concatenation, as PNA and multi-aggregation layers use it. sum, mean, min and max are bit for bit
    `spmm`'s. With n = max(degree, 1): var = max(Q / n - mean^2, 0), Q the fp32 (fp64) sum of squared messages, and
    std = sqrt(var) where var > 1e-5, else 0; neither passes a gradient where its clamp is active, which keeps the
    gradient finite on constant and one-entry rows. `other` is 2-D (bf16, f16, f32, f64). Differentiable in the values
    and `other`; only the caches a requested gradient reads are built."""
    if other.dim() != 2:
        raise RuntimeError("spmm_multi: other must be 2-D [N, K], got " + str(other.dim()) + "-D")
    N = src.size(1)
    if other.size(0) != N:
        raise RuntimeError("spmm_multi: other must have " + str(N) + " rows (the sparse sizes), got " + str(other.size(0)))
    rowptr, col, value = src.csr()
    st = src.storage
    row, colptr, csr2csc = st._row, st._colptr, st._csr2csc
    row_csc: Optional[Tensor] = None
    if value is not None:
        value = value.to(other.dtype)
        if value.requires_grad:
            row = st.row()
    if other.requires_grad:     # A^T a and A_{v^2}^T b run on the CSC view
        row = st.row()
        csr2csc = st.csr2csc()
        colptr = st.colptr()
        row_csc = st.row_csc()
    return torch.ops.tsb200.spmm_multi(row, rowptr, col, value, colptr, csr2csc, other, row_csc, aggrs)


def spmm_softmax_aggr(src: SparseTensor, other: Tensor, t: Optional[Tensor] = None) -> Tensor:
    """Softmax aggregation of every row's messages p_e = value[e] * other[col[e]], per feature column k:
    out[m, k] = sum_e softmax_e(t_k p_e) p_e over the entries of row m, as PyG's SoftmaxAggregation and GENConv's
    default aggregation compute it, in one gather pass with no [E, K] temporary. `other` is 2-D [N, K] (bf16, f16,
    f32, f64); `t` is the temperature in float32 (float64 for f64) of shape [] or [1] (one for all columns) or [K], or
    None for t = 1 (not learnable). The softmax runs online in fp32 (fp64), shifted by each row's own maximum, so rows
    far from the column's global maximum do not underflow. An empty row gives 0; t = 0 gives `spmm(src, other,
    "mean")`, and a negative t a soft minimum. Differentiable in the values, `other` and `t`; only a gradient to
    `other` builds the CSC view."""
    if other.dim() != 2:
        raise RuntimeError("spmm_softmax_aggr: other must be 2-D [N, K], got " + str(other.dim()) + "-D")
    N = src.size(1)
    if other.size(0) != N:
        raise RuntimeError("spmm_softmax_aggr: other must have " + str(N) + " rows (the sparse sizes), got "
                           + str(other.size(0)))
    rowptr, col, value = src.csr()
    st = src.storage
    colptr: Optional[Tensor] = None
    csr2csc: Optional[Tensor] = None
    row_csc: Optional[Tensor] = None
    if value is not None:
        value = value.to(other.dtype)
    if other.requires_grad:     # the column-wise backward runs on the CSC view
        csr2csc = st.csr2csc()
        colptr = st.colptr()
        row_csc = st.row_csc()
    return torch.ops.tsb200.spmm_softmax_aggr(rowptr, col, value, colptr, csr2csc, other, row_csc, t)


def spmm_fp8(src: SparseTensor, x8: Tensor, scale: Tensor, reduce: str = "sum",
             out_dtype: torch.dtype = torch.bfloat16, residual: Optional[Tensor] = None,
             residual_scale: Optional[Tensor] = None) -> Tensor:
    """`src @ (x8 * scale)` over an FP8 (e4m3) dense operand `x8` [N, K] (K % 16 == 0) with a float32 `scale` of
    shape [] or [N] (see `quantize_fp8`), reduce in sum/add/mean/min/max, result in `out_dtype` (bf16, f16, f32).
    The entry values are cast to `out_dtype` first, as `spmm` casts them to the dense dtype. Forward only: no
    gradient flows, and a `value` or `scale` that requires grad is refused while grad mode is on.
    With `residual` (e4m3 [M, K]) and `residual_scale` (float32 [] or [M]), sum / mean only, the kernel adds
    `residual_scale[m] * residual[m]` to row m of the float32 result before rounding it to `out_dtype`."""
    rowptr, col, value = src.csr()
    if value is not None:
        value = value.to(out_dtype)
    if reduce == "add":
        reduce = "sum"
    if reduce != "sum" and reduce != "mean" and reduce != "min" and reduce != "max":
        raise ValueError("unknown reduce '" + reduce + "'")
    return torch.ops.tsb200.spmm_fp8(rowptr, col, value, x8, scale, reduce, out_dtype, residual, residual_scale)[0]


def spmm_fp8_quant(src: SparseTensor, x8: Tensor, scale: Tensor, reduce: str = "sum",
                   residual: Optional[Tensor] = None, residual_scale: Optional[Tensor] = None) -> Tuple[Tensor, Tensor]:
    """One FP8 propagation hop: `src @ (x8 * scale)` as `spmm_fp8(..., torch.float32)` computes it, returned as
    `(y8, y_scale)` = `quantize_fp8(y, per_row=True)` of that float32 result, bit for bit, without materialising y:
    the kernels quantise each row as they store it. The pair is the `x8` / `scale` of the next hop, so repeated
    propagation (SIGN, APPNP, label propagation) stays in e4m3. K <= 2048 columns; entry values are cast to float32.
    Forward only: a `value` or `scale` that requires grad is refused while grad mode is on.
    With `residual` (e4m3 [M, K]) and `residual_scale` (float32 [] or [M]), sum / mean only, the rows quantised are
    `y[m] + residual_scale[m] * residual[m]` (one fp32 product and one fp32 add), so a propagation step with a fixed
    residual term stays in e4m3: APPNP `X = (1 - a) A X + a H` takes entry values times (1 - a) and `residual_scale`
    times a (see README)."""
    rowptr, col, value = src.csr()
    if value is not None:
        value = value.to(torch.float32)
    if reduce == "add":
        reduce = "sum"
    if reduce != "sum" and reduce != "mean" and reduce != "min" and reduce != "max":
        raise ValueError("unknown reduce '" + reduce + "'")
    y8, y_scale, _ = torch.ops.tsb200.spmm_fp8_quant(rowptr, col, value, x8, scale, reduce, residual, residual_scale)
    return y8, y_scale


def quantize_fp8(x: Tensor, per_row: bool = True) -> Tuple[Tensor, Tensor]:
    """A 2-D floating `x` [N, K] as `(x8, scale)` for `spmm_fp8`: scale = amax|x| / 448 (e4m3's largest finite value)
    per row ([N]) or over the whole tensor ([]), 1 where that amax is not > 0 (all-zero and NaN rows), and
    x8 = e4m3(x.float() / scale), rounded to nearest even; magnitudes past 464 and inf become NaN.
    A CUDA `x` is quantised by one streaming kernel (`torch.ops.tsb200.quantize_fp8`, two launches for a per-tensor
    scale) without float temporaries, bit for bit the CPU result; bf16, f16 and f32 are read as they are, other dtypes
    through `.float()`, and a column slice of a wider matrix is read in place. The torch expression below is the
    definition: it runs for a CPU `x`, and for an `x` that requires grad while grad mode is on, whose `scale` keeps
    its autograd history."""
    if x.dim() != 2:
        raise ValueError("quantize_fp8 expects a 2-D tensor [N, K]")
    if x.is_cuda and not (x.requires_grad and torch.is_grad_enabled()):
        if x.dtype != torch.bfloat16 and x.dtype != torch.float16 and x.dtype != torch.float32:
            x = x.float()
        return torch.ops.tsb200.quantize_fp8(x, per_row)
    xf = x.float()
    amax = xf.abs().amax(dim=1) if per_row else xf.abs().amax()
    scale = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    x8 = (xf / (scale.unsqueeze(1) if per_row else scale)).to(torch.float8_e4m3fn)
    return x8, scale


def sddmm(src: SparseTensor, a: Tensor, b: Tensor) -> Tensor:
    """Edge scores `out[e] = <a[row_e], b[col_e]>` for every stored entry of `src` (M x N), in CSR order, without an
    E x K temporary: `a` [M, K] and `b` [N, K] share a floating dtype (bf16, f16, f32, f64), accumulated in fp32
    (fp64 for fp64) and rounded once. `src`'s values are ignored: only its structure is used. Differentiable in `a` and
    `b`; the gradients are SpMMs with the incoming gradient as values, on the CSR view for `a` and on the cached CSC
    view for `b`. To score arbitrary pairs (i, j), build `SparseTensor(row=i, col=j, value=arange)` and scatter the
    scores back through its permuted values (see README)."""
    rowptr, col, _ = src.csr()
    st = src.storage
    M, N = src.sparse_sizes()
    if a.dim() == 2 and b.dim() == 2 and (a.size(0) != M or b.size(0) != N):
        raise RuntimeError("sddmm: a must have " + str(M) + " rows and b " + str(N) + " rows (the sparse sizes), got "
                           + str(a.size(0)) + " and " + str(b.size(0)))
    row = st.row()
    colptr, csr2csc = st._colptr, st._csr2csc
    row_csc: Optional[Tensor] = None
    if b.requires_grad:     # grad_b = A(g)^T @ a runs on the CSC view
        csr2csc = st.csr2csc()
        colptr = st.colptr()
        row_csc = st.row_csc()
    return torch.ops.tsb200.sddmm(row, rowptr, col, colptr, csr2csc, row_csc, a, b)


def sddmm_fp8(src: SparseTensor, a8: Tensor, a_scale: Tensor, b8: Tensor, b_scale: Tensor,
              out_dtype: torch.dtype = torch.float32) -> Tensor:
    """`sddmm` over two FP8 (e4m3) operands with float32 scales of shape [] or [rows] (see `quantize_fp8`):
    `out[e] = round_out(fl32(a_scale[r] * b_scale[c]) * sum_k a8[r, k] * b8[c, k])`, the sum in fp32 (every e4m3
    product is exact). `a8` [M, K] and `b8` [N, K] contiguous and 16-byte aligned, K % 16 == 0 and K <= 2048 (a
    ValueError otherwise); out_dtype bf16, f16 or f32. `src`'s values are ignored. Forward only: a scale that requires
    grad is refused while grad mode is on."""
    rowptr, col, _ = src.csr()
    N = src.sparse_size(1)
    if b8.dim() == 2 and b8.size(0) != N:
        raise RuntimeError("sddmm_fp8: b8 must have " + str(N) + " rows (the sparse sizes), got " + str(b8.size(0)))
    return torch.ops.tsb200.sddmm_fp8(rowptr, col, a8, a_scale, b8, b_scale, out_dtype)


def spmm_heads(src: SparseTensor, x: Tensor) -> Tensor:
    """Multi-head message passing: `out[m, h] = sum_e value[e, h] * x[col_e, h]` over the entries of row m, for `x`
    [N, H, D] and a value of `src` of shape [E, H] (or none: every weight 1), `out` [M, H, D], without an E x H*D
    temporary. The value is cast to x's dtype (bf16, f16, f32, f64); fp32 accumulation (fp64 for fp64), one rounding.
    Differentiable in the value (an `sddmm_heads`) and in `x` (an `spmm_heads` on the cached CSC view). With H = 1 the
    result is `spmm`'s, bit for bit."""
    rowptr, col, value = src.csr()
    st = src.storage
    N = src.sparse_size(1)
    if x.dim() == 3 and x.size(0) != N:
        raise RuntimeError("spmm_heads: x must have " + str(N) + " rows (the sparse sizes), got " + str(x.size(0)))
    row, colptr, csr2csc = st._row, st._colptr, st._csr2csc
    row_csc: Optional[Tensor] = None
    if value is not None:
        value = value.to(x.dtype)
    if x.requires_grad:     # grad_x = A^T @ grad_out per head runs on the CSC view
        row = st.row()
        csr2csc = st.csr2csc()
        colptr = st.colptr()
        row_csc = st.row_csc()
    return torch.ops.tsb200.spmm_heads(row, rowptr, col, value, colptr, csr2csc, x, row_csc)


def sddmm_heads(src: SparseTensor, a: Tensor, b: Tensor) -> Tensor:
    """Multi-head edge scores `s[e, h] = <a[row_e, h], b[col_e, h]>` for `a` [M, H, D] and `b` [N, H, D], `s` [E, H]
    in CSR order, without an E x H*D temporary; dtypes and accumulation as `sddmm`, whose result it is for H = 1.
    `src`'s values are ignored. Differentiable in `a` and `b` (`spmm_heads` on the CSR and the cached CSC view)."""
    rowptr, col, _ = src.csr()
    st = src.storage
    M, N = src.sparse_sizes()
    if a.dim() == 3 and b.dim() == 3 and (a.size(0) != M or b.size(0) != N):
        raise RuntimeError("sddmm_heads: a must have " + str(M) + " rows and b " + str(N) + " rows (the sparse sizes), "
                           "got " + str(a.size(0)) + " and " + str(b.size(0)))
    row = st.row()
    colptr, csr2csc = st._colptr, st._csr2csc
    row_csc: Optional[Tensor] = None
    if b.requires_grad:     # grad_b = A(g)^T @ a per head runs on the CSC view
        csr2csc = st.csr2csc()
        colptr = st.colptr()
        row_csc = st.row_csc()
    return torch.ops.tsb200.sddmm_heads(row, rowptr, col, colptr, csr2csc, row_csc, a, b)


def spspmm_sum(src: SparseTensor, other: SparseTensor) -> SparseTensor:
    M, Kd = src.sparse_sizes()
    Kb, N = other.sparse_sizes()
    assert Kd == Kb, "inner dimensions differ"
    rowptr_a, col_a, val_a = src.csr()
    rowptr_b, col_b, val_b = other.csr()
    want_value = val_a is not None or val_b is not None   # a missing side counts as all-ones
    if val_a is not None and val_a.dim() > 1:
        raise RuntimeError("spspmm: multi-dimensional values are not supported")
    if val_b is not None and val_b.dim() > 1:
        raise RuntimeError("spspmm: multi-dimensional values are not supported")
    if val_a is not None and val_b is not None and val_a.dtype != val_b.dtype:
        val_b = val_b.to(val_a.dtype)
    rowptr_c, row_c, col_c, val_c = torch.ops.tsb200.spspmm(rowptr_a, col_a, val_a, rowptr_b, col_b, val_b, M, Kd, N,
                                                            want_value)
    return SparseTensor(row_c, rowptr_c, col_c, val_c, (M, N), True, True)


def spspmm_add(src: SparseTensor, other: SparseTensor) -> SparseTensor:
    return spspmm_sum(src, other)


def spspmm(src: SparseTensor, other: SparseTensor, reduce: str = "sum") -> SparseTensor:
    if reduce == "sum" or reduce == "add":
        return spspmm_sum(src, other)
    elif reduce == "mean" or reduce == "min" or reduce == "max":
        raise NotImplementedError("spspmm with reduce='" + reduce + "'")
    else:
        raise ValueError("unknown reduce '" + reduce + "'")


@torch.jit._overload  # noqa: F811
def matmul(src, other, reduce):  # noqa: F811
    # type: (SparseTensor, Tensor, str) -> Tensor
    pass


@torch.jit._overload  # noqa: F811
def matmul(src, other, reduce):  # noqa: F811
    # type: (SparseTensor, SparseTensor, str) -> SparseTensor
    pass


def matmul(src, other, reduce="sum"):  # noqa: F811
    """`src @ other`: a dense `other` gives a dense result (reduce in sum/add/mean/min/max over each row's
    entries); a SparseTensor `other` gives a SparseTensor (sum only)."""
    if isinstance(other, Tensor):
        return spmm(src, other, reduce)
    elif isinstance(other, SparseTensor):
        return spspmm(src, other, reduce)
    raise ValueError("cannot multiply a SparseTensor with this operand")


SparseTensor.spmm = lambda self, other, reduce="sum", residual=None, residual_scale=None: spmm(
    self, other, reduce, residual, residual_scale)
SparseTensor.spmm_fp8 = lambda self, x8, scale, reduce="sum", out_dtype=torch.bfloat16, residual=None, \
    residual_scale=None: spmm_fp8(self, x8, scale, reduce, out_dtype, residual, residual_scale)
SparseTensor.spmm_fp8_quant = lambda self, x8, scale, reduce="sum", residual=None, residual_scale=None: spmm_fp8_quant(
    self, x8, scale, reduce, residual, residual_scale)
SparseTensor.sddmm = lambda self, a, b: sddmm(self, a, b)
SparseTensor.sddmm_fp8 = lambda self, a8, a_scale, b8, b_scale, out_dtype=torch.float32: sddmm_fp8(
    self, a8, a_scale, b8, b_scale, out_dtype)
SparseTensor.spmm_heads = lambda self, x: spmm_heads(self, x)
SparseTensor.spmm_multi = lambda self, other, aggrs: spmm_multi(self, other, aggrs)
SparseTensor.spmm_softmax_aggr = lambda self, other, t=None: spmm_softmax_aggr(self, other, t)
SparseTensor.sddmm_heads = lambda self, a, b: sddmm_heads(self, a, b)
SparseTensor.spspmm = lambda self, other, reduce="sum": spspmm(self, other, reduce)
SparseTensor.matmul = lambda self, other, reduce="sum": matmul(self, other, reduce)
SparseTensor.__matmul__ = lambda self, other: matmul(self, other, "sum")
