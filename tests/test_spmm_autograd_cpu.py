"""Mean aggregation's `grad_mat` weights, bit for bit, with the tensor-level kernels routed through the oracle (no GPU).

`SPMMMean.backward` forms grad_mat as a sum SpMM on the CSC view whose per-entry weights are value / count(row) (or
1 / count). The weights are formed in the accumulator type (fp32, fp64 for fp64) and rounded once to the dense dtype,
because the forward and the value gradient divide by the exact count: a count rounded to bf16 (above 256) or f16 (above
2048) first would give a row of degree 257 the weights of a row of degree 256.

Every row below has private columns, so each column of the CSC view holds one entry; with grad_out = 1, grad_mat[c]
is that entry's weight (the oracle's sum of one term times 1 is exact in every dtype). The expected weights are the
quotient in the accumulator type rounded once; `old` is the count-rounded-first formula, which the test uses to show
where the two differ (bf16 / f16 rows of a degree the dtype cannot hold) and that they agree everywhere else.
"""
import pytest
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import ops

MEAN_DEGREES = (1, 3, 255, 256, 257, 259, 300, 1001, 2047, 2048, 2049, 2051, 4100)
DTYPES = (torch.bfloat16, torch.float16, torch.float32, torch.float64)


def _id(p):
    return str(p).replace("torch.", "")


def private_column_case(dtype, has_value, seed=0):
    """CSR (rowptr, col, value) with one row per degree in MEAN_DEGREES and every entry in a column of its own, the
    columns shuffled so the CSC permutation is not the identity."""
    g = torch.Generator().manual_seed(seed)
    deg = torch.tensor(MEAN_DEGREES)
    rowptr = torch.zeros(deg.numel() + 1, dtype=torch.long)
    rowptr[1:] = deg.cumsum(0)
    E = int(rowptr[-1])
    col = torch.randperm(E, generator=g)
    value = torch.randn(E, generator=g, dtype=torch.float64).to(dtype) if has_value else None
    return rowptr, col, value


def mean_weights(rowptr, col, value, dtype):
    """-> (new, old, representable), per column of the CSC view (= per entry here): `new` the weight value / count
    (1 / count without values) in the accumulator type rounded once to `dtype`; `old` the same with the count rounded
    to `dtype` first; `representable` whether the entry's row degree is exact in `dtype`."""
    acc = torch.float64 if dtype == torch.float64 else torch.float32
    E = col.numel()
    d = torch.repeat_interleave(rowptr[1:] - rowptr[:-1], rowptr[1:] - rowptr[:-1])
    num = value.to(acc) if value is not None else torch.ones(E, dtype=acc)
    new = (num / d.to(acc)).to(dtype)
    cnt = d.to(dtype)
    old = value / cnt if value is not None else cnt.reciprocal()
    rep = cnt.to(torch.float64) == d.to(torch.float64)
    out = [torch.empty_like(t) for t in (new, old, rep)]
    for o, t in zip(out, (new, old, rep)):
        o[col] = t
    return tuple(out)


def bits(t):
    t = t.cpu().contiguous()
    return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def check_weight_expectations(new, old, rep, dtype, has_value):
    """The two formulas agree wherever the count is representable (and everywhere in fp32 / fp64); in bf16 / f16
    without values they differ on some rows, so a grad_mat equal to `new` cannot come from the old formula."""
    same = bits(new) == bits(old)
    assert bool(same[rep].all()), "weights of a representable degree differ between the two formulas"
    if dtype in (torch.float32, torch.float64):
        assert bool(same.all())
    elif not has_value:
        assert not bool(same.all())


def assert_rows_equal_weights(grad_mat, new, what):
    """grad_mat[c, k] == +0 + new[c] * 1: the sums start at +0, so a weight of -0 (an underflowed quotient) gives +0."""
    exp = (new.cpu() + 0.0).view(-1, 1).expand(grad_mat.shape)
    ok = bits(grad_mat) == bits(exp)
    if not bool(ok.all()):
        c, k = (int(j) for j in (~ok).nonzero()[0])
        raise AssertionError(f"{what}: {int((~ok).sum())} grad_mat elements differ from the weight, first at "
                             f"column {c}, k {k}: {grad_mat[c, k].item()!r} vs {new[c].item()!r}")


@pytest.fixture
def oracle_kernels(monkeypatch, oracle):
    """Route ops.py's tensor-level SpMM kernels through the oracle, so the autograd Functions run on CPU tensors."""
    monkeypatch.setattr(ops, "spmm_fw", lambda rowptr, col, value, mat, reduce: oracle.spmm(rowptr, col, value, mat,
                                                                                           reduce))
    monkeypatch.setattr(ops, "spmm_value_bw", oracle.spmm_value_bw)
    return oracle


@pytest.mark.parametrize("has_value", [True, False], ids=["value", "novalue"])
@pytest.mark.parametrize("dtype", DTYPES, ids=_id)
def test_mean_weights_bit_for_bit(oracle_kernels, dtype, has_value):
    rowptr, col, value = private_column_case(dtype, has_value)
    M, E, K = rowptr.numel() - 1, col.numel(), 3
    new, old, rep = mean_weights(rowptr, col, value, dtype)
    check_weight_expectations(new, old, rep, dtype, has_value)
    v = value.clone().requires_grad_() if has_value else None
    a = ts.SparseTensor(rowptr=rowptr, col=col, value=v, sparse_sizes=(M, E), is_sorted=True, trust_data=True)
    x = torch.randn(E, K, generator=torch.Generator().manual_seed(1), dtype=torch.float64).to(dtype).requires_grad_()
    out = ts.matmul(a, x, "mean")
    (gm,) = torch.autograd.grad(out, x, torch.ones_like(out))
    assert_rows_equal_weights(gm, new, f"{dtype} value={has_value}")
