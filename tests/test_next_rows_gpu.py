"""SURVEY §8(f) "next" rows on the GPU vs golden vectors from the unmodified reference: row/column
reductions (torch_sparse/reduce.py), sparse + sparse (add.py:38-56, spadd.py:5-18), narrow (narrow.py)."""
from pathlib import Path

import pytest
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import ops
from util import assert_spspmm_values, random_csr, segment_sum_ref_bound

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
D = torch.load(Path(__file__).resolve().parent / "golden" / "next_rows.pt", weights_only=False)


def _mk(kind):
    i = D["in"]
    v = {"v": i["va"], "v2": i["va2"], "nv": None}[kind]
    return ts.SparseTensor(row=i["ra"].to(DEV), col=i["ca"].to(DEV), value=None if v is None else v.to(DEV),
                           sparse_sizes=(i["M"], i["N"]))


@pytest.mark.parametrize("kind", ["v", "v2", "nv"])
def test_reductions_vs_reference(kind):
    a = _mk(kind)
    for op in ("sum", "mean", "min", "max"):
        for dim in (None, 0, 1, -1):
            ref = D["reduce"][f"{kind}_{op}_{dim}"]
            if ref is None:
                continue
            dim_eff = 1 if (kind == "nv" and dim == -1) else dim
            got = getattr(ts, op)(a, dim_eff)
            assert got.shape == ref.shape, (kind, op, dim)
            if op in ("min", "max"):
                assert torch.equal(got.cpu().to(ref.dtype), ref), (kind, op, dim)
            else:
                assert torch.allclose(got.cpu().to(ref.dtype), ref, rtol=1e-12, atol=1e-12), (kind, op, dim)


def test_add_spadd_narrow_vs_reference():
    i = D["in"]
    a = _mk("v")
    b = ts.SparseTensor(row=i["rb"].to(DEV), col=i["cb"].to(DEV), value=i["vb"].to(DEV), sparse_sizes=(i["M"], i["N"]))
    c = a + b
    assert torch.equal(c.storage.row().cpu(), D["add"]["row"]) and torch.equal(c.storage.col().cpu(), D["add"]["col"])
    assert torch.allclose(c.storage.value().cpu(), D["add"]["value"], rtol=1e-12, atol=1e-12)
    idx, v = ts.spadd(torch.stack([i["ra"], i["ca"]]).to(DEV), i["va"].to(DEV), torch.stack([i["rb"], i["cb"]]).to(DEV),
                      i["vb"].to(DEV), i["M"], i["N"])
    assert torch.equal(idx.cpu(), D["spadd"]["index"])
    assert torch.allclose(v.cpu(), D["spadd"]["value"], rtol=1e-12, atol=1e-12)
    n0 = ts.narrow(a, 0, 5, 20)
    assert n0.sparse_sizes() == tuple(D["narrow0"]["sizes"])
    assert torch.equal(n0.storage.rowptr().cpu(), D["narrow0"]["rowptr"]) and torch.equal(n0.storage.col().cpu(), D["narrow0"]["col"])
    assert torch.equal(n0.storage.value().cpu(), D["narrow0"]["value"])
    n1 = ts.narrow(a, 1, 4, 15)
    assert n1.sparse_sizes() == tuple(D["narrow1"]["sizes"])
    assert torch.equal(n1.storage.row().cpu(), D["narrow1"]["row"]) and torch.equal(n1.storage.col().cpu(), D["narrow1"]["col"])
    assert torch.equal(n1.storage.value().cpu(), D["narrow1"]["value"])
    # row slice feeds SpMM directly (the multi-GPU partitioner)
    x = torch.randn(i["N"], 8, device=DEV, dtype=torch.float64)
    assert torch.allclose(n0 @ x, (a @ x)[5:25], atol=1e-12)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.int64])
@pytest.mark.parametrize("reduce", ["sum", "mean", "min", "max"])
def test_segment_reduce_vs_oracle(oracle, dtype, reduce):
    row, rowptr, col = random_csr(300, 200, 9, seed=3, power_law=True, empty_rows=(0, 5, 299), long_rows=[(7, 190)])
    g = torch.Generator().manual_seed(1)
    v = torch.randn(col.numel(), 2, generator=g)
    v = (v * 10).round().to(dtype) if dtype == torch.int64 else v.to(dtype)
    perm = torch.randperm(col.numel(), generator=g)
    for p in (None, perm):
        out = ops.segment_reduce(rowptr.to(DEV), v.to(DEV), reduce, perm=None if p is None else p.to(DEV)).cpu()
        if dtype == torch.int64 or reduce in ("min", "max"):
            assert torch.equal(out, oracle.segment_reduce(rowptr, v, reduce, perm=p))
        else:  # warp-tree summation order differs from the sequential oracle: the rounding bound
            ref, bound = segment_sum_ref_bound(oracle, rowptr, v, p, mean=reduce == "mean")
            assert_spspmm_values(out, ref, bound, f"{dtype} {reduce} perm={p is not None}")


def test_mul_vs_reference_and_gcn_flow():
    """row / column scaling (torch_sparse/mul.py:22-40) vs golden, then the GCN normalisation flow
    D^-1/2 (A) D^-1/2 X built from sum(dim) + mul + matmul against a dense computation."""
    i = D["in"]
    a = _mk("v")
    mr = ts.mul(a, D["mul"]["dr"].to(DEV))
    mc = a * D["mul"]["dc"].to(DEV)
    assert torch.equal(mr.storage.value().cpu(), D["mul"]["row_scaled"])
    assert torch.equal(mc.storage.value().cpu(), D["mul"]["col_scaled"])
    adj = ts.SparseTensor(row=i["ra"].to(DEV), col=i["ca"].to(DEV), value=i["va"].abs().to(DEV) + 0.1,
                          sparse_sizes=(i["M"], i["N"]))
    deg_r = adj.sum(dim=1).clamp(min=1e-12)
    deg_c = adj.sum(dim=0).clamp(min=1e-12)
    norm = adj.mul(deg_r.pow(-0.5).view(-1, 1)).mul(deg_c.pow(-0.5).view(1, -1))
    x = torch.randn(i["N"], 16, device=DEV, dtype=torch.float64)
    dense = adj.to_dense()
    ref = (deg_r.pow(-0.5).view(-1, 1) * dense * deg_c.pow(-0.5).view(1, -1)) @ x
    assert torch.allclose(norm @ x, ref, atol=1e-10)


# ---- §8(f) ranks 2 and 4: to_symmetric, index_select, index_select_nnz (golden: tests/golden/next_rows2.pt) ----
D2 = torch.load(Path(__file__).resolve().parent / "golden" / "next_rows2.pt", weights_only=False)


def _mk2(case, tag):
    i = case["in"]
    v = {"v": i["v"], "v2": i["v2"], "nv": None}[tag]
    return ts.SparseTensor(row=i["row"].to(DEV), col=i["col"].to(DEV), value=None if v is None else v.to(DEV),
                           sparse_sizes=(i["M"], i["N"]))


def _same(got, ref, what):
    if ref is None:
        assert got is None, what
    elif ref.dtype.is_floating_point:
        assert torch.allclose(got.cpu(), ref, rtol=1e-12, atol=1e-12), what
    else:
        assert torch.equal(got.cpu(), ref), what


@pytest.mark.parametrize("name", list(D2["cases"].keys()))
@pytest.mark.parametrize("tag", ["v", "v2", "nv"])
def test_index_select_vs_reference(name, tag):
    case = D2["cases"][name]
    i = case["in"]
    a = _mk2(case, tag)
    s0 = a.index_select(0, i["idx0"].to(DEV))
    ref = case[f"sel0_{tag}"]
    assert s0.sparse_sizes() == tuple(ref["sizes"])
    for k in ("rowptr", "row", "col", "value"):
        _same(getattr(s0.storage, k)(), ref[k], (name, tag, "sel0", k))   # indices bit-exact, values are gathered
    s1 = a.index_select(1, i["idx1"].to(DEV))
    ref = case[f"sel1_{tag}"]
    assert s1.sparse_sizes() == tuple(ref["sizes"])
    for k in ("row", "col", "value", "colptr"):
        _same(getattr(s1.storage, k)(), ref[k], (name, tag, "sel1", k))
    for lay in ("coo", "csc"):
        sn = a.index_select_nnz(i["idxe"].to(DEV), lay)
        ref = case[f"selnnz_{lay}_{tag}"]
        for k in ("row", "col", "value"):
            _same(getattr(sn.storage, k)(), ref[k], (name, tag, "selnnz", lay, k))
    # the gathered rows feed SpMM directly (mini-batch path): rows of the product are the selected rows
    if tag == "v":
        x = torch.randn(i["N"], 16, device=DEV, dtype=torch.float64)
        assert torch.allclose(s0 @ x, (a @ x)[i["idx0"].to(DEV)], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("name", list(D2["cases"].keys()))
def test_to_symmetric_vs_reference(name):
    case = D2["cases"][name]
    for tag in ("v", "v2", "nv"):
        a = _mk2(case, tag)
        for red in ("sum", "mean", "min", "max"):
            if f"sym_{red}_{tag}" not in case:
                continue
            ref = case[f"sym_{red}_{tag}"]
            s = a.to_symmetric(red)
            assert s.sparse_sizes() == tuple(ref["sizes"])
            for k in ("row", "col", "value"):
                _same(getattr(s.storage, k)(), ref[k], (name, tag, red, k))


@pytest.mark.parametrize("dtype", [torch.half, torch.float, torch.double, torch.int, torch.long, torch.bfloat16])
def test_add_and_sparse_sparse_mul_reference_cases(dtype):
    """The assertions of test/test_add.py:12-30 and test/test_mul.py:12-30, 41-57 (those tests end with a
    @torch.jit.script over SparseTensor arguments, which this package does not provide)."""
    rowA = torch.tensor([0, 0, 1, 2, 2], device=DEV)
    colA = torch.tensor([0, 2, 1, 0, 1], device=DEV)
    A = ts.SparseTensor(row=rowA, col=colA, value=torch.tensor([1, 2, 4, 1, 3], dtype=dtype, device=DEV))
    rowB = torch.tensor([0, 0, 1, 2, 2], device=DEV)
    colB = torch.tensor([1, 2, 2, 1, 2], device=DEV)
    B = ts.SparseTensor(row=rowB, col=colB, value=torch.tensor([2, 3, 1, 2, 4], dtype=dtype, device=DEV))
    r, c, v = (A + B).coo()
    assert r.tolist() == [0, 0, 0, 1, 1, 2, 2, 2] and c.tolist() == [0, 1, 2, 1, 2, 0, 1, 2]
    assert v.tolist() == [1, 2, 5, 4, 1, 1, 5, 4]
    r, c, v = (A * B).coo()
    assert r.tolist() == [0, 2] and c.tolist() == [2, 1] and v.tolist() == [6, 6]
    A1 = ts.SparseTensor(row=torch.tensor([0], device=DEV), col=torch.tensor([1], device=DEV),
                         value=torch.tensor([1], dtype=dtype, device=DEV))
    B1 = ts.SparseTensor(row=torch.tensor([1], device=DEV), col=torch.tensor([0], device=DEV),
                         value=torch.tensor([2], dtype=dtype, device=DEV))
    r, c, v = (A1 * B1).coo()
    assert r.tolist() == [] and c.tolist() == [] and v.tolist() == []


def test_dense_vector_add_mul_variants_and_getitem():
    """torch_sparse/add.py:21-37,59-104, mul.py:82-125, tensor.py:624-671 vs dense arithmetic."""
    g = torch.Generator().manual_seed(5)
    M, N = 12, 9
    dense = (torch.randn(M, N, generator=g, dtype=torch.float64) * (torch.rand(M, N, generator=g) < 0.4)).to(DEV)
    A = ts.SparseTensor.from_dense(dense)
    mask = (dense != 0).to(dense.dtype)
    r = torch.randn(M, 1, generator=g, dtype=torch.float64).to(DEV)
    c = torch.randn(1, N, generator=g, dtype=torch.float64).to(DEV)
    assert torch.allclose((A + r).to_dense(), (dense + r) * mask) and torch.allclose((c + A).to_dense(), (dense + c) * mask)
    assert torch.allclose((A * r).to_dense(), dense * r) and torch.allclose((c * A).to_dense(), dense * c)
    S = ts.SparseTensor.from_dense(dense, has_value=False)
    assert torch.allclose((S + r).to_dense(), (1 + r) * mask) and torch.allclose((S * c).to_dense(), c * mask)
    nnzv = torch.randn(A.nnz(), generator=g, dtype=torch.float64).to(DEV)
    assert torch.allclose(A.mul_nnz(nnzv).storage.value(), A.storage.value() * nnzv)
    assert torch.allclose(A.add_nnz(nnzv).storage.value(), A.storage.value() + nnzv)
    B = A.clone()
    B *= r
    B += c
    assert torch.allclose(B.to_dense(), (dense * r + c) * mask)
    # __getitem__: slices, index / bool tensors, Ellipsis
    idx = torch.tensor([3, 0, 3, 7], device=DEV)
    keep = torch.zeros(N, dtype=torch.bool, device=DEV)
    keep[[1, 4, 8]] = True
    assert torch.equal(A[2:7, :4].to_dense(), dense[2:7, :4])
    assert torch.equal(A[idx].to_dense(), dense[idx])
    assert torch.equal(A[idx, keep].to_dense(), dense[idx][:, keep])
    assert torch.equal(A[..., 2:5].to_dense(), dense[:, 2:5])
    assert torch.equal(A[5].to_dense(), dense[5:6])
    # sparse_reshape / is_symmetric / __eq__
    assert torch.equal(A.sparse_reshape(6, -1).to_dense(), dense.reshape(6, 18))
    sym = A[:9, :9].to_symmetric()
    assert sym.is_symmetric() and not A[:9, :9].is_symmetric()
    assert A == ts.SparseTensor.from_dense(dense) and A != A.set_value(A.storage.value() + 1, layout="coo")
