"""Multi-head SpMM and SDDMM (`spmm_heads`, `sddmm_heads`): per-head edge weights over [N, H, D] operands.

Kernels run through tsb200_spmm_heads / tsb200_sddmm_heads into NaN-prefilled outputs on the structured matrix `small`
(test_spmm_kernels_gpu: empty rows, rows of up to 4100 nnz, a 32-row block over the item budget) at every work-item
size (TSB200_SPMM_ITEM_SHIFT = 0 ... 5). Cases cover every row width of the vector kernels (16 B ... 2048 B and a
second column tile), several head widths per width, and the generic kernels (fp64, D = 3, an unaligned operand).

Bounds, per (row or entry, head): |out - ref64| <= 1/2 ulp_T + (n + 1) 2^-24 sum|terms|, n the number of terms; data of
multiples of 1/2 make every fp32 partial sum exact, and the result must then be fp64's rounded once, bit for bit.
"""
import os

import pytest
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import SparseTensor, ops
from pytorch_sparse_b200._lib import lib
from test_spmm_kernels_gpu import DEV, assert_bits_equal, assert_sum_bound, small  # noqa: F401

pytestmark = pytest.mark.gpu
ENV = "TSB200_SPMM_ITEM_SHIFT"
U32 = 2.0 ** -24
U64 = 2.0 ** -52
BF, F16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64

# (dtype, H, D): row widths 16 B ... 4096 B (two column tiles for SpMM), several head widths per width; SDDMM row-wise
# kernels up to 64 vectors with HL = D * size / 16 a power of two, and generic cases
CASES = [(BF, 1, 8), (F32, 1, 4), (BF, 2, 8), (F32, 2, 4), (BF, 4, 8), (F32, 4, 4), (F16, 2, 16),
         (BF, 8, 8), (BF, 4, 16), (F32, 2, 16), (F32, 8, 4),
         (BF, 1, 128), (BF, 2, 64), (BF, 8, 16), (BF, 16, 8), (F16, 4, 32), (F32, 8, 8),
         (BF, 4, 64), (F32, 4, 32), (BF, 1, 256),
         (BF, 8, 64), (F16, 2, 256), (F32, 16, 16),
         (BF, 16, 64), (F32, 4, 128), (BF, 32, 64), (F32, 8, 128),
         (F64, 2, 8), (F32, 4, 3), (F16, 3, 8)]


def _id(c):
    return f"{str(c[0]).split('.')[-1]}-H{c[1]}-D{c[2]}"


def coo_row(rowptr):
    return torch.repeat_interleave(torch.arange(rowptr.numel() - 1), rowptr[1:] - rowptr[:-1])


def operands(shape, dtype, g, exact):
    if exact:
        return (torch.randint(-4, 5, shape, generator=g).double() / 2).to(dtype)
    return torch.randn(shape, generator=g, dtype=torch.float64).to(dtype)


def spmm_ref(rowptr, col, value, x):
    """fp64 sum and sum of |terms| per (row, head, column), and the row degrees."""
    row = coo_row(rowptr)
    M = rowptr.numel() - 1
    xv = x.double()[col]
    v = value.double()[:, :, None] if value is not None else torch.ones(col.numel(), x.size(1), 1, dtype=F64)
    ref = torch.zeros((M,) + tuple(x.shape[1:]), dtype=F64).index_add_(0, row, xv * v)
    S = torch.zeros_like(ref).index_add_(0, row, (xv * v).abs())
    return ref, S, (rowptr[1:] - rowptr[:-1]).double()[:, None, None]


def sddmm_ref(rowptr, col, a, b):
    row = coo_row(rowptr)
    p = a.double()[row] * b.double()[col]
    return p.sum(-1), p.abs().sum(-1)


def call_spmm(rowptr, col, value, x, M, plan=None):
    N, H, D = x.shape
    out = torch.full((M, H, D), float("nan"), dtype=x.dtype, device=DEV)
    dt = ops._dtype_code(x.dtype)
    E = col.numel()
    if plan is not None:
        nws = lib.tsb200_spmm_fw_planned_workspace_bytes(H * D, plan.n_long, plan.n_slot, 0)
        pl = (ops._p(plan.data), plan.data.numel(), plan.n_seg, plan.n_long, plan.n_slot)
    else:
        nws = lib.tsb200_spmm_fw_workspace_bytes(1, M, H * D, E, dt, 0)
        pl = (None, 0, 0, 0, 0)
    ws = torch.empty(max(nws, 1), dtype=torch.uint8, device=DEV)
    rc = lib.tsb200_spmm_heads(ops._p(rowptr), ops._p(col), ops._p(value), ops._p(x), ops._p(out), M, N, H, D, E,
                               dt, *pl, ops._p(ws), nws, ops._stream(torch.device(DEV)))
    assert rc == 0, rc
    return out


def call_sddmm(rowptr, col, a, b):
    M, H, D = a.shape
    N, E = b.size(0), col.numel()
    out = torch.full((E, H), float("nan"), dtype=a.dtype, device=DEV)
    dt = ops._dtype_code(a.dtype)
    nws = lib.tsb200_spmm_value_bw_workspace_bytes(1, M, H * D, E, dt)
    ws = torch.empty(max(nws, 1), dtype=torch.uint8, device=DEV)
    rc = lib.tsb200_sddmm_heads(ops._p(rowptr), ops._p(col), ops._p(a), ops._p(b), ops._p(out), M, N, H, D, E, dt,
                                ops._p(ws), nws, ops._stream(torch.device(DEV)))
    assert rc == 0, rc
    return out


def unaligned(t):
    """the same values at an address 2 elements off a 16-byte boundary"""
    buf = torch.empty(t.numel() + 2, dtype=t.dtype, device=DEV)
    v = buf[2:].view(t.shape)
    v.copy_(t)
    return v


@pytest.mark.parametrize("case", CASES, ids=_id)
def test_kernels_every_item_size(small, monkeypatch, case):
    dtype, H, D = case
    rowptr_c, col_c, M, N = small["rowptr"], small["col"], small["M"], small["N"]
    E = col_c.numel()
    rowptr, col = rowptr_c.to(DEV), col_c.to(DEV)
    u = U64 if dtype == F64 else U32
    for exact in (True, False):
        g = torch.Generator().manual_seed(H * 1000 + D + exact)
        x_c, v_c = operands((N, H, D), dtype, g, exact), operands((E, H), dtype, g, exact)
        a_c = operands((M, H, D), dtype, g, exact)
        x, v, a = x_c.to(DEV), v_c.to(DEV), a_c.to(DEV)
        if dtype == F16 and H == 3:    # 16-byte heads at an unaligned address: the generic kernels
            x, a = unaligned(x), unaligned(a)
        ref, S, deg = spmm_ref(rowptr_c, col_c, v_c, x_c)
        ref1, S1, _ = spmm_ref(rowptr_c, col_c, None, x_c)
        dref, dS = sddmm_ref(rowptr_c, col_c, a_c, x_c)
        results = []
        for s in range(6):
            monkeypatch.setenv(ENV, str(s))
            out = call_spmm(rowptr, col, v, x, M)
            out1 = call_spmm(rowptr, col, None, x, M)
            sc = call_sddmm(rowptr, col, a, x)
            what = f"{_id(case)} shift {s} exact={exact}"
            if exact:
                assert_bits_equal(out, ref.to(dtype), "spmm_heads " + what)
                assert_bits_equal(out1, ref1.to(dtype), "spmm_heads no value " + what)
                assert_bits_equal(sc, dref.to(dtype), "sddmm_heads " + what)
            else:
                assert_sum_bound(out, ref, S, deg + 1, dtype, u=u, what="spmm_heads " + what)
                assert_sum_bound(out1, ref1, S1, deg + 1, dtype, u=u, what="spmm_heads no value " + what)
                assert_sum_bound(sc, dref, dS, D + 1, dtype, u=u, what="sddmm_heads " + what)
            results.append((out, sc))
        # a dot is formed by one lane group whatever the item size; so is a row sum over rows wider than 128 bytes
        for out, sc in results[1:]:
            if H * D * x.element_size() > 128:
                assert_bits_equal(out, results[0][0], "spmm_heads across item sizes " + _id(case))
            assert_bits_equal(sc, results[0][1], "sddmm_heads across item sizes " + _id(case))


@pytest.mark.parametrize("case", [c for c in CASES if c[0] != F64 and (c[2] * c[0].itemsize) % 16 == 0
                                  and c[1] * c[2] * c[0].itemsize > 128], ids=_id)
def test_planned_equals_unplanned(small, case):
    dtype, H, D = case
    rowptr, col, M, N = small["rowptr"].to(DEV), small["col"].to(DEV), small["M"], small["N"]
    g = torch.Generator().manual_seed(7)
    x = operands((N, H, D), dtype, g, False).to(DEV)
    v = operands((col.numel(), H), dtype, g, False).to(DEV)
    plan = ops.spmm_plan(rowptr, col.numel())
    assert_bits_equal(call_spmm(rowptr, col, v, x, M, plan), call_spmm(rowptr, col, v, x, M), "planned " + _id(case))


@pytest.mark.parametrize("dtype,K", [(BF, 8), (BF, 64), (BF, 128), (F16, 256), (F32, 32), (BF, 1024), (F32, 1024),
                                     (F32, 6), (F64, 16)])
def test_one_head_is_the_single_head_operator(small, monkeypatch, dtype, K):
    monkeypatch.setenv("TSB200_AUTO_PLAN", "0")    # both unplanned (narrow rows may differ between the two paths)
    rowptr, col, M, N = small["rowptr"].to(DEV), small["col"].to(DEV), small["M"], small["N"]
    row = coo_row(small["rowptr"]).to(DEV)
    g = torch.Generator().manual_seed(K)
    x = operands((N, K), dtype, g, False).to(DEV)
    a = operands((M, K), dtype, g, False).to(DEV)
    v = operands((col.numel(),), dtype, g, False).to(DEV)
    for s in range(6):
        monkeypatch.setenv(ENV, str(s))
        with torch.no_grad():
            assert_bits_equal(call_spmm(rowptr, col, v[:, None], x[:, None], M)[:, 0],
                              ops.spmm_fw(rowptr, col, v, x, "sum")[0], f"spmm H=1 K={K}")
            vecs = K * x.element_size() // 16
            if (K * x.element_size()) % 16 == 0 and 4 <= vecs <= 32 and vecs & (vecs - 1) == 0:
                assert_bits_equal(call_sddmm(rowptr, col, a[:, None], x[:, None])[:, 0],
                                  ops.spmm_value_bw(row, rowptr, col, x, a, "sum"), f"sddmm H=1 K={K}")


def test_empty_extents():
    rowptr = torch.zeros(4, dtype=torch.int64, device=DEV)
    col = torch.zeros(0, dtype=torch.int64, device=DEV)
    x = torch.randn(5, 2, 8, device=DEV)
    assert torch.equal(call_spmm(rowptr, col, torch.zeros(0, 2, device=DEV), x, 3), torch.zeros(3, 2, 8, device=DEV))
    assert call_sddmm(rowptr, col, torch.randn(3, 2, 8, device=DEV), x).shape == (0, 2)
    empty_m = torch.zeros(1, dtype=torch.int64, device=DEV)
    assert call_spmm(empty_m, col, None, x, 0).shape == (0, 2, 8)
    rp = torch.tensor([0, 2, 3], device=DEV)
    c = torch.tensor([0, 4, 1], device=DEV)
    assert call_spmm(rp, c, torch.zeros(3, 0, device=DEV), torch.zeros(5, 0, 8, device=DEV), 2).shape == (2, 0, 8)
    assert call_sddmm(rp, c, torch.zeros(2, 0, 8, device=DEV), torch.zeros(5, 0, 8, device=DEV)).shape == (3, 0)
    torch.cuda.synchronize()


# ---- autograd ---------------------------------------------------------------------------------------------------
def random_src(M, N, deg, seed, dtype=None, H=None):
    g = torch.Generator().manual_seed(seed)
    E = M * deg
    row = torch.randint(0, M, (E,), generator=g)
    col = torch.randint(0, N, (E,), generator=g)
    row[: M // 4] = col[: M // 4] % M     # a few repeated columns (hub columns in the CSC view)
    col[: E // 3] = torch.randint(0, 4, (E // 3,), generator=g)
    src = SparseTensor(row=row.to(DEV), col=col.to(DEV), sparse_sizes=(M, N))
    return src


def gather_spmm(src, value, x):
    row, col, _ = src.coo()
    out = torch.zeros((src.size(0),) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    return out.index_add(0, row, x[col] * value[..., None])


def gather_sddmm(src, a, b):
    row, col, _ = src.coo()
    return (a[row] * b[col]).sum(-1)


@pytest.mark.parametrize("dtype,H,D", [(BF, 8, 16), (F32, 4, 8), (F16, 2, 64), (F32, 3, 3)])
@pytest.mark.parametrize("want", ["value", "x", "both"])
def test_spmm_heads_gradients(dtype, H, D, want):
    src = random_src(300, 200, 6, H * D)
    E = src.nnz()
    g = torch.Generator().manual_seed(3)
    x0 = torch.randn(200, H, D, generator=g, dtype=F64)
    v0 = torch.randn(E, H, generator=g, dtype=F64)
    go = torch.randn(300, H, D, generator=g, dtype=F64).to(dtype).to(DEV)
    x = x0.to(dtype).to(DEV).requires_grad_(want != "value")
    v = v0.to(dtype).to(DEV).requires_grad_(want != "x")
    out = src.set_value(v, layout="csr").spmm_heads(x)
    out.backward(go)
    go = go.double()
    xr, vr = x.detach().double().requires_grad_(), v.detach().double().requires_grad_()
    ref = gather_spmm(src, vr, xr)
    ref.backward(go)
    row, col, _ = src.coo()
    deg = torch.bincount(col, minlength=200).double()
    if want != "x":
        S = (go[row].abs() * x.detach().double()[col].abs()).sum(-1)
        assert_sum_bound(v.grad, vr.grad.cpu(), S.cpu(), D + 1, dtype, what="grad value")
    else:
        assert v.grad is None
    if want != "value":
        S = torch.zeros(200, H, D, dtype=F64, device=DEV).index_add_(
            0, col, (v.detach().double()[..., None] * go[row]).abs())
        assert_sum_bound(x.grad, xr.grad.cpu(), S.cpu(), (deg.max() + 1).item(), dtype, what="grad x")
    else:
        assert x.grad is None


@pytest.mark.parametrize("dtype,H,D", [(BF, 8, 16), (F32, 4, 8), (F16, 2, 64), (F32, 3, 3)])
@pytest.mark.parametrize("want", ["a", "b", "both"])
def test_sddmm_heads_gradients(dtype, H, D, want):
    src = random_src(300, 200, 6, H * D + 1)
    g = torch.Generator().manual_seed(4)
    a0 = torch.randn(300, H, D, generator=g, dtype=F64)
    b0 = torch.randn(200, H, D, generator=g, dtype=F64)
    go = torch.randn(src.nnz(), H, generator=g, dtype=F64).to(dtype).to(DEV)
    a = a0.to(dtype).to(DEV).requires_grad_(want != "b")
    b = b0.to(dtype).to(DEV).requires_grad_(want != "a")
    s = ts.sddmm_heads(src, a, b)
    s.backward(go)
    go = go.double()
    ar, br = a.detach().double().requires_grad_(), b.detach().double().requires_grad_()
    gather_sddmm(src, ar, br).backward(go)
    row, col, _ = src.coo()
    if want != "b":
        S = torch.zeros(300, H, D, dtype=F64, device=DEV).index_add_(0, row, (go[..., None] * br.detach()[col]).abs())
        n = torch.bincount(row, minlength=300).max().item() + 1
        assert_sum_bound(a.grad, ar.grad.cpu(), S.cpu(), n, dtype, what="grad a")
    if want != "a":
        S = torch.zeros(200, H, D, dtype=F64, device=DEV).index_add_(0, col, (go[..., None] * ar.detach()[row]).abs())
        n = torch.bincount(col, minlength=200).max().item() + 1
        assert_sum_bound(b.grad, br.grad.cpu(), S.cpu(), n, dtype, what="grad b")


def test_gradcheck_fp64():
    src = random_src(20, 15, 3, 1)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(15, 2, 3, generator=g, dtype=F64).to(DEV).requires_grad_()
    v = torch.randn(src.nnz(), 2, generator=g, dtype=F64).to(DEV).requires_grad_()
    a = torch.randn(20, 2, 3, generator=g, dtype=F64).to(DEV).requires_grad_()
    assert torch.autograd.gradcheck(lambda v, x: src.set_value(v, layout="csr").spmm_heads(x), (v, x))
    assert torch.autograd.gradcheck(lambda a, x: src.sddmm_heads(a, x), (a, x))


def test_value_gradient_builds_no_csc_view():
    src = random_src(100, 80, 4, 9)
    x = torch.randn(80, 2, 8, device=DEV)
    v = torch.randn(src.nnz(), 2, device=DEV, requires_grad=True)
    adj = src.set_value(v, layout="csr")
    adj.spmm_heads(x).sum().backward()
    st = adj.storage
    assert st._csr2csc is None and st._colptr is None
    assert v.grad is not None


@pytest.mark.parametrize("dtype", [F32, BF])
def test_readme_attention_layer(dtype):
    M, H, D = 200, 4, 16
    adj = random_src(M, M, 5, 11)
    g = torch.Generator().manual_seed(6)
    q0, k0, v0 = (torch.randn(M, H, D, generator=g, dtype=F64) for _ in range(3))
    q, k, v = (t.to(dtype).to(DEV).requires_grad_() for t in (q0, k0, v0))

    row = adj.storage.row()
    s = adj.sddmm_heads(q, k) * D ** -0.5                       # [E, H]
    m = adj.set_value(s.detach(), layout="csr").max(dim=1)      # [M, H], native segment max
    p = (s - m[row]).exp()
    alpha = p / adj.set_value(p, layout="csr").sum(dim=1)[row]  # row softmax per head
    out = adj.set_value(alpha, layout="csr").spmm_heads(v)      # [M, H, D]
    go = torch.randn(M, H, D, generator=g, dtype=F64).to(DEV)
    out.backward(go.to(dtype))

    # dense masked multi-head attention in fp64; duplicate entries count once per stored entry
    qr, kr, vr = (t.detach().double().requires_grad_() for t in (q, k, v))
    r, c, _ = adj.coo()
    cnt = torch.zeros(M, M, dtype=F64, device=DEV).index_put_((r, c), torch.ones_like(r, dtype=F64), accumulate=True)
    logits = torch.einsum("mhd,nhd->hmn", qr, kr) * D ** -0.5
    logits = logits + cnt.log()                                 # -inf off the structure, log(multiplicity) on it
    has = cnt.sum(1) > 0
    att = torch.softmax(logits[:, has], dim=-1)
    ref = torch.einsum("hmn,nhd->mhd", att, vr)
    ref.backward(go[has])
    tol = 2e-2 if dtype == BF else 1e-4
    torch.testing.assert_close(out[has].double(), ref, atol=tol, rtol=tol)
    for t, tr in ((q, qr), (k, kr), (v, vr)):
        torch.testing.assert_close(t.grad.double(), tr.grad, atol=5 * tol, rtol=5 * tol)


def test_forward_peak_allocation():
    src = random_src(4000, 4000, 8, 13)
    H, D = 8, 16
    x = torch.randn(4000, H, D, device=DEV, dtype=BF)
    v = torch.randn(src.nnz(), H, device=DEV, dtype=BF)
    adj = src.set_value(v, layout="csr")
    a = torch.randn(4000, H, D, device=DEV, dtype=BF)
    for _ in range(3):    # builds the cached plan and CSR views
        adj.spmm_heads(x)
        adj.sddmm_heads(a, x)
    E = src.nnz()
    for fn, out_bytes, ws in ((lambda: adj.spmm_heads(x), 4000 * H * D * 2,
                               lib.tsb200_spmm_fw_workspace_bytes(1, 4000, H * D, E, 3, 0)),
                              (lambda: adj.sddmm_heads(a, x), E * H * 2,
                               lib.tsb200_spmm_value_bw_workspace_bytes(1, 4000, H * D, E, 3))):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        y = fn()
        torch.cuda.synchronize()
        assert torch.cuda.max_memory_allocated() - base <= out_bytes + ws + (1 << 20)
        del y
    assert os.environ.get("TSB200_AUTO_PLAN", "1") == "1"
