"""Softmax-aggregation SpMM (tsb200_spmm_fw_softmax_aggr, `spmm_softmax_aggr`) and its backward on the H100.

Forward calls go through the C ABI into NaN-prefilled outputs between guard zones, with a guarded workspace of exactly
the stated size, and every const input is compared before and after: an element a kernel fails to write, a write
outside an output or the workspace, or a write to an input cannot pass.

Error bound of the forward (test_random_within_bound). The reference is the definition in fp64 over the messages p
as the kernels form them (p = fl(v x): exact for bf16 / f16, rounded once in fp32 for f32). Per row and column, with n
the degree, u the unit roundoff of the accumulator (2^-24; 2^-53 for fp64), Y = max_e |t p_e| and P = max_e |p_e|:
  * y = fl(t p), y - mu and the log2(e) scaling each round once, so every exp argument is off by at most 3 u (|y| +
    |mu|) <= 6 u Y in absolute terms; ex2.approx adds a relative error of at most 2^-22 (fp64 exp: 2^-52).
    Each weight is also multiplied by at most n rescale factors with the same errors, so every weight carries a
    relative error of at most d = (n + 1) (2^-22 + 6 u Y) (fp64: 2^-52 + 6 u Y), to first order.
  * s and a are sums of n non-negative weights and of n terms |w p| <= w P: each is off by at most n u of its
    magnitude, plus one rounding per rescale and merge (another n u).
  * a / s with weights of relative error d moves by at most 2 d P; the sums' errors move it by at most 4 n u P; the
    division rounds once (u). Then the result is rounded once to T (u_T |z|).
So |out - ref| <= u_T |ref| + (1 + u_T) B with B = 2 d P + 4 (n + 1) u P + u |ref|; the test allows 2 B, plus
2^-25 for f16, whose subnormal results (below 2^-14) round to a spacing of 2^-24.
"""
import ctypes
import importlib

import pytest
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import ops
from pytorch_sparse_b200._lib import lib
from test_spmm_kernels_gpu import build_csr
from test_spmm_multi_gpu import _guard_ok, _guarded, _power_law, call_spmm
from test_spmm_res_gpu import ROW_BYTES, _id, _stream, _vp

tsm = importlib.import_module("pytorch_sparse_b200.matmul")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FLOATS = (torch.bfloat16, torch.float16, torch.float32)
MEAN = 1
UT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 2.0 ** -24, torch.float64: 2.0 ** -53}
WS_GUARD = 256 * 16


@pytest.fixture(scope="module")
def mat():
    """Empty rows, rows of 1 ... 1300 nnz (segments past 256 and the combine), a 32-row block over the item budget."""
    M, N = 32 * 40 + 13, 3000
    specials = {5: 1, 37: 31, 38: 32, 39: 33, 200: 255, 201: 256, 202: 257, 500: 512, 501: 513, 900: 1300}
    rowptr, col = build_csr(M, N, 4, 11, specials, blocks=[64], tie_rows={300: 40, 301: 600},
                            empty_rows=(0, M // 2, M - 1))
    return dict(M=M, N=N, rowptr=rowptr, col=col)


def _acc(dtype):
    return torch.float64 if dtype == torch.float64 else torch.float32


def call_smx(rowptr, col, value, x, t, plan=None, want_lse=True):
    """tsb200_spmm_fw_softmax_aggr into NaN-prefilled, guarded outputs and a guarded workspace of exactly the stated
    size; the inputs must come back unchanged. Returns (out, lse)."""
    M, E = rowptr.numel() - 1, col.numel()
    N, K = x.shape
    dt = ops._DTYPES[x.dtype]
    ob, out = _guarded((M, K), x.dtype, float("nan"))
    lb, lse = _guarded((M, K), _acc(x.dtype), float("nan")) if want_lse else (None, None)
    if plan is None:
        pl, nws = (None, 0, 0, 0, 0), lib.tsb200_spmm_fw_softmax_aggr_workspace_bytes(K, E, 0, 0, 0)
    else:
        pl = (_vp(plan.data), plan.data.numel(), plan.n_seg, plan.n_long, plan.n_slot)
        nws = lib.tsb200_spmm_fw_softmax_aggr_workspace_bytes(K, E, 1, plan.n_long, plan.n_slot)
    wb = torch.full((nws + 2 * WS_GUARD,), 0xA5, dtype=torch.uint8, device=DEV)
    ws = wb[WS_GUARD:WS_GUARD + nws]
    inputs = [a.clone() for a in (rowptr, col, value, x, t) if a is not None]
    plan_in = plan.data.clone() if plan is not None else None
    stride = 0 if t.numel() == 1 else 1
    rc = lib.tsb200_spmm_fw_softmax_aggr(_vp(rowptr), _vp(col), _vp(value), _vp(x), _vp(t), stride, _vp(out),
                                         _vp(lse), M, N, K, E, dt, *pl, _vp(ws) if nws else None, nws, _stream())
    assert rc == 0, rc
    torch.cuda.synchronize()
    assert _guard_ok(ob, float("nan")), "write before / after out"
    assert lb is None or _guard_ok(lb, float("nan")), "write before / after lse"
    assert (wb[:WS_GUARD] == 0xA5).all() and (wb[WS_GUARD + nws:] == 0xA5).all(), "write outside the workspace"
    for a, b in zip(inputs, [a for a in (rowptr, col, value, x, t) if a is not None]):
        assert torch.equal(_bits(a), _bits(b)), "a const input changed"
    assert plan is None or torch.equal(plan_in, plan.data), "the plan changed"
    return out, lse


def _operands(m, dtype, K, with_value, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(m["N"], K, generator=g) * scale).to(dtype).to(DEV)
    v = (torch.rand(m["col"].numel(), generator=g) * 2 - 0.5).to(dtype).to(DEV) if with_value else None
    return m["rowptr"].to(DEV), m["col"].to(DEV), v, x


def _bits(a):
    return a.view(torch.int16 if a.element_size() == 2 else torch.int32 if a.element_size() == 4 else torch.int64)


def assert_t0_is_mean(rowptr, col, v, x, plan):
    t = torch.zeros((), dtype=_acc(x.dtype), device=DEV)
    out, lse = call_smx(rowptr, col, v, x, t, plan)
    ref, _ = call_spmm(rowptr, col, v, x, MEAN, plan)
    assert torch.equal(_bits(out), _bits(ref))
    deg = (rowptr[1:] - rowptr[:-1]).to(lse.dtype)[:, None]
    torch.testing.assert_close(lse, deg.log().expand_as(lse), msg="lse of t = 0 is log(degree)")


def _t0_cases():
    for rb in ROW_BYTES:
        for dtype in FLOATS:
            for with_value in (True, False):
                if dtype == torch.float32 and with_value:
                    continue   # p is rounded before it is summed: not spmm's fused product
                yield rb, dtype, with_value


@pytest.mark.parametrize("planned", [False, True])
@pytest.mark.parametrize("row_bytes,dtype,with_value", list(_t0_cases()), ids=_id)
def test_t0_is_mean_bitwise(mat, monkeypatch, row_bytes, dtype, with_value, planned):
    monkeypatch.setenv("TSB200_SPMM_ITEM_SHIFT", "5")   # the same work items as the mean kernels
    esz = torch.tensor([], dtype=dtype).element_size()
    rowptr, col, v, x = _operands(mat, dtype, row_bytes // esz, with_value)
    assert_t0_is_mean(rowptr, col, v, x, ops.spmm_plan(rowptr, col.numel()) if planned else None)


@pytest.mark.parametrize("shift", range(6))
@pytest.mark.parametrize("K", [8, 64, 128, 512])
def test_t0_is_mean_every_item_size(mat, monkeypatch, shift, K):
    monkeypatch.setenv("TSB200_SPMM_ITEM_SHIFT", str(shift))
    rowptr, col, v, x = _operands(mat, torch.bfloat16, K, True, seed=shift)
    assert_t0_is_mean(rowptr, col, v, x, None)
    assert_t0_is_mean(rowptr, col, v, x, ops.spmm_plan(rowptr, col.numel()))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=_id)
@pytest.mark.parametrize("K", [16, 128])
def test_t0_is_mean_power_law(dtype, K):
    m = _power_law(20000, 5000, seed=7)
    rowptr, col, v, x = _operands(m, dtype, K, True)
    assert_t0_is_mean(rowptr, col, v, x, None)
    assert_t0_is_mean(rowptr, col, v, x, ops.spmm_plan(rowptr, col.numel()))


def reference(rowptr, col, v, x, t):
    """(out, lse, B) in fp64 by the definition over the messages as the kernels form them, and the bound B of the
    module docstring (without the final rounding to T)."""
    xd, M = x.double().cpu(), rowptr.numel() - 1
    rp, colc = rowptr.cpu(), col.cpu()
    vd = v.double().cpu() if v is not None else torch.ones(col.numel(), dtype=torch.float64)
    row = torch.repeat_interleave(torch.arange(M), rp[1:] - rp[:-1])
    p = xd[colc] * vd[:, None]
    if x.dtype == torch.float32:
        p = p.float().double()
    y = t.double().cpu() * p
    K = x.size(1)
    mu = torch.full((M, K), float("-inf"), dtype=torch.float64).index_reduce_(0, row, y, "amax")
    w = torch.exp(y - mu[row])
    s = torch.zeros(M, K, dtype=torch.float64).index_add_(0, row, w)
    a = torch.zeros_like(s).index_add_(0, row, w * p)
    n = (rp[1:] - rp[:-1]).double()[:, None]
    out = torch.where(n > 0, a / s, torch.zeros_like(a))
    lse = mu + s.log()
    P = torch.zeros_like(s).index_reduce_(0, row, p.abs(), "amax")
    Y = torch.zeros_like(s).index_reduce_(0, row, y.abs(), "amax")
    u = 2.0 ** -53 if x.dtype == torch.float64 else 2.0 ** -24
    ex = 2.0 ** -52 if x.dtype == torch.float64 else 2.0 ** -22
    d = (n + 1) * (ex + 6 * u * Y)
    B = 2 * d * P + 4 * (n + 1) * u * P + u * out.abs()
    return out, lse, B


def assert_within_bound(out, ref, B, dtype):
    got = out.double().cpu()
    uT = UT[dtype]
    sub = 2.0 ** -25 if dtype == torch.float16 else 0   # f16 results below 2^-14 round to a spacing of 2^-24
    bound = uT * ref.abs() + (1 + uT) * 2 * B + sub
    bad = ~((got - ref).abs() <= bound)
    assert not bad.any(), f"{int(bad.sum())} elements outside the bound, worst {((got - ref).abs() - bound).max()}"


T_KINDS = ["scalar", "channel", "negative"]


def _t(kind, K, dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    acc = _acc(dtype)
    if kind == "scalar":
        return torch.tensor(1.7, dtype=acc, device=DEV)
    if kind == "negative":
        return torch.tensor([-2.5], dtype=acc, device=DEV)
    return (torch.rand(K, generator=g) * 6 - 2).to(acc).to(DEV)


@pytest.mark.parametrize("planned", [False, True])
@pytest.mark.parametrize("t_kind", T_KINDS)
@pytest.mark.parametrize("dtype", FLOATS + (torch.float64,), ids=_id)
@pytest.mark.parametrize("row_bytes", ROW_BYTES)
def test_random_within_bound(mat, row_bytes, dtype, t_kind, planned):
    esz = torch.tensor([], dtype=dtype).element_size()
    if row_bytes % esz:
        pytest.skip("not a whole number of elements")
    K = row_bytes // esz
    rowptr, col, v, x = _operands(mat, dtype, K, True, seed=K)
    t = _t(t_kind, K, dtype, seed=K)
    plan = ops.spmm_plan(rowptr, col.numel()) if planned else None
    out, lse = call_smx(rowptr, col, v, x, t, plan)
    ref, ref_lse, B = reference(rowptr, col, v, x, t)
    assert not out.isnan().any() and not lse.isnan().any()
    assert_within_bound(out, ref, B, dtype)
    fin = ref_lse.isfinite()
    assert torch.equal(lse.cpu().isinf(), ~fin)
    torch.testing.assert_close(lse.double().cpu()[fin], ref_lse[fin], rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("t_kind", T_KINDS)
@pytest.mark.parametrize("case", ["fp64", "odd_k", "unaligned", "e0"])
def test_generic_path_within_bound(mat, case, t_kind):
    dtype = torch.float64 if case == "fp64" else torch.float32
    K = 13 if case == "odd_k" else 32
    rowptr, col, v, x = _operands(mat, dtype, K, True)
    if case == "unaligned":     # the dense operand 4 bytes past a 16-byte boundary
        xb = torch.empty(x.numel() + 1, dtype=dtype, device=DEV)
        xu = xb[1:].view(x.shape)
        xu.copy_(x)
        x = xu
    if case == "e0":
        rowptr, col, v = torch.zeros_like(rowptr), col[:0], v[:0]
    t = _t(t_kind, K, dtype)
    out, lse = call_smx(rowptr, col, v, x, t)
    ref, _, B = reference(rowptr, col, v, x, t)
    assert_within_bound(out, ref, B, dtype)
    if case == "e0":
        assert (out == 0).all() and (lse == float("-inf")).all()


@pytest.mark.parametrize("dtype", FLOATS + (torch.float64,), ids=_id)
@pytest.mark.parametrize("K", [8, 128])
def test_one_entry_and_empty_rows_exact(mat, dtype, K):
    rowptr, col, v, x = _operands(mat, dtype, K, True, seed=3)
    t = _t("channel", K, dtype)
    out, lse = call_smx(rowptr, col, v, x, t)
    deg = (rowptr[1:] - rowptr[:-1]).cpu()
    one = torch.nonzero(deg == 1).flatten()
    empty = torch.nonzero(deg == 0).flatten()
    assert one.numel() > 0 and empty.numel() > 0
    e = rowptr.cpu()[one]
    p = x.to(_acc(dtype)).cpu()[col.cpu()[e]] * v.to(_acc(dtype)).cpu()[e, None]
    assert torch.equal(out.cpu()[one], p.to(dtype))
    assert torch.equal(lse.cpu()[one], t.cpu() * p)
    assert (out.cpu()[empty] == 0).all() and (lse.cpu()[empty] == float("-inf")).all()


def test_nan_propagates(mat):
    rowptr, col, v, x = _operands(mat, torch.bfloat16, 64, True, seed=4)
    x[int(col[1000]), 3] = float("nan")
    t = _t("channel", 64, torch.bfloat16)
    t[9] = float("nan")
    out, _ = call_smx(rowptr, col, v, x, t)
    rowc = torch.repeat_interleave(torch.arange(mat["M"], device=DEV), rowptr[1:] - rowptr[:-1])
    hit = torch.zeros(mat["M"], dtype=torch.bool, device=DEV)
    hit[rowc[col == int(col[1000])]] = True
    deg = rowptr[1:] - rowptr[:-1]
    assert torch.equal(out[:, 3].isnan(), hit)
    assert torch.equal(out[:, 9].isnan(), deg > 0)
    others = torch.ones(64, dtype=torch.bool)
    others[[3, 9]] = False
    assert not out[:, others.to(DEV)].isnan().any()


def test_row_far_below_the_global_max():
    """A row whose messages lie near -200 while the column's global max is near +200: the fused result is finite and
    within the bound; the global-shift composition spmm(A, e * x) / spmm(A, e) with e = exp(t x - max_k t x) gives
    0 / 0 = NaN there."""
    M, N, K = 4, 64, 16
    g = torch.Generator().manual_seed(5)
    x = torch.randn(N, K, generator=g)
    x[:32] += 200
    x[32:] -= 200
    rowptr = torch.tensor([0, 32, 64, 70, 80])
    col = torch.cat([torch.arange(32), torch.arange(32, 64), torch.arange(26, 32), torch.arange(40, 50)])
    rowptr, col, x = rowptr.to(DEV), col.to(DEV), x.to(DEV)
    t = torch.tensor(1.0, device=DEV)
    out, _ = call_smx(rowptr, col, None, x, t)
    ref, _, B = reference(rowptr, col, None, x, t)
    assert out.isfinite().all()
    assert_within_bound(out, ref, B, torch.float32)
    A = ts.SparseTensor(rowptr=rowptr, col=col, sparse_sizes=(M, N))
    e = torch.exp(t * x - (t * x).amax(0))
    shifted = tsm.spmm_sum(A, e * x) / tsm.spmm_sum(A, e)
    assert shifted[1].isnan().all() and shifted[3].isnan().all()
    assert shifted[0].isfinite().all()


# ---- gradients --------------------------------------------------------------------------------------------------------
def definition(rowptr, col, value, x, t):
    """The forward by its definition in torch (fp64 autograd): per row the softmax of t p over the entries, per column."""
    M = rowptr.numel() - 1
    row = torch.repeat_interleave(torch.arange(M, device=x.device), rowptr[1:] - rowptr[:-1])
    p = x[col] * (value[:, None] if value is not None else 1)
    y = t * p
    mu = torch.full((M, x.size(1)), float("-inf"), dtype=x.dtype, device=x.device)
    mu = mu.index_reduce(0, row, y.detach(), "amax")
    w = torch.exp(y - mu[row])
    s = torch.zeros(M, x.size(1), dtype=x.dtype, device=x.device).index_add(0, row, w)
    a = torch.zeros_like(s).index_add(0, row, w * p)
    return torch.where(s > 0, a / s.clamp(min=1e-300), torch.zeros_like(a))


def _graph(seed, M=300, N=200, K=32, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    deg = torch.randint(0, 12, (M,), generator=g)
    deg[7] = 700   # a row the forward cuts into segments
    rowptr = torch.cat([torch.zeros(1, dtype=torch.long), deg.cumsum(0)])
    col = torch.randint(N, (int(rowptr[-1]),), generator=g)
    value = torch.rand(col.numel(), generator=g, dtype=torch.float64) + 0.5
    x = torch.randn(N, K, generator=g, dtype=torch.float64)
    return rowptr.to(DEV), col.to(DEV), value.to(dtype).to(DEV), x.to(dtype).to(DEV)


@pytest.mark.parametrize("t_kind", ["scalar", "channel"])
@pytest.mark.parametrize("wrt", [("x",), ("v",), ("t",), ("x", "v", "t")])
def test_gradients_match_fp64_definition(t_kind, wrt):
    rowptr, col, value, x = _graph(11)
    M, N, K = rowptr.numel() - 1, x.size(0), x.size(1)
    t0 = torch.tensor(0.8, device=DEV) if t_kind == "scalar" else torch.linspace(-1.5, 2.0, K, device=DEV)
    v1 = value.clone().requires_grad_("v" in wrt)
    A = ts.SparseTensor(rowptr=rowptr, col=col, value=v1, sparse_sizes=(M, N))
    x1 = x.clone().requires_grad_("x" in wrt)
    t1 = t0.clone().requires_grad_("t" in wrt)
    out = tsm.spmm_softmax_aggr(A, x1, t1)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
    leaves = {"x": x1, "v": v1, "t": t1}
    got = torch.autograd.grad(out, [leaves[k] for k in wrt], g)
    x2, v2, t2 = x.double().requires_grad_(), value.double().requires_grad_(), t0.double().requires_grad_()
    ref = definition(rowptr, col, v2, x2, t2)
    want = torch.autograd.grad(ref, [{"x": x2, "v": v2, "t": t2}[k] for k in wrt], g.double())
    torch.testing.assert_close(out.double(), ref.detach(), rtol=2e-5, atol=2e-5)
    for k, a, b in zip(wrt, got, want):
        assert a.shape == b.shape and a.dtype == leaves[k].dtype, k
        scale = b.abs().max().item() + 1
        torch.testing.assert_close(a.double(), b, rtol=1e-4, atol=1e-4 * scale, msg=k)


def test_gradcheck_fp64():
    rowptr, col, value, x = _graph(12, M=20, N=15, K=5, dtype=torch.float64)
    M, N = rowptr.numel() - 1, x.size(0)
    A = ts.SparseTensor(rowptr=rowptr, col=col, sparse_sizes=(M, N))
    rowptr, col, _ = A.csr()   # the storage's order, which its CSC view indexes
    st = A.storage
    colptr, csr2csc, row_csc = st.colptr(), st.csr2csc(), st.row_csc()
    for t in (torch.tensor(0.7, dtype=torch.float64, device=DEV),
              torch.linspace(-1, 1.5, 5, dtype=torch.float64, device=DEV)):
        args = (value.clone().requires_grad_(), x.clone().requires_grad_(), t.clone().requires_grad_())
        assert torch.autograd.gradcheck(
            lambda v, xx, tt: ops.SPMMSoftmaxAggr.apply(rowptr, col, v, colptr, csr2csc, xx, row_csc, tt), args)


@pytest.mark.parametrize("t_kind", ["scalar", "channel"])
def test_temperature_gradient_reproducible(t_kind):
    rowptr, col, value, x = _graph(13, M=5000, N=3000, K=64, dtype=torch.bfloat16)
    M, N, K = rowptr.numel() - 1, x.size(0), x.size(1)
    A = ts.SparseTensor(rowptr=rowptr, col=col, value=value, sparse_sizes=(M, N))
    grads = []
    for _ in range(2):
        t = (torch.tensor(1.1, device=DEV) if t_kind == "scalar" else torch.full((K,), 1.1, device=DEV))
        t.requires_grad_()
        tsm.spmm_softmax_aggr(A, x, t).float().pow(2).sum().backward()
        grads.append(t.grad)
    assert torch.equal(grads[0], grads[1])


def _split_graph(seed, dtype, K):
    """A sorted CSR matrix whose rows and columns the backward's row-split kernels defer: a row of 700 entries (three
    segments) and one of 300 (two), a 32-row block of 40 entries per row (over the item budget: single-segment
    deferrals), a hub column holding every fourth entry (over a thousand: several segments), empty rows and columns."""
    g = torch.Generator().manual_seed(seed)
    M, N = 600, 400
    deg = torch.randint(0, 12, (M,), generator=g)
    deg[7], deg[8] = 700, 300
    deg[64:96] = 40
    deg[::37] = 0
    rowptr = torch.cat([torch.zeros(1, dtype=torch.long), deg.cumsum(0)])
    E = int(rowptr[-1])
    col = torch.randint(N - 1, (E,), generator=g)   # column N - 1 stays empty
    col[::4] = 3
    row = torch.repeat_interleave(torch.arange(M), deg)
    col = col[torch.argsort(row * N + col, stable=True)]
    value = (torch.rand(E, generator=g, dtype=torch.float64) + 0.5).to(dtype)
    x = torch.randn(N, K, generator=g, dtype=torch.float64).to(dtype)
    return rowptr.to(DEV), col.to(DEV), value.to(DEV), x.to(DEV)


def _grad_bounds(rowptr, col, v, x, t, g, uT):
    """Error bounds of the three gradients (module docstring of this test): the saved result o is rounded to T (and
    off from the exact one by up to u_T |o| more), which moves every d_e by |g alpha t| 2 u_T |o| and every
    alpha (p - o)^2 by alpha 2 |p - o| 2 u_T |o|; every other term carries a relative error of at most
    c = 2^-20 + (n + 4) 2^-24 (the fp32 exp, products and the n-term sums, n the longest row or column). Returns the
    bounds of grad_x, grad_v and grad_t (per column) before the final rounding to T."""
    M, N = rowptr.numel() - 1, x.size(0)
    rp, colc = rowptr.cpu(), col.cpu()
    row = torch.repeat_interleave(torch.arange(M), rp[1:] - rp[:-1])
    xd, vd, td, gd = x.double().cpu(), v.double().cpu(), t.double().cpu(), g.double().cpu()
    p = xd[colc] * vd[:, None]
    y = td * p
    mu = torch.full((M, x.size(1)), float("-inf"), dtype=torch.float64).index_reduce_(0, row, y, "amax")
    w = torch.exp(y - mu[row])
    s = torch.zeros_like(mu).index_add_(0, row, w)
    o = torch.zeros_like(mu).index_add_(0, row, w * p) / s.clamp(min=1e-300)
    al = w / s[row]
    n = max(int((rp[1:] - rp[:-1]).max()), int(torch.bincount(colc, minlength=N).max()))
    c = 2.0 ** -20 + (n + 4) * 2.0 ** -24
    do = 2 * uT * o.abs()[row]
    dp = p - o[row]
    gr = gd.abs()[row]
    dd = gr * al * (td.abs() * do + c * (1 + td * dp).abs())
    bx = torch.zeros_like(xd).index_add_(0, colc, vd.abs()[:, None] * dd)
    bv = (xd[colc].abs() * dd).sum(1)
    bt = (gr * al * (2 * dp.abs() * do + c * dp * dp)).sum(0)
    return bx, bv, bt


@pytest.mark.parametrize("t_kind", ["scalar", "channel"])
@pytest.mark.parametrize("dtype,K", [(torch.bfloat16, 8), (torch.bfloat16, 128), (torch.bfloat16, 512),
                                     (torch.float16, 64), (torch.float16, 256), (torch.float32, 4),
                                     (torch.float32, 32), (torch.float32, 256), (torch.float32, 13)], ids=_id)
def test_gradients_row_split_within_bound(dtype, K, t_kind):
    """grad_x, grad_v and grad_t against fp64 autograd of the definition, through the row-split backward kernels
    (every width of one column tile, deferred and multi-segment rows and columns) and, at K = 13, the generic ones."""
    rowptr, col, value, x = _split_graph(21, dtype, K)
    M, N = rowptr.numel() - 1, x.size(0)
    t0 = torch.tensor(0.8, device=DEV) if t_kind == "scalar" else torch.linspace(-1.5, 2.0, K, device=DEV)
    v1, x1, t1 = value.clone().requires_grad_(), x.clone().requires_grad_(), t0.clone().requires_grad_()
    A = ts.SparseTensor(rowptr=rowptr, col=col, value=v1, sparse_sizes=(M, N), is_sorted=True, trust_data=True)
    out = tsm.spmm_softmax_aggr(A, x1, t1)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(3)).to(dtype).to(DEV)
    gx, gv, gt = torch.autograd.grad(out, [x1, v1, t1], g)
    x2, v2, t2 = x.double().requires_grad_(), value.double().requires_grad_(), t0.double().requires_grad_()
    ref = definition(rowptr, col, v2, x2, t2)
    rx, rv, rt = torch.autograd.grad(ref, [x2, v2, t2], g.double())
    uT = UT[dtype]
    bx, bv, bt = _grad_bounds(rowptr, col, value, x, t0, g, uT)
    sub = 2.0 ** -25 if dtype == torch.float16 else 0
    for name, got, want, b, u in (("x", gx, rx, bx, uT), ("v", gv, rv, bv, uT)):
        err = (got.double().cpu() - want.cpu()).abs()
        bound = u * want.abs().cpu() + 2 * b + sub
        assert (err <= bound).all(), f"grad_{name}: {int((err > bound).sum())} outside, worst {(err - bound).max()}"
    bt = bt if t_kind == "channel" else bt.sum()
    err = (gt.double().cpu() - rt.cpu()).abs()
    assert (err <= 2.0 ** -24 * rt.abs().cpu() + 2 * bt).all(), f"grad_t: {err} vs {bt}"


@pytest.mark.parametrize("wrt", ["v", "t"])
def test_value_or_temperature_gradient_builds_no_csc_view(wrt):
    rowptr, col, value, x = _graph(14)
    M, N = rowptr.numel() - 1, x.size(0)
    A = ts.SparseTensor(rowptr=rowptr, col=col, value=value.requires_grad_(wrt == "v"), sparse_sizes=(M, N))
    t = torch.tensor(0.9, device=DEV, requires_grad=wrt == "t")
    tsm.spmm_softmax_aggr(A, x, t).sum().backward()
    assert A.storage._csr2csc is None and A.storage._colptr is None
    A = ts.SparseTensor(rowptr=rowptr, col=col, value=value.detach(), sparse_sizes=(M, N))
    x.requires_grad_()
    tsm.spmm_softmax_aggr(A, x, t).sum().backward()
    assert A.storage._csr2csc is not None and x.grad is not None


@pytest.mark.parametrize("dtype,K", [(torch.bfloat16, 8), (torch.bfloat16, 512), (torch.float16, 128),
                                     (torch.float32, 64), (torch.float32, 13), (torch.float64, 16)], ids=_id)
def test_backward_footprint(dtype, K):
    """The backward kernels write every element of their outputs and nothing around them, use no more than their stated
    workspace, and leave their inputs; run twice, the second time over the first call's workspace, they give the same
    bits (no atomics, a fixed segment order)."""
    rowptr, col, value, x = _split_graph(15, dtype, K)
    M, N = rowptr.numel() - 1, x.size(0)
    E = col.numel()
    t = torch.linspace(-1, 1, K, dtype=_acc(dtype), device=DEV)
    out, lse = ops.spmm_fw_softmax_aggr(rowptr, col, value, x, t, want_lse=True)
    g = torch.randn(M, K, device=DEV).to(dtype)
    A = ts.SparseTensor(rowptr=rowptr, col=col, sparse_sizes=(M, N), is_sorted=True, trust_data=True)
    colptr, perm, row_csc = A.storage.colptr(), A.storage.csr2csc(), A.storage.row_csc()
    v_csc = value[perm]
    inputs = [a.clone() for a in (rowptr, col, value, x, t, g, out, lse, colptr, row_csc, v_csc)]
    dt = ops._DTYPES[dtype]
    nws = lib.tsb200_spmm_softmax_aggr_bw_workspace_bytes(K, E)
    wb = torch.full((nws + 2 * WS_GUARD,), 0xA5, dtype=torch.uint8, device=DEV)
    ws = wb[WS_GUARD:WS_GUARD + nws]
    runs = []
    for _ in range(2):
        vb, gv = _guarded((E,), dtype, float("nan"))
        ub, U = _guarded((M, K), _acc(dtype), float("nan"))
        mb, gm = _guarded((N, K), dtype, float("nan"))
        assert lib.tsb200_spmm_softmax_aggr_bw_rows(_vp(rowptr), _vp(col), _vp(value), _vp(x), _vp(t), 1, _vp(g),
                                                    _vp(out), _vp(lse), _vp(gv), _vp(U), M, N, K, E, dt,
                                                    _vp(ws) if nws else None, nws, _stream()) == 0
        assert lib.tsb200_spmm_softmax_aggr_bw_cols(_vp(colptr), _vp(row_csc), _vp(v_csc), _vp(x), _vp(t), 1,
                                                    _vp(g), _vp(out), _vp(lse), _vp(gm), M, N, K, E, dt,
                                                    _vp(ws) if nws else None, nws, _stream()) == 0
        torch.cuda.synchronize()
        for b in (vb, ub, mb):
            assert _guard_ok(b, float("nan"))
        assert (wb[:WS_GUARD] == 0xA5).all() and (wb[WS_GUARD + nws:] == 0xA5).all(), "write outside the workspace"
        assert not gv.isnan().any() and not U.isnan().any() and not gm.isnan().any()
        runs.append((gv, U, gm))
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(_bits(a), _bits(b))
    for a, b in zip(inputs, (rowptr, col, value, x, t, g, out, lse, colptr, row_csc, v_csc)):
        assert torch.equal(a, b)


# ---- a GENConv-style layer ------------------------------------------------------------------------------------------
def _genconv_torch(rowptr, col, x, t, eps=1e-7):
    """GENConv's softmax aggregation as a torch composition (PyG's SoftmaxAggregation: per-column softmax of t * msg
    over each row's entries, by scatter-max shift), with messages relu(x_j) + eps."""
    M = rowptr.numel() - 1
    row = torch.repeat_interleave(torch.arange(M, device=x.device), rowptr[1:] - rowptr[:-1])
    msg = x[col].relu() + eps
    y = t * msg
    mx = torch.full((M, x.size(1)), float("-inf"), device=x.device).index_reduce(0, row, y.detach(), "amax")
    e = torch.exp(y - mx[row])
    s = torch.zeros(M, x.size(1), device=x.device).index_add(0, row, e)
    alpha = e / s[row]
    return torch.zeros(M, x.size(1), device=x.device).index_add(0, row, alpha * msg)


def test_genconv_layer_matches_torch_composition():
    rowptr, col, _, x = _graph(16, M=2000, N=2000, K=64)
    M, N, K = rowptr.numel() - 1, x.size(0), x.size(1)
    A = ts.SparseTensor(rowptr=rowptr, col=col, sparse_sizes=(M, N))
    lin = torch.nn.Linear(K, K).to(DEV)
    eps = 1e-7

    def run(fused):
        t = torch.tensor(1.0, device=DEV, requires_grad=True)
        h = x.clone().requires_grad_()
        if fused:
            agg = tsm.spmm_softmax_aggr(A, h.relu() + eps, t)
        else:
            agg = _genconv_torch(rowptr, col, h, t, eps)
        out = lin(agg + h[:M])
        out.square().mean().backward()
        return out.detach(), h.grad, t.grad

    (o1, gx1, gt1), (o2, gx2, gt2) = run(True), run(False)
    torch.testing.assert_close(o1, o2, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(gx1, gx2, rtol=1e-3, atol=1e-3 * gx2.abs().max().item())
    torch.testing.assert_close(gt1, gt2, rtol=1e-3, atol=1e-6)
