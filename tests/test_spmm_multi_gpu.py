"""Multi-aggregation SpMM (tsb200_spmm_fw_multi, `spmm_multi`): sum, mean, min, max, var and std of every row's
messages from one gather pass.

The sum, mean, min and max slices and both args are bit for bit what tsb200_spmm_fw / tsb200_spmm_fw_planned return
on the same path and at the same work-item size; var and std are checked against fp64 sums of the definition. Calls go
through the C ABI into NaN-prefilled outputs inside a guarded buffer, so an element a kernel fails to write, or writes
outside its output, cannot pass.
"""
import ctypes
import importlib

import pytest
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import ops
from pytorch_sparse_b200._lib import lib
from test_spmm_kernels_gpu import build_csr
from test_spmm_res_gpu import ROW_BYTES, _id, _stream, _vp, _ws

tsm = importlib.import_module("pytorch_sparse_b200.matmul")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FLOATS = (torch.bfloat16, torch.float16, torch.float32)
SUM, MEAN, MIN, MAX, VAR, STD = range(6)
G = 4096  # guard elements on each side of every output and workspace


@pytest.fixture(scope="module")
def mat():
    """Empty rows, rows of 1 ... 1300 nnz (segments past 256 and the combine), a 32-row block over the item budget."""
    M, N = 32 * 40 + 13, 3000
    specials = {5: 1, 37: 31, 38: 32, 39: 33, 200: 255, 201: 256, 202: 257, 500: 512, 501: 513, 900: 1300}
    rowptr, col = build_csr(M, N, 4, 11, specials, blocks=[64], tie_rows={300: 40, 301: 600},
                            empty_rows=(0, M // 2, M - 1))
    return dict(M=M, N=N, rowptr=rowptr, col=col)


def _guarded(shape, dtype, fill):
    n = 1
    for s in shape:
        n *= s
    buf = torch.full((n + 2 * G,), fill, dtype=dtype, device=DEV)
    return buf, buf[G:G + n].view(shape)


def _guard_ok(buf, fill):
    head, tail = buf[:G], buf[-G:]
    if buf.dtype.is_floating_point and fill != fill:
        return bool(head.isnan().all() and tail.isnan().all())
    return bool((head == fill).all() and (tail == fill).all())


def call_multi(rowptr, col, value, x, codes, plan=None, args=True):
    """tsb200_spmm_fw_multi into NaN-prefilled, guarded outputs and a guarded workspace of exactly the stated size.
    Returns (out, arg_min, arg_max)."""
    M, E = rowptr.numel() - 1, col.numel()
    K = x.size(1)
    N = x.size(0)
    dt = ops._DTYPES[x.dtype]
    A = len(codes)
    ob, out = _guarded((M, A, K), x.dtype, float("nan"))
    nb = lb = amin = amax = None
    if args and MIN in codes:
        nb, amin = _guarded((M, K), torch.int64, -7)
    if args and MAX in codes:
        lb, amax = _guarded((M, K), torch.int64, -7)
    if plan is None:
        pl, nws = (None, 0, 0, 0, 0), lib.tsb200_spmm_fw_multi_workspace_bytes(K, E, 0, 0, 0)
    else:
        pl = (_vp(plan.data), plan.data.numel(), plan.n_seg, plan.n_long, plan.n_slot)
        nws = lib.tsb200_spmm_fw_multi_workspace_bytes(K, E, 1, plan.n_long, plan.n_slot)
    wb = torch.full((nws + 2 * 256 * 16,), 0xA5, dtype=torch.uint8, device=DEV)
    ws = wb[256 * 16:256 * 16 + nws]
    xin = x.clone()
    rc = lib.tsb200_spmm_fw_multi(_vp(rowptr), _vp(col), _vp(value), _vp(x),
                                  (ctypes.c_int * A)(*codes), A, _vp(out), _vp(amin), _vp(amax), M, N, K, E, dt, *pl, _vp(ws) if nws else None, nws, _stream())
    assert rc == 0, rc
    torch.cuda.synchronize()
    assert _guard_ok(ob, float("nan")), "write before / after out"
    for b in (nb, lb):
        assert b is None or _guard_ok(b, -7), "write before / after an arg output"
    assert (wb[:256 * 16] == 0xA5).all() and (wb[256 * 16 + nws:] == 0xA5).all(), "write outside the workspace"
    assert torch.equal(xin, x), "the dense operand changed"
    return out, amin, amax


def call_spmm(rowptr, col, value, x, red, plan=None):
    M, E = rowptr.numel() - 1, col.numel()
    N, K = x.shape
    dt = ops._DTYPES[x.dtype]
    out = torch.full((M, K), float("nan"), dtype=x.dtype, device=DEV)
    arg = torch.full((M, K), -7, dtype=torch.int64, device=DEV) if red >= 2 else None
    pl, nws = _ws(plan, M, K, E, dt, red)
    ws = torch.empty(max(nws, 256), dtype=torch.uint8, device=DEV)
    if plan is None:
        rc = lib.tsb200_spmm_fw(_vp(rowptr), _vp(col), _vp(value), _vp(x), _vp(out), _vp(arg), 1, M, N, K, E, dt, red,
                                _vp(ws), nws, _stream())
    else:
        rc = lib.tsb200_spmm_fw_planned(_vp(rowptr), _vp(col), _vp(value), _vp(x), _vp(out), _vp(arg), M, N, K, E, dt,
                                        red, *pl, _vp(ws), nws, _stream())
    assert rc == 0, rc
    return out, arg


def _operands(m, dtype, K, with_value, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(m["N"], K, generator=g).to(dtype).to(DEV)
    v = (torch.rand(m["col"].numel(), generator=g) * 2 - 0.5).to(dtype).to(DEV) if with_value else None
    return m["rowptr"].to(DEV), m["col"].to(DEV), v, x


def assert_same_as_spmm(rowptr, col, v, x, plan):
    out, amin, amax = call_multi(rowptr, col, v, x, [MAX, SUM, STD, MIN, MEAN, VAR], plan)
    for red, sl in ((SUM, 1), (MEAN, 4), (MIN, 3), (MAX, 0)):
        ref, arg = call_spmm(rowptr, col, v, x, red, plan)
        assert torch.equal(out[:, sl].view(torch.int16 if x.element_size() == 2 else torch.int32),
                           ref.view(torch.int16 if x.element_size() == 2 else torch.int32)), f"reduce {red}"
        if red == MIN:
            assert torch.equal(amin, arg)
        if red == MAX:
            assert torch.equal(amax, arg)
    return out


@pytest.mark.parametrize("planned", [False, True])
@pytest.mark.parametrize("with_value", [True, False])
@pytest.mark.parametrize("dtype", FLOATS, ids=_id)
@pytest.mark.parametrize("row_bytes", ROW_BYTES)
def test_bitwise_sum_mean_min_max(mat, row_bytes, dtype, with_value, planned):
    esz = torch.tensor([], dtype=dtype).element_size()
    if row_bytes % esz:
        pytest.skip("not a whole number of elements")
    rowptr, col, v, x = _operands(mat, dtype, row_bytes // esz, with_value)
    plan = ops.spmm_plan(rowptr, col.numel()) if planned else None
    assert_same_as_spmm(rowptr, col, v, x, plan)


@pytest.mark.parametrize("shift", range(6))
@pytest.mark.parametrize("K", [8, 64, 128, 512])
def test_bitwise_every_item_size(mat, monkeypatch, shift, K):
    monkeypatch.setenv("TSB200_SPMM_ITEM_SHIFT", str(shift))
    rowptr, col, v, x = _operands(mat, torch.bfloat16, K, True, seed=shift)
    assert_same_as_spmm(rowptr, col, v, x, None)
    assert_same_as_spmm(rowptr, col, v, x, ops.spmm_plan(rowptr, col.numel()))


def _power_law(M, N, seed):
    g = torch.Generator().manual_seed(seed)
    deg = (torch.rand(M, generator=g) ** -1.6).long().clamp(max=4000)
    deg[::97] = 0
    rowptr = torch.zeros(M + 1, dtype=torch.long)
    rowptr[1:] = deg.cumsum(0)
    col = torch.randint(N, (int(rowptr[-1]),), generator=g)
    return dict(M=M, N=N, rowptr=rowptr, col=col)


@pytest.mark.parametrize("dtype", FLOATS, ids=_id)
@pytest.mark.parametrize("K", [16, 128])
def test_bitwise_power_law(dtype, K):
    m = _power_law(20000, 5000, K)
    rowptr, col, v, x = _operands(m, dtype, K, True)
    assert_same_as_spmm(rowptr, col, v, x, None)
    assert_same_as_spmm(rowptr, col, v, x, ops.spmm_plan(rowptr, col.numel()))


@pytest.mark.parametrize("case", ["fp64", "odd_k", "unaligned", "e0"])
def test_bitwise_generic_path(mat, case):
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
    out, amin, amax = call_multi(rowptr, col, v, x, [MAX, SUM, STD, MIN, MEAN, VAR], None)
    for red, sl in ((SUM, 1), (MEAN, 4), (MIN, 3), (MAX, 0)):
        if col.numel():
            ref, arg = call_spmm(rowptr, col, v, x, red)
        else:
            ref, arg = torch.zeros_like(out[:, 0]), torch.zeros_like(amin)
        assert torch.equal(out[:, sl], ref), red
        if red == MIN:
            assert torch.equal(amin, arg)
        if red == MAX:
            assert torch.equal(amax, arg)
    if case == "e0":
        assert (out == 0).all()


def _ref_var(rowptr, col, v, x):
    """fp64 var of the definition, from the products rounded as the kernels form them (exact for 16-bit operands)."""
    xd, M = x.double().cpu(), rowptr.numel() - 1
    colc, rp = col.cpu(), rowptr.cpu()
    vd = v.double().cpu() if v is not None else torch.ones(col.numel(), dtype=torch.float64)
    row = torch.repeat_interleave(torch.arange(M), rp[1:] - rp[:-1])
    p = xd[colc] * vd[:, None]
    if x.dtype == torch.float32:
        p = p.float().double()
    S = torch.zeros(M, x.size(1), dtype=torch.float64).index_add_(0, row, p)
    Q = torch.zeros_like(S).index_add_(0, row, p * p)
    n = (rp[1:] - rp[:-1]).clamp(min=1).double()[:, None]
    mu = S / n
    return (Q / n - mu * mu).clamp(min=0), Q / n + mu * mu, n


@pytest.mark.parametrize("planned", [False, True])
@pytest.mark.parametrize("dtype", FLOATS + (torch.float64,), ids=_id)
@pytest.mark.parametrize("K", [8, 128, 1032])
def test_var_std_bound(mat, dtype, K, planned):
    rowptr, col, v, x = _operands(mat, dtype, K, True, seed=K)
    plan = ops.spmm_plan(rowptr, col.numel()) if planned and dtype != torch.float64 else None
    out, _, _ = call_multi(rowptr, col, v, x, [STD, VAR], plan, args=False)
    var, scale, n = _ref_var(rowptr, col, v, x)
    u = 2.0 ** -53 if dtype == torch.float64 else 2.0 ** -24
    uT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 2.0 ** -24, torch.float64: 2.0 ** -53}[dtype]
    ev = 4 * (n + 4) * u * scale + (2.0 ** -25 if dtype == torch.float16 else 0)   # f16 subnormal results
    got_var = out[:, 1].double().cpu()
    assert ((got_var - var).abs() <= ev + uT * var).all()
    got_std = out[:, 0].double().cpu()
    hi = var > 1e-5 + 2 * ev
    lo = var < 1e-5 - 2 * ev
    sd = var.sqrt()
    assert ((got_std - sd).abs() <= (ev / sd.clamp(min=1e-3) + 2 * uT * sd))[hi].all()
    assert (got_std[lo] == 0).all()


def test_constant_and_one_entry_rows():
    M, N, K = 64, 40, 64
    deg = torch.tensor([1] * 16 + [5] * 16 + [0] * 8 + [300] * 8 + [3] * 16)
    rowptr = torch.zeros(M + 1, dtype=torch.long)
    rowptr[1:] = deg.cumsum(0)
    E = int(rowptr[-1])
    g = torch.Generator().manual_seed(3)
    col = torch.randint(N, (E,), generator=g)
    x = torch.randn(N, K, generator=g)
    x[7] = 0.375                                   # rows 16.. gather only this constant dense row
    col[int(rowptr[16]):] = 7                      # rows of 5 and of 300 entries (several segments), and empty rows
    for dtype in FLOATS + (torch.float64,):
        xd = x.to(dtype).to(DEV)
        out, _, _ = call_multi(rowptr.to(DEV), col.to(DEV), None, xd, [VAR, STD], None, args=False)
        assert (out[:, 1] == 0).all(), dtype
        assert (out[:16, 0] == 0).all() and (out[16:, 0] == 0).all(), dtype


@pytest.mark.parametrize("codes", [[MEAN, MIN, MAX, STD], [SUM, MAX], [STD, SUM], [MIN], [VAR, MEAN]])
def test_order_subsets_and_null_args(mat, codes):
    rowptr, col, v, x = _operands(mat, torch.bfloat16, 64, True)
    full, fmin, fmax = call_multi(rowptr, col, v, x, [SUM, MEAN, MIN, MAX, VAR, STD])
    for args in (True, False):
        out, amin, amax = call_multi(rowptr, col, v, x, codes, args=args)
        for a, c in enumerate(codes):
            assert torch.equal(out[:, a].view(torch.int16), full[:, c].view(torch.int16))
        if args and MIN in codes:
            assert torch.equal(amin, fmin)
        if args and MAX in codes:
            assert torch.equal(amax, fmax)


def test_inputs_untouched(mat):
    rowptr, col, v, x = _operands(mat, torch.float32, 128, True)
    before = [t.clone() for t in (rowptr, col, v, x)]
    plan = ops.spmm_plan(rowptr, col.numel())
    pdata = plan.data.clone()
    call_multi(rowptr, col, v, x, [SUM, MIN, MAX, STD], plan)
    for a, b in zip(before, (rowptr, col, v, x)):
        assert torch.equal(a, b)
    assert torch.equal(pdata, plan.data)


# ---- the public operator and its gradients --------------------------------------------------------------------------
def _sparse(M, N, E, seed, dtype):
    g = torch.Generator().manual_seed(seed)
    row, col = torch.randint(M, (E,), generator=g), torch.randint(N, (E,), generator=g)
    val = (torch.rand(E, generator=g) + 0.5).to(dtype)
    return ts.SparseTensor(row=row.to(DEV), col=col.to(DEV), value=val.to(DEV), sparse_sizes=(M, N)).coalesce()


def test_gradcheck_fp64():
    A = _sparse(12, 9, 50, 0, torch.float64)
    rowptr, col, value = A.csr()
    x = torch.randn(9, 6, dtype=torch.float64, device=DEV, requires_grad=True)
    v = value.detach().clone().requires_grad_()

    def f(v_, x_):
        B = ts.SparseTensor(rowptr=rowptr, col=col, value=v_, sparse_sizes=(12, 9))
        return tsm.spmm_multi(B, x_, ["mean", "min", "max", "std", "var", "sum"])

    assert torch.autograd.gradcheck(f, (v, x), eps=1e-6, atol=1e-6, rtol=1e-5)


def _definition(A, x, aggrs):
    """fp64 torch composition of the definition, differentiable."""
    rowptr, col, value = A.csr()
    M = rowptr.numel() - 1
    row = torch.repeat_interleave(torch.arange(M, device=DEV), rowptr[1:] - rowptr[:-1])
    p = x[col] * value[:, None]
    n = (rowptr[1:] - rowptr[:-1]).clamp(min=1).to(x.dtype)[:, None]
    S = x.new_zeros(M, x.size(1)).index_add(0, row, p)
    Q = x.new_zeros(M, x.size(1)).index_add(0, row, p * p)
    mu = S / n
    d = Q / n - mu * mu
    var = torch.where(d > 0, d, torch.zeros_like(d))
    std = torch.where(var > 1e-5, var.clamp(min=1e-300).sqrt(), torch.zeros_like(var))
    idx = row[:, None].expand_as(p)
    mn = x.new_full((M, x.size(1)), float("inf")).scatter_reduce(0, idx, p, "amin")
    mx = x.new_full((M, x.size(1)), float("-inf")).scatter_reduce(0, idx, p, "amax")
    empty = (rowptr[1:] == rowptr[:-1])[:, None]
    mn, mx = mn.masked_fill(empty, 0), mx.masked_fill(empty, 0)
    st = {"sum": S, "mean": mu, "min": mn, "max": mx, "var": var, "std": std}
    return torch.stack([st[a] for a in aggrs], 1)


@pytest.mark.parametrize("dtype", FLOATS, ids=_id)
def test_gradients_against_fp64(dtype):
    A = _sparse(3000, 2000, 40000, 1, dtype)
    aggrs = ["mean", "min", "max", "std", "var", "sum"]
    g = torch.Generator().manual_seed(2)
    x0 = torch.randn(2000, 64, generator=g)
    go = torch.randn(3000, 6, 64, generator=g)
    if dtype != torch.float32:   # min / max compare products rounded to 16 bits, whose ties fp64 does not see
        go[:, 1:3] = 0
    x = x0.to(dtype).to(DEV).requires_grad_()
    A.requires_grad_()
    out = tsm.spmm_multi(A, x, aggrs)
    gx, gv = torch.autograd.grad(out, [x, A.storage.value()], go.to(dtype).to(DEV))
    rowptr, col, value = A.csr()
    Ad = ts.SparseTensor(rowptr=rowptr, col=col, value=value.detach().double().requires_grad_(),
                         sparse_sizes=A.sparse_sizes())
    xd = x.detach().double().requires_grad_()
    ref = _definition(Ad, xd, aggrs)
    rgx, rgv = torch.autograd.grad(ref, [xd, Ad.storage.value()], go.double().to(DEV))
    uT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 2.0 ** -20}[dtype]
    for got, want in ((gx, rgx), (gv, rgv)):
        err = (got.double() - want).abs()
        scale = want.abs().max()
        assert err.max() <= 64 * uT * scale, (err.max().item(), scale.item())


def test_pna_layer_end_to_end(monkeypatch):
    monkeypatch.setenv("TSB200_AUTO_PLAN", "0")         # both sides unplanned, at the same work-item size
    monkeypatch.setenv("TSB200_SPMM_ITEM_SHIFT", "5")
    A = _sparse(5000, 5000, 80000, 4, torch.float32)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(5000, 32, generator=g).to(DEV)
    deg = A.storage.rowcount().clamp(min=1).float()[:, None]
    logd = torch.log(deg + 1)
    delta = logd.mean()
    agg = tsm.spmm_multi(A, x, ["mean", "min", "max", "std"]).flatten(1)
    out = torch.cat([agg, agg * (logd / delta), agg * (delta / logd)], -1)
    mean = tsm.spmm(A, x, "mean")
    mn, mx = tsm.spmm(A, x, "min"), tsm.spmm(A, x, "max")
    v = A.storage.value()
    A2 = A.set_value(v * v, layout="csr")              # the messages' squares (v x)^2 = v^2 x^2
    var = (tsm.spmm(A2, x * x, "mean") - mean * mean).clamp(min=0)
    std = torch.where(var > 1e-5, var.sqrt(), torch.zeros_like(var))
    ref_agg = torch.cat([mean, mn, mx, std], -1)
    ref = torch.cat([ref_agg, ref_agg * (logd / delta), ref_agg * (delta / logd)], -1)
    assert torch.equal(agg[:, :96], ref_agg[:, :96])
    # the two var formulas round differently, so std may fall on either side of its 1e-5 threshold right next to it
    far = torch.cat([torch.ones_like(ref_agg[:, :96], dtype=torch.bool), (var - 1e-5).abs() > 1e-6], -1).repeat(1, 3)
    assert far[:, 96:128].float().mean() > 0.99
    torch.testing.assert_close(out[far], ref[far], rtol=1e-4, atol=1e-4)
