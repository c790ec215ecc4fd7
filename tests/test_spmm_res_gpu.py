"""SpMM with a residual of the operand's type added in the store epilogue (tsb200_spmm_fw_res, `spmm(...,
residual=, residual_scale=)`).

The definition: with y the fp32 (fp64) row result of tsb200_spmm_fw / tsb200_spmm_fw_planned on the same path,
    out[m, k] = round_T(fl(y[m, k] + fl(s[m] * r[m, k])))   (one IEEE product, one IEEE add)
so s = 0 with a finite r gives spmm's bits, and an f32 result is fl32(spmm + fl32(s * r)) bit for bit. Calls go through
the C ABI into NaN-prefilled outputs, so an element a kernel fails to write cannot pass on what was there.
"""
import ctypes
import importlib

import pytest
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import ops
from pytorch_sparse_b200._lib import lib
from test_spmm_kernels_gpu import build_csr, half_ulp

tsm = importlib.import_module("pytorch_sparse_b200.matmul")  # the module; the package's `matmul` is a function
pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FLOATS = (torch.bfloat16, torch.float16, torch.float32)
# dense-row bytes 16 ... 4096 (every shape of the vector path) and 4112 (a second column tile)
ROW_BYTES = (16, 32, 64, 128, 256, 512, 1024, 2048, 4096, 4112)


def _id(p):
    return str(p).replace("torch.", "")


def _vp(t, offset=0):
    return None if t is None else ctypes.c_void_p(t.data_ptr() + offset)


@pytest.fixture(scope="module")
def mat():
    """The structured matrix of the per-family tests: empty rows, rows of 1 ... 1300 nnz (segments past 256 and the
    combine), a 32-row block over the 1024-nnz item budget."""
    M, N = 32 * 40 + 13, 3000
    specials = {5: 1, 37: 31, 38: 32, 39: 33, 200: 255, 201: 256, 202: 257, 500: 512, 501: 513, 900: 1300}
    rowptr, col = build_csr(M, N, 4, 11, specials, blocks=[64], tie_rows={300: 40, 301: 600},
                            empty_rows=(0, M // 2, M - 1))
    return dict(M=M, N=N, rowptr=rowptr, col=col)


def _ws(plan, M, K, E, dt, red):
    if plan is None:
        nws = lib.tsb200_spmm_fw_workspace_bytes(1, M, K, E, dt, red)
        return (None, 0, 0, 0, 0), nws
    nws = lib.tsb200_spmm_fw_planned_workspace_bytes(K, plan.n_long, plan.n_slot, red)
    return (_vp(plan.data), plan.data.numel(), plan.n_seg, plan.n_long, plan.n_slot), nws


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def call_res(rowptr, col, value, x, r, s, reduce, plan=None, r_off=0, expect_rc=0):
    """tsb200_spmm_fw_res into a NaN-prefilled output; r_off shifts the residual pointer by that many elements."""
    M, E = rowptr.numel() - 1, col.numel()
    N, K = x.shape
    red, dt = ops._REDUCE[reduce], ops._DTYPES[x.dtype]
    out = torch.full((M, K), float("nan"), dtype=x.dtype, device=DEV)
    pl, nws = _ws(plan, M, K, E, dt, red)
    ws = torch.empty(max(nws, 256), dtype=torch.uint8, device=DEV)
    rc = lib.tsb200_spmm_fw_res(_vp(rowptr), _vp(col), _vp(value), _vp(x), _vp(r, r_off * r.element_size()), _vp(s),
                                0 if s.dim() == 0 else 1, _vp(out), M, N, K, E, dt, red, *pl, _vp(ws), nws, _stream())
    assert rc == expect_rc, rc
    return out


def call_spmm(rowptr, col, value, x, reduce, plan=None):
    """tsb200_spmm_fw / tsb200_spmm_fw_planned into a NaN-prefilled output."""
    M, E = rowptr.numel() - 1, col.numel()
    N, K = x.shape
    red, dt = ops._REDUCE[reduce], ops._DTYPES[x.dtype]
    out = torch.full((M, K), float("nan"), dtype=x.dtype, device=DEV)
    pl, nws = _ws(plan, M, K, E, dt, red)
    ws = torch.empty(max(nws, 256), dtype=torch.uint8, device=DEV)
    if plan is None:
        rc = lib.tsb200_spmm_fw(_vp(rowptr), _vp(col), _vp(value), _vp(x), _vp(out), None, 1, M, N, K, E, dt, red,
                                _vp(ws), nws, _stream())
    else:
        rc = lib.tsb200_spmm_fw_planned(_vp(rowptr), _vp(col), _vp(value), _vp(x), _vp(out), None, M, N, K, E, dt, red,
                                        *pl, _vp(ws), nws, _stream())
    assert rc == 0, rc
    return out


def assert_bits(a, b, what):
    """Bit for bit, NaN equal to NaN."""
    a, b = a.cpu(), b.cpu()
    bits = {2: torch.int16, 4: torch.int32, 8: torch.int64}[a.element_size()]
    ok = (a.view(bits) == b.view(bits)) | (a.isnan() & b.isnan())
    if not bool(ok.all()):
        i = tuple(int(j) for j in (~ok).nonzero()[0])
        raise AssertionError(f"{what}: {int((~ok).sum())} elements differ, first at {i}: {a[i].item()!r} vs "
                             f"{b[i].item()!r}")


def operands(mat, K, dtype, has_value, scale, seed=0):
    g = torch.Generator().manual_seed(seed)
    M, N, E = mat["M"], mat["N"], mat["col"].numel()
    x = torch.randn(N, K, generator=g, dtype=torch.float64).to(dtype)
    v = torch.randn(E, generator=g, dtype=torch.float64).to(dtype) if has_value else None
    r = torch.randn(M, K, generator=g, dtype=torch.float64).to(dtype)
    sdt = torch.float64 if dtype == torch.float64 else torch.float32
    s = {"none": torch.ones((), dtype=sdt), "scalar": torch.tensor(0.75, dtype=sdt),
         "row": (torch.rand(M, generator=g, dtype=torch.float64) * 2 - 0.5).to(sdt)}[scale]
    return x, v, r, s


def ref_bound(rowptr, col, v, x, r, s, mean, dtype):
    """fp64 reference and the bound 1/2 ulp_T + (deg + 2) u (sum |v x| (/deg for a mean) + |s r|)."""
    rowptr, col, x, r = rowptr.cpu(), col.cpu(), x.cpu().double(), r.cpu().double()
    M = rowptr.numel() - 1
    row = torch.repeat_interleave(torch.arange(M), rowptr[1:] - rowptr[:-1])
    vv = torch.ones(col.numel(), dtype=torch.float64) if v is None else v.cpu().double()
    y = torch.zeros(M, x.size(1), dtype=torch.float64).index_add_(0, row, vv[:, None] * x[col])
    S = torch.zeros_like(y).index_add_(0, row, (vv[:, None] * x[col]).abs())
    deg = (rowptr[1:] - rowptr[:-1]).double()[:, None]
    if mean:
        y, S = y / deg.clamp(min=1), S / deg.clamp(min=1)
    sr = s.cpu().double()
    sr = sr[:, None] * r if sr.dim() == 1 else sr * r
    ref = y + sr
    u = 2.0 ** -53 if dtype == torch.float64 else 2.0 ** -24
    bound = (deg + 2) * u * (S + sr.abs())
    if dtype != torch.float64:
        bound = bound + half_ulp(ref.abs() + bound, dtype)
    return ref, bound


def assert_bound(out, ref, bound, what):
    err = (out.cpu().double() - ref).abs()
    ok = err <= bound
    if not bool(ok.all()):
        i = tuple(int(j) for j in (~ok).nonzero()[0])
        raise AssertionError(f"{what}: {int((~ok).sum())} out of bound, first at {i}: {out.cpu()[i].item()!r} vs "
                             f"{ref[i].item()!r} (bound {bound[i].item():.3e})")


# ---- every shape x dtype x reduce x value x scale, planned and unplanned --------------------------------------------
@pytest.mark.parametrize("scale", ["none", "scalar", "row"])
@pytest.mark.parametrize("has_value", [True, False], ids=["value", "novalue"])
@pytest.mark.parametrize("reduce", ["sum", "mean"])
@pytest.mark.parametrize("dtype", FLOATS, ids=_id)
@pytest.mark.parametrize("row_bytes", ROW_BYTES)
def test_forward_every_shape(mat, row_bytes, dtype, reduce, has_value, scale):
    K = row_bytes // torch.tensor([], dtype=dtype).element_size()
    rowptr, col = mat["rowptr"].to(DEV), mat["col"].to(DEV)
    E = col.numel()
    x, v, r, s = operands(mat, K, dtype, has_value, scale)
    xd, vd, rd, sd = x.to(DEV), None if v is None else v.to(DEV), r.to(DEV), s.to(DEV)
    plan = ops.spmm_plan(rowptr, E)
    ref, bound = ref_bound(rowptr, col, v, x, r, s, reduce == "mean", dtype)
    for pl in (None, plan):
        what = f"{dtype} K={K} {reduce} {'planned' if pl else 'unplanned'}"
        y = call_spmm(rowptr, col, vd, xd, reduce, pl)
        out = call_res(rowptr, col, vd, xd, rd, sd, reduce, pl)
        assert_bits(call_res(rowptr, col, vd, xd, rd, torch.zeros_like(sd), reduce, pl), y, what + " s=0")
        if dtype == torch.float32:
            sr = sd[:, None] * rd if sd.dim() == 1 else sd * rd
            assert_bits(out, y + sr, what + " fl32(spmm + fl32(s r))")
        assert_bound(out, ref, bound, what)


@pytest.mark.parametrize("shift", range(6))
@pytest.mark.parametrize("row_bytes", (16, 32, 64, 128, 256, 512, 1024, 2048, 4096))
def test_item_sizes(mat, row_bytes, shift, monkeypatch):
    """Every work-item size on every shape, planned and unplanned: s = 0 gives spmm's bits at the same size, and f32
    gives fl32(spmm + fl32(s r))."""
    monkeypatch.setenv("TSB200_SPMM_ITEM_SHIFT", str(shift))
    rowptr, col = mat["rowptr"].to(DEV), mat["col"].to(DEV)
    plan = ops.spmm_plan(rowptr, col.numel())
    for dtype in (torch.float32, torch.bfloat16):
        K = row_bytes // torch.tensor([], dtype=dtype).element_size()
        x, v, r, s = [t.to(DEV) for t in operands(mat, K, dtype, True, "row", seed=shift)]
        for reduce in ("sum", "mean"):
            for pl in (None, plan):
                what = f"shift {shift} {dtype} K={K} {reduce} {'planned' if pl else 'unplanned'}"
                y = call_spmm(rowptr, col, v, x, reduce, pl)
                assert_bits(call_res(rowptr, col, v, x, r, torch.zeros_like(s), reduce, pl), y, what + " s=0")
                if dtype == torch.float32:
                    assert_bits(call_res(rowptr, col, v, x, r, s, reduce, pl), y + s[:, None] * r, what + " f32")


# ---- the generic kernel: partial widths, fp64, a misaligned residual -------------------------------------------------
@pytest.mark.parametrize("dtype,K", [(torch.float32, 3), (torch.float32, 37), (torch.bfloat16, 12),
                                     (torch.float16, 100), (torch.float64, 2), (torch.float64, 64),
                                     (torch.float64, 130)], ids=_id)
@pytest.mark.parametrize("reduce", ["sum", "mean"])
def test_generic(mat, dtype, K, reduce):
    rowptr, col = mat["rowptr"].to(DEV), mat["col"].to(DEV)
    x, v, r, s = operands(mat, K, dtype, True, "row")
    xd, vd, rd, sd = x.to(DEV), v.to(DEV), r.to(DEV), s.to(DEV)
    y = call_spmm(rowptr, col, vd, xd, reduce)
    assert_bits(call_res(rowptr, col, vd, xd, rd, torch.zeros_like(sd), reduce), y, f"{dtype} K={K} s=0")
    out = call_res(rowptr, col, vd, xd, rd, sd, reduce)
    if dtype in (torch.float32, torch.float64):
        assert_bits(out, y + sd[:, None] * rd, f"{dtype} K={K} fl(spmm + fl(s r))")
    ref, bound = ref_bound(rowptr, col, v, x, r, s, reduce == "mean", dtype)
    assert_bound(out, ref, bound, f"{dtype} K={K}")
    A = ts.SparseTensor(rowptr=rowptr, col=col, value=vd, sparse_sizes=(mat["M"], mat["N"]))
    rp, c, va = A.csr()   # the tensor sorts each row's columns: its own CSR is what the public API multiplies
    assert_bits(tsm.spmm(A, xd, reduce, residual=rd, residual_scale=sd), call_res(rp, c, va, xd, rd, sd, reduce),
                "public API")


@pytest.mark.parametrize("dtype", FLOATS, ids=_id)
def test_misaligned_residual(mat, dtype):
    """A residual that is not 16-byte aligned runs the generic kernel: same formula, within the bound."""
    rowptr, col = mat["rowptr"].to(DEV), mat["col"].to(DEV)
    M, K = mat["M"], 64
    x, v, r, s = operands(mat, K, dtype, True, "row")
    buf = torch.empty(M * K + 1, dtype=dtype, device=DEV)
    buf[1:] = r.to(DEV).flatten()
    out = call_res(rowptr, col, v.to(DEV), x.to(DEV), buf, s.to(DEV), "sum", r_off=1)
    ref, bound = ref_bound(rowptr, col, v, x, r, s, False, dtype)
    assert_bound(out, ref, bound, f"{dtype} misaligned")
    if dtype == torch.float32:
        y = ops.spmm_fw(rowptr, col, v.to(DEV), x.to(DEV), "sum")[0]
        assert_bound(out, (y.double() + s.to(DEV).double()[:, None] * r.to(DEV).double()).cpu(), bound, "vs spmm")


# ---- exact sums against a CPU replay; specials ------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", FLOATS + (torch.float64,), ids=_id)
@pytest.mark.parametrize("K", (8, 128, 1024))
def test_exact_sums_replay(mat, dtype, K):
    """Small integers (every product and sum exact in fp32) and power-of-two scales: the result is the fp64 replay
    rounded once, bit for bit, planned and unplanned."""
    g = torch.Generator().manual_seed(K)
    M, N = mat["M"], mat["N"]
    rowptr, col = mat["rowptr"].to(DEV), mat["col"].to(DEV)
    x = torch.randint(-3, 4, (N, K), generator=g).to(dtype)
    v = torch.randint(-2, 3, (col.numel(),), generator=g).to(dtype)
    r = torch.randint(-8, 9, (M, K), generator=g).to(dtype)
    sdt = torch.float64 if dtype == torch.float64 else torch.float32
    s = (2.0 ** torch.randint(-2, 3, (M,), generator=g)).to(sdt)
    ref, _ = ref_bound(rowptr, col, v, x, r, s, False, dtype)
    plan = ops.spmm_plan(rowptr, col.numel())
    for pl in (None, plan):
        out = call_res(rowptr, col, v.to(DEV), x.to(DEV), r.to(DEV), s.to(DEV), "sum", pl)
        assert_bits(out, ref.to(dtype), f"{dtype} K={K} replay")


@pytest.mark.parametrize("dtype", FLOATS + (torch.float64,), ids=_id)
@pytest.mark.parametrize("K", (64, 6))
def test_specials(mat, dtype, K):
    """NaN and +-inf in r propagate; a -0 residual on an empty row gives +0."""
    M = mat["M"]
    rowptr, col = mat["rowptr"].to(DEV), mat["col"].to(DEV)
    x, v, r, s = [t.to(DEV) for t in operands(mat, K, dtype, True, "scalar")]
    r[3, 1], r[5, 2], r[900, 0] = float("nan"), float("inf"), float("-inf")
    empty = [0, M // 2, M - 1]
    r[empty] = -0.0
    out = call_res(rowptr, col, v, x, r, s, "sum").cpu()
    assert out[3, 1].isnan() and out[5, 2] == float("inf") and out[900, 0] == float("-inf")
    e = out[empty]
    assert bool((e == 0).all()) and not bool(torch.signbit(e).any())


def test_empty_matrix_and_rows():
    """E = 0 writes round(fl(+0 + s r)); M = 0 writes nothing."""
    for dtype, K in [(dt, k) for dt in FLOATS + (torch.float64,) for k in (32, 6)]:   # residual-only / generic kernel
        M, N = 70, 5
        rowptr = torch.zeros(M + 1, dtype=torch.long, device=DEV)
        col = torch.empty(0, dtype=torch.long, device=DEV)
        x = torch.randn(N, K, device=DEV).to(dtype)
        r = torch.randn(M, K, device=DEV).to(dtype)
        r[1] = -0.0
        sdt = torch.float64 if dtype == torch.float64 else torch.float32
        s = torch.rand(M, device=DEV, dtype=sdt)
        out = call_res(rowptr, col, None, x, r, s, "mean")
        want = (s[:, None] * r.to(sdt)).to(dtype)   # fl(s r) in the accumulator type, rounded once
        assert_bits(out, want + 0.0, f"{dtype} E=0")
        assert not bool(torch.signbit(out[1]).any())
        out0 = call_res(torch.zeros(1, dtype=torch.long, device=DEV), col, None, x, r[:0], s[:0], "sum")
        assert out0.shape == (0, K)


# ---- public API ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", FLOATS, ids=_id)
@pytest.mark.parametrize("reduce", ["sum", "add", "mean"])
def test_public_api_bits(mat, dtype, reduce, monkeypatch):
    """spmm(..., residual=, residual_scale=) and SparseTensor.spmm give the C ABI's bits, unplanned and planned."""
    monkeypatch.setenv("TSB200_AUTO_PLAN", "0")
    M, N, K = mat["M"], mat["N"], 128
    rowptr, col = mat["rowptr"].to(DEV), mat["col"].to(DEV)
    x, v, r, s = [t.to(DEV) for t in operands(mat, K, dtype, True, "row")]
    A = ts.SparseTensor(rowptr=rowptr, col=col, value=v, sparse_sizes=(M, N))
    rowptr, col, v = A.csr()   # the tensor sorts each row's columns: its own CSR is what the public API multiplies
    want = call_res(rowptr, col, v, x, r, s, reduce)
    assert_bits(tsm.spmm(A, x, reduce, residual=r, residual_scale=s), want, "spmm")
    assert_bits(A.spmm(x, reduce, residual=r, residual_scale=s), want, "SparseTensor.spmm")
    plan = ops.spmm_plan(rowptr, col.numel())
    assert_bits(ops.spmm_fw_res(rowptr, col, v, x, r, s, reduce, plan=plan),
                call_res(rowptr, col, v, x, r, s, reduce, plan), "ops planned")
    one = call_res(rowptr, col, v, x, r, torch.ones((), device=DEV), reduce)
    assert_bits(tsm.spmm(A, x, reduce, residual=r), one, "residual_scale None")


# ---- gradients -------------------------------------------------------------------------------------------------------
def _small(seed=0, M=40, N=30):
    g = torch.Generator().manual_seed(seed)
    deg = torch.randint(0, 9, (M,), generator=g)
    deg[3], deg[7] = 0, 300
    row = torch.repeat_interleave(torch.arange(M), deg)
    col = torch.randint(N, (row.numel(),), generator=g)
    return row, col, M, N


@pytest.mark.parametrize("reduce", ["sum", "mean"])
@pytest.mark.parametrize("scale", ["none", "scalar", "row"])
@pytest.mark.parametrize("dtype", (torch.float32, torch.bfloat16, torch.float64), ids=_id)
def test_gradients(dtype, scale, reduce):
    """Gradients to each input alone and to all together against fp64 autograd of the composition."""
    row, col, M, N = _small()
    K = 16
    g = torch.Generator().manual_seed(1)
    v0 = torch.randn(row.numel(), generator=g, dtype=torch.float64)
    x0 = torch.randn(N, K, generator=g, dtype=torch.float64)
    r0 = torch.randn(M, K, generator=g, dtype=torch.float64)
    s0 = None if scale == "none" else (torch.tensor(0.6, dtype=torch.float64) if scale == "scalar"
                                       else torch.rand(M, generator=g, dtype=torch.float64))
    go = torch.randn(M, K, generator=g, dtype=torch.float64)
    sdt = torch.float64 if dtype == torch.float64 else torch.float32
    names = ["value", "x", "residual"] + ([] if s0 is None else ["scale"])
    deg = torch.bincount(row, minlength=M).double().clamp(min=1)[:, None]
    for want in [[n] for n in names] + [names]:
        leaves = {"value": v0, "x": x0, "residual": r0, "scale": s0}
        ref = {k: (t.clone().requires_grad_(k in want) if t is not None else None) for k, t in leaves.items()}
        y = torch.zeros(M, K, dtype=torch.float64).index_add(0, row, ref["value"][:, None] * ref["x"][col])
        if reduce == "mean":
            y = y / deg
        sr = ref["residual"] if s0 is None else (ref["scale"][:, None] if s0.dim() == 1 else ref["scale"]) * ref["residual"]
        (y + sr).backward(go)
        dev = {k: (t.to(DEV, sdt if k == "scale" else dtype).requires_grad_(k in want) if t is not None else None)
               for k, t in leaves.items()}
        A = ts.SparseTensor(row=row.to(DEV), col=col.to(DEV), value=dev["value"], sparse_sizes=(M, N))
        out = tsm.spmm(A, dev["x"], reduce, residual=dev["residual"], residual_scale=dev["scale"])
        out.backward(go.to(DEV, dtype))
        tol = 1e-9 if dtype == torch.float64 else (2e-5 if dtype == torch.float32 else 3e-2)
        for k in want:
            a, b = dev[k].grad.cpu().double(), ref[k].grad
            err = ((a - b).abs() / (b.abs().max() + 1e-30)).max().item()
            assert err <= tol, f"{dtype} {scale} {reduce} grad {k} (want {want}): {err:.3e}"
        if "residual" in want:
            s_dev = dev["scale"]
            gr = go.to(DEV, dtype).to(sdt)
            if s_dev is not None:
                gr = gr * (s_dev.detach()[:, None] if s_dev.dim() == 1 else s_dev.detach())
            assert_bits(dev["residual"].grad, gr.to(dtype) + 0.0, "grad_residual rounded once")


@pytest.mark.parametrize("reduce", ["sum", "mean"])
def test_gradcheck_fp64(reduce):
    row, col, M, N = _small(2, M=12, N=9)
    g = torch.Generator().manual_seed(3)
    v = torch.randn(row.numel(), generator=g, dtype=torch.float64).to(DEV).requires_grad_()
    x = torch.randn(N, 4, generator=g, dtype=torch.float64).to(DEV).requires_grad_()
    r = torch.randn(M, 4, generator=g, dtype=torch.float64).to(DEV).requires_grad_()
    s = torch.rand(M, generator=g, dtype=torch.float64).to(DEV).requires_grad_()
    rd, cd = row.to(DEV), col.to(DEV)

    def f(v, x, r, s):
        return tsm.spmm(ts.SparseTensor(row=rd, col=cd, value=v, sparse_sizes=(M, N)), x, reduce, residual=r,
                        residual_scale=s)
    assert torch.autograd.gradcheck(f, (v, x, r, s))


def test_residual_only_gradient_builds_no_csc_view():
    row, col, M, N = _small()
    A = ts.SparseTensor(row=row.to(DEV), col=col.to(DEV), value=torch.randn(row.numel(), device=DEV),
                        sparse_sizes=(M, N))
    x = torch.randn(N, 16, device=DEV)
    r = torch.randn(M, 16, device=DEV, requires_grad=True)
    s = torch.rand(M, device=DEV, requires_grad=True)
    st = A.storage
    for reduce in ("sum", "mean"):
        tsm.spmm(A, x, reduce, residual=r, residual_scale=s).sum().backward()
        assert st._csr2csc is None and st._colptr is None and st._row_csc is None and st._rowcount is None


# ---- recipes ---------------------------------------------------------------------------------------------------------
def test_appnp_chain():
    """10 APPNP hops X <- (1 - a) A X + a H with (1 - a) folded into the values, in bf16, against fp64: each hop adds at
    most the one-hop bound on top of the previous hop's error carried through the (norm <= 1) operator."""
    g = torch.Generator().manual_seed(5)
    M, K, alpha = 3000, 64, 0.1
    row = torch.randint(M, (30000,), generator=g)
    col = torch.randint(M, (30000,), generator=g)
    A = ts.SparseTensor(row=row.to(DEV), col=col.to(DEV), sparse_sizes=(M, M)).coalesce()
    rp, c, _ = A.csr()
    deg = (rp[1:] - rp[:-1]).double().clamp(min=1)
    w = ((1 - alpha) / deg[torch.repeat_interleave(torch.arange(M, device=DEV), rp[1:] - rp[:-1])])
    An = A.set_value(w.to(torch.bfloat16), layout="csr")
    h = torch.randn(M, K, generator=g, dtype=torch.float64)
    xb, x64 = h.to(DEV, torch.bfloat16), h.to(DEV)
    s = torch.tensor(alpha, device=DEV)
    w64 = w.double()
    row_d = torch.repeat_interleave(torch.arange(M, device=DEV), rp[1:] - rp[:-1])
    hb = h.to(DEV, torch.bfloat16)
    for _ in range(10):
        xb = An.spmm(xb, residual=hb, residual_scale=s)
        x64 = torch.zeros(M, K, dtype=torch.float64, device=DEV).index_add_(0, row_d, w64[:, None] * x64[c]) \
            + alpha * hb.double()
    err = (xb.double() - x64).abs().max().item()
    assert err <= 10 * (2.0 ** -8 * x64.abs().max().item() + 64 * 2.0 ** -24 * 4), err


def test_gcn_self_loops():
    """GCN with self-loops as a per-row residual scale: values d^-1/2[row] w d^-1/2[col] (d = deg + 1), residual x,
    residual_scale 1/d, against the structural A + I product in fp64."""
    g = torch.Generator().manual_seed(6)
    M, K = 2000, 32
    row = torch.randint(M, (20000,), generator=g)
    col = torch.randint(M, (20000,), generator=g)
    keep = row != col
    A = ts.SparseTensor(row=row[keep].to(DEV), col=col[keep].to(DEV), sparse_sizes=(M, M)).coalesce()
    rp, c, _ = A.csr()
    r_ = torch.repeat_interleave(torch.arange(M, device=DEV), rp[1:] - rp[:-1])
    d = (rp[1:] - rp[:-1]).double() + 1
    dis = d.rsqrt()
    vals = (dis[r_] * dis[c]).float()
    x = torch.randn(M, K, generator=g).to(DEV)
    out = A.set_value(vals, layout="csr").spmm(x, residual=x, residual_scale=(1 / d).float())
    # structural reference: A + I normalised, in fp64
    rows = torch.cat([r_, torch.arange(M, device=DEV)])
    cols = torch.cat([c, torch.arange(M, device=DEV)])
    wv = dis[rows] * dis[cols]
    ref = torch.zeros(M, K, dtype=torch.float64, device=DEV).index_add_(0, rows, wv[:, None] * x.double()[cols])
    S = torch.zeros_like(ref).index_add_(0, rows, (wv[:, None] * x.double()[cols]).abs())
    degp = torch.bincount(rows, minlength=M).double()[:, None]
    bound = (degp + 3) * 2.0 ** -24 * S
    assert bool(((out.double() - ref).abs() <= bound).all())


def test_forward_peak_memory(mat):
    rowptr, col = mat["rowptr"].to(DEV), mat["col"].to(DEV)
    M, K = mat["M"], 256
    x, v, r, s = [t.to(DEV) for t in operands(mat, K, torch.bfloat16, True, "row")]
    ops.spmm_fw_res(rowptr, col, v, x, r, s)  # first call: plan cache entry
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = ops.spmm_fw_res(rowptr, col, v, x, r, s)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    ws = max(lib.tsb200_spmm_fw_workspace_bytes(1, M, K, col.numel(), 3, 0), 1 << 16)
    assert peak <= out.numel() * out.element_size() + ws + (1 << 20), peak
