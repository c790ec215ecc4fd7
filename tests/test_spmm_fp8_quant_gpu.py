"""SpMM from an FP8 (e4m3) operand to an e4m3 result with per-row scales (tsb200_spmm_fw_fp8_quant, `spmm_fp8_quant`).

The definition: with y the float32 result of tsb200_spmm_fw_fp8 on the same path (planned or unplanned),
(y8, y_scale) is bit for bit `quantize_fp8(y.cpu(), per_row=True)` (CPU torch: IEEE divisions, the non-saturating
float8_e4m3fn cast), and arg_out is that call's arg_out. NaN equals NaN in any encoding.

The library is called directly into prefilled outputs (y8 0x7f, y_scale NaN, arg_out -1), so an element a kernel fails
to write cannot pass on what was there. The structured matrix of the fp8 tests has empty rows, rows of 1 ... 1300 nnz
(multi-segment rows past 256), a 32-row block over the 1024-nnz item budget and rows with duplicate columns.

Unplanned calls may run at another occupancy than the float32 call they are compared with, hence another work-item
size, and a row the budget defers in one call may not be deferred in the other: it is then summed in another order.
So unplanned sums are compared bit for bit on data where every fp32 sum is exact, and within the rounding bound on
random data. Min/max are exact everywhere.
"""
import ctypes

import pytest
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import ops
from pytorch_sparse_b200._lib import lib
from test_fp8_cpu import e4m3_half_ulp
from test_spmm_fp8_gpu import DEV, ERR_UNSUPPORTED, REDUCES, U32, _dev, call_fp8, make_scale, make_values, make_x8
from test_spmm_kernels_gpu import build_csr, unreferenced_rows

pytestmark = pytest.mark.gpu
KS = (16, 32, 64, 128, 256, 512, 1024, 2048, 48, 400)   # every fp8 dispatch shape, and two partial widths


@pytest.fixture(scope="module")
def mat():
    M, N = 32 * 40 + 13, 3000
    specials = {5: 1, 37: 31, 38: 32, 39: 33, 200: 255, 201: 256, 202: 257, 500: 512, 501: 513, 900: 1300}
    rowptr, col = build_csr(M, N, 4, 11, specials, blocks=[64], tie_rows={300: 40, 301: 600},
                            empty_rows=(0, M // 2, M - 1))
    return dict(M=M, N=N, rowptr=rowptr, col=col)


def _vp(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def call_quant(rowptr, col, value, x8, scale, reduce, plan=None, expect_rc=0, y8=None):
    """tsb200_spmm_fw_fp8_quant into prefilled outputs (y8 0x7f, y_scale NaN, arg_out -1); unplanned when plan is None."""
    M, E = rowptr.numel() - 1, col.numel()
    N, K = x8.shape
    red = ops._REDUCE[reduce]
    if y8 is None:
        y8 = torch.full((M, K), 0x7F, dtype=torch.uint8, device=DEV).view(torch.float8_e4m3fn)
    ys = torch.full((M,), float("nan"), device=DEV)
    arg = torch.full((M, K), -1, dtype=torch.int64, device=DEV) if red >= 2 else None
    if plan is None:
        nws = lib.tsb200_spmm_fw_workspace_bytes(1, M, K, E, 0, red)
        pl, plb, counts = None, 0, (0, 0, 0)
    else:
        nws = lib.tsb200_spmm_fw_planned_workspace_bytes(K, plan.n_long, plan.n_slot, red)
        pl, plb, counts = _vp(plan.data), plan.data.numel(), (plan.n_seg, plan.n_long, plan.n_slot)
    ws = torch.empty(max(nws, 256), dtype=torch.uint8, device=DEV)
    stride = 0 if scale.dim() == 0 else 1
    rc = lib.tsb200_spmm_fw_fp8_quant(_vp(rowptr), _vp(col), _vp(value), _vp(x8), _vp(scale), stride, _vp(y8),
                                      _vp(ys), _vp(arg), M, N, K, E, red, pl, plb, *counts, _vp(ws), nws,
                                      ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == expect_rc, rc
    return y8, ys, arg


# ---- comparisons ------------------------------------------------------------------------------------------------------
def _nan8(b):
    return (b & 0x7F) == 0x7F


def assert_q_equal(y8, ys, ref8, refs, what):
    """e4m3 bytes and fp32 scales bit for bit, NaN equal to NaN in any encoding."""
    a, b = y8.cpu().view(torch.uint8), ref8.cpu().view(torch.uint8)
    ok = (a == b) | (_nan8(a) & _nan8(b))
    if not bool(ok.all()):
        i = tuple(int(j) for j in (~ok).nonzero()[0])
        raise AssertionError(f"{what}: {int((~ok).sum())} e4m3 elements differ, first at {i}: "
                             f"0x{int(a[i]):02x} vs 0x{int(b[i]):02x} (scale {ys.cpu()[i[0]].item()!r})")
    sa, sb = ys.cpu(), refs.cpu()
    ok = (sa.view(torch.int32) == sb.view(torch.int32)) | (sa.isnan() & sb.isnan())
    if not bool(ok.all()):
        i = int((~ok).nonzero()[0])
        raise AssertionError(f"{what}: {int((~ok).sum())} scales differ, first at row {i}: "
                             f"{sa[i].item()!r} vs {sb[i].item()!r}")


def check_against_f32(rowptr, col, v, x8, sc, reduce, plan, what):
    """spmm_fp8_quant against CPU quantize_fp8 of the float32 spmm_fp8 on the same path, arg_out included."""
    y, arg_f = call_fp8(rowptr, col, v, x8, sc, reduce, torch.float32, plan=plan)
    ref8, refs = ts.quantize_fp8(y.cpu(), per_row=True)
    y8, ys, arg = call_quant(rowptr, col, v, x8, sc, reduce, plan=plan)
    assert_q_equal(y8, ys, ref8, refs, what)
    if arg is not None:
        assert torch.equal(arg, arg_f), f"{what}: arg_out differs"
    return y8, ys


def sum_bound_check(y8, ys, rowptr_c, col_c, v_c, x8_c, sc_c, reduce, what):
    """Dequantised result against the fp64 sum: |y - ref| <= e (the fp32 chain, as in test_spmm_fp8_gpu) and the
    quantisation of y: 1/2 ulp_e4m3(y / s) s (1 + 2^-22) + 2^-22 |y| (the division and the product back)."""
    M = rowptr_c.numel() - 1
    deg = (rowptr_c[1:] - rowptr_c[:-1]).double().view(-1, 1)
    row = torch.repeat_interleave(torch.arange(M), deg.view(-1).long())
    s_e = sc_c[col_c] if sc_c.dim() == 1 else sc_c.expand(col_c.numel())
    v = torch.ones(col_c.numel()) if v_c is None else v_c
    t = (v.double() * s_e.double()).view(-1, 1) * x8_c.double()[col_c]
    K = t.size(1)
    ref = torch.zeros(M, K, dtype=torch.float64).index_add_(0, row, t)
    S = torch.zeros(M, K, dtype=torch.float64).index_add_(0, row, t.abs())
    e = (deg + 2) * U32 * S
    if reduce == "mean":
        cnt = deg.clamp(min=1)
        ref, e = ref / cnt, e / cnt
    s = ys.cpu().double().view(-1, 1)
    q = y8.cpu().double()
    got = q * s
    yabs = got.abs() + e4m3_half_ulp(q) * s
    bound = e + e4m3_half_ulp(q) * s * (1 + 2.0 ** -22) + 2.0 ** -22 * yabs
    ok = (got - ref).abs() <= bound
    if not bool(ok.all()):
        i = tuple(int(j) for j in (~ok).nonzero()[0])
        raise AssertionError(f"{what}: {int((~ok).sum())} elements out of bound, first at {i}: "
                             f"got {got[i].item()!r} ref {ref[i].item()!r} bound {bound[i].item():.3e}")


# ---- every shape x reduction x value x scale, planned and unplanned -------------------------------------------------
def exact_operands(N, K, E, seed, per_row):
    """Data on which every fp32 sum of the matrix is exact, in any order: x8 integers in [-4, 4], power-of-two scales
    2^-2 ... 2^2, values multiples of 1/8 in [-2, 2]. A term is a multiple of 2^-5 below 2^5, a row of <= 1300 terms
    sums below 2^16: at most 21 significant bits."""
    g = torch.Generator().manual_seed(seed)
    x8 = torch.randint(-4, 5, (N, K), generator=g).float()
    x8[unreferenced_rows(N)] = float("nan")
    s = torch.ldexp(torch.ones(N), torch.randint(-2, 3, (N,), generator=g))
    v = torch.randint(-16, 17, (E,), generator=g).float() / 8
    return x8.to(torch.float8_e4m3fn), (s if per_row else s[7].clone()), v


@pytest.mark.parametrize("per_row", [True, False], ids=["rowscale", "tensorscale"])
@pytest.mark.parametrize("has_value", [True, False], ids=["value", "novalue"])
@pytest.mark.parametrize("K", KS)
def test_quant_vs_quantize_f32(mat, K, has_value, per_row):
    rowptr_c, col_c, N = mat["rowptr"], mat["col"], mat["N"]
    E = col_c.numel()
    rowptr, col = _dev(rowptr_c, col_c)
    plan = ops.spmm_plan(rowptr, E)
    assert plan.n_long > 0 and plan.n_seg > plan.n_long
    for ties, reduces in ((False, ("sum", "mean")), (True, ("min", "max"))):
        x8_c = make_x8(N, K, K + ties, ties)
        sc_c = make_scale(N, K + 2, per_row)
        v_c = make_values(E, K + 3, ties) if has_value else None
        x8, sc, v = _dev(x8_c, sc_c, v_c)
        for reduce in reduces:
            what = f"K={K} value={has_value} per_row={per_row} {reduce}"
            check_against_f32(rowptr, col, v, x8, sc, reduce, plan, what + " planned")
            if reduce in ("min", "max"):
                check_against_f32(rowptr, col, v, x8, sc, reduce, None, what + " unplanned")
            else:
                y8, ys, _ = call_quant(rowptr, col, v, x8, sc, reduce)
                sum_bound_check(y8, ys, rowptr_c, col_c, v_c, x8_c, sc_c, reduce, what + " unplanned")
    # exact sums: the unplanned result is bit-equal whatever order the kernel adds in
    x8_c, sc_c, v_c = exact_operands(N, K, E, K + 5, per_row)
    x8, sc, v = _dev(x8_c, sc_c, v_c if has_value else None)
    for reduce in ("sum", "mean"):
        check_against_f32(rowptr, col, v, x8, sc, reduce, None, f"K={K} exact {reduce} unplanned")
        check_against_f32(rowptr, col, v, x8, sc, reduce, plan, f"K={K} exact {reduce} planned")


# ---- edge rows --------------------------------------------------------------------------------------------------------
def edge_problem(K):
    """64 rows of 1 ... 8 nnz (no row is deferred, so planned and unplanned add in the same order) over 64 dense rows
    that make, per row: a NaN in the sum, +-inf, results past 448 (scale > 1), results spanning 2^-9 ... 448 after
    scaling (e4m3 subnormals), +-0, and ordinary rows."""
    g = torch.Generator().manual_seed(K)
    M = N = 64
    deg = torch.randint(1, 9, (M,), generator=g)
    rowptr = torch.zeros(M + 1, dtype=torch.long)
    rowptr[1:] = deg.cumsum(0)
    E = int(rowptr[-1])
    col = torch.randint(N, (E,), generator=g)
    row = torch.repeat_interleave(torch.arange(M), deg)
    x = torch.randn(N, K, generator=g) * 8
    kind = torch.arange(N) % 8
    x[kind == 1, 3] = float("nan")                                            # NaN entries
    x[kind == 2] = torch.where(x[kind == 2] > 0, 448.0, -448.0)              # +-448: times a huge value -> +-inf
    span = torch.ldexp(torch.ones(K), torch.linspace(-9, 8, K).round().int())  # 2^-9 ... 2^8 per row, signs mixed
    x[kind == 3] = span * torch.where(torch.rand(K, generator=g) < 0.5, -1.0, 1.0)
    x[kind == 4] = -0.0
    x8 = x.to(torch.float8_e4m3fn)
    v = torch.randn(E, generator=g)
    rk = row % 8
    col = torch.where((rk >= 1) & (rk <= 4), rk, col)                        # rows of kind k gather dense row k only
    v = torch.where(rk == 1, 50.0, v)                                         # NaN at column 3, others past 464
    v = torch.where(rk == 2, 3e38, v)                                         # +-inf in every column
    v = torch.where(rk == 3, 1.0, v)                                          # deg * span: subnormal after scaling
    v = torch.where(rk == 4, v.abs() + 0.5, v)                                # min / max of -0 products: -0
    v = torch.where(rk == 5, v * 100, v)                                      # results far past 448
    return rowptr, col, v, x8


@pytest.mark.parametrize("K", (16, 128, 256, 1024))
def test_quant_edge_rows(K):
    rowptr_c, col_c, v_c, x8_c = edge_problem(K)
    rowptr, col, v, x8 = _dev(rowptr_c, col_c, v_c, x8_c)
    plan = ops.spmm_plan(rowptr, col.numel())
    assert plan.n_seg == 0
    seen = dict(nan_row=False, inf_scale=False, big_scale=False, subnormal=False, neg_zero=False)
    for per_row in (True, False):
        sc = _dev(make_scale(64, K, per_row, pow2=True))[0]
        for reduce in REDUCES:
            for p in (plan, None):
                y8, ys = check_against_f32(rowptr, col, v, x8, sc, reduce, p, f"K={K} {reduce} per_row={per_row}")
                b, s = y8.cpu().view(torch.uint8), ys.cpu()
                seen["nan_row"] |= bool((_nan8(b).any(1) & (s == 1)).any())
                seen["inf_scale"] |= bool(s.isinf().any())
                seen["big_scale"] |= bool(((s > 1) & s.isfinite()).any())
                seen["subnormal"] |= bool((((b & 0x78) == 0) & ((b & 0x07) != 0)).any())
                seen["neg_zero"] |= bool((b == 0x80).any())
    assert all(seen.values()), seen


# ---- chained hops -----------------------------------------------------------------------------------------------------
def test_chained_hops():
    """Three hops X_{h+1} = A X_h in e4m3 on a square matrix, against fp64 propagation of the first dequantised
    operand. The bound is computed, not tuned: with x_h the dequantised operand of hop h and y the fp32 result,
        e_{h+1} = |A| e_h + (deg + 2) 2^-24 |A| |x_h| + 1/2 ulp_e4m3(y / s) s (1 + 2^-22) + 2^-22 |y|."""
    M = 3000
    rowptr_c, col_c = build_csr(M, M, 6, 7, {10: 300, 11: 900}, blocks=[128], tie_rows={}, empty_rows=(0, M // 3))
    E = col_c.numel()
    g = torch.Generator().manual_seed(8)
    v_c = torch.rand(E, generator=g) * 0.3
    K = 128
    x0 = torch.randn(M, K, generator=g)
    x8, sc = ts.quantize_fp8(x0, per_row=True)
    rowptr, col, v = _dev(rowptr_c, col_c, v_c)
    a = ts.SparseTensor(rowptr=rowptr, col=col, value=v, sparse_sizes=(M, M))
    A = torch.sparse_csr_tensor(rowptr_c, col_c, v_c.double(), (M, M))
    Aabs = torch.sparse_csr_tensor(rowptr_c, col_c, v_c.double().abs(), (M, M))
    deg = (rowptr_c[1:] - rowptr_c[:-1]).double().view(-1, 1)
    ref = x8.double() * sc.double().view(-1, 1)          # the first dequantised operand, exactly
    e = torch.zeros(M, K, dtype=torch.float64)
    x8, sc = _dev(x8, sc)
    for h in range(3):
        xh = x8.cpu().double() * sc.cpu().double().view(-1, 1)
        x8, sc = a.spmm_fp8_quant(x8, sc)
        assert x8.dtype == torch.float8_e4m3fn and sc.shape == (M,)
        q, s = x8.cpu().double(), sc.cpu().double().view(-1, 1)
        got = q * s
        hu = e4m3_half_ulp(q) * s
        ref = A @ ref
        e = Aabs @ e + (deg + 2) * U32 * (Aabs @ xh.abs()) + hu * (1 + 2.0 ** -22) + 2.0 ** -22 * (got.abs() + hu)
        err = (got - ref).abs()
        assert bool((err <= e).all()), f"hop {h + 1}: max err / bound {float((err / e).nan_to_num(0).max()):.3f}"
        assert float(got.abs().max()) > 0


# ---- public API -------------------------------------------------------------------------------------------------------
def test_quant_public_api(mat):
    g = torch.Generator().manual_seed(4)
    E = mat["col"].numel()
    rowptr, col = _dev(mat["rowptr"], mat["col"])
    a = ts.SparseTensor(rowptr=rowptr, col=col, value=torch.randn(E, generator=g).to(DEV),
                        sparse_sizes=(mat["M"], mat["N"]))
    x8, sc = ts.quantize_fp8(torch.randn(mat["N"], 64, generator=g).to(DEV), per_row=True)
    for _ in range(2):   # from here on every call uses the cached plan of `a`
        ts.spmm_fp8(a, x8, sc)
    for reduce in REDUCES:
        y8, ys = a.spmm_fp8_quant(x8, sc, reduce)
        ref8, refs = ts.quantize_fp8(ts.spmm_fp8(a, x8, sc, reduce, torch.float32).cpu(), per_row=True)
        assert_q_equal(y8, ys, ref8, refs, f"public {reduce}")
    y8, ys = ts.spmm_fp8_quant(a, x8, sc)
    y8a, ysa = ts.spmm_fp8_quant(a, x8, sc, "add")
    assert torch.equal(y8.view(torch.uint8), y8a.view(torch.uint8)) and torch.equal(ys, ysa)
    # the result is the next hop's operand: a matrix with M columns reads its rows
    M = mat["M"]
    sq = ts.SparseTensor(row=torch.randint(M, (4 * M,), generator=g).to(DEV),
                         col=torch.randint(M, (4 * M,), generator=g).to(DEV), sparse_sizes=(M, M)).coalesce()
    out = ts.spmm_fp8(sq, y8, ys, "sum", torch.float32)
    ref = ts.spmm_fp8(sq, y8.float().to(torch.float8_e4m3fn), ys, "sum", torch.float32)
    assert out.shape == (M, 64) and bool(out.isfinite().all()) and torch.equal(out, ref)
    with pytest.raises(ValueError):
        ts.spmm_fp8_quant(a, x8, sc, "prod")
    # an empty matrix: zeros, scale 1
    a0 = ts.SparseTensor(row=torch.empty(0, dtype=torch.long, device=DEV),
                         col=torch.empty(0, dtype=torch.long, device=DEV), sparse_sizes=(7, mat["N"]))
    y8, ys = a0.spmm_fp8_quant(x8, sc, "max")
    assert bool((y8.view(torch.uint8) == 0).all()) and bool((ys == 1).all())


# ---- errors -----------------------------------------------------------------------------------------------------------
def test_quant_errors(mat):
    N, E = mat["N"], mat["col"].numel()
    rowptr, col = _dev(mat["rowptr"], mat["col"])
    x8 = torch.zeros(N, 32, device=DEV).to(torch.float8_e4m3fn)
    sc = torch.ones(N, device=DEV)
    a = ts.SparseTensor(rowptr=rowptr, col=col, value=torch.ones(E, device=DEV), sparse_sizes=(mat["M"], N))

    # the C-ABI: K % 16, K > 2048, misaligned x8 / y8
    call_quant(rowptr, col, None, torch.zeros(N, 24, device=DEV).to(torch.float8_e4m3fn), sc, "sum",
               expect_rc=ERR_UNSUPPORTED)
    call_quant(rowptr, col, None, torch.zeros(N, 2064, device=DEV).to(torch.float8_e4m3fn), sc, "sum",
               expect_rc=ERR_UNSUPPORTED)
    buf = torch.zeros(N * 32 + 1, device=DEV).to(torch.float8_e4m3fn)
    call_quant(rowptr, col, None, buf[1:].view(N, 32), sc, "sum", expect_rc=ERR_UNSUPPORTED)
    M = mat["M"]
    ybuf = torch.zeros(M * 32 + 16, dtype=torch.uint8, device=DEV)
    call_quant(rowptr, col, None, x8, sc, "sum", y8=ybuf[1:1 + M * 32].view(M, 32), expect_rc=ERR_UNSUPPORTED)
    # E == 0: zeros, scale 1, arg_out 0
    rp0 = torch.zeros(8, dtype=torch.long, device=DEV)
    y8, ys, arg = call_quant(rp0, torch.empty(0, dtype=torch.long, device=DEV), None, x8, sc, "max")
    assert bool((y8.view(torch.uint8) == 0).all()) and bool((ys == 1).all()) and bool((arg == 0).all())

    # the Python layers
    def raises(fn, match):
        with pytest.raises(RuntimeError, match=match):
            fn()
    raises(lambda: ts.spmm_fp8_quant(a, torch.zeros(N, 24, device=DEV).to(torch.float8_e4m3fn), sc), "multiple of 16")
    raises(lambda: ts.spmm_fp8_quant(a, torch.zeros(N, 2064, device=DEV).to(torch.float8_e4m3fn), sc),
           "at most 2048")
    raises(lambda: ts.spmm_fp8_quant(a, torch.zeros(N, 32, device=DEV, dtype=torch.bfloat16), sc), "float8_e4m3fn")
    raises(lambda: ts.spmm_fp8_quant(a, x8, sc.double()), "float32")
    raises(lambda: ts.spmm_fp8_quant(a, x8, torch.ones(N + 1, device=DEV)), r"shape \[\] or \[N\]")
    raises(lambda: ts.spmm_fp8_quant(a, x8.cpu(), sc), "must be CUDA tensor")
    raises(lambda: ops.spmm_fw_fp8_quant(rowptr, col, torch.ones(E, device=DEV, dtype=torch.bfloat16), x8, sc, "sum"),
           "dtype")
    raises(lambda: ts.spmm_fp8_quant(a, x8, sc.clone().requires_grad_()), "forward only")
    av = ts.SparseTensor(rowptr=rowptr, col=col, value=torch.ones(E, device=DEV).requires_grad_(),
                         sparse_sizes=(mat["M"], N))
    raises(lambda: ts.spmm_fp8_quant(av, x8, sc), "forward only")
    with torch.no_grad():
        ts.spmm_fp8_quant(av, x8, sc.clone().requires_grad_())
