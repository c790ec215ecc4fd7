"""FP8 SpMM with a per-row e4m3 residual added in the store epilogue (tsb200_spmm_fw_fp8_res, the `residual=` /
`residual_scale=` arguments of `spmm_fp8` and `spmm_fp8_quant`).

The definition: with y the float32 result of tsb200_spmm_fw_fp8 on the same path (planned or unplanned),
    rho = fl32(r_scale[m] * float(r8[m, k])),   z = fl32(y + rho)   (CPU fp32: one IEEE product, one IEEE add)
and the result is z rounded to the output dtype, or `quantize_fp8(z.cpu(), per_row=True)` for an e4m3 result.

The library is called directly into prefilled outputs (NaN, e4m3 0x7f, NaN scales), so an element a kernel fails to
write cannot pass on what was there. Planned calls are bit-exact against that replay. Unplanned calls may run at
another occupancy than the float32 call they are compared with, hence another work-item size and other deferred rows
(see test_spmm_fp8_quant_gpu): they are bit-exact on data where every fp32 sum is exact and within the rounding bound
on random data.
"""
import ctypes

import pytest
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import ops
from pytorch_sparse_b200._lib import lib
from test_fp8_cpu import e4m3_half_ulp
from test_spmm_fp8_gpu import DEV, ERR_UNSUPPORTED, U32, Replay, _dev, call_fp8, make_scale, make_values, make_x8
from test_spmm_fp8_quant_gpu import _nan8, assert_q_equal, call_quant, edge_problem, exact_operands
from test_spmm_kernels_gpu import build_csr, half_ulp

pytestmark = pytest.mark.gpu
E4M3 = torch.float8_e4m3fn
KS = (16, 32, 64, 128, 256, 512, 1024, 2048, 48, 400)   # every fp8 dispatch shape, and two partial widths
OUTS = (torch.bfloat16, torch.float16, torch.float32, E4M3)


@pytest.fixture(scope="module")
def mat():
    """The structured matrix of the fp8 tests: empty rows, rows of 1 ... 1300 nnz (multi-segment rows past 256), a
    32-row block over the 1024-nnz item budget."""
    M, N = 32 * 40 + 13, 3000
    specials = {5: 1, 37: 31, 38: 32, 39: 33, 200: 255, 201: 256, 202: 257, 500: 512, 501: 513, 900: 1300}
    rowptr, col = build_csr(M, N, 4, 11, specials, blocks=[64], tie_rows={300: 40, 301: 600},
                            empty_rows=(0, M // 2, M - 1))
    return dict(M=M, N=N, rowptr=rowptr, col=col)


def _vp(t, offset=0):
    return None if t is None else ctypes.c_void_p(t.data_ptr() + offset)


def call_res(rowptr, col, value, x8, scale, r8, rsc, reduce, out_dtype, plan=None, expect_rc=0, r8_off=0, rsc_off=0):
    """tsb200_spmm_fw_fp8_res into prefilled outputs; out_dtype float8_e4m3fn selects the e4m3 result (value f32).
    r8 = None calls it without a residual. Returns (out, out_scale or None, arg_out or None)."""
    M, E = rowptr.numel() - 1, col.numel()
    N, K = x8.shape
    red = ops._REDUCE[reduce]
    q8 = out_dtype == E4M3
    dt = 0 if q8 else ops._FP8_OUT[out_dtype]
    if q8:
        out = torch.full((M, K), 0x7F, dtype=torch.uint8, device=DEV).view(E4M3)
        ys = torch.full((M,), float("nan"), device=DEV)
    else:
        out = torch.full((M, K), float("nan"), dtype=out_dtype, device=DEV)
        ys = None
    arg = torch.full((M, K), -1, dtype=torch.int64, device=DEV) if red >= 2 else None
    if plan is None:
        nws = lib.tsb200_spmm_fw_workspace_bytes(1, M, K, E, 0, red)
        pl, plb, counts = None, 0, (0, 0, 0)
    else:
        nws = lib.tsb200_spmm_fw_planned_workspace_bytes(K, plan.n_long, plan.n_slot, red)
        pl, plb, counts = _vp(plan.data), plan.data.numel(), (plan.n_seg, plan.n_long, plan.n_slot)
    ws = torch.empty(max(nws, 256), dtype=torch.uint8, device=DEV)
    stride = 0 if scale.dim() == 0 else 1
    rstride = 0 if rsc is None or rsc.dim() == 0 else 1
    rc = lib.tsb200_spmm_fw_fp8_res(_vp(rowptr), _vp(col), _vp(value), _vp(x8), _vp(scale), stride,
                                    _vp(r8, r8_off), _vp(rsc, rsc_off), rstride, _vp(out), _vp(ys), _vp(arg),
                                    M, N, K, E, dt, red, pl, plb, *counts, _vp(ws), nws,
                                    ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == expect_rc, rc
    return out, ys, arg


def rho_of(r8_c, rsc_c):
    """fl32(r_scale[m] * r8[m, k]) on the CPU."""
    return (rsc_c.view(-1, 1) if rsc_c.dim() == 1 else rsc_c) * r8_c.float()


def finish(z, out_dtype):
    """z rounded to the output dtype, or quantised per row (CPU)."""
    return ts.quantize_fp8(z, per_row=True) if out_dtype == E4M3 else z.to(out_dtype)


def assert_out_equal(out, ys, ref, what):
    """Bit for bit, NaN equal to NaN in any encoding."""
    if isinstance(ref, tuple):
        assert_q_equal(out, ys, ref[0], ref[1], what)
        return
    a, b = out.cpu(), ref.cpu()
    bits = {2: torch.int16, 4: torch.int32}[a.element_size()]
    ok = (a.view(bits) == b.view(bits)) | (a.isnan() & b.isnan())
    if not bool(ok.all()):
        i = tuple(int(j) for j in (~ok).nonzero()[0])
        raise AssertionError(f"{what}: {int((~ok).sum())} elements differ, first at {i}: "
                             f"{a[i].item()!r} vs {b[i].item()!r}")


def make_residual(M, K, seed, per_row):
    g = torch.Generator().manual_seed(seed)
    r8 = (torch.randn(M, K, generator=g) * 3).to(E4M3)
    s = torch.rand(M, generator=g) * 0.5 + 0.01
    return r8, (s if per_row else s[3].clone())


def check_vs_replay(rowptr, col, v32, x8, sc, r8, rsc, r8_c, rsc_c, reduce, out_dtype, plan, what):
    """The planned / exact-data rule: bit-exact against the f32 result on the same path plus rho, then rounded. A
    16-bit result takes 16-bit values; the f32 call gets those values widened."""
    v = v32 if v32 is None or out_dtype in (torch.float32, E4M3) else v32.to(out_dtype)
    y, _ = call_fp8(rowptr, col, None if v is None else v.float(), x8, sc, reduce, torch.float32, plan=plan)
    out, ys, _ = call_res(rowptr, col, v, x8, sc, r8, rsc, reduce, out_dtype, plan=plan)
    assert_out_equal(out, ys, finish(y.cpu() + rho_of(r8_c, rsc_c), out_dtype), what)
    return out, ys


def bound_check(out, ys, rep, reduce, rho, out_dtype, what):
    """An unplanned result on random data against the fp64 sum plus rho: the fp32 chain's e (as in
    test_spmm_fp8_gpu), the add's rounding 2^-24 |z|, then the rounding to the output dtype or the e4m3
    quantisation (as in test_spmm_fp8_quant_gpu)."""
    ref, S = rep.sums()
    e = (rep.deg + 2) * U32 * S
    if reduce == "mean":
        ref, e = ref / rep.cnt, e / rep.cnt
    ref = ref + rho.double()
    if out_dtype == E4M3:
        s = ys.cpu().double().view(-1, 1)
        q = out.cpu().double()
        got = q * s
        hu = e4m3_half_ulp(q) * s
        zabs = got.abs() + hu
        bound = e + U32 * zabs + hu * (1 + 2.0 ** -22) + 2.0 ** -22 * zabs
    else:
        got = out.cpu().double()
        zabs = ref.abs() + e
        bound = e + U32 * zabs + half_ulp(zabs * (1 + 2.0 ** -22), out_dtype)
    ok = (got - ref).abs() <= bound
    if not bool(ok.all()):
        i = tuple(int(j) for j in (~ok).nonzero()[0])
        raise AssertionError(f"{what}: {int((~ok).sum())} elements out of bound, first at {i}: "
                             f"got {got[i].item()!r} ref {ref[i].item()!r} bound {bound[i].item():.3e}")


# ---- 1. every shape x path ---------------------------------------------------------------------------------------------
SCALES = [(True, True), (False, False), (True, False), (False, True)]   # (input scale per row, residual scale per row)


@pytest.mark.parametrize("has_value", [True, False], ids=["value", "novalue"])
@pytest.mark.parametrize("K", KS + (2064,))
def test_residual_vs_replay(mat, K, has_value):
    rowptr_c, col_c, M, N = mat["rowptr"], mat["col"], mat["M"], mat["N"]
    E = col_c.numel()
    rowptr, col = _dev(rowptr_c, col_c)
    plan = ops.spmm_plan(rowptr, E)
    assert plan.n_long > 0 and plan.n_seg > plan.n_long
    outs = OUTS if K <= 2048 else OUTS[:3]     # a second column tile: no e4m3 result
    for per_row_in, per_row_res in SCALES:
        x8_c = make_x8(N, K, K, False)
        sc_c = make_scale(N, K + 2, per_row_in)
        v_c = make_values(E, K + 3, False) if has_value else None
        r8_c, rsc_c = make_residual(M, K, K + 4, per_row_res)
        rep = Replay(rowptr_c, col_c, v_c, x8_c, sc_c)
        rho = rho_of(r8_c, rsc_c)
        x8, sc, v, r8, rsc = _dev(x8_c, sc_c, v_c, r8_c, rsc_c)
        for reduce in ("sum", "mean"):
            for out_dtype in outs:
                what = f"K={K} value={has_value} scales={per_row_in, per_row_res} {reduce} {out_dtype}"
                check_vs_replay(rowptr, col, v, x8, sc, r8, rsc, r8_c, rsc_c, reduce, out_dtype, plan,
                                what + " planned")
                vo = v if v is None or out_dtype in (torch.float32, E4M3) else v.to(out_dtype)
                out, ys, _ = call_res(rowptr, col, vo, x8, sc, r8, rsc, reduce, out_dtype)
                bound_check(out, ys, rep, reduce, rho, out_dtype, what + " unplanned")
    # exact sums: the unplanned result is bit-equal whatever order the kernel adds in
    x8_c, sc_c, v_c = exact_operands(N, K, E, K + 5, True)
    r8_c, rsc_c = make_residual(M, K, K + 6, True)
    rsc_c = torch.ldexp(torch.ones(M), torch.randint(-3, 1, (M,), generator=torch.Generator().manual_seed(K)))
    x8, sc, v, r8, rsc = _dev(x8_c, sc_c, v_c if has_value else None, r8_c, rsc_c)
    for reduce in ("sum", "mean"):
        for out_dtype in outs:
            what = f"K={K} exact {reduce} {out_dtype}"
            for p in (None, plan):
                check_vs_replay(rowptr, col, v, x8, sc, r8, rsc, r8_c, rsc_c, reduce, out_dtype, p,
                                what + (" planned" if p else " unplanned"))


# ---- 2. edge rows ------------------------------------------------------------------------------------------------------
def edge_residual(K):
    """edge_problem with every 8th row emptied (rows 7 mod 8), and a residual per row kind (row mod 8): NaN in r8,
    r_scale 3e38 times +-448 (+-inf), a zero residual under the subnormal rows, a -0 residual, +-448 times 50
    (far past the row's own amax), e4m3 subnormals, ordinary values (rows 0 and 7; rows 15 mod 16 get -0)."""
    rowptr_c, col_c, v_c, x8_c = edge_problem(K)
    M = rowptr_c.numel() - 1
    row = torch.repeat_interleave(torch.arange(M), rowptr_c[1:] - rowptr_c[:-1])
    keep = row % 8 != 7
    deg = torch.bincount(row[keep], minlength=M)
    rowptr_c = torch.zeros(M + 1, dtype=torch.long)
    rowptr_c[1:] = deg.cumsum(0)
    col_c, v_c = col_c[keep], v_c[keep]
    g = torch.Generator().manual_seed(K + 1)
    r = torch.randn(M, K, generator=g) * 4
    rs = torch.rand(M, generator=g) + 0.25
    kind = torch.arange(M) % 8
    r[kind == 1, 5] = float("nan")
    r[kind == 2] = torch.where(r[kind == 2] > 0, 448.0, -448.0)
    rs[kind == 2] = 3e38
    r[kind == 3] = 0.0
    r[kind == 4] = -0.0
    r[kind == 5] = torch.where(r[kind == 5] > 0, 448.0, -448.0)
    rs[kind == 5] = 50.0
    r[kind == 6] = torch.ldexp(torch.ones(K), torch.randint(-9, -6, (K,), generator=g).int())
    r[torch.arange(M) % 16 == 15] = -0.0
    return rowptr_c, col_c, v_c, x8_c, r.to(E4M3), rs


@pytest.mark.parametrize("K", (16, 128, 256, 1024))
def test_residual_edge_rows(K):
    rowptr_c, col_c, v_c, x8_c, r8_c, rsc_c = edge_residual(K)
    M = rowptr_c.numel() - 1
    rowptr, col, v, x8, r8, rsc = _dev(rowptr_c, col_c, v_c, x8_c, r8_c, rsc_c)
    plan = ops.spmm_plan(rowptr, col.numel())
    empty = torch.arange(M) % 8 == 7
    negz = torch.arange(M) % 16 == 15
    seen = dict(nan=False, inf=False, big_scale=False, subnormal=False, neg_zero_row=False)
    for per_row in (True, False):
        sc = _dev(make_scale(64, K, per_row, pow2=True))[0]
        for reduce in ("sum", "mean"):
            for out_dtype in OUTS:
                for p in (plan, None):
                    what = f"K={K} per_row={per_row} {reduce} {out_dtype} {'planned' if p else 'unplanned'}"
                    out, ys = check_vs_replay(rowptr, col, v, x8, sc, r8, rsc, r8_c, rsc_c, reduce, out_dtype, p, what)
                    # empty rows are exactly the rounded / quantised rho; a -0 residual there gives +0
                    rho = rho_of(r8_c, rsc_c)[empty]
                    ref = finish(torch.zeros_like(rho) + rho, out_dtype)
                    if out_dtype == E4M3:
                        assert_q_equal(out[empty.to(DEV)], ys[empty.to(DEV)], ref[0], ref[1], what + " empty rows")
                        b = out.cpu().view(torch.uint8)
                        assert bool((b[negz] == 0).all()) and bool((ys.cpu()[negz] == 1).all())
                        s = ys.cpu()
                        seen["inf"] |= bool(s.isinf().any())
                        seen["big_scale"] |= bool(((s > 1) & s.isfinite()).any())
                        seen["subnormal"] |= bool((((b & 0x78) == 0) & ((b & 0x07) != 0)).any())
                        seen["nan"] |= bool(_nan8(b).any())
                    else:
                        assert_out_equal(out[empty.to(DEV)], None, ref, what + " empty rows")
                        o = out.cpu().float()
                        assert bool((o[negz] == 0).all()) and not bool(o[negz].signbit().any())
                        seen["inf"] |= bool(o.isinf().any())
                        seen["nan"] |= bool(o.isnan().any())
                    seen["neg_zero_row"] = True
    assert all(seen.values()), seen


@pytest.mark.parametrize("out_dtype", OUTS, ids=lambda d: str(d).replace("torch.", ""))
def test_residual_empty_matrix(out_dtype):
    """E == 0 with a residual: every row is fl32(+0 + rho), rounded or quantised (a -0 residual gives +0)."""
    M, N, K = 37, 50, 64
    r8_c, rsc_c = make_residual(M, K, 9, True)
    r8_c[3] = -0.0
    r8_c[4, 7] = float("nan")
    rowptr, col = _dev(torch.zeros(M + 1, dtype=torch.long), torch.empty(0, dtype=torch.long))
    x8, sc, r8, rsc = _dev(torch.zeros(N, K).to(E4M3), torch.ones(N), r8_c, rsc_c)
    for reduce in ("sum", "mean"):
        out, ys, _ = call_res(rowptr, col, None, x8, sc, r8, rsc, reduce, out_dtype)
        rho = rho_of(r8_c, rsc_c)
        assert_out_equal(out, ys, finish(torch.zeros_like(rho) + rho, out_dtype), f"E=0 {reduce} {out_dtype}")
        if out_dtype != E4M3:
            assert not bool(out.cpu().float()[3].signbit().any())
    # through the public API
    a0 = ts.SparseTensor(row=torch.empty(0, dtype=torch.long, device=DEV),
                         col=torch.empty(0, dtype=torch.long, device=DEV), sparse_sizes=(M, N))
    rho = rho_of(r8_c, rsc_c)
    if out_dtype == E4M3:
        y8, ys = a0.spmm_fp8_quant(x8, sc, residual=r8, residual_scale=rsc)
        assert_out_equal(y8, ys, finish(torch.zeros_like(rho) + rho, out_dtype), "E=0 public")
    else:
        out = a0.spmm_fp8(x8, sc, "mean", out_dtype, residual=r8, residual_scale=rsc)
        assert_out_equal(out, None, finish(torch.zeros_like(rho) + rho, out_dtype), "E=0 public")


# ---- 3. no change without a residual -------------------------------------------------------------------------------
@pytest.mark.parametrize("K", (64, 256, 2048))
def test_no_residual_is_unchanged(mat, K):
    """res8 = NULL: the new entry point is bit-identical to tsb200_spmm_fw_fp8 / _quant, min / max included."""
    rowptr_c, col_c, N = mat["rowptr"], mat["col"], mat["N"]
    E = col_c.numel()
    rowptr, col = _dev(rowptr_c, col_c)
    plan = ops.spmm_plan(rowptr, E)
    x8, sc, v = _dev(make_x8(N, K, K, False), make_scale(N, K, True), make_values(E, K, False))
    for reduce in ("sum", "mean", "min", "max"):
        for p in (plan, None):
            for out_dtype in OUTS:
                what = f"K={K} {reduce} {out_dtype} {'planned' if p else 'unplanned'}"
                if out_dtype == E4M3:
                    y8, ys, arg = call_quant(rowptr, col, v, x8, sc, reduce, plan=p)
                    out, ys2, arg2 = call_res(rowptr, col, v, x8, sc, None, None, reduce, out_dtype, plan=p)
                    assert torch.equal(out.view(torch.uint8), y8.view(torch.uint8)), what
                    assert torch.equal(ys.view(torch.int32), ys2.view(torch.int32)), what
                else:
                    vo = v.to(out_dtype)
                    y, arg = call_fp8(rowptr, col, vo, x8, sc, reduce, out_dtype, plan=p)
                    out, _, arg2 = call_res(rowptr, col, vo, x8, sc, None, None, reduce, out_dtype, plan=p)
                    bits = {2: torch.int16, 4: torch.int32}[y.element_size()]
                    assert torch.equal(out.view(bits), y.view(bits)), what
                if arg is not None:
                    assert torch.equal(arg, arg2), what


# ---- 4. chained propagation ------------------------------------------------------------------------------------------
def propagate(M, K, coef_a, coef_r, x0, h, hops, seed):
    """hops of X <- coef_a A X + coef_r H in e4m3 through the public API (entry values times coef_a, r_scale times
    coef_r, folded once), against fp64 propagation of the dequantised x_0 and H. The bound extends the one of
    test_spmm_fp8_quant_gpu.test_chained_hops: with x_h the dequantised operand of hop h and z the fp32 result,
        e_{h+1} = |A'| e_h + (deg + 4) 2^-24 |A'| |x_h|        (the fp32 chain, the weight, the coef_a fold and
                                                               coef_a's own fp32 rounding)
                  + 3 * 2^-24 |coef_r H| + 2^-24 |z|           (the r_scale fold and coef_r's rounding, the product;
                                                               the add)
                  + 1/2 ulp_e4m3(z / s) s (1 + 2^-22) + 2^-22 |z|
    with A' = coef_a A. Returns the largest error / bound over the hops."""
    rowptr_c, col_c = build_csr(M, M, 6, seed, {10: 300, 11: 900}, blocks=[128], tie_rows={},
                                empty_rows=(0, M // 3))
    E = col_c.numel()
    deg = (rowptr_c[1:] - rowptr_c[:-1]).double().view(-1, 1)
    row = torch.repeat_interleave(torch.arange(M), deg.view(-1).long())
    g = torch.Generator().manual_seed(seed)
    v_c = torch.rand(E, generator=g) + 0.1
    v_c = v_c / deg.view(-1)[row].float()          # a row-stochastic A
    x8, sc = ts.quantize_fp8(x0, per_row=True)
    h8, hs = ts.quantize_fp8(h, per_row=True)
    rowptr, col = _dev(rowptr_c, col_c)
    a = ts.SparseTensor(rowptr=rowptr, col=col, value=(v_c * coef_a).to(DEV), sparse_sizes=(M, M))
    A = torch.sparse_csr_tensor(rowptr_c, col_c, v_c.double() * coef_a, (M, M))
    Aabs = torch.sparse_csr_tensor(rowptr_c, col_c, (v_c.double() * coef_a).abs(), (M, M))
    H = h8.double() * hs.double().view(-1, 1)
    ref = x8.double() * sc.double().view(-1, 1)
    e = torch.zeros(M, K, dtype=torch.float64)
    x8, sc, h8d, rs = _dev(x8, sc, h8, hs * coef_r)
    worst = 0.0
    for _ in range(hops):
        xh = x8.cpu().double() * sc.cpu().double().view(-1, 1)
        x8, sc = a.spmm_fp8_quant(x8, sc, residual=h8d, residual_scale=rs)
        q, s = x8.cpu().double(), sc.cpu().double().view(-1, 1)
        got = q * s
        hu = e4m3_half_ulp(q) * s
        zabs = got.abs() + hu
        ref = A @ ref + coef_r * H
        e = (Aabs @ e + (deg + 4) * U32 * (Aabs @ xh.abs()) + 3 * U32 * (coef_r * H).abs() + U32 * zabs
             + hu * (1 + 2.0 ** -22) + 2.0 ** -22 * zabs)
        err = (got - ref).abs()
        assert bool((err <= e).all()), f"max err / bound {float((err / e).nan_to_num(0).max()):.3f}"
        worst = max(worst, float((err / e).nan_to_num(0).max()))
        assert float(got.abs().max()) > 0
    return worst


def test_appnp_hops():
    """10 APPNP hops X <- (1 - a) A X + a H, a = 0.1, H = X_0."""
    M, K = 3000, 128
    g = torch.Generator().manual_seed(8)
    x0 = torch.randn(M, K, generator=g)
    propagate(M, K, 0.9, 0.1, x0, x0, 10, 7)


def test_label_propagation_hops():
    """5 label-propagation hops Y <- a A Y + (1 - a) Y_0, a = 0.9, one-hot Y_0 over 40 classes padded to K = 48."""
    M, K = 3000, 48
    g = torch.Generator().manual_seed(9)
    y0 = torch.zeros(M, K)
    y0[torch.arange(M), torch.randint(40, (M,), generator=g)] = 1.0
    y0[torch.rand(M, generator=g) < 0.5] = 0.0            # unlabelled nodes
    propagate(M, K, 0.9, 0.1, y0, y0, 5, 5)


# ---- 5. public API -----------------------------------------------------------------------------------------------------
def test_residual_public_api(mat):
    g = torch.Generator().manual_seed(4)
    M, N, E = mat["M"], mat["N"], mat["col"].numel()
    rowptr, col = _dev(mat["rowptr"], mat["col"])
    # values exact in bf16, so the bf16 result (values cast to bf16) and the f32 one sum the same terms
    a = ts.SparseTensor(rowptr=rowptr, col=col, value=torch.randn(E, generator=g).bfloat16().float().to(DEV),
                        sparse_sizes=(M, N))
    x8, sc = ts.quantize_fp8(torch.randn(N, 64, generator=g).to(DEV), per_row=True)
    r8, rs = ts.quantize_fp8(torch.randn(M, 64, generator=g).to(DEV), per_row=True)
    for _ in range(2):   # from here on every call uses the cached plan of `a`
        ts.spmm_fp8(a, x8, sc)
    for reduce in ("sum", "mean"):
        y = ts.spmm_fp8(a, x8, sc, reduce, torch.float32).cpu()
        z = y + rho_of(r8.cpu(), rs.cpu())
        for out_dtype in (torch.bfloat16, torch.float32):
            out = a.spmm_fp8(x8, sc, reduce, out_dtype, residual=r8, residual_scale=rs)
            assert_out_equal(out, None, z.to(out_dtype), f"public {reduce} {out_dtype}")
        y8, ys = a.spmm_fp8_quant(x8, sc, reduce, residual=r8, residual_scale=rs)
        ref8, refs = ts.quantize_fp8(z, per_row=True)
        assert_q_equal(y8, ys, ref8, refs, f"public quant {reduce}")
        y8b, ysb = ts.spmm_fp8_quant(a, x8, sc, reduce, r8, rs)
        assert torch.equal(y8.view(torch.uint8), y8b.view(torch.uint8)) and torch.equal(ys, ysb)
    # "add" is "sum"; a per-tensor residual scale
    y8, ys = ts.spmm_fp8_quant(a, x8, sc, "sum", r8, rs[5])
    y8a, ysa = ts.spmm_fp8_quant(a, x8, sc, "add", r8, rs[5])
    assert torch.equal(y8.view(torch.uint8), y8a.view(torch.uint8)) and torch.equal(ys, ysa)
    # the registered operators, with and without the new arguments
    rowptr_s, col_s, val_s = a.csr()
    out0, _ = torch.ops.tsb200.spmm_fp8(rowptr_s, col_s, val_s.bfloat16(), x8, sc, "sum", torch.bfloat16)
    assert torch.equal(out0, ts.spmm_fp8(a, x8, sc))
    out1, _ = torch.ops.tsb200.spmm_fp8(rowptr_s, col_s, val_s.bfloat16(), x8, sc, "sum", torch.bfloat16,
                                        residual=r8, residual_scale=rs)
    assert torch.equal(out1, a.spmm_fp8(x8, sc, residual=r8, residual_scale=rs))
    q0 = torch.ops.tsb200.spmm_fp8_quant(rowptr_s, col_s, val_s, x8, sc, "sum")
    q1 = torch.ops.tsb200.spmm_fp8_quant(rowptr_s, col_s, val_s, x8, sc, "sum", r8, rs)
    assert torch.equal(q0[0].view(torch.uint8), a.spmm_fp8_quant(x8, sc)[0].view(torch.uint8))
    assert torch.equal(q1[0].view(torch.uint8), a.spmm_fp8_quant(x8, sc, residual=r8, residual_scale=rs)[0]
                       .view(torch.uint8))
    # the result of one hop is the next hop's operand (and residual)
    sq = ts.SparseTensor(row=torch.randint(M, (4 * M,), generator=g).to(DEV),
                         col=torch.randint(M, (4 * M,), generator=g).to(DEV), sparse_sizes=(M, M)).coalesce()
    y8, ys = a.spmm_fp8_quant(x8, sc, residual=r8, residual_scale=rs)
    for _ in range(2):   # the plan of `sq`
        ts.spmm_fp8(sq, y8, ys)
    y8n, ysn = sq.spmm_fp8_quant(y8, ys, residual=y8, residual_scale=ys)
    z = ts.spmm_fp8(sq, y8, ys, "sum", torch.float32).cpu() + rho_of(y8.cpu(), ys.cpu())
    ref8, refs = ts.quantize_fp8(z, per_row=True)
    assert_q_equal(y8n, ysn, ref8, refs, "second hop")


# ---- 6. errors ---------------------------------------------------------------------------------------------------------
def test_residual_errors(mat):
    M, N, E = mat["M"], mat["N"], mat["col"].numel()
    rowptr, col = _dev(mat["rowptr"], mat["col"])
    x8 = torch.zeros(N, 32, device=DEV).to(E4M3)
    sc = torch.ones(N, device=DEV)
    r8 = torch.zeros(M, 32, device=DEV).to(E4M3)
    rs = torch.ones(M, device=DEV)

    # the C-ABI: min / max, misaligned res8 / res_scale, K > 2048 with an e4m3 result
    for reduce in ("min", "max"):
        for out_dtype in (torch.bfloat16, E4M3):
            call_res(rowptr, col, None, x8, sc, r8, rs, reduce, out_dtype, expect_rc=ERR_UNSUPPORTED)
    rbuf = torch.zeros(M * 32 + 16, dtype=torch.uint8, device=DEV).view(E4M3)
    call_res(rowptr, col, None, x8, sc, rbuf[:M * 32].view(M, 32), rs, "sum", torch.float32, r8_off=1,
             expect_rc=ERR_UNSUPPORTED)
    call_res(rowptr, col, None, x8, sc, r8, torch.ones(M + 1, device=DEV), "sum", E4M3, rsc_off=2,
             expect_rc=ERR_UNSUPPORTED)
    wide = torch.zeros(N, 2064, device=DEV).to(E4M3)
    call_res(rowptr, col, None, wide, sc, torch.zeros(M, 2064, device=DEV).to(E4M3), rs, "sum", E4M3,
             expect_rc=ERR_UNSUPPORTED)

    # the Python layers
    a = ts.SparseTensor(rowptr=rowptr, col=col, value=torch.ones(E, device=DEV), sparse_sizes=(M, N))

    def raises(fn, match):
        with pytest.raises(RuntimeError, match=match):
            fn()
    for f in (lambda **kw: a.spmm_fp8(x8, sc, "sum", torch.float32, **kw), lambda **kw: a.spmm_fp8_quant(x8, sc, **kw)):
        raises(lambda: f(residual=r8.float(), residual_scale=rs), "float8_e4m3fn")
        raises(lambda: f(residual=torch.zeros(M, 48, device=DEV).to(E4M3), residual_scale=rs), r"shape \[M, K\]")
        raises(lambda: f(residual=r8[:-1], residual_scale=rs), r"shape \[M, K\]")
        raises(lambda: f(residual=r8), "both or neither")
        raises(lambda: f(residual_scale=rs), "both or neither")
        raises(lambda: f(residual=r8, residual_scale=torch.ones(M + 1, device=DEV)), r"shape \[\] or \[M\]")
        raises(lambda: f(residual=r8, residual_scale=rs.double()), "float32")
        raises(lambda: f(residual=r8.cpu(), residual_scale=rs), "must be CUDA tensor")
        raises(lambda: f(residual=r8, residual_scale=rs.clone().requires_grad_()), "forward only")
        with torch.no_grad():
            f(residual=r8, residual_scale=rs.clone().requires_grad_())
    for reduce in ("min", "max"):
        raises(lambda: a.spmm_fp8(x8, sc, reduce, residual=r8, residual_scale=rs), "sum")
        raises(lambda: a.spmm_fp8_quant(x8, sc, reduce, residual=r8, residual_scale=rs), "sum")
