"""SpMM over an FP8 (e4m3) dense operand (tsb200_spmm_fw_fp8, `spmm_fp8`): every dispatch shape, reduction, output
dtype, value / no value and per-tensor / per-row scale, planned and unplanned, against an exact replay on the CPU.

The library is called directly with outputs prefilled with NaN (arg_out with -1), so an element a kernel fails to write
cannot pass on what the allocator left in the buffer. The structured matrix (`build_csr` of the kernel-family tests)
has empty rows, rows of 1 ... 1300 nnz (multi-segment rows past 256), a 32-row block over the 1024-nnz item budget and
rows with duplicate columns (tied extrema); dense rows no entry references are NaN.

Semantics replayed (entry e, column c): w_e = fl32(v_e * scale[c]), q = x8[c, k] widened to fp32 (exact).
  sum / mean: checked in fp64 against ref = sum_e v_e s_c q (each term exact in fp64). The kernel rounds w_e once
  (relative 2^-24), folds deg terms with FFMA (one rounding each), the mean divides once, and the result is rounded
  once to the output dtype; as in util.segment_sum_ref_bound this gives, with S = sum_e |v_e s_c q|,
      |out - ref| <= 1/2 ulp_out(|ref| + e) + e,   e = (deg + 2) 2^-24 S  (divided by max(deg, 1) for the mean)
  (deg + 1 roundings of the fp32 chain plus the weight's, and one spare for the division and second-order terms).
  min / max: p = round_out(fl32(w_e * q)) compared strictly, the smallest e wins ties, out = p: replayed with the
  same fp32 operations in torch and compared bit for bit, arg_out included.
"""
import ctypes

import pytest
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import ops
from pytorch_sparse_b200._lib import lib
from test_spmm_kernels_gpu import NAN_ROWS, build_csr, half_ulp, plan_budget_rows, unreferenced_rows

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U32 = 2.0 ** -24
ERR_UNSUPPORTED = -2
OUTS = (torch.bfloat16, torch.float16, torch.float32)
REDUCES = ("sum", "mean", "min", "max")
# every dispatch shape (dense-row bytes = K: group-per-row 16..128 B, vec16, vec32 CH = 1, 2, 4), partial widths
# (a vector count that is not a power of two) and a second column tile
KS = (16, 32, 64, 128, 256, 512, 1024, 2048)
KS_PARTIAL = (48, 400, 2064)


def _id(p):
    return str(p).replace("torch.", "")


@pytest.fixture(scope="module")
def mat():
    M, N = 32 * 40 + 13, 3000
    specials = {5: 1, 37: 31, 38: 32, 39: 33, 200: 255, 201: 256, 202: 257, 500: 512, 501: 513, 900: 1300}
    rowptr, col = build_csr(M, N, 4, 11, specials, blocks=[64], tie_rows={300: 40, 301: 600},
                            empty_rows=(0, M // 2, M - 1))
    return dict(M=M, N=N, rowptr=rowptr, col=col)


# ---- operands ----------------------------------------------------------------------------------------------------------
E4M3_SPECIAL = torch.tensor([float("nan"), 0.0, -0.0])


def make_x8(N, K, seed, ties):
    """e4m3 [N, K]: randn / 4-ish magnitudes (sums), or few distinct values with NaN and +-0 (min/max, many ties).
    Unreferenced rows are NaN."""
    g = torch.Generator().manual_seed(seed)
    if ties:
        x = torch.tensor([-2.0, -1.0, -0.5, 0.5, 1.0, 3.0])[torch.randint(6, (N, K), generator=g)]
        pick = torch.rand(N, K, generator=g) < 0.08
        x = torch.where(pick, E4M3_SPECIAL[torch.randint(3, (N, K), generator=g)], x)
    else:
        x = torch.randn(N, K, generator=g) * 4
    x[unreferenced_rows(N)] = float("nan")
    return x.to(torch.float8_e4m3fn)


def make_scale(N, seed, per_row, pow2=False):
    g = torch.Generator().manual_seed(seed)
    if pow2:
        s = torch.ldexp(torch.ones(N), torch.randint(-3, 4, (N,), generator=g))
    else:
        s = torch.rand(N, generator=g) * 1.5 + 0.05
    return s if per_row else s[7].clone()


def make_values(E, seed, ties):
    """multiples of 1/64 in [-4, 4] (exact in bf16, f16 and f32, so one value array serves every out dtype)."""
    g = torch.Generator().manual_seed(seed)
    if ties:
        return torch.tensor([-1.0, -0.5, 0.5, 1.0, 2.0, 0.0, -0.0])[torch.randint(7, (E,), generator=g)]
    return torch.randint(-256, 257, (E,), generator=g).float() / 64


# ---- direct library calls ----------------------------------------------------------------------------------------------
def _vp(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def call_fp8(rowptr, col, value, x8, scale, reduce, out_dtype, plan=None, expect_rc=0):
    """tsb200_spmm_fw_fp8 into NaN / -1 prefilled outputs; unplanned when plan is None."""
    M, E = rowptr.numel() - 1, col.numel()
    N, K = x8.shape
    red, dt = ops._REDUCE[reduce], ops._FP8_OUT.get(out_dtype, 1)
    out = torch.full((M, K), float("nan"), dtype=out_dtype, device=DEV)
    arg = torch.full((M, K), -1, dtype=torch.int64, device=DEV) if red >= 2 else None
    if plan is None:
        nws = lib.tsb200_spmm_fw_workspace_bytes(1, M, K, E, 0, red)
        pl, plb, counts = None, 0, (0, 0, 0)
    else:
        nws = lib.tsb200_spmm_fw_planned_workspace_bytes(K, plan.n_long, plan.n_slot, red)
        pl, plb, counts = _vp(plan.data), plan.data.numel(), (plan.n_seg, plan.n_long, plan.n_slot)
    ws = torch.empty(max(nws, 256), dtype=torch.uint8, device=DEV)
    stride = 0 if scale.dim() == 0 else 1
    rc = lib.tsb200_spmm_fw_fp8(_vp(rowptr), _vp(col), _vp(value), _vp(x8), _vp(scale), stride, _vp(out), _vp(arg),
                                M, N, K, E, dt, red, pl, plb, *counts, _vp(ws), nws,
                                ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == expect_rc, rc
    return out, arg


# ---- the replay -------------------------------------------------------------------------------------------------------
class Replay:
    """CPU reference of one (matrix, value, x8, scale): exact fp64 sums and |terms|, and the fp32 min/max replay."""

    def __init__(self, rowptr, col, value, x8, scale):
        self.rowptr, self.col = rowptr, col
        M, E = rowptr.numel() - 1, col.numel()
        self.M, self.E = M, E
        deg = rowptr[1:] - rowptr[:-1]
        self.row = torch.repeat_interleave(torch.arange(M), deg)
        self.deg = deg.double().view(-1, 1)
        self.cnt = self.deg.clamp(min=1)
        self.q = x8.float()[col]                                   # [E, K], exact
        self.v = torch.ones(E) if value is None else value.float()
        self.s = scale[col] if scale.dim() == 1 else scale.expand(E)
        self.w = self.v * self.s                                    # fl32(v * s)
        self._sum = None

    def sums(self):
        if self._sum is None:
            t = (self.v.double() * self.s.double()).view(-1, 1) * self.q.double()
            K = t.size(1)
            ref = torch.zeros(self.M, K, dtype=torch.float64).index_add_(0, self.row, t)
            S = torch.zeros(self.M, K, dtype=torch.float64).index_add_(0, self.row, torch.nan_to_num(t.abs(), nan=0.0))
            self._sum = ref, S
        return self._sum

    def minmax(self, reduce, out_dtype):
        E, K = self.E, self.q.size(1)
        p = (self.w.view(-1, 1) * self.q).to(out_dtype).float()
        fin = torch.finfo(out_dtype)
        is_min = reduce == "min"
        init = fin.max if is_min else fin.min
        hole = float("inf") if is_min else -float("inf")
        cand = (p < init) if is_min else (p > init)               # False on NaN
        key = torch.where(cand, p, torch.full_like(p, hole))
        idx = self.row.view(-1, 1).expand(E, K)
        ext = torch.full((self.M, K), hole).scatter_reduce(0, idx, key, "amin" if is_min else "amax")
        win = cand & (key == ext[self.row])
        first = torch.where(win, torch.arange(E).view(-1, 1).expand(E, K), torch.full((E, K), E))
        arg = torch.full((self.M, K), E, dtype=torch.int64).scatter_reduce(0, idx, first, "amin")
        val = torch.where(arg < E, p.gather(0, arg.clamp(max=max(E - 1, 0))), torch.full((self.M, K), init))
        val = torch.where(self.deg == 0, torch.zeros_like(val), val)
        return val.to(out_dtype), arg

    def check(self, reduce, out, arg, out_dtype, what):
        if reduce in ("min", "max"):
            ref, rarg = self.minmax(reduce, out_dtype)
            assert_bits_equal(out, ref, f"{what} {reduce} out")
            assert torch.equal(arg.cpu(), rarg), f"{what} {reduce}: arg_out differs"
            return
        ref, S = self.sums()
        e = (self.deg + 2) * U32 * S
        if reduce == "mean":
            ref, e = ref / self.cnt, e / self.cnt
        o = out.cpu().double()
        bound = e + half_ulp(ref.abs() + e, out_dtype)
        ok = (o - ref).abs() <= bound
        if not bool(ok.all()):
            i = tuple(int(j) for j in (~ok).nonzero()[0])
            raise AssertionError(f"{what} {reduce}: {int((~ok).sum())} elements out of bound, first at {i}: "
                                 f"out {o[i].item()!r} ref {ref[i].item()!r} bound {bound[i].item():.3e}")


def bits(t):
    t = t.cpu().contiguous()
    return t.view({2: torch.int16, 4: torch.int32}[t.element_size()])


def assert_bits_equal(a, b, what=""):
    x, y = bits(a), bits(b)
    ok = x == y
    if not bool(ok.all()):
        i = tuple(int(j) for j in (~ok).nonzero()[0])
        raise AssertionError(f"{what}: {int((~ok).sum())} elements differ, first at {i}: "
                             f"{a.cpu()[i].item()!r} vs {b.cpu()[i].item()!r}")


def _dev(*ts_):
    return [None if t is None else t.to(DEV) for t in ts_]


# ---- every shape x reduction x out dtype x value x scale, planned and unplanned -------------------------------------
@pytest.mark.parametrize("per_row", [True, False], ids=["rowscale", "tensorscale"])
@pytest.mark.parametrize("has_value", [True, False], ids=["value", "novalue"])
@pytest.mark.parametrize("K", KS + KS_PARTIAL)
def test_fp8_vs_replay(mat, K, has_value, per_row):
    rowptr_c, col_c, N = mat["rowptr"], mat["col"], mat["N"]
    E = col_c.numel()
    rowptr, col = _dev(rowptr_c, col_c)
    plan = ops.spmm_plan(rowptr, E)
    assert plan.n_long > 0 and plan.n_seg > plan.n_long
    budget = plan_budget_rows(rowptr_c)
    assert budget.any()
    for ties, reduces in ((False, ("sum", "mean")), (True, ("min", "max"))):
        x8_c = make_x8(N, K, K + ties, ties)
        sc_c = make_scale(N, K + 2, per_row)
        v_c = make_values(E, K + 3, ties) if has_value else None
        rep = Replay(rowptr_c, col_c, v_c, x8_c, sc_c)
        x8, sc = _dev(x8_c, sc_c)
        for out_dtype in OUTS:
            v = None if v_c is None else v_c.to(out_dtype).to(DEV)
            for reduce in reduces:
                what = f"K={K} {_id(out_dtype)} value={has_value} per_row={per_row}"
                out_u, arg_u = call_fp8(rowptr, col, v, x8, sc, reduce, out_dtype)
                rep.check(reduce, out_u, arg_u, out_dtype, what + " unplanned")
                out_p, arg_p = call_fp8(rowptr, col, v, x8, sc, reduce, out_dtype, plan=plan)
                rep.check(reduce, out_p, arg_p, out_dtype, what + " planned")
                if reduce in ("min", "max"):
                    assert_bits_equal(out_p, out_u, what + " planned vs unplanned")
                    assert torch.equal(arg_p, arg_u)
                elif K <= 128:
                    # group-per-row kernel: a row the plan defers for the item budget is summed by the segment kernel's
                    # lane groups instead (DESIGN §3.1); every other row is bit-identical
                    keep = ~budget.to(DEV)
                    assert_bits_equal(out_p[keep], out_u[keep], what + " planned vs unplanned")
                else:
                    assert_bits_equal(out_p, out_u, what + " planned vs unplanned")


def test_fp8_nan_in_sums(mat):
    """A NaN in x8 makes exactly the sums that gather it NaN (sum and mean, planned and unplanned)."""
    rowptr_c, col_c, N = mat["rowptr"], mat["col"], mat["N"]
    E = col_c.numel()
    rowptr, col = _dev(rowptr_c, col_c)
    plan = ops.spmm_plan(rowptr, E)
    x8_c = make_x8(N, 256, 5, ties=True)       # NaN, +-0 and ties
    sc_c = make_scale(N, 6, True)
    rep = Replay(rowptr_c, col_c, None, x8_c, sc_c)
    ref, _ = rep.sums()
    x8, sc = _dev(x8_c, sc_c)
    for reduce in ("sum", "mean"):
        for p in (None, plan):
            out, _ = call_fp8(rowptr, col, None, x8, sc, reduce, torch.float32, plan=p)
            assert torch.equal(out.cpu().isnan(), ref.isnan()), f"{reduce}: NaN pattern"


# ---- the public function, cross-checks --------------------------------------------------------------------------------
def _sparse(mat, value):
    rowptr, col = _dev(mat["rowptr"], mat["col"])
    return ts.SparseTensor(rowptr=rowptr, col=col, value=value, sparse_sizes=(mat["M"], mat["N"]))


@pytest.mark.parametrize("per_row", [True, False], ids=["rowscale", "tensorscale"])
def test_fp8_matches_f32_matmul(mat, per_row):
    """f32 output against the existing matmul on the dequantised operand x8.float() * scale: with power-of-two scales
    both paths form the same exact products, so min/max values and arg_out agree bit for bit; sums agree within the
    bound (the two kernels add a row's terms in different orders)."""
    N, E = mat["N"], mat["col"].numel()
    K = 128
    for ties, reduces in ((False, ("sum", "mean")), (True, ("min", "max"))):
        x8_c = make_x8(N, K, 21 + ties, ties)
        x8_c[unreferenced_rows(N)] = 0.0     # the dequantised operand must not differ from x8 where nothing reads it
        sc_c = make_scale(N, 22, per_row, pow2=True)
        v_c = make_values(E, 23, ties)
        x8, sc = _dev(x8_c, sc_c)
        a = _sparse(mat, v_c.to(DEV))
        xd = x8.float() * (sc.view(-1, 1) if per_row else sc)
        rep = Replay(mat["rowptr"], mat["col"], v_c, x8_c, sc_c)
        for reduce in reduces:
            got = ts.spmm_fp8(a, x8, sc, reduce, torch.float32)
            assert got.dtype == torch.float32 and got.shape == (mat["M"], K)
            want = ts.matmul(a, xd, reduce)
            if reduce in ("min", "max"):
                assert_bits_equal(got, want, f"{reduce} vs matmul")
                _, arg = ops.spmm_fw_fp8(a.storage.rowptr(), a.storage.col(), a.storage.value(), x8, sc, reduce,
                                         torch.float32)
                _, arg_ref = ops.spmm_fw(a.storage.rowptr(), a.storage.col(), a.storage.value(), xd, reduce)
                assert torch.equal(arg, arg_ref)
            else:
                rep.check(reduce, got, None, torch.float32, "spmm_fp8")
                rep.check(reduce, want, None, torch.float32, "matmul")


def test_fp8_public_api(mat):
    """SparseTensor.spmm_fp8, 'add' == 'sum', value cast to out_dtype, quantize_fp8 output accepted, every out dtype."""
    g = torch.Generator().manual_seed(3)
    E = mat["col"].numel()
    a = _sparse(mat, (torch.randn(E, generator=g)).to(DEV))
    x = torch.randn(mat["N"], 64, generator=g).to(DEV)
    for per_row in (True, False):
        x8, sc = ts.quantize_fp8(x, per_row)
        for _ in range(2):   # from here on every call uses the cached plan of `a` (narrow rows: see test_fp8_vs_replay)
            ts.spmm_fp8(a, x8, sc)
        assert x8.dtype == torch.float8_e4m3fn and sc.dtype == torch.float32
        for out_dtype in OUTS:
            s = a.spmm_fp8(x8, sc, "sum", out_dtype)
            assert s.dtype == out_dtype
            assert torch.equal(bits(ts.spmm_fp8(a, x8, sc, "add", out_dtype)), bits(s))
        default = ts.spmm_fp8(a, x8, sc)
        assert default.dtype == torch.bfloat16
    with pytest.raises(ValueError):
        ts.spmm_fp8(a, x8, sc, "prod")


def test_fp8_empty_and_narrow():
    """E == 0 (zeros, arg_out 0), M == 0, and a matrix whose only entries sit in one row."""
    x8 = torch.ones(10, 32, device=DEV).to(torch.float8_e4m3fn)
    sc = torch.ones(10, device=DEV)
    a0 = ts.SparseTensor(row=torch.empty(0, dtype=torch.long, device=DEV),
                         col=torch.empty(0, dtype=torch.long, device=DEV), sparse_sizes=(7, 10))
    for reduce in REDUCES:
        out = ts.spmm_fp8(a0, x8, sc, reduce)
        assert out.shape == (7, 32) and bool((out == 0).all())
    rowptr = torch.zeros(8, dtype=torch.long, device=DEV)
    out, arg = call_fp8(rowptr, torch.empty(0, dtype=torch.long, device=DEV), None, x8, sc, "max", torch.bfloat16)
    assert bool((out.float() == 0).all()) and bool((arg == 0).all())
    a1 = ts.SparseTensor(row=torch.zeros(3, dtype=torch.long, device=DEV), col=torch.tensor([1, 4, 9], device=DEV),
                         sparse_sizes=(3, 10))
    out = ts.spmm_fp8(a1, x8, sc, "sum", torch.float32)
    assert torch.equal(out[0].cpu(), torch.full((32,), 3.0)) and bool((out[1:] == 0).all())


# ---- errors -----------------------------------------------------------------------------------------------------------
def test_fp8_errors(mat):
    N, E = mat["N"], mat["col"].numel()
    rowptr, col = _dev(mat["rowptr"], mat["col"])
    x8 = torch.zeros(N, 32, device=DEV).to(torch.float8_e4m3fn)
    sc = torch.ones(N, device=DEV)
    a = _sparse(mat, torch.ones(E, device=DEV))

    # the C-ABI
    call_fp8(rowptr, col, None, torch.zeros(N, 24, device=DEV).to(torch.float8_e4m3fn), sc, "sum", torch.bfloat16,
             expect_rc=ERR_UNSUPPORTED)
    call_fp8(rowptr, col, None, x8, sc, "sum", torch.float64, expect_rc=ERR_UNSUPPORTED)
    buf = torch.zeros(N * 32 + 1, device=DEV).to(torch.float8_e4m3fn)
    call_fp8(rowptr, col, None, buf[1:].view(N, 32), sc, "sum", torch.bfloat16, expect_rc=ERR_UNSUPPORTED)

    # the Python layers
    def raises(fn, match):
        with pytest.raises(RuntimeError, match=match):
            fn()
    raises(lambda: ts.spmm_fp8(a, torch.zeros(N, 24, device=DEV).to(torch.float8_e4m3fn), sc), "multiple of 16")
    raises(lambda: ts.spmm_fp8(a, torch.zeros(2, N, 32, device=DEV).to(torch.float8_e4m3fn), sc), "2-D")
    raises(lambda: ts.spmm_fp8(a, torch.zeros(N, 32, device=DEV, dtype=torch.bfloat16), sc), "float8_e4m3fn")
    raises(lambda: ts.spmm_fp8(a, torch.zeros(N, 32, device=DEV).to(torch.float8_e5m2), sc), "float8_e4m3fn")
    raises(lambda: ts.spmm_fp8(a, x8, sc.double()), "float32")
    raises(lambda: ts.spmm_fp8(a, x8, torch.ones(N + 1, device=DEV)), r"shape \[\] or \[N\]")
    raises(lambda: ts.spmm_fp8(a, x8, torch.ones(N, 1, device=DEV)), r"shape \[\] or \[N\]")
    raises(lambda: ts.spmm_fp8(a, x8, sc, "sum", torch.float64), "out_dtype")
    raises(lambda: ts.spmm_fp8(a, x8.cpu(), sc), "must be CUDA tensor")
    raises(lambda: ts.spmm_fp8(a, x8, sc.cpu()), "must be CUDA tensor")
    raises(lambda: ops.spmm_fw_fp8(rowptr, col, torch.ones(E, device=DEV), x8, sc, "sum", torch.bfloat16), "dtype")
    # forward only
    raises(lambda: ts.spmm_fp8(a, x8, sc.clone().requires_grad_()), "forward only")
    av = _sparse(mat, torch.ones(E, device=DEV).requires_grad_())
    raises(lambda: ts.spmm_fp8(av, x8, sc), "forward only")
    with torch.no_grad():
        ts.spmm_fp8(av, x8, sc.clone().requires_grad_())
    # matmul / spmm with a float8 operand keep refusing it
    with pytest.raises(RuntimeError):
        ts.matmul(a, x8)
