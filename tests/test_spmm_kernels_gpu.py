"""SpMM forward: every kernel family of the dispatch against the oracle, with error bounds taken from the kernels'
rounding model.

`dispatch_shape` (csrc/spmm_fw.cu) picks a kernel family from the width of a dense row; each family is instantiated
per dtype x reduction x {plain, ACC (column blocks through an fp32 partial), PLAN}. The table below restates that
dispatch; every row of it runs on one structured matrix built to give the queue, the budget deferral, the
multi-segment combine and the tie rules work, and on a large-M variant whose work items are full size (32 rows).

Outputs are prefilled with NaN (arg_out with -1) and the library is called directly, so an element a kernel fails to
write cannot pass on what the allocator left in the buffer.

Bounds (DESIGN §3.1: products of 16-bit values are exact in fp32, accumulated in fp32, rounded once at the store):
  sum   |out - ref64| <= 1/2 ulp_T(ref64) + (deg + 1) * 2^-24 * S,   S = (|A| |B|)[m, k], deg = row length
  mean  the sum's error / deg, plus one fp32 rounding of the division
  acc   P column blocks: deg + P instead of deg + 1
min / max values and arg_out are bit-exact (compared as bit patterns) with the oracle in the storage dtype.
"""
import ctypes
import re

import pytest
import torch

import pytorch_sparse_b200  # noqa: F401  (loads the library)
from pytorch_sparse_b200 import ops
from pytorch_sparse_b200._lib import lib
from util import launched_kernels

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REDUCES = ["sum", "mean", "min", "max"]
U32 = 2.0 ** -24                     # unit roundoff of the fp32 accumulators
ERR_UNSUPPORTED = -2
F16S = (torch.bfloat16, torch.float16)
FLOATS = (torch.float32, torch.bfloat16, torch.float16)

# ---- the dispatch, restated ----------------------------------------------------------------------------------------
# family -> (LPR, CH, U, MINB) of the main kernel; gpr = group-per-row kernel (its CH is 1)
KERNEL = {
    "gpr1": (1, 1, 4, 5), "gpr2": (2, 1, 4, 5), "gpr4": (4, 1, 4, 5), "gpr8": (8, 1, 4, 5),
    "vec16": (16, 1, 6, 3), "vec32ch1": (32, 1, 4, 5), "vec32ch2": (32, 2, 4, 3), "vec32ch4": (32, 4, 2, 3),
    "tiled": (32, 4, 2, 3),
}
# family -> (fp32 K values, 16-bit K values): full width first, then partial width (vector count not a power of two)
FAMILIES = {
    "gpr1": ((4,), (8,)),
    "gpr2": ((8,), (16,)),
    "gpr4": ((16, 12), (32, 24)),
    "gpr8": ((32, 20), (64, 40)),
    "vec16": ((64, 40), (128, 72)),
    "vec32ch1": ((128, 68), (256, 200)),
    "vec32ch2": ((256, 132), (512, 392)),
    "vec32ch4": ((512, 260), (1024, 520)),
    "tiled": ((516, 1100), (1032,)),
}


def family_of(dtype, K, aligned=True):
    """The kernel family tsb200_spmm_fw runs for a dense row of K elements of `dtype`."""
    es = torch.empty(0, dtype=dtype).element_size()
    if dtype not in FLOATS or (K * es) % 16 or not aligned:
        return "generic"
    vecs = K * es // 16
    for lim, fam in ((1, "gpr1"), (2, "gpr2"), (4, "gpr4"), (8, "gpr8"), (16, "vec16"), (32, "vec32ch1"),
                     (64, "vec32ch2"), (128, "vec32ch4")):
        if vecs <= lim:
            return fam
    return "tiled"


def n_tiles(dtype, K):
    vec = 16 // torch.empty(0, dtype=dtype).element_size()
    return -(-K // (32 * 4 * vec))


TABLE = [(dt, K) for fam, (k32, k16) in FAMILIES.items() for dt in FLOATS for K in (k32 if dt == torch.float32 else k16)]
assert all(family_of(dt, K) == fam for fam, (k32, k16) in FAMILIES.items()
           for dt in FLOATS for K in (k32 if dt == torch.float32 else k16))


def _id(p):
    return str(p).replace("torch.", "")


# ---- structured matrices ---------------------------------------------------------------------------------------------
SPECIAL_DEGREES = [1, 31, 32, 33, 255, 256, 257, 512, 513, 4100]
BLOCK_DEG = 48           # 32 rows x 48 nnz = 1536 > the 1024-nnz item budget
NAN_ROWS = 64            # dense rows never referenced by any nnz (column 0 and the last NAN_ROWS - 1): NaN-filled


def build_csr(M, N, mean_deg, seed, specials, blocks, tie_rows, empty_rows):
    """CSR with unsorted, duplicate columns. specials: {row: degree}; blocks: first rows of 32-row blocks of degree
    BLOCK_DEG; tie_rows: {row: degree} whose columns come from 6 dense rows only (duplicate extrema)."""
    g = torch.Generator().manual_seed(seed)
    deg = torch.poisson(torch.full((M,), float(mean_deg)), generator=g).long()
    for r0 in blocks:
        deg[r0:r0 + 32] = BLOCK_DEG
    for r, d in list(specials.items()) + list(tie_rows.items()):
        deg[r] = d
    deg[list(empty_rows)] = 0
    rowptr = torch.zeros(M + 1, dtype=torch.long)
    rowptr[1:] = deg.cumsum(0)
    E = int(rowptr[-1])
    col = torch.randint(1, N - NAN_ROWS + 1, (E,), generator=g)
    tie_cols = torch.randint(1, N - NAN_ROWS + 1, (6,), generator=g)
    for r, d in tie_rows.items():
        col[rowptr[r]:rowptr[r + 1]] = tie_cols[torch.randint(6, (d,), generator=g)]
    return rowptr, col


def unreferenced_rows(N):
    return torch.cat([torch.tensor([0]), torch.arange(N - NAN_ROWS + 1, N)])


@pytest.fixture(scope="module")
def small():
    """M not a multiple of 32; empty rows at 0, M/2, M-1; one row of every degree in SPECIAL_DEGREES; one 32-row
    aligned block over the item budget; two rows (one multi-segment) with duplicate extrema."""
    M, N = 32 * 70 + 13, 4600
    specials = {r: d for r, d in zip([5, 37, 38, 39, 200, 201, 202, 500, 501, 1500], SPECIAL_DEGREES)}
    rowptr, col = build_csr(M, N, 4, 1, specials, blocks=[64], tie_rows={300: 40, 301: 600},
                            empty_rows=(0, M // 2, M - 1))
    return dict(M=M, N=N, rowptr=rowptr, col=col)


LARGE_M = 600_017


@pytest.fixture(scope="module")
def large():
    """About 600k rows: M * B >= 32 * 16 * 8 * SMs, so the work item is 32 rows for any occupancy. The budget block is
    repeated every 4096 rows. Checked against the oracle on a sample of whole 32-row groups."""
    M, N = LARGE_M, 40_000
    specials = {4096 * 7 + 5: 4100, 4096 * 9 + 3: 513, 4096 * 11 + 31: 257, 4096 * 13: 256, 4096 * 20 + 1: 33}
    blocks = list(range(2048, M - 32, 4096))
    rowptr, col = build_csr(M, N, 1, 2, specials, blocks, tie_rows={4096 * 30 + 2: 700}, empty_rows=(0, M // 2, M - 1))
    g = torch.Generator().manual_seed(3)
    groups = set(blocks[:16]) | {r & ~31 for r in specials} | {4096 * 30, 0, (M // 2) & ~31, (M - 1) & ~31}
    groups |= set((torch.randint((M - 1) // 32, (32,), generator=g) * 32).tolist())
    rows = torch.cat([torch.arange(r, min(r + 32, M)) for r in sorted(groups)])
    return dict(M=M, N=N, rowptr=rowptr, col=col, rows=rows)


def sub_csr(rowptr, col, rows):
    """The rows `rows` of a CSR matrix as their own CSR; `idx` maps its nnz to the full matrix's."""
    s, e = rowptr[rows], rowptr[rows + 1]
    lens = e - s
    sp = torch.zeros(rows.numel() + 1, dtype=torch.long)
    sp[1:] = lens.cumsum(0)
    idx = torch.repeat_interleave(s - sp[:-1], lens) + torch.arange(int(sp[-1]))
    return sp, col[idx], idx


def plan_budget_rows(rowptr, group=32):
    """Rows deferred for the 1024-nnz budget of their `group`-row work item (not for their length): the plan's rule
    with the default 32, an unplanned call's with the size of its items."""
    deg = rowptr[1:] - rowptr[:-1]
    M = deg.numel()
    d = torch.cat([deg, deg.new_zeros((-M) % group)]).view(-1, group)
    cum = torch.where(d > 256, 0, d).cumsum(1)
    return ((d > 0) & (d <= 256) & (cum > 1024)).view(-1)[:M]


# ---- operands --------------------------------------------------------------------------------------------------------
def dense(N, K, dtype, seed, quantized, B=None):
    """randn (sums) or multiples of 1/2 in [-2, 2] with signed zeros (min/max: many exact ties); unreferenced rows NaN."""
    g = torch.Generator().manual_seed(seed)
    shape = (N, K) if B is None else (B, N, K)
    if quantized:
        x = torch.randint(-4, 5, shape, generator=g).double() * 0.5
        x = torch.where(torch.rand(shape, generator=g) < 0.05, torch.tensor(-0.0, dtype=torch.float64), x)
    else:
        x = torch.randn(shape, generator=g, dtype=torch.float64)
    x[..., unreferenced_rows(N), :] = float("nan")
    return x.to(dtype)


def values(E, dtype, seed, quantized):
    g = torch.Generator().manual_seed(seed)
    if quantized:
        return torch.tensor([-1.0, -0.5, 0.5, 1.0, 2.0, 0.0, -0.0], dtype=torch.float64)[
            torch.randint(7, (E,), generator=g)].to(dtype)
    return torch.randn(E, generator=g, dtype=torch.float64).to(dtype)


# ---- direct library calls, outputs prefilled ------------------------------------------------------------------------
def _vp(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _prefilled(sizes, dtype, arg):
    fill = float("nan") if dtype.is_floating_point else -7777
    out = torch.full(sizes, fill, dtype=dtype, device=DEV)
    return out, (torch.full(sizes, -1, dtype=torch.int64, device=DEV) if arg else None)


def call_fw(rowptr, col, value, mat, reduce):
    """tsb200_spmm_fw into NaN / -1 prefilled outputs."""
    M, E = rowptr.numel() - 1, col.numel()
    N, K = mat.shape[-2:]
    B = mat.numel() // (N * K)
    sizes = list(mat.shape[:-2]) + [M, K]
    red, dt = ops._REDUCE[reduce], ops._dtype_code(mat.dtype)
    out, arg = _prefilled(sizes, mat.dtype, red >= 2)
    nws = lib.tsb200_spmm_fw_workspace_bytes(B, M, K, E, dt, red)
    ws = torch.empty(max(nws, 1), dtype=torch.uint8, device=DEV)
    rc = lib.tsb200_spmm_fw(_vp(rowptr), _vp(col), _vp(value), _vp(mat), _vp(out), _vp(arg), B, M, N, K, E, dt, red,
                            _vp(ws), nws, _stream())
    assert rc == 0, rc
    return out, arg


def call_planned(plan, rowptr, col, value, mat, reduce, expect_rc=0):
    """tsb200_spmm_fw_planned into NaN / -1 prefilled outputs (B = 1)."""
    M, E = rowptr.numel() - 1, col.numel()
    N, K = mat.shape[-2:]
    red, dt = ops._REDUCE[reduce], ops._dtype_code(mat.dtype)
    out, arg = _prefilled([M, K], mat.dtype, red >= 2)
    nws = lib.tsb200_spmm_fw_planned_workspace_bytes(K, plan.n_long, plan.n_slot, red)
    ws = torch.empty(max(nws, 1), dtype=torch.uint8, device=DEV)
    rc = lib.tsb200_spmm_fw_planned(_vp(rowptr), _vp(col), _vp(value), _vp(mat), _vp(out), _vp(arg), M, N, K, E, dt,
                                    red, _vp(plan.data), plan.data.numel(), plan.n_seg, plan.n_long, plan.n_slot,
                                    _vp(ws), nws, _stream())
    assert rc == expect_rc, rc
    return out, arg


def call_acc_blocks(rowptr, col, value, mat, P):
    """A sum assembled from P column blocks of A through tsb200_spmm_fw_acc (modes 1, 2, 3); partial and out
    prefilled with NaN."""
    M, N, K = rowptr.numel() - 1, mat.size(-2), mat.size(-1)
    dt = ops._dtype_code(mat.dtype)
    row = torch.repeat_interleave(torch.arange(M, device=DEV), rowptr[1:] - rowptr[:-1])
    partial = torch.full((M, K), float("nan"), dtype=torch.float32, device=DEV)
    out = torch.full((M, K), float("nan"), dtype=mat.dtype, device=DEV)
    bounds = [N * c // P for c in range(P + 1)]
    for c in range(P):
        keep = (col >= bounds[c]) & (col < bounds[c + 1])
        rp = torch.zeros(M + 1, dtype=torch.long, device=DEV)
        rp[1:] = torch.bincount(row[keep], minlength=M).cumsum(0)
        cl = col[keep].contiguous()
        v = None if value is None else value[keep].contiguous()
        E = cl.numel()
        nws = lib.tsb200_spmm_fw_workspace_bytes(1, M, K, E, dt, 0)
        ws = torch.empty(max(nws, 1), dtype=torch.uint8, device=DEV)
        mode = 1 if c == 0 else (3 if c == P - 1 else 2)
        rc = lib.tsb200_spmm_fw_acc(_vp(rp), _vp(cl), _vp(v), _vp(mat), _vp(out), _vp(partial), mode, 1, M, N, K, E,
                                    dt, _vp(ws), nws, _stream())
        assert rc == 0, rc
    return out


# ---- bounds ----------------------------------------------------------------------------------------------------------
PREC = {torch.float32: (24, -126), torch.bfloat16: (8, -126), torch.float16: (11, -14), torch.float64: (53, -1022)}


def half_ulp(x, dtype):
    """1/2 ulp of |x| (float64) in `dtype`, subnormals included."""
    p, emin = PREC[dtype]
    _, e = torch.frexp(x)
    e = torch.where(x == 0, torch.full_like(e, emin), (e - 1).clamp(min=emin))
    return torch.ldexp(torch.full_like(x, 0.5), (e - (p - 1)).double())


def assert_sum_bound(out, ref, S, n, dtype, cnt=None, u=U32, what=""):
    """|out - ref| <= 1/2 ulp_T + n * u * S; for a mean `ref` is the mean, S and n those of the sum, cnt the row
    degree (>= 1): the sum's error / cnt plus one rounding of the division."""
    out = out.cpu().double()
    e = n * u * S
    if cnt is not None:
        e = e / cnt
        e = e + u * (ref.abs() + e)
    bound = e + half_ulp(ref.abs() + e, dtype)
    ok = (out - ref).abs() <= bound
    if not bool(ok.all()):
        i = tuple(int(j) for j in (~ok).nonzero()[0])
        raise AssertionError(f"{what}: {int((~ok).sum())} elements out of bound, first at {i}: "
                             f"out {out[i].item()!r} ref {ref[i].item()!r} bound {bound[i].item():.3e}")


def bits(t):
    t = t.cpu().contiguous()
    return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def assert_bits_equal(out, ref, what=""):
    a, b = bits(out), bits(ref)
    ok = a == b
    if not bool(ok.all()):
        i = tuple(int(j) for j in (~ok).nonzero()[0])
        raise AssertionError(f"{what}: {int((~ok).sum())} elements differ, first at {i}: "
                             f"{out.cpu()[i].item()!r} vs {ref.cpu()[i].item()!r}")


class Ref:
    """Oracle results of one (matrix, value, mat): fp64 sum and |A||B| on the upcast inputs, min/max in the storage
    dtype; each computed once and shared by every call checked against it."""

    def __init__(self, oracle, rowptr, col, value, mat):
        self.o, self.rowptr, self.col, self.value, self.mat = oracle, rowptr, col, value, mat
        self._c = {}
        deg = (rowptr[1:] - rowptr[:-1]).double()
        self.deg = deg.view(-1, 1)
        self.cnt = deg.clamp(min=1).view(-1, 1)

    def _get(self, key, fn):
        if key not in self._c:
            self._c[key] = fn()
        return self._c[key]

    def sum64(self):
        v = None if self.value is None else self.value.double()
        return self._get("sum", lambda: self.o.spmm(self.rowptr, self.col, v, self.mat.double(), "sum")[0])

    def S(self):
        v = None if self.value is None else self.value.double().abs()
        mat = torch.nan_to_num(self.mat.double(), nan=0.0).abs()
        return self._get("S", lambda: self.o.spmm(self.rowptr, self.col, v, mat, "sum")[0])

    def minmax(self, reduce):
        return self._get(reduce, lambda: self.o.spmm(self.rowptr, self.col, self.value, self.mat, reduce))

    def check(self, reduce, out, arg, what, extra_terms=1):
        if reduce in ("min", "max"):
            ref, rarg = self.minmax(reduce)
            assert_bits_equal(out, ref, f"{what} {reduce} out")
            assert torch.equal(arg.cpu(), rarg), f"{what} {reduce}: arg_out differs"
        elif reduce == "sum":
            assert_sum_bound(out, self.sum64(), self.S(), self.deg + extra_terms, self.mat.dtype, what=f"{what} sum")
        else:
            assert_sum_bound(out, self.sum64() / self.cnt, self.S(), self.deg + extra_terms, self.mat.dtype,
                             cnt=self.cnt, what=f"{what} mean")


def _dev(*ts):
    return [None if t is None else t.to(DEV) for t in ts]


# ---- 1. the dispatch table against the library ----------------------------------------------------------------------
@pytest.mark.parametrize("dtype,K", [(dt, ks[0]) for fam, (k32, k16) in FAMILIES.items() for dt in FLOATS
                                     for ks in [k32 if dt == torch.float32 else k16]], ids=_id)
def test_dispatch_table_matches_library(small, dtype, K):
    """The kernel each table row names is the kernel the library launches (unplanned and planned), with the table's
    (LPR, CH, U, CTAs/SM) and one launch per column tile."""
    rowptr, col = _dev(small["rowptr"], small["col"])
    mat = dense(small["N"], K, dtype, 0, False).to(DEV)
    fam = family_of(dtype, K)
    plan = ops.spmm_plan(rowptr, col.numel())
    for planned in (False, True):
        names = launched_kernels(lambda: call_planned(plan, rowptr, col, None, mat, "sum") if planned
                          else call_fw(rowptr, col, None, mat, "sum"), r"spmm_(gpr|vec)_kernel<")
        if fam.startswith("gpr"):
            got = [int(m.group(1)) for n in names for m in [re.search(r"spmm_gpr_kernel<[^,]+, \d+, (\d+), (\d+), (\d+)", n)]
                   if m and m.group(2) == "4" and m.group(3) == "5"]
            assert got and set(got) == {KERNEL[fam][0]}, (fam, names)
            assert not any("spmm_vec_kernel" in n for n in names), names
        else:
            got = [tuple(int(x) for x in m.groups()) for n in names
                   for m in [re.search(r"spmm_vec_kernel<[^,]+, \d+, (\d+), (\d+), (\d+), (\d+)", n)] if m]
            assert set(got) == {KERNEL[fam]}, (fam, names)
            assert len(got) == n_tiles(dtype, K), (fam, names)
            assert not any("spmm_gpr_kernel" in n for n in names), names


def test_generic_cases_match_table_and_oracle(oracle, small):
    """Where the table says "generic" (K*size not a multiple of 16 B, fp64, integers, a 2-byte-misaligned bf16 value)
    the planned entry point refuses with TSB200_ERR_UNSUPPORTED and the unplanned call runs the generic kernel:
    bit-exact with the oracle for fp32 / fp64 / integers (same sequential walk, separate multiply and add), within the
    sum bound for bf16 / f16; everywhere else in the table the planned entry point accepts the call."""
    rowptr_c, col_c = small["rowptr"], small["col"]
    rowptr, col = _dev(rowptr_c, col_c)
    E, N = col.numel(), small["N"]
    plan = ops.spmm_plan(rowptr, E)
    cases = [(torch.float32, 6, True), (torch.float64, 8, True), (torch.int64, 4, True), (torch.int32, 3, True),
             (torch.float16, 5, True), (torch.bfloat16, 8, False)]
    for dtype, K, aligned in cases:
        assert family_of(dtype, K, aligned) == "generic"
        if dtype.is_floating_point:
            mat_c = dense(N, K, dtype, 5, False)
            val_c = values(E, dtype, 6, False)
        else:
            g = torch.Generator().manual_seed(5)
            mat_c = torch.randint(-50, 50, (N, K), generator=g).to(dtype)
            val_c = torch.randint(-5, 5, (E,), generator=g).to(dtype)
        mat = mat_c.to(DEV)
        if aligned:
            val = val_c.to(DEV)
        else:
            buf = torch.empty(E + 1, dtype=dtype, device=DEV)
            buf[1:] = val_c.to(DEV)
            val = buf[1:]
            assert val.data_ptr() % 4 == 2
        ref = Ref(oracle, rowptr_c, col_c, val_c, mat_c)
        for reduce in REDUCES:
            call_planned(plan, rowptr, col, val, mat, reduce, expect_rc=ERR_UNSUPPORTED)
            out, arg = call_fw(rowptr, col, val, mat, reduce)
            what = f"generic {dtype} K={K}"
            if dtype in F16S or reduce in ("min", "max"):
                ref.check(reduce, out, arg, what)
            else:
                exact, _ = oracle.spmm(rowptr_c, col_c, val_c, mat_c, reduce)
                assert_bits_equal(out, exact, f"{what} {reduce}")
    # the vector path accepts every other table row
    for dtype, K in TABLE:
        mat = torch.zeros(N, K, dtype=dtype, device=DEV)
        call_planned(plan, rowptr, col, None, mat, "sum")


# ---- 2-4. every family x dtype x reduction x value x {plain, planned, ACC} on the structured matrix -----------------
@pytest.mark.parametrize("has_value", [True, False], ids=["value", "novalue"])
@pytest.mark.parametrize("dtype,K", TABLE, ids=_id)
def test_family_vs_oracle(oracle, small, dtype, K, has_value):
    rowptr_c, col_c = small["rowptr"], small["col"]
    E, N = col_c.numel(), small["N"]
    fam = family_of(dtype, K)
    rowptr, col = _dev(rowptr_c, col_c)
    plan = ops.spmm_plan(rowptr, E)
    assert plan.n_long > 0 and plan.n_seg > plan.n_long
    budget = plan_budget_rows(rowptr_c)
    assert budget.any()
    for quantized, reduces in ((False, ("sum", "mean")), (True, ("min", "max"))):
        mat_c = dense(N, K, dtype, K, quantized)
        val_c = values(E, dtype, K + 1, quantized) if has_value else None
        mat, val = _dev(mat_c, val_c)
        ref = Ref(oracle, rowptr_c, col_c, val_c, mat_c)
        for reduce in reduces:
            what = f"{fam} {dtype} K={K} value={has_value}"
            out_u, arg_u = call_fw(rowptr, col, val, mat, reduce)
            ref.check(reduce, out_u, arg_u, what + " unplanned")
            out_p, arg_p = call_planned(plan, rowptr, col, val, mat, reduce)
            ref.check(reduce, out_p, arg_p, what + " planned")
            if reduce in ("min", "max"):
                assert_bits_equal(out_p, out_u, what + " planned vs unplanned")
                assert torch.equal(arg_p, arg_u)
            elif fam.startswith("gpr"):
                # the group-per-row kernel walks a row with one lane group; a row the plan defers for the item budget
                # is summed by the segment kernel's lane groups instead (the unplanned call, with items shrunk to
                # fewer rows for this small matrix, keeps it): only the order of those rows' sums differs
                keep = ~budget.to(DEV)
                assert_bits_equal(out_p[keep], out_u[keep], what + " planned vs unplanned")
            else:
                assert_bits_equal(out_p, out_u, what + " planned vs unplanned")
        if has_value and not quantized:
            out_a = call_acc_blocks(rowptr, col, val, mat, 3)
            assert_sum_bound(out_a, ref.sum64(), ref.S(), ref.deg + 3, dtype, what=f"{what} acc P=3")


@pytest.mark.parametrize("fam", [f for f in FAMILIES if f != "tiled"])
def test_family_batched(oracle, small, fam):
    """B = 3 with a different dense operand per batch (unplanned; the planned path is B = 1 only)."""
    rowptr_c, col_c = small["rowptr"], small["col"]
    E, N = col_c.numel(), small["N"]
    rowptr, col = _dev(rowptr_c, col_c)
    for dtype in FLOATS:
        K = FAMILIES[fam][0 if dtype == torch.float32 else 1][-1]
        for quantized, reduces in ((False, ("sum", "mean")), (True, ("min", "max"))):
            mat_c = dense(N, K, dtype, 40 + K, quantized, B=3)
            val_c = values(E, dtype, 41, quantized)
            mat, val = _dev(mat_c, val_c)
            ref = Ref(oracle, rowptr_c, col_c, val_c, mat_c)
            for reduce in reduces:
                out, arg = call_fw(rowptr, col, val, mat, reduce)
                ref.check(reduce, out, arg, f"{fam} {dtype} K={K} B=3")


# one full-width K per family, dtypes rotating so that each of fp32, bf16 and f16 appears
LARGE_TABLE = [("gpr1", torch.float32), ("gpr2", torch.bfloat16), ("gpr4", torch.float16), ("gpr8", torch.float32),
               ("vec16", torch.bfloat16), ("vec32ch1", torch.float16), ("vec32ch2", torch.float32),
               ("vec32ch4", torch.bfloat16)]


@pytest.mark.parametrize("fam,dtype", LARGE_TABLE, ids=_id)
def test_family_full_size_items(oracle, large, fam, dtype):
    """32-row work items: budget deferral of whole rows, the item's ring aligned across many rows; planned and
    unplanned results bit-identical (the same rows are deferred); every output written; a sample of whole 32-row
    groups against the oracle."""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    assert large["M"] >= 32 * 16 * 8 * sms
    K = FAMILIES[fam][0 if dtype == torch.float32 else 1][0]
    rowptr_c, col_c, rows, N = large["rowptr"], large["col"], large["rows"], large["N"]
    E = col_c.numel()
    rowptr, col = _dev(rowptr_c, col_c)
    plan = ops.spmm_plan(rowptr, E)
    sp, scol, idx = sub_csr(rowptr_c, col_c, rows)
    rows_d = rows.to(DEV)
    for quantized, reduces in ((False, ("sum", "mean")), (True, ("min", "max"))):
        mat_c = dense(N, K, dtype, 7, quantized)
        val_c = values(E, dtype, 8, quantized)
        mat, val = _dev(mat_c, val_c)
        ref = Ref(oracle, sp, scol, val_c[idx], mat_c)
        for reduce in reduces:
            what = f"{fam} {dtype} K={K} M={large['M']}"
            out_u, arg_u = call_fw(rowptr, col, val, mat, reduce)
            out_p, arg_p = call_planned(plan, rowptr, col, val, mat, reduce)
            assert_bits_equal(out_p, out_u, what + f" {reduce} planned vs unplanned")
            if arg_u is not None:
                assert torch.equal(arg_p, arg_u)
                assert bool((arg_u >= 0).all()), "arg_out element not written"
            else:
                assert not bool(out_u.isnan().any()), "output element not written (or a NaN row leaked)"
            arg_s = None
            if arg_u is not None:  # back to the sample's own nnz numbering
                a = arg_u[rows_d].cpu()
                glob = torch.cat([idx, torch.tensor([E])])
                arg_s = torch.searchsorted(glob, a)
                arg_s = torch.where(glob[arg_s.clamp(max=idx.numel())] == a, arg_s, -1)
                arg_s = torch.where(a == E, idx.numel(), arg_s)
            ref.check(reduce, out_u[rows_d], arg_s, what)


# ---- 5. non-finite and signed-zero data ------------------------------------------------------------------------------
def nonfinite_case(dtype, K, seed):
    """A matrix and operands with NaN, +-inf, -0.0 and +0.0: row 1 has only NaN products (NaN values), row 2 only -inf
    products, row 3 (700 nnz, three segments) a finite winner in its second segment only, row 4 only +-0 products;
    every other row mixes everything."""
    g = torch.Generator().manual_seed(seed)
    M, N = 300, 500
    deg = torch.poisson(torch.full((M,), 6.0), generator=g).long()
    deg[[1, 2, 3, 4, 0, M - 1]] = torch.tensor([9, 9, 700, 40, 0, 0])
    rowptr = torch.zeros(M + 1, dtype=torch.long)
    rowptr[1:] = deg.cumsum(0)
    E = int(rowptr[-1])
    col = torch.randint(1, N - NAN_ROWS + 1, (E,), generator=g)
    x = torch.randn(N, K, generator=g, dtype=torch.float64)
    special = torch.tensor([float("nan"), float("inf"), -float("inf"), 0.0, -0.0], dtype=torch.float64)
    pick = torch.rand(N, K, generator=g) < 0.1
    x = torch.where(pick, special[torch.randint(5, (N, K), generator=g)], x)
    x[unreferenced_rows(N)] = float("nan")
    x[N - NAN_ROWS] = -float("inf")      # an all -inf row...
    x[N - NAN_ROWS - 1] = 0.0             # ...an all +0 row and an all -0 row, referenced only by rows 2 and 4
    x[N - NAN_ROWS - 2] = -0.0
    v = torch.randn(E, generator=g, dtype=torch.float64)
    v = torch.where(torch.rand(E, generator=g) < 0.1, special[torch.randint(5, (E,), generator=g)], v)
    s = lambda r: slice(int(rowptr[r]), int(rowptr[r + 1]))  # noqa: E731
    v[s(1)] = float("nan")
    col[s(2)] = N - NAN_ROWS
    v[s(2)] = torch.rand(9, generator=g, dtype=torch.float64) + 0.5
    v[s(3)] = float("nan")
    v[int(rowptr[3]) + 300: int(rowptr[3]) + 310] = 1.0
    col[int(rowptr[3]) + 300: int(rowptr[3]) + 310] = torch.randint(1, N - NAN_ROWS - 2, (10,), generator=g)
    x[col[int(rowptr[3]) + 300: int(rowptr[3]) + 310]] = 1.0
    col[s(4)] = torch.tensor([N - NAN_ROWS - 1, N - NAN_ROWS - 2])[torch.randint(2, (40,), generator=g)]
    v[s(4)] = torch.tensor([1.0, -1.0, 0.0, -0.0], dtype=torch.float64)[torch.randint(4, (40,), generator=g)]
    return rowptr, col, v.to(dtype), x.to(dtype)


@pytest.mark.parametrize("dtype,K", [(dt, ks[0]) for fam, (k32, k16) in FAMILIES.items() for dt in FLOATS
                                     for ks in [k32 if dt == torch.float32 else k16]], ids=_id)
def test_nonfinite_and_signed_zero(oracle, dtype, K):
    """min/max: values and arg_out bit-exact with the oracle, which defines a non-empty row without a winner (all NaN
    products; all -inf products under max) like an empty row: (lowest() / max(), arg = E). sum/mean: the NaN and +-inf
    pattern of the fp64 oracle, and no NaN from an unreferenced dense row in any finite output."""
    rowptr_c, col_c, val_c, mat_c = nonfinite_case(dtype, K, K)
    rowptr, col, val, mat = _dev(rowptr_c, col_c, val_c, mat_c)
    E = col.numel()
    plan = ops.spmm_plan(rowptr, E)
    for value_c, value in ((val_c, val), (None, None)):
        for reduce in REDUCES:
            outs = [call_fw(rowptr, col, value, mat, reduce), call_planned(plan, rowptr, col, value, mat, reduce)]
            what = f"{dtype} K={K} value={value is not None} {reduce}"
            if reduce in ("min", "max"):
                ref, rarg = oracle.spmm(rowptr_c, col_c, value_c, mat_c, reduce)
                for out, arg in outs:
                    assert_bits_equal(out, ref, what)
                    assert torch.equal(arg.cpu(), rarg), what + ": arg_out differs"
                if value is not None:
                    lim = torch.finfo(dtype).max if reduce == "min" else torch.finfo(dtype).min
                    assert bool((ref[1] == lim).all()) and bool((rarg[1] == E).all())
                    if reduce == "max":
                        assert bool((ref[2] == lim).all()) and bool((rarg[2] == E).all())
                    a3 = rarg[3]
                    assert bool(((a3 >= rowptr_c[3] + 256) & (a3 < rowptr_c[3] + 512)).all())
            else:
                v64 = None if value_c is None else value_c.double()
                ref, _ = oracle.spmm(rowptr_c, col_c, v64, mat_c.double(), reduce)
                for out, _ in outs:
                    o = out.cpu().double()
                    assert torch.equal(o.isnan(), ref.isnan()), what + ": NaN pattern"
                    assert torch.equal(o.isposinf(), ref.isposinf()) and torch.equal(o.isneginf(), ref.isneginf()), \
                        what + ": inf pattern"
