"""SDDMM as a public operator: `sddmm` (every float dtype, through tsb200_spmm_value_bw, differentiable) and `sddmm_fp8`
(two e4m3 operands with per-row or per-tensor scales, tsb200_sddmm_fp8).

Kernels are called through the C-ABI into NaN-prefilled outputs, so an entry a kernel fails to write cannot pass; the
public calls are then compared with those results bit for bit. The structured matrix `small` (test_spmm_kernels_gpu)
has empty rows, rows of 1 ... 4100 nnz (segments past 256) and a 32-row block over the 1024-nnz item budget, and
every row-wise kernel runs at every work-item size (TSB200_SPMM_ITEM_SHIFT = 0 ... 5). A dot product is summed by one
lane group in a fixed lane order whatever the item size or kernel (row or segment), so results must not change with
the item size.

Float path: |out - ref64| <= 1/2 ulp_T + (K + 1) u sum_k |a b| against a CPU fp64 reference (u = 2^-24, 2^-52 for
fp64), bit for bit where every partial sum is exact. Gradients are SpMMs (each element a sum of n terms):
(n + 1) 2^-24 sum|terms| + 1/2 ulp_T.
FP8 path: d_e = sum_k qa qb (each product exact in fp32), s_e = fl32(sa[r] sb[c]), out = round_out(fl32(s_e d_e)).
The CPU replay forms d_e exactly in fp64: bit for bit where d_e is exact in fp32, otherwise
|out - s_e d_e| <= 1/2 ulp_out + (K + 2) 2^-24 s_e sum_k |qa qb|.
"""
import ctypes
import json
import subprocess
import sys
from pathlib import Path

import pytest
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import SparseTensor, ops
from pytorch_sparse_b200._lib import lib
from test_spmm_backward_kernels_gpu import call_value_bw, sddmm_family
from test_spmm_kernels_gpu import (DEV, _dev, _id, assert_bits_equal, assert_sum_bound, build_csr, half_ulp,  # noqa: F401
                                   small)

pytestmark = pytest.mark.gpu
ENV = "TSB200_SPMM_ITEM_SHIFT"
SHIFTS = range(6)
U32 = 2.0 ** -24
E4M3 = torch.float8_e4m3fn
OUTS = (torch.bfloat16, torch.float16, torch.float32)


def coo_row(rowptr):
    return torch.repeat_interleave(torch.arange(rowptr.numel() - 1), rowptr[1:] - rowptr[:-1])


def src_of(m, device=DEV):
    """The structured matrix as a SparseTensor (CSR order kept: its columns are unsorted within a row)."""
    rowptr, col = m["rowptr"], m["col"]
    return SparseTensor(row=coo_row(rowptr).to(device), rowptr=rowptr.to(device), col=col.to(device),
                        sparse_sizes=(m["M"], m["N"]), is_sorted=True, trust_data=True)


def dots64(x, y, row, col, chunk=4096):
    """sum_k x[row_e, k] * y[col_e, k] in fp64 on the CPU, in chunks of entries."""
    x, y = x.cpu().double(), y.cpu().double()
    out = torch.empty(row.numel(), dtype=torch.float64)
    for i in range(0, row.numel(), chunk):
        out[i:i + chunk] = (x[row[i:i + chunk]] * y[col[i:i + chunk]]).sum(-1)
    return out


# ---- float path: every path of tsb200_spmm_value_bw -----------------------------------------------------------------
# (dtype, K): every row-wise family at full and partial width, the nnz-parallel kernel below 3 and above 64 vectors,
# and the generic kernel (fp64, rows that are not a multiple of 16 bytes)
FLOAT_CASES = [(torch.float32, 12), (torch.float16, 24), (torch.bfloat16, 32), (torch.float32, 32),
               (torch.bfloat16, 64), (torch.float32, 64), (torch.float16, 128), (torch.float32, 100),
               (torch.bfloat16, 256), (torch.float32, 256), (torch.float16, 392), (torch.bfloat16, 512),
               (torch.float32, 8), (torch.bfloat16, 8), (torch.float32, 300), (torch.bfloat16, 600),
               (torch.float64, 16), (torch.float64, 5), (torch.float32, 6), (torch.bfloat16, 7)]
FAMILIES = {sddmm_family(dt, K, 1) for dt, K in FLOAT_CASES}
assert FAMILIES == {"row4", "row8", "row16", "row32", "row32ch2", "nnz1", "nnz4", "nnz32strided", "generic"}, FAMILIES


def float_operands(M, N, K, dtype, seed, exact):
    """randn, or multiples of 1/2 in [-2, 2] (every fp32 partial sum exact)."""
    g = torch.Generator().manual_seed(seed)
    if exact:
        a = torch.randint(-4, 5, (M, K), generator=g).double() / 2
        b = torch.randint(-4, 5, (N, K), generator=g).double() / 2
    else:
        a = torch.randn(M, K, generator=g, dtype=torch.float64)
        b = torch.randn(N, K, generator=g, dtype=torch.float64)
    return a.to(dtype), b.to(dtype)


def float_bound_check(out, a, b, row, col, what):
    dtype = a.dtype
    ref = dots64(a, b, row, col)
    S = dots64(a.abs(), b.abs(), row, col)
    K = a.size(1)
    u = 2.0 ** -52 if dtype == torch.float64 else U32
    assert_sum_bound(out, ref, S, K + 1, dtype, u=u, what=what)


@pytest.mark.parametrize("exact", [False, True], ids=["random", "exact"])
@pytest.mark.parametrize("dtype,K", FLOAT_CASES, ids=_id)
def test_float_paths_every_item_size(small, monkeypatch, dtype, K, exact):
    rowptr_c, col_c, M, N = small["rowptr"], small["col"], small["M"], small["N"]
    row_c = coo_row(rowptr_c)
    a_c, b_c = float_operands(M, N, K, dtype, K, exact)
    row, rowptr, col, a, b = _dev(row_c, rowptr_c, col_c, a_c, b_c)
    src = src_of(small)
    ref_exact = dots64(a_c, b_c, row_c, col_c).to(dtype) if exact else None
    first = None
    for s in SHIFTS:
        monkeypatch.setenv(ENV, str(s))
        what = f"sddmm {sddmm_family(dtype, K, 1)} {dtype} K={K} shift={s}"
        out = call_value_bw(row, rowptr, col, b, a, "sum")        # grad := a, mat := b
        if exact:
            assert_bits_equal(out, ref_exact, what + " exact")
        else:
            float_bound_check(out, a_c, b_c, row_c, col_c, what)
        if first is None:
            first = out
        assert_bits_equal(out, first, what + " vs shift 0")
        assert_bits_equal(ts.sddmm(src, a, b), out, what + " public")
        assert_bits_equal(src.sddmm(a, b), out, what + " method")


def test_float_unaligned_rows_take_the_generic_kernel(small):
    """A 16-byte multiple row starting 4 bytes past an aligned address: the generic kernel, same bound."""
    rowptr_c, col_c, M, N = small["rowptr"], small["col"], small["M"], small["N"]
    row_c = coo_row(rowptr_c)
    a_c, b_c = float_operands(M, N, 64, torch.float32, 5, False)
    buf = torch.empty(M * 64 + 1, dtype=torch.float32, device=DEV)
    a = buf[1:].view(M, 64)
    a.copy_(a_c)
    assert a.data_ptr() % 16 == 4 and a.is_contiguous()
    b = b_c.to(DEV)
    src = src_of(small)
    out = call_value_bw(*_dev(row_c, rowptr_c, col_c), b, a, "sum")
    float_bound_check(out, a_c, b_c, row_c, col_c, "sddmm unaligned")
    assert_bits_equal(ts.sddmm(src, a, b), out, "sddmm unaligned public")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float64])
def test_float_empty(dtype):
    for M, N in ((5, 7), (0, 7)):          # E = 0 with rows, and M = 0
        src = SparseTensor(row=torch.empty(0, dtype=torch.long, device=DEV), col=torch.empty(0, dtype=torch.long,
                           device=DEV), sparse_sizes=(M, N))
        a = torch.randn(M, 32, device=DEV, dtype=dtype, requires_grad=True)
        b = torch.randn(N, 32, device=DEV, dtype=dtype, requires_grad=True)
        out = ts.sddmm(src, a, b)
        assert out.shape == (0,) and out.dtype == dtype
        out.sum().backward()
        assert torch.equal(a.grad, torch.zeros_like(a)) and torch.equal(b.grad, torch.zeros_like(b))
    src = SparseTensor(row=torch.tensor([0, 2], device=DEV), col=torch.tensor([1, 1], device=DEV), sparse_sizes=(3, 2))
    out = ts.sddmm(src, torch.empty(3, 0, device=DEV, dtype=dtype), torch.empty(2, 0, device=DEV, dtype=dtype))
    assert torch.equal(out, torch.zeros(2, device=DEV, dtype=dtype)) and not bool(out.signbit().any())


# ---- autograd -----------------------------------------------------------------------------------------------------------
def grad_bound_check(got, ref, S, n, dtype, what):
    assert_sum_bound(got, ref, S, n + 1, dtype, what=what)


@pytest.mark.parametrize("dtype,K", [(torch.float32, 32), (torch.bfloat16, 128), (torch.float16, 512),
                                     (torch.float32, 6)], ids=_id)
@pytest.mark.parametrize("need", ["both", "a", "b"])
def test_autograd_against_fp64_torch(small, dtype, K, need):
    rowptr_c, col_c, M, N = small["rowptr"], small["col"], small["M"], small["N"]
    row_c = coo_row(rowptr_c)
    a_c, b_c = float_operands(M, N, K, dtype, 7, False)
    w_c = torch.randn(row_c.numel(), generator=torch.Generator().manual_seed(8), dtype=torch.float64).to(dtype)
    a = a_c.to(DEV).requires_grad_(need in ("both", "a"))
    b = b_c.to(DEV).requires_grad_(need in ("both", "b"))
    src = src_of(small)
    out = ts.sddmm(src, a, b)
    assert out.requires_grad
    (out * w_c.to(DEV)).sum().backward()
    # fp64 torch autograd of the expression on the same operands
    a64 = a_c.double().requires_grad_()
    b64 = b_c.double().requires_grad_()
    ((a64[row_c] * b64[col_c]).sum(-1) * w_c.double()).sum().backward()
    w = w_c.double().abs().view(-1, 1)
    if need in ("both", "a"):
        S = torch.zeros(M, K, dtype=torch.float64).index_add_(0, row_c, w * b_c.double().abs()[col_c])
        n = torch.bincount(row_c, minlength=M).double().view(-1, 1)
        grad_bound_check(a.grad, a64.grad, S, n, dtype, f"grad_a {dtype} K={K} {need}")
    else:
        assert a.grad is None
    if need in ("both", "b"):
        S = torch.zeros(N, K, dtype=torch.float64).index_add_(0, col_c, w * a_c.double().abs()[row_c])
        n = torch.bincount(col_c, minlength=N).double().view(-1, 1)
        grad_bound_check(b.grad, b64.grad, S, n, dtype, f"grad_b {dtype} K={K} {need}")
    else:
        assert b.grad is None


def test_gradcheck_fp64():
    g = torch.Generator().manual_seed(3)
    M, N, K = 13, 9, 5
    row = torch.randint(M, (40,), generator=g)
    col = torch.randint(N, (40,), generator=g)
    src = SparseTensor(row=row.to(DEV), col=col.to(DEV), sparse_sizes=(M, N))   # duplicates kept
    a = torch.randn(M, K, generator=g, dtype=torch.float64).to(DEV).requires_grad_()
    b = torch.randn(N, K, generator=g, dtype=torch.float64).to(DEV).requires_grad_()
    assert torch.autograd.gradcheck(lambda x, y: ts.sddmm(src, x, y), (a, b))
    assert torch.autograd.gradcheck(lambda x: ts.sddmm(src, x, b.detach()), (a,))
    assert torch.autograd.gradcheck(lambda y: ts.sddmm(src, a.detach(), y), (b,))


def test_gradient_to_b_needs_the_csc_view(small):
    rowptr, col = _dev(small["rowptr"], small["col"])
    row = coo_row(small["rowptr"]).to(DEV)
    a = torch.randn(small["M"], 16, device=DEV)
    b = torch.randn(small["N"], 16, device=DEV, requires_grad=True)
    with pytest.raises(RuntimeError, match="Argument `colptr` is missing"):
        torch.ops.tsb200.sddmm(row, rowptr, col, None, None, None, a, b)


# ---- memory: no E x K temporary ------------------------------------------------------------------------------------------
def peak_above(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


def test_peak_memory():
    M = N = 200_000
    E0 = 16 * M
    g = torch.Generator(device=DEV).manual_seed(0)
    key = torch.unique(torch.randint(M, (E0,), generator=g, device=DEV) * N +
                       torch.randint(N, (E0,), generator=g, device=DEV))
    src = SparseTensor(row=key // N, col=key % N, sparse_sizes=(M, N), is_sorted=True, trust_data=True)
    src.storage.rowptr()
    E, K = src.nnz(), 128
    nws = lib.tsb200_sddmm_fp8_workspace_bytes(M, K, E)
    assert nws == lib.tsb200_spmm_value_bw_workspace_bytes(1, M, K, E, 3)
    a = torch.randn(M, K, device=DEV, dtype=torch.bfloat16)
    b = torch.randn(N, K, device=DEV, dtype=torch.bfloat16)
    out, peak = peak_above(lambda: ts.sddmm(src, a, b))
    assert peak <= E * 2 + nws + (1 << 20), (peak, E)
    a8, sa = ts.quantize_fp8(a)
    b8, sb = ts.quantize_fp8(b, per_row=False)
    for dt in OUTS:
        out8, peak = peak_above(lambda: ts.sddmm_fp8(src, a8, sa, b8, sb, dt))
        assert peak <= E * out8.element_size() + nws + (1 << 20), (peak, E, dt)


# ---- FP8 path ------------------------------------------------------------------------------------------------------------
FP8_KS = (16, 32, 48, 64, 128, 256, 400, 512, 1024, 2048)


@pytest.fixture(scope="module")
def fp8mat():
    """A smaller structured matrix for the wide FP8 rows: empty rows, rows of 1 ... 1300 nnz, a budget block."""
    M, N = 32 * 40 + 13, 3000
    specials = {5: 1, 37: 31, 38: 32, 39: 33, 200: 255, 201: 256, 202: 257, 500: 512, 501: 513, 900: 1300}
    rowptr, col = build_csr(M, N, 4, 11, specials, blocks=[64], tie_rows={300: 40, 301: 600},
                            empty_rows=(0, M // 2, M - 1))
    return dict(M=M, N=N, rowptr=rowptr, col=col)


def _vp(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def call_sddmm_fp8(rowptr, col, a8, sa, b8, sb, out_dtype, expect_rc=0):
    """tsb200_sddmm_fp8 into a NaN-prefilled output."""
    M, E = rowptr.numel() - 1, col.numel()
    N, K = b8.shape
    out = torch.full((E,), float("nan"), dtype=out_dtype, device=DEV)
    nws = lib.tsb200_sddmm_fp8_workspace_bytes(M, K, E)
    ws = torch.empty(max(nws, 256), dtype=torch.uint8, device=DEV)
    rc = lib.tsb200_sddmm_fp8(_vp(rowptr), _vp(col), _vp(a8), _vp(sa), 0 if sa.dim() == 0 else 1, _vp(b8), _vp(sb),
                              0 if sb.dim() == 0 else 1, _vp(out), M, N, K, E, ops._FP8_OUT[out_dtype], _vp(ws), nws,
                              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == expect_rc, rc
    return out


def fp8_operand(rows, K, seed, exact):
    """e4m3 [rows, K]: multiples of 1/2 in [-2, 2] (every fp32 partial sum of products exact), or randn * 4."""
    g = torch.Generator().manual_seed(seed)
    if exact:
        x = torch.randint(-4, 5, (rows, K), generator=g).float() / 2
    else:
        x = torch.randn(rows, K, generator=g) * 4
    return x.to(E4M3)


def fp8_scale(rows, seed, per_row, pow2):
    g = torch.Generator().manual_seed(seed)
    if pow2:
        s = torch.ldexp(torch.ones(rows), torch.randint(-3, 4, (rows,), generator=g))
    else:
        s = torch.rand(rows, generator=g) * 1.5 + 0.05
    return s if per_row else s[3].clone()


def replay(a8, sa, b8, sb, row, col):
    """(s_e in fp32, d_e exact in fp64, sum_k |qa qb| in fp64) on the CPU."""
    qa, qb = a8.cpu().float(), b8.cpu().float()
    sa_e = sa.cpu().expand(a8.size(0))[row] if sa.dim() == 0 else sa.cpu()[row]
    sb_e = sb.cpu().expand(b8.size(0))[col] if sb.dim() == 0 else sb.cpu()[col]
    return sa_e * sb_e, dots64(qa, qb, row, col), dots64(qa.abs(), qb.abs(), row, col)


def expected_bits(s, d, out_dtype):
    """round_out(fl32(s * d)) for d exact in fp32."""
    d32 = d.float()
    assert torch.equal(d32.double(), d), "the data is not exact-sum data"
    return (s * d32).to(out_dtype)


def fp8_bound_check(out, s, d, S, K, what):
    ref = s.double() * d
    e = (K + 2) * U32 * s.double().abs() * S
    bound = e + half_ulp(ref.abs() + e, out.dtype)
    err = (out.cpu().double() - ref).abs()
    ok = err <= bound
    if not bool(ok.all()):
        i = int((~ok).nonzero()[0])
        raise AssertionError(f"{what}: {int((~ok).sum())} of {ok.numel()} out of bound, first at {i}: "
                             f"{out[i].item()!r} vs {ref[i].item()!r} (bound {bound[i].item():.3e})")


@pytest.mark.parametrize("exact", [False, True], ids=["random", "exact"])
@pytest.mark.parametrize("K", FP8_KS)
def test_fp8_every_shape_scale_output_and_item_size(fp8mat, monkeypatch, K, exact):
    rowptr_c, col_c, M, N = fp8mat["rowptr"], fp8mat["col"], fp8mat["M"], fp8mat["N"]
    row_c = coo_row(rowptr_c)
    a8_c, b8_c = fp8_operand(M, K, K, exact), fp8_operand(N, K, K + 1, exact)
    rowptr, col, a8, b8 = _dev(rowptr_c, col_c, a8_c, b8_c)
    src = src_of(fp8mat)
    _, d, S = replay(a8_c, torch.ones(()), b8_c, torch.ones(()), row_c, col_c)
    for a_row in (True, False):
        for b_row in (True, False):
            sa_c, sb_c = fp8_scale(M, 1, a_row, exact), fp8_scale(N, 2, b_row, exact)
            s = (sa_c.expand(M)[row_c] if sa_c.dim() == 0 else sa_c[row_c]) * \
                (sb_c.expand(N)[col_c] if sb_c.dim() == 0 else sb_c[col_c])
            sa, sb = _dev(sa_c, sb_c)
            for out_dtype in OUTS:
                what = f"sddmm_fp8 K={K} a_row={a_row} b_row={b_row} {_id(out_dtype)}"
                want = expected_bits(s, d, out_dtype) if exact else None
                first = None
                for sh in SHIFTS:
                    monkeypatch.setenv(ENV, str(sh))
                    out = call_sddmm_fp8(rowptr, col, a8, sa, b8, sb, out_dtype)
                    if exact:
                        assert_bits_equal(out, want, f"{what} shift={sh}")
                    elif first is None:
                        fp8_bound_check(out, s, d, S, K, f"{what} shift={sh}")
                    if first is None:
                        first = out
                    assert_bits_equal(out, first, f"{what} shift={sh} vs shift 0")
                assert_bits_equal(ts.sddmm_fp8(src, a8, sa, b8, sb, out_dtype), first, what + " public")
                assert_bits_equal(src.sddmm_fp8(a8, sa, b8, sb, out_dtype), first, what + " method")


def _cdiv(a, b):
    return -(-a // b)


# The grid check profiles in a process of its own: a profiler session here would leave this pytest process's CUDA
# profiling state different from what the later kernel-name and grid checks of the suite start from.
GRID_PROBE = """
import json, sys
from pathlib import Path
sys.path[:0] = [sys.argv[1], str(Path(sys.argv[1]).parent)]
import os, torch
from test_sddmm_gpu import DEV, call_sddmm_fp8, fp8_operand
from test_spmm_item_sizes_gpu import kernel_grids
M, N = int(sys.argv[3]), 4600
g = torch.Generator().manual_seed(0)
deg = torch.randint(0, 9, (M,), generator=g)
rowptr = torch.zeros(M + 1, dtype=torch.long)
rowptr[1:] = deg.cumsum(0)
col = torch.randint(N, (int(rowptr[-1]),), generator=g)
rowptr, col = rowptr.to(DEV), col.to(DEV)
a8, b8 = fp8_operand(M, 128, 1, False).to(DEV), fp8_operand(N, 128, 2, False).to(DEV)
one = torch.ones((), device=DEV)
grids = {}
for s in range(2, 6):
    os.environ["TSB200_SPMM_ITEM_SHIFT"] = str(s)
    grids[s] = kernel_grids(lambda: call_sddmm_fp8(rowptr, col, a8, one, b8, one, torch.float32),
                            r"sddmm_vec_kernel<.*fp8", Path(sys.argv[2]))
print(json.dumps(grids))
"""


def _cdiv(a, b):
    return -(-a // b)


def test_fp8_override_reaches_the_new_kernels(tmp_path):
    """One item per warp: the main e4m3 kernel runs ceil(ceil(M / 2^s) / 8) CTAs at shifts 2 ... 5 (M = 2253: 71, 36,
    18 and 9, fewer than any persistent grid)."""
    M = 2253
    script = tmp_path / "grid_probe.py"
    script.write_text(GRID_PROBE)
    res = subprocess.run([sys.executable, str(script), str(Path(__file__).resolve().parent), str(tmp_path), str(M)],
                         capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stderr[-4000:]
    grids = json.loads(res.stdout.strip().splitlines()[-1])
    for s in range(2, 6):
        assert [tuple(g) for g in grids[str(s)]] == [(_cdiv(_cdiv(M, 1 << s), 8), 1, 1)], (s, grids)


def test_fp8_special_values(fp8mat):
    """NaN in either operand or scale propagates; a dot of +-0 products is +0 (the sum starts at +0), times a negative
    scale -0; e4m3 subnormals (2^-9 ... 7 * 2^-9) multiply exactly."""
    rowptr_c, col_c, M, N = fp8mat["rowptr"], fp8mat["col"], fp8mat["M"], fp8mat["N"]
    row_c = coo_row(rowptr_c)
    K = 48
    g = torch.Generator().manual_seed(5)
    a = torch.randint(-4, 5, (M, K), generator=g).float() / 2
    b = torch.randint(-4, 5, (N, K), generator=g).float() / 2
    a[10] = -0.0                                             # every product -0 or +0
    a[11, ::2] = -0.0
    a[11, 1::2] = 0.0
    a[15] = 0.0                                              # a zero dot under a negative scale
    sub = torch.arange(1, 8).float() * 2.0 ** -9            # e4m3 subnormals
    a[12] = sub[torch.randint(7, (K,), generator=g)]
    b[: N // 2, :8] = sub[torch.randint(7, (N // 2, 8), generator=g)]
    a8_c, b8_c = a.to(E4M3), b.to(E4M3)
    a8_c.view(torch.uint8)[13, 5] = 0x7F                    # NaN encodings in a row of a and in some rows of b
    b8_c.view(torch.uint8)[7::97, 9] = 0xFF
    sa_c = fp8_scale(M, 3, True, True)
    sa_c[14] = float("nan")
    sa_c[15] = -0.5
    sb_c = fp8_scale(N, 4, True, True)
    s, d, _ = replay(a8_c, sa_c, b8_c, sb_c, row_c, col_c)
    nan = d.isnan() | s.isnan()
    assert bool(nan.any()) and bool((~nan).any())
    rowptr, col, a8, b8, sa, sb = _dev(rowptr_c, col_c, a8_c, b8_c, sa_c, sb_c)
    for out_dtype in OUTS:
        out = call_sddmm_fp8(rowptr, col, a8, sa, b8, sb, out_dtype).cpu()
        assert torch.equal(out.isnan(), nan), out_dtype
        assert_bits_equal(out[~nan], expected_bits(s[~nan], d[~nan], out_dtype), f"special values {_id(out_dtype)}")
        zero_rows = ((row_c == 10) | (row_c == 11)) & ~nan
        assert bool(zero_rows.any()) and bool((out[zero_rows] == 0).all())
        assert not bool(out[zero_rows].signbit().any())
        neg = (row_c == 15) & ~nan
        assert bool(neg.any()) and bool((out[neg] == 0).all()) and bool(out[neg].signbit().all())


def test_fp8_matches_float_sddmm_on_dequantised_operands(fp8mat):
    rowptr_c, col_c, M, N = fp8mat["rowptr"], fp8mat["col"], fp8mat["M"], fp8mat["N"]
    row_c = coo_row(rowptr_c)
    src = src_of(fp8mat)
    g = torch.Generator().manual_seed(9)
    for K in (64, 400, 2048):
        a = (torch.randn(M, K, generator=g) * torch.logspace(-2, 2, M).view(-1, 1)).to(DEV)
        b = torch.randn(N, K, generator=g).to(DEV)
        for per_row in (True, False):
            a8, sa = ts.quantize_fp8(a, per_row)
            b8, sb = ts.quantize_fp8(b, per_row)
            af = a8.float() * (sa.view(-1, 1) if per_row else sa)
            bf = b8.float() * (sb.view(-1, 1) if per_row else sb)
            want = ts.sddmm(src, af, bf).cpu().double()
            got = ts.sddmm_fp8(src, a8, sa, b8, sb, torch.float32)
            S = dots64(af.abs(), bf.abs(), row_c, col_c)
            # both are within (K + 2) 2^-24 S of the exact dot of the dequantised operands
            assert bool(((got.cpu().double() - want).abs() <= 2 * (K + 3) * U32 * S + 1e-38).all()), (K, per_row)
            # the native and the CPU quantize_fp8 give the same operands, hence the same scores
            a8h, sah = ts.quantize_fp8(a.cpu(), per_row)
            b8h, sbh = ts.quantize_fp8(b.cpu(), per_row)
            again = ts.sddmm_fp8(src, *_dev(a8h, sah, b8h, sbh), torch.float32)
            assert_bits_equal(again, got, f"native vs CPU quantize_fp8 K={K} per_row={per_row}")


def test_fp8_empty():
    for M, N, E in ((5, 7, 0), (0, 7, 0)):
        src = SparseTensor(row=torch.empty(E, dtype=torch.long, device=DEV),
                           col=torch.empty(E, dtype=torch.long, device=DEV), sparse_sizes=(M, N))
        a8 = torch.zeros(M, 32, dtype=E4M3, device=DEV)
        b8 = torch.zeros(N, 32, dtype=E4M3, device=DEV)
        out = ts.sddmm_fp8(src, a8, torch.ones(M, device=DEV), b8, torch.ones((), device=DEV), torch.bfloat16)
        assert out.shape == (0,) and out.dtype == torch.bfloat16
    src = SparseTensor(row=torch.tensor([0, 2], device=DEV), col=torch.tensor([1, 1], device=DEV), sparse_sizes=(3, 2))
    out = ts.sddmm_fp8(src, torch.empty(3, 0, dtype=E4M3, device=DEV), torch.ones((), device=DEV),
                       torch.empty(2, 0, dtype=E4M3, device=DEV), torch.ones((), device=DEV))
    assert torch.equal(out, torch.zeros(2, device=DEV)) and not bool(out.signbit().any())


def test_errors():
    src = SparseTensor(row=torch.tensor([0, 1, 1], device=DEV), col=torch.tensor([1, 0, 2], device=DEV),
                       sparse_sizes=(2, 3))
    rowptr, col, _ = src.csr()
    row = src.storage.row()
    a = torch.randn(2, 16, device=DEV)
    b = torch.randn(3, 16, device=DEV)
    # float path
    with pytest.raises(RuntimeError, match="not implemented for 'torch.int64'"):
        ts.sddmm(src, a.long(), b.long())
    with pytest.raises(RuntimeError, match="same dtype"):
        ts.sddmm(src, a, b.double())
    with pytest.raises(RuntimeError, match="a must be 2-D"):
        ts.sddmm(src, a.view(2, 4, 4), b)
    with pytest.raises(RuntimeError, match="b must be 2-D"):
        torch.ops.tsb200.sddmm(row, rowptr, col, None, None, None, a, b.view(-1))
    with pytest.raises(RuntimeError, match="the sparse sizes"):
        ts.sddmm(src, a, b[:2])
    with pytest.raises(RuntimeError, match=r"a must be \[M, K\]"):
        ts.sddmm(src, a[:, :8], b)
    with pytest.raises(RuntimeError, match=r"a must be \[M, K\]"):
        ops.sddmm(row, rowptr, col, None, None, None, a[:1], b)
    with pytest.raises(RuntimeError, match="b must have 3 rows"):
        ops.sddmm(row, rowptr, col, src.storage.colptr(), src.storage.csr2csc(), None, a, torch.randn(4, 16,
                  device=DEV))
    # fp8 path
    a8, sa = ts.quantize_fp8(a)
    b8, sb = ts.quantize_fp8(b, per_row=False)
    ok = ts.sddmm_fp8(src, a8, sa, b8, sb)
    assert ok.dtype == torch.float32 and ok.shape == (3,)
    with pytest.raises(RuntimeError, match="forward only"):
        ts.sddmm_fp8(src, a8, sa.clone().requires_grad_(), b8, sb)
    with pytest.raises(RuntimeError, match="forward only"):
        ts.sddmm_fp8(src, a8, sa, b8, sb.clone().requires_grad_())
    with torch.no_grad():
        ts.sddmm_fp8(src, a8, sa.clone().requires_grad_(), b8, sb)
    with pytest.raises(RuntimeError, match="a8 must be torch.float8_e4m3fn"):
        ts.sddmm_fp8(src, a, sa, b8, sb)
    with pytest.raises(RuntimeError, match="b8 must be torch.float8_e4m3fn"):
        ts.sddmm_fp8(src, a8, sa, b8.to(torch.float8_e5m2), sb)
    with pytest.raises(RuntimeError, match="b8 must be 2-D"):
        ts.sddmm_fp8(src, a8, sa, b8.view(3, 2, 8), sb)
    with pytest.raises(RuntimeError, match="the sparse sizes"):
        ts.sddmm_fp8(src, a8, sa, b8[:2], sb)
    with pytest.raises(RuntimeError, match=r"a8 must be \[M, K\]"):
        ts.sddmm_fp8(src, a8[:1], sa[:1], b8, sb)
    w8 = torch.zeros(2, 24, dtype=E4M3, device=DEV)
    with pytest.raises(ValueError, match="multiple of 16"):
        ts.sddmm_fp8(src, w8, sa, torch.zeros(3, 24, dtype=E4M3, device=DEV), sb)
    with pytest.raises(ValueError, match="at most 2048"):
        ts.sddmm_fp8(src, torch.zeros(2, 2064, dtype=E4M3, device=DEV), sa,
                     torch.zeros(3, 2064, dtype=E4M3, device=DEV), sb)
    with pytest.raises(RuntimeError, match="contiguous and 16-byte aligned"):
        ts.sddmm_fp8(src, torch.zeros(16, 2, dtype=E4M3, device=DEV).t(), sa, b8, sb)
    buf = torch.zeros(3 * 16 + 1, dtype=E4M3, device=DEV)
    with pytest.raises(RuntimeError, match="contiguous and 16-byte aligned"):
        ts.sddmm_fp8(src, a8, sa, buf[1:].view(3, 16), sb)
    with pytest.raises(RuntimeError, match="out_dtype must be"):
        ts.sddmm_fp8(src, a8, sa, b8, sb, torch.float64)
    with pytest.raises(RuntimeError, match="a_scale must be float32"):
        ts.sddmm_fp8(src, a8, sa.double(), b8, sb)
    with pytest.raises(RuntimeError, match=r"b_scale must have shape \[\] or \[3\]"):
        ts.sddmm_fp8(src, a8, sa, b8, torch.ones(2, device=DEV))
    with pytest.raises(RuntimeError, match="a_scale must be CUDA tensor"):
        ts.sddmm_fp8(src, a8, sa.cpu(), b8, sb)
    # the C-ABI refuses a short workspace on a real launch
    call = lib.tsb200_sddmm_fp8
    ws = torch.empty(256, dtype=torch.uint8, device=DEV)
    out = torch.empty(3, device=DEV)
    assert call(_vp(rowptr), _vp(col), _vp(a8), _vp(sa), 1, _vp(b8), _vp(sb), 0, _vp(out), 2, 3, 16, 3, 0, _vp(ws), 1,
                None) == -3
