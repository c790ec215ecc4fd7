"""SpMM backward kernels against the oracle, with error bounds taken from the kernels' rounding model.

* tsb200_spmm_value_bw (SDDMM): every family of `dispatch_sddmm` (row-wise, B = 1, 3..64 vectors per dense row) and of
  `dispatch_value_vec` (nnz-parallel: B = 1 with 1, 2 or > 64 vectors, any B otherwise), and the generic kernel, on the
  structured matrices of test_spmm_kernels_gpu (segments, budget deferral, full-size items). Bound:
  |out - ref64| <= 1/2 ulp_T(ref64) + (K*B + 1) * u * sum|mat * grad|; a mean adds the roundings of the division.
* tsb200_spmm_minmax_bw: every feature slice width (TSB200_MMBW_LSL, read on every call), both / one gradient, with and
  without values, arg_out from the forward kernel itself (so it holds the E sentinel of empty and no-winner rows).
  The kernel adds exact (16-bit) or once-rounded (fp32) products with fp32 atomics in any order:
  |out - ref64| <= (n + 1) * 2^-24 * sum|terms|, n = the number of terms routed to that element.
Outputs are prefilled with NaN, so an element a kernel fails to write cannot pass.
"""
import ctypes

import pytest
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import ops
from pytorch_sparse_b200._lib import lib
from test_spmm_kernels_gpu import (DEV, F16S, NAN_ROWS, _dev, _id, _stream, _vp, assert_bits_equal,  # noqa: F401
                                   assert_sum_bound, call_fw, dense, large, small, sub_csr, values)

pytestmark = pytest.mark.gpu
U = {torch.float32: 2.0 ** -24, torch.bfloat16: 2.0 ** -24, torch.float16: 2.0 ** -24, torch.float64: 2.0 ** -53}


def sddmm_family(dtype, K, B):
    """The kernel family tsb200_spmm_value_bw runs (with a workspace and aligned operands)."""
    es = torch.empty(0, dtype=dtype).element_size()
    if dtype not in (torch.float32, torch.bfloat16, torch.float16) or (K * es) % 16:
        return "generic"
    vecs = K * es // 16
    if B == 1 and 3 <= vecs <= 64:
        for lim, fam in ((4, "row4"), (8, "row8"), (16, "row16"), (32, "row32"), (64, "row32ch2")):
            if vecs <= lim:
                return fam
    for lim, fam in ((1, "nnz1"), (4, "nnz4"), (8, "nnz8"), (16, "nnz16"), (32, "nnz32")):
        if vecs <= lim:
            return fam
    return "nnz32strided"


# (dtype, K, B): every row-wise family at full and partial width, every nnz-parallel family at B = 1 / 2 / 3
ROWWISE = [(torch.float32, K, 1) for K in (12, 16, 20, 32, 40, 64, 128, 200, 256)] + \
          [(dt, K, 1) for dt in F16S for K in (24, 32, 40, 64, 72, 128, 256, 392, 512)]
NNZ = [(torch.float32, K, 1) for K in (4, 8, 300)] + [(dt, K, 1) for dt in F16S for K in (8, 16, 600)] + \
      [(torch.float32, K, B) for B in (2, 3) for K in (4, 12, 32, 40, 128, 200)] + \
      [(dt, K, B) for dt in F16S for B in (2, 3) for K in (8, 24, 64, 72, 256, 392)]
GENERIC = [(torch.float32, 6, 1), (torch.float64, 8, 1), (torch.float64, 8, 2), (torch.bfloat16, 7, 1),
           (torch.float16, 12, 2)]
assert {sddmm_family(*c) for c in ROWWISE} == {"row4", "row8", "row16", "row32", "row32ch2"}
assert {sddmm_family(*c) for c in NNZ} == {"nnz1", "nnz4", "nnz8", "nnz16", "nnz32", "nnz32strided"}
assert {sddmm_family(*c) for c in GENERIC} == {"generic"}


def call_value_bw(row, rowptr, col, mat, grad, reduce):
    """tsb200_spmm_value_bw into a NaN-prefilled output."""
    E = row.numel()
    N, K = mat.shape[-2:]
    M = grad.size(-2)
    B = mat.numel() // (N * K)
    dt = ops._dtype_code(mat.dtype)
    out = torch.full((E,), float("nan"), dtype=mat.dtype, device=DEV)
    nws = lib.tsb200_spmm_value_bw_workspace_bytes(B, M, K, E, dt)
    ws = torch.empty(max(nws, 1), dtype=torch.uint8, device=DEV)
    rc = lib.tsb200_spmm_value_bw(_vp(row), _vp(rowptr), _vp(col), _vp(mat), _vp(grad), _vp(out), B, M, N, K, E, dt,
                                  ops._REDUCE[reduce], _vp(ws) if nws else None, nws, _stream())
    assert rc == 0, rc
    return out


def check_value_bw(oracle, rowptr_c, col_c, mat_c, grad_c, reduce, out, what):
    M = rowptr_c.numel() - 1
    row_c = torch.repeat_interleave(torch.arange(M), rowptr_c[1:] - rowptr_c[:-1])
    K = mat_c.size(-1)
    B = mat_c.numel() // (mat_c.size(-2) * K)
    ref = oracle.spmm_value_bw(row_c, rowptr_c, col_c, mat_c.double(), grad_c.double(), "sum")
    S = oracle.spmm_value_bw(row_c, rowptr_c, col_c, mat_c.double().abs(), grad_c.double().abs(), "sum")
    n = K * B + 1
    cnt = None
    if reduce == "mean":
        cnt = (rowptr_c[1:] - rowptr_c[:-1]).clamp(min=1)[row_c].double()
        ref = ref / cnt
    u = U[mat_c.dtype]
    if reduce == "mean":
        # the row-wise kernel multiplies by a rounded reciprocal (two roundings), the others divide (one)
        e = n * u * S / cnt
        e = e + (2 * u + u * u) * (ref.abs() + e)
        assert_sum_bound(out, ref, e, 1.0, mat_c.dtype, u=1.0, what=what)
    else:
        assert_sum_bound(out, ref, S, n, mat_c.dtype, u=u, what=what)


def _operands(N, M, K, B, dtype, seed):
    mat = dense(N, K, dtype, seed, False, B=None if B == 1 else B)
    g = torch.Generator().manual_seed(seed + 1)
    grad = torch.randn((M, K) if B == 1 else (B, M, K), generator=g, dtype=torch.float64).to(dtype)
    return mat, grad


@pytest.mark.parametrize("reduce", ["sum", "mean"])
@pytest.mark.parametrize("dtype,K,B", ROWWISE + NNZ + GENERIC, ids=_id)
def test_value_bw_family(oracle, small, dtype, K, B, reduce):
    rowptr_c, col_c, N, M = small["rowptr"], small["col"], small["N"], small["M"]
    mat_c, grad_c = _operands(N, M, K, B, dtype, K + B)
    row = torch.repeat_interleave(torch.arange(M), rowptr_c[1:] - rowptr_c[:-1])
    out = call_value_bw(*_dev(row, rowptr_c, col_c, mat_c, grad_c), reduce)
    check_value_bw(oracle, rowptr_c, col_c, mat_c, grad_c, reduce, out,
                   f"value_bw {sddmm_family(dtype, K, B)} {dtype} K={K} B={B} {reduce}")


@pytest.mark.parametrize("dtype,K", [(torch.float32, 16), (torch.bfloat16, 64), (torch.float16, 128),
                                     (torch.float32, 128), (torch.bfloat16, 512)], ids=_id)
def test_value_bw_full_size_items(oracle, large, dtype, K):
    """Row-wise SDDMM with 32-row items (budget deferral into the segment kernel); every nnz written, a sample of
    whole 32-row groups against the oracle."""
    rowptr_c, col_c, N, M, rows = large["rowptr"], large["col"], large["N"], large["M"], large["rows"]
    mat_c, grad_c = _operands(N, M, K, 1, dtype, 3)
    row = torch.repeat_interleave(torch.arange(M), rowptr_c[1:] - rowptr_c[:-1])
    for reduce in ("sum", "mean"):
        out = call_value_bw(*_dev(row, rowptr_c, col_c, mat_c, grad_c), reduce)
        assert not bool(out.isnan().any()), "value_bw: an nnz was not written"
        sp, scol, idx = sub_csr(rowptr_c, col_c, rows)
        check_value_bw(oracle, sp, scol, mat_c, grad_c[rows], reduce, out[idx.to(DEV)],
                       f"value_bw {dtype} K={K} M={M} {reduce}")


# ---- fused min/max backward ------------------------------------------------------------------------------------------
def call_minmax_bw(col, value, mat, grad_out, arg_out, need_value, need_mat):
    """tsb200_spmm_minmax_bw into zeroed fp32 / fp64 accumulators (as the library requires), returned unrounded."""
    N, K = mat.shape[-2:]
    M = grad_out.size(-2)
    E = col.numel()
    B = mat.numel() // (N * K)
    acc = torch.float64 if mat.dtype == torch.float64 else torch.float32
    gv = torch.zeros(E, dtype=acc, device=DEV) if need_value else None
    gm = torch.zeros(mat.shape, dtype=acc, device=DEV) if need_mat else None
    rc = lib.tsb200_spmm_minmax_bw(_vp(col), _vp(value), _vp(mat), _vp(grad_out), _vp(arg_out), _vp(gv), _vp(gm),
                                   B, M, N, K, E, ops._dtype_code(mat.dtype), _stream())
    assert rc == 0, rc
    return gv, gm


def check_accumulated(got, ref, S, n, u, what):
    got = got.cpu().double()
    bound = (n + 1) * u * S
    ok = (got - ref).abs() <= bound
    if not bool(ok.all()):
        i = tuple(int(j) for j in (~ok).nonzero()[0])
        raise AssertionError(f"{what}: {int((~ok).sum())} out of bound, first at {i}: {got[i].item()!r} vs "
                             f"{ref[i].item()!r} (bound {bound[i].item():.3e})")


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("K", [40, 100, 256])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16, torch.float64], ids=_id)
def test_minmax_bw_slices(oracle, small, monkeypatch, dtype, K, B):
    rowptr_c, col_c, N, M = small["rowptr"], small["col"], small["N"], small["M"]
    E = col_c.numel()
    g = torch.Generator().manual_seed(K + B)
    mat_c = dense(N, K, dtype, K, False, B=None if B == 1 else B)
    mat_c = torch.nan_to_num(mat_c, nan=1.0)
    val_c = torch.randn(E, generator=g, dtype=torch.float64)
    val_c[rowptr_c[500]:rowptr_c[501]] = float("nan")  # a multi-segment row without a winner: arg_out = E
    val_c = val_c.to(dtype)
    grad_c = torch.randn(mat_c.shape[:-2] + (M, K), generator=g, dtype=torch.float64).to(dtype)
    rowptr, col, val, mat, grad = _dev(rowptr_c, col_c, val_c, mat_c, grad_c)
    full = max(0, (K - 1).bit_length())
    for reduce in ("min", "max"):
        _, arg = call_fw(rowptr, col, val, mat, reduce)  # the forward's own arg_out (E sentinels included)
        assert bool((arg == E).any())
        arg_c = arg.cpu()
        for value_c, value in ((val_c, val), (None, None)):
            v64 = None if value_c is None else value_c.double()
            ones = None if value_c is None else torch.ones(E, dtype=torch.float64)
            for need_value, need_mat in ((True, True), (True, False), (False, True)):
                ref_v, ref_m = oracle.spmm_minmax_bw(col_c, v64, mat_c.double(), grad_c.double(), arg_c,
                                                     need_value, need_mat)
                S_v, S_m = oracle.spmm_minmax_bw(col_c, None if v64 is None else v64.abs(), mat_c.double().abs(),
                                                 grad_c.double().abs(), arg_c, need_value, need_mat)
                n_v, n_m = oracle.spmm_minmax_bw(col_c, ones, torch.ones(mat_c.shape, dtype=torch.float64),
                                                 torch.ones(grad_c.shape, dtype=torch.float64), arg_c,
                                                 need_value, need_mat)
                for lsl in sorted({0, 1, 3, 6, full}):
                    monkeypatch.setenv("TSB200_MMBW_LSL", str(lsl))
                    gv, gm = call_minmax_bw(col, value, mat, grad, arg, need_value, need_mat)
                    what = f"{dtype} K={K} B={B} {reduce} value={value is not None} lsl={lsl}"
                    if need_value:
                        check_accumulated(gv, ref_v, S_v, n_v, U[dtype], what + " grad_value")
                    if need_mat:
                        check_accumulated(gm, ref_m, S_m, n_m, U[dtype], what + " grad_mat")


def test_matmul_max_backward_planned_equals_unplanned():
    """ts.matmul(..., "max") twice on the same SparseTensor in f16 at K = 128: the second call takes the auto-plan path
    (planned forward kernel). Outputs and both gradients are bit-identical. Operands are multiples of 1/4, so every
    gradient sum is exact in fp32 and the atomics' order cannot change a bit."""
    g = torch.Generator().manual_seed(9)
    M, N, K = 3000, 2000, 128
    deg = torch.poisson(torch.full((M,), 10.0), generator=g).long()
    deg[[3, 4, 5]] = torch.tensor([1500, 700, 300])
    deg[[0, 10]] = 0
    rowptr = torch.zeros(M + 1, dtype=torch.long)
    rowptr[1:] = deg.cumsum(0)
    E = int(rowptr[-1])
    col = torch.randint(N, (E,), generator=g)
    q = lambda *s: (torch.randint(-8, 9, s, generator=g) * 0.25).half().to(DEV)  # noqa: E731
    v, x, go = q(E).requires_grad_(), q(N, K).requires_grad_(), q(M, K)
    a = ts.SparseTensor(rowptr=rowptr.to(DEV), col=col.to(DEV), value=v, sparse_sizes=(M, N), is_sorted=True,
                        trust_data=True)
    ops._PLAN_CACHE.clear()
    res = []
    for _ in range(2):
        out = ts.matmul(a, x, "max")
        res.append((out.detach(),) + torch.autograd.grad(out, (v, x), go))
        res[-1] += (any(ent[1] is not None for ent in ops._PLAN_CACHE.values()),)
    assert res[0][-1] is False and res[1][-1] is True, "the second call did not take the planned path"
    for t0, t1 in zip(res[0][:-1], res[1][:-1]):
        assert_bits_equal(t1, t0, "planned vs unplanned matmul max")
