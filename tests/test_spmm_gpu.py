"""GPU parity of the CSR SpMM forward/backward against the oracle (CPU restatement of
csrc/cpu/spmm_cpu.cpp) — mirrors test/test_matmul.py::test_spmm of the reference."""
from itertools import product

import pytest
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import ops
from util import fast_random_csr, random_csr

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REDUCES = ["sum", "mean", "min", "max"]
# fp tolerances stated by BASELINE.json north_star: 1e-5 rel fp32, 1e-2 rel bf16 (fp16 ~ 2e-3)
TOL = {torch.float32: 1e-5, torch.float64: 1e-12, torch.bfloat16: 1e-2, torch.float16: 2e-3}


def _abs_bound(rowptr, col, value, mat):
    """componentwise normaliser |A| @ |B| (SURVEY §8d parity checks), fp64 on CPU via the oracle."""
    import oracle
    v = None if value is None else value.double().abs()
    out, _ = oracle.spmm(rowptr, col, v, mat.double().abs(), "sum")
    return out


def _check_forward(oracle, rowptr, col, value, mat, reduce):
    out, arg = ops.spmm_fw(rowptr.to(DEV), col.to(DEV), None if value is None else value.to(DEV), mat.to(DEV), reduce)
    # reference semantics in exact arithmetic: oracle in fp64 on the (upcast) inputs
    ref64, arg64 = oracle.spmm(rowptr, col, None if value is None else value.double(), mat.double(), reduce)
    tol = TOL.get(mat.dtype)
    if mat.dtype.is_floating_point:
        bound = _abs_bound(rowptr, col, value, mat).clamp_min(1e-30)
        if reduce == "mean":
            pass  # |mean| <= |sum| bound still valid
        err = ((out.cpu().double() - ref64).abs() / bound).max().item() if out.numel() else 0.0
        assert err <= tol, f"{reduce} {mat.dtype}: rel err {err:.3e} > {tol}"
    else:
        assert torch.equal(out.cpu(), ref64.to(mat.dtype))
    if reduce in ("min", "max"):
        # the reference compares products rounded to the storage dtype: oracle in the storage dtype
        ref_t, arg_t = oracle.spmm(rowptr, col, value, mat, reduce)
        assert torch.equal(arg.cpu(), arg_t), f"arg_out mismatch ({reduce}, {mat.dtype})"
        assert torch.equal(out.cpu(), ref_t), f"min/max values must be bit-exact ({reduce}, {mat.dtype})"
    return out, arg


@pytest.mark.parametrize("dtype,reduce", list(product([torch.float32, torch.bfloat16, torch.float16, torch.float64,
                                                       torch.int32, torch.int64], REDUCES)))
def test_reference_shape(oracle, dtype, reduce):
    """10x8 with empty rows 2-3 / empty cols 2-3, other [2, 8, 2] — test/test_matmul.py:18-25."""
    torch.manual_seed(1)
    dense = torch.randn(10, 8)
    dense[2:4, :] = 0
    dense[:, 2:4] = 0
    if not dtype.is_floating_point:
        dense = (dense * 4).round()
    src = ts.SparseTensor.from_dense(dense.to(dtype))
    rowptr, col, value = src.csr()
    other = torch.randn(2, 8, 2)
    other = (other * 4).round().to(dtype) if not dtype.is_floating_point else other.to(dtype)
    _check_forward(oracle, rowptr, col, value, other, reduce)
    _check_forward(oracle, rowptr, col, None, other, reduce)


SHAPES = [  # (M, N, K, avg_deg, power_law)
    (300, 200, 128, 16, False),
    (257, 300, 32, 5, False),
    (100, 90, 256, 12, True),
    (64, 50, 8, 3, False),
    (50, 70, 520, 6, False),    # bf16: 65 vectors -> CH=4 tile path
    (40, 60, 1100, 4, False),   # fp32: 275 vectors -> column-tiled launches
    (33, 20, 7, 4, False),      # odd K -> generic kernel
]


@pytest.mark.parametrize("shape,dtype,reduce", list(product(SHAPES, [torch.float32, torch.bfloat16], REDUCES)))
def test_random_shapes(oracle, shape, dtype, reduce):
    M, N, K, deg, pl = shape
    row, rowptr, col = random_csr(M, N, deg, seed=M + K, power_law=pl, empty_rows=(0, M // 2, M - 1))
    g = torch.Generator().manual_seed(7)
    value = torch.randn(col.numel(), generator=g).to(dtype)
    mat = torch.randn(N, K, generator=g).to(dtype)
    _check_forward(oracle, rowptr, col, value, mat, reduce)


@pytest.mark.parametrize("dtype,reduce", list(product([torch.float32, torch.bfloat16], REDUCES)))
def test_long_rows_and_budget(oracle, dtype, reduce):
    """rows longer than the 256-nnz segment length (multi-segment combine), a row of exactly 256/257,
    and a dense 32-row block that exceeds the 1024-nnz item budget (single-segment deferral)."""
    M, N, K = 200, 1500, 64
    long_rows = [(5, 1400), (6, 256), (7, 257), (100, 700)] + [(r, 60) for r in range(128, 160)]
    row, rowptr, col = random_csr(M, N, 4, seed=3, empty_rows=(0, 8, 199), long_rows=long_rows)
    g = torch.Generator().manual_seed(11)
    value = torch.randn(col.numel(), generator=g).to(dtype)
    mat = torch.randn(N, K, generator=g).to(dtype)
    _check_forward(oracle, rowptr, col, value, mat, reduce)
    _check_forward(oracle, rowptr, col, None, mat, reduce)


def test_ties_keep_first(oracle):
    """duplicate maxima: strict compare keeps the smallest nnz index (csrc/cpu/reducer.h:63-67)."""
    rowptr = torch.tensor([0, 600, 600, 603])
    col = torch.cat([torch.arange(600) % 7, torch.tensor([1, 1, 2])])
    value = torch.ones(603)
    mat = torch.ones(7, 16)
    for reduce in ("min", "max"):
        out, arg = _check_forward(oracle, rowptr, col, value, mat, reduce)
        assert arg[0].eq(0).all() and arg[1].eq(603).all() and arg[2].eq(600).all()
        assert out[1].eq(0).all()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float64])
@pytest.mark.parametrize("reduce", ["sum", "mean"])
def test_value_bw(oracle, dtype, reduce):
    for (M, N, K, B) in [(120, 90, 128, 1), (60, 40, 32, 2), (30, 20, 6, 3)]:
        row, rowptr, col = random_csr(M, N, 6, seed=K, power_law=True, empty_rows=(1,))
        g = torch.Generator().manual_seed(5)
        mat = torch.randn(B, N, K, generator=g).to(dtype)
        grad = torch.randn(B, M, K, generator=g).to(dtype)
        out = ops.spmm_value_bw(row.to(DEV), rowptr.to(DEV), col.to(DEV), mat.to(DEV), grad.to(DEV), reduce)
        ref = oracle.spmm_value_bw(row, rowptr, col, mat.double(), grad.double(), reduce)
        bound = oracle.spmm_value_bw(row, rowptr, col, mat.double().abs(), grad.double().abs(), reduce)
        err = ((out.cpu().double() - ref).abs() / bound.clamp_min(1e-30)).max().item()
        assert err <= TOL[dtype], f"value_bw {dtype} {reduce}: {err:.3e}"


@pytest.mark.parametrize("dtype,reduce", list(product([torch.float32, torch.float64, torch.bfloat16, torch.float16],
                                                      ["sum", "add", "mean", "min", "max"])))
def test_autograd_like_reference(oracle, dtype, reduce):
    """forward + grad wrt value + grad wrt other through matmul(), as test/test_matmul.py:12-51,
    expected values from dense autograd in fp64."""
    torch.manual_seed(3)
    dense = torch.randn(10, 8, dtype=torch.float64)
    dense[2:4, :] = 0
    dense[:, 2:4] = 0
    src = ts.SparseTensor.from_dense(dense.to(dtype).to(DEV)).requires_grad_()
    row, col, value = src.coo()
    other = torch.randn(2, 8, 2, dtype=torch.float64).to(dtype).to(DEV).requires_grad_()

    # expected: fp64 dense formulation of the same reduction
    v64 = value.detach().double().cpu().requires_grad_()
    o64 = other.detach().double().cpu().requires_grad_()
    r, c = row.cpu(), col.cpu()
    src_col = o64.index_select(-2, c) * v64.unsqueeze(-1)  # [2, E, 2]
    M = 10
    if reduce in ("sum", "add", "mean"):
        exp = torch.zeros(2, M, 2, dtype=torch.float64).index_add(-2, r, src_col)
        if reduce == "mean":
            cnt = torch.bincount(r, minlength=M).clamp(min=1).view(1, M, 1)
            exp = exp / cnt
    else:
        fill = float("inf") if reduce == "min" else float("-inf")
        exp = torch.full((2, M, 2), fill, dtype=torch.float64)
        idx = r.view(1, -1, 1).expand_as(src_col)
        exp = exp.scatter_reduce(-2, idx, src_col, reduce="amin" if reduce == "min" else "amax", include_self=True)
        exp = torch.where(torch.isinf(exp), torch.zeros_like(exp), exp)
    grad_out = torch.randn(2, M, 2, dtype=torch.float64)
    exp.backward(grad_out)

    out = ts.matmul(src, other, reduce)
    out.backward(grad_out.to(dtype).to(DEV))
    atol = 1e-1 if dtype in (torch.float16, torch.bfloat16) else (1e-5 if dtype == torch.float32 else 1e-10)
    assert torch.allclose(exp, out.detach().double().cpu(), atol=atol)
    assert torch.allclose(v64.grad, value.grad.double().cpu(), atol=atol)
    assert torch.allclose(o64.grad, other.grad.double().cpu(), atol=atol)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_minmax_backward_vs_oracle(oracle, dtype):
    M, N, K = 150, 120, 64
    row, rowptr, col = random_csr(M, N, 8, seed=9, power_law=True, empty_rows=(3, 4))
    g = torch.Generator().manual_seed(2)
    value = torch.randn(col.numel(), generator=g).to(dtype)
    mat = torch.randn(N, K, generator=g).to(dtype)
    grad_out = torch.randn(M, K, generator=g).to(dtype)
    for reduce in ("min", "max"):
        _, arg = oracle.spmm(rowptr, col, value, mat, reduce)
        gv, gm = ops.spmm_minmax_bw(col.to(DEV), value.to(DEV), mat.to(DEV), grad_out.to(DEV), arg.to(DEV), True, True)
        rv, rm = oracle.spmm_minmax_bw(col, value.double(), mat.double(), grad_out.double(), arg)
        tol = 1e-5 if dtype == torch.float32 else 2e-2
        assert torch.allclose(gv.double().cpu(), rv, rtol=tol, atol=tol)
        assert torch.allclose(gm.double().cpu(), rm, rtol=tol, atol=tol)


def test_full_size_properties():
    """BASELINE config 2 at full size (1M x 1M, ~16 nnz/row, F=128 bf16): size-independent properties —
    linearity in the dense operand, row-sum identity with an all-ones operand, agreement of the
    bf16 result with the fp32 kernel on the same (bf16-representable) inputs, and row-block
    decomposition (SpMM of a row slice == slice of the SpMM)."""
    M = N = 1_000_000
    F = 128
    row, rowptr, col = fast_random_csr(M, N, 16, seed=1, device=DEV)
    E = col.numel()
    g = torch.Generator(device=DEV).manual_seed(2)
    value = (torch.rand(E, generator=g, device=DEV) + 0.5).bfloat16()
    x = torch.randn(N, F, generator=g, device=DEV).bfloat16()
    y, _ = ops.spmm_fw(rowptr, col, value, x, "sum")
    y32, _ = ops.spmm_fw(rowptr, col, value.float(), x.float(), "sum")
    absb, _ = ops.spmm_fw(rowptr, col, value.float().abs(), x.float().abs(), "sum")
    err = ((y.float() - y32).abs() / absb.clamp_min(1e-20)).max().item()
    assert err <= 1e-2, err
    # all-ones operand: out[m, :] == sum of the row's values (exactly representable check in fp32)
    ones = torch.ones(N, 8, device=DEV)
    rs, _ = ops.spmm_fw(rowptr, col, value.float(), ones, "sum")
    rowsum = torch.zeros(M, device=DEV).index_add_(0, row, value.float())
    assert torch.allclose(rs[:, 0], rowsum, rtol=1e-5, atol=1e-5)
    # linearity: A(2x) == 2 A(x) exactly (power-of-two scaling)
    y2, _ = ops.spmm_fw(rowptr, col, value, (x.float() * 2).bfloat16(), "sum")
    assert torch.equal(y2.float(), (y.float() * 2).bfloat16().float())
    # row-block decomposition. The value slice is copied: a bf16 slice that starts at an odd entry is not 4-byte
    # aligned and takes the generic kernel, whose separate multiply and add round differently. Where it starts
    # depends on the matrix, and the CUDA generator draws a different one on GPUs with different SM counts.
    r0, r1 = 123_456, 345_678
    sub = rowptr[r0:r1 + 1]
    lo, hi = int(sub[0]), int(sub[-1])
    ys, _ = ops.spmm_fw(sub - lo, col[lo:hi], value[lo:hi].clone(), x, "sum")
    assert torch.equal(ys, y[r0:r1])
    # max: arg_out points at an entry of the row whose product equals the output
    ym, am = ops.spmm_fw(rowptr, col, value, x, "max")
    nonempty = (rowptr[1:] - rowptr[:-1]) > 0
    am_ne = am[nonempty]
    assert (am_ne >= rowptr[:-1][nonempty].unsqueeze(1)).all() and (am_ne < rowptr[1:][nonempty].unsqueeze(1)).all()
    pick = torch.randint(M, (4096,), device=DEV)
    pick = pick[nonempty[pick]]
    k = torch.arange(F, device=DEV)
    a = am[pick]
    prod = (value[a].float() * x[col[a], k.unsqueeze(0).expand_as(a)].float()).bfloat16()
    assert torch.equal(prod, ym[pick])


@pytest.mark.parametrize("wl", ["c2", "c2_f32", "c2_f256"])
def test_full_size_c2_vs_oracle(oracle, wl):
    """BASELINE configs[1] at FULL size and its F = 32 / F = 256 variants (north_star: F in {32, 128, 256}),
    directly against the oracle (fp32 restatement on the bf16 inputs, OpenMP over rows): every output within 1e-2
    of the |A||B| bound, and the fp32 kernel within 1e-5."""
    import bench
    w = bench.WORKLOADS[wl]
    rowptr, col, value, N = bench.gen_matrix(w, 0, 1)
    x = bench.gen_dense(w, 0, N)
    vb, xb = value.bfloat16(), x.bfloat16()
    ref, _ = oracle.spmm(rowptr, col, vb.float(), xb.float(), "sum")          # exact products, fp32 sums
    bound, _ = oracle.spmm(rowptr, col, vb.float().abs(), xb.float().abs(), "sum")
    bound.clamp_(min=1e-20)
    d = [t.to(DEV) for t in (rowptr, col)]
    out_bf16, _ = ops.spmm_fw(d[0], d[1], vb.to(DEV), xb.to(DEV), "sum")
    err = ((out_bf16.cpu().float() - ref).abs() / bound).max().item()
    assert err <= 1e-2, err
    out_f32, _ = ops.spmm_fw(d[0], d[1], vb.float().to(DEV), xb.float().to(DEV), "sum")
    err32 = ((out_f32.cpu() - ref).abs() / bound).max().item()
    assert err32 <= 1e-5, err32


def test_full_size_c3_max_vs_oracle(oracle):
    """BASELINE configs[2] at FULL size (500k x 500k power-law, F=256 fp32, max): values and arg_out
    BIT-EXACT against the oracle, including the rows split into segments and the empty rows."""
    import bench
    w = bench.WORKLOADS["c3"]
    rowptr, col, value, N = bench.gen_matrix(w, 0, 1)
    x = bench.gen_dense(w, 0, N)
    ref, rarg = oracle.spmm(rowptr, col, value, x, "max")
    out, arg = ops.spmm_fw(rowptr.to(DEV), col.to(DEV), value.to(DEV), x.to(DEV), "max")
    assert torch.equal(arg.cpu(), rarg)
    assert torch.equal(out.cpu(), ref)
    # backward through the fused min/max kernel vs the oracle's restatement of the ATen chain
    g = torch.Generator().manual_seed(3)
    go = torch.randn(w["M"], w["F"], generator=g)
    gv, gm = ops.spmm_minmax_bw(col.to(DEV), value.to(DEV), x.to(DEV), go.to(DEV), arg, True, True)
    rv, rm = oracle.spmm_minmax_bw(col, value.double(), x.double(), go.double(), rarg)
    # north_star tolerance: 1e-5 relative in fp32, against the componentwise |A||B| normaliser (SURVEY §8d) — the
    # same routing applied to the absolute values bounds every accumulated sum. The kernel adds in fp32 with atomics
    # (run-dependent order): the error of a sum of n terms is <= n * 2^-24 * sum|terms|, n <= K = 256 for
    # grad_value and <= the column degree for grad_mat, i.e. <= 1.6e-5 worst case and ~sqrt(n) * 6e-8 in practice.
    bv, bm = oracle.spmm_minmax_bw(col, value.double().abs(), x.double().abs(), go.double().abs(), rarg)
    assert ((gv.cpu().double() - rv).abs() <= 1e-5 * bv + 1e-30).all()
    assert ((gm.cpu().double() - rm).abs() <= 1e-5 * bm + 1e-30).all()


@pytest.mark.parametrize("dtype,K", [(torch.float32, 64), (torch.bfloat16, 128), (torch.float16, 32)])
@pytest.mark.parametrize("P", [2, 3])
def test_column_block_accumulate_modes_vs_oracle(oracle, dtype, K, P):
    """tsb200_spmm_fw_acc: a SUM SpMM assembled from P column blocks through the fp32 partial (first / middle / last
    block modes), on a power-law matrix whose long rows go through the segment queue and the combine kernel —
    against the oracle's single pass on the same inputs."""
    from pytorch_sparse_b200.parallel import split_column_chunks
    M, N = 3000, 3 * 1024
    row, rowptr, col = random_csr(M, N, 12, seed=5, power_law=True, empty_rows=(0, 7, 2999),
                                  long_rows=[(3, 3000), (4, 700), (5, 257), (6, 256)])
    g = torch.Generator().manual_seed(6)
    value = torch.randn(col.numel(), generator=g).to(dtype)
    x = torch.randn(N, K, generator=g).to(dtype)
    parts, _ = split_column_chunks(rowptr.to(DEV), col.to(DEV), value.to(DEV), N, 1, P)   # world = 1: ids unchanged
    partial = torch.empty(M, K, dtype=torch.float32, device=DEV)
    out = torch.empty(M, K, dtype=dtype, device=DEV)
    xd = x.to(DEV)
    for c, (rp, cl, v) in enumerate(parts):
        ops.spmm_fw_acc(rp, cl, v, xd, partial, out, 1 if c == 0 else (3 if c == P - 1 else 2))
    ref, _ = oracle.spmm(rowptr, col, value.float(), x.float(), "sum")
    bound, _ = oracle.spmm(rowptr, col, value.float().abs(), x.float().abs(), "sum")
    tol = 1e-5 if dtype == torch.float32 else 1e-2
    assert ((out.cpu().float() - ref).abs() <= tol * bound + 1e-30).all()
    single, _ = ops.spmm_fw(rowptr.to(DEV), col.to(DEV), value.to(DEV), xd, "sum")
    assert ((out.float() - single.float()).abs().cpu() <= tol * bound + 1e-30).all()


@pytest.mark.parametrize("split", ["feature", "column"])
def test_pipelined_row_sharded_spmm_single_rank(oracle, split):
    """PipelinedRowShardedSpMM on one rank (the gather degenerates to local copies): both splits reproduce the
    plain SpMM; the slice-major fast path round-trips."""
    from pytorch_sparse_b200.parallel import PipelinedRowShardedSpMM
    M = N = 2048
    row, rowptr, col = random_csr(M, N, 9, seed=11, empty_rows=(1,), long_rows=[(2, 600)])
    g = torch.Generator().manual_seed(12)
    value = torch.randn(col.numel(), generator=g).bfloat16()
    x = torch.randn(N, 128, generator=g).bfloat16()
    a = ts.SparseTensor(rowptr=rowptr.to(DEV), col=col.to(DEV), value=value.to(DEV), sparse_sizes=(M, N),
                        is_sorted=True, trust_data=True)
    pipe = PipelinedRowShardedSpMM(a, block=N, chunks=4, split=split)
    y = pipe(x.to(DEV))
    ref, _ = oracle.spmm(rowptr, col, value.float(), x.float(), "sum")
    bound, _ = oracle.spmm(rowptr, col, value.float().abs(), x.float().abs(), "sum")
    assert ((y.cpu().float() - ref).abs() <= 1e-2 * bound + 1e-30).all()
    if split == "feature":
        xs = pipe.to_sliced(x.to(DEV))
        assert torch.equal(pipe.from_sliced(xs).cpu(), x)
        assert torch.equal(pipe.from_sliced(pipe.forward_sliced(xs)), y)


@pytest.mark.parametrize("dtype,K,reduce", [(torch.bfloat16, 128, "sum"), (torch.float32, 256, "max"),
                                            (torch.float32, 32, "sum"), (torch.float16, 64, "mean"),
                                            (torch.bfloat16, 256, "min"), (torch.float32, 128, "sum")])
@pytest.mark.parametrize("has_value", [True, False])
def test_planned_spmm_matches_unplanned_and_oracle(oracle, dtype, K, reduce, has_value):
    """tsb200_spmm_plan + tsb200_spmm_fw_planned (one memset + one kernel: row items, then the plan's segments drained
    by the same warps, multi-segment rows combined by the last finisher) on a power-law matrix with empty rows, rows
    of exactly / just over the segment length and rows of thousands of nnz — against the unplanned call and the oracle."""
    M, N = 5000, 4096
    row, rowptr, col = random_csr(M, N, 14, seed=31, power_law=True, empty_rows=(0, 1, 4999),
                                  long_rows=[(3, 4000), (4, 1025), (5, 257), (6, 256), (40, 600), (41, 600)])
    g = torch.Generator().manual_seed(32)
    value = torch.randn(col.numel(), generator=g).to(dtype) if has_value else None
    x = torch.randn(N, K, generator=g).to(dtype)
    d_rowptr, d_col = rowptr.to(DEV), col.to(DEV)
    d_value = None if value is None else value.to(DEV)
    plan = ops.spmm_plan(d_rowptr, col.numel())
    assert plan.n_seg > 0 and plan.n_long > 0 and plan.n_slot >= 2 * plan.n_long
    out_p, arg_p = ops.spmm_fw(d_rowptr, d_col, d_value, x.to(DEV), reduce, plan=plan)
    out_u, arg_u = ops.spmm_fw(d_rowptr, d_col, d_value, x.to(DEV), reduce)
    ref, ref_arg = oracle.spmm(rowptr, col, value, x, reduce)
    if reduce in ("min", "max"):
        assert torch.equal(out_p, out_u) and torch.equal(arg_p, arg_u)
        assert torch.equal(out_p.cpu(), ref) and torch.equal(arg_p.cpu(), ref_arg)
    else:
        vf = None if value is None else value.float().abs()
        bound, _ = oracle.spmm(rowptr, col, vf, x.float().abs(), "sum")
        if reduce == "mean":
            bound = bound / (rowptr[1:] - rowptr[:-1]).clamp(min=1).view(-1, 1)
        fref, _ = oracle.spmm(rowptr, col, None if value is None else value.float(), x.float(), reduce)
        tol = 1e-5 if dtype == torch.float32 else 1e-2
        assert ((out_p.cpu().float() - fref).abs() <= tol * bound + 1e-30).all()
        assert ((out_p.float() - out_u.float()).abs().cpu() <= tol * bound + 1e-30).all()
    # a matrix without long rows: the plan is empty and the call is a single kernel
    r2, rp2, c2 = random_csr(300, 200, 5, seed=33)
    plan2 = ops.spmm_plan(rp2.to(DEV), c2.numel())
    assert plan2.n_seg == 0 and plan2.n_long == 0
    x2 = torch.randn(200, K, generator=g).to(dtype)
    o2, a2 = ops.spmm_fw(rp2.to(DEV), c2.to(DEV), None, x2.to(DEV), reduce, plan=plan2)
    o3, a3 = ops.spmm_fw(rp2.to(DEV), c2.to(DEV), None, x2.to(DEV), reduce)
    assert torch.equal(o2, o3) and (a2 is None or torch.equal(a2, a3))
