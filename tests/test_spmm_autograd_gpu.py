"""SpMM autograd end to end: `ts.matmul(A, X, reduce)` and the registered `torch.ops.tsb200.spmm_*` operators followed
by `torch.autograd.grad`, on every kernel path of the forward, of the CSC-view product that forms grad_mat and of the
value gradient, against fp64 references from the oracle, with bounds from the kernels' rounding model.

grad_mat of sum / mean is a sum SpMM on the CSC view (colptr, the cached row_csc, value[csr2csc], and for mean the
weights value / count); its reference is an fp64 index_add over the COO entries, which reads none of the storage's CSC
caches. Hub columns give the CSC view rows of 1, 255, 256, 257, 600 and 4100 entries (segments, the multi-segment
combine), a 32-row block over the item budget and empty rows; the dense rows no entry references are NaN.

Bounds (T the storage dtype, u = 2^-24 the unit roundoff of the fp32 accumulators):
  forward sum / mean, grad_value    as test_spmm_kernels_gpu / test_spmm_backward_kernels_gpu bound them
  grad_mat sum    1/2 ulp_T(ref) + (n_c + 1) u S_c, n_c the column's entry count, S_c = (|A^T| |G|)[c, k]
  grad_mat mean   ref = sum_e (v_e / d_r) g over exact quotients; 1/2 ulp_T(ref) + (n_c + 1) u sum|w_e g|
                  + sum_e delta_e |g|, delta_e = 1/2 ulp_T(v_e / d_r) + u |v_e / d_r| (the weight's fp32 quotient and
                  its rounding to T; for T = f32 the second term only)
  min / max       values and arg_out bit for bit with the oracle in T; both gradients against the oracle's fp64
                  backward with that arg, (n + 1) u S + 1/2 ulp_T(ref) (fp32 accumulators rounded once to T)
The grad_mat rows of columns without entries are +0, compared as bit patterns.
"""
import pytest
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import ops
from test_spmm_autograd_cpu import check_weight_expectations, mean_weights, private_column_case
from test_spmm_backward_kernels_gpu import check_accumulated, check_value_bw, sddmm_family
from test_spmm_kernels_gpu import (BLOCK_DEG, DEV, FAMILIES, FLOATS, NAN_ROWS, SPECIAL_DEGREES, U32, Ref, _id,
                                   assert_bits_equal, assert_sum_bound, build_csr, dense, family_of, half_ulp,
                                   plan_budget_rows, sub_csr, values)

pytestmark = pytest.mark.gpu
REDUCES = ("sum", "add", "mean", "min", "max")
HUB_DEGREES = (1, 255, 256, 257, 600, 4100)

# (dtype, K, B): the first (full-width) K of every forward family per dtype and an odd K (generic), each at B = 1 and
# B = 2. grad_mat has the forward's K, so it runs the same families; B = 2 reaches the nnz-parallel value gradients.
GRID = [(dt, ks[0], B) for fam, (k32, k16) in FAMILIES.items() for dt in FLOATS
        for ks in [k32 if dt == torch.float32 else k16] for B in (1, 2)] + \
       [(dt, 7, B) for dt in FLOATS for B in (1, 2)]
assert {family_of(dt, K) for dt, K, _ in GRID} == set(FAMILIES) | {"generic"}
assert {sddmm_family(dt, K, B) for dt, K, B in GRID} == {"row4", "row8", "row16", "row32", "row32ch2", "nnz1", "nnz4",
                                                         "nnz8", "nnz16", "nnz32", "nnz32strided", "generic"}


# ---- matrices ------------------------------------------------------------------------------------------------------
def coo_row(rowptr):
    return torch.repeat_interleave(torch.arange(rowptr.numel() - 1), rowptr[1:] - rowptr[:-1])


def with_hub_columns(rowptr, col, N, counts, seed, keep_rows=()):
    """`col` with entries moved so that column c holds exactly counts[c] entries (0: an empty column); the entries of
    `keep_rows` stay where they are. Row degrees do not change."""
    g = torch.Generator().manual_seed(seed)
    col = col.clone()
    movable = ~torch.isin(coo_row(rowptr), torch.tensor(list(keep_rows), dtype=torch.long))
    reserved = torch.tensor(sorted(counts), dtype=torch.long)
    assert not bool(torch.isin(col[~movable], reserved).any())
    pool = torch.arange(1, N - NAN_ROWS + 1)
    pool = pool[~torch.isin(pool, reserved)]
    clash = movable & torch.isin(col, reserved)
    col[clash] = pool[torch.randint(pool.numel(), (int(clash.sum()),), generator=g)]
    pos = movable.nonzero().view(-1)
    pos = pos[torch.randperm(pos.numel(), generator=g)]
    at = 0
    for c, n in counts.items():
        col[pos[at:at + n]] = c
        at += n
    assert at <= pos.numel()
    return col


def sparse(rowptr, col, value, N):
    M = rowptr.numel() - 1
    return ts.SparseTensor(rowptr=rowptr.to(DEV), col=col.to(DEV), value=value, sparse_sizes=(M, N), is_sorted=True,
                           trust_data=True)


@pytest.fixture(scope="module")
def small():
    """test_spmm_kernels_gpu's structured matrix (empty rows, every SPECIAL_DEGREES row, a 32-row block over the item
    budget, duplicate columns, tie rows) with hub columns of HUB_DEGREES entries, 32 consecutive columns of BLOCK_DEG
    entries and three empty columns among the referenced ones."""
    M, N = 32 * 70 + 13, 4600
    specials = {r: d for r, d in zip([5, 37, 38, 39, 200, 201, 202, 500, 501, 1500], SPECIAL_DEGREES)}
    rowptr, col = build_csr(M, N, 4, 1, specials, blocks=[64], tie_rows={300: 40, 301: 600},
                            empty_rows=(0, M // 2, M - 1))
    counts = dict(zip(range(100, 106), HUB_DEGREES))
    counts.update({c: BLOCK_DEG for c in range(1024, 1056)})
    counts.update({c: 0 for c in (2000, 2001, 3333)})
    col = with_hub_columns(rowptr, col, N, counts, 4, keep_rows=(300, 301))
    colcount = torch.bincount(col, minlength=N)
    for c, n in counts.items():
        assert int(colcount[c]) == n
    return dict(M=M, N=N, rowptr=rowptr, col=col, row=coo_row(rowptr), colcount=colcount)


LARGE_M = 600_017


@pytest.fixture(scope="module")
def large():
    """A square matrix of about 600k rows, so that both the forward and the CSC view run 32-row work items, with rows
    and columns of 256, 257 and 4100 entries and budget blocks in both views. Checked on a sample of whole 32-row
    groups of each view."""
    M = N = LARGE_M
    specials = {4096 * 7 + 5: 4100, 4096 * 11 + 31: 257, 4096 * 13: 256}
    blocks = list(range(2048, M - 32, 4096 * 8))
    rowptr, col = build_csr(M, N, 1, 2, specials, blocks, tie_rows={}, empty_rows=(0, M // 2, M - 1))
    hubs = {4096 * 5 + 7: 4100, 4096 * 9 + 3: 257, 4096 * 15: 256}
    cblocks = [4096 * 3, 4096 * 17]
    counts = dict(hubs)
    for b in cblocks:
        counts.update({c: BLOCK_DEG for c in range(b, b + 32)})
    col = with_hub_columns(rowptr, col, N, counts, 5)
    g = torch.Generator().manual_seed(6)

    def groups(marked, n):
        s = {r & ~31 for r in marked} | {0, (n // 2) & ~31, (n - 1) & ~31}
        s |= set((torch.randint((n - 1) // 32, (24,), generator=g) * 32).tolist())
        return torch.cat([torch.arange(r, min(r + 32, n)) for r in sorted(s)])

    return dict(M=M, N=N, rowptr=rowptr, col=col, row=coo_row(rowptr),
                rows=groups(list(specials) + blocks[:4], M), cols=groups(list(hubs) + cblocks, N))


# ---- references ----------------------------------------------------------------------------------------------------
def csc_sum(col, w, Gr, N):
    """fp64 sum_e w_e Gr[e] into row col_e of an N-row result (w None: ones); Gr [..., E, K] holds each entry's row
    of grad_out."""
    src = Gr if w is None else Gr * w.view(-1, 1)
    return torch.zeros(Gr.shape[:-2] + (N, Gr.size(-1)), dtype=torch.float64).index_add_(-2, col, src)


def assert_rounded(got, ref, S, n, dtype, what):
    """An fp32 accumulation of n terms (fp32 atomics in any order), rounded once to `dtype`."""
    if dtype == torch.float32:
        check_accumulated(got, ref, S, n, U32, what)
    else:
        assert_sum_bound(got, ref, S, n + 1, dtype, what=what)


def check_grad_mat(reduce, gm, row, col, rowptr, v, G, N, colcount, dtype, what):
    """grad_mat of sum / mean against the fp64 index_add over the COO entries (row, col, v): N result rows, colcount
    the entries of each."""
    v64 = None if v is None else v.cpu().double()
    Gr = G.cpu().index_select(-2, row).double()
    Ga = Gr.abs()
    n = colcount.double().view(-1, 1)
    if reduce in ("sum", "add"):
        ref = csc_sum(col, v64, Gr, N)
        S = csc_sum(col, None if v64 is None else v64.abs(), Ga, N)
        assert_sum_bound(gm, ref, S, n + 1, dtype, what=what + " grad_mat")
        return
    d = (rowptr[1:] - rowptr[:-1]).clamp(min=1).double()[row]
    w = (torch.ones_like(d) if v64 is None else v64) / d
    delta = U32 * w.abs()
    if dtype != torch.float32:
        delta = delta + half_ulp(w.abs(), dtype)
    ref = csc_sum(col, w, Gr, N)
    e = (n + 1) * U32 * csc_sum(col, w.abs() + delta, Ga, N) + csc_sum(col, delta, Ga, N)
    assert_sum_bound(gm, ref, e, 1.0, dtype, u=1.0, what=what + " grad_mat")


def minmax_refs(oracle, col, v, X, G, arg):
    """The oracle's fp64 min/max backward with the given arg: (ref, S, n) for (grad_value, grad_mat)."""
    v64 = None if v is None else v.cpu().double()
    X64, G64 = X.cpu().double(), G.cpu().double()
    need_v = v is not None
    ref = oracle.spmm_minmax_bw(col, v64, X64, G64, arg, need_v, True)
    S = oracle.spmm_minmax_bw(col, None if v64 is None else v64.abs(), torch.nan_to_num(X64, nan=0.0).abs(),
                              G64.abs(), arg, need_v, True)
    ones = None if v is None else torch.ones_like(v64)
    n = oracle.spmm_minmax_bw(col, ones, torch.ones_like(X64), torch.ones_like(G64), arg, need_v, True)
    return ref, S, n


def assert_empty_columns_zero(gm, colcount, what):
    empty = (colcount == 0).nonzero().view(-1).to(gm.device)
    z = gm.index_select(-2, empty)
    assert_bits_equal(z, torch.zeros_like(z), what + " grad_mat of empty columns")


def run(a, x, reduce, G, v=None):
    """matmul and backward through torch.autograd.grad -> (out, grad_value or None, grad_mat or None)."""
    out = ts.matmul(a, x, reduce)
    inputs = [t for t in (v, x) if t is not None and t.requires_grad]
    grads = list(torch.autograd.grad(out, inputs, G))
    gv = grads.pop(0) if v is not None and v.requires_grad else None
    gm = grads.pop(0) if x.requires_grad else None
    return out.detach(), gv, gm


def grad_out(shape, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g, dtype=torch.float64).to(dtype)


# ---- 1. every family x dtype x B x reduction x value, end to end ---------------------------------------------------
@pytest.mark.parametrize("has_value", [True, False], ids=["value", "novalue"])
@pytest.mark.parametrize("dtype,K,B", GRID, ids=_id)
def test_autograd_vs_fp64(oracle, small, dtype, K, B, has_value):
    rowptr, col, row, N, M = small["rowptr"], small["col"], small["row"], small["N"], small["M"]
    E = col.numel()
    bshape = () if B == 1 else (B,)
    for quantized, reduces in ((False, ("sum", "add", "mean")), (True, ("min", "max"))):
        X = dense(N, K, dtype, K + B, quantized, B=None if B == 1 else B)
        v = values(E, dtype, K + 1, quantized) if has_value else None
        G = grad_out(bshape + (M, K), dtype, K + 2)
        ref = Ref(oracle, rowptr, col, v, X)
        for reduce in reduces:
            what = f"{family_of(dtype, K)} {dtype} K={K} B={B} value={has_value} {reduce}"
            vd = None if v is None else v.to(DEV).requires_grad_()
            xd = X.to(DEV).requires_grad_()
            a = sparse(rowptr, col, vd, N)
            out, gv, gm = run(a, xd, reduce, G.to(DEV), vd)
            if reduce in ("min", "max"):
                with torch.no_grad():
                    out_op, arg = getattr(torch.ops.tsb200, f"spmm_{reduce}")(*a.csr(), xd)
                assert_bits_equal(out, out_op, what + " matmul vs op")
                ref.check(reduce, out, arg, what)
                (rv, rm), (Sv, Sm), (nv, nm) = minmax_refs(oracle, col, v, X, G, arg.cpu())
                if has_value:
                    assert_rounded(gv, rv, Sv, nv, dtype, what + " grad_value")
                assert_rounded(gm, rm, Sm, nm, dtype, what + " grad_mat")
            else:
                ref.check("sum" if reduce == "add" else reduce, out, None, what)
                if has_value:
                    check_value_bw(oracle, rowptr, col, X, G, "mean" if reduce == "mean" else "sum", gv,
                                   what + " grad_value")
                check_grad_mat(reduce, gm, row, col, rowptr, v, G, N, small["colcount"], dtype, what)
            assert_empty_columns_zero(gm, small["colcount"], what)


# ---- 2. 32-row work items in both views --------------------------------------------------------------------------
def _compact(col_s):
    """Column indices of a sample renumbered over the dense rows it references -> (referenced rows, local indices)."""
    return torch.unique(col_s, return_inverse=True)


@pytest.mark.parametrize("dtype,K", [(torch.float32, 16), (torch.bfloat16, 128), (torch.float16, 64)], ids=_id)
def test_autograd_full_size_items(oracle, large, dtype, K):
    rowptr, col, row, N, M = large["rowptr"], large["col"], large["row"], large["N"], large["M"]
    rows, cols = large["rows"], large["cols"]
    E = col.numel()
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    assert M >= 32 * 16 * 8 * sms and N >= 32 * 16 * 8 * sms
    colcount = torch.bincount(col, minlength=N)
    sp, scol, idx = sub_csr(rowptr, col, rows)                # sampled rows of the CSR view
    uc, scol_l = _compact(scol)
    csel = torch.isin(col, cols).nonzero().view(-1)           # entries of the sampled columns (CSC view)
    cpos = torch.searchsorted(cols, col[csel])
    g = torch.Generator().manual_seed(7)
    for quantized, reduces in ((False, ("sum", "mean")), (True, ("max",))):
        if quantized:
            X = (torch.randint(-4, 5, (N, K), generator=g) * 0.5).to(dtype)
        else:
            X = torch.randn(N, K, generator=g).to(dtype)
        X[torch.cat([torch.tensor([0]), torch.arange(N - NAN_ROWS + 1, N)])] = float("nan")
        v = values(E, dtype, 8, quantized)
        G = torch.randn(M, K, generator=g).to(dtype)
        Gs = G[rows]
        for reduce in reduces:
            what = f"{dtype} K={K} M=N={M} {reduce}"
            vd, xd = v.to(DEV).requires_grad_(), X.to(DEV).requires_grad_()
            a = sparse(rowptr, col, vd, N)
            out, gv, gm = run(a, xd, reduce, G.to(DEV), vd)
            rows_d = rows.to(DEV)
            gv_s, gm_s = gv[idx.to(DEV)], gm[cols.to(DEV)]
            if reduce == "max":
                with torch.no_grad():
                    _, arg = torch.ops.tsb200.spmm_max(*a.csr(), xd)
                arg = arg.cpu()
                ref, rarg = oracle.spmm(sp, scol_l, v[idx], X[uc], "max")
                assert_bits_equal(out[rows_d], ref, what + " out")
                glob = torch.where(rarg < idx.numel(), idx[rarg.clamp(max=idx.numel() - 1)], E)
                assert torch.equal(arg[rows], glob), what + ": arg_out differs"
                (rv, _), (Sv, _), (nv, _) = minmax_refs(oracle, scol_l, v[idx], X[uc], Gs, rarg)
                assert_rounded(gv_s, rv, Sv, nv, dtype, what + " grad_value")
                # grad_mat[c, k] = sum over the column's entries e won by arg[row_e, k] of v_e G[row_e, k]
                r_e = row[csel]
                won = (arg[r_e] == csel.view(-1, 1)).double()
                terms = won * v[csel].double().view(-1, 1) * G[r_e].double()
                rm = torch.zeros(cols.numel(), K, dtype=torch.float64).index_add_(0, cpos, terms)
                Sm = torch.zeros_like(rm).index_add_(0, cpos, terms.abs())
                nm = torch.zeros_like(rm).index_add_(0, cpos, won)
                assert_rounded(gm_s, rm, Sm, nm, dtype, what + " grad_mat")
            else:
                Ref(oracle, sp, scol_l, v[idx], X[uc]).check(reduce, out[rows_d], None, what)
                check_value_bw(oracle, sp, scol_l, X[uc], Gs, reduce, gv_s, what + " grad_value")
                check_grad_mat(reduce, gm_s, row[csel], cpos, rowptr, v[csel], G, cols.numel(), colcount[cols],
                               dtype, what)
            assert not bool(gm.isnan().any()), what + ": grad_mat has a NaN"
            assert_empty_columns_zero(gm, colcount, what)


# ---- 3. which gradients, value dtype, reference-schema operators --------------------------------------------------
@pytest.mark.parametrize("reduce", REDUCES)
def test_value_only_mat_only_both(oracle, small, reduce):
    """Each gradient alone equals, bit for bit, the same gradient taken together with the other (f16, K = 128: rows of
    256 bytes, where a planned and an unplanned product give the same bits; quantized operands, so the min/max
    atomics' order changes nothing). A value-only backward builds no CSC view."""
    rowptr, col, N, M = small["rowptr"], small["col"], small["N"], small["M"]
    dtype, K = torch.float16, 128
    X = dense(N, K, dtype, 11, True)
    v = values(col.numel(), dtype, 12, True)
    G = (torch.randint(-8, 9, (M, K), generator=torch.Generator().manual_seed(13)) * 0.25).to(dtype).to(DEV)
    res = {}
    for need_v, need_x in ((True, True), (True, False), (False, True)):
        vd = v.to(DEV).requires_grad_(need_v)
        xd = X.to(DEV).requires_grad_(need_x)
        a = sparse(rowptr, col, vd, N)
        res[need_v, need_x] = run(a, xd, reduce, G, vd)
        if not need_x:
            keys = a.storage.cached_keys()
            assert "csr2csc" not in keys and "colptr" not in keys, keys
    both = res[True, True]
    assert_bits_equal(res[True, False][0], both[0], f"{reduce} out")
    assert_bits_equal(res[True, False][1], both[1], f"{reduce} value only")
    assert_bits_equal(res[False, True][2], both[2], f"{reduce} mat only")
    assert res[True, False][2] is None and res[False, True][1] is None


@pytest.mark.parametrize("reduce", REDUCES)
def test_value_dtype_differs_from_mat(oracle, small, reduce):
    """f32 values with a bf16 dense operand: matmul casts the values to bf16, and the value gradient comes back through
    the cast as f32, equal to the bf16 value gradient of the same product (quantized operands, so the min/max
    atomics' order changes nothing)."""
    rowptr, col, N, M = small["rowptr"], small["col"], small["N"], small["M"]
    K = 64
    X = dense(N, K, torch.bfloat16, 21, True).to(DEV)
    v32 = values(col.numel(), torch.float32, 22, True).to(DEV)
    G = (torch.randint(-8, 9, (M, K), generator=torch.Generator().manual_seed(23)) * 0.25).to(torch.bfloat16).to(DEV)
    outs = []
    for v in (v32.clone().requires_grad_(), v32.to(torch.bfloat16).requires_grad_()):
        ops._PLAN_CACHE.clear()
        outs.append(run(sparse(rowptr, col, v, N), X.clone().requires_grad_(), reduce, G, v))
    (o32, g32, m32), (o16, g16, m16) = outs
    assert g32.dtype == torch.float32 and g16.dtype == torch.bfloat16
    assert_bits_equal(o32, o16, f"{reduce} out")
    assert_bits_equal(g32, g16.float(), f"{reduce} grad_value through the cast")
    assert_bits_equal(m32, m16, f"{reduce} grad_mat")


@pytest.mark.parametrize("reduce", ["sum", "mean"])
@pytest.mark.parametrize("dtype,K", [(torch.float32, 12), (torch.bfloat16, 40), (torch.float16, 256)], ids=_id)
def test_reference_schema_ops_match_matmul(small, dtype, K, reduce):
    """torch.ops.tsb200.spmm_sum / spmm_mean without row_csc (gathered in the backward) give the gradients of the
    matmul path that passes the storage's cached row_csc, bit for bit."""
    rowptr, col, N, M = small["rowptr"], small["col"], small["N"], small["M"]
    X = dense(N, K, dtype, 31, False).to(DEV)
    v = values(col.numel(), dtype, 32, False).to(DEV)
    G = grad_out((M, K), dtype, 33).to(DEV)
    vd, xd = v.clone().requires_grad_(), X.clone().requires_grad_()
    a = sparse(rowptr, col, vd, N)
    ops._PLAN_CACHE.clear()
    want = run(a, xd, reduce, G, vd)
    st = a.storage
    rp, cl, _ = a.csr()
    ops._PLAN_CACHE.clear()
    if reduce == "sum":
        out = torch.ops.tsb200.spmm_sum(st.row(), rp, cl, vd, st.colptr(), st.csr2csc(), xd)
    else:
        out = torch.ops.tsb200.spmm_mean(st.row(), rp, cl, vd, st.rowcount(), st.colptr(), st.csr2csc(), xd)
    got = (out.detach(),) + torch.autograd.grad(out, (vd, xd), G)
    for t0, t1, name in zip(want, got, ("out", "grad_value", "grad_mat")):
        assert_bits_equal(t1, t0, f"{dtype} K={K} {reduce} {name}")


# ---- 4. the planned backward ---------------------------------------------------------------------------------------
def _has_plan(t):
    key = t.untyped_storage()._cdata
    return any(k[0] == key and ent[1] is not None for k, ent in ops._PLAN_CACHE.items())


@pytest.mark.parametrize("reduce", ["sum", "mean"])
@pytest.mark.parametrize("dtype,K", [(torch.float16, 128), (torch.float32, 64), (torch.bfloat16, 32),
                                     (torch.float32, 8)], ids=_id)
def test_planned_backward(oracle, small, dtype, K, reduce):
    """matmul and backward twice on one SparseTensor: the second forward uses the plan of rowptr and the second
    grad_mat the plan of colptr. Rows wider than 128 bytes: outputs and both gradients bit-identical. Narrower rows:
    bit-identical outside the rows a plan defers for the item budget (which the unplanned call's smaller items keep,
    DESIGN §3.1), and both calls within the bound."""
    rowptr, col, row, N, M = small["rowptr"], small["col"], small["row"], small["N"], small["M"]
    X = dense(N, K, dtype, 41, False)
    v = values(col.numel(), dtype, 42, False)
    G = grad_out((M, K), dtype, 43)
    vd, xd = v.to(DEV).requires_grad_(), X.to(DEV).requires_grad_()
    a = sparse(rowptr, col, vd, N)
    ops._PLAN_CACHE.clear()
    res = [run(a, xd, reduce, G.to(DEV), vd) for _ in range(2)]
    rp, colptr = a.storage.rowptr(), a.storage.colptr()
    assert _has_plan(rp) and _has_plan(colptr), "the second call did not use a plan for both rowptr and colptr"
    what = f"{dtype} K={K} {reduce}"
    if K * X.element_size() > 128:
        for t0, t1, name in zip(res[0], res[1], ("out", "grad_value", "grad_mat")):
            assert_bits_equal(t1, t0, f"{what} planned vs unplanned {name}")
        return
    keep_r = ~plan_budget_rows(rowptr)
    keep_c = ~plan_budget_rows(colptr.cpu())
    assert not bool(keep_c.all())
    assert_bits_equal(res[1][0][keep_r.to(DEV)], res[0][0][keep_r.to(DEV)], what + " planned vs unplanned out")
    assert_bits_equal(res[1][1], res[0][1], what + " planned vs unplanned grad_value")
    assert_bits_equal(res[1][2][keep_c.to(DEV)], res[0][2][keep_c.to(DEV)], what + " planned vs unplanned grad_mat")
    ref = Ref(oracle, rowptr, col, v, X)
    for out, gv, gm in res:
        ref.check(reduce, out, None, what)
        check_value_bw(oracle, rowptr, col, X, G, reduce, gv, what + " grad_value")
        check_grad_mat(reduce, gm, row, col, rowptr, v, G, N, small["colcount"], dtype, what)


# ---- 5. gradcheck in fp64 -------------------------------------------------------------------------------------------
def gradcheck_case(reduce, seed=51):
    """7 rows of degrees 300, 0, 5, 400, 1, 9, 17 over 512 columns; column 7 holds at least 280 entries of rows 0 and 3.
    For min / max: distinct values and entries, every row's extremes ahead of the runner-up by more than 1e-4."""
    g = torch.Generator().manual_seed(seed)
    M, N, K = 7, 512, 3
    deg = torch.tensor([300, 0, 5, 400, 1, 9, 17])
    rowptr = torch.zeros(M + 1, dtype=torch.long)
    rowptr[1:] = deg.cumsum(0)
    col = torch.cat([torch.randperm(N, generator=g)[:int(d)] for d in deg])
    E = int(rowptr[-1])
    assert col.numel() == E
    col[0:150] = 7
    col[int(rowptr[3]):int(rowptr[3]) + 130] = 7
    if reduce in ("min", "max"):
        v = 1 + torch.randperm(E, generator=g).double() / E
        x = (torch.randperm(N * K, generator=g).double() + 1).view(N, K) / (N * K)
        x = x * torch.where(torch.rand(N, K, generator=g) < 0.5, -1.0, 1.0).double()
        p = v.view(-1, 1) * x[col]
        for r in range(M):
            s = p[int(rowptr[r]):int(rowptr[r + 1])].sort(dim=0).values
            if s.size(0) > 1:
                assert bool((s[1] - s[0]).min() > 1e-4) and bool((s[-1] - s[-2]).min() > 1e-4), (seed, r)
    else:
        v = torch.randn(E, generator=g, dtype=torch.float64)
        x = torch.randn(N, K, generator=g, dtype=torch.float64)
    return rowptr, col, v, x


@pytest.mark.parametrize("reduce", ["sum", "mean", "min", "max"])
def test_gradcheck_fp64(reduce):
    """fp64 (the generic kernel) on rows longer than 256 entries and a hub column: checks the algebra of the four
    backward compositions, not the fast paths."""
    rowptr, col, v, x = gradcheck_case(reduce)
    M, N = rowptr.numel() - 1, x.size(0)
    assert int(torch.bincount(col, minlength=N)[7]) >= 280
    vd, xd = v.to(DEV).requires_grad_(), x.to(DEV).requires_grad_()
    rp, cl = rowptr.to(DEV), col.to(DEV)

    def f(val, mat):
        return ts.matmul(ts.SparseTensor(rowptr=rp, col=cl, value=val, sparse_sizes=(M, N), is_sorted=True,
                                         trust_data=True), mat, reduce)
    assert torch.autograd.gradcheck(f, (vd, xd), nondet_tol=1e-12)


# ---- 6. mean weights bit for bit -------------------------------------------------------------------------------------
@pytest.mark.parametrize("has_value", [True, False], ids=["value", "novalue"])
@pytest.mark.parametrize("kind", ["gpr", "vec"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32, torch.float64], ids=_id)
def test_mean_weights_bit_for_bit(oracle, dtype, kind, has_value):
    """Rows of degree 1 ... 4100 on private columns, grad_out = 1: grad_mat[c] is the weight of column c's one entry,
    value / count formed in fp32 (fp64) and rounded once (see test_spmm_autograd_cpu). The value gradient of the same
    call divides by the same count: within its bound of the fp64 quotient."""
    K = {"gpr": 32, "vec": 256}[kind] // torch.empty(0, dtype=dtype).element_size()
    rowptr, col, value = private_column_case(dtype, has_value)
    M, E = rowptr.numel() - 1, col.numel()
    new, old, rep = mean_weights(rowptr, col, value, dtype)
    check_weight_expectations(new, old, rep, dtype, has_value)
    X = grad_out((E, K), dtype, 61)
    vd = None if value is None else value.to(DEV).requires_grad_()
    a = sparse(rowptr, col, vd, E)
    G = torch.ones(M, K, dtype=dtype, device=DEV)
    _, gv, gm = run(a, X.to(DEV).requires_grad_(), "mean", G, vd)
    assert_bits_equal(gm, (new + 0.0).view(-1, 1).expand(E, K), f"{dtype} K={K} value={has_value} weights")
    if has_value:
        check_value_bw(oracle, rowptr, col, X, G.cpu(), "mean", gv, f"{dtype} K={K} grad_value")
