"""Sparse softmax (`softmax(src, dim)`, `ops.segment_softmax`, tsb200_segment_softmax / _bw) on the GPU.

The structured matrix has empty rows and rows of 1, 2, 31, 32, 33, 127, 128, 129, 255, 256, 257, 4100 and 60 000
entries: both sides of the short (<= 32 entries: 8 lanes per segment), medium (<= 128: a warp) and long (a CTA,
three passes) paths of the one kernel. Its transpose gives the same column lengths for dim = 0.

Forward bound against fp64 `torch.softmax` of each segment, first order, per entry j of a segment of n entries with
R = min(max_k |v_k - m|, 104) (beyond 104 every fp32 exp is 0, and those entries are covered by the floor):
  fl(v_j - m) adds at most R u to the exponent, so e_j is off by a factor of (1 + (R + 4) u): R u from the
  subtraction, 4 u from expf's 2 ulp; S = sum e_k then by (R + 4 + (n - 1)) u; the division adds u. So
      |out_j - ref_j| <= ref_j (2R + n + 8) u + 1/2 ulp_T(ref_j) + floor,   u = 2^-24
  and for fp64 (exp's 1 ulp = 2 u, no final rounding) ref_j (2R + n + 6) 2^-53 + floor. The floor covers results in
  the subnormal range: half the smallest subnormal of T plus one of fp32 (an e_j that is subnormal in fp32).
Backward bound against alpha_j (g_j - sum_k alpha_k g_k) in fp64 over the stored alpha: the FMA dot of n terms (no term
rounded more than n times) is off by n u sum_k alpha_k |g_k|, and g_j - dot and the product each round once, relative
to at most |g_j| + sum_k alpha_k |g_k|, so
      |grad_j - ref_j| <= alpha_j ((n + 2) sum_k alpha_k |g_k| + 2 |g_j|) u + 1/2 ulp_T(ref_j) + floor.
For fp64 the reference's own dot rounds as often as the kernel's, so the backward bound takes u = 2 * 2^-53.
"""
import ctypes
import subprocess
import sys
from pathlib import Path

import pytest
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import SparseTensor, ops
from pytorch_sparse_b200._lib import lib
from util import launched_kernels

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF, F16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
DTYPES = (BF, F16, F32, F64)
CODE = {F32: 0, F64: 1, F16: 2, BF: 3}
LENGTHS = [0, 1, 2, 0, 31, 32, 33, 127, 128, 129, 255, 256, 257, 4100, 60000, 0, 3, 17]
DS = (1, 2, 3, 4, 8, 16, 64)
_STORE = {BF: (8, -133), F16: (11, -24), F32: (24, -149), F64: (53, -1074)}   # precision, exponent of min subnormal


def structured(lengths=LENGTHS, seed=0):
    """Rows of the given lengths over N = max + 7 columns, sorted random columns per row."""
    g = torch.Generator().manual_seed(seed)
    N = max(lengths) + 7
    rows, cols = [], []
    for r, n in enumerate(lengths):
        rows.append(torch.full((n,), r, dtype=torch.long))
        cols.append(torch.randperm(N, generator=g)[:n].sort().values)
    return SparseTensor(row=torch.cat(rows).to(DEV), col=torch.cat(cols).to(DEV), sparse_sizes=(len(lengths), N))


def segments(ptr, perm, E):
    """(segment id, position in `value`) of every entry, in segment order."""
    ptr = ptr.cpu()
    seg = torch.repeat_interleave(torch.arange(ptr.numel() - 1), ptr[1:] - ptr[:-1])
    pos = torch.arange(E) if perm is None else perm.cpu()
    return seg, pos


def ref_softmax(ptr, value, perm=None):
    """fp64 softmax per segment and column, in `value`'s order; also n and R (see the module docstring)."""
    v = value.detach().cpu().double().reshape(value.size(0), -1)
    E, D = v.shape
    seg, pos = segments(ptr, perm, E)
    S = ptr.numel() - 1
    x = v[pos]
    idx = seg[:, None].expand(-1, D)
    m = torch.full((S, D), -float("inf"), dtype=F64).scatter_reduce(0, idx, x, "amax")
    lo = torch.full((S, D), float("inf"), dtype=F64).scatter_reduce(0, idx, x, "amin")
    e = torch.exp(x - m[seg])
    tot = torch.zeros(S, D, dtype=F64).index_add_(0, seg, e)
    out = torch.empty_like(v)
    out[pos] = e / tot[seg]
    n = torch.empty(E, 1, dtype=F64)
    n[pos] = (ptr[1:] - ptr[:-1]).cpu().double()[seg][:, None]
    R = torch.empty_like(v)
    R[pos] = (m - lo).clamp(max=104.0)[seg]
    return out, n, R


def ulp_half(x, dtype):
    p, emin = _STORE[dtype]
    e = torch.floor(torch.log2(x.abs().clamp(min=2.0 ** -1074)))
    return torch.where(x == 0, torch.zeros_like(x), 2.0 ** (e - p)).clamp(min=2.0 ** (emin - 1))


def floor_of(dtype):
    return 2.0 ** (_STORE[dtype][1] - 1) + (2.0 ** -149 if dtype != F64 else 0.0)


def assert_forward(out, ptr, value, perm=None, what=""):
    ref, n, R = ref_softmax(ptr, value, perm)
    o = out.detach().cpu().double().reshape(ref.shape)
    if value.dtype == F64:
        bound = ref * (2 * R + n + 6) * 2.0 ** -53 + floor_of(F64)
    else:
        bound = ref * (2 * R + n + 8) * 2.0 ** -24 + ulp_half(torch.maximum(ref, o), value.dtype) + floor_of(value.dtype)
    err = (o - ref).abs()
    bad = ~(err <= bound)
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())} of {o.numel()} out of bound, first {bad.nonzero()[0]}: "
                                 f"{o[bad][0].item()!r} vs {ref[bad][0].item()!r}")
    # each segment sums to 1 within n times the bound
    seg, pos = segments(ptr, perm, o.size(0))
    D = o.size(1)
    tot = torch.zeros(ptr.numel() - 1, D, dtype=F64).index_add_(0, seg, o[pos])
    bsum = torch.zeros_like(tot).index_add_(0, seg, (bound * n)[pos])
    has = (ptr[1:] - ptr[:-1]).cpu() > 0
    assert bool(((tot - 1).abs() <= bsum)[has].all()), what


def assert_backward(grad, ptr, alpha, g, perm=None, what=""):
    a = alpha.detach().cpu().double().reshape(alpha.size(0), -1)
    gg = g.detach().cpu().double().reshape(a.shape)
    E, D = a.shape
    seg, pos = segments(ptr, perm, E)
    S = ptr.numel() - 1
    dot = torch.zeros(S, D, dtype=F64).index_add_(0, seg, (a * gg)[pos])
    mag = torch.zeros(S, D, dtype=F64).index_add_(0, seg, (a * gg.abs())[pos])
    n = (ptr[1:] - ptr[:-1]).cpu().double()[:, None]
    ref, bound = torch.empty_like(a), torch.empty_like(a)
    ref[pos] = a[pos] * (gg[pos] - dot[seg])
    bound[pos] = a[pos] * ((n[seg] + 2) * mag[seg] + 2 * gg[pos].abs())
    o = grad.detach().cpu().double().reshape(a.shape)
    if alpha.dtype == F64:
        bound = bound * 2.0 ** -52 + floor_of(F64)
    else:
        bound = bound * 2.0 ** -24 + ulp_half(torch.maximum(ref.abs(), o.abs()), alpha.dtype) + floor_of(alpha.dtype)
    bad = ~((o - ref).abs() <= bound)
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {o.numel()} out of bound"


def bits(t):
    return t.detach().contiguous().view(torch.uint8)


def scores(E, D, dtype, seed=1, scale=4.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(E, D, generator=g, dtype=F64) * scale).to(dtype).to(DEV)


def c_call(ptr, value, perm, out):
    E = value.size(0)
    return lib.tsb200_segment_softmax(ctypes.c_void_p(ptr.data_ptr()),
                                      None if perm is None else ctypes.c_void_p(perm.data_ptr()),
                                      ctypes.c_void_p(value.data_ptr()), ctypes.c_void_p(out.data_ptr()),
                                      ptr.numel() - 1, E, value.numel() // E, CODE[value.dtype],
                                      ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))


@pytest.fixture(scope="module")
def mats():
    a = structured()
    return {"rows": a, "cols": a.t()}


@pytest.mark.parametrize("dim", [1, 0])
@pytest.mark.parametrize("D", DS)
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda t: str(t).split(".")[-1])
def test_forward_backward_bounds(mats, dtype, D, dim):
    for name, src in mats.items():
        st = src.storage
        ptr, perm = (st.rowptr(), None) if dim == 1 else (st.colptr(), st.csr2csc())
        v = scores(src.nnz(), D, dtype, seed=D)
        out = torch.full_like(v, float("nan"))
        assert c_call(ptr, v, perm, out) == 0
        torch.cuda.synchronize()
        assert not bool(out.isnan().any()), "an entry was not written"
        assert_forward(out, ptr, v, perm, f"{name} dim={dim} D={D}")
        vv = v.clone().requires_grad_()
        res = ts.softmax(src.set_value(vv, layout="csr"), dim).storage.value()
        assert torch.equal(bits(res), bits(out)), "C-ABI and public API differ"
        g = scores(src.nnz(), D, dtype, seed=100 + D, scale=1.0)
        (grad,) = torch.autograd.grad(res, vv, g)
        assert_backward(grad, ptr, res, g, perm, f"{name} dim={dim} D={D}")


def _isolated(body, timeout=900):
    """Runs `body()` of this module in a fresh interpreter. The profiler (CUPTI), CUDA-graph and near-full-memory state
    these tests create belongs to the whole process; left in the pytest process, later profiler sessions of other test
    files recorded no kernels at all."""
    here = Path(__file__).resolve().parent
    code = (f"import sys; sys.path[:0] = [{str(here.parent)!r}, {str(here)!r}]; "
            f"import test_softmax_gpu as t; t.{body}()")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", code], capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, f"{body} failed:\n{r.stdout[-4000:]}\n{r.stderr[-4000:]}"


def test_kernel_instantiations():
    """The vector width and form follow D and the operands' alignment; the length paths live in the same kernel."""
    _isolated("_kernel_instantiations")


def _kernel_instantiations():
    src = structured()
    E = src.nnz()
    base = scores(E * 8 + 2, 1, BF).view(-1)
    aligned = base[: E * 8].view(E, 8)
    shifted = base[2: E * 8 + 2].view(E, 8)        # 4 bytes off a 16-byte boundary
    cases = [(aligned, r"SoftmaxFw<__nv_bfloat16, 8, true>"), (shifted, r"SoftmaxFw<__nv_bfloat16, 8, false>"),
             (scores(E, 3, BF), r"SoftmaxFw<__nv_bfloat16, 1, false>"),
             (scores(E, 2, F32), r"SoftmaxFw<float, 2, true>"), (scores(E, 4, F64), r"SoftmaxFw<double, 2, true>")]
    ptr = src.storage.rowptr()
    for v, pat in cases:
        names = launched_kernels(lambda: ops.segment_softmax(ptr, v), pat)
        assert any(pat in n for n in names), (pat, names)
    # the scalar form computes the bits of the vector form, forward and backward
    g = scores(E, 8, BF, seed=5)
    out_a, out_s = ops.segment_softmax(ptr, shifted.clone()), ops.segment_softmax(ptr, shifted)
    assert torch.equal(bits(out_a), bits(out_s))
    gs = base[1: E * 8 + 1].view(E, 8)             # 2 bytes off
    names = launched_kernels(lambda: ops.segment_softmax_bw(ptr, out_s, gs, None), r"SoftmaxBw<__nv_bfloat16, 8, false>")
    assert any("SoftmaxBw<__nv_bfloat16, 8, false>" in n for n in names)
    assert torch.equal(bits(ops.segment_softmax_bw(ptr, out_a, gs.clone(), None)),
                       bits(ops.segment_softmax_bw(ptr, out_s, gs, None)))


def test_special_values_bit_for_bit():
    lengths = [1, 1, 3, 5, 40, 200, 2, 4, 3, 3, 2, 300]
    src = structured(lengths, seed=3)
    E = src.nnz()
    ptr = src.storage.rowptr().cpu()
    for dtype in DTYPES:
        v = torch.randn(E, 2, dtype=F64, generator=torch.Generator().manual_seed(2))
        s = lambda r: slice(int(ptr[r]), int(ptr[r + 1]))   # noqa: E731
        v[s(2)] = 0.75                         # constant, n = 3
        v[s(3)] = -2.5                         # constant, n = 5
        v[s(4)] = 1.0                          # constant, n = 40 (short/medium boundary region)
        v[s(5)] = 0.5                          # constant, n = 200 (the CTA path)
        v[s(6)][0] = float("nan")              # NaN
        v[s(7)][1] = float("inf")              # +inf
        v[s(8)] = -float("inf")                # all -inf
        v[s(9)][0] = -float("inf")             # -inf next to finite entries
        v[s(11)][7] = float("nan")             # NaN on the CTA path
        out = ts.softmax(src.set_value(v.to(dtype).to(DEV), layout="csr"), 1).storage.value().cpu()
        one = torch.ones(1, dtype=dtype)
        assert torch.equal(out[s(0)], one.expand(1, 2)) and torch.equal(out[s(1)], one.expand(1, 2))
        for r, n in ((2, 3), (3, 5), (4, 40), (5, 200)):
            want = torch.tensor(1.0 / n, dtype=F32 if dtype != F64 else F64).to(dtype)
            assert torch.equal(out[s(r)], want.expand(n, 2)), (dtype, n)
        for r in (6, 7, 8, 11):
            assert bool(out[s(r)].isnan().all()), (dtype, r)
        z = out[s(9)][0]
        assert bool((z == 0).all()) and not bool(torch.signbit(z).any())
        assert not bool(out[s(9)][1:].isnan().any())
    # +-3e38 in f32 does not overflow
    v = torch.zeros(E, 1, dtype=F32)
    v[s(3)] = torch.tensor([3e38, -3e38, 3e38, -3e38, 0.0])[:, None]
    out = ts.softmax(src.set_value(v.to(DEV), layout="csr"), 1).storage.value().cpu()
    assert out[s(3)].view(-1).tolist() == [0.5, 0.0, 0.5, 0.0, 0.0]


def test_one_entry_gradient_is_positive_zero():
    src = structured([1, 1, 4, 1], seed=4)
    for dtype in DTYPES:
        v = scores(src.nnz(), 3, dtype).requires_grad_()
        a = ts.softmax(src.set_value(v, layout="csr"), 1).storage.value()
        (gr,) = torch.autograd.grad(a, v, scores(src.nnz(), 3, dtype, seed=9))
        ones = torch.tensor([0, 1, 6]).to(DEV)
        z = gr[ones]
        assert bool((z == 0).all()) and not bool(torch.signbit(z).any())


@pytest.mark.parametrize("dim", [0, 1])
def test_gradcheck_fp64(dim):
    src = structured([0, 1, 3, 7, 2, 40, 5], seed=5)
    v = scores(src.nnz(), 2, F64, scale=1.0).requires_grad_()
    assert torch.autograd.gradcheck(lambda x: ts.softmax(src.set_value(x, layout="csr"), dim).storage.value(), (v,))


def test_double_backward_raises():
    src = structured([3, 5], seed=6)
    v = scores(src.nnz(), 1, F64).requires_grad_()
    a = ts.softmax(src.set_value(v, layout="csr"), 1).storage.value()
    (gr,) = torch.autograd.grad(a, v, torch.ones_like(a), create_graph=True)
    with pytest.raises(RuntimeError):
        torch.autograd.grad(gr.sum(), v)


def test_row_softmax_builds_no_csc_view():
    src = structured([3, 0, 50, 300], seed=7)
    v = scores(src.nnz(), 4, F32).requires_grad_()
    adj = src.set_value(v, layout="csr")
    att = adj.softmax(dim=1)
    att.storage.value().sum().backward()
    for st in (adj.storage, att.storage):
        assert st._csr2csc is None and st._colptr is None
    assert v.grad is not None


def test_properties_bit_for_bit(mats):
    src = mats["rows"]
    E = src.nnz()
    for dtype in (BF, F32):
        v = scores(E, 6, dtype)
        a = src.set_value(v, layout="csr")
        by_col = ts.softmax(a, 0).storage.value()
        t = a.t()     # its CSR order is a's CSC order
        by_row_t = ts.softmax(t, 1).storage.value()
        perm = a.storage.csr2csc()
        assert torch.equal(bits(by_col[perm]), bits(by_row_t))
        # a row depends only on itself
        full = ts.softmax(a, 1)
        rows = torch.tensor([13, 5, 14, 1, 6]).to(DEV)
        sub = ts.softmax(a.index_select(0, rows), 1)
        rp, sp = full.storage.rowptr().cpu(), sub.storage.rowptr().cpu()
        fv, sv = full.storage.value().cpu(), sub.storage.value().cpu()
        for i, r in enumerate(rows.tolist()):
            assert torch.equal(bits(fv[rp[r]:rp[r + 1]]), bits(sv[sp[i]:sp[i + 1]]))
        # trailing dimensions are flattened
        v3 = ts.softmax(src.set_value(v.view(E, 2, 3), layout="csr"), 1).storage.value()
        assert v3.shape == (E, 2, 3) and torch.equal(bits(v3.reshape(E, 6)), bits(full.storage.value()))
        # two calls give the same bits
        again = ts.softmax(a, 1).storage.value()
        assert torch.equal(bits(again), bits(full.storage.value()))


def test_cuda_graph_replay():
    _isolated("_cuda_graph_replay")


def _cuda_graph_replay():
    src = structured()
    st = src.storage
    ptr = st.rowptr()
    E = src.nnz()
    v = scores(E, 8, BF)
    g = scores(E, 8, BF, seed=3)
    ref = ops.segment_softmax(ptr, v)
    ref_g = ops.segment_softmax_bw(ptr, ref, g, None)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.segment_softmax(ptr, v)     # warm-up off the default stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ops.segment_softmax(ptr, v)
        gin = ops.segment_softmax_bw(ptr, out, g, None)
    out.zero_()
    gin.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(bits(out), bits(ref)) and torch.equal(bits(gin), bits(ref_g))


def random_src(M, N, deg, seed):
    g = torch.Generator().manual_seed(seed)
    E = M * deg
    row = torch.randint(0, M, (E,), generator=g)
    col = torch.randint(0, N, (E,), generator=g)
    col[: E // 3] = torch.randint(0, 4, (E // 3,), generator=g)    # hub columns and duplicate entries
    return SparseTensor(row=row.to(DEV), col=col.to(DEV), sparse_sizes=(M, N))


@pytest.mark.parametrize("dtype", [F32, BF])
def test_readme_attention_layer(dtype):
    M, H, D = 200, 4, 16
    adj = random_src(M, M, 5, 11)
    g = torch.Generator().manual_seed(6)
    q0, k0, v0 = (torch.randn(M, H, D, generator=g, dtype=F64) for _ in range(3))
    q, k, v = (t.to(dtype).to(DEV).requires_grad_() for t in (q0, k0, v0))
    go = torch.randn(M, H, D, generator=g, dtype=F64).to(DEV)

    s = adj.sddmm_heads(q, k) * D ** -0.5                       # [E, H]
    att = adj.set_value(s, layout="csr").softmax(dim=1)         # row softmax per head
    out = att.spmm_heads(v)                                     # [M, H, D]
    grads = torch.autograd.grad(out, (q, k, v), go.to(dtype))

    # dense masked multi-head attention in fp64; duplicate entries count once per stored entry
    qr, kr, vr = (t.detach().double().requires_grad_() for t in (q, k, v))
    r, c, _ = adj.coo()
    cnt = torch.zeros(M, M, dtype=F64, device=DEV).index_put_((r, c), torch.ones_like(r, dtype=F64), accumulate=True)
    logits = torch.einsum("mhd,nhd->hmn", qr, kr) * D ** -0.5 + cnt.log()
    has = cnt.sum(1) > 0
    ref = torch.einsum("hmn,nhd->mhd", torch.softmax(logits[:, has], dim=-1), vr)
    ref.backward(go[has])
    tol = 2e-2 if dtype == BF else 1e-4
    torch.testing.assert_close(out[has].double(), ref, atol=tol, rtol=tol)
    for t, tr in zip(grads, (qr, kr, vr)):
        torch.testing.assert_close(t.double(), tr.grad, atol=5 * tol, rtol=5 * tol)

    # the composed recipe this replaces
    q2, k2, v2 = (t.detach().clone().requires_grad_() for t in (q, k, v))
    row = adj.storage.row()
    s2 = adj.sddmm_heads(q2, k2) * D ** -0.5
    m = adj.set_value(s2.detach(), layout="csr").max(dim=1)
    p = (s2 - m[row]).exp()
    alpha = p / adj.set_value(p, layout="csr").sum(dim=1)[row]
    out2 = adj.set_value(alpha, layout="csr").spmm_heads(v2)
    grads2 = torch.autograd.grad(out2, (q2, k2, v2), go.to(dtype))
    torch.testing.assert_close(out.double(), out2.double(), atol=tol, rtol=tol)
    for a, b in zip(grads, grads2):
        torch.testing.assert_close(a.double(), b.double(), atol=5 * tol, rtol=5 * tol)


def test_script_reaches_the_kernel():
    src = structured([3, 0, 40], seed=8)
    v = scores(src.nnz(), 2, F32)
    fn = torch.jit.script(ts.softmax)
    a = fn(src.set_value(v, layout="csr"), 1).storage.value()
    assert torch.equal(a, ts.softmax(src.set_value(v, layout="csr"), 1).storage.value())


def test_peak_allocation():
    src = structured([16] * 4000 + [3000], seed=9)
    E, D = src.nnz(), 8
    st = src.storage
    ptr, perm = st.rowptr(), st.csr2csc()
    cptr = st.colptr()
    v = scores(E, D, BF).requires_grad_()
    g = scores(E, D, BF, seed=2)
    for p, pm in ((ptr, None), (cptr, perm)):
        for _ in range(2):
            torch.autograd.grad(ops.segment_softmax(p, v, pm), v, g)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out = ops.segment_softmax(p, v, pm)
        torch.cuda.synchronize()
        assert torch.cuda.max_memory_allocated() - base <= E * D * 2 + (1 << 20)
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        (gr,) = torch.autograd.grad(out, v, g)
        torch.cuda.synchronize()
        assert torch.cuda.max_memory_allocated() - base <= E * D * 2 + (1 << 20)
        del out, gr


BIG_E, BIG_D, BIG_DEG = (1 << 28) + (1 << 16), 8, 16


def test_offsets_past_2_31():
    """E * D > 2^31 elements (bf16, rows of 16 entries, D = 8): forward and backward, the rows around element 2^31."""
    need = 4 * BIG_E * BIG_D * 2 + (2 << 30)
    if torch.cuda.mem_get_info()[0] < max(need, 24 << 30):
        pytest.skip("needs 24 GB of free device memory")
    _isolated("_offsets_past_2_31")


def _offsets_past_2_31():
    E, D, deg = BIG_E, BIG_D, BIG_DEG
    S = E // deg
    ptr = torch.arange(0, E + 1, deg, device=DEV)
    gen = torch.Generator(device=DEV).manual_seed(0)
    v = torch.randn(E, D, device=DEV, generator=gen, dtype=BF).mul_(3)
    out = ops.segment_softmax(ptr, v)
    g = torch.randn(E, D, device=DEV, generator=gen, dtype=BF)
    grad = ops.segment_softmax_bw(ptr, out, g, None)
    torch.cuda.synchronize()
    r0 = (1 << 31) // (deg * D)
    for lo in (0, r0 - 3, S - 4):
        a, b = lo * deg, (lo + 4) * deg          # rows lo .. lo + 3; r0 starts at element 2^31
        sub = torch.arange(0, b - a + 1, deg)
        assert_forward(out[a:b], sub, v[a:b], None, f"rows {lo}..")
        assert_backward(grad[a:b], sub, out[a:b], g[a:b], None, f"rows {lo}..")
