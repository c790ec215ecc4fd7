"""SpSpMM: every row path, column window and single-pass schedule of csrc/spspmm.cu against the oracle, with error
bounds taken from the kernel's rounding model.

`spspmm_kernel` chooses its path per row at run time: flat rows (one window, <= 128 A entries, <= 2048 products, the
products kept in registers) or general rows (re-walked per pass, in 128-entry A batches, window by window), with the
output of a window staged in shared memory when it has <= 2048 columns; the window size and the scan-chunk width follow
from N. Nothing outside the kernel shows which path ran, so the inputs are built for it: the dispatch is restated
below, every row of every input is classified with it, and the test asserts that each class occurs at its boundary.

The C-ABI is called directly, in both modes (symbolic + numeric, bound + single pass), into outputs prefilled with a
sentinel (-7777 indices, NaN values) between guard zones, so an element a kernel fails to write, or writes past its
end, cannot go unnoticed.

Values (util.spspmm_ref_bound): randn data within (n + 1) 2^-24 S (fp32) / 2 (n + 1) 2^-53 S (fp64) of the oracle,
n = products per entry, S = sum |a||b|, and exactly +0 where S = 0. Quantized data ({0, -0, +-1/2, +-1, +-2}) makes
every sum exact, so the order of the atomics cannot matter: bit-exact with the oracle, never -0 (the sum starts at +0,
as torch.sparse.mm's does), and with +-inf entries the same NaN positions.
"""
import collections
import ctypes
import functools
import re

import pytest
import torch

import pytorch_sparse_b200  # noqa: F401  (loads the library)
from pytorch_sparse_b200 import ops
from pytorch_sparse_b200._lib import lib
from util import ORACLE_MAX_N, assert_spspmm_values, launched_kernels, oracle_spspmm, spspmm_ref_bound

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENTINEL = -7777
GUARD = 64                      # sentinel-filled elements on each side of every output array

# ---- the dispatch, restated -----------------------------------------------------------------------------------------
THREADS = 256
STAGE_CAP = 2048                # products of a flat row; output columns of a staged window
A_BATCH = 128                   # A entries staged per batch
MAX_WINDOW = 1 << 18            # bits of the shared-memory bitmap


def window_bits_for(N):
    w = 1024
    while w < N and w < MAX_WINDOW:
        w <<= 1
    return w


def log2_wpt_for(window_bits):
    wpt = max((window_bits >> 5) // THREADS, 4)
    lw = 2
    while (1 << lw) < wpt:
        lw += 1
    return lw


def n_chunks(window_bits):
    return (window_bits >> 5) >> log2_wpt_for(window_bits)


EMPTY, FLAT, GENERAL1, GENERAL_N = 0, 1, 2, 3
CLASS_NAME = {EMPTY: "empty", FLAT: "flat", GENERAL1: "general single-batch", GENERAL_N: "general multi-batch"}

# N = 1, every power of two from 1024 to 2^18 and one N inside each interval, then multi-window widths
N_SINGLE = [1, 33, 1000, 1024, 1500, 2048, 3000, 4096, 6000, 8192, 12000, 16384, 20000, 32768, 40000, 65536, 100_000,
            131_072, 200_000, 262_144]
N_MULTI = [262_145, 3 * MAX_WINDOW + 5]
N_HUGE = (1 << 32) + 5          # columns 2^31 - 1, 2^31, 2^32 and N - 1
N_ALL = N_SINGLE + N_MULTI + [N_HUGE]

_PAIRS = {(window_bits_for(N), log2_wpt_for(window_bits_for(N))) for N in N_SINGLE}
assert _PAIRS == {(1 << k, 2 if k <= 15 else k - 13) for k in range(10, 19)}
assert all(n_chunks(1 << k) <= THREADS for k in range(10, 19))
assert {1 << k for k in range(10, 19)} <= set(N_SINGLE) and 1 in N_SINGLE
assert all(any((1 << k) < N < (1 << (k + 1)) for N in N_SINGLE) for k in range(10, 18))


# ---- structured operands ----------------------------------------------------------------------------------------------
class Case:
    def __init__(self, N, rows, brows):
        self.N, self.M, self.Kd = N, len(rows), len(brows)
        self.rpa, self.ca = _csr(rows)
        self.rpb, self.cb = _csr(brows)
        self.nnz_a, self.nnz_b = self.ca.numel(), self.cb.numel()

    @functools.cached_property
    def dev(self):
        return [t.to(DEV) for t in (self.rpa, self.ca, self.rpb, self.cb)]


def _csr(rows):
    lens = torch.tensor([len(r) for r in rows], dtype=torch.long)
    rp = torch.zeros(len(rows) + 1, dtype=torch.long)
    rp[1:] = lens.cumsum(0)
    cols = [torch.as_tensor(r, dtype=torch.long).view(-1) for r in rows]
    return rp, (torch.cat(cols) if cols else torch.empty(0, dtype=torch.long))


@functools.lru_cache(maxsize=None)
def structured(N, seed=0):
    """A (about 4000 rows, more than the grid has CTAs) times B (N columns). B rows are column-sorted and may repeat a
    column; A rows may be unsorted and repeat an entry. Rows on every class boundary are interleaved with random
    rows: empty rows, rows whose B rows are all empty, 2048 / 2049 products, 128 / 129 A entries, one B row of
    2048 / 2049 entries, 2048 products onto 1024 adjacent columns (one contended bitmap word per 32 lanes, the lost-bit
    repair), one column taking all 2048 products of a row, windows of 2048 / 2049 columns; for N beyond one window
    rows in two far-apart windows with empty windows between, columns on both sides of each window edge, and for the
    widest N the columns 2^31 - 1, 2^31, 2^32 - 1, 2^32 and N - 1."""
    g = torch.Generator().manual_seed(seed + N % 100_003)
    W = window_bits_for(N)
    huge = N > ORACLE_MAX_N
    # random columns anywhere for N up to a few windows; for the widest N in the two windows around 2^31, so that only
    # the rows built for it span many windows (each window costs the row a few barriers)
    lo, span = ((1 << 31) - MAX_WINDOW, 2 * MAX_WINDOW) if huge else (0, N)

    def rnd(n):
        return lo + torch.randint(span, (n,), generator=g)

    brows = []

    def B(cols):
        brows.append(torch.as_tensor(cols, dtype=torch.long).view(-1).sort().values)
        return len(brows) - 1

    empty = [B([]) for _ in range(3)]
    short = []
    for _ in range(48):
        c = rnd(int(torch.randint(1, 24, (1,), generator=g)))
        short.append(B(torch.cat([c, c[: int(torch.randint(0, 3, (1,), generator=g))]])))   # duplicate columns
    one = [B(rnd(1)) for _ in range(8)]
    len17 = B(rnd(17))
    l2048, l2049 = B(rnd(2048)), B(rnd(2049))
    c0 = int(rnd(1))
    dense1 = B((c0 + torch.arange(1024)) % N)
    dense2 = B((c0 + 512 + torch.arange(1024)) % N)
    same16 = B([int(rnd(1))] * 16)

    special = [
        [empty[0]], [empty[1], empty[0], empty[1]],                  # P = 0
        [l2048], [l2049],                                            # one B row of 2048 / 2049 entries
        [same16] * 128,                                              # n_a = 128, P = 2048 onto one column
        [same16] * 64 + [len17] + [same16] * 63,                     # n_a = 128, P = 2049
        [one[i % 8] for i in range(128)], [one[i % 8] for i in range(129)],      # n_a = 128 / 129
        [one[(3 * i) % 8] for i in range(300)] + [short[0], empty[2]],            # three A batches
        [dense1, dense1], [dense2, dense1], [dense1, dense1, one[0]],             # contended bitmap words
        [short[5], short[5], short[2], short[9], short[2]],                       # unsorted, repeated k
    ]
    if W >= 4096:   # a window of 2048 columns (staged when the row is general) and one of 2049 (unstaged)
        wbase = lo if huge else (W if N >= 2 * W else 0)
        wspan = min(W, N - wbase)
        wc = wbase + torch.randperm(wspan, generator=g)[:2049]
        w2048, w2049 = B(wc[:2048]), B(wc)
        special += [[w2048], [w2048, B(wc[:1])], [w2049], [one[1], w2049]]
    if N > MAX_WINDOW:
        far_lo, far_hi = B([3]), B([N - 2])
        last = (N - 1) // W
        ks = range(1, last + 1) if not huge else [1, 2, 1 << 13, (1 << 13) + 1, 1 << 14]
        edge = B([k * W + d for k in ks for d in (-1, 0)])
        special += [[far_lo, far_hi], [edge]]
        if huge:
            special += [[B([(1 << 31) - 1, 1 << 31, (1 << 32) - 1, 1 << 32, N - 1])],
                        [B([(1 << 31) - 1]), B([1 << 31])]]
        else:
            special += [[far_hi, one[2], far_lo], [edge, dense1], [B([W - 1]), B([W])], [B([last * W - 1, last * W])]]

    rows = [[]]
    for r in special:
        rows.append(r)
        for _ in range(int(torch.randint(0, 40, (1,), generator=g))):
            k = int(torch.randint(1, 9, (1,), generator=g))
            pool = short + one + empty[:1]
            rows.append([pool[int(j)] for j in torch.randint(len(pool), (k,), generator=g)])
        rows += [[]] * int(torch.randint(0, 2, (1,), generator=g))
    while len(rows) < 4000:
        k = int(torch.randint(0, 9, (1,), generator=g))
        rows.append([short[int(j)] for j in torch.randint(len(short), (k,), generator=g)])
    rows.append([])
    return Case(N, rows, brows)


def classify(case):
    """Per row: its class; and the number of distinct columns of every (row, window) of a general row."""
    n_a = case.rpa[1:] - case.rpa[:-1]
    deg_b = case.rpb[1:] - case.rpb[:-1]
    arow = torch.repeat_interleave(torch.arange(case.M), n_a)
    plen = deg_b[case.ca]
    P = torch.zeros(case.M, dtype=torch.long).index_add_(0, arow, plen)
    W = window_bits_for(case.N)
    multi = case.N > W
    flat = (n_a > 0) & (n_a <= A_BATCH) & (P <= STAGE_CAP) & torch.tensor(not multi)
    cls = torch.where(n_a == 0, EMPTY, torch.where(flat, FLAT, torch.where(n_a <= A_BATCH, GENERAL1, GENERAL_N)))
    # every product's (row, column)
    prow = torch.repeat_interleave(arow, plen)
    start = torch.repeat_interleave(case.rpb[case.ca], plen)
    first = torch.repeat_interleave(torch.cumsum(plen, 0) - plen, plen)
    pcol = case.cb[start + torch.arange(prow.numel()) - first]
    key = torch.unique(prow * case.N + pcol)
    urow, ucol = key // case.N, key % case.N
    rw, wcount = torch.unique(torch.stack([urow, ucol // W]), dim=1, return_counts=True)
    general_w = (cls[rw[0]] == GENERAL1) | (cls[rw[0]] == GENERAL_N)
    return dict(cls=cls, n_a=n_a, P=P, win_count=wcount[general_w])


def boundaries(case):
    """The class boundaries this input reaches."""
    c = classify(case)
    cls, n_a, P = c["cls"], c["n_a"], c["P"]
    flat, gen = cls == FLAT, (cls == GENERAL1) | (cls == GENERAL_N)
    hit = {CLASS_NAME[k] for k in cls.unique().tolist()}
    facts = {
        "flat P=2048": flat & (P == 2048), "general P=2049": gen & (P == 2049),
        "flat n_a=128": flat & (n_a == 128), "general multi-batch n_a=129": (cls == GENERAL_N) & (n_a == 129),
        "flat one B row of 2048": flat & (n_a == 1) & (P == 2048),
        "general one B row of 2049": gen & (n_a == 1) & (P == 2049),
    }
    hit |= {k for k, m in facts.items() if bool(m.any())}
    if bool((c["win_count"] <= STAGE_CAP).any()):
        hit.add("staged")
    if bool((c["win_count"] > STAGE_CAP).any()):
        hit.add("unstaged")
    if bool((c["win_count"] == 2048).any()):
        hit.add("staged window of 2048")
    if bool((c["win_count"] == 2049).any()):
        hit.add("unstaged window of 2049")
    if case.N == MAX_WINDOW and bool(flat.any()):
        hit.add("flat at N=2^18")
    if case.N == MAX_WINDOW + 1 and not bool(flat.any()) and bool(gen.any()):
        hit.add("only general at N=2^18+1")
    return hit


def test_row_classes_cover_every_path():
    """Every class of the restated dispatch occurs, and at each of its boundaries, across the inputs below."""
    want = {"empty", "flat", "general single-batch", "general multi-batch", "staged", "unstaged", "flat P=2048",
            "general P=2049", "flat n_a=128", "general multi-batch n_a=129", "flat one B row of 2048",
            "general one B row of 2049", "staged window of 2048", "unstaged window of 2049", "flat at N=2^18",
            "only general at N=2^18+1"}
    hit = set()
    for N in N_ALL:
        b = boundaries(structured(N))
        assert {"empty", "general multi-batch"} <= b, (N, b)
        assert ("flat" in b) == (N <= MAX_WINDOW), (N, b)
        hit |= b
    assert want <= hit, want - hit


# ---- direct library calls -------------------------------------------------------------------------------------------
def _vp(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


class Guarded:
    """An n-element device array between two GUARD-element guard zones, all prefilled with the sentinel."""

    def __init__(self, n, dtype):
        self.n, self.fill = n, (float("nan") if dtype.is_floating_point else SENTINEL)
        self.whole = torch.full((n + 2 * GUARD,), self.fill, dtype=dtype, device=DEV)
        self.t = self.whole[GUARD:GUARD + n]

    def untouched(self, lo, hi):
        x = self.whole[GUARD + lo:GUARD + hi]
        return bool(x.isnan().all()) if self.whole.dtype.is_floating_point else bool((x == SENTINEL).all())

    def guards_intact(self):
        return self.untouched(-GUARD, 0) and self.untouched(self.n, self.n + GUARD)


def _host_scalar():
    return torch.full((1,), -1, dtype=torch.long).pin_memory()


def _workspace(case):
    nws = lib.tsb200_spspmm_workspace_bytes(case.M, case.Kd, case.N, case.nnz_a, case.nnz_b)
    return torch.empty(max(nws, 1), dtype=torch.uint8, device=DEV), nws


def call_bound(case):
    rpa, ca, rpb, cb = case.dev
    ws, nws = _workspace(case)
    h = _host_scalar()
    assert lib.tsb200_spspmm_bound(_vp(ca), _vp(rpb), case.nnz_a, _vp(ws), nws, _vp(h), _stream()) == 0
    torch.cuda.synchronize()
    return int(h)


def call_two_phase(case, va, vb, dtype, with_row=True):
    """tsb200_spspmm_symbolic + tsb200_spspmm_numeric; dtype None = structure only."""
    rpa, ca, rpb, cb = case.dev
    ws, nws = _workspace(case)
    h = _host_scalar()
    rp = Guarded(case.M + 1, torch.long)
    rc = lib.tsb200_spspmm_symbolic(_vp(rpa), _vp(ca), _vp(rpb), _vp(cb), case.M, case.Kd, case.N, case.nnz_a,
                                    case.nnz_b, _vp(rp.t), _vp(ws), nws, _vp(h), _stream())
    assert rc == 0, rc
    torch.cuda.synchronize()
    nnz = int(h)
    row, col = Guarded(nnz, torch.long), Guarded(nnz, torch.long)
    val = Guarded(nnz, dtype) if dtype is not None else None
    rc = lib.tsb200_spspmm_numeric(_vp(rpa), _vp(ca), _vp(va), _vp(rpb), _vp(cb), _vp(vb), case.M, case.Kd, case.N,
                                   case.nnz_a, case.nnz_b, _vp(rp.t), _vp(row.t) if with_row else None, _vp(col.t),
                                   _vp(val.t) if val else None, ops._dtype_code(dtype) if val else 0, _vp(ws), nws,
                                   _stream())
    assert rc == 0, rc
    torch.cuda.synchronize()
    outs = [rp, row, col] + ([val] if val else [])
    assert all(o.guards_intact() for o in outs), "two-phase: write outside an output array"
    if not with_row:
        assert row.untouched(0, nnz), "two-phase: row_c = NULL, yet row indices were written"
    return nnz, rp.t.cpu(), (row.t.cpu() if with_row else None), col.t.cpu(), (val.t.cpu() if val else None)


def call_fused(case, va, vb, dtype, with_row=True, capacity=None):
    """tsb200_spspmm_bound + tsb200_spspmm_fused into arrays of `capacity` (default: the bound) entries."""
    rpa, ca, rpb, cb = case.dev
    bound = call_bound(case)
    cap = bound if capacity is None else capacity
    ws, nws = _workspace(case)
    h = _host_scalar()
    rp = Guarded(case.M + 1, torch.long)
    row, col = Guarded(cap, torch.long), Guarded(cap, torch.long)
    val = Guarded(cap, dtype) if dtype is not None else None
    rc = lib.tsb200_spspmm_fused(_vp(rpa), _vp(ca), _vp(va), _vp(rpb), _vp(cb), _vp(vb), case.M, case.Kd, case.N,
                                 case.nnz_a, case.nnz_b, _vp(rp.t), _vp(row.t) if with_row else None, _vp(col.t),
                                 _vp(val.t) if val else None, cap, ops._dtype_code(dtype) if val else 0, _vp(ws), nws,
                                 _vp(h), _stream())
    assert rc == 0, rc
    torch.cuda.synchronize()
    nnz = int(h)
    outs = [rp, row, col] + ([val] if val else [])
    assert all(o.guards_intact() for o in outs), "fused: write outside an output array"
    if nnz >= 0:
        assert all(o.untouched(nnz, cap) for o in outs[1:]), "fused: entries [nnz(C), capacity) were written"
    if not with_row:
        assert row.untouched(0, cap), "fused: row_c = NULL, yet row indices were written"
    n = max(nnz, 0)
    return nnz, rp.t.cpu(), (row.t[:n].cpu() if with_row else None), col.t[:n].cpu(), (val.t[:n].cpu() if val else None)


MODES = {"two_phase": call_two_phase, "fused": call_fused}


# ---- references and comparisons ---------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def oracle_structure(oracle, N):
    c = structured(N)
    rp, r, col, _ = oracle_spspmm(oracle, c.rpa, c.ca, None, c.rpb, c.cb, None, c.M, c.Kd, c.N, want_value=False)
    return rp, r, col


def _where(case, row):
    """Describes failing output entries by the class of their row."""
    def describe(bad):
        cls = classify(case)["cls"]
        cnt = collections.Counter(CLASS_NAME[int(k)] for k in cls[row[bad]])
        return "failing entries by row class: " + ", ".join(f"{k} {v}" for k, v in sorted(cnt.items()))
    return describe


def check_structure(oracle, case, out, what):
    rp, r, col = oracle_structure(oracle, case.N)
    nnz, orp, orow, ocol, _ = out
    assert nnz == r.numel(), (what, nnz, r.numel())
    assert torch.equal(orp, rp), what + ": rowptr"
    assert torch.equal(ocol, col), what + ": col"
    if orow is not None:
        assert torch.equal(orow, r), what + ": row"


def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int64)


def assert_bits_equal(v, ref, where, what):
    """Bit-exact except that NaN must meet NaN; no -0 anywhere."""
    nan = ref.isnan()
    bad = (v.isnan() != nan) | (~nan & (_bits(v) != _bits(ref))) | ((v == 0) & torch.signbit(v))
    if bool(bad.any()):
        i = int(bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {v.numel()} values differ, first at {i}: {v[i].item()!r} vs "
                             f"{ref[i].item()!r}; {where(bad)}")


def randn_values(n, dtype, seed):
    """randn with 5 % signed zeros (entries whose every product is zero must come out +0)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, generator=g, dtype=torch.float64)
    z = torch.rand(n, generator=g) < 0.05
    x = torch.where(z, torch.where(torch.rand(n, generator=g) < 0.5, -0.0, 0.0), x)
    return x.to(dtype)


def quantized_values(n, dtype, seed, inf=False):
    g = torch.Generator().manual_seed(seed)
    q = torch.tensor([0.0, -0.0, 0.5, -0.5, 1.0, -1.0, 2.0, -2.0], dtype=torch.float64)
    x = q[torch.randint(q.numel(), (n,), generator=g)]
    if inf:
        pick = torch.rand(n, generator=g) < 0.01
        x = torch.where(pick, torch.where(torch.rand(n, generator=g) < 0.5, -torch.inf, torch.inf), x)
    return x.to(dtype)


SIDES = [("A", "B"), ("A", "-"), ("-", "B"), ("-", "-")]


def _sides(va, vb, sides):
    return (va if sides[0] == "A" else None), (vb if sides[1] == "B" else None)


# ---- every N x dtype: structure, randn values, quantized values ------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("N", N_ALL)
def test_paths_vs_oracle(oracle, N, dtype):
    case = structured(N)
    rpa, ca, rpb, cb = case.rpa, case.ca, case.rpb, case.cb
    args = (case.M, case.Kd, case.N)
    deg_b = rpb[1:] - rpb[:-1]
    assert call_bound(case) == int(deg_b[ca].sum())          # the bound is the exact number of products
    for mode, call in MODES.items():                         # structure only, row_c as a buffer and as NULL
        for with_row in (True, False):
            check_structure(oracle, case, call(case, None, None, None, with_row), f"{mode} N={N} structure")
    _, row_ref, _ = oracle_structure(oracle, N)
    where = _where(case, row_ref)

    va, vb = randn_values(case.nnz_a, dtype, 1), randn_values(case.nnz_b, dtype, 2)
    va_d, vb_d = va.to(DEV), vb.to(DEV)
    for sides in SIDES:
        a, b = _sides(va, vb, sides)
        ref, bound = spspmm_ref_bound(oracle, rpa, ca, a, rpb, cb, b, *args, dtype)
        for mode, call in MODES.items():
            what = f"{mode} N={N} {dtype} randn {sides}"
            out = call(case, *_sides(va_d, vb_d, sides), dtype, with_row=sides != ("A", "-"))
            check_structure(oracle, case, out, what)
            assert_spspmm_values(out[4], ref, bound, what, where)

    for inf in (False, True):
        va, vb = quantized_values(case.nnz_a, dtype, 3 + inf, inf), quantized_values(case.nnz_b, dtype, 5 + inf, inf)
        va_d, vb_d = va.to(DEV), vb.to(DEV)
        for sides in (SIDES if not inf else SIDES[:1]):
            a, b = _sides(va, vb, sides)
            ones = lambda t, n: torch.ones(n, dtype=dtype) if t is None else t  # noqa: E731
            ref = oracle_spspmm(oracle, rpa, ca, ones(a, case.nnz_a), rpb, cb, ones(b, case.nnz_b), *args)[3]
            if inf:
                assert bool(ref.isnan().any()) and bool(ref.isinf().any())
            for mode, call in MODES.items():
                what = f"{mode} N={N} {dtype} quantized{' +-inf' if inf else ''} {sides}"
                out = call(case, *_sides(va_d, vb_d, sides), dtype, with_row=sides != ("-", "B"))
                check_structure(oracle, case, out, what)
                assert_bits_equal(out[4], ref, where, what)


@pytest.mark.parametrize("N", [1, 3000, 65_536, 262_144, 262_145, 3 * MAX_WINDOW + 5, N_HUGE])
def test_vs_torch_sparse_mm(N):
    """On duplicate-free operands, bit for bit with torch.sparse.mm on the CPU (COO, the reference's own call), in
    fp32 and fp64, quantized values with signed zeros and +-inf. B's columns are relabelled 0..U-1 for the CPU call
    (ATen's Gustavson keeps an N-long accumulator)."""
    case = structured(N)
    ka = torch.unique(torch.repeat_interleave(torch.arange(case.M), case.rpa[1:] - case.rpa[:-1]) * case.Kd + case.ca)
    kb = torch.unique(torch.repeat_interleave(torch.arange(case.Kd), case.rpb[1:] - case.rpb[:-1]) * case.N + case.cb)
    ra, ca = ka // case.Kd, ka % case.Kd
    rb, cb = kb // case.N, kb % case.N
    dd = Case(N, [ca[ra == i] for i in range(case.M)], [cb[rb == k] for k in range(case.Kd)])
    uniq = torch.unique(cb)
    for dtype in (torch.float32, torch.float64):
        va, vb = quantized_values(ca.numel(), dtype, 7, True), quantized_values(cb.numel(), dtype, 8, True)
        A = torch.sparse_coo_tensor(torch.stack([ra, ca]), va, (case.M, case.Kd))
        Bt = torch.sparse_coo_tensor(torch.stack([rb, torch.searchsorted(uniq, cb)]), vb, (case.Kd, uniq.numel()))
        ref = torch.sparse.mm(A, Bt).coalesce()
        rrow, rcol, rval = ref.indices()[0], uniq[ref.indices()[1]], ref.values()
        for mode, call in MODES.items():
            nnz, rp, row, col, val = call(dd, va.to(DEV), vb.to(DEV), dtype)
            what = f"{mode} N={N} {dtype} vs torch.sparse.mm"
            assert torch.equal(row, rrow) and torch.equal(col, rcol), what
            assert_bits_equal(val, rval, lambda bad: "", what)


# ---- the C-ABI contracts ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [6000, 3 * MAX_WINDOW + 5])
def test_fused_capacity(oracle, N):
    """Too small an output: the single pass returns -1 and writes nothing past `capacity` (guard zone intact); with
    the bound as capacity, entries [nnz(C), capacity) keep the sentinel (checked in call_fused)."""
    case = structured(N)
    va, vb = randn_values(case.nnz_a, torch.float32, 1).to(DEV), randn_values(case.nnz_b, torch.float32, 2).to(DEV)
    nnz = call_fused(case, va, vb, torch.float32)[0]
    assert 0 < nnz < call_bound(case)
    for cap in (nnz - 1, 0):
        assert call_fused(case, va, vb, torch.float32, capacity=cap)[0] == -1
        assert call_fused(case, None, None, None, capacity=cap)[0] == -1
    check_structure(oracle, case, call_fused(case, va, vb, torch.float32, capacity=nnz), f"N={N} capacity = nnz")


def test_bound_loops_over_a_large_a():
    """nnz_a > 8 * 1024 * SMs: the bound kernel's grid is capped and each thread loops; the bound stays exact."""
    sms = lib.tsb200_sm_count()
    g = torch.Generator().manual_seed(11)
    Kd = 1000
    deg = torch.randint(0, 50, (Kd,), generator=g)
    rpb = torch.zeros(Kd + 1, dtype=torch.long)
    rpb[1:] = deg.cumsum(0)
    E = 8 * 1024 * sms + 12_345
    ca = torch.randint(Kd, (E,), generator=g)
    ws = torch.empty(256, dtype=torch.uint8, device=DEV)
    h = _host_scalar()
    assert lib.tsb200_spspmm_bound(_vp(ca.to(DEV)), _vp(rpb.to(DEV)), E, _vp(ws), 256, _vp(h), _stream()) == 0
    torch.cuda.synchronize()
    assert int(h) == int(deg[ca].sum())


def test_lookback_across_rows_without_output(oracle):
    """A tall matrix whose rows mostly produce 0 or 1 entries, with runs of 40, 100 and 1000 rows without output and
    the first row with output at index >= 64. Rows without output never publish a prefix, so a row only finds its
    offset by walking back (distance to the previous row with output) / 32 steps at least: a correct rowptr_c shows
    that the multi-step walks ran."""
    g = torch.Generator().manual_seed(12)
    M, N = 300_000, 64
    brows = [[], [5], [7, 9]]                     # B row 0 is empty: an A row on it is not empty but has no output
    kind = torch.randint(0, 4, (M,), generator=g)  # 0: empty A row, 1: A row on the empty B row, 2-3: output
    kind[:100] = torch.randint(0, 2, (100,), generator=g)
    for start, run in ((5000, 40), (90_000, 100), (200_000, 1000)):
        kind[start:start + run] = torch.randint(0, 2, (run,), generator=g)
    rows = [[] if k == 0 else [0] if k == 1 else [int(k) - 1] for k in kind.tolist()]
    case = Case(N, rows, brows)
    rpa, ca, rpb, cb = case.dev
    ws, nws = _workspace(case)
    h = _host_scalar()
    bound = call_bound(case)
    rowc, colc = Guarded(bound, torch.long), Guarded(bound, torch.long)
    rpc = Guarded(M + 1, torch.long)
    assert lib.tsb200_spspmm_fused(_vp(rpa), _vp(ca), None, _vp(rpb), _vp(cb), None, M, case.Kd, N, case.nnz_a,
                                   case.nnz_b, _vp(rpc.t), _vp(rowc.t), _vp(colc.t), None, bound, 0, _vp(ws), nws,
                                   _vp(h), _stream()) == 0
    torch.cuda.synchronize()
    rp, _, col, _ = oracle.spspmm(case.rpa, case.ca, None, case.rpb, case.cb, None, M, case.Kd, N, False)
    nnz = int(h)
    assert nnz == col.numel() and torch.equal(rpc.t.cpu(), rp) and torch.equal(colc.t[:nnz].cpu(), col)
    out_rows = ((rp[1:] - rp[:-1]) > 0).nonzero().view(-1)
    assert int(out_rows[0]) >= 64
    prev = torch.cat([torch.tensor([-1]), out_rows[:-1]])
    need = torch.where(prev < 0, (out_rows + 31) // 32, (out_rows - prev + 31) // 32)
    assert int(need.sum()) > out_rows.numel() + 1000 // 32, "the input forces no multi-step walk"


def test_null_operands_after_the_memsets():
    """The symbolic and single-pass entry points zero rowptr_c and their scalars before they check the operands (the
    checks the CPU table cannot reach): a NULL operand, or a NULL col_c with room for output, returns -1 and leaves
    rowptr_c all zeros."""
    case = structured(3000)
    ws, nws = _workspace(case)
    rp = torch.empty(case.M + 1, dtype=torch.long, device=DEV)
    col = torch.empty(16, dtype=torch.long, device=DEV)
    sizes = (case.M, case.Kd, case.N, case.nnz_a, case.nnz_b)

    def symbolic(rpa, ca, rpb, cb, col_c):
        return lib.tsb200_spspmm_symbolic(rpa, ca, rpb, cb, *sizes, _vp(rp), _vp(ws), nws, None, _stream())

    def fused(rpa, ca, rpb, cb, col_c):
        return lib.tsb200_spspmm_fused(rpa, ca, None, rpb, cb, None, *sizes, _vp(rp), None, col_c, None, 16, 0, _vp(ws),
                                       nws, None, _stream())

    good = [_vp(t) for t in case.dev] + [_vp(col)]
    calls = [(fn, j) for fn in (symbolic, fused) for j in range(4)] + [(fused, 4)]
    for fn, j in calls:
        args = list(good)
        args[j] = None
        what = f"{fn.__name__}: {['rowptr_a', 'col_a', 'rowptr_b', 'col_b', 'col_c'][j]} = NULL"
        rp.fill_(SENTINEL)
        assert fn(*args) == -1, what
        torch.cuda.synchronize()
        assert bool((rp == 0).all()), what + ": rowptr_c not zeroed"


# ---- edge extents through ops.spspmm ------------------------------------------------------------------------------------
def _edge_cases():
    g = torch.Generator().manual_seed(13)

    def rand_rows(M, deg_hi, Kd):
        return [torch.randint(Kd, (int(torch.randint(0, deg_hi, (1,), generator=g)),), generator=g) for _ in range(M)]

    def rand_brows(Kd, N, deg_hi):
        return [torch.randint(N, (int(torch.randint(0, deg_hi, (1,), generator=g)),), generator=g) for _ in range(Kd)]

    return {
        "M=0": (0, 7, 10, [], rand_brows(7, 10, 4)),
        "nnz_a=0": (5, 7, 10, [[]] * 5, rand_brows(7, 10, 4)),
        "nnz_b=0": (5, 7, 10, rand_rows(5, 6, 7), [[]] * 7),
        "N=1": (40, 30, 1, rand_rows(40, 12, 30), rand_brows(30, 1, 5)),
        "one A row of 5000": (1, 300, 4000, [torch.randint(300, (5000,), generator=g)], rand_brows(300, 4000, 6)),
        "M=3 (fewer rows than CTAs)": (3, 50, 500, rand_rows(3, 60, 50), rand_brows(50, 500, 30)),
    }


@pytest.mark.parametrize("mode", ["two_phase", "fused", "auto"])
@pytest.mark.parametrize("name", list(_edge_cases()))
def test_edge_extents(oracle, monkeypatch, mode, name):
    monkeypatch.setenv("TSB200_SPSPMM", mode)
    M, Kd, N, rows, brows = _edge_cases()[name]
    rpa, ca = _csr(rows)
    rpb, cb = _csr(brows)
    for dtype in (torch.float32, torch.float64):
        va, vb = randn_values(ca.numel(), dtype, 1), randn_values(cb.numel(), dtype, 2)
        rp, r, c, v = ops.spspmm(rpa.to(DEV), ca.to(DEV), va.to(DEV), rpb.to(DEV), cb.to(DEV), vb.to(DEV), M, Kd, N,
                                 True)
        orp, orow, oc, _ = oracle.spspmm(rpa, ca, va, rpb, cb, vb, M, Kd, N)
        what = f"{mode} {name} {dtype}"
        assert torch.equal(rp.cpu(), orp) and torch.equal(r.cpu(), orow) and torch.equal(c.cpu(), oc), what
        ref, bound = spspmm_ref_bound(oracle, rpa, ca, va, rpb, cb, vb, M, Kd, N, dtype)
        assert v.dtype == dtype
        assert_spspmm_values(v, ref, bound, what)


# ---- TSB200_SPSPMM=auto -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_auto_mode_kernels(monkeypatch, dtype):
    """auto takes the single pass when the product bound fits easily (a small product always does); two_phase runs
    the symbolic and the numeric kernel. Each numeric kernel runs in the dtype it was given."""
    case = structured(3000)
    rpa, ca, rpb, cb = case.dev
    va, vb = randn_values(case.nnz_a, dtype, 1).to(DEV), randn_values(case.nnz_b, dtype, 2).to(DEV)
    T = "float" if dtype == torch.float32 else "double"

    def kernels(mode, patterns):
        monkeypatch.setenv("TSB200_SPSPMM", mode)
        names = launched_kernels(lambda: ops.spspmm(rpa, ca, va, rpb, cb, vb, case.M, case.Kd, case.N, True),
                                 patterns)
        return {m.groups() for n in names for m in [re.search(r"spspmm_kernel<(\d), (float|double)>", n)] if m}, names

    got, names = kernels("auto", [r"spspmm_kernel<"])
    assert got == {("2", T)}, names
    got, names = kernels("two_phase", [r"spspmm_kernel<0,", r"spspmm_kernel<1,"])
    assert got == {("0", "float"), ("1", T)}, names
