"""Coalesce, format conversion and segment reduce: every kernel path of csrc/coalesce.cu and csrc/convert.cu against the
oracle, bit for bit where the kernel's arithmetic order is the oracle's, else within an error bound taken from the
kernel's rounding model (util.segment_sum_ref_bound).

The C-ABI is called directly, into outputs prefilled with a sentinel (-7777 indices, NaN values) between guard zones,
so an element a kernel fails to write, or writes past its end, cannot go unnoticed. The dispatch decisions that nothing
outside a kernel shows (the coalesce key mode, the skipped sort, the grid-stride caps) are restated below and every
input is checked to reach the branch it was built for; the coalesce key mode and the skipped sort are also read back
from the workspace the sort phase leaves behind.

Rules pinned here (include/tsb200.h): sums and means start at +0, so a run of -0 gives +0; min / max compare strictly
from the segment's first entry, so a NaN there is the result and a NaN anywhere else never is, and the arg is the first
entry attaining the extreme; coalesce keys row * N + col are one 64-bit word, so M * N <= 2^64.
"""
import ctypes
import functools

import pytest
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import ops
from pytorch_sparse_b200._lib import Tsb200Error, lib
from util import assert_spspmm_values, segment_sum_ref_bound

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENTINEL = -7777
GUARD = 64
ERR_UNSUPPORTED = -2
REDUCES = ["sum", "mean", "min", "max"]
RED = {"sum": 0, "mean": 1, "min": 2, "max": 3}
FLOATS = [torch.float32, torch.float64, torch.bfloat16, torch.float16]
ALL_DTYPES = FLOATS + [torch.int32, torch.int64]
DT_ID = {torch.float32: "f32", torch.float64: "f64", torch.bfloat16: "bf16", torch.float16: "f16",
         torch.int32: "i32", torch.int64: "i64"}


# ---- the dispatch, restated ------------------------------------------------------------------------------------------
@functools.cache
def sms():
    return lib.tsb200_sm_count()


def grid_stride_cap():
    """Threads of a capped 1-D grid (coalesce, ind2ptr, csr2csc, segment_reduce_bw): sm_count * 32 blocks of 256."""
    return sms() * 32 * 256


def warp_cap():
    """Warps of a capped grid (ptr2ind: 32 rows per warp; segment_reduce: one segment per warp)."""
    return grid_stride_cap() // 32


def key_mode(M, N, E):
    """(bits, ebits, ib) of tsb200_coalesce_sort: the key row * N + col takes bits = ceil(log2(M N)) (1..64); the
    input position takes ebits = ceil(log2 E) (>= 1); packed (ib = ebits, position in the key's low bits) iff
    bits + ebits <= 64, else unpacked (ib = 0, a separate 32-bit payload)."""
    mk = max(M, 1) * max(N, 1)
    bits = 1
    while bits < 64 and (1 << bits) < mk:
        bits += 1
    ebits = 1
    while (1 << ebits) < E:
        ebits += 1
    return bits, ebits, (ebits if bits + ebits <= 64 else 0)


def bits_for(n):
    """Key bits of the csr2csc sort: values in [0, n)."""
    b = 1
    while b < 63 and (1 << b) < n:
        b += 1
    return b


assert key_mode(1 << 26, 1 << 26, 4096)[2] == 12 and key_mode(1 << 26, 1 << 26, 4097)[2] == 0
assert key_mode(1 << 32, 1 << 32, 1)[2] == 0 and key_mode(7, 5, 1) == (6, 1, 1)


# ---- direct library calls --------------------------------------------------------------------------------------------
def _vp(t):
    """Raw pointer of a tensor the caller keeps alive until the work that reads it has finished (a temporary such
    as `_vp(x.to(DEV))` is freed at once, and its memory may be handed to the next allocation before the launch)."""
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


class Guarded:
    """An n-element device array between two GUARD-element guard zones, all prefilled with the sentinel."""

    def __init__(self, n, dtype):
        self.n, self.dtype = n, dtype
        fill = float("nan") if dtype.is_floating_point else SENTINEL
        self.whole = torch.full((n + 2 * GUARD,), fill, dtype=dtype, device=DEV)
        self.t = self.whole[GUARD:GUARD + n]

    def untouched(self, lo, hi):
        x = self.whole[GUARD + lo:GUARD + hi]
        return bool(x.isnan().all()) if self.dtype.is_floating_point else bool((x == SENTINEL).all())

    def guards_intact(self):
        return self.untouched(-GUARD, 0) and self.untouched(self.n, self.n + GUARD)

    def get(self):
        assert self.guards_intact(), "write outside an output array"
        return self.t.cpu()


def _bits(t):
    return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()]) if t.dtype.is_floating_point \
        else t


def assert_same(got, ref, what):
    """Bit for bit, except that NaN must meet NaN (any payload)."""
    got, ref = got.cpu(), ref.cpu()
    assert got.shape == ref.shape and got.dtype == ref.dtype, (what, got.shape, ref.shape, got.dtype, ref.dtype)
    if got.dtype.is_floating_point:
        nan = ref.isnan()
        bad = (got.isnan() != nan) | (~nan & (_bits(got) != _bits(ref)))
    else:
        bad = got != ref
    if bool(bad.any()):
        i = int(bad.reshape(-1).nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {got.numel()} differ, first at flat {i}: "
                             f"{got.reshape(-1)[i].item()!r} vs {ref.reshape(-1)[i].item()!r}")


class Coalesced:
    """tsb200_coalesce_sort, then tsb200_coalesce_perm; what the sort phase left in the workspace."""

    def __init__(self, row, col, M, N):
        self.E, self.M, self.N = row.numel(), M, N
        self.row, self.col = row.to(DEV), col.to(DEV)
        self.nws = lib.tsb200_coalesce_workspace_bytes(self.E, M, N)
        self.ws = torch.empty(max(self.nws, 1), dtype=torch.uint8, device=DEV)
        h = torch.full((1,), -1, dtype=torch.long).pin_memory()
        rc = lib.tsb200_coalesce_sort(_vp(self.row), _vp(self.col), self.E, M, N, _vp(self.ws), self.nws, _vp(h),
                                      _stream())
        assert rc == 0, rc
        torch.cuda.synchronize()
        self.n_unique = int(h)
        sc = self.ws[:32].cpu().view(torch.int32)
        self.sorted_ran, self.ib = bool(sc[0]), int(sc[6])     # scalars: [0] unsorted flag, [4..6] {keys, perm, ib}
        perm = Guarded(self.E, torch.long)
        assert lib.tsb200_coalesce_perm(self.E, _vp(perm.t), _vp(self.ws), _stream()) == 0
        torch.cuda.synchronize()
        self.perm = perm.get()

    def emit(self, value=None, reduce="sum", outs=("row", "col", "perm", "seg", "count", "arg")):
        """tsb200_coalesce_emit into guarded outputs; the outputs not in `outs` are passed as NULL."""
        nu, E = self.n_unique, self.E
        D = (value.numel() // max(E, 1) if E else 0) if value is not None else 1
        sizes = {"row": nu, "col": nu, "perm": nu, "seg": E, "count": nu, "arg": nu * D}
        g = {k: Guarded(sizes[k], torch.long) for k in outs}
        vo = Guarded(nu * D, value.dtype) if value is not None else None
        vin = value.to(DEV).contiguous() if value is not None else None
        rc = lib.tsb200_coalesce_emit(E, self.N, nu, _vp(vin), D, ops._dtype_code(value.dtype) if vin is not None
                                      else 0, RED[reduce], *[_vp(g[k].t) if k in g else None
                                                             for k in ("row", "col")], _vp(vo.t) if vo else None,
                                      *[_vp(g[k].t) if k in g else None for k in ("perm", "seg", "count", "arg")],
                                      _vp(self.ws), _stream())
        assert rc == 0, rc
        torch.cuda.synchronize()
        res = {k: v.get() for k, v in g.items()}
        if vo is not None:
            res["value"] = vo.get()
            if D == 0:
                assert vo.guards_intact()
        return res


# ---- references ------------------------------------------------------------------------------------------------------
def oracle_coalesce_index(oracle, row, col):
    """oracle.coalesce_index on rows and columns relabelled 0..U-1 in order (the oracle's keys are signed int64, the
    kernel's go up to 2^64 - 1; an order-preserving relabelling changes neither the order nor the runs).
    -> (perm, row', col', seg_ptr)."""
    ur, uc = torch.unique(row), torch.unique(col)
    perm, r, c, seg = oracle.coalesce_index(torch.searchsorted(ur, row), torch.searchsorted(uc, col),
                                            max(uc.numel(), 1))
    return perm, ur[r], uc[c], seg


def oracle_coalesce_values(oracle, row, col, value, reduce):
    """-> (value', arg): the oracle on the storage dtype for f32 / f64 / i32 / i64; for bf16 / f16 on the values
    widened to f32 (the kernel's accumulator, same order) and rounded once to the storage dtype."""
    ur, uc = torch.unique(row), torch.unique(col)
    r, c = torch.searchsorted(ur, row), torch.searchsorted(uc, col)
    wide = value.float() if value.dtype in (torch.bfloat16, torch.float16) else value
    _, _, v, arg = oracle.coalesce(r, c, wide, ur.numel(), max(uc.numel(), 1), reduce, return_arg=True)
    return v.to(value.dtype), arg


# ---- coalesce inputs -------------------------------------------------------------------------------------------------
def _dups(keys_r, keys_c, g, lo=1, hi=3):
    """Every (row, col) 1..3 times, in key order."""
    reps = torch.randint(lo, hi + 1, (keys_r.numel(),), generator=g)
    return torch.repeat_interleave(keys_r, reps), torch.repeat_interleave(keys_c, reps)


def _unique_keys(M, N, n, g):
    r = torch.randint(M, (n,), generator=g, dtype=torch.long)
    c = torch.randint(N, (n,), generator=g, dtype=torch.long)
    k = torch.unique(torch.stack([r, c], 1), dim=0)
    return k[:, 0].contiguous(), k[:, 1].contiguous()


def _shuffle(row, col, g):
    p = torch.randperm(row.numel(), generator=g)
    return row[p], col[p]


@functools.cache
def coalesce_cases():
    """name -> (row, col, M, N, expect_sort_ran)."""
    g = torch.Generator().manual_seed(20)
    cases = {}
    r, c = _dups(*_unique_keys(3000, 2000, 6000, g), g)
    cases["shuffled, 1-3 copies"] = (*_shuffle(r, c, g), 3000, 2000, True)
    cases["sorted with duplicates"] = (r, c, 3000, 2000, False)
    r, c = _dups(*_unique_keys(500, 700, 3000, g), g)
    r, c = r[:2048].clone(), c[:2048].clone()
    while bool((r[255] == r[256]) & (c[255] == c[256])):      # make entries 255, 256 two distinct keys
        r, c = r[1:].clone(), c[1:].clone()
    r[[255, 256]], c[[255, 256]] = r[[256, 255]], c[[256, 255]]
    cases["one descending pair across a 256-entry block"] = (r, c, 500, 700, True)
    cap = grid_stride_cap()
    r, c = _dups(*_unique_keys(1 << 20, 1 << 12, cap, g), g, 1, 2)
    r, c = r[:cap + 4096].clone(), c[:cap + 4096].clone()
    while bool((r[cap - 1] == r[cap]) & (c[cap - 1] == c[cap])):
        r, c = torch.cat([r[:1], r]), torch.cat([c[:1], c])
    r[[cap - 1, cap]], c[[cap - 1, cap]] = r[[cap, cap - 1]], c[[cap, cap - 1]]
    cases["one descending pair past the grid-stride cap"] = (r, c, 1 << 20, 1 << 12, True)
    r, c = _dups(*_unique_keys(4000, 4000, 4000, g), g)
    r = torch.cat([r, torch.full((1 << 17,), 1234)])
    c = torch.cat([c, torch.full((1 << 17,), 567)])
    cases["a run of 2^17 duplicates"] = (*_shuffle(r, c, g), 4000, 4000, True)
    big = [0, 1, (1 << 31) - 1, 1 << 31, (1 << 32) - 2, (1 << 32) - 1]
    kr = torch.tensor(big).repeat_interleave(len(big))
    kc = torch.tensor(big).repeat(len(big))
    r, c = _dups(kr, kc, g)
    cases["rows / cols at 2^31 - 1, 2^31, 2^32 - 1 (M = N = 2^32)"] = (*_shuffle(r, c, g), 1 << 32, 1 << 32, True)
    for E in (4096, 4097):
        r, c = _dups(*_unique_keys(1 << 26, 1 << 26, 3000, g), g)
        r, c = _shuffle(r[:E], c[:E], g)
        r[-1], c[-1] = (1 << 26) - 1, (1 << 26) - 1                  # the largest key
        cases[f"M = N = 2^26, E = {E}"] = (r, c, 1 << 26, 1 << 26, True)
    for E in (1024, 1025):
        r, c = _dups(*_unique_keys(1 << 27, 1 << 26, 1000, g), g)
        cases[f"M = 2^27, N = 2^26, E = {E}"] = (*_shuffle(r[:E], c[:E], g), 1 << 27, 1 << 26, True)
    cases["E = 1"] = (torch.tensor([5]), torch.tensor([3]), 9, 4, False)
    cases["E = 2, one key"] = (torch.tensor([5, 5]), torch.tensor([3, 3]), 9, 4, False)
    return cases


def test_coalesce_cases_reach_every_branch():
    """Across the inputs: packed and unpacked keys on both sides of a boundary (M = N = 2^26: 52 + 12 bits packed,
    52 + 13 not; M = 2^27, N = 2^26: E = 2^10 / 2^10 + 1), E = 1, a skipped sort with duplicates, a sort started by
    a pair at a block boundary and by one past the grid-stride cap, and keys above 2^63."""
    modes = {name: key_mode(M, N, r.numel()) for name, (r, c, M, N, _) in coalesce_cases().items()}
    assert modes["M = N = 2^26, E = 4096"] == (52, 12, 12) and modes["M = N = 2^26, E = 4097"] == (52, 13, 0)
    assert modes["M = 2^27, N = 2^26, E = 1024"] == (53, 10, 10) and modes["M = 2^27, N = 2^26, E = 1025"][2] == 11
    assert modes["E = 1"][1] == 1
    assert {m[2] == 0 for m in modes.values()} == {True, False}
    r, c, M, N, _ = coalesce_cases()["one descending pair past the grid-stride cap"]
    assert r.numel() > grid_stride_cap()
    for name, (r, c, M, N, ran) in coalesce_cases().items():
        desc = (r[1:] < r[:-1]) | ((r[1:] == r[:-1]) & (c[1:] < c[:-1]))
        assert bool(desc.any()) == ran, name
        if name.startswith("one descending pair"):
            assert int(desc.sum()) == 1
            i = int(desc.nonzero()[0]) + 1
            assert i % 256 == 0 and (i == 256 or i == grid_stride_cap()), (name, i)


@pytest.mark.parametrize("name", list(coalesce_cases()))
def test_coalesce_structure(oracle, name):
    """n_unique, the key mode, the skipped sort, row' / col', the full sorted perm, perm_out, seg_out (run id of
    every input entry) and count_out against the oracle, each optional output as a buffer and as NULL."""
    row, col, M, N, ran = coalesce_cases()[name]
    co = Coalesced(row, col, M, N)
    assert co.ib == key_mode(M, N, row.numel())[2], (name, co.ib)
    assert co.sorted_ran == ran, name
    perm, r, c, seg = oracle_coalesce_index(oracle, row, col)
    nu = r.numel()
    assert co.n_unique == nu, name
    assert torch.equal(co.perm, perm), name
    count = seg[1:] - seg[:-1]
    seg_in = torch.empty_like(perm)
    seg_in[perm] = torch.repeat_interleave(torch.arange(nu), count)
    want = {"row": r, "col": c, "perm": perm[seg[:-1]], "seg": seg_in, "count": count}
    full = co.emit(outs=tuple(want))
    for k, v in want.items():
        assert torch.equal(full[k], v), (name, k)
    for drop in want:                                          # each output NULL in turn; the others unchanged
        part = co.emit(outs=tuple(k for k in want if k != drop))
        for k in part:
            assert torch.equal(part[k], want[k]), (name, "without", drop, k)


def coalesce_values(n, dtype, g, special):
    """randn (floats) or small integers; `special`: values from {+-0, +-1, 2, +-inf, NaN} (ties, signed zeros, NaN as
    the first and as a later entry of runs)."""
    if not dtype.is_floating_point:
        return torch.randint(-60, 60, (n,), generator=g).to(dtype)
    if special:
        q = torch.tensor([0.0, -0.0, 1.0, -1.0, 2.0, float("inf"), float("-inf"), float("nan")], dtype=torch.float64)
        w = torch.tensor([4, 4, 3, 3, 3, 1, 1, 1], dtype=torch.float)
        return q[torch.multinomial(w, n, replacement=True, generator=g)].to(dtype)
    x = torch.randn(n, generator=g, dtype=torch.float64)
    z = torch.rand(n, generator=g) < 0.05
    return torch.where(z, torch.where(torch.rand(n, generator=g) < 0.5, -0.0, 0.0), x).to(dtype)


VALUE_CASES = ["shuffled, 1-3 copies", "a run of 2^17 duplicates", "M = N = 2^26, E = 4097",
               "rows / cols at 2^31 - 1, 2^31, 2^32 - 1 (M = N = 2^32)", "E = 1"]


@pytest.mark.parametrize("dtype", ALL_DTYPES, ids=DT_ID.get)
def test_coalesce_values(oracle, dtype):
    """All four reductions, D in {1, 3, 33}, bit for bit against the oracle (the kernel adds each run in input order,
    as the oracle does; bf16 / f16 against the fp32 oracle on the widened values, rounded once), the arg of min / max
    included. Special values for floats: runs of +-0, ties, +-inf, NaN first and later in a run."""
    g = torch.Generator().manual_seed(21)
    for name in VALUE_CASES:
        row, col, M, N, _ = coalesce_cases()[name]
        co = Coalesced(row, col, M, N)
        E = row.numel()
        Ds = (1, 3, 33) if E < 100_000 else (1, 3)
        for D in Ds:
            for special in ((False, True) if dtype.is_floating_point else (False,)):
                v = coalesce_values(E * D, dtype, g, special).reshape(E, D) if D > 1 else \
                    coalesce_values(E, dtype, g, special)
                for reduce in REDUCES:
                    what = f"{name} {dtype} D={D} {reduce}{' special' if special else ''}"
                    ref, arg = oracle_coalesce_values(oracle, row, col, v, reduce)
                    out = co.emit(v, reduce, outs=("row", "arg"))
                    assert_same(out["value"].reshape(ref.shape), ref, what)
                    if reduce in ("min", "max"):
                        assert torch.equal(out["arg"].reshape(arg.shape), arg), what
                    else:
                        assert out["arg"].eq(SENTINEL).all(), what + ": arg written for " + reduce
                    if reduce in ("sum", "mean") and dtype.is_floating_point:
                        assert not bool(torch.signbit(out["value"][out["value"] == 0]).any()), what + ": -0"


def test_coalesce_signed_zero_runs(oracle):
    """Runs of -0 and of mixed +-0 sum (and average) to +0, single entries included, through the C-ABI and through
    ops.coalesce; a run of -0 keeps -0 for min / max."""
    z = -0.0
    runs = [[z], [0.0], [z, z], [z, 0.0], [0.0, z], [z] * 40, [1.5, z], [z, -1.0, 1.0]]
    value = torch.tensor([x for r in runs for x in r])
    row = torch.repeat_interleave(torch.arange(len(runs)), torch.tensor([len(r) for r in runs]))
    g = torch.Generator().manual_seed(22)
    p = torch.randperm(row.numel(), generator=g)
    row, value = row[p], value[p]
    col = torch.zeros_like(row)
    for dtype in FLOATS:
        v = value.to(dtype)
        co = Coalesced(row, col, len(runs), 1)
        for reduce in REDUCES:
            ref, _ = oracle_coalesce_values(oracle, row, col, v, reduce)
            got = co.emit(v, reduce, outs=())["value"]
            assert_same(got, ref, f"{dtype} {reduce}")
            _, _, got2 = ops.coalesce(row.to(DEV), col.to(DEV), v.to(DEV), len(runs), 1, reduce)
            assert_same(got2, ref, f"ops.coalesce {dtype} {reduce}")
            if reduce in ("sum", "mean"):
                assert not bool(torch.signbit(got).any()), (dtype, reduce, got)
            else:
                assert bool(torch.signbit(got[5])), (dtype, reduce, "min / max of a run of -0 is -0")


def test_coalesce_d0_and_no_value():
    """D = 0 writes no value (the output guards and the row' / col' stay right); value_in NULL emits the structure."""
    row, col, M, N, _ = coalesce_cases()["shuffled, 1-3 copies"]
    co = Coalesced(row, col, M, N)
    ref = co.emit(outs=("row", "col"))
    out = co.emit(torch.empty(row.numel(), 0), "sum", outs=("row", "col", "arg"))
    assert out["value"].numel() == 0 and torch.equal(out["row"], ref["row"]) and torch.equal(out["col"], ref["col"])
    assert bool(out["arg"].eq(SENTINEL).all())


def test_coalesce_key_wider_than_64_bits():
    """M * N > 2^64 would wrap row * N + col: refused; M * N = 2^64 (keys up to 2^64 - 1) is accepted."""
    row = torch.tensor([0, (1 << 32) - 1], device=DEV)
    col = torch.tensor([0, (1 << 32) - 1], device=DEV)
    ws = torch.empty(lib.tsb200_coalesce_workspace_bytes(2, 0, 0), dtype=torch.uint8, device=DEV)
    for M, N, want in (((1 << 32) + 1, 1 << 32, ERR_UNSUPPORTED), (1 << 32, (1 << 32) + 1, ERR_UNSUPPORTED),
                       (1 << 62, 5, ERR_UNSUPPORTED), (1 << 32, 1 << 32, 0)):
        assert lib.tsb200_coalesce_sort(_vp(row), _vp(col), 2, M, N, _vp(ws), ws.numel(), None, _stream()) == want, \
            (M, N)
    torch.cuda.synchronize()
    with pytest.raises(Tsb200Error):
        ops.coalesce(row, col, None, (1 << 32) + 1, 1 << 32)
    with pytest.raises(Tsb200Error):
        ops.sort_perm(row.flip(0), col, (1 << 32) + 1, 1 << 32)
    r, c, _ = ops.coalesce(row.flip(0), col.flip(0), None, 1 << 32, 1 << 32)
    assert r.tolist() == [0, (1 << 32) - 1] and c.tolist() == [0, (1 << 32) - 1]


@pytest.mark.parametrize("name", ["shuffled, 1-3 copies", "sorted with duplicates",
                                  "one descending pair past the grid-stride cap",
                                  "rows / cols at 2^31 - 1, 2^31, 2^32 - 1 (M = N = 2^32)"])
def test_sort_perm(oracle, name):
    """ops.sort_perm: None when the input is sorted, else the oracle's stable permutation."""
    row, col, M, N, ran = coalesce_cases()[name]
    p = ops.sort_perm(row.to(DEV), col.to(DEV), M, N)
    if not ran:
        assert p is None
        return
    assert torch.equal(p.cpu(), oracle_coalesce_index(oracle, row, col)[0])


# ---- ptr2ind / ind2ptr -----------------------------------------------------------------------------------------------
def _ptr(lengths):
    p = torch.zeros(len(lengths) + 1, dtype=torch.long)
    p[1:] = torch.as_tensor(lengths, dtype=torch.long).cumsum(0)
    return p


@functools.cache
def ptr2ind_cases():
    g = torch.Generator().manual_seed(23)
    rnd = lambda n, hi=5: torch.randint(0, hi, (n,), generator=g).tolist()  # noqa: E731
    cases = {f"M = {M}": rnd(M) for M in (1, 31, 32, 33, 64, 65)}
    cases["M = 1, 100 entries"] = [100]
    cases["an all-empty 32-row block"] = rnd(32) + [0] * 32 + rnd(33)
    cases["blocks starting / ending with empty rows"] = [0, 0, 0] + rnd(26) + [0, 0, 0] + [0] * 5 + rnd(22) + [0] * 5
    cases["one row of 33, 100 and 1000 in a block"] = [0] * 7 + [33] + [0] * 24 + rnd(10) + [100] + rnd(21) + [1000]
    cases["empty rows then one entry at the end"] = [0] * 95 + [1]
    return cases


@pytest.mark.parametrize("name", list(ptr2ind_cases()))
def test_ptr2ind(oracle, name):
    ptr = _ptr(ptr2ind_cases()[name])
    M, E = ptr.numel() - 1, int(ptr[-1])
    out = Guarded(E, torch.long)
    ptr_d = ptr.to(DEV)
    assert lib.tsb200_ptr2ind(_vp(ptr_d), M, E, _vp(out.t), _stream()) == 0
    torch.cuda.synchronize()
    assert torch.equal(out.get(), oracle.ptr2ind(ptr, E)), name
    assert torch.equal(ops.ind2ptr(out.t, M).cpu(), ptr), name + " (ind2ptr back)"


def test_ptr2ind_past_the_warp_grid():
    """M > sm_count * 32 * 8 blocks of 32 rows: warps loop; entries in rows past the first pass, in the last block,
    and in blocks of the second pass that start and end empty."""
    nblk = warp_cap() + 1000
    M = nblk * 32 - 7
    g = torch.Generator().manual_seed(24)
    lengths = torch.zeros(M, dtype=torch.long)
    rows = torch.randint(M, (200_000,), generator=g)
    lengths[rows] = torch.randint(1, 4, (200_000,), generator=g)
    lengths[warp_cap() * 32 + 40] = 70                             # a long row in the first block of the second pass
    lengths[-3:] = torch.tensor([2, 0, 1])
    ptr = torch.zeros(M + 1, dtype=torch.long)
    ptr[1:] = lengths.cumsum(0)
    E = int(ptr[-1])
    out = Guarded(E, torch.long)
    ptr_d = ptr.to(DEV)
    assert lib.tsb200_ptr2ind(_vp(ptr_d), M, E, _vp(out.t), _stream()) == 0
    torch.cuda.synchronize()
    assert torch.equal(out.get(), torch.repeat_interleave(torch.arange(M), lengths))


def _ind2ptr_call(ind, M):
    out = Guarded(M + 1, torch.long)
    ind_d = ind.to(DEV)
    assert lib.tsb200_ind2ptr(_vp(ind_d) if ind.numel() else None, ind.numel(), M, _vp(out.t), _stream()) == 0
    torch.cuda.synchronize()
    return out.get()


def test_ind2ptr(oracle):
    """E << M, M << E, leading and trailing empty rows, E = 0, and M + 1 past the grid-stride cap."""
    g = torch.Generator().manual_seed(25)
    cases = {
        "E << M": (torch.randint(100_000, (50,), generator=g).sort().values, 100_000),
        "M << E": (torch.randint(5, (100_000,), generator=g).sort().values, 5),
        "leading / trailing empty rows": (torch.randint(40, 60, (500,), generator=g).sort().values, 100),
        "one row": (torch.zeros(77, dtype=torch.long), 1),
        "E = 0": (torch.empty(0, dtype=torch.long), 9),
        "M + 1 past the grid cap": (torch.randint(grid_stride_cap() + 500, (5000,), generator=g).sort().values,
                                    grid_stride_cap() + 500),
    }
    assert cases["M + 1 past the grid cap"][1] + 1 > grid_stride_cap()
    for name, (ind, M) in cases.items():
        assert torch.equal(_ind2ptr_call(ind, M), oracle.ind2ptr(ind, M)), name


# ---- csr2csc ---------------------------------------------------------------------------------------------------------
N_CSC = [1, 2, 3, 4, 5, 255, 256, 257, 4096, 4097, 65_536, 65_537, 1 << 20, (1 << 20) + 1]
N_HUGE_CSC = (1 << 32) - 1
assert {bits_for(n) for n in N_CSC} == {1, 2, 3, 8, 9, 12, 13, 16, 17, 20, 21}


def _csr_for(N, g, M=300, E=3000):
    cols = torch.randint(N, (E,), generator=g)
    cols[:4] = torch.tensor([N - 1, 0, N // 2, N - 1]).clamp(max=N - 1)
    rows = torch.randint(M, (E,), generator=g)
    k = torch.unique(rows * N + cols)                              # row-major sorted, duplicate-free
    return k // N, k % N, M


def _csc_call(row, col, M, N, with_colptr=True, with_row=True):
    E = row.numel()
    nws = lib.tsb200_csr2csc_workspace_bytes(E, M, N)
    ws = torch.empty(max(nws, 1), dtype=torch.uint8, device=DEV)
    perm, row_csc = Guarded(E, torch.long), Guarded(E, torch.long)
    colptr = Guarded(N + 1, torch.long) if with_colptr else None
    rd, cd = row.to(DEV), col.to(DEV)
    rc = lib.tsb200_csr2csc(_vp(rd), _vp(cd), E, M, N, _vp(perm.t), _vp(colptr.t) if colptr else None,
                            _vp(row_csc.t) if with_row else None, _vp(ws), nws, _stream())
    torch.cuda.synchronize()
    if rc != 0:
        return rc
    if not with_row:
        assert row_csc.untouched(0, E)
    return perm.get(), (colptr.get() if colptr else None), (row_csc.get() if with_row else None)


@pytest.mark.parametrize("N", N_CSC + [N_HUGE_CSC])
def test_csr2csc(oracle, N):
    """The permutation, colptr and row_csc bit for bit against oracle.csr2csc / ind2ptr at N on both sides of the
    sort's bit boundaries (it sorts ceil(log2 N) bits), with columns at 0 and N - 1; colptr and row_csc also NULL.
    N = 2^32 - 1: columns at 2^31 - 1, 2^31 and 2^32 - 2 (colptr would be 32 GB: NULL only)."""
    g = torch.Generator().manual_seed(26 + N % 1000)
    if N == N_HUGE_CSC:
        big = torch.tensor([0, 12345, (1 << 31) - 1, 1 << 31, N - 2, N - 1])
        M = 40
        key = torch.unique(torch.randint(M, (400,), generator=g) * 8 + torch.randint(6, (400,), generator=g))
        row, col = key // 8, big[key % 8]
    else:
        row, col, M = _csr_for(N, g)
    assert int(col.max()) == N - 1
    uc = torch.unique(col)
    perm = oracle.csr2csc(row, torch.searchsorted(uc, col), M)
    colptr = oracle.ind2ptr(col[perm], N) if N != N_HUGE_CSC else None
    for with_colptr in ((True, False) if N != N_HUGE_CSC else (False,)):
        for with_row in (True, False):
            p, cp, rcsc = _csc_call(row, col, M, N, with_colptr, with_row)
            assert torch.equal(p, perm), (N, with_colptr, with_row)
            if with_colptr:
                assert torch.equal(cp, colptr), N
            if with_row:
                assert torch.equal(rcsc, row[perm]), N


def test_csr2csc_edges():
    """E = 0 zeroes colptr (and writes nothing else); N = 2^32 is refused."""
    e = torch.empty(0, dtype=torch.long)
    _, cp, _ = _csc_call(e, e, 5, 17)
    assert cp.tolist() == [0] * 18
    row, col = torch.tensor([0, 1]), torch.tensor([3, 1])
    assert _csc_call(row, col, 2, 1 << 32, with_colptr=False) == ERR_UNSUPPORTED


# ---- segment reduce --------------------------------------------------------------------------------------------------
SEG_LENGTHS = [0, 1, 2, 31, 32, 33, 63, 64, 65, 1000, 0, 100_003, 3, 0]
TIE_LEN = 100                     # tie segments: equal extremes at positions j, j + 1, j + 32 (j = 5, 31)


@functools.cache
def segment_case():
    """Pointers over SEG_LENGTHS, four tie segments, and random short segments -> (ptr, tie segment ids)."""
    g = torch.Generator().manual_seed(27)
    lengths = list(SEG_LENGTHS)
    ties = []
    for _ in range(4):
        ties.append(len(lengths))
        lengths.append(TIE_LEN)
    lengths += torch.randint(0, 40, (200,), generator=g).tolist()
    return _ptr(lengths), ties


def segment_values(ptr, ties, D, dtype, g):
    """randn (5 % signed zeros) or integers in [-50, 50); in the tie segments -64 (min) at j, j + 1, j + 32 of
    segments 0, 1 and +64 (max) at the same positions of segments 2, 3, for j = 5 / 31."""
    E = int(ptr[-1])
    if dtype.is_floating_point:
        x = torch.randn(E, D, generator=g, dtype=torch.float64)
        z = torch.rand(E, D, generator=g) < 0.05
        x = torch.where(z, torch.where(torch.rand(E, D, generator=g) < 0.5, -0.0, 0.0), x)
    else:
        x = torch.randint(-50, 50, (E, D), generator=g).double()
    for k, s in enumerate(ties):
        j = int(ptr[s]) + (5 if k % 2 == 0 else 31)
        x[[j, j + 1, j + 32]] = -64.0 if k < 2 else 64.0
    return x.to(dtype)


def oracle_minmax(oracle, ptr, v, reduce, perm):
    wide = v.float() if v.dtype in (torch.bfloat16, torch.float16) else v
    out, arg = oracle.segment_reduce(ptr, wide, reduce, perm=perm, return_arg=True)
    return out.to(v.dtype), arg


def call_segment_reduce(ptr, v, reduce, perm=None, with_arg=True):
    S = ptr.numel() - 1
    D = v.size(1) if v.dim() > 1 else 1
    out = Guarded(S * D, v.dtype)
    arg = Guarded(S * D, torch.long) if with_arg else None
    vd = v.to(DEV).contiguous()
    ptr_d, perm_d = ptr.to(DEV), (perm.to(DEV) if perm is not None else None)
    rc = lib.tsb200_segment_reduce(_vp(ptr_d), _vp(perm_d), _vp(vd),
                                   _vp(out.t), _vp(arg.t) if arg else None, S, D, ops._dtype_code(v.dtype), RED[reduce],
                                   _stream())
    assert rc == 0, rc
    torch.cuda.synchronize()
    o = out.get().reshape((S,) + tuple(v.shape[1:]))
    a = arg.get().reshape(o.shape) if arg else None
    return o, a


def check_segment_reduce(oracle, ptr, v, reduce, perm, what):
    out, arg = call_segment_reduce(ptr, v, reduce, perm)
    if reduce in ("min", "max"):
        ref, ref_arg = oracle_minmax(oracle, ptr, v, reduce, perm)
        assert_same(out, ref, what)
        assert torch.equal(arg, ref_arg), what + ": arg"
    else:
        assert bool(arg.eq(SENTINEL).all()), what + ": arg written for " + reduce
        if v.dtype.is_floating_point:
            ref, bound = segment_sum_ref_bound(oracle, ptr, v, perm, mean=reduce == "mean")
            assert_spspmm_values(out, ref, bound, what)
        else:
            assert_same(out, oracle.segment_reduce(ptr, v, reduce, perm=perm), what)
    return out, arg


@pytest.mark.parametrize("dtype", ALL_DTYPES, ids=DT_ID.get)
def test_segment_reduce(oracle, dtype):
    """All four reductions, D in {1, 3, 33}, with and without perm, over segments of 0, 1, 2, 31, 32, 33, 63, 64, 65,
    1000 and 100003 entries: min / max and integers bit for bit with the arg (-1 for empty segments), sums within the
    rounding bound, exactly +0 where every entry is 0 (and for empty segments)."""
    ptr, ties = segment_case()
    E = int(ptr[-1])
    g = torch.Generator().manual_seed(28)
    for D in (1, 3, 33):
        v = segment_values(ptr, ties, D, dtype, g)
        v = v.view(-1) if D == 1 else v
        perm = torch.randperm(E, generator=g)
        vp = torch.empty_like(v)
        vp[perm] = v                      # through perm, the segments hold the same entries in the same order
        for reduce in REDUCES:
            what = f"{dtype} D={D} {reduce}"
            out, arg = check_segment_reduce(oracle, ptr, v, reduce, None, what)
            outp, argp = check_segment_reduce(oracle, ptr, vp, reduce, perm, what + " perm")
            if reduce in ("min", "max"):
                assert_same(outp, out, what + " perm vs no perm")
                assert torch.equal(argp, torch.where(arg >= 0, perm[arg.clamp(min=0)], arg)), what
                for s, j in zip(ties[:2] if reduce == "min" else ties[2:], (5, 31)):
                    assert bool((arg[s] == int(ptr[s]) + j).all()), (what, "tie at", j, arg[s])


def test_segment_reduce_past_the_warp_grid(oracle):
    """S > sm_count * 32 * 8 segments: each warp loops over segments; f32 and i64, D = 3."""
    S = warp_cap() + 777
    g = torch.Generator().manual_seed(29)
    ptr = _ptr(torch.randint(0, 6, (S,), generator=g).tolist())
    E = int(ptr[-1])
    for dtype in (torch.float32, torch.int64):
        v = (torch.randn(E, 3, generator=g) * 10).to(dtype)
        for reduce in REDUCES:
            check_segment_reduce(oracle, ptr, v, reduce, None, f"S={S} {dtype} {reduce}")


NAN = float("nan")
INF = float("inf")
SPECIAL_SEGMENTS = {
    "NaN at 1, minimum at 17 (40)": [float(i) for i in range(40)],
    "NaN first (40)": [NAN] + [float(i) for i in range(39)],
    "NaN at every later lane start (64)": [5.0] + [NAN] * 31 + [float(-i) for i in range(32)],
    "NaN at 33 (70)": [float(i % 7) for i in range(70)],
    "all NaN but the first (40)": [3.0] + [NAN] * 39,
    "-0 x 1": [-0.0], "-0 x 2": [-0.0, -0.0], "-0 x 40": [-0.0] * 40, "+0, -0": [0.0, -0.0], "-0, +0": [-0.0, 0.0],
    "-0 x 33 then +0": [-0.0] * 33 + [0.0],
    "+-inf": [INF, 1.0, -INF, 2.0], "inf, 1": [1.0, INF] * 20, "-inf only": [-INF] * 35,
    "ties at 0, 1, 32": [1.0, 1.0] + [2.0] * 30 + [1.0, 2.0],
}
SPECIAL_SEGMENTS["NaN at 1, minimum at 17 (40)"][1] = NAN
SPECIAL_SEGMENTS["NaN at 1, minimum at 17 (40)"][17] = -100.0
SPECIAL_SEGMENTS["NaN at 33 (70)"][33] = NAN


@pytest.mark.parametrize("reduce", REDUCES)
@pytest.mark.parametrize("dtype", FLOATS, ids=DT_ID.get)
def test_segment_reduce_nan_signed_zero_inf(oracle, dtype, reduce):
    """Bit for bit against the oracle: min / max compare strictly from the segment's first entry (NaN there is the
    result, a NaN elsewhere never is, whichever lane meets it first), sums of -0 runs are +0, +-inf propagate; every
    value here is exact, so the sum order cannot matter. Also as a duplicate run of coalesce."""
    names = list(SPECIAL_SEGMENTS)
    ptr = _ptr([len(SPECIAL_SEGMENTS[k]) for k in names])
    v = torch.tensor([x for k in names for x in SPECIAL_SEGMENTS[k]], dtype=torch.float64).to(dtype)
    E = v.numel()
    g = torch.Generator().manual_seed(30)
    perm = torch.randperm(E, generator=g)
    vp = torch.empty_like(v)
    vp[perm] = v
    row = torch.repeat_interleave(torch.arange(len(names)), ptr[1:] - ptr[:-1])
    co = Coalesced(row, torch.zeros_like(row), len(names), 1)
    for pv, pp in ((v, None), (vp, perm)):
        out, arg = call_segment_reduce(ptr, pv, reduce, pp)
        wide = pv.float() if dtype in (torch.bfloat16, torch.float16) else pv
        ref, ref_arg = oracle.segment_reduce(ptr, wide, reduce, perm=pp, return_arg=True)
        what = f"{dtype} {reduce} perm={pp is not None}"
        for i, k in enumerate(names):
            assert_same(out[i:i + 1], ref[i:i + 1].to(dtype), f"{what} segment '{k}'")
            if reduce in ("min", "max"):
                assert int(arg[i]) == int(ref_arg[i]), f"{what} segment '{k}': arg {int(arg[i])} vs {int(ref_arg[i])}"
    cref, carg = oracle_coalesce_values(oracle, row, torch.zeros_like(row), v, reduce)
    cout = co.emit(v, reduce, outs=("arg",))
    assert_same(cout["value"], cref, f"coalesce {dtype} {reduce}")
    if reduce in ("min", "max"):
        assert torch.equal(cout["arg"], carg)
    seg_out, _ = call_segment_reduce(ptr, v, reduce)
    assert_same(seg_out, cout["value"], f"segment_reduce vs coalesce {dtype} {reduce}")
    if reduce == "min":
        i = names.index("NaN at 1, minimum at 17 (40)")
        out, arg = call_segment_reduce(ptr, v, "min")
        assert float(out[i]) == -100.0 and int(arg[i]) == int(ptr[i]) + 17


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.int64], ids=DT_ID.get)
def test_row_reductions_equal_coalesce(oracle, dtype):
    """SparseTensor.min / max / sum(dim=1) against coalesce(row, zeros, value, op) on the same entries: min / max bit
    for bit, sum within the rounding bound of both (integers exact)."""
    g = torch.Generator().manual_seed(31)
    M, N = 500, 300
    lengths = torch.randint(0, 70, (M,), generator=g)
    lengths[::17] = 0
    ptr = _ptr(lengths.tolist())
    E = int(ptr[-1])
    row = torch.repeat_interleave(torch.arange(M), lengths)
    col = torch.cat([torch.randperm(N, generator=g)[:int(n)].sort().values for n in lengths])
    v = segment_values(ptr, [], 2, dtype, g)
    a = ts.SparseTensor(row=row.to(DEV), col=col.to(DEV), value=v.to(DEV), sparse_sizes=(M, N))
    nonempty = lengths > 0
    for op in ("sum", "min", "max"):
        got = getattr(ts, op)(a, 1).cpu()
        r, _, cv = ops.coalesce(row.to(DEV), torch.zeros(E, dtype=torch.long, device=DEV), v.to(DEV), M, 1, op)
        assert torch.equal(r.cpu(), nonempty.nonzero().view(-1))
        if op == "sum" and dtype.is_floating_point:
            ref, bound = segment_sum_ref_bound(oracle, ptr, v)
            assert_spspmm_values(got, ref, bound, f"{dtype} sum(dim=1)")
            assert_spspmm_values(cv.cpu(), ref[nonempty], bound[nonempty], f"{dtype} coalesce sum")
        else:
            assert_same(got[nonempty], cv.cpu(), f"{dtype} {op}(dim=1) vs coalesce")
            assert bool((got[~nonempty] == 0).all()), f"{dtype} {op}(dim=1): empty rows"


# ---- segment reduce backward -----------------------------------------------------------------------------------------
def call_segment_reduce_bw(seg, count, arg, grad_out, E, reduce):
    S = grad_out.size(0)
    D = grad_out.numel() // max(S, 1)
    gin = Guarded(E * D, grad_out.dtype)
    grad_out = grad_out.contiguous()
    rc = lib.tsb200_segment_reduce_bw(_vp(seg), _vp(count), _vp(arg), _vp(grad_out), _vp(gin.t), E, S,
                                      D, ops._dtype_code(grad_out.dtype), RED[reduce], _stream())
    torch.cuda.synchronize()
    return rc, gin


def bw_inputs(source, reduce, dtype, D, g):
    """(seg, count, arg, E, S, value) as the forward that feeds the backward leaves them: the coalesce emit, or the
    row (dim=1) / column (dim=0) reduction of reduce.py (segment reduce over rowptr, or over colptr through csr2csc)."""
    if source == "coalesce":
        E, M, N = 3000, 40, 30
        row, col = torch.randint(M, (E,), generator=g), torch.randint(N, (E,), generator=g)
        v = torch.randint(-4, 5, (E, D), generator=g).to(dtype).squeeze(1)     # small integers: many ties
        _, _, vo, bw = ops._coalesce_raw(row.to(DEV), col.to(DEV), v.to(DEV), M, N, reduce, want_bw=True)
        seg, count, arg = bw
        return seg, count, arg, E, vo.size(0), (row, col, v, N)
    M, N = 200, 150
    lengths = torch.randint(0, 30, (M,), generator=g)
    row = torch.repeat_interleave(torch.arange(M), lengths)
    col = torch.cat([torch.randperm(N, generator=g)[:int(n)].sort().values for n in lengths])
    E = row.numel()
    v = torch.randint(-4, 5, (E, D), generator=g).to(dtype).squeeze(1)
    a = ts.SparseTensor(row=row.to(DEV), col=col.to(DEV), value=v.to(DEV), sparse_sizes=(M, N))
    st = a.storage
    if source == "dim1":
        ptr, perm, seg = st.rowptr(), None, st.row()
    else:
        ptr, perm, seg = st.colptr(), st.csr2csc(), st.col()
    _, arg = ops._segment_reduce_raw(ptr, v.to(DEV), reduce, perm, want_arg=True)
    count = ptr[1:] - ptr[:-1]
    return seg, (count if reduce == "mean" else None), arg, E, ptr.numel() - 1, None


@pytest.mark.parametrize("source", ["coalesce", "dim1", "dim0"])
@pytest.mark.parametrize("dtype", FLOATS, ids=DT_ID.get)
def test_segment_reduce_bw(oracle, dtype, source):
    """Bit for bit: sum = grad_out[seg]; mean = (grad_out[seg] / count[seg]) in the accumulator dtype, rounded once;
    min / max = grad_out[seg] at the arg entry, 0 elsewhere. For coalesce in f64 also against oracle.coalesce_value_bw.
    D in {1, 3}; every element of grad_in is written, nothing outside it."""
    g = torch.Generator().manual_seed(32)
    for D in (1, 3):
        for reduce in REDUCES:
            seg, count, arg, E, S, small = bw_inputs(source, reduce, dtype, D, g)
            grad_out = torch.randn(S, D, generator=g, dtype=torch.float64).to(dtype)
            rc, gin = call_segment_reduce_bw(seg, count, arg, grad_out.to(DEV), E, reduce)
            assert rc == 0, rc
            got = gin.get().reshape(E, D)
            s = seg.cpu()
            go = grad_out[s]
            if reduce == "sum":
                want = go
            elif reduce == "mean":
                acc = torch.float64 if dtype == torch.float64 else torch.float32
                want = (go.to(acc) / count.cpu()[s].clamp(min=1).to(acc).view(-1, 1)).to(dtype)
            else:
                hit = arg.cpu().reshape(S, D)[s] == torch.arange(E).view(-1, 1)
                want = torch.where(hit, go, torch.zeros_like(go))
                assert int(hit.sum()) == int((arg.cpu() >= 0).sum())        # one entry per non-empty (segment, d)
            what = f"{source} {dtype} D={D} {reduce}"
            assert_same(got, want, what)
            if small is not None and dtype == torch.float64:
                row, col, v, N = small
                ref = oracle.coalesce_value_bw(row, col, v, N, "add" if reduce == "sum" else reduce,
                                               grad_out.reshape((S,) + tuple(v.shape[1:])))
                assert torch.equal(got.reshape(ref.shape), ref), what + " vs oracle"


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64], ids=DT_ID.get)
def test_segment_reduce_bw_refuses_integers(dtype):
    seg = torch.zeros(4, dtype=torch.long, device=DEV)
    grad_out = torch.ones(1, 2, dtype=dtype, device=DEV)
    for reduce in REDUCES:
        count = torch.tensor([4], device=DEV)
        arg = torch.zeros(1, 2, dtype=torch.long, device=DEV)
        rc, gin = call_segment_reduce_bw(seg, count, arg, grad_out, 4, reduce)
        assert rc == ERR_UNSUPPORTED, (dtype, reduce, rc)
        assert gin.untouched(-GUARD, 4 * 2 + GUARD), "written without a launch"
