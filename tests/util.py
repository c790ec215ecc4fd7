"""Shared generators / comparison helpers for the parity tests."""
import torch


def random_csr(M, N, avg_deg, seed, power_law=False, empty_rows=(), long_rows=(), device="cpu"):
    """Random CSR structure: sorted unique columns per row; optional power-law degrees, forced empty
    rows and forced long rows [(row, degree)]."""
    g = torch.Generator().manual_seed(seed)
    if power_law:
        u = torch.rand(M, generator=g).clamp_(min=1e-6)
        deg = (avg_deg / 3.0 * u.pow(-1 / 1.5)).floor().long().clamp_(max=N)
    else:
        deg = torch.poisson(torch.full((M,), float(avg_deg)), generator=g).long().clamp_(max=N)
    for r in empty_rows:
        deg[r] = 0
    for r, d in long_rows:
        deg[r] = min(d, N)
    rows, cols = [], []
    for m in range(M):
        d = int(deg[m])
        if d == 0:
            continue
        c = torch.randperm(N, generator=g)[:d].sort().values
        rows.append(torch.full((d,), m, dtype=torch.long))
        cols.append(c)
    row = torch.cat(rows) if rows else torch.empty(0, dtype=torch.long)
    col = torch.cat(cols) if cols else torch.empty(0, dtype=torch.long)
    rowptr = torch.zeros(M + 1, dtype=torch.long)
    rowptr[1:] = torch.cumsum(deg, 0)
    return row.to(device), rowptr.to(device), col.to(device)


def fast_random_csr(M, N, avg_deg, seed, device):
    """Large uniform random CSR generated on `device` (SURVEY §8d G2 recipe): E0 = avg_deg*M random
    (row, col) pairs, sorted + deduplicated."""
    g = torch.Generator(device=device).manual_seed(seed)
    E0 = int(avg_deg * M)
    row = torch.randint(M, (E0,), generator=g, device=device)
    col = torch.randint(N, (E0,), generator=g, device=device)
    key = torch.unique(row * N + col)  # sorted
    row, col = key // N, key % N
    rowptr = torch.zeros(M + 1, dtype=torch.long, device=device)
    rowptr[1:] = torch.cumsum(torch.bincount(row, minlength=M), 0)
    return row, rowptr, col


def rel_err_bound(out, ref, absmax):
    """max |out - ref| / max(|A||B| normaliser)"""
    return ((out.double() - ref.double()).abs() / absmax.double().clamp_min(1e-30)).max().item()


# ---- SpSpMM against the oracle -------------------------------------------------------------------------------------
ORACLE_MAX_N = 1 << 20   # wider B: the oracle runs on B's columns relabelled 0..U-1 (its arrays are N long)


def oracle_spspmm(oracle, rpa, ca, va, rpb, cb, vb, M, Kd, N, want_value=True):
    """oracle.spspmm; for N > ORACLE_MAX_N on B's distinct columns relabelled 0..U-1 in order and mapped back (an
    order-preserving relabelling changes neither the structure nor any sum)."""
    if N <= ORACLE_MAX_N:
        return oracle.spspmm(rpa, ca, va, rpb, cb, vb, M, Kd, N, want_value)
    cb = cb.cpu()
    uniq = torch.unique(cb)
    rp, r, c, v = oracle.spspmm(rpa, ca, va, rpb, torch.searchsorted(uniq, cb), vb, M, Kd, max(uniq.numel(), 1),
                                want_value)
    return rp, r, uniq[c], v


def spspmm_ref_bound(oracle, rpa, ca, va, rpb, cb, vb, M, Kd, N, dtype):
    """Reference values of C = A @ B and the per-entry error bound of a kernel that forms each product in `dtype` and
    adds it with one rounding (atomics in any order): n products per entry, S = sum |a||b| (oracle on |A|, |B|)
      fp32: |v - ref64| <= (n + 1) 2^-24 S   against the oracle on the inputs cast to fp64 (exact products)
      fp64: |v - ref|   <= 2 (n + 1) 2^-53 S against the oracle in fp64
    None stands for all-ones values. Entries with S = 0 must be exactly +0."""
    ones = lambda t, n: torch.ones(n, dtype=torch.float64) if t is None else t.cpu().double()  # noqa: E731
    a, b = ones(va, ca.numel()), ones(vb, cb.numel())
    args = (M, Kd, N)
    ref = oracle_spspmm(oracle, rpa, ca, a, rpb, cb, b, *args)[3]
    S = oracle_spspmm(oracle, rpa, ca, a.abs(), rpb, cb, b.abs(), *args)[3]
    n = oracle_spspmm(oracle, rpa, ca, torch.ones_like(a), rpb, cb, torch.ones_like(b), *args)[3]
    u = 2.0 ** -24 if dtype == torch.float32 else 2.0 * 2.0 ** -53
    return ref, (n + 1) * u * S


def assert_spspmm_values(v, ref, bound, what="", where=None):
    """|v - ref| <= bound elementwise, and every entry with bound 0 (no non-zero product) is +0, bit for bit.
    `where(bad)` may describe the failing entries (a boolean mask) in the message."""
    v = v.cpu()
    err = (v.double() - ref).abs()
    ok = (err <= bound) & ~((bound == 0) & ((v != 0) | torch.signbit(v)))
    if not bool(ok.all()):
        i = int((~ok).nonzero()[0])
        raise AssertionError(f"{what}: {int((~ok).sum())} of {v.numel()} values out of bound, first at {i}: "
                             f"{v[i].item()!r} vs {ref[i].item()!r} (bound {bound[i].item():.3e})"
                             + (f"; {where(~ok)}" if where else ""))


_STORE_U = {torch.bfloat16: (2.0 ** -8, 2.0 ** -134), torch.float16: (2.0 ** -11, 2.0 ** -25)}


def segment_sum_ref_bound(oracle, ptr, value, perm=None, mean=False):
    """Reference values of a segment sum (or mean) and the per-entry error bound of a kernel that adds the segment's
    n entries in any order in its accumulator (fp32 for fp32 / bf16 / f16, fp64 for fp64), divides once for the mean
    and rounds once to the storage dtype. Against the oracle in fp64 on the values widened, with S = sum |v|:
      sum : (n + 1) 2^-24 S (fp32 accumulator) or 2 (n + 1) 2^-53 S (fp64)
      mean: (n + 2) u S / n (one more rounding, by the division)
      bf16 / f16: plus 1/2 ulp of the storage dtype (relative 2^-8 / 2^-11 of the result, or half its smallest
      subnormal). Entries with S = 0 (empty segments, all-zero segments) must be exactly +0."""
    ptr, v = ptr.cpu(), value.cpu().double()
    op = "mean" if mean else "sum"
    ref = oracle.segment_reduce(ptr, v, op, perm=perm)
    S = oracle.segment_reduce(ptr, v.abs(), "sum", perm=perm)
    n = (ptr[1:] - ptr[:-1]).double().view((-1,) + (1,) * (v.dim() - 1))
    u = 2.0 * 2.0 ** -53 if value.dtype == torch.float64 else 2.0 ** -24
    bound = ((n + 2) * u * S / n.clamp(min=1)) if mean else ((n + 1) * u * S)
    if value.dtype in _STORE_U:
        rel, sub = _STORE_U[value.dtype]
        bound = bound + torch.where(S > 0, rel * (ref.abs() + bound) + sub, torch.zeros_like(S))
    return ref, bound


def launched_kernels(fn, pattern=None):
    """Names of the kernels `fn` launches. A profiling session that delivers no kernel record at all, or none whose
    name matches the regular expression `pattern` (with a list of expressions: none for one of them), is repeated:
    every call profiled here launches such kernels, and the profiler now and then drops a record."""
    import re
    from torch.profiler import ProfilerActivity, profile
    patterns = [] if pattern is None else [pattern] if isinstance(pattern, str) else list(pattern)
    names = []
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if "kernel" in e.name]
        if names and all(any(re.search(p, n) for n in names) for p in patterns):
            return names
    raise AssertionError(f"the profiler recorded no kernel{'' if pattern is None else ' matching ' + pattern}: {names}")
