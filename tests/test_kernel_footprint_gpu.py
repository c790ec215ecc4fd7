"""Where every SpMM-family kernel writes: nothing outside its outputs and workspace, every output element it promises,
the same bits from a reused workspace or plan as from a zeroed one, and no byte of an input changed.

Each output, workspace and plan lives inside one uint8 device buffer between two GUARD-byte zones of the byte PAT,
compared byte for byte after the call. An output starts at exactly the alignment the ABI requires and no more (16 B
rows and arg_out on the vector paths, 4 B scales, the element size on the generic paths, placed at that offset mod 256)
and is filled with SENT bytes: all-ones is a NaN no kernel computes (the GPU's NaN is positive) and -1 as an index, so
an element still all SENT was not written. Workspaces and plans are exactly their `*_bytes` size, 256-byte aligned.

Every case runs the entry point three times on the same workspace: (a) zero-filled, (b) after a call of the same
entry point on another matrix of the same shape and nnz (the degrees of the first in reverse order), which leaves the
bytes the caching allocator would hand back, and (c) once more. The three results must be bit-identical, bit-identical
to the existing tests' unguarded call, and within the fp64 reference bound those tests use. The inputs (structure,
values, operands, scales, residuals, arg_out, grad_out, plans) are snapshotted on the CPU before and compared after.

The segment-queue counters are read back from the unplanned workspace on the worst-case degree patterns derived in
test_kernel_footprint_cpu.py and compared with the Python restatement of the deferral rule.
"""
import ctypes

import pytest
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import ops
from pytorch_sparse_b200._lib import lib
from test_heads_gpu import CASES as HEAD_CASES, spmm_ref as heads_ref, sddmm_ref as heads_sddmm_ref, unaligned
from test_heads_gpu import call_sddmm as call_sddmm_heads, call_spmm as call_spmm_heads
from test_kernel_footprint_cpu import (BUDGET_WINDOW, capacities, planned_ws, plan_layout, queue_counts, worst_budget,
                                       worst_long, worst_mixed, ws_layout)
from test_quantize_fp8_gpu import assert_same_bits, make_rows
from test_sddmm_gpu import expected_bits, fp8_operand, fp8_scale, replay as sddmm_fp8_replay
from test_softmax_gpu import assert_backward, assert_forward, c_call as softmax_unguarded, scores, structured
from test_spmm_backward_kernels_gpu import (call_minmax_bw, call_value_bw, check_accumulated, check_value_bw,
                                            sddmm_family)
from test_spmm_fp8_gpu import KS, KS_PARTIAL, Replay, call_fp8, make_scale, make_values, make_x8
from test_spmm_fp8_gpu import mat as fp8_mat  # noqa: F401
from test_spmm_kernels_gpu import (DEV, FAMILIES, NAN_ROWS, TABLE, U32, Ref, _id, assert_bits_equal, assert_sum_bound,
                                   call_fw, call_planned, dense, family_of, large, small, sub_csr, values)  # noqa: F401
from test_spmm_res_gpu import call_res as call_res_unguarded, ref_bound as res_ref_bound, assert_bound

pytestmark = pytest.mark.gpu
GUARD = 4096          # wider than a column tile's row store (32 lanes x 4 x 16 B = 2 KiB: what a tile that ignored the
PAT = 0xA5            # column bound could write past the last row) and the index ring's reach of 64 entries
SENT = 0xFF
ENV = "TSB200_SPMM_ITEM_SHIFT"
E4M3 = torch.float8_e4m3fn
SUM, MEAN, MIN, MAX = 0, 1, 2, 3
RED = {"sum": SUM, "mean": MEAN, "min": MIN, "max": MAX}


# ---- guarded buffers ---------------------------------------------------------------------------------------------------
class Guarded:
    """`nbytes` bytes at an address of exactly `align` mod 256 (0: 256-aligned), between two GUARD-byte zones of PAT,
    in one uint8 device buffer (the caching allocator hands out 512-byte aligned blocks)."""

    def __init__(self, nbytes, align, fill=SENT):
        self.off, self.n = GUARD + align, nbytes
        self.raw = torch.full((self.off + nbytes + GUARD,), PAT, dtype=torch.uint8, device=DEV)
        assert self.raw.data_ptr() % 512 == 0
        self.body = self.raw[self.off:self.off + nbytes]
        if fill is not None:
            self.body.fill_(fill)

    @property
    def p(self):
        return ctypes.c_void_p(self.raw.data_ptr() + self.off)

    def t(self, dtype, shape):
        return self.body.view(dtype).view(shape)

    def check_guards(self, what):
        lo, hi = self.raw[:self.off].cpu(), self.raw[self.off + self.n:].cpu()
        for zone, name, rel in ((lo, "before", lambda i: self.off - i), (hi, "past the end", lambda i: i + 1)):
            bad = (zone != PAT).nonzero().view(-1)
            if bad.numel():
                i = int(bad[0] if name == "past the end" else bad[-1])
                raise AssertionError(f"{what}: {bad.numel()} guard bytes {name} overwritten, nearest {rel(i)} bytes "
                                     f"{name} (0x{int(zone[i]):02x})")


class Out:
    """An output of `dtype` and `shape` at exactly `align`; `full`: the ABI promises every element is written."""

    def __init__(self, dtype, shape, align, full=True, fill=SENT):
        self.dtype, self.shape, self.align, self.full, self.fill = dtype, tuple(shape), align, full, fill
        es = torch.empty(0, dtype=dtype).element_size()
        self.nbytes = es * int(torch.Size(self.shape).numel())
        self.es = es

    def make(self):
        return Guarded(self.nbytes, self.align, self.fill)


def unwritten(g, es):
    """Elements of a guarded output still holding only SENT bytes."""
    return (g.body.view(-1, es) == SENT).all(1) if g.n else torch.zeros(0, dtype=torch.bool, device=DEV)


def snapshot(tensors):
    return [None if t is None else t.detach().reshape(-1).view(torch.uint8).cpu().clone() if t.numel() else None
            for t in tensors]


def same_bytes(a, b):
    return a.n == b.n and torch.equal(a.body, b.body)


def footprint(launch, outs, ws_bytes, main, other, inputs, what, reruns_equal=True, guarded_inputs=()):
    """Runs launch(args, outs, ws) for (a) main in zeroed workspaces, (b) other then main, (c) main again; checks every
    guard (those around the Guarded inputs, i.e. plans, included), the promised writes, the reruns' bits (unless the
    kernel accumulates with atomics in any order) and the inputs; returns run (a)'s outputs as typed tensors."""
    ws = {k: Guarded(n, 0, fill=0) for k, n in ws_bytes.items()}
    before = snapshot(inputs)
    runs = []
    for tag, args in (("a", main), ("other", other), ("b", main), ("c", main)):
        if args is None:
            continue
        o = {k: s.make() for k, s in outs.items()}
        launch(args, o, ws)
        torch.cuda.synchronize()
        for k, g in o.items():
            g.check_guards(f"{what} [{tag}] {k}")
            if outs[k].full:
                miss = unwritten(g, outs[k].es)
                assert not bool(miss.any()), (f"{what} [{tag}] {k}: {int(miss.sum())} elements not written, first "
                                              f"{int(miss.nonzero()[0])}")
        for k, g in ws.items():
            g.check_guards(f"{what} [{tag}] workspace {k}")
        for i, g in enumerate(guarded_inputs):
            g.check_guards(f"{what} [{tag}] guarded input {i}")
        if tag != "other":
            runs.append(o)
    for o in runs[1:] if reruns_equal else []:
        for k in outs:
            assert same_bytes(o[k], runs[0][k]), f"{what} {k}: a reused workspace changed the result"
    after = snapshot(inputs)
    for i, (x, y) in enumerate(zip(before, after)):
        assert (x is None) == (y is None) and (x is None or torch.equal(x, y)), f"{what}: input {i} was written"
    return {k: runs[0][k].t(s.dtype, s.shape) for k, s in outs.items()}


def _vp(t):
    return None if t is None or t.numel() == 0 else ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def flipped(rowptr, col):
    """The matrix with the degrees of `rowptr` in reverse row order: same M, E, multiset of columns and long rows."""
    deg = (rowptr[1:] - rowptr[:-1]).flip(0)
    rp = torch.zeros_like(rowptr)
    rp[1:] = deg.cumsum(0)
    return rp, col.flip(0).contiguous()


def set_shift(monkeypatch, shift):
    if shift is None:
        monkeypatch.delenv(ENV, raising=False)
    else:
        monkeypatch.setenv(ENV, str(shift))


def _es(dtype):
    return torch.empty(0, dtype=dtype).element_size()


def _dev(*ts_):
    return [None if t is None else t.to(DEV) for t in ts_]


def other_of(m):
    rp, c = flipped(m["rowptr"], m["col"])
    return rp.to(DEV), c.to(DEV)


@pytest.fixture(scope="module")
def small_other(small):
    return other_of(small)


@pytest.fixture(scope="module")
def fp8_other(fp8_mat):
    return other_of(fp8_mat)


# ---- tsb200_spmm_fw ----------------------------------------------------------------------------------------------------
def guarded_fw(rowptr, col, value, mat, reduce, other, vec=True, what=""):
    M, E = rowptr.numel() - 1, col.numel()
    N, K = mat.shape[-2:]
    B = mat.numel() // (N * K)
    red, dt = RED[reduce], ops._dtype_code(mat.dtype)
    arg = red >= MIN
    outs = {"out": Out(mat.dtype, (B, M, K), 16 if vec else _es(mat.dtype))}
    if arg:
        outs["arg"] = Out(torch.int64, (B, M, K), 16 if vec else 8)
    nws = lib.tsb200_spmm_fw_workspace_bytes(B, M, K, E, dt, red)

    def launch(a, o, w):
        rc = lib.tsb200_spmm_fw(_vp(a[0]), _vp(a[1]), _vp(value), _vp(mat), o["out"].p, o["arg"].p if arg else None,
                                B, M, N, K, E, dt, red, w["ws"].p, nws, _stream())
        assert rc == 0, rc

    r = footprint(launch, outs, {"ws": nws}, (rowptr, col), other, [rowptr, col, value, mat], what)
    shape = list(mat.shape[:-2]) + [M, K]
    return r["out"].view(shape), (r["arg"].view(shape) if arg else None)


@pytest.mark.parametrize("has_value", [True, False], ids=["value", "novalue"])
@pytest.mark.parametrize("dtype,K", TABLE, ids=_id)
def test_spmm_fw(oracle, small, small_other, monkeypatch, dtype, K, has_value):
    """Every family at full and partial width (two column tiles for `tiled`), all four reductions, B = 1 and 3, the
    automatic item size and items of 1 and 32 rows."""
    rowptr_c, col_c, N = small["rowptr"], small["col"], small["N"]
    E = col_c.numel()
    rowptr, col = _dev(rowptr_c, col_c)
    fam = family_of(dtype, K)
    for B in (1, 3):
        for quantized, reduces in ((False, ("sum", "mean")), (True, ("min", "max"))):
            mat_c = dense(N, K, dtype, K + B, quantized, B=None if B == 1 else B)
            val_c = values(E, dtype, K + 1, quantized) if has_value else None
            mat, val = _dev(mat_c, val_c)
            ref = Ref(oracle, rowptr_c, col_c, val_c, mat_c)
            for shift, reduce in [(s, r) for s in ((None, 0, 5) if B == 1 else (None,)) for r in reduces]:
                set_shift(monkeypatch, shift)
                what = f"spmm_fw {fam} {dtype} K={K} B={B} shift={shift} value={has_value} {reduce}"
                out, arg = guarded_fw(rowptr, col, val, mat, reduce, small_other, what=what)
                ref.check(reduce, out, arg, what)
                out_u, arg_u = call_fw(rowptr, col, val, mat, reduce)
                assert_bits_equal(out, out_u, what + " vs unguarded")
                if arg is not None:
                    assert torch.equal(arg, arg_u), what + " arg vs unguarded"


def test_spmm_fw_generic(oracle, small, small_other):
    """The generic kernel: fp64 (outputs at 8 B), bf16 values at a 2-byte aligned address, 24-byte fp32 rows."""
    rowptr_c, col_c, N = small["rowptr"], small["col"], small["N"]
    E = col_c.numel()
    rowptr, col = _dev(rowptr_c, col_c)
    for dtype, K, aligned in ((torch.float64, 8, True), (torch.bfloat16, 8, False), (torch.float32, 6, True)):
        assert family_of(dtype, K, aligned) == "generic"
        for quantized, reduces in ((False, ("sum", "mean")), (True, ("min", "max"))):
            mat_c = dense(N, K, dtype, 5, quantized)
            val_c = values(E, dtype, 6, quantized)
            mat = mat_c.to(DEV)
            if aligned:
                val = val_c.to(DEV)
            else:
                buf = torch.empty(E + 1, dtype=dtype, device=DEV)
                buf[1:] = val_c.to(DEV)
                val = buf[1:]
                assert val.data_ptr() % 4 == 2
            ref = Ref(oracle, rowptr_c, col_c, val_c, mat_c)
            for reduce in reduces:
                what = f"spmm_fw generic {dtype} K={K} {reduce}"
                out, arg = guarded_fw(rowptr, col, val, mat, reduce, small_other, vec=False, what=what)
                ref.check(reduce, out, arg, what)
                out_u, arg_u = call_fw(rowptr, col, val, mat, reduce)
                assert_bits_equal(out, out_u, what + " vs unguarded")


@pytest.mark.parametrize("fam,dtype", [("gpr4", torch.float32), ("vec32ch2", torch.bfloat16)], ids=_id)
def test_spmm_fw_full_size_items(oracle, large, fam, dtype):
    """32-row items at full occupancy, fully guarded; a sample of whole 32-row groups against the oracle."""
    K = FAMILIES[fam][0 if dtype == torch.float32 else 1][0]
    rowptr_c, col_c, rows, N = large["rowptr"], large["col"], large["rows"], large["N"]
    E = col_c.numel()
    rowptr, col = _dev(rowptr_c, col_c)
    other = other_of(large)
    sp, scol, idx = sub_csr(rowptr_c, col_c, rows)
    for quantized, reduce in ((False, "sum"), (True, "max")):
        mat_c = dense(N, K, dtype, 7, quantized)
        val_c = values(E, dtype, 8, quantized)
        mat, val = _dev(mat_c, val_c)
        what = f"spmm_fw {fam} {dtype} K={K} M={large['M']} {reduce}"
        out, arg = guarded_fw(rowptr, col, val, mat, reduce, other, what=what)
        out_u, arg_u = call_fw(rowptr, col, val, mat, reduce)
        assert_bits_equal(out, out_u, what + " vs unguarded")
        ref = Ref(oracle, sp, scol, val_c[idx], mat_c)
        rows_d = rows.to(DEV)
        if reduce == "sum":
            ref.check(reduce, out[rows_d], None, what)
        else:
            assert torch.equal(arg, arg_u)
            a = arg[rows_d].cpu()
            glob = torch.cat([idx, torch.tensor([E])])
            arg_s = torch.searchsorted(glob, a)
            arg_s = torch.where(a == E, idx.numel(), arg_s)
            ref.check(reduce, out[rows_d], arg_s, what)


# ---- tsb200_spmm_plan + tsb200_spmm_fw_planned -------------------------------------------------------------------------
class GPlan:
    """A plan built into a guarded buffer of exactly tsb200_spmm_plan_bytes, optionally over another matrix's plan."""

    def __init__(self, rowptr, E, dirty_from=None, buf=None):
        M = rowptr.numel() - 1
        nb = lib.tsb200_spmm_plan_bytes(M, E)
        assert nb == plan_layout(M, E)
        self.buf = buf if buf is not None else Guarded(nb, 0, fill=0)
        if dirty_from is not None:
            self._build(dirty_from, E)
        self.counts = self._build(rowptr, E)
        self.buf.check_guards("plan")
        self.nb = nb

    def _build(self, rowptr, E):
        counts = (ctypes.c_int64 * 3)()
        rc = lib.tsb200_spmm_plan(_vp(rowptr), rowptr.numel() - 1, E, self.buf.p, self.buf.n, counts, _stream())
        assert rc == 0, rc
        torch.cuda.synchronize()
        return tuple(counts)

    @property
    def args(self):
        return (self.buf.p, self.nb) + self.counts


def guarded_planned(plan, other_plan, rowptr, col, value, mat, reduce, other, what):
    M, E = rowptr.numel() - 1, col.numel()
    N, K = mat.shape
    red, dt = RED[reduce], ops._dtype_code(mat.dtype)
    arg = red >= MIN
    _, n_long, n_slot = plan.counts
    nws = lib.tsb200_spmm_fw_planned_workspace_bytes(K, n_long, n_slot, red)
    assert nws == planned_ws(K, n_long, n_slot, arg)
    assert other_plan.counts[1:] == plan.counts[1:]
    outs = {"out": Out(mat.dtype, (M, K), 16)}
    if arg:
        outs["arg"] = Out(torch.int64, (M, K), 16)

    def launch(a, o, w):
        rp, c, pl = a
        rc = lib.tsb200_spmm_fw_planned(_vp(rp), _vp(c), _vp(value), _vp(mat), o["out"].p,
                                        o["arg"].p if arg else None, M, N, K, E, dt, red, *pl.args, w["ws"].p, nws,
                                        _stream())
        assert rc == 0, rc

    r = footprint(launch, outs, {"ws": nws}, (rowptr, col, plan), (*other, other_plan),
                  [rowptr, col, value, mat, plan.buf.body, other_plan.buf.body], what,
                  guarded_inputs=(plan.buf, other_plan.buf))
    return r["out"], r.get("arg")


@pytest.fixture(scope="module")
def small_plans(small, small_other):
    rowptr = small["rowptr"].to(DEV)
    E = small["col"].numel()
    clean = GPlan(rowptr, E)
    other = GPlan(small_other[0], E)
    dirty = GPlan(rowptr, E, dirty_from=small_other[0])
    assert dirty.counts == clean.counts == queue_counts((small["rowptr"][1:] - small["rowptr"][:-1]).tolist())
    return clean, dirty, other


@pytest.mark.parametrize("dtype,K", TABLE, ids=_id)
def test_spmm_planned(oracle, small, small_other, small_plans, dtype, K):
    """Planned products from a plan built in a zeroed buffer and one built over another matrix's plan: guarded,
    in reused planned workspaces, bit-identical to each other and to the unguarded planned call; the plan unchanged."""
    rowptr_c, col_c, N = small["rowptr"], small["col"], small["N"]
    E = col_c.numel()
    rowptr, col = _dev(rowptr_c, col_c)
    clean, dirty, other = small_plans
    plan_ref = ops.spmm_plan(rowptr, E)
    for quantized, reduces in ((False, ("sum", "mean")), (True, ("min", "max"))):
        mat_c = dense(N, K, dtype, K, quantized)
        val_c = values(E, dtype, K + 1, quantized)
        mat, val = _dev(mat_c, val_c)
        ref = Ref(oracle, rowptr_c, col_c, val_c, mat_c)
        for reduce in reduces:
            what = f"planned {family_of(dtype, K)} {dtype} K={K} {reduce}"
            res = [guarded_planned(p, other, rowptr, col, val, mat, reduce, small_other, what + f" plan {i}")
                   for i, p in enumerate((clean, dirty))]
            ref.check(reduce, res[0][0], res[0][1], what)
            out_u, arg_u = call_planned(plan_ref, rowptr, col, val, mat, reduce)
            for out, arg in res:
                assert_bits_equal(out, out_u, what + " vs unguarded")
                if arg is not None:
                    assert torch.equal(arg, arg_u), what


# ---- tsb200_spmm_fw_acc ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,K", [(torch.float32, 12), (torch.bfloat16, 40), (torch.float32, 260),
                                     (torch.bfloat16, 1032)], ids=_id)
def test_spmm_fw_acc(oracle, small, small_other, dtype, K):
    """Modes 1 -> 2 -> 3 over P = 3 column blocks; partial and out guarded; each block's workspace exact."""
    rowptr_c, col_c, N, M = small["rowptr"], small["col"], small["N"], small["M"]
    E = col_c.numel()
    mat_c = dense(N, K, dtype, K, False)
    val_c = values(E, dtype, K + 1, False)
    rowptr, col, mat, val = _dev(rowptr_c, col_c, mat_c, val_c)
    dt = ops._dtype_code(dtype)
    P = 3
    bounds = [N * c // P for c in range(P + 1)]

    def blocks(rp, c, v):
        row = torch.repeat_interleave(torch.arange(M, device=DEV), rp[1:] - rp[:-1])
        out = []
        for b in range(P):
            keep = (c >= bounds[b]) & (c < bounds[b + 1])
            bp = torch.zeros(M + 1, dtype=torch.long, device=DEV)
            bp[1:] = torch.bincount(row[keep], minlength=M).cumsum(0)
            out.append((bp, c[keep].contiguous(), v[keep].contiguous()))
        return out

    main = blocks(rowptr, col, val)
    oth = blocks(*small_other, val)
    nws = [lib.tsb200_spmm_fw_workspace_bytes(1, M, K, bc.numel(), dt, SUM) for _, bc, _ in main]
    assert nws == [lib.tsb200_spmm_fw_workspace_bytes(1, M, K, bc.numel(), dt, SUM) for _, bc, _ in oth]
    outs = {"partial": Out(torch.float32, (M, K), 16), "out": Out(dtype, (M, K), 16)}

    def launch(a, o, w):
        for b, (bp, bc, bv) in enumerate(a):
            mode = 1 if b == 0 else (3 if b == P - 1 else 2)
            rc = lib.tsb200_spmm_fw_acc(_vp(bp), _vp(bc), _vp(bv), _vp(mat), o["out"].p, o["partial"].p, mode, 1, M,
                                        N, K, bc.numel(), dt, w[b].p, nws[b], _stream())
            assert rc == 0, rc

    flat = [t for blk in main + oth for t in blk]
    r = footprint(launch, outs, dict(enumerate(nws)), main, oth, [mat, *flat], f"acc {dtype} K={K}")
    ref = Ref(oracle, rowptr_c, col_c, val_c, mat_c)
    assert_sum_bound(r["out"], ref.sum64(), ref.S(), ref.deg + P, dtype, what=f"acc {dtype} K={K}")


# ---- tsb200_spmm_fw_fp8 / _fp8_quant / _fp8_res ------------------------------------------------------------------------
def fp8_call(fn, rowptr, col, value, x8, scale, reduce, out_dtype, plan, other, other_plan, res=None, what=""):
    """fn in ("fp8", "quant", "res"); res = (res8, res_scale) for "res" (out_dtype E4M3: an e4m3 result)."""
    M, E = rowptr.numel() - 1, col.numel()
    N, K = x8.shape
    red = RED[reduce]
    arg = red >= MIN
    q8 = fn == "quant" or out_dtype == E4M3
    acc_dt = 0 if q8 else ops._FP8_OUT[out_dtype]
    if plan is None:
        nws = lib.tsb200_spmm_fw_workspace_bytes(1, M, K, E, 0, red)
    else:
        nws = lib.tsb200_spmm_fw_planned_workspace_bytes(K, plan.counts[1], plan.counts[2], red)
    outs = {"out": Out(E4M3 if q8 else out_dtype, (M, K), 16)}
    if q8:
        outs["scale"] = Out(torch.float32, (M,), 4)
    if arg:
        outs["arg"] = Out(torch.int64, (M, K), 16)
    stride = 0 if scale.dim() == 0 else 1

    def launch(a, o, w):
        rp, c, pl = a
        pa = pl.args if pl is not None else (None, 0, 0, 0, 0)
        ar = o["arg"].p if arg else None
        if fn == "fp8":
            rc = lib.tsb200_spmm_fw_fp8(_vp(rp), _vp(c), _vp(value), _vp(x8), _vp(scale), stride, o["out"].p, ar,
                                        M, N, K, E, acc_dt, red, *pa, w["ws"].p, nws, _stream())
        elif fn == "quant":
            rc = lib.tsb200_spmm_fw_fp8_quant(_vp(rp), _vp(c), _vp(value), _vp(x8), _vp(scale), stride, o["out"].p,
                                              o["scale"].p, ar, M, N, K, E, red, *pa, w["ws"].p, nws, _stream())
        else:
            r8, rs = res
            rc = lib.tsb200_spmm_fw_fp8_res(_vp(rp), _vp(c), _vp(value), _vp(x8), _vp(scale), stride, _vp(r8),
                                            _vp(rs), 0 if rs.dim() == 0 else 1, o["out"].p,
                                            o["scale"].p if q8 else None, ar, M, N, K, E, acc_dt, red, *pa, w["ws"].p,
                                            nws, _stream())
        assert rc == 0, rc

    inputs = [rowptr, col, value, x8, scale] + (list(res) if res else [])
    if plan is not None:
        inputs += [plan.buf.body, other_plan.buf.body]
    return footprint(launch, outs, {"ws": nws}, (rowptr, col, plan), (*other, other_plan), inputs, what,
                     guarded_inputs=() if plan is None else (plan.buf, other_plan.buf))


@pytest.fixture(scope="module")
def fp8_plans(fp8_mat, fp8_other):
    rowptr = fp8_mat["rowptr"].to(DEV)
    E = fp8_mat["col"].numel()
    return GPlan(rowptr, E, dirty_from=fp8_other[0]), GPlan(fp8_other[0], E)


@pytest.mark.parametrize("per_row", [True, False], ids=["rowscale", "tensorscale"])
@pytest.mark.parametrize("K", KS + KS_PARTIAL)
def test_spmm_fp8(fp8_mat, fp8_other, fp8_plans, K, per_row):
    """The fp8 forward (every out dtype, all reductions), its e4m3 result (K <= 2048; out bytes and out_scale guarded
    separately) and its residual (sum / mean), planned and unplanned."""
    rowptr_c, col_c, N, M = fp8_mat["rowptr"], fp8_mat["col"], fp8_mat["N"], fp8_mat["M"]
    E = col_c.numel()
    rowptr, col = _dev(rowptr_c, col_c)
    plan, other_plan = fp8_plans
    g = torch.Generator().manual_seed(K)
    r8 = (torch.randn(M, K, generator=g) * 8).to(E4M3).to(DEV)
    rs = (torch.rand(M, generator=g) + 0.25 if per_row else torch.tensor(0.375)).to(DEV)
    rho = rs.view(-1, 1) * r8.float() if per_row else rs * r8.float()
    for ties, reduces in ((False, ("sum", "mean")), (True, ("min", "max"))):
        x8_c = make_x8(N, K, K + ties, ties)
        sc_c = make_scale(N, K + 2, per_row)
        v_c = make_values(E, K + 3, ties)
        rep = Replay(rowptr_c, col_c, v_c, x8_c, sc_c)
        x8, sc = _dev(x8_c, sc_c)
        for pl in (None, plan):
            tag = "planned" if pl is not None else "unplanned"
            for reduce in reduces:
                for out_dtype in (torch.bfloat16, torch.float16, torch.float32):
                    v = v_c.to(out_dtype).to(DEV)
                    what = f"fp8 K={K} {_id(out_dtype)} per_row={per_row} {reduce} {tag}"
                    r = fp8_call("fp8", rowptr, col, v, x8, sc, reduce, out_dtype, pl, fp8_other, other_plan,
                                 what=what)
                    rep.check(reduce, r["out"], r.get("arg"), out_dtype, what)
                    out_u, arg_u = call_fp8(rowptr, col, v, x8, sc, reduce, out_dtype, plan=None if pl is None
                                            else ops.spmm_plan(rowptr, E))
                    assert_bits_equal(r["out"], out_u, what + " vs unguarded")
                    if out_dtype != torch.float32:
                        continue
                    y, arg_y = r["out"], r.get("arg")
                    if reduce in ("sum", "mean"):
                        z = y + rho
                        w = what.replace("fp8", "fp8_res")
                        rr = fp8_call("res", rowptr, col, v, x8, sc, reduce, out_dtype, pl, fp8_other, other_plan,
                                      res=(r8, rs), what=w)
                        assert_bits_equal(rr["out"], z, w)
                        for od in (torch.bfloat16, torch.float16):
                            rr = fp8_call("res", rowptr, col, v.to(od), x8, sc, reduce, od, pl, fp8_other,
                                          other_plan, res=(r8, rs), what=w + f" {_id(od)}")
                            # round_out(fl32(y + rho)) with y the fp32 result: one rounding of z
                            assert_bits_equal(rr["out"], z.to(od), w + f" {_id(od)}")
                    if K > 2048:
                        continue
                    w = what.replace("fp8", "fp8_quant")
                    rq = fp8_call("quant", rowptr, col, v, x8, sc, reduce, out_dtype, pl, fp8_other, other_plan,
                                  what=w)
                    assert_same_bits(rq["out"], rq["scale"], *ts.quantize_fp8(y.cpu(), True), w)
                    if arg_y is not None:
                        assert torch.equal(rq["arg"], arg_y), w
                    if reduce in ("sum", "mean"):
                        w = what.replace("fp8", "fp8_res e4m3")
                        rq = fp8_call("res", rowptr, col, v, x8, sc, reduce, E4M3, pl, fp8_other, other_plan,
                                      res=(r8, rs), what=w)
                        assert_same_bits(rq["out"], rq["scale"], *ts.quantize_fp8((y + rho).cpu(), True), w)


# ---- tsb200_spmm_fw_res ------------------------------------------------------------------------------------------------
def res_call(rowptr, col, value, x, r, s, reduce, plan, other, other_plan, what, vec=True):
    M, E = rowptr.numel() - 1, col.numel()
    N, K = x.shape
    red, dt = RED[reduce], ops._dtype_code(x.dtype)
    if plan is None:
        nws = lib.tsb200_spmm_fw_workspace_bytes(1, M, K, E, dt, red)
    else:
        nws = lib.tsb200_spmm_fw_planned_workspace_bytes(K, plan.counts[1], plan.counts[2], red)
    outs = {"out": Out(x.dtype, (M, K), 16 if vec else _es(x.dtype))}

    def launch(a, o, w):
        rp, c, pl = a
        pa = pl.args if pl is not None else (None, 0, 0, 0, 0)
        rc = lib.tsb200_spmm_fw_res(_vp(rp), _vp(c), _vp(value), _vp(x), _vp(r), _vp(s), 0 if s.dim() == 0 else 1,
                                    o["out"].p, M, N, K, E, dt, red, *pa, w["ws"].p, nws, _stream())
        assert rc == 0, rc

    inputs = [rowptr, col, value, x, r, s] + ([plan.buf.body, other_plan.buf.body] if plan is not None else [])
    return footprint(launch, outs, {"ws": nws}, (rowptr, col, plan), None if other is None else (*other, other_plan),
                     inputs, what, guarded_inputs=() if plan is None else (plan.buf, other_plan.buf))["out"]


@pytest.mark.parametrize("dtype,K", [(torch.float32, 4), (torch.bfloat16, 16), (torch.float16, 40),
                                     (torch.float32, 68), (torch.bfloat16, 392), (torch.float32, 1028),
                                     (torch.float64, 8), (torch.float32, 6)], ids=_id)
def test_spmm_fw_res(small, small_other, small_plans, dtype, K):
    """Scalar and per-row residual scales, planned and unplanned, and the generic kernel (fp64, 24-byte rows)."""
    rowptr_c, col_c, N, M = small["rowptr"], small["col"], small["N"], small["M"]
    E = col_c.numel()
    rowptr, col = _dev(rowptr_c, col_c)
    vec = family_of(dtype, K) != "generic"
    _, plan, other_plan = small_plans
    g = torch.Generator().manual_seed(K)
    x = torch.randn(N, K, generator=g, dtype=torch.float64).to(dtype)
    v = torch.randn(E, generator=g, dtype=torch.float64).to(dtype)
    r = torch.randn(M, K, generator=g, dtype=torch.float64).to(dtype)
    sdt = torch.float64 if dtype == torch.float64 else torch.float32
    xd, vd, rd = _dev(x, v, r)
    for s in (torch.tensor(0.75, dtype=sdt), (torch.rand(M, generator=g, dtype=torch.float64) * 2 - 0.5).to(sdt)):
        sd = s.to(DEV)
        for reduce in ("sum", "mean"):
            ref, bound = res_ref_bound(rowptr_c, col_c, v, x, r, s, reduce == "mean", dtype)
            for pl in ((None, plan) if vec else (None,)):
                what = f"spmm_fw_res {dtype} K={K} {reduce} per_row={s.dim()} {'planned' if pl else 'unplanned'}"
                out = res_call(rowptr, col, vd, xd, rd, sd, reduce, pl, small_other, other_plan, what, vec)
                assert_bound(out, ref, bound, what)
                u = call_res_unguarded(rowptr, col, vd, xd, rd, sd, reduce,
                                       None if pl is None else ops.spmm_plan(rowptr, E))
                assert_bits_equal(out, u, what + " vs unguarded")


@pytest.mark.parametrize("dtype,K", [(torch.float32, 4), (torch.bfloat16, 200), (torch.float32, 1100),
                                     (torch.float64, 8), (torch.bfloat16, 7)], ids=_id)
def test_spmm_fw_res_residual_only(dtype, K):
    """E = 0: the residual-only kernels (vector rows) or the generic kernel write round(fl(+0 + s r))."""
    M = 1000
    rowptr = torch.zeros(M + 1, dtype=torch.long, device=DEV)
    col = torch.empty(0, dtype=torch.long, device=DEV)
    g = torch.Generator().manual_seed(K)
    x = torch.randn(3, K, generator=g, dtype=torch.float64).to(dtype).to(DEV)
    r = torch.randn(M, K, generator=g, dtype=torch.float64).to(dtype).to(DEV)
    sdt = torch.float64 if dtype == torch.float64 else torch.float32
    vec = family_of(dtype, K) != "generic"
    for s in (torch.tensor(-1.5, dtype=sdt, device=DEV), torch.rand(M, generator=g, dtype=sdt).to(DEV)):
        what = f"residual only {dtype} K={K} per_row={s.dim()}"
        out = res_call(rowptr, col, None, x, r, s, "sum", None, None, None, what, vec)
        acc = torch.float64 if dtype == torch.float64 else torch.float32
        sr = (s.view(-1, 1) if s.dim() else s).to(acc) * r.to(acc)
        assert_bits_equal(out, (torch.zeros_like(sr) + sr).to(dtype), what)


# ---- tsb200_spmm_heads / tsb200_sddmm_heads ----------------------------------------------------------------------------
HEADS = [c for c in HEAD_CASES if c in ((torch.bfloat16, 1, 8), (torch.float32, 2, 4), (torch.float16, 2, 16),
                                        (torch.bfloat16, 2, 64), (torch.float32, 8, 8), (torch.bfloat16, 8, 64),
                                        (torch.float32, 8, 128), (torch.float64, 2, 8), (torch.float32, 4, 3),
                                        (torch.float16, 3, 8))]


@pytest.mark.parametrize("case", HEADS, ids=lambda c: f"{str(c[0]).split('.')[-1]}-H{c[1]}-D{c[2]}")
def test_heads(small, small_other, small_plans, case):
    dtype, H, D = case
    rowptr_c, col_c, M, N = small["rowptr"], small["col"], small["M"], small["N"]
    E = col_c.numel()
    rowptr, col = _dev(rowptr_c, col_c)
    es = _es(dtype)
    misaligned = dtype == torch.float16 and H == 3
    vec = dtype != torch.float64 and (D * es) % 16 == 0 and not misaligned
    al = 16 if vec else es
    g = torch.Generator().manual_seed(H * 100 + D)
    x_c = torch.randn(N, H, D, generator=g, dtype=torch.float64).to(dtype)
    v_c = torch.randn(E, H, generator=g, dtype=torch.float64).to(dtype)
    a_c = torch.randn(M, H, D, generator=g, dtype=torch.float64).to(dtype)
    x, v, a = _dev(x_c, v_c, a_c)
    if misaligned:   # 16-byte heads two elements off a 16-byte boundary: the generic kernels
        x, a = unaligned(x), unaligned(a)
    dt = ops._dtype_code(dtype)
    u = 2.0 ** -53 if dtype == torch.float64 else U32
    _, plan, other_plan = small_plans
    ref, S, deg = heads_ref(rowptr_c, col_c, v_c, x_c)
    for pl in ((None, plan) if vec else (None,)):
        nws = (lib.tsb200_spmm_fw_workspace_bytes(1, M, H * D, E, dt, SUM) if pl is None else
               lib.tsb200_spmm_fw_planned_workspace_bytes(H * D, pl.counts[1], pl.counts[2], SUM))

        def launch(args, o, w):
            rp, c, p_ = args
            pa = p_.args if p_ is not None else (None, 0, 0, 0, 0)
            rc = lib.tsb200_spmm_heads(_vp(rp), _vp(c), _vp(v), _vp(x), o["out"].p, M, N, H, D, E, dt, *pa,
                                       w["ws"].p, nws, _stream())
            assert rc == 0, rc

        what = f"spmm_heads {dtype} H={H} D={D} {'planned' if pl else 'unplanned'}"
        inputs = [rowptr, col, v, x] + ([pl.buf.body, other_plan.buf.body] if pl is not None else [])
        out = footprint(launch, {"out": Out(dtype, (M, H, D), al)}, {"ws": nws}, (rowptr, col, pl),
                        (*small_other, other_plan), inputs, what,
                        guarded_inputs=() if pl is None else (pl.buf, other_plan.buf))["out"]
        assert_sum_bound(out, ref, S, deg + 1, dtype, u=u, what=what)
        assert_bits_equal(out, call_spmm_heads(rowptr, col, v, x, M, None if pl is None else ops.spmm_plan(rowptr, E)),
                          what + " vs unguarded")
    dref, dS = heads_sddmm_ref(rowptr_c, col_c, a_c, x_c)
    nws = lib.tsb200_spmm_value_bw_workspace_bytes(1, M, H * D, E, dt)

    def launch_sddmm(args, o, w):
        rc = lib.tsb200_sddmm_heads(_vp(args[0]), _vp(args[1]), _vp(a), _vp(x), o["out"].p, M, N, H, D, E, dt,
                                    w["ws"].p, nws, _stream())
        assert rc == 0, rc

    what = f"sddmm_heads {dtype} H={H} D={D}"
    out = footprint(launch_sddmm, {"out": Out(dtype, (E, H), es)}, {"ws": nws}, (rowptr, col), small_other,
                    [rowptr, col, a, x], what)["out"]
    assert_sum_bound(out, dref, dS, D + 1, dtype, u=u, what=what)
    assert_bits_equal(out, call_sddmm_heads(rowptr, col, a, x), what + " vs unguarded")


# ---- tsb200_spmm_value_bw / tsb200_sddmm_fp8 ---------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,K,B,ws", [(torch.float32, 12, 1, True), (torch.bfloat16, 72, 1, True),
                                          (torch.float16, 512, 1, True), (torch.float32, 256, 1, True),
                                          (torch.float32, 4, 1, True), (torch.bfloat16, 600, 1, True),
                                          (torch.float32, 40, 1, False), (torch.bfloat16, 24, 2, False),
                                          (torch.float32, 200, 3, False), (torch.float64, 8, 2, False),
                                          (torch.bfloat16, 7, 1, True)], ids=_id)
def test_value_bw(oracle, small, small_other, dtype, K, B, ws):
    """Row-wise with a workspace, nnz-parallel (no workspace, or B > 1) and generic."""
    rowptr_c, col_c, N, M = small["rowptr"], small["col"], small["N"], small["M"]
    E = col_c.numel()
    mat_c = dense(N, K, dtype, K + B, False, B=None if B == 1 else B)
    g = torch.Generator().manual_seed(K)
    grad_c = torch.randn(mat_c.shape[:-2] + (M, K), generator=g, dtype=torch.float64).to(dtype)
    row_c = torch.repeat_interleave(torch.arange(M), rowptr_c[1:] - rowptr_c[:-1])
    row, rowptr, col, mat, grad = _dev(row_c, rowptr_c, col_c, mat_c, grad_c)
    orp, ocol = small_other
    orow = torch.repeat_interleave(torch.arange(M, device=DEV), orp[1:] - orp[:-1])
    dt = ops._dtype_code(dtype)
    nws = lib.tsb200_spmm_value_bw_workspace_bytes(B, M, K, E, dt) if ws else 0
    fam = sddmm_family(dtype, K, B) if ws else "nnz"
    for reduce in ("sum", "mean"):
        def launch(a, o, w):
            rc = lib.tsb200_spmm_value_bw(_vp(a[0]), _vp(a[1]), _vp(a[2]), _vp(mat), _vp(grad), o["out"].p, B, M, N, K,
                                          E, dt, RED[reduce], w["ws"].p if ws else None, nws, _stream())
            assert rc == 0, rc

        what = f"value_bw {fam} {dtype} K={K} B={B} {reduce}"
        out = footprint(launch, {"out": Out(dtype, (E,), _es(dtype))}, {"ws": nws}, (row, rowptr, col),
                        (orow, orp, ocol), [row, rowptr, col, mat, grad], what)["out"]
        check_value_bw(oracle, rowptr_c, col_c, mat_c, grad_c, reduce, out, what)
        if ws or lib.tsb200_spmm_value_bw_workspace_bytes(B, M, K, E, dt) == 0:
            # the existing caller passes a workspace whenever one is sized: the same kernel as here
            u = call_value_bw(row, rowptr, col, mat, grad, reduce)
        else:
            # it would take the row-wise kernel; the nnz-parallel one unguarded, into a NaN-prefilled output
            u = torch.full((E,), float("nan"), dtype=dtype, device=DEV)
            assert lib.tsb200_spmm_value_bw(_vp(row), _vp(rowptr), _vp(col), _vp(mat), _vp(grad), _vp(u), B, M, N, K,
                                            E, dt, RED[reduce], None, 0, _stream()) == 0
        assert_bits_equal(out, u, what + " vs unguarded")


@pytest.mark.parametrize("K", [16, 64, 400, 2048])
def test_sddmm_fp8(small, small_other, K):
    rowptr_c, col_c, N, M = small["rowptr"], small["col"], small["N"], small["M"]
    E = col_c.numel()
    rowptr, col = _dev(rowptr_c, col_c)
    row_c = torch.repeat_interleave(torch.arange(M), rowptr_c[1:] - rowptr_c[:-1])
    nws = lib.tsb200_sddmm_fp8_workspace_bytes(M, K, E)
    for per_row in (True, False):
        a8, b8 = _dev(fp8_operand(M, K, K, True), fp8_operand(N, K, K + 1, True))
        sa, sb = _dev(fp8_scale(M, K, per_row, True), fp8_scale(N, K + 1, per_row, True))
        s, d, _ = sddmm_fp8_replay(a8, sa, b8, sb, row_c, col_c)
        for out_dtype in (torch.bfloat16, torch.float16, torch.float32):
            def launch(a, o, w):
                rc = lib.tsb200_sddmm_fp8(_vp(a[0]), _vp(a[1]), _vp(a8), _vp(sa), 0 if sa.dim() == 0 else 1, _vp(b8),
                                          _vp(sb), 0 if sb.dim() == 0 else 1, o["out"].p, M, N, K, E,
                                          ops._FP8_OUT[out_dtype], w["ws"].p, nws, _stream())
                assert rc == 0, rc

            what = f"sddmm_fp8 K={K} per_row={per_row} {_id(out_dtype)}"
            out = footprint(launch, {"out": Out(out_dtype, (E,), _es(out_dtype))}, {"ws": nws}, (rowptr, col),
                            small_other, [rowptr, col, a8, sa, b8, sb], what)["out"]
            assert_bits_equal(out, expected_bits(s, d, out_dtype), what)


# ---- tsb200_spmm_minmax_bw ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,K,B", [(torch.float32, 40, 1), (torch.bfloat16, 256, 2), (torch.float64, 100, 1)],
                         ids=_id)
def test_minmax_bw(oracle, small, dtype, K, B):
    """grad_value[E] and grad_mat[B, N, K] zero-filled inside guards; what no arg_out entry points at stays +0."""
    rowptr_c, col_c, N, M = small["rowptr"], small["col"], small["N"], small["M"]
    E = col_c.numel()
    g = torch.Generator().manual_seed(K)
    mat_c = torch.nan_to_num(dense(N, K, dtype, K, False, B=None if B == 1 else B), nan=1.0)
    val_c = torch.randn(E, generator=g, dtype=torch.float64).to(dtype)
    grad_c = torch.randn(mat_c.shape[:-2] + (M, K), generator=g, dtype=torch.float64).to(dtype)
    rowptr, col, val, mat, grad = _dev(rowptr_c, col_c, val_c, mat_c, grad_c)
    acc = torch.float64 if dtype == torch.float64 else torch.float32
    for reduce in ("min", "max"):
        _, arg = call_fw(rowptr, col, val, mat, reduce)
        arg_c = arg.cpu()

        def launch(a, o, w):
            rc = lib.tsb200_spmm_minmax_bw(_vp(col), _vp(val), _vp(mat), _vp(grad), _vp(arg), o["gv"].p, o["gm"].p,
                                           B, M, N, K, E, ops._dtype_code(dtype), _stream())
            assert rc == 0, rc

        outs = {"gv": Out(acc, (E,), _es(acc), full=False, fill=0),
                "gm": Out(acc, tuple(mat.shape), _es(acc), full=False, fill=0)}
        what = f"minmax_bw {dtype} K={K} B={B} {reduce}"
        r = footprint(launch, outs, {}, (), None, [col, val, mat, grad, arg], what, reruns_equal=False)
        ref_v, ref_m = oracle.spmm_minmax_bw(col_c, val_c.double(), mat_c.double(), grad_c.double(), arg_c, True, True)
        S_v, S_m = oracle.spmm_minmax_bw(col_c, val_c.double().abs(), mat_c.double().abs(), grad_c.double().abs(),
                                         arg_c, True, True)
        ones = torch.ones(E, dtype=torch.float64)
        n_v, n_m = oracle.spmm_minmax_bw(col_c, ones, torch.ones(mat_c.shape, dtype=torch.float64),
                                         torch.ones(grad_c.shape, dtype=torch.float64), arg_c, True, True)
        check_accumulated(r["gv"], ref_v, S_v, n_v, U32 if dtype != torch.float64 else 2.0 ** -53, what + " gv")
        check_accumulated(r["gm"], ref_m, S_m, n_m, U32 if dtype != torch.float64 else 2.0 ** -53, what + " gm")
        # elements no arg_out entry routes a term to: +0, bit for bit
        for got, n in ((r["gv"], n_v), (r["gm"], n_m)):
            untouched = (n == 0).to(DEV)
            bits = got.view({4: torch.int32, 8: torch.int64}[_es(acc)])
            assert bool((bits[untouched] == 0).all()), what + ": an element without terms is not +0"


# ---- tsb200_segment_softmax / _bw --------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32, torch.float64], ids=_id)
@pytest.mark.parametrize("D", [1, 3, 8])
def test_segment_softmax(dtype, D):
    """Row form and column form; vector and scalar forms (odd D, and the operand one element off its alignment);
    segments from 1 to 60000 entries."""
    a = structured()
    code = ops._dtype_code(dtype)
    es = _es(dtype)
    for dim, src in ((1, a), (0, a)):
        st = src.storage
        ptr, perm = (st.rowptr(), None) if dim == 1 else (st.colptr(), st.csr2csc())
        E, S = src.nnz(), ptr.numel() - 1
        for off in (0, 1):
            v = scores(E, D, dtype, seed=D)
            g = scores(E, D, dtype, seed=100 + D, scale=1.0)
            if off:   # one element past a 16-byte boundary
                vb = torch.empty(E * D + 1, dtype=dtype, device=DEV)
                vb[1:] = v.reshape(-1)
                v = vb[1:].view(E, D)
            al = es if off else 16

            def fwd(args, o, w):
                assert lib.tsb200_segment_softmax(_vp(ptr), _vp(perm), _vp(v), o["out"].p, S, E, D, code,
                                                  _stream()) == 0

            what = f"softmax {dtype} D={D} dim={dim} off={off}"
            inputs = [ptr, perm, v]
            out = footprint(fwd, {"out": Out(dtype, (E, D), al)}, {}, (), None, inputs, what)["out"]
            assert_forward(out, ptr, v, perm, what)
            u = torch.full_like(v, float("nan"))
            assert softmax_unguarded(ptr, v, perm, u) == 0
            assert_bits_equal(out, u, what + " vs unguarded")
            alpha = out.clone()

            def bwd(args, o, w):
                assert lib.tsb200_segment_softmax_bw(_vp(ptr), _vp(perm), _vp(alpha), _vp(g), o["gin"].p, S, E, D,
                                                     code, _stream()) == 0

            gin = footprint(bwd, {"gin": Out(dtype, (E, D), al)}, {}, (), None, [ptr, perm, alpha, g],
                            what + " bw")["gin"]
            assert_backward(gin, ptr, alpha, g, perm, what + " bw")
            u = torch.full_like(v, float("nan"))
            assert lib.tsb200_segment_softmax_bw(_vp(ptr), _vp(perm), _vp(alpha), _vp(g), _vp(u), S, E, D, code,
                                                 _stream()) == 0
            assert_bits_equal(gin, u, what + " bw vs unguarded")


# ---- tsb200_quantize_fp8 -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32], ids=_id)
@pytest.mark.parametrize("K,ld", [(16, 16), (400, 424), (1000, 1008), (4096, 4096), (15, 15), (15, 40)])
def test_quantize_fp8(dtype, K, ld):
    """Short rows (<= 2 KB in registers), long rows, and the element-wise kernel (K * size not a multiple of 16, or
    a row pitch ld > K); x8 and scale guarded; the per-tensor workspace is exactly 4 bytes."""
    g = torch.Generator().manual_seed(K + ld)
    N = 1037
    xc = make_rows(N, K, dtype, g)
    wide = torch.full((N, ld), float("nan"), dtype=dtype, device=DEV)
    wide[:, :K] = xc.to(DEV)
    code = ops._dtype_code(dtype)
    for per_row in (1, 0):
        def launch(a, o, w):
            rc = lib.tsb200_quantize_fp8(_vp(wide), N, K, ld, code, per_row, o["x8"].p, o["scale"].p,
                                         w["ws"].p if not per_row else None, 0 if per_row else 4, _stream())
            assert rc == 0, rc

        outs = {"x8": Out(E4M3, (N, K), 16), "scale": Out(torch.float32, (N if per_row else 1,), 4)}
        what = f"quantize_fp8 {dtype} K={K} ld={ld} per_row={per_row}"
        r = footprint(launch, outs, {} if per_row else {"ws": 4}, (), None, [wide], what)
        assert_same_bits(r["x8"], r["scale"] if per_row else r["scale"][0], *ts.quantize_fp8(xc, bool(per_row)), what)


# ---- the segment queues at their worst case ----------------------------------------------------------------------------
def worst_matrix(pattern, N=512, seed=0):
    deg = {"budget": worst_budget(40), "long": worst_long(32 * 20), "mixed": worst_mixed(20, 32 * 10)}[pattern]
    deg = torch.tensor(deg, dtype=torch.long)
    rowptr = torch.zeros(deg.numel() + 1, dtype=torch.long)
    rowptr[1:] = deg.cumsum(0)
    # columns of the dense rows the operands keep finite (dense() fills row 0 and the last NAN_ROWS - 1 with NaN)
    col = torch.randint(1, N - NAN_ROWS + 1, (int(rowptr[-1]),), generator=torch.Generator().manual_seed(seed))
    return dict(M=deg.numel(), N=N, rowptr=rowptr, col=col, deg=deg.tolist())


def read_counters(ws):
    return tuple(ws.body[4:16].view(torch.int32).cpu().tolist())


@pytest.mark.parametrize("pattern", ["budget", "long", "mixed"])
def test_segment_queue_worst_case(oracle, monkeypatch, pattern):
    """Counters [1..3] of the unplanned workspace after the SpMM forward (sum, max), the row-wise SDDMM, spmm_heads and
    the fp8 forward equal the restated counts at every item size and B, within the capacities; the plan's counts are
    the restated plan counts; every output is written and within its bound."""
    m = worst_matrix(pattern)
    rowptr_c, col_c, N, M, deg = m["rowptr"], m["col"], m["N"], m["M"], m["deg"]
    E = col_c.numel()
    rowptr, col = _dev(rowptr_c, col_c)
    other = other_of(m)
    K = 64
    dtype = torch.bfloat16
    for shift in range(6):
        monkeypatch.setenv(ENV, str(shift))
        for B in (1, 3):
            want = queue_counts(deg, 1 << shift, B)
            caps = capacities(B, E)
            assert all(w <= c for w, c in zip(want, caps)), (want, caps)
            for quantized, reduce in ((False, "sum"), (True, "max")):
                mat_c = dense(N, K, dtype, shift, quantized, B=None if B == 1 else B)
                val_c = values(E, dtype, shift + 1, quantized)
                mat, val = _dev(mat_c, val_c)
                ws = Guarded(lib.tsb200_spmm_fw_workspace_bytes(B, M, K, E, 3, RED[reduce]), 0, fill=0)
                red = RED[reduce]
                outs = [Out(dtype, (B, M, K), 16).make()]
                if red >= MIN:
                    outs.append(Out(torch.int64, (B, M, K), 16).make())
                rc = lib.tsb200_spmm_fw(_vp(rowptr), _vp(col), _vp(val), _vp(mat), outs[0].p,
                                        outs[1].p if red >= MIN else None, B, M, N, K, E, 3, red, ws.p, ws.n,
                                        _stream())
                assert rc == 0
                torch.cuda.synchronize()
                what = f"worst {pattern} shift={shift} B={B} spmm {reduce}"
                assert read_counters(ws) == want, (what, read_counters(ws), want)
                for o in outs:
                    o.check_guards(what)
                    assert not bool(unwritten(o, o.body.numel() // (B * M * K)).any()), what
                ws.check_guards(what)
                shape = list(mat.shape[:-2]) + [M, K]
                out = outs[0].t(dtype, shape)
                arg = outs[1].t(torch.int64, shape) if red >= MIN else None
                Ref(oracle, rowptr_c, col_c, val_c, mat_c).check(reduce, out, arg, what)
            # the row-wise SDDMM (B = 1)
            if B == 1:
                mat_c = dense(N, K, dtype, 9, False)
                grad_c = dense(M, K, dtype, 10, False)
                grad_c = torch.nan_to_num(grad_c, nan=0.5)
                row = torch.repeat_interleave(torch.arange(M), rowptr_c[1:] - rowptr_c[:-1]).to(DEV)
                nws = lib.tsb200_spmm_value_bw_workspace_bytes(1, M, K, E, 3)
                ws = Guarded(nws, 0, fill=0)
                out = Out(dtype, (E,), 2).make()
                mat, grad = _dev(mat_c, grad_c)
                assert lib.tsb200_spmm_value_bw(_vp(row), _vp(rowptr), _vp(col), _vp(mat), _vp(grad), out.p, 1, M, N,
                                                K, E, 3, SUM, ws.p, nws, _stream()) == 0
                torch.cuda.synchronize()
                what = f"worst {pattern} shift={shift} sddmm"
                # the SDDMM writes each segment's dots directly: no long rows, no partial slots
                assert read_counters(ws) == (want[0], 0, 0), (what, read_counters(ws), want)
                out.check_guards(what)
                ws.check_guards(what)
                assert not bool(unwritten(out, 2).any()), what
                check_value_bw(oracle, rowptr_c, col_c, mat_c, grad_c, "sum", out.t(dtype, (E,)), what)
                # spmm_heads, H = 2
                H, D = 2, K // 2
                x_c = torch.randn(N, H, D, generator=torch.Generator().manual_seed(shift), dtype=torch.float64).to(dtype)
                v_c = torch.randn(E, H, generator=torch.Generator().manual_seed(shift + 1),
                                  dtype=torch.float64).to(dtype)
                x, v = _dev(x_c, v_c)
                nws = lib.tsb200_spmm_fw_workspace_bytes(1, M, K, E, 3, SUM)
                ws = Guarded(nws, 0, fill=0)
                out = Out(dtype, (M, H, D), 16).make()
                assert lib.tsb200_spmm_heads(_vp(rowptr), _vp(col), _vp(v), _vp(x), out.p, M, N, H, D, E, 3, None, 0,
                                             0, 0, 0, ws.p, nws, _stream()) == 0
                torch.cuda.synchronize()
                what = f"worst {pattern} shift={shift} heads"
                assert read_counters(ws) == want, (what, read_counters(ws), want)
                out.check_guards(what)
                ws.check_guards(what)
                ref, S, d = heads_ref(rowptr_c, col_c, v_c, x_c)
                assert_sum_bound(out.t(dtype, (M, H, D)), ref, S, d + 1, dtype, what=what)
                # fp8 forward
                x8_c = make_x8(N, K, shift, False)
                sc_c = make_scale(N, shift, True)
                v32 = make_values(E, shift, False)
                x8, sc, v32d = _dev(x8_c, sc_c, v32)
                for reduce in ("sum", "max"):
                    r = fp8_call("fp8", rowptr, col, v32d, x8, sc, reduce, torch.float32, None, other, None,
                                 what=f"worst {pattern} shift={shift} fp8 {reduce}")
                    rep = Replay(rowptr_c, col_c, v32, x8_c, sc_c)
                    rep.check(reduce, r["out"], r.get("arg"), torch.float32, f"worst {pattern} fp8")
                    nws = lib.tsb200_spmm_fw_workspace_bytes(1, M, K, E, 0, RED[reduce])
                    ws = Guarded(nws, 0, fill=0)
                    o = Out(torch.float32, (M, K), 16).make()
                    ao = Out(torch.int64, (M, K), 16).make() if reduce == "max" else None
                    assert lib.tsb200_spmm_fw_fp8(_vp(rowptr), _vp(col), _vp(v32d), _vp(x8), _vp(sc), 1, o.p,
                                                  ao.p if ao else None, M, N, K, E, 0, RED[reduce], None, 0, 0, 0, 0,
                                                  ws.p, nws, _stream()) == 0
                    torch.cuda.synchronize()
                    assert read_counters(ws) == want, (f"worst {pattern} fp8", read_counters(ws), want)
    # last, so that a queue too short for these patterns shows as unwritten rows above before any size comparison
    assert GPlan(rowptr, E).counts == queue_counts(deg)


def test_worst_case_layouts_match():
    """The workspaces of the worst-case runs are the restated layouts."""
    for pattern in ("budget", "long", "mixed"):
        m = worst_matrix(pattern)
        E, M = m["col"].numel(), m["M"]
        for B in (1, 3):
            for red in (SUM, MAX):
                assert lib.tsb200_spmm_fw_workspace_bytes(B, M, 64, E, 3, red) == ws_layout(B, 64, E, red == MAX)[
                    "total"]
        assert sum(m["deg"]) == E and (pattern != "budget" or m["deg"][:32] == BUDGET_WINDOW)
