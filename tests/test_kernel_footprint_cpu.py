"""The workspace and plan layouts of the SpMM-family kernels, restated in Python and checked against the library's own
size functions without a GPU, and the worst case of the deferred-segment queues derived from the deferral rule.

`test_kernel_footprint_gpu.py` sizes every workspace and plan exactly and reads the queue counters back through this
restatement, so it is kept honest here.

The deferral rule (csrc/spmm_common.cuh, defer_row): in a work item of up to 32 rows, a row with deg > 256 nnz is long;
a row with 0 < deg <= 256 is deferred when the prefix sum, over the item's rows in order, of the degrees of the rows
that are not long exceeds 1024. A deferred row becomes ceil(deg / 256) segments; a row of more than one segment also
takes one long-row record and one partial slot per segment. With EB = E * B the queues hold
    seg_cap = EB/32 + EB/128 + 64,   long_cap = EB/256 + 64,   slot_cap = EB/128 + 64   (integer division).
"""
import ctypes

import pytest

from pytorch_sparse_b200._lib import lib

F32, F64, F16, BF16, I32 = 0, 1, 2, 3, 4
SUM, MEAN, MIN, MAX = 0, 1, 2, 3
SEGMENT_BYTES, LONGROW_BYTES = 32, 24
LONG_T, SEG, ITEM_CAP = 256, 256, 1024


def align256(n):
    return (n + 255) // 256 * 256


def capacities(B, E):
    EB = E * (B if B > 0 else 1)
    return EB // 32 + EB // 128 + 64, EB // LONG_T + 64, EB // 128 + 64


def ws_layout(B, K, E, arg, partials=True):
    """Byte offsets of the unplanned workspace: counters, segments, long rows, fp32 partials, int64 arg partials."""
    seg_cap, long_cap, slot_cap = capacities(B, E)
    off = {"counters": 0}
    total = 256
    off["segs"] = total; total += align256(seg_cap * SEGMENT_BYTES)
    off["longs"] = total; total += align256(long_cap * LONGROW_BYTES)
    off["part_val"] = total; total += align256(slot_cap * K * 4) if partials else 0
    off["part_arg"] = total; total += align256(slot_cap * K * 8) if partials and arg else 0
    off["total"] = total
    return off


def plan_layout(M, E):
    seg_cap, long_cap, _ = capacities(1, E)
    total = 256                                          # header: counters 1..3 are the three counts
    total += align256(((M + 31) // 32 + 1) * 4)          # one deferral mask word per 32-row group
    total += align256(seg_cap * SEGMENT_BYTES)
    total += align256(seg_cap * 4)                       # long-row index of every segment
    total += align256(long_cap * LONGROW_BYTES)
    return total


def planned_ws(K, n_long, n_slot, arg):
    total = 256 + align256(max(n_long, 1) * 4)           # counters, then the per-long-row completion counts
    total += align256(max(n_slot, 1) * K * 4)
    total += align256(max(n_slot, 1) * K * 8) if arg else 0
    return total


def fw_workspace_bytes(B, M, K, E, dtype, reduce):
    if dtype not in (F32, F16, BF16) or B <= 0 or K <= 0 or E <= 0:
        return 0
    return ws_layout(B, K, E, reduce in (MIN, MAX))["total"]


def value_bw_workspace_bytes(B, M, K, E, dtype):
    if dtype not in (F32, F16, BF16) or B != 1 or K <= 0 or E <= 0:
        return 0
    return ws_layout(1, K, E, False, False)["total"]


def sddmm_fp8_workspace_bytes(M, K, E):
    return 0 if K <= 0 or E <= 0 else ws_layout(1, K, E, False, False)["total"]


# ---- the deferral rule and the queue counts ----------------------------------------------------------------------------
def deferred(deg, group):
    """Per row (a list of degrees): whether the items of `group` rows (aligned to multiples of `group`) defer it."""
    out = []
    for g0 in range(0, len(deg), group):
        cum = 0
        for d in deg[g0:g0 + group]:
            cum += 0 if d > LONG_T else d
            out.append(d > 0 and (d > LONG_T or cum > ITEM_CAP))
    return out


def queue_counts(deg, group=32, B=1):
    """(segments, long rows, partial slots) pushed by B batches of items of `group` rows: the counters [1], [2] and [3]
    of an unplanned workspace after the call, and with group = 32 and B = 1 the counts of tsb200_spmm_plan."""
    n_seg = n_long = n_slot = 0
    for d, dfr in zip(deg, deferred(deg, group)):
        if dfr:
            s = -(-d // SEG)
            n_seg += s
            if s > 1:
                n_long += 1
                n_slot += s
    return n_seg * B, n_long * B, n_slot * B


# Worst cases of the queues per nnz (derivation):
# * Budget deferral. In one item the rows that are not long and not deferred sum to at most 1024 nnz, and a row is
#   only deferred once that prefix has passed 1024. A deferred row of d nnz adds one segment for d nnz, so the most
#   segments per nnz come from the smallest prefix that passes 1024 and then the most rows of one nnz. Rows of at most
#   256 nnz need four rows to reach 1024 (4 x 256), which leaves 28 rows of one nnz, each deferred: 28 segments per
#   1052 nnz, 0.0266 per nnz. No long row or slot is involved.
# * Long rows. A row of d > 256 nnz gives ceil(d / 256) segments and slots and one long row; per nnz that is largest at
#   d = 257: 2 segments, 1 long row and 2 slots per 257 nnz (0.00778 segments and slots, 0.00389 long rows per nnz).
#   Long rows add nothing to the budget prefix, so mixing them into a budget window only lowers its rate.
# Against the capacities: 28/1052 < 1/32 + 1/128 = 0.039 segments, 1/257 < 1/256 long rows and 2/257 < 1/128 slots per
# nnz, before the + 64 of each capacity. Smaller items (1 << s rows, s < 5) defer fewer rows: 2^s - 4 per
# 1024 + 2^s - 4 nnz for s >= 3, none for s <= 2, since four rows of 256 already fill a 4-row item.
BUDGET_WINDOW = [256] * 4 + [1] * 28
LONG_ROW = 257


def worst_budget(windows):
    return BUDGET_WINDOW * windows


def worst_long(rows):
    return [LONG_ROW] * rows


def worst_mixed(windows, rows):
    """Budget windows, then 32-row groups of long rows, alternating."""
    deg = []
    for i in range(max(windows, rows // 32 + 1)):
        if i < windows:
            deg += BUDGET_WINDOW
        deg += [LONG_ROW] * min(32, max(rows - 32 * i, 0))
    return deg


def assert_within_capacity(deg, B=1):
    E = sum(deg)
    caps = capacities(B, E)
    for s in range(6):
        got = queue_counts(deg, 1 << s, B)
        assert all(g <= c for g, c in zip(got, caps)), (s, B, got, caps)


# ---- the restatement against the library -------------------------------------------------------------------------------
GRID = [(B, M, K, E, dt, red) for B in (0, 1, 2, 3, 7) for M in (0, 1, 100, 70_000) for K in (0, 1, 4, 12, 64, 1100)
        for E in (0, 1, 31, 1000, 12_345, 3_000_000) for dt in (F32, F64, F16, BF16, I32) for red in (SUM, MEAN, MIN, MAX)
        if (M, dt, red) in ((100, F32, SUM), (100, BF16, MAX), (0, F16, MEAN), (70_000, F32, MIN), (1, F64, SUM),
                            (100, I32, MAX))]


def test_fw_workspace_bytes():
    for B, M, K, E, dt, red in GRID:
        assert lib.tsb200_spmm_fw_workspace_bytes(B, M, K, E, dt, red) == fw_workspace_bytes(B, M, K, E, dt, red), \
            (B, M, K, E, dt, red)


def test_value_bw_and_sddmm_fp8_workspace_bytes():
    for B, M, K, E, dt, _ in GRID:
        assert lib.tsb200_spmm_value_bw_workspace_bytes(B, M, K, E, dt) == value_bw_workspace_bytes(B, M, K, E, dt), \
            (B, M, K, E, dt)
        assert lib.tsb200_sddmm_fp8_workspace_bytes(M, K, E) == sddmm_fp8_workspace_bytes(M, K, E), (M, K, E)


def test_plan_and_planned_workspace_bytes():
    for M in (0, 1, 31, 32, 33, 100, 4097, 600_017):
        for E in (0, 1, 255, 1000, 1052, 12_345, 3_000_000):
            assert lib.tsb200_spmm_plan_bytes(M, E) == plan_layout(M, E), (M, E)
    for K in (0, 1, 8, 64, 1100):
        for n_long in (0, 1, 3, 1000):
            for n_slot in (0, 1, 8, 5000):
                for red in (SUM, MEAN, MIN, MAX):
                    assert (lib.tsb200_spmm_fw_planned_workspace_bytes(K, n_long, n_slot, red)
                            == planned_ws(K, n_long, n_slot, red in (MIN, MAX))), (K, n_long, n_slot, red)


def test_workspace_offsets_are_256_byte_aligned():
    for B, M, K, E, dt, red in GRID:
        L = ws_layout(max(B, 1), K, E, red in (MIN, MAX))
        assert all(v % 256 == 0 for v in L.values()), L


def test_deferral_rule_restated():
    """The Python rule agrees with the torch restatement the kernel tests use (plan_budget_rows) on budget rows."""
    import torch
    g = torch.Generator().manual_seed(0)
    deg = torch.randint(0, 300, (32 * 50 + 7,), generator=g)
    deg[::5] = torch.randint(0, 3, (deg[::5].numel(),), generator=g)
    rowptr = torch.zeros(deg.numel() + 1, dtype=torch.long)
    rowptr[1:] = deg.cumsum(0)
    from test_spmm_kernels_gpu import plan_budget_rows
    for s in range(6):
        want = plan_budget_rows(rowptr, 1 << s).tolist()
        got = [dfr and d <= LONG_T for d, dfr in zip(deg.tolist(), deferred(deg.tolist(), 1 << s))]
        assert got == want, s


def test_worst_case_rates():
    """The two worst windows give the counts of the derivation."""
    assert queue_counts(BUDGET_WINDOW) == (28, 0, 0) and sum(BUDGET_WINDOW) == 1052
    assert queue_counts(BUDGET_WINDOW, group=16) == (12, 0, 0)     # the second 16-row item defers nothing
    assert queue_counts(BUDGET_WINDOW, group=4) == (0, 0, 0)
    assert queue_counts([LONG_ROW]) == (2, 1, 2)
    # any deviation from the window makes it no worse: one nnz more in a deferred row or one row fewer in the prefix
    for i in range(32):
        for delta in (-1, 1):
            d = list(BUDGET_WINDOW)
            d[i] = max(d[i] + delta, 0)
            n = queue_counts(d)[0]
            assert n * 1052 <= 28 * sum(d), (i, delta, n)


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("pattern", ["budget", "long", "mixed"])
def test_worst_cases_fit_the_capacities(pattern, B):
    for n in (1, 2, 3, 10, 100, 1000):
        deg = {"budget": worst_budget(n), "long": worst_long(32 * n), "mixed": worst_mixed(n, 32 * n)}[pattern]
        assert_within_capacity(deg, B)


def test_capacity_margin():
    """The budget pattern at its worst uses under 70 % of the segment queue; the long rows' slots over 99 % of theirs
    at large E (2/257 against 1/128), so the + 64 is what covers short matrices of such rows."""
    deg = worst_budget(10_000)
    seg_cap = capacities(1, sum(deg))[0]
    assert queue_counts(deg)[0] < 0.7 * seg_cap
    deg = worst_long(100_000)
    _, long_cap, slot_cap = capacities(1, sum(deg))
    n_seg, n_long, n_slot = queue_counts(deg)
    assert n_long <= long_cap and n_slot <= slot_cap and n_slot > 0.99 * (slot_cap - 64)


def test_library_loads_without_a_device():
    assert isinstance(lib, ctypes.CDLL)
