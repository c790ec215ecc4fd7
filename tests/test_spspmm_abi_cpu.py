"""Return codes of the 5 C entry points of `csrc/spspmm.cu`, without a GPU: negative extents and capacity, the M < 2^31
limit, unsupported value dtypes, required NULLs, the workspace size rules, the nothing-to-do cases, and the order in
which these checks run.

Pointers are fake (`P` = 256) and never dereferenced. The table runs in a child interpreter that sees no CUDA device
(CUDA_VISIBLE_DEVICES=""), so a call that passes validation fails at its first CUDA call with a positive CUDA error:
those rows expect `CUDA`, never a particular code. The symbolic and single-pass entry points zero `rowptr_c` and their
scalars before they check the operands, so a NULL operand reaches that first CUDA call here; the GPU test
`test_null_operands_after_the_memsets` checks what they return after it. Without a device CUB reports no temporary
bytes, so workspace sizes are not pinned: the table passes a workspace no layout reaches (`BIG`) or one of 1 byte."""
import json
import os
import subprocess
import sys
from pathlib import Path

import pytest

F32, F64, F16 = 0, 1, 2
INVALID, UNSUPPORTED, WORKSPACE = -1, -2, -3
CUDA = "cuda"   # passed validation: the first CUDA call fails with a positive code
SIZE = "size"   # a workspace size (> 0)

P = 256               # a fake pointer
W = 1 << 20           # a fake workspace
BIG = 1 << 62         # a byte count no layout reaches
M_MAX = (1 << 31) - 1  # the most rows the symbolic and single-pass kernels take

# argument names and defaults of each entry point, in signature order; the defaults pass validation
BASE = {
    "spspmm_workspace_bytes": dict(M=1000, Kd=100, N=100, nnz_a=1000, nnz_b=1000),
    "spspmm_symbolic": dict(rowptr_a=P, col_a=P, rowptr_b=P, col_b=P, M=1000, Kd=100, N=100, nnz_a=1000, nnz_b=1000,
                            rowptr_c=P, ws=W, wsb=BIG, nnz_host=None, stream=None),
    "spspmm_numeric": dict(rowptr_a=P, col_a=P, val_a=P, rowptr_b=P, col_b=P, val_b=P, M=1000, Kd=100, N=100,
                           nnz_a=1000, nnz_b=1000, rowptr_c=P, row_c=P, col_c=P, val_c=P, dtype=F32, ws=W, wsb=BIG,
                           stream=None),
    "spspmm_bound": dict(col_a=P, rowptr_b=P, nnz_a=1000, ws=W, wsb=BIG, bound_host=None, stream=None),
    "spspmm_fused": dict(rowptr_a=P, col_a=P, val_a=P, rowptr_b=P, col_b=P, val_b=P, M=1000, Kd=100, N=100,
                         nnz_a=1000, nnz_b=1000, rowptr_c=P, row_c=P, col_c=P, val_c=P, capacity=5000, dtype=F32,
                         ws=W, wsb=BIG, nnz_host=None, stream=None),
}

OPERANDS = ("rowptr_a", "col_a", "rowptr_b", "col_b")


def negatives(fn, *names):
    return [(fn, {n: -1}, INVALID) for n in names]


TABLE = [
    # ---- tsb200_spspmm_workspace_bytes
    ("spspmm_workspace_bytes", {}, SIZE), ("spspmm_workspace_bytes", dict(M=0), SIZE),
    ("spspmm_workspace_bytes", dict(Kd=-1, N=-1, nnz_a=-1, nnz_b=-1), SIZE),
    ("spspmm_workspace_bytes", dict(M=-1), 0),

    # ---- tsb200_spspmm_symbolic: memsets before the operand checks
    ("spspmm_symbolic", {}, CUDA),
    *negatives("spspmm_symbolic", "M", "Kd", "N", "nnz_a", "nnz_b"),
    ("spspmm_symbolic", dict(rowptr_c=None), INVALID),
    ("spspmm_symbolic", dict(M=M_MAX), CUDA), ("spspmm_symbolic", dict(M=M_MAX + 1), UNSUPPORTED),
    ("spspmm_symbolic", dict(M=1 << 40), UNSUPPORTED),
    ("spspmm_symbolic", dict(ws=None), WORKSPACE), ("spspmm_symbolic", dict(wsb=1), WORKSPACE),
    ("spspmm_symbolic", dict(M=0, wsb=1), WORKSPACE),
    ("spspmm_symbolic", dict(M=0), CUDA), ("spspmm_symbolic", dict(nnz_a=0), CUDA),
    ("spspmm_symbolic", dict(nnz_b=0), CUDA),
    *[("spspmm_symbolic", {n: None}, CUDA) for n in OPERANDS],
    ("spspmm_symbolic", dict(M=-1, rowptr_c=None), INVALID),
    ("spspmm_symbolic", dict(M=M_MAX + 1, rowptr_c=None), INVALID),
    ("spspmm_symbolic", dict(M=M_MAX + 1, ws=None), UNSUPPORTED),

    # ---- tsb200_spspmm_numeric: no CUDA call before its operand checks, and no limit on M
    ("spspmm_numeric", {}, CUDA), ("spspmm_numeric", dict(dtype=F64), CUDA),
    ("spspmm_numeric", dict(row_c=None), CUDA),
    ("spspmm_numeric", dict(val_a=None, val_b=None), CUDA),
    ("spspmm_numeric", dict(val_c=None, dtype=9), CUDA),      # structure only: the dtype is not read
    *negatives("spspmm_numeric", "M", "Kd", "N", "nnz_a", "nnz_b"),
    ("spspmm_numeric", dict(M=0), 0), ("spspmm_numeric", dict(nnz_a=0), 0), ("spspmm_numeric", dict(nnz_b=0), 0),
    ("spspmm_numeric", dict(M=0, **{n: None for n in (*OPERANDS, "rowptr_c", "col_c")}, ws=None), 0),
    *[("spspmm_numeric", {n: None}, INVALID) for n in (*OPERANDS, "rowptr_c", "col_c")],
    ("spspmm_numeric", dict(dtype=F16), UNSUPPORTED), ("spspmm_numeric", dict(dtype=9), UNSUPPORTED),
    ("spspmm_numeric", dict(M=M_MAX + 1), CUDA), ("spspmm_numeric", dict(M=1 << 40), CUDA),
    ("spspmm_numeric", dict(ws=None), WORKSPACE), ("spspmm_numeric", dict(wsb=1), WORKSPACE),
    ("spspmm_numeric", dict(M=-1, rowptr_a=None), INVALID),
    ("spspmm_numeric", dict(nnz_a=0, rowptr_c=None), 0),
    ("spspmm_numeric", dict(rowptr_a=None, dtype=F16), INVALID),
    ("spspmm_numeric", dict(dtype=F16, ws=None), UNSUPPORTED),

    # ---- tsb200_spspmm_bound: only the 256-byte scalar block
    ("spspmm_bound", {}, CUDA), ("spspmm_bound", dict(wsb=256), CUDA),
    ("spspmm_bound", dict(wsb=255), WORKSPACE), ("spspmm_bound", dict(wsb=1), WORKSPACE),
    ("spspmm_bound", dict(ws=None), WORKSPACE),
    ("spspmm_bound", dict(nnz_a=-1), INVALID), ("spspmm_bound", dict(nnz_a=-1, ws=None), INVALID),
    ("spspmm_bound", dict(nnz_a=0), CUDA), ("spspmm_bound", dict(nnz_a=0, col_a=None, rowptr_b=None), CUDA),
    ("spspmm_bound", dict(col_a=None), CUDA), ("spspmm_bound", dict(rowptr_b=None), CUDA),

    # ---- tsb200_spspmm_fused: memsets before the operand checks
    ("spspmm_fused", {}, CUDA), ("spspmm_fused", dict(dtype=F64), CUDA),
    ("spspmm_fused", dict(row_c=None), CUDA), ("spspmm_fused", dict(val_a=None, val_b=None), CUDA),
    ("spspmm_fused", dict(val_c=None, dtype=9), CUDA),
    ("spspmm_fused", dict(capacity=0), CUDA), ("spspmm_fused", dict(capacity=0, col_c=None), CUDA),
    *negatives("spspmm_fused", "M", "Kd", "N", "nnz_a", "nnz_b", "capacity"),
    ("spspmm_fused", dict(rowptr_c=None), INVALID),
    ("spspmm_fused", dict(M=M_MAX), CUDA), ("spspmm_fused", dict(M=M_MAX + 1), UNSUPPORTED),
    ("spspmm_fused", dict(M=1 << 40), UNSUPPORTED),
    ("spspmm_fused", dict(dtype=F16), UNSUPPORTED), ("spspmm_fused", dict(dtype=9), UNSUPPORTED),
    ("spspmm_fused", dict(ws=None), WORKSPACE), ("spspmm_fused", dict(wsb=1), WORKSPACE),
    ("spspmm_fused", dict(M=0, wsb=1), WORKSPACE),
    ("spspmm_fused", dict(M=0), CUDA), ("spspmm_fused", dict(nnz_a=0), CUDA), ("spspmm_fused", dict(nnz_b=0), CUDA),
    *[("spspmm_fused", {n: None}, CUDA) for n in (*OPERANDS, "col_c")],
    ("spspmm_fused", dict(capacity=-1, M=M_MAX + 1), INVALID),
    ("spspmm_fused", dict(M=M_MAX + 1, dtype=F16), UNSUPPORTED),
    ("spspmm_fused", dict(M=M_MAX + 1, ws=None), UNSUPPORTED),
    ("spspmm_fused", dict(dtype=F16, ws=None), UNSUPPORTED),
]


def _label(i, row):
    fn, over, _ = row
    return f"{i:03d}-{fn}(" + ",".join(f"{k}={v}" for k, v in over.items()) + ")"


def _run():
    """In the child: refuse to call anything if a CUDA device is visible, else print every row's result as JSON."""
    import torch
    assert torch.cuda.device_count() == 0, "a CUDA device is visible: no entry point is called"
    from pytorch_sparse_b200 import _lib
    codes = []
    for fn, over, _ in TABLE:
        args = dict(BASE[fn])
        assert set(over) <= set(args), (fn, over)
        args.update(over)
        codes.append(getattr(_lib.lib, "tsb200_" + fn)(*args.values()))
    print(json.dumps(codes))


@pytest.fixture(scope="module")
def codes():
    here = Path(__file__).resolve().parent
    code = f"import sys; sys.path[:0] = [{str(here.parent)!r}, {str(here)!r}]; import {Path(__file__).stem} as t; t._run()"
    flags = ["-s"] if sys.flags.no_user_site else []
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, *flags, "-c", code], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, f"the table failed to run:\n{r.stdout[-4000:]}\n{r.stderr[-4000:]}"
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_covers_every_entry_point():
    from pytorch_sparse_b200 import _lib
    src = Path(__file__).resolve().parent.parent / "pytorch_sparse_b200" / "csrc" / "spspmm.cu"
    names = {line.split("(")[0].split()[-1] for line in src.read_text().splitlines() if line.startswith('extern "C"')}
    assert len(names) == 5 and names == {"tsb200_" + fn for fn in BASE}
    for fn, args in BASE.items():
        assert len(args) == len(_lib.SIGNATURES["tsb200_" + fn][1]), fn
    assert {fn for fn, _, _ in TABLE} == set(BASE)


@pytest.mark.parametrize("i", range(len(TABLE)), ids=[_label(i, row) for i, row in enumerate(TABLE)])
def test_return_code(codes, i):
    fn, over, want = TABLE[i]
    got = codes[i]
    if want == CUDA:
        assert got > 0, f"tsb200_{fn}({over}): {got}, want a CUDA error (validation passed)"
    elif want == SIZE:
        assert got > 0, f"tsb200_{fn}({over}): {got}, want a workspace size"
    else:
        assert got == want, f"tsb200_{fn}({over}): {got}, want {want}"
