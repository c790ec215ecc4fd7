"""SpMM with a residual without a GPU: the operator schema, TorchScript, the exports, every argument error of
`ops.spmm_fw_res` and `spmm(..., residual=)`, and the return codes of tsb200_spmm_fw_res.

The return-code table runs in a child interpreter that sees no CUDA device, as tests/test_rowsplit_abi_cpu.py does: a
call that passes validation fails at its first CUDA call with a positive CUDA error (`CUDA`). A short workspace tells the
vector path (which reports it, -3) from the generic kernel (which reads no workspace)."""
import importlib
import json
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import ops
from test_rowsplit_abi_cpu import (BF16, BIG, CUDA, E_MAX, F16, F32, F64, I32, INVALID, MAX, MEAN, MIN, MIS, N_MAX, P,
                                   PLANNED, SUM, UNSUPPORTED, W, WORKSPACE, negatives, plan_faults, workspace_faults)

tsm = importlib.import_module("pytorch_sparse_b200.matmul")  # the module; the package's `matmul` is a function
FN = "spmm_fw_res"
BASE = dict(rowptr=P, col=P, value=P, mat=P, res=P, res_scale=P, res_stride=1, out=P, M=64, N=64, K=64, E=1000,
            dtype=BF16, reduce=SUM, plan=None, pb=0, ns=0, nl=0, nsl=0, ws=W, wsb=BIG, stream=None)

TABLE = [
    (FN, {}, CUDA), (FN, dict(PLANNED), CUDA), (FN, dict(reduce=MEAN, res_stride=0), CUDA),
    (FN, dict(dtype=F32, value=None), CUDA), (FN, dict(dtype=F16), CUDA),
    # the generic kernel: fp64, partial widths; it reads no workspace and no plan
    (FN, dict(dtype=F64, wsb=1), CUDA), (FN, dict(PLANNED, dtype=F64, pb=1), CUDA),
    (FN, dict(K=12, wsb=1), CUDA), (FN, dict(dtype=F32, K=3, wsb=1), CUDA),
    *negatives(FN, "M", "N", "K", "E", "ns", "nl", "nsl"),
    (FN, dict(reduce=-1), INVALID), (FN, dict(reduce=4), INVALID),
    (FN, dict(dtype=9), INVALID), (FN, dict(dtype=-1), INVALID), (FN, dict(dtype=I32), UNSUPPORTED),
    (FN, dict(res_stride=2), INVALID), (FN, dict(res_stride=-1), INVALID),
    (FN, dict(reduce=MIN), UNSUPPORTED), (FN, dict(reduce=MAX), UNSUPPORTED),
    (FN, dict(M=0), 0), (FN, dict(K=0), 0), (FN, dict(M=0, res=None), 0),
    *[(FN, {n: None}, INVALID) for n in ("rowptr", "out", "res", "res_scale", "col", "mat")],
    (FN, dict(E=0, col=None, mat=None, ws=None), CUDA),    # every row empty: the residual alone
    (FN, dict(E=0, res=None), INVALID),
    # alignments: res_scale to its element size; res 16 B for the vector path, else the generic kernel
    (FN, dict(res_scale=P + 2), UNSUPPORTED), (FN, dict(res_scale=P + 4), CUDA),
    (FN, dict(dtype=F64, res_scale=P + 4), UNSUPPORTED), (FN, dict(dtype=F64, res_scale=P + 8), CUDA),
    (FN, dict(res=P + 8, wsb=1), CUDA), (FN, dict(res=P + 16, wsb=1), WORKSPACE),
    (FN, dict(mat=P + 8, wsb=1), CUDA), (FN, dict(mat=P + 16, wsb=1), WORKSPACE),
    (FN, dict(out=P + 8, wsb=1), CUDA),
    (FN, dict(col=P + 4, wsb=1), CUDA), (FN, dict(col=P + 8, wsb=1), WORKSPACE),
    (FN, dict(value=P + 2, wsb=1), CUDA), (FN, dict(value=P + 4, wsb=1), WORKSPACE),
    # workspace and plan faults of the vector path
    *workspace_faults(FN),
    *plan_faults(FN, **PLANNED),
    (FN, dict(PLANNED, ws=MIS, wsb=1), WORKSPACE),
    # extent limits of the vector path, at and just past each boundary
    (FN, dict(E=E_MAX, wsb=1), WORKSPACE), (FN, dict(E=E_MAX + 1, wsb=1), CUDA),
    (FN, dict(N=N_MAX, wsb=1), WORKSPACE), (FN, dict(N=N_MAX + 1, wsb=1), CUDA),
    (FN, dict(dtype=F32, K=(1 << 29) - 4, wsb=1), WORKSPACE), (FN, dict(dtype=F32, K=1 << 29, wsb=1), CUDA),
]


def _run():
    """In the child: refuse to call anything if a CUDA device is visible, else print every row's result as JSON."""
    assert torch.cuda.device_count() == 0, "a CUDA device is visible: no entry point is called"
    from pytorch_sparse_b200 import _lib
    codes = []
    for fn, over, _ in TABLE:
        args = dict(BASE)
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


def test_signature():
    from pytorch_sparse_b200 import _lib
    assert len(BASE) == len(_lib.SIGNATURES["tsb200_" + FN][1])
    header = (Path(__file__).resolve().parent.parent / "include" / "tsb200.h").read_text()
    assert "TSB200_API int tsb200_spmm_fw_res(" in header


@pytest.mark.parametrize("i", range(len(TABLE)),
                         ids=[f"{i:03d}-" + ",".join(f"{k}={v}" for k, v in o.items()) for i, (_, o, _) in enumerate(TABLE)])
def test_return_code(codes, i):
    fn, over, want = TABLE[i]
    got = codes[i]
    if want == CUDA:
        assert got > 0, f"tsb200_{fn}({over}): {got}, want a CUDA error (validation passed)"
    else:
        assert got == want, f"tsb200_{fn}({over}): {got}, want {want}"


# ---- Python surface ---------------------------------------------------------------------------------------------------
def test_schema_and_exports():
    assert ts.torch_ops.REGISTERED["tsb200"]
    schema = str(torch.ops.tsb200.spmm_res.default._schema)
    assert "Tensor residual, Tensor? residual_scale, str reduce" in schema
    assert callable(ops.spmm_fw_res) and ops.SPMMRes is not None and callable(ops.spmm_res)
    assert callable(tsm.spmm_res) and ts.SparseTensor.spmm is not None


def test_torchscript():
    def f(src: ts.SparseTensor, x: torch.Tensor, r: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
        return tsm.spmm(src, x, "mean", residual=r, residual_scale=s)

    g = torch.jit.script(f)
    assert "tsb200::spmm_res" in str(g.inlined_graph)


def test_scale_without_residual():
    A = ts.SparseTensor(row=torch.tensor([0]), col=torch.tensor([0]), sparse_sizes=(1, 1))
    with pytest.raises(ValueError, match="residual_scale needs a residual"):
        tsm.spmm(A, torch.ones(1, 1), residual_scale=torch.ones(()))


@pytest.fixture
def no_device_check(monkeypatch):
    """The device checks come first and need CUDA tensors; past them every check runs on CPU tensors."""
    monkeypatch.setattr(ops, "_check_cuda", lambda t, name: None)


def test_cpu_tensors_refused():
    x = torch.ones(3, 4)
    with pytest.raises(RuntimeError, match="rowptr must be CUDA tensor"):
        ops.spmm_fw_res(torch.zeros(3, dtype=torch.long), torch.zeros(0, dtype=torch.long), None, x, torch.ones(2, 4))


@pytest.mark.parametrize("kw,msg", [
    (dict(reduce="max"), "a residual is only added to reduce='sum' / 'mean' results, not min / max"),
    (dict(reduce="min"), "a residual is only added to reduce='sum' / 'mean' results, not min / max"),
    (dict(reduce="prod"), "unknown reduce 'prod'"),
    (dict(mat=torch.ones(2, 3, 4)), "a residual needs a 2-D dense operand \\[N, K\\], got 3-D"),
    (dict(residual=torch.ones(2, 4, dtype=torch.float64)), "residual must have the dense operand's dtype torch.float32"),
    (dict(residual=torch.ones(3, 4)), "residual must have the result's shape \\[M, K\\] = \\[2, 4\\], got \\[3, 4\\]"),
    (dict(residual=torch.ones(2, 5)), "residual must have the result's shape"),
    (dict(residual=torch.ones(2)), "residual must have the result's shape"),
    (dict(residual=torch.ones(4, 2).t()), "residual must be contiguous"),
    (dict(residual_scale=torch.ones((), dtype=torch.float64)),
     "residual_scale must be torch.float32 for a torch.float32 operand, got torch.float64"),
    (dict(residual_scale=torch.ones(3)), "residual_scale must have shape \\[\\] or \\[M\\] = \\[2\\], got \\[3\\]"),
    (dict(residual_scale=torch.ones(2, 1)), "residual_scale must have shape"),
    (dict(mat=torch.ones(3, 4, dtype=torch.float64), residual=torch.ones(2, 4, dtype=torch.float64),
          residual_scale=torch.ones(())), "residual_scale must be torch.float64 for a torch.float64 operand"),
])
def test_argument_errors(no_device_check, kw, msg):
    args = dict(rowptr=torch.zeros(3, dtype=torch.long), col=torch.zeros(0, dtype=torch.long), value=None,
                mat=torch.ones(3, 4), residual=torch.ones(2, 4), residual_scale=None, reduce="sum")
    args.update(kw)
    err = ValueError if kw.get("reduce") == "prod" else RuntimeError
    with pytest.raises(err, match=msg):
        ops.spmm_fw_res(**args)
