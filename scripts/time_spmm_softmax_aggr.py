"""Softmax-aggregation SpMM against the compositions it replaces, at C2 (1M x 1M, 16 nnz/row) and the power-law C3 shape.

    a  gather        PyG's SoftmaxAggregation in torch: the messages v * x[col] as an [E, K] tensor, a per-row max by
                     scatter, exp, a per-row sum by scatter, the weighted messages summed by index_add
    b  library       this library's pieces: the [E, K] logits t * v * x[col], the native row softmax over them
                     (`softmax(A, 1)`), then `spmm_heads` with D = 1 and the weights alpha * v
    c  global shift  (no values only) spmm(A, e * x) / spmm(A, e) with e = exp(t x - max_n t x): two SpMMs and no
                     [E, K] temporary; its largest error against the fused result is reported (rows far below the
                     column's global maximum underflow to 0 / 0)
    d  fused         spmm_softmax_aggr(A, x, t)

with a learnable per-column t, at C2 bf16 F = 128, C2 f32 F = 64 (both with and without values) and C3 f32 F = 64.
Each arm is timed as a forward under no_grad and as forward + backward to x, the values and t. The arms alternate
within one job (ROUNDS rounds of CALLS timed calls each, CUDA events); every line carries the card's name and power
limit, the median and the spread ((max - min) / min), the peak of max_memory_allocated above the operands, and the
largest difference of each arm from the fused result in the same run. An arm that runs out of memory is reported
as such.

    python scripts/time_spmm_softmax_aggr.py [--rounds 5] [--calls 20] [--out DIR]
"""
import argparse
import importlib
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

import bench  # noqa: E402
import pytorch_sparse_b200 as ts  # noqa: E402
from time_fp8 import DEV, card  # noqa: E402
from time_fp8_hops import peak_extra  # noqa: E402
from time_spmm_res import rounds  # noqa: E402

tsm = importlib.import_module("pytorch_sparse_b200.matmul")  # the module; the package's `matmul` is a function


def gather(A, x, t):
    rowptr, col, value = A.csr()
    M = rowptr.numel() - 1
    row = A.storage.row()
    msg = x[col] if value is None else x[col] * value[:, None]
    y = (t * msg.float()).to(x.dtype) if x.dtype != torch.float32 else t * msg
    mx = torch.full((M, x.size(1)), float("-inf"), device=x.device, dtype=y.dtype)
    mx = mx.index_reduce(0, row, y.detach(), "amax")
    e = torch.exp(y - mx[row])
    s = torch.zeros_like(mx).index_add(0, row, e)
    alpha = e / s[row]
    return torch.zeros_like(mx).index_add(0, row, alpha * msg)


def library(A, x, t):
    rowptr, col, value = A.csr()
    msg = x[col] if value is None else x[col] * value[:, None]
    y = (t * msg.float()).to(x.dtype)
    alpha = ts.softmax(A.set_value(y, layout="csr"), 1).storage.value()
    w = alpha if value is None else alpha * value[:, None]
    return tsm.spmm_heads(A.set_value(w, layout="csr"), x.unsqueeze(-1)).squeeze(-1)


def global_shift(A, x, t):
    tx = (t * x.float())
    e = torch.exp(tx - tx.amax(0)).to(x.dtype)
    return tsm.spmm(A, e * x, "sum") / tsm.spmm(A, e, "sum")


def fused(A, x, t):
    return tsm.spmm_softmax_aggr(A, x, t)


def guarded(fn):
    """fn, or the string "out of memory" when it runs out of device memory."""
    try:
        return fn()
    except torch.cuda.OutOfMemoryError:
        torch.cuda.empty_cache()
        return "out of memory"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/time_spmm_softmax_aggr.jsonl")
    args = ap.parse_args()
    lines = [dict(card(), kind="card")]
    print(json.dumps(lines[0]), flush=True)

    def emit(d):
        print(json.dumps(d), flush=True)
        lines.append(d)

    for wname, dtype, F, with_value in (("c2", torch.bfloat16, 128, True), ("c2", torch.bfloat16, 128, False),
                                        ("c2", torch.float32, 64, True), ("c2", torch.float32, 64, False),
                                        ("c3", torch.float32, 64, True)):
        w = bench.WORKLOADS[wname]
        rowptr_h, col_h, value_h, N = bench.gen_matrix(w, 0, 1)
        M = w["M"]
        A = ts.SparseTensor(rowptr=rowptr_h.to(DEV), col=col_h.to(DEV),
                            value=value_h.to(DEV, dtype) if with_value else None,
                            sparse_sizes=(M, N), is_sorted=True, trust_data=True)
        A.storage.row()
        x = bench.gen_dense(dict(w, F=F), 0, N).to(DEV, dtype)
        t = torch.linspace(0.5, 2.0, F, device=DEV)
        fns = {"a_gather": gather, "b_library": library, "d_fused": fused}
        if not with_value:
            fns["c_global_shift"] = global_shift
        tag = {"workload": wname, "dtype": str(dtype), "F": F, "values": with_value}

        with torch.no_grad():
            arms = {k: (lambda f=f: f(A, x, t)) for k, f in fns.items()}
            ref = fused(A, x, t).double()
            ok = {}
            diff = {}
            for k, fn in arms.items():
                o = guarded(fn)
                ok[k] = not isinstance(o, str)
                diff[k] = float((o.double() - ref).abs().nan_to_num(float("inf")).max()) if ok[k] else o
                del o
            live = {k: fn for k, fn in arms.items() if ok[k]}
            res = rounds(live, args.rounds, args.calls)
            peak = {k: round(peak_extra(fn) / 2 ** 20, 1) for k, fn in live.items()}
        emit({"kind": "forward", **tag, **res, "peak_MB_above_operands": peak, "max_abs_diff_vs_fused": diff,
              "max_abs_fused": float(ref.abs().max()),
              "fused_over": {k: round(res["median_ms"]["d_fused"] / v, 4) for k, v in res["median_ms"].items()}})
        del ref

        if with_value:
            A.requires_grad_()
        xg = x.detach().requires_grad_()
        tg = t.detach().requires_grad_()
        go = torch.randn(M, F, device=DEV, dtype=dtype)

        def fb(f):
            def run():
                xg.grad = tg.grad = None
                if with_value:
                    A.storage.value().grad = None
                f(A, xg, tg).backward(go)
                return xg.grad
            return run

        arms = {k: fb(f) for k, f in fns.items() if k != "c_global_shift"}
        gref = arms["d_fused"]().double().clone()
        ok, diff = {}, {}
        for k, fn in arms.items():
            o = guarded(fn)
            ok[k] = not isinstance(o, str)
            diff[k] = float((o.double() - gref).abs().max()) if ok[k] else o
        live = {k: fn for k, fn in arms.items() if ok[k]}
        res = rounds(live, args.rounds, max(args.calls // 4, 3))
        peak = {k: round(peak_extra(fn) / 2 ** 20, 1) for k, fn in live.items()}
        emit({"kind": "forward_backward", **tag, **res, "peak_MB_above_operands": peak,
              "max_abs_diff_grad_x_vs_fused": diff, "max_abs_grad_x": float(gref.abs().max()),
              "fused_over": {k: round(res["median_ms"]["d_fused"] / v, 4) for k, v in res["median_ms"].items()}})
        A.requires_grad_(False)
        del arms, gref, go, xg, tg, A, x
        torch.cuda.empty_cache()
    if args.out:
        out = Path(args.out)
        out.mkdir(parents=True, exist_ok=True)
        (out / "time_spmm_softmax_aggr.jsonl").write_text("".join(json.dumps(d) + "\n" for d in lines))


if __name__ == "__main__":
    main()
