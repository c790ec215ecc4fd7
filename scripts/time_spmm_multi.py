"""Multi-aggregation SpMM against the composition it replaces, at C2 (1M x 1M, 16 nnz/row) and the power-law C3 shape.

    a  composition   one spmm per aggregator, and for std a second mean over an x * x temporary with the squared
                     values (the messages' squares v^2 x^2): mean, min, max, var = (mean - mean^2).clamp(0), std;
                     concatenated
    b  fused         spmm_multi(src, x, aggrs).flatten(1)

for aggrs (mean, min, max, std) and (sum, max), at C2 bf16 F = 128, C2 f32 F = 64 and C3 f32 F = 64 (scripts/
bench_extra.py's matrix). Each arm is timed as a forward under no_grad and as forward + backward to x and the values.
The arms alternate within one job (ROUNDS rounds of CALLS timed calls each, CUDA events); every line carries the card's
name and power limit, the median and the spread ((max - min) / min), the peak of max_memory_allocated above the
operands, and the largest difference of the composition from the fused result in the same run.

    python scripts/time_spmm_multi.py [--rounds 5] [--calls 20] [--out DIR]
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


def composition(A, x, aggrs):
    parts = []
    mean = None
    for a in aggrs:
        if a in ("mean", "var", "std") and mean is None:
            mean = tsm.spmm(A, x, "mean")
        if a == "sum":
            parts.append(tsm.spmm(A, x, "sum"))
        elif a == "mean":
            parts.append(mean)
        elif a in ("min", "max"):
            parts.append(tsm.spmm(A, x, a))
        else:
            v = A.storage.value()
            A2 = A if v is None else A.set_value(v * v, layout="csr")   # the messages' squares: v^2 x^2
            var = (tsm.spmm(A2, x * x, "mean") - mean * mean).clamp(min=0)
            std = torch.where(var > 1e-5, var.clamp(min=1e-5).sqrt(), torch.zeros_like(var))
            parts.append(var if a == "var" else std)
    return torch.cat(parts, -1)


def fused(A, x, aggrs):
    return tsm.spmm_multi(A, x, list(aggrs)).flatten(1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/time_spmm_multi.jsonl")
    args = ap.parse_args()
    lines = [dict(card(), kind="card")]
    print(json.dumps(lines[0]), flush=True)

    def emit(d):
        print(json.dumps(d), flush=True)
        lines.append(d)

    for wname, dtype, F in (("c2", torch.bfloat16, 128), ("c2", torch.float32, 64), ("c3", torch.float32, 64)):
        w = bench.WORKLOADS[wname]
        rowptr_h, col_h, value_h, N = bench.gen_matrix(w, 0, 1)
        M = w["M"]
        A = ts.SparseTensor(rowptr=rowptr_h.to(DEV), col=col_h.to(DEV), value=value_h.to(DEV, dtype),
                            sparse_sizes=(M, N), is_sorted=True, trust_data=True)
        x = bench.gen_dense(dict(w, F=F), 0, N).to(DEV, dtype)
        for aggrs in (("mean", "min", "max", "std"), ("sum", "max")):
            with torch.no_grad():
                arms = {"a_composition": lambda: composition(A, x, aggrs), "b_fused": lambda: fused(A, x, aggrs)}
                outs = {k: fn() for k, fn in arms.items()}
                res = rounds(arms, args.rounds, args.calls)
                peak = {k: round(peak_extra(fn) / 2 ** 20, 1) for k, fn in arms.items()}
            diff = float((outs["a_composition"].double() - outs["b_fused"].double()).abs().max())
            del outs
            emit({"kind": "forward", "workload": wname, "dtype": str(dtype), "F": F, "aggrs": list(aggrs), **res,
                  "fused_over_composition": round(res["median_ms"]["b_fused"] / res["median_ms"]["a_composition"], 4),
                  "peak_MB_above_operands": peak, "max_abs_diff_composition_vs_fused": diff})

            Ag = A.requires_grad_()
            xg = x.detach().requires_grad_()
            go = torch.randn(M, len(aggrs) * F, device=DEV, dtype=dtype)

            def fb(f):
                def run():
                    xg.grad = None
                    Ag.storage.value().grad = None
                    f(Ag, xg, aggrs).backward(go)
                    return xg.grad
                return run

            arms = {"a_composition": fb(composition), "b_fused": fb(fused)}
            res = rounds(arms, args.rounds, max(args.calls // 4, 3))
            peak = {k: round(peak_extra(fn) / 2 ** 20, 1) for k, fn in arms.items()}
            ga = arms["a_composition"]().double().clone()
            gb = arms["b_fused"]().double()
            emit({"kind": "forward_backward", "workload": wname, "dtype": str(dtype), "F": F, "aggrs": list(aggrs),
                  **res,
                  "fused_over_composition": round(res["median_ms"]["b_fused"] / res["median_ms"]["a_composition"], 4),
                  "peak_MB_above_operands": peak, "max_abs_diff_grad_x": float((ga - gb).abs().max()),
                  "max_abs_grad_x": float(gb.abs().max())})
            A.requires_grad_(False)
            del arms, ga, gb, go, xg
            torch.cuda.empty_cache()
        del A, x
        torch.cuda.empty_cache()
    if args.out:
        out = Path(args.out)
        out.mkdir(parents=True, exist_ok=True)
        (out / "time_spmm_multi.jsonl").write_text("".join(json.dumps(d) + "\n" for d in lines))


if __name__ == "__main__":
    main()
