"""SpMM forward at C2 (1M x 1M, 16 nnz/row, uniform columns) over an FP8 (e4m3) dense operand against the bf16 operand,
at F = 128 and F = 256, all with bf16 output and the cached plan:

    bf16       ops.spmm_fw(rowptr, col, value, x_bf16, "sum", plan)        (what matmul runs)
    fp8_tensor ops.spmm_fw_fp8(..., x8, scale [],  "sum", bf16, plan)
    fp8_row    ops.spmm_fw_fp8(..., x8, scale [N], "sum", bf16, plan)

The variants alternate within one job (ROUNDS rounds of CALLS timed calls each, CUDA events); each round's ms per call
is printed with the card's name and power limit. Also printed: the gathered-byte model, and per fp8 variant the largest
error against the exactly dequantised operand (fp64 reference through the library's fp64 path) relative to the kernel's
bound (must be <= 1), and the largest difference to the bf16 result relative to the quantisation bound.

    python scripts/time_fp8.py [--rounds 5] [--calls 40] [--out DIR]
"""
import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

import bench  # noqa: E402
import pytorch_sparse_b200 as ts  # noqa: E402
from pytorch_sparse_b200 import ops  # noqa: E402

DEV = "cuda:0"


def card():
    name = torch.cuda.get_device_name(DEV)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = f"unavailable ({e})"
    return {"name": name, "power_limit,max_sm_clock": q}


def time_calls(fn, calls):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/time_fp8.jsonl")
    args = ap.parse_args()
    lines = [dict(card(), kind="card")]
    print(json.dumps(lines[0]), flush=True)

    w = bench.WORKLOADS["c2"]
    rowptr_h, col_h, value_h, N = bench.gen_matrix(w, 0, 1)
    rp, c = rowptr_h.to(DEV), col_h.to(DEV)
    v = value_h.bfloat16().to(DEV)
    M, E = w["M"], c.numel()
    plan = ops.spmm_plan(rp, E)
    for F in (128, 256):
        x = bench.gen_dense(dict(w, F=F), 0, N).to(DEV)
        xb = x.bfloat16()
        x8t, st = ts.quantize_fp8(x, per_row=False)
        x8r, sr = ts.quantize_fp8(x, per_row=True)
        variants = {
            "bf16": lambda: ops.spmm_fw(rp, c, v, xb, "sum", plan=plan),
            "fp8_tensor": lambda: ops.spmm_fw_fp8(rp, c, v, x8t, st, "sum", torch.bfloat16, plan=plan),
            "fp8_row": lambda: ops.spmm_fw_fp8(rp, c, v, x8r, sr, "sum", torch.bfloat16, plan=plan),
        }
        gathered = {"bf16": E * F * 2, "fp8_tensor": E * F, "fp8_row": E * F}
        model = {"kind": "bytes", "F": F, "E": E,
                 "gathered_dense_rows_GB": {k: b / 1e9 for k, b in gathered.items()},
                 "per_row_scale_sectors_GB": E * 32 / 1e9,
                 "note": "uniform random columns over an operand larger than L2: the gathered rows come from DRAM"}
        print(json.dumps(model), flush=True)
        lines.append(model)
        for fn in variants.values():   # warm-up: module load, grid-size queries, plan
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        ms = {k: [] for k in variants}
        for _ in range(args.rounds):
            for k, fn in variants.items():
                ms[k].append(time_calls(fn, args.calls))
        res = {"kind": "time", "F": F, "calls_per_round": args.calls,
               "ms": {k: [round(t, 4) for t in ts_] for k, ts_ in ms.items()},
               "median_ms": {k: round(statistics.median(ts_), 4) for k, ts_ in ms.items()},
               "spread": {k: round((max(ts_) - min(ts_)) / min(ts_), 4) for k, ts_ in ms.items()}}
        print(json.dumps(res), flush=True)
        lines.append(res)

        # accuracy: fp8 against its exactly dequantised operand, and against the bf16 result
        out_b = variants["bf16"]()[0].double()
        v64 = v.double()
        deg = (rp[1:] - rp[:-1]).double().view(-1, 1)
        acc = {"kind": "accuracy", "F": F}
        for k, x8, s in (("fp8_tensor", x8t, st), ("fp8_row", x8r, sr)):
            s_rows = (s.expand(N) if s.dim() == 0 else s).double().view(-1, 1)
            xd = x8.double() * s_rows
            ref = ops.spmm_fw(rp, c, v64, xd, "sum")[0]
            S = ops.spmm_fw(rp, c, v64.abs(), xd.abs(), "sum")[0]
            out = variants[k]()[0].double()
            e = (deg + 2) * 2.0 ** -24 * S
            kern_bound = e + (ref.abs() + e) * 2.0 ** -8 + 2.0 ** -134      # + 1/2 ulp of bf16
            # quantisation: |x - q s| <= 2^-4 |x| + 2^-10 s per element (1/2 ulp of e4m3); x itself differs from its
            # bf16 copy by 2^-9 |x|; both results are rounded to bf16
            xq = ((2.0 ** -4 + 2.0 ** -9) * x.double().abs() + 2.0 ** -10 * s_rows).contiguous()
            q_bound = ops.spmm_fw(rp, c, v64.abs(), xq, "sum")[0] + 2.0 ** -8 * (out.abs() + out_b.abs()) + 2.0 ** -133
            acc[k] = {"max_err_over_kernel_bound": float(((out - ref).abs() / kern_bound).max()),
                      "max_diff_to_bf16_over_quant_bound": float(((out - out_b).abs() / q_bound).max()),
                      "max_abs_diff_to_bf16": float((out - out_b).abs().max()),
                      "max_abs_bf16_out": float(out_b.abs().max())}
            del xd, ref, S, out, xq, q_bound
        print(json.dumps(acc), flush=True)
        lines.append(acc)
        del x, xb, x8t, x8r, out_b
        torch.cuda.empty_cache()

    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        with open(Path(args.out) / "time_fp8.jsonl", "w") as f:
            f.write("".join(json.dumps(l) + "\n" for l in lines))


if __name__ == "__main__":
    main()
