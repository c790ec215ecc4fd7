"""FP8 (e4m3) quantisation of a dense operand, N = 1M rows, K = 128 and 256, bf16 and f32 inputs, per-row and
per-tensor scales:

    i   torch     the pure-torch quantize_fp8 expression as it stood before the native quantiser (inlined below)
    ii  native    ts.quantize_fp8 on the CUDA tensor: tsb200_quantize_fp8

and the FP8-result hop at C2 (1M x 1M, 16 nnz/row, uniform columns), per-row input scale, planned:

    c_torch   spmm_fp8 -> bf16, then (i) per row
    c_native  spmm_fp8 -> bf16, then (ii) per row
    d         spmm_fp8_quant (quantised in the kernel's store epilogue)

The arms of a shape alternate within one job (ROUNDS rounds of CALLS timed calls each, CUDA events); the card's name,
power limit and max SM clock are read in the same run. Printed per shape: ms per call of each round, the median and
the spread ((max - min) / min); the byte model (x read once per row scale, twice per tensor scale; N K + 4 N bytes
written) and the rate it gives at the median; the peak of torch.cuda.max_memory_allocated above the input for each
arm; and the number of e4m3 bytes and scales where (ii) differs from (i) run on x.cpu() (must be 0), and where (i) run
on the GPU differs from (i) on the CPU.

    python scripts/time_fp8_quant.py [--rounds 5] [--calls 40] [--out DIR]
"""
import argparse
import json
import statistics
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

import bench  # noqa: E402
import pytorch_sparse_b200 as ts  # noqa: E402
from pytorch_sparse_b200 import ops  # noqa: E402
from time_fp8 import DEV, card, time_calls  # noqa: E402
from time_fp8_hops import peak_extra  # noqa: E402

HBM_TBPS = 3.35   # H100 SXM data sheet


def torch_quantize_fp8(x, per_row):
    """quantize_fp8 as it was before the native quantiser: pure torch, on the device of x."""
    xf = x.float()
    amax = xf.abs().amax(dim=1) if per_row else xf.abs().amax()
    scale = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    x8 = (xf / (scale.unsqueeze(1) if per_row else scale)).to(torch.float8_e4m3fn)
    return x8, scale


def n_differ(a8, a, b8, b):
    return {"x8_bytes": int((a8.cpu().view(torch.uint8) != b8.cpu().view(torch.uint8)).sum()),
            "scales": int((a.cpu().view(torch.int32) != b.cpu().view(torch.int32)).sum())}


def alternate(arms, rounds, calls):
    for fn in arms.values():       # warm-up: module load, grid-size queries
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            ms[k].append(time_calls(fn, calls))
    return {"ms": {k: [round(t, 4) for t in v] for k, v in ms.items()},
            "median_ms": {k: round(statistics.median(v), 4) for k, v in ms.items()},
            "spread": {k: round((max(v) - min(v)) / min(v), 4) for k, v in ms.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/time_fp8_quant.jsonl")
    args = ap.parse_args()
    lines = [dict(card(), kind="card")]
    print(json.dumps(lines[0]), flush=True)

    def emit(d):
        print(json.dumps(d), flush=True)
        lines.append(d)

    w = bench.WORKLOADS["c2"]
    N = w["M"]
    for K in (128, 256):
        base = bench.gen_dense(dict(w, F=K), 0, N)
        for dtype in (torch.bfloat16, torch.float32):
            x = base.to(dtype).to(DEV)
            xc = x.cpu()
            for per_row in (True, False):
                arms = {"i_torch": lambda: torch_quantize_fp8(x, per_row),
                        "ii_native": lambda: ts.quantize_fp8(x, per_row)}
                res = alternate(arms, args.rounds, args.calls)
                size = x.element_size()
                read = N * K * size * (1 if per_row else 2)
                written = N * K + (4 * N if per_row else 4)
                t = res["median_ms"]["ii_native"] * 1e-3
                ref8, refs = torch_quantize_fp8(xc, per_row)
                emit({"kind": "quantize", "N": N, "K": K, "dtype": str(dtype).split(".")[1],
                      "scale": "per_row" if per_row else "per_tensor", "calls_per_round": args.calls, **res,
                      "bytes_model": {"read_MB": read / 1e6, "written_MB": written / 1e6,
                                      "min_ms_at_3.35TBps": round((read + written) / (HBM_TBPS * 1e12) * 1e3, 4),
                                      "native_TBps": round((read + written) / t / 1e12, 3)},
                      "peak_MB_above_input": {k: round(peak_extra(fn) / 2 ** 20, 1) for k, fn in arms.items()},
                      "native_vs_cpu_differ": n_differ(*ts.quantize_fp8(x, per_row), ref8, refs),
                      "torch_gpu_vs_cpu_differ": n_differ(*torch_quantize_fp8(x, per_row), ref8, refs)})
                del ref8, refs
            del x, xc
            torch.cuda.empty_cache()
        del base

    rowptr_h, col_h, value_h, Nc = bench.gen_matrix(w, 0, 1)
    rp, c = rowptr_h.to(DEV), col_h.to(DEV)
    vb, v32 = value_h.bfloat16().to(DEV), value_h.float().to(DEV)
    plan = ops.spmm_plan(rp, c.numel())
    for K in (128, 256):
        x8, sr = ts.quantize_fp8(bench.gen_dense(dict(w, F=K), 0, Nc).to(DEV), True)
        arms = {
            "c_torch": lambda: torch_quantize_fp8(
                ops.spmm_fw_fp8(rp, c, vb, x8, sr, "sum", torch.bfloat16, plan=plan)[0], True),
            "c_native": lambda: ts.quantize_fp8(
                ops.spmm_fw_fp8(rp, c, vb, x8, sr, "sum", torch.bfloat16, plan=plan)[0], True),
            "d_fp8_quant": lambda: ops.spmm_fw_fp8_quant(rp, c, v32, x8, sr, "sum", plan=plan)[:2],
        }
        res = alternate(arms, args.rounds, args.calls)
        emit({"kind": "hop", "K": K, "calls_per_round": args.calls, **res,
              "peak_MB_above_operands": {k: round(peak_extra(fn) / 2 ** 20, 1) for k, fn in arms.items()}})
        del x8, sr
        torch.cuda.empty_cache()

    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        with open(Path(args.out) / "time_fp8_quant.jsonl", "w") as f:
            f.write("".join(json.dumps(l) + "\n" for l in lines))


if __name__ == "__main__":
    main()
