"""Edge scores s_e = <a[row_e], b[col_e]> over the C2 matrix of bench.py (1M x 1M, 16 nnz/row, uniform columns) at
F = 128 and F = 256:

    (a) torch      (a[row] * b[col]).sum(-1) in bf16          (what users write today; three E x F temporaries)
    (b) sddmm      ts.sddmm(src, a, b) in bf16                (tsb200_spmm_value_bw, row-wise kernel)
    (c) fp8_row    ts.sddmm_fp8(src, a8, sa[M], b8, sb[N], torch.bfloat16)
    (d) fp8_tensor ts.sddmm_fp8(src, a8, sa[], b8, sb[], torch.bfloat16)

The arms alternate within one job (ROUNDS rounds of CALLS timed calls each, CUDA events); printed: each round's ms per
call, the median and the spread (max - min) / min, the peak torch.cuda.max_memory_allocated above the operands of one
call, a byte model, and the card's name and power limit read in the same run. Checks in the same run:
(b) against (a) within the sum of both rounding bounds, and (c), (d) against the f32 `sddmm` of their dequantised
operands within the FP8 kernel's bound plus the f32 kernel's; each printed as the largest error over its bound (<= 1).

    python scripts/time_sddmm.py [--rounds 5] [--calls 40] [--out DIR]
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

DEV = "cuda:0"
U = 2.0 ** -24
BF16_HALF_ULP, BF16_HALF_MIN = 2.0 ** -8, 2.0 ** -134     # relative 1/2 ulp of bf16, half its smallest subnormal


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


def peak_above(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


def max_ratio(err, bound):
    return float((err / bound).max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/time_sddmm.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_sddmm.py measures on the GPU: no CUDA device")
    lines = [dict(card(), kind="card")]
    print(json.dumps(lines[0]), flush=True)

    w = bench.WORKLOADS["c2"]
    rowptr_h, col_h, _, N = bench.gen_matrix(w, 0, 1)
    M = w["M"]
    src = ts.SparseTensor(rowptr=rowptr_h.to(DEV), col=col_h.to(DEV), sparse_sizes=(M, N), is_sorted=True,
                          trust_data=True)
    row, col = src.storage.row(), src.storage.col()
    E = col.numel()
    for F in (128, 256):
        a = bench.gen_dense(dict(w, F=F), 1, M).to(DEV).bfloat16()
        b = bench.gen_dense(dict(w, F=F), 0, N).to(DEV).bfloat16()
        a8r, sar = ts.quantize_fp8(a, per_row=True)
        b8r, sbr = ts.quantize_fp8(b, per_row=True)
        a8t, sat = ts.quantize_fp8(a, per_row=False)
        b8t, sbt = ts.quantize_fp8(b, per_row=False)
        arms = {
            "torch": lambda: (a[row] * b[col]).sum(-1),
            "sddmm": lambda: ts.sddmm(src, a, b),
            "fp8_row": lambda: ts.sddmm_fp8(src, a8r, sar, b8r, sbr, torch.bfloat16),
            "fp8_tensor": lambda: ts.sddmm_fp8(src, a8t, sat, b8t, sbt, torch.bfloat16),
        }
        # byte model: index stream, one gathered b row per entry, one a row per CSR row, the scores; the torch
        # expression gathers an a row per entry too (and writes and reads its E x F temporaries, not counted here)
        model = {"kind": "bytes", "F": F, "E": E, "M": M}
        for k, s, idx, a_rows in (("torch", 2, 16, E), ("sddmm", 2, 8, M), ("fp8_row", 1, 8, M),
                                  ("fp8_tensor", 1, 8, M)):
            gb = {"index": idx * E, "gathered_rows": E * F * s, "row_operand": a_rows * F * s, "scores": 2 * E}
            if k == "fp8_row":
                gb["scales"] = 4 * E + 4 * M
            model[k] = {n: round(v / 1e9, 4) for n, v in gb.items()}
            model[k]["total_GB"] = round(sum(gb.values()) / 1e9, 4)
            model[k]["data_sheet_minimum_ms"] = round(sum(gb.values()) / 3.35e12 * 1e3, 4)
        print(json.dumps(model), flush=True)
        lines.append(model)

        outs, peak = {}, {}
        for k, fn in arms.items():          # warm-up (module load, grid-size queries) and peak memory of one call
            for _ in range(2):
                fn()
            outs[k], peak[k] = peak_above(fn)
        lines.append({"kind": "peak_MB_above_operands", "F": F, **{k: round(v / 2 ** 20, 1) for k, v in peak.items()}})
        print(json.dumps(lines[-1]), flush=True)

        ms = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, fn in arms.items():
                ms[k].append(time_calls(fn, args.calls))
        res = {"kind": "time", "F": F, "calls_per_round": args.calls,
               "ms": {k: [round(t, 4) for t in v] for k, v in ms.items()},
               "median_ms": {k: round(statistics.median(v), 4) for k, v in ms.items()},
               "spread": {k: round((max(v) - min(v)) / min(v), 4) for k, v in ms.items()}}
        print(json.dumps(res), flush=True)
        lines.append(res)

        # checks. (a) rounds every product to bf16 (1/2 ulp: 2^-9 relative) and sums in fp32; (b) sums exact products
        # in fp32 (F + 1 roundings); both round once to bf16.
        acc = {"kind": "accuracy", "F": F}
        S = ts.sddmm(src, a.float().abs(), b.float().abs()).double() * (1 + 2.0 ** -10)
        ref_a, ref_b = outs["torch"].double(), outs["sddmm"].double()
        e = (2.0 ** -9 + 2 * (F + 1) * U) * S
        bound = e + BF16_HALF_ULP * (ref_a.abs() + ref_b.abs() + 2 * e) + 2 * BF16_HALF_MIN
        acc["sddmm_vs_torch_over_bound"] = max_ratio((ref_a - ref_b).abs(), bound)
        acc["sddmm_vs_torch_max_abs"] = float((ref_a - ref_b).abs().max())
        # (c), (d): fl32(s_e * d_e) against the f32 kernel on the dequantised operands fl32(q * s); both within
        # (F + 1) 2^-24 of the exact dot of the dequantised values, the FP8 arm 3 more roundings (two dequantisations
        # it does not perform, and s_e), then 1/2 ulp of bf16
        for k, a8, sa, b8, sb in (("fp8_row", a8r, sar, b8r, sbr), ("fp8_tensor", a8t, sat, b8t, sbt)):
            af = a8.float() * (sa.view(-1, 1) if sa.dim() else sa)
            bf = b8.float() * (sb.view(-1, 1) if sb.dim() else sb)
            ref = ts.sddmm(src, af, bf).double()
            Sq = ts.sddmm(src, af.abs(), bf.abs()).double() * (1 + 2.0 ** -10)
            got = outs[k].double()
            e = (2 * F + 6) * U * Sq
            bound = e + BF16_HALF_ULP * (ref.abs() + e) + BF16_HALF_MIN
            acc[k + "_vs_dequantised_f32_over_bound"] = max_ratio((got - ref).abs(), bound)
            acc[k + "_vs_sddmm_bf16_max_abs"] = float((got - ref_b).abs().max())
            del af, bf, ref, Sq, got
        acc["sddmm_max_abs_score"] = float(ref_b.abs().max())
        print(json.dumps(acc), flush=True)
        lines.append(acc)
        del a, b, a8r, b8r, a8t, b8t, outs, S, ref_a, ref_b, bound, e
        torch.cuda.empty_cache()

    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        with open(Path(args.out) / "time_sddmm.jsonl", "w") as f:
            f.write("".join(json.dumps(line) + "\n" for line in lines))


if __name__ == "__main__":
    main()
