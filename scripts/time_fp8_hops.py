"""One FP8 propagation hop X_{h+1} = A X_h at C2 (1M x 1M, 16 nnz/row, uniform columns), F = 128 and 256, planned:

    a  bf16 -> bf16          ops.spmm_fw(rowptr, col, value_bf16, x_bf16, "sum", plan)
    b  fp8 -> bf16           ops.spmm_fw_fp8(..., x8, scale [N], "sum", bf16, plan)
    c  b, then quantize_fp8  the e4m3 operand of the next hop from the bf16 result
    d  fp8 -> fp8            ops.spmm_fw_fp8_quant(..., x8, scale [N], "sum", plan): quantised in the kernel epilogue

The variants alternate within one job (ROUNDS rounds of CALLS timed calls each, CUDA events); each round's ms per hop
is printed with the card's name and power limit, the median and the spread ((max - min) / min). Also printed: the
per-hop peak of torch.cuda.max_memory_allocated above what the operands hold, for a, c and d; the written-byte model
(2 M K for a bf16 result against M K + 4 M for e4m3 and its scales); and the error of 3 chained hops of c and d
against fp64 propagation of the first dequantised operand, as a fraction of the computed bound
    e_{h+1} = |A| e_h + (deg + 2) 2^-24 |A| |x_h| + 1/2 ulp_e4m3(y / s) s (1 + 2^-22) + 2^-22 |y|
(for c plus 2^-8 |y|: the bf16 rounding of y before it is quantised, and torch's CUDA division).

    python scripts/time_fp8_hops.py [--rounds 5] [--calls 40] [--out DIR]
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


def e4m3_half_ulp(y):
    _, e = torch.frexp(y.abs())
    e = torch.clamp(e - 1, min=-6)
    return torch.ldexp(torch.full_like(y, 0.5), (e - 3).to(torch.int32))


def peak_extra(fn):
    """Bytes allocated at the peak of one call, above what was allocated before it (the call's outputs included)."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del out
    return peak


def chain_error(rp, c, v, x8, s, hop, extra_rel, hops=3):
    """Largest |got - ref| / bound of each of `hops` chained hops (fp64 reference and bound on the GPU); `v` = the
    values the hop uses."""
    v64, a64 = v.double(), v.double().abs()
    deg = (rp[1:] - rp[:-1]).double().view(-1, 1)
    ref = x8.double() * s.double().view(-1, 1)
    e = torch.zeros_like(ref)
    res = []
    for _ in range(hops):
        xh = x8.double() * s.double().view(-1, 1)
        x8, s = hop(x8, s)
        q, sd = x8.double(), s.double().view(-1, 1)
        got = q * sd
        hu = e4m3_half_ulp(q) * sd
        ref = ops.spmm_fw(rp, c, v64, ref, "sum")[0]
        yabs = got.abs() + hu
        e = (ops.spmm_fw(rp, c, a64, e, "sum")[0] + (deg + 2) * 2.0 ** -24 * ops.spmm_fw(rp, c, a64, xh.abs(), "sum")[0]
             + hu * (1 + 2.0 ** -22) + (2.0 ** -22 + extra_rel) * yabs)
        r = (got - ref).abs() / e
        res.append(float(r[e > 0].max()))
        del xh, q, got, hu, yabs, r
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/time_fp8_hops.jsonl")
    args = ap.parse_args()
    lines = [dict(card(), kind="card")]
    print(json.dumps(lines[0]), flush=True)

    w = bench.WORKLOADS["c2"]
    rowptr_h, col_h, value_h, N = bench.gen_matrix(w, 0, 1)
    rp, c = rowptr_h.to(DEV), col_h.to(DEV)
    vb, v32 = value_h.bfloat16().to(DEV), value_h.float().to(DEV)
    M, E = w["M"], c.numel()
    plan = ops.spmm_plan(rp, E)
    for F in (128, 256):
        x = bench.gen_dense(dict(w, F=F), 0, N).to(DEV)
        xb = x.bfloat16()
        x8, sr = ts.quantize_fp8(x, per_row=True)
        del x

        def hop_c(x8_, s_):
            return ts.quantize_fp8(ops.spmm_fw_fp8(rp, c, vb, x8_, s_, "sum", torch.bfloat16, plan=plan)[0], True)

        def hop_d(x8_, s_):
            return ops.spmm_fw_fp8_quant(rp, c, v32, x8_, s_, "sum", plan=plan)[:2]

        variants = {
            "a_bf16": lambda: ops.spmm_fw(rp, c, vb, xb, "sum", plan=plan),
            "b_fp8_to_bf16": lambda: ops.spmm_fw_fp8(rp, c, vb, x8, sr, "sum", torch.bfloat16, plan=plan),
            "c_fp8_bf16_quantize": lambda: hop_c(x8, sr),
            "d_fp8_quant": lambda: hop_d(x8, sr),
        }
        model = {"kind": "bytes", "F": F, "M": M, "E": E,
                 "written_GB": {"bf16 (2MK)": 2 * M * F / 1e9, "e4m3 + scales (MK + 4M)": (M * F + 4 * M) / 1e9},
                 "note": "b and c also carry a bf16 value per nnz, d an f32 one (2 more bytes per nnz)"}
        print(json.dumps(model), flush=True)
        lines.append(model)
        for fn in variants.values():   # warm-up: module load, grid-size queries
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        mem = {"kind": "peak_alloc", "F": F,
               "MB_above_operands": {k: round(peak_extra(variants[k]) / 2 ** 20, 1)
                                     for k in ("a_bf16", "c_fp8_bf16_quantize", "d_fp8_quant")}}
        print(json.dumps(mem), flush=True)
        lines.append(mem)
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
        if F == 128:
            acc = {"kind": "chain_error_over_bound", "F": F, "hops": 3,
                   "c_fp8_bf16_quantize": chain_error(rp, c, vb, x8, sr, hop_c, 2.0 ** -8),
                   "d_fp8_quant": chain_error(rp, c, v32, x8, sr, hop_d, 0.0)}
            print(json.dumps(acc), flush=True)
            lines.append(acc)
        del xb, x8, sr
        torch.cuda.empty_cache()

    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        with open(Path(args.out) / "time_fp8_hops.jsonl", "w") as f:
            f.write("".join(json.dumps(l) + "\n" for l in lines))


if __name__ == "__main__":
    main()
