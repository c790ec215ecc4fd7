"""One APPNP hop X_{h+1} = (1 - a) A X_h + a H at C2 (1M x 1M, 16 nnz/row, uniform columns), a = 0.1, F = 128 and
256, per-row scales, planned calls. The entry values are folded once: v' = (1 - a) v.

    a  bf16 APPNP hop        ops.spmm_fw(rowptr, col, v'_bf16, x_bf16, "sum", plan), then out.add_(h_bf16, alpha=a)
    b  unfused FP8 hop       ops.spmm_fw_fp8(..., v'_f32, x8, scale, "sum", float32, plan), + (a h_scale) * h8 in
                             torch, then quantize_fp8: the e4m3 operand of the next hop through float copies
    c  fused FP8 hop         ops.spmm_fw_fp8_quant(..., residual=h8, residual_scale=a h_scale): the residual is added
                             in the store epilogue, before the row is quantised
    d  spmm_fp8_quant        c without the residual: what the residual costs is c - d

The variants alternate within one job (ROUNDS rounds of CALLS timed calls each, CUDA events); each round's ms per hop
is printed with the card's name and power limit, the median and the spread ((max - min) / min). Also printed: the
per-hop peak of torch.cuda.max_memory_allocated above what the operands hold, for a, b and c; the byte model (the
residual adds M K + 4 M read bytes); and the error of 10 chained APPNP hops of b and c against fp64 APPNP of the
dequantised x_0 and h, as a fraction of the computed bound (x_h the dequantised operand of hop h, z the fp32 result,
A' = (1 - a) A):
    e_{h+1} = |A'| e_h + (deg + 4) 2^-24 |A'| |x_h|      (the fp32 chain, the weight, the fold of v' and of 1 - a)
              + 3 * 2^-24 |a H| + 2^-24 |z|              (the fold of a h_scale and of a, the product; the add)
              + 1/2 ulp_e4m3(z / s) s (1 + 2^-22) + 2^-22 |z|

    python scripts/time_fp8_appnp.py [--rounds 5] [--calls 40] [--hops 10] [--out DIR]
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
from time_fp8_hops import e4m3_half_ulp, peak_extra  # noqa: E402

ALPHA = 0.1
U = 2.0 ** -24


def chain_error(rp, c, v, x8, s, h8, hs, hop, hops):
    """Largest |got - ref| / bound of each of `hops` chained APPNP hops (fp64 reference and bound on the GPU); `v` =
    the unfolded values."""
    v64 = v.double() * (1 - ALPHA)
    a64 = v64.abs()
    deg = (rp[1:] - rp[:-1]).double().view(-1, 1)
    aH = ALPHA * h8.double() * hs.double().view(-1, 1)
    ref = x8.double() * s.double().view(-1, 1)
    e = torch.zeros_like(ref)
    res = []
    for _ in range(hops):
        xh = x8.double() * s.double().view(-1, 1)
        x8, s = hop(x8, s)
        q, sd = x8.double(), s.double().view(-1, 1)
        got = q * sd
        hu = e4m3_half_ulp(q) * sd
        ref = ops.spmm_fw(rp, c, v64, ref, "sum")[0] + aH
        zabs = got.abs() + hu
        e = (ops.spmm_fw(rp, c, a64, e, "sum")[0] + (deg + 4) * U * ops.spmm_fw(rp, c, a64, xh.abs(), "sum")[0]
             + 3 * U * aH.abs() + U * zabs + hu * (1 + 2.0 ** -22) + 2.0 ** -22 * zabs)
        r = (got - ref).abs() / e
        res.append(round(float(r[e > 0].max()), 4))
        del xh, q, got, hu, zabs, r
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--hops", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/time_fp8_appnp.jsonl")
    args = ap.parse_args()
    lines = [dict(card(), kind="card")]
    print(json.dumps(lines[0]), flush=True)

    w = bench.WORKLOADS["c2"]
    rowptr_h, col_h, value_h, N = bench.gen_matrix(w, 0, 1)
    rp, c = rowptr_h.to(DEV), col_h.to(DEV)
    v32 = value_h.float().to(DEV)
    va32 = v32 * (1 - ALPHA)             # folded once, outside the loop
    vab = va32.bfloat16()
    M, E = w["M"], c.numel()
    plan = ops.spmm_plan(rp, E)
    for F in (128, 256):
        x = bench.gen_dense(dict(w, F=F), 0, N).to(DEV)
        h = bench.gen_dense(dict(w, F=F), 1, M).to(DEV)
        xb, hb = x.bfloat16(), h.bfloat16()
        x8, sr = ts.quantize_fp8(x, per_row=True)
        h8, hs = ts.quantize_fp8(h, per_row=True)
        rs = hs * ALPHA
        del x, h

        def hop_a():
            out = ops.spmm_fw(rp, c, vab, xb, "sum", plan=plan)[0]
            return out.add_(hb, alpha=ALPHA)

        def hop_b(x8_, s_):
            y = ops.spmm_fw_fp8(rp, c, va32, x8_, s_, "sum", torch.float32, plan=plan)[0]
            return ts.quantize_fp8(y + rs.view(-1, 1) * h8.float(), True)

        def hop_c(x8_, s_):
            return ops.spmm_fw_fp8_quant(rp, c, va32, x8_, s_, "sum", plan=plan, residual=h8, residual_scale=rs)[:2]

        variants = {
            "a_bf16_add": hop_a,
            "b_fp8_f32_add_quantize": lambda: hop_b(x8, sr),
            "c_fp8_residual": lambda: hop_c(x8, sr),
            "d_fp8_quant": lambda: ops.spmm_fw_fp8_quant(rp, c, va32, x8, sr, "sum", plan=plan),
        }
        model = {"kind": "bytes", "F": F, "M": M, "E": E,
                 "residual_read_GB (MK + 4M)": (M * F + 4 * M) / 1e9,
                 "gathered_GB (E K + 4 E)": (E * F + 4 * E) / 1e9,
                 "index_value_GB (12 E)": 12 * E / 1e9,
                 "written_GB (MK + 4M)": (M * F + 4 * M) / 1e9}
        print(json.dumps(model), flush=True)
        lines.append(model)
        for fn in variants.values():   # warm-up: module load, grid-size queries
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        mem = {"kind": "peak_alloc", "F": F,
               "MB_above_operands": {k: round(peak_extra(variants[k]) / 2 ** 20, 1)
                                     for k in ("a_bf16_add", "b_fp8_f32_add_quantize", "c_fp8_residual")}}
        print(json.dumps(mem), flush=True)
        lines.append(mem)
        ms = {k: [] for k in variants}
        for _ in range(args.rounds):
            for k, fn in variants.items():
                ms[k].append(time_calls(fn, args.calls))
        med = {k: statistics.median(ts_) for k, ts_ in ms.items()}
        res = {"kind": "time", "F": F, "calls_per_round": args.calls,
               "ms": {k: [round(t, 4) for t in ts_] for k, ts_ in ms.items()},
               "median_ms": {k: round(t, 4) for k, t in med.items()},
               "spread": {k: round((max(ts_) - min(ts_)) / min(ts_), 4) for k, ts_ in ms.items()},
               "c_over_d": round(med["c_fp8_residual"] / med["d_fp8_quant"] - 1, 4)}
        print(json.dumps(res), flush=True)
        lines.append(res)
        if F == 128:
            acc = {"kind": "chain_error_over_bound", "F": F, "hops": args.hops,
                   "b_fp8_f32_add_quantize": chain_error(rp, c, v32, x8, sr, h8, hs, hop_b, args.hops),
                   "c_fp8_residual": chain_error(rp, c, v32, x8, sr, h8, hs, hop_c, args.hops)}
            print(json.dumps(acc), flush=True)
            lines.append(acc)
        del xb, hb, x8, sr, h8, hs, rs
        torch.cuda.empty_cache()

    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        with open(Path(args.out) / "time_fp8_appnp.jsonl", "w") as f:
            f.write("".join(json.dumps(l) + "\n" for l in lines))


if __name__ == "__main__":
    main()
