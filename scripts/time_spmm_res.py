"""SpMM with a fused residual at C2 (1M x 1M, 16 nnz/row), planned calls, against the unfused forms it replaces.

    a  spmm + add_        ops.spmm_fw(...) then out.add_(r, alpha=s)
    b  spmm + mul_ + add_ ops.spmm_fw(...) over the unfolded values, then out.mul_(1 - s).add_(r, alpha=s)
                          (PyG's APPNP form)
    c  fused              ops.spmm_fw_res(..., residual=r, residual_scale=s)
    d  spmm alone         what the residual costs is c - d

for bf16 F = 128 and 256 and f32 F = 64; then a 10-hop APPNP chain, forward and forward + backward, a against c; and
GCN propagation with structural self-loops (adj + I, normalised, one SpMM over E + M entries) against the per-row
residual form (values d^-1/2 w d^-1/2, residual x, residual_scale 1/d). The arms alternate within one job (ROUNDS
rounds of CALLS timed calls each, CUDA events); each line carries the card's name and power limit, the median and the
spread ((max - min) / min), the peak of max_memory_allocated above the operands, and the largest difference of each arm
from c in the same run. Byte model: the residual adds one coalesced read of M K s bytes, against 3 M K s for add_ and
5 M K s for mul_ + add_.

    python scripts/time_spmm_res.py [--rounds 5] [--calls 40] [--hops 10] [--out DIR]
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

ALPHA = 0.1


def rounds(variants, n_rounds, calls):
    for fn in variants.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in variants}
    for _ in range(n_rounds):
        for k, fn in variants.items():
            ms[k].append(time_calls(fn, calls))
    return {"ms": {k: [round(t, 4) for t in v] for k, v in ms.items()},
            "median_ms": {k: round(statistics.median(v), 4) for k, v in ms.items()},
            "spread": {k: round((max(v) - min(v)) / min(v), 4) for k, v in ms.items()}}


def maxdiff(outs, ref):
    return {k: float((o.double() - outs[ref].double()).abs().max()) for k, o in outs.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--hops", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/time_spmm_res.jsonl")
    args = ap.parse_args()
    lines = [dict(card(), kind="card")]
    print(json.dumps(lines[0]), flush=True)

    def emit(d):
        print(json.dumps(d), flush=True)
        lines.append(d)

    w = bench.WORKLOADS["c2"]
    rowptr_h, col_h, value_h, N = bench.gen_matrix(w, 0, 1)
    rp, c = rowptr_h.to(DEV), col_h.to(DEV)
    M, E = w["M"], c.numel()
    plan = ops.spmm_plan(rp, E)
    for dtype, F in ((torch.bfloat16, 128), (torch.bfloat16, 256), (torch.float32, 64)):
        v = (value_h.float() * (1 - ALPHA)).to(DEV, dtype)   # (1 - a) folded into the values once
        v1 = value_h.float().to(DEV, dtype)                  # unfolded, for (b)
        x = bench.gen_dense(dict(w, F=F), 0, N).to(DEV, dtype)
        r = bench.gen_dense(dict(w, F=F), 1, M).to(DEV, dtype)
        s = torch.tensor(ALPHA, device=DEV)
        arms = {
            "a_spmm_add": lambda: ops.spmm_fw(rp, c, v, x, "sum", plan=plan)[0].add_(r, alpha=ALPHA),
            "b_spmm_mul_add": lambda: ops.spmm_fw(rp, c, v1, x, "sum", plan=plan)[0].mul_(1 - ALPHA).add_(r, alpha=ALPHA),
            "c_fused": lambda: ops.spmm_fw_res(rp, c, v, x, r, s, plan=plan),
            "d_spmm": lambda: ops.spmm_fw(rp, c, v, x, "sum", plan=plan)[0],
        }
        outs = {k: fn() for k, fn in arms.items() if k != "d_spmm"}
        res = rounds(arms, args.rounds, args.calls)
        es = torch.tensor([], dtype=dtype).element_size()
        emit({"kind": "hop", "dtype": str(dtype), "F": F, **res,
              "c_over_d": round(res["median_ms"]["c_fused"] / res["median_ms"]["d_spmm"] - 1, 4),
              "peak_MB_above_operands": {k: round(peak_extra(fn) / 2 ** 20, 1) for k, fn in arms.items()},
              "max_abs_diff_vs_c": maxdiff(outs, "c_fused"), "max_abs_c": float(outs["c_fused"].abs().max()),
              "bytes_GB": {"residual_read (M K s)": M * F * es / 1e9, "add_ (3 M K s)": 3 * M * F * es / 1e9,
                           "mul_add_ (5 M K s)": 5 * M * F * es / 1e9}})
        del arms, outs, x, r, v, v1
        torch.cuda.empty_cache()

    # 10-hop APPNP chain in bf16, F = 128, forward and forward + backward
    F = 128
    A = ts.SparseTensor(rowptr=rp, col=c, value=(value_h.float() * (1 - ALPHA)).to(DEV, torch.bfloat16),
                        sparse_sizes=(M, N))
    h0 = bench.gen_dense(dict(w, F=F), 1, M).to(DEV, torch.bfloat16)
    s = torch.tensor(ALPHA, device=DEV)

    def chain(fused, backward):
        h = h0.detach().requires_grad_(backward)
        x = h
        for _ in range(args.hops):
            x = A.spmm(x, residual=h, residual_scale=s) if fused else A.spmm(x).add(h, alpha=ALPHA)
        if backward:
            x.float().sum().backward()
        return x.detach()

    chains = {"a_fw": lambda: chain(False, False), "c_fw": lambda: chain(True, False),
              "a_fwbw": lambda: chain(False, True), "c_fwbw": lambda: chain(True, True)}
    res = rounds(chains, args.rounds, max(1, args.calls // 10))
    emit({"kind": "appnp_chain", "hops": args.hops, "F": F, **res,
          "max_rel_diff_a_vs_c": float((chain(False, False).double() - (xc := chain(True, False).double())).abs().max()
                                       / xc.abs().max())})
    del A, h0, chains

    # GCN propagation, F = 128 bf16: structural self-loops against the per-row residual
    row = torch.repeat_interleave(torch.arange(M, device=DEV), rp[1:] - rp[:-1])
    adj = ts.SparseTensor(row=row, col=c, value=torch.ones(E, device=DEV), sparse_sizes=(M, N))
    loops = adj + ts.SparseTensor.eye(M, dtype=torch.float32, device=DEV)
    lr, lc, _ = loops.coo()
    d = (rp[1:] - rp[:-1]).double() + 1
    dl = torch.bincount(lr, minlength=M).double()
    gl = loops.set_value((dl.rsqrt()[lr] * dl.rsqrt()[lc]).to(torch.bfloat16), layout="coo")
    ga = adj.set_value((d.rsqrt()[row] * d.rsqrt()[c]).to(torch.bfloat16), layout="coo")
    x = bench.gen_dense(dict(w, F=F), 0, N).to(DEV, torch.bfloat16)
    inv = (1 / d).float()
    gcn = {"structural_self_loops": lambda: gl.spmm(x), "residual_self_loops": lambda: ga.spmm(x, residual=x,
                                                                                              residual_scale=inv)}
    outs = {k: fn() for k, fn in gcn.items()}
    res = rounds(gcn, args.rounds, args.calls)
    emit({"kind": "gcn", "F": F, "E": E, "E_with_loops": lr.numel(), **res,
          "peak_MB_above_operands": {k: round(peak_extra(fn) / 2 ** 20, 1) for k, fn in gcn.items()},
          "max_abs_diff_vs_residual": maxdiff(outs, "residual_self_loops")})

    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        with open(Path(args.out) / "time_spmm_res.jsonl", "w") as f:
            f.write("".join(json.dumps(l) + "\n" for l in lines))


if __name__ == "__main__":
    main()
