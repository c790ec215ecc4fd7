"""Multi-head SpMM / SDDMM at C2 (1M x 1M, 16 nnz per row, uniform columns, planned calls).

Arms per (H, D, dtype):
  (a) torch gather:  index_add_(0, row, x[col] * alpha[..., None])  and  (a[row] * b[col]).sum(-1)
  (b) per-head loop of spmm / sddmm over contiguous head slices x[:, h]
  (c) spmm_heads / sddmm_heads
  (d) one attention layer (README recipe), forward + backward, against the same layer in torch gather form
Method: warm-up, then 5 alternated rounds of 40 calls per arm; median and spread (max - min over rounds) of the per-call
time, and max_memory_allocated above the operands. Every arm's output is checked against (c) in the same run, within
the summation bound of the dtype the arm accumulates in.

    python scripts/time_heads.py [--rounds 5] [--calls 40] [--out time_heads.json]
"""
import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import pytorch_sparse_b200 as ts
from pytorch_sparse_b200 import SparseTensor, ops

SHAPES = [(8, 16, torch.bfloat16), (4, 64, torch.bfloat16), (8, 8, torch.float32)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return q or torch.cuda.get_device_name()


def timed(fn, calls):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(calls):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / calls


def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    r = fn()
    torch.cuda.synchronize()
    p = torch.cuda.max_memory_allocated() - base
    del r
    return p


def run_arms(arms, rounds, calls):
    for fn in arms.values():   # warm-up (plans, CSC views, allocator)
        fn()
        fn()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            times[k].append(timed(fn, calls))
    return {k: {"median_ms": statistics.median(v), "spread_ms": max(v) - min(v),
                "peak_above_operands_MB": peak(arms[k]) / 2 ** 20} for k, v in times.items()}


def close(x, ref, S, n, dtype, what):
    """|x - ref| <= (n + 2) eps_T S: both sides summed n terms of total magnitude S, the torch arms in the dtype itself
    (bf16 products and bf16 index_add_), the native ones in fp32; returns the largest |x - ref| / S"""
    eps = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -23
    d = (x.float() - ref.float()).abs()
    assert bool((d <= (n + 2) * eps * S.float() + 1e-30).all()), f"{what}: max |diff| {d.max().item():.3e}"
    return (d / S.float().clamp(min=1e-30)).max().item()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda")
    N, deg = args.n, 16
    g = torch.Generator(device=dev).manual_seed(0)
    row = torch.arange(N, device=dev).repeat_interleave(deg)
    col = torch.randint(0, N, (N * deg,), device=dev, generator=g)
    col = col.view(N, deg).sort(dim=1).values.view(-1)
    adj0 = SparseTensor(row=row, col=col, sparse_sizes=(N, N), is_sorted=True, trust_data=True)
    rowptr = adj0.storage.rowptr()
    E = col.numel()
    res = {"card_and_power_limit": card(), "N": N, "nnz_per_row": deg, "rounds": args.rounds, "calls": args.calls,
           "shapes": []}
    print(res["card_and_power_limit"], flush=True)
    for H, D, dt in SHAPES:
        x = torch.randn(N, H, D, device=dev, dtype=dt, generator=g)
        a = torch.randn(N, H, D, device=dev, dtype=dt, generator=g)
        alpha = torch.rand(E, H, device=dev, dtype=dt, generator=g)
        adj = adj0.set_value(alpha, layout="csr")
        slices = [x[:, h].contiguous() for h in range(H)]
        aslices = [a[:, h].contiguous() for h in range(H)]
        vals = [alpha[:, h].contiguous() for h in range(H)]
        ops.spmm_plan(rowptr, E)
        with torch.no_grad():
            spmm = {
                "a_gather": lambda: torch.zeros(N, H, D, device=dev, dtype=dt).index_add_(0, row, x[col] * alpha[..., None]),
                "b_per_head": lambda: torch.stack([ops.spmm_fw(rowptr, col, vals[h], slices[h], "sum")[0]
                                                   for h in range(H)], 1),
                "c_spmm_heads": lambda: adj.spmm_heads(x),
            }
            sddmm = {
                "a_gather": lambda: (a[row] * x[col]).sum(-1),
                "b_per_head": lambda: torch.stack([adj0.sddmm(aslices[h], slices[h]) for h in range(H)], 1),
                "c_sddmm_heads": lambda: adj0.sddmm_heads(a, x),
            }
            ref = spmm["c_spmm_heads"]()
            S = adj0.set_value(alpha.abs(), layout="csr").spmm_heads(x.abs())
            errs = {k: close(fn(), ref, S, deg, dt, f"spmm {k} H={H} D={D}") for k, fn in spmm.items()}
            sref = sddmm["c_sddmm_heads"]()
            S = adj0.sddmm_heads(a.abs(), x.abs())
            errs.update({"sddmm_" + k: close(fn(), sref, S, D, dt, f"sddmm {k} H={H} D={D}") for k, fn in sddmm.items()})
            t_spmm = run_arms(spmm, args.rounds, args.calls)
            t_sddmm = run_arms(sddmm, args.rounds, args.calls)
        q = a.clone().requires_grad_()
        k = x.clone().requires_grad_()
        v = x.flip(0).contiguous().requires_grad_()

        def layer_native():
            s = adj0.sddmm_heads(q, k) * D ** -0.5
            m = adj0.set_value(s.detach(), layout="csr").max(dim=1)
            p = (s - m[row]).exp()
            al = p / adj0.set_value(p, layout="csr").sum(dim=1)[row]
            out = adj0.set_value(al, layout="csr").spmm_heads(v)
            out.sum().backward()
            return out.detach()

        def layer_gather():
            s = (q[row] * k[col]).sum(-1) * D ** -0.5
            m = torch.full((N, H), float("-inf"), device=dev, dtype=dt).scatter_reduce(0, row[:, None].expand(-1, H),
                                                                                    s.detach(), "amax")
            p = (s - m[row]).exp()
            den = torch.zeros(N, H, device=dev, dtype=dt).index_add(0, row, p)
            al = p / den[row]
            out = torch.zeros(N, H, D, device=dev, dtype=dt).index_add(0, row, v[col] * al[..., None])
            out.sum().backward()
            return out.detach()

        lg, ln = layer_gather(), layer_native()
        errs["layer_gather"] = (lg.float() - ln.float()).abs().max().item()   # outputs are convex mixes of rows of v
        assert errs["layer_gather"] <= (0.1 if dt == torch.bfloat16 else 1e-4), f"layer H={H} D={D}: {errs}"
        t_layer = run_arms({"d_layer_native": layer_native, "d_layer_gather": layer_gather}, args.rounds,
                           max(1, args.calls // 4))
        entry = {"H": H, "D": D, "dtype": str(dt).split(".")[-1], "spmm": t_spmm, "sddmm": t_sddmm,
                 "layer_fw_bw": t_layer, "max_rel_err_vs_native": errs}
        res["shapes"].append(entry)
        print(json.dumps(entry), flush=True)
        del x, a, alpha, adj, slices, aslices, vals, q, k, v
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
