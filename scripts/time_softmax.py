"""Sparse softmax over [E, H] scores: the native `softmax` against the compositions it replaces.

Workloads: the C2 structure (1M x 1M, 16 entries per row, uniform columns) and the C3 power-law matrix
(bench.gen_matrix(WORKLOADS["c3"]), rows of up to ~50 000 entries); scores [E, H] with H in {1, 8} in bf16 and H = 8 in
f32, softmax over rows, and once over columns (C2, H = 8, bf16).
Arms per workload:
  (a) the README composition (segment max, exp, segment sum, divide), forward alone and forward + backward
  (b) the torch gather form (scatter_reduce amax, index_add), forward alone and forward + backward
  (c) the native softmax, forward alone, backward alone (the kernel over a stored result) and forward + backward
  (d) at C2 only: one attention layer (time_heads.py's three (H, D) shapes), forward + backward, the README composition
      against the native softmax
Method (as time_heads.py): warm-up, then 5 alternated rounds of 40 calls per arm; median and spread (max - min over
rounds) of the per-call time, and max_memory_allocated above the operands. Every arm's result is checked against (c)
in the same run: |x - ref| <= (R + n + 8) eps_T ref + eps_T 2^-8 for an arm that works in the storage dtype T, R the
entry's |s - m| and n its segment's length (the gather form adds in T; the native result itself is tested against
fp64 in tests/test_softmax_gpu.py).
Byte model of (c): forward 8 (S + 1) + 2 s E H (+ 8 E for the column permutation), backward 8 (S + 1) + 3 s E H, as a
rate against the H100 SXM data-sheet 3.35 TB/s.

    python scripts/time_softmax.py [--rounds 5] [--calls 40] [--out time_softmax.json]
"""
import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import bench  # noqa: E402
import pytorch_sparse_b200 as ts  # noqa: E402
from pytorch_sparse_b200 import SparseTensor, ops  # noqa: E402

HBM = 3.35e12
LAYER_SHAPES = [(8, 16, torch.bfloat16), (4, 64, torch.bfloat16), (8, 8, torch.float32)]


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
    for fn in arms.values():   # warm-up (CSR / CSC views, allocator)
        fn()
        fn()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            times[k].append(timed(fn, calls))
    return {k: {"median_ms": statistics.median(v), "spread_ms": max(v) - min(v),
                "peak_above_operands_MB": peak(arms[k]) / 2 ** 20} for k, v in times.items()}


def c2_matrix(dev, N=1 << 20, deg=16):
    g = torch.Generator(device=dev).manual_seed(0)
    row = torch.arange(N, device=dev).repeat_interleave(deg)
    col = torch.randint(0, N, (N * deg,), device=dev, generator=g).view(N, deg).sort(dim=1).values.view(-1)
    return SparseTensor(row=row, col=col, sparse_sizes=(N, N), is_sorted=True, trust_data=True)


def c3_matrix(dev):
    rp, c, _, N = bench.gen_matrix(bench.WORKLOADS["c3"], 0, 1)
    return SparseTensor(rowptr=rp.to(dev), col=c.to(dev), sparse_sizes=(rp.numel() - 1, N), is_sorted=True,
                        trust_data=True)


def softmax_arms(adj, s, g, dim):
    """forward and forward + backward of the three forms, over scores s [E, H] with upstream gradient g"""
    st = adj.storage
    seg = st.row() if dim == 1 else st.col()
    S = adj.sparse_size(1 - dim)
    H = s.size(1)

    def composed(x):
        m = adj.set_value(x.detach(), layout="csr").max(dim=dim)
        p = (x - m[seg]).exp()
        return p / adj.set_value(p, layout="csr").sum(dim=dim)[seg]

    def gather(x):
        idx = seg[:, None].expand(-1, H)
        m = torch.full((S, H), float("-inf"), device=x.device, dtype=x.dtype).scatter_reduce(0, idx, x.detach(), "amax")
        p = (x - m[seg]).exp()
        return p / torch.zeros(S, H, device=x.device, dtype=x.dtype).index_add(0, seg, p)[seg]

    def native(x):
        return ts.softmax(adj.set_value(x, layout="csr"), dim).storage.value()

    sr = s.detach().requires_grad_()
    ptr, perm = (st.rowptr(), None) if dim == 1 else (st.colptr(), st.csr2csc())
    alpha = native(s)
    fw = {"a_composed_fw": lambda: composed(s), "b_gather_fw": lambda: gather(s), "c_native_fw": lambda: native(s),
          "c_native_bw": lambda: ops.segment_softmax_bw(ptr, alpha, g, perm)}
    fwbw = {"a_composed_fw_bw": lambda: torch.autograd.grad(composed(sr), sr, g)[0],
            "b_gather_fw_bw": lambda: torch.autograd.grad(gather(sr), sr, g)[0],
            "c_native_fw_bw": lambda: torch.autograd.grad(native(sr), sr, g)[0]}
    return fw, fwbw, alpha


def check(arms, ref, s, adj, dim, what):
    """|x - ref| <= (R + n + 8) eps_T ref + eps_T 2^-8 (see the module docstring); returns the largest |x - ref|"""
    eps = 2.0 ** -8 if ref.dtype == torch.bfloat16 else 2.0 ** -23
    st = adj.storage
    seg = st.row() if dim == 1 else st.col()
    m = adj.set_value(s, layout="csr").max(dim=dim).float()
    n = (st.rowcount() if dim == 1 else st.colcount())[seg].float()[:, None]
    R = (m[seg] - s.float()).abs() + n
    worst = 0.0
    for k, fn in arms.items():
        with torch.no_grad():
            x = fn().float()
        d = (x - ref.float()).abs()
        assert bool((d <= (R + 8) * eps * ref.float() + eps * 2 ** -8).all()), f"{what} {k}: max |diff| {d.max():.3e}"
        worst = max(worst, d.max().item())
    return worst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda")
    res = {"card_and_power_limit": card(), "rounds": args.rounds, "calls": args.calls, "softmax": [], "layer": []}
    print(res["card_and_power_limit"], flush=True)
    gen = torch.Generator(device=dev).manual_seed(1)
    cases = [("c2", 1, 1, torch.bfloat16), ("c2", 1, 8, torch.bfloat16), ("c2", 1, 8, torch.float32),
             ("c2", 0, 8, torch.bfloat16), ("c3", 1, 1, torch.bfloat16), ("c3", 1, 8, torch.bfloat16),
             ("c3", 1, 8, torch.float32)]
    mats = {"c2": c2_matrix(dev), "c3": c3_matrix(dev)}
    for name, dim, H, dt in cases:
        adj = mats[name]
        E, S = adj.nnz(), adj.sparse_size(1 - dim)
        s = torch.randn(E, H, device=dev, dtype=dt, generator=gen) * 2
        g = torch.randn(E, H, device=dev, dtype=dt, generator=gen)
        fw, fwbw, alpha = softmax_arms(adj, s, g, dim)
        err = check({k: v for k, v in fw.items() if k != "c_native_bw"}, alpha, s, adj, dim, f"{name} dim={dim} H={H}")
        t = run_arms(fw, args.rounds, args.calls)
        t.update(run_arms(fwbw, args.rounds, args.calls))
        sz = s.element_size()
        bytes_fw = 8 * (S + 1) + 2 * sz * E * H + (8 * E if dim == 0 else 0)
        bytes_bw = 8 * (S + 1) + 3 * sz * E * H + (8 * E if dim == 0 else 0)
        entry = {"matrix": name, "dim": dim, "S": S, "E": E, "H": H, "dtype": str(dt).split(".")[-1],
                 "max_abs_diff_vs_native": err, "times": t,
                 "model_bytes_fw": bytes_fw, "model_bytes_bw": bytes_bw,
                 "fw_rate_of_3.35TBs": bytes_fw / (t["c_native_fw"]["median_ms"] * 1e-3) / HBM,
                 "bw_rate_of_3.35TBs": bytes_bw / (t["c_native_bw"]["median_ms"] * 1e-3) / HBM}
        res["softmax"].append(entry)
        print(json.dumps(entry), flush=True)
        del s, g, fw, fwbw, alpha
        torch.cuda.empty_cache()
    del mats["c3"]
    adj0 = mats["c2"]
    N = adj0.sparse_size(0)
    row = adj0.storage.row()
    for H, D, dt in LAYER_SHAPES:
        q = torch.randn(N, H, D, device=dev, dtype=dt, generator=gen).requires_grad_()
        k = torch.randn(N, H, D, device=dev, dtype=dt, generator=gen).requires_grad_()
        v = torch.randn(N, H, D, device=dev, dtype=dt, generator=gen).requires_grad_()

        def layer_composed():
            s = adj0.sddmm_heads(q, k) * D ** -0.5
            m = adj0.set_value(s.detach(), layout="csr").max(dim=1)
            p = (s - m[row]).exp()
            al = p / adj0.set_value(p, layout="csr").sum(dim=1)[row]
            out = adj0.set_value(al, layout="csr").spmm_heads(v)
            out.sum().backward()
            return out.detach()

        def layer_native():
            s = adj0.sddmm_heads(q, k) * D ** -0.5
            out = adj0.set_value(s, layout="csr").softmax(dim=1).spmm_heads(v)
            out.sum().backward()
            return out.detach()

        diff = (layer_composed().float() - layer_native().float()).abs().max().item()  # convex mixes of rows of v
        assert diff <= (0.1 if dt == torch.bfloat16 else 1e-4), f"layer H={H} D={D}: {diff}"
        t = run_arms({"d_layer_composed": layer_composed, "d_layer_native": layer_native}, args.rounds,
                     max(1, args.calls // 4))
        entry = {"H": H, "D": D, "dtype": str(dt).split(".")[-1], "max_abs_diff": diff, "layer_fw_bw": t}
        res["layer"].append(entry)
        print(json.dumps(entry), flush=True)
        del q, k, v
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
