"""SpMM forward, C2-style inputs: column panels against the single launch (development helper).

A is split into P contiguous column blocks, one launch per block with an fp32 partial (tsb200_spmm_fw_acc), so that
each launch gathers from N/P dense rows only.

    python scripts/sweep_col_panels.py [--F 128] [--M 1000000] [--panels 2,4]
"""
import argparse, sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
import torch
from pytorch_sparse_b200 import ops
from pytorch_sparse_b200.parallel import split_column_chunks
from util import fast_random_csr

ap = argparse.ArgumentParser()
ap.add_argument("--M", type=int, default=1_000_000)
ap.add_argument("--N", type=int, default=0)
ap.add_argument("--F", type=int, default=128)
ap.add_argument("--deg", type=int, default=16)
ap.add_argument("--panels", default="2,4")
ap.add_argument("--steps", type=int, default=40)
a = ap.parse_args()
dev = "cuda:0"
N = a.N or a.M
row, rowptr, col = fast_random_csr(a.M, N, a.deg, 1, dev)
g = torch.Generator(device=dev).manual_seed(2)
val = (torch.rand(col.numel(), generator=g, device=dev) + 0.5).bfloat16()
x = torch.randn(N, a.F, generator=g, device=dev).bfloat16()
E = col.numel()


def timeit(fn, steps):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


ms = timeit(lambda: ops.spmm_fw(rowptr, col, val, x, "sum"), a.steps)
ref = ops.spmm_fw(rowptr, col, val, x, "sum")[0]
print(f"panels=1  F={a.F} N={N}: {ms:.4f} ms  {2 * E * a.F / ms / 1e6:.0f} GFLOP/s", flush=True)

for P in [int(v) for v in a.panels.split(",") if v != ""]:
    if N % P:
        continue
    parts, _ = split_column_chunks(rowptr, col, val, N, 1, P)      # world = 1: column ids unchanged
    partial = torch.empty(a.M, a.F, dtype=torch.float32, device=dev)
    out = torch.empty(a.M, a.F, dtype=torch.bfloat16, device=dev)

    def run():
        for c, (rp, cl, v) in enumerate(parts):
            ops.spmm_fw_acc(rp, cl, v, x, partial, out, 1 if c == 0 else (3 if c == P - 1 else 2))
    ms = timeit(run, a.steps)
    err = (out.float() - ref.float()).abs().max().item()
    print(f"panels={P}  F={a.F} N={N}: {ms:.4f} ms  (max |diff| vs single pass {err:.3e})", flush=True)
