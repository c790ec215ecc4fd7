"""Go/no-go probe for a feature-sliced SpMM forward (DESIGN §3.1), measured with the library's existing kernels.

Times, alternated `--rounds` times on the C2 matrix (1M x 1M, 16 nnz/row, bf16):
  * the full product at F = 128 (X is 256 MB, 5x the L2);
  * one slice pass: the same matrix against a contiguous [N, 16] X (32 MB, one 32 B slice of every row);
  * the same pass with N = 250 000 columns (8 MB X: certainly L2-resident);
  * the slice-major copy of the F = 128 operand, x.view(N, 8, 16).permute(1, 0, 2).contiguous().
Projected sliced time = 8 * t(pass) + t(copy).
"""
import argparse, sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
import torch
from pytorch_sparse_b200 import ops
from util import fast_random_csr

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--steps", type=int, default=30)
a = ap.parse_args()
dev = "cuda:0"
M, F, S = 1_000_000, 128, 16


def timed(fn, steps=a.steps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def problem(N):
    _, rowptr, col = fast_random_csr(M, N, 16, 1, dev)
    g = torch.Generator(device=dev).manual_seed(2)
    val = (torch.rand(col.numel(), generator=g, device=dev) + 0.5).bfloat16()
    return rowptr, col, val, g


rowptr, col, val, g = problem(M)
x = torch.randn(M, F, generator=g, device=dev).bfloat16()
x16 = torch.randn(M, S, generator=g, device=dev).bfloat16()
rp_s, col_s, val_s, g_s = problem(250_000)
x16_s = torch.randn(250_000, S, generator=g_s, device=dev).bfloat16()
cases = {
    "F=128 (today)": lambda: ops.spmm_fw(rowptr, col, val, x, "sum"),
    "F=16 pass, N=1M (32 MB X)": lambda: ops.spmm_fw(rowptr, col, val, x16, "sum"),
    "F=16 pass, N=250k (8 MB X)": lambda: ops.spmm_fw(rp_s, col_s, val_s, x16_s, "sum"),
    "slice-major copy of X": lambda: x.view(M, F // S, S).permute(1, 0, 2).contiguous(),
}
res = {k: [] for k in cases}
for r in range(a.rounds):
    for k, fn in cases.items():
        res[k].append(timed(fn))
print(f"{torch.cuda.get_device_name(0)}, L2 {torch.cuda.get_device_properties(0).L2_cache_size >> 20} MB, "
      f"E = {col.numel()}")
for k, v in res.items():
    print(f"{k:32s} " + "  ".join(f"{t:.4f}" for t in v) + " ms")
med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
proj = (F // S) * med["F=16 pass, N=1M (32 MB X)"] + med["slice-major copy of X"]
print(f"projected sliced = {F // S} x pass + copy = {proj:.4f} ms = {proj / med['F=128 (today)']:.3f} x today")
