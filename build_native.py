"""Build libtsb200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

    python build_native.py [--force] [--verbose]

Stand-alone on purpose (it lives outside the package): importing `pytorch_sparse_b200` requires the
library to exist, so the build step must not import it.

No torch headers are involved: the library is plain CUDA C++ behind `include/tsb200.h`.
Objects are cached next to the sources (`csrc/_build/`) keyed on source + header mtimes and flags.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent
PKG = ROOT / "pytorch_sparse_b200"
CSRC = PKG / "csrc"
INCLUDE = ROOT / "include"
BUILD = CSRC / "_build"
LIB = PKG / "libtsb200.so"

SOURCES = ["spmm_fw.cu", "spmm_softmax_aggr.cu", "spmm_bw.cu", "convert.cu", "coalesce.cu", "spspmm.cu", "quant.cu",
           "softmax.cu", "host_api.cu"]

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    *GENCODE,
    "-O3", "-lineinfo", "-std=c++17", "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
    "-cudart", "shared",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found (set NVCC=/path/to/nvcc)")


def _stamp(src: Path) -> str:
    h = hashlib.sha1()
    h.update(" ".join(NVCC_FLAGS).encode())
    for f in [src, *sorted(CSRC.glob("*.cuh")), *sorted(INCLUDE.glob("*.h"))]:
        h.update(f.name.encode())
        h.update(str(f.stat().st_mtime_ns).encode())
    return h.hexdigest()


def _compile(src_name: str, force: bool, verbose: bool) -> Path:
    src = CSRC / src_name
    obj = BUILD / (src.stem + ".o")
    stamp_file = BUILD / (src.stem + ".stamp")
    stamp = _stamp(src)
    if not force and obj.exists() and stamp_file.exists() and stamp_file.read_text() == stamp:
        return obj
    cmd = [_nvcc(), *NVCC_FLAGS, "-I", str(INCLUDE), "-c", str(src), "-o", str(obj)]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
        print(" ".join(cmd), flush=True)
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src_name}:\n{res.stdout}\n{res.stderr}")
    if verbose:
        print(res.stderr, flush=True)
    stamp_file.write_text(stamp)
    return obj


def build(force: bool = False, verbose: bool = False) -> Path:
    BUILD.mkdir(parents=True, exist_ok=True)
    with ThreadPoolExecutor(max_workers=min(len(SOURCES), os.cpu_count() or 4)) as ex:
        objs = list(ex.map(lambda s: _compile(s, force, verbose), SOURCES))
    newest = max(o.stat().st_mtime_ns for o in objs)
    if force or not LIB.exists() or LIB.stat().st_mtime_ns < newest:
        cmd = [_nvcc(), "-shared", "-cudart", "shared", *GENCODE,
               "-Xlinker", "-rpath", "-Xlinker", "/usr/local/cuda/lib64",
               "-o", str(LIB), *map(str, objs)]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
    return LIB


if __name__ == "__main__":
    lib = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(lib)
