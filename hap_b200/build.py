"""Builds libhap_b200.so (sm_90a, H100) in-tree with nvcc.  `python -m hap_b200.build`"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libhap_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-fmad=false",             # FMAs are written explicitly (bc_block.cuh) so the CPU twin matches bit for bit
    "-Xcompiler", "-fPIC",
    "-shared", "--cudart", "shared",
]


def nvcc() -> str:
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def sources():
    return [os.path.abspath(__file__)] + [os.path.join(SRC, f) for f in sorted(os.listdir(SRC))] + [os.path.join(ROOT, "include", f) for f in ("hap.h", "hap_b200.h")]


def up_to_date() -> bool:
    if not os.path.exists(OUT):
        return False
    t = os.path.getmtime(OUT)
    return all(os.path.getmtime(s) <= t for s in sources())


def build(force: bool = False, verbose: bool = False, extra_flags=(), out: str = OUT) -> str:
    """extra_flags / out: variant builds for A/B measurements (loaded through HAPB200_LIBRARY); the product is OUT."""
    if not force and out == OUT and up_to_date():
        return OUT
    cmd = [nvcc()] + NVCC_FLAGS + list(extra_flags) + (["-Xptxas", "-v"] if verbose else []) + ["-o", out, os.path.join(SRC, "hap_api.cu")]
    p = subprocess.run(cmd, capture_output=True, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stdout + p.stderr)
        raise RuntimeError("nvcc failed")
    if verbose:
        print(p.stderr)
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
