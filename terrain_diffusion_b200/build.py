"""Build libtdx.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

Usage:  python -m terrain_diffusion_b200.build [--force] [--verbose]
The .so is written next to this file so it travels with the source tree (it is git-ignored).
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB = PKG / "libtdx.so"
STAMP = PKG / ".libtdx.stamp"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
    "--expt-relaxed-constexpr",
    "-cudart", "static",
]


if os.environ.get("TDX_DEBUG_HOOKS") == "1":      # trace clocks / launch timeline for tools/trace_igemm.py etc.
    NVCC_FLAGS.append("-DTDX_DEBUG_HOOKS=1")


def _sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


def _digest() -> str:
    h = hashlib.sha256()
    for p in sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h"))
                    + [PKG.parent / "include" / "tdx.h"]):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    digest = _digest()
    if not force and LIB.exists() and STAMP.exists() and STAMP.read_text().strip() == digest:
        return LIB
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc, *NVCC_FLAGS, "-o", str(LIB), *map(str, _sources()), "-ldl"]
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
        print(" ".join(cmd), flush=True)
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("nvcc failed building libtdx.so")
    if verbose:
        sys.stderr.write(res.stdout + res.stderr)
    STAMP.write_text(digest)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(LIB)
