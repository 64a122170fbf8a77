"""In-tree build of the native pieces for sm_90a (H100); no JIT cache, the .so files sit next to the sources.  `python -m ai00_server_b200.build` or `__graft_entry__.build()`."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200rwkv.so")
SYNTH = os.path.join(HERE, "_synthfill.so")
ORACLE_C = os.path.join(ROOT, "oracle", "liboracle_ref.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-shared",
]


def _newer(target: str, sources: list[str]) -> bool:
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in sources)


def _run(cmd: list[str]) -> None:
    print("+", " ".join(cmd), flush=True)
    subprocess.check_call(cmd)


def build_engine(force: bool = False, verbose_ptxas: bool = False) -> str:
    srcs = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh"))]
    srcs.append(os.path.join(ROOT, "include", "b200rwkv.h"))
    if force or not _newer(LIB, srcs):
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose_ptxas else []) + [os.path.join(CSRC, "engine.cu"), "-o", LIB]
        _run(cmd)
    return LIB


def build_synth(force: bool = False) -> str:
    src = os.path.join(CSRC, "synth_fill.c")
    if force or not _newer(SYNTH, [src]):
        _run(["gcc", "-O3", "-fopenmp", "-mf16c", "-mavx2", "-ffp-contract=off", "-shared", "-fPIC", src, "-o", SYNTH])
    return SYNTH


def build_oracle(force: bool = False) -> str | None:
    src = os.path.join(ROOT, "oracle", "rwkv_ref.c")
    if not os.path.exists(src):
        return None
    if force or not _newer(ORACLE_C, [src]):
        _run(["gcc", "-O3", "-fopenmp", "-mf16c", "-mavx2", "-mfma", "-shared", "-fPIC", src, "-o", ORACLE_C, "-lm"])
    return ORACLE_C


def build_all(force: bool = False) -> None:
    build_synth(force)
    build_oracle(force)
    build_engine(force)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv)
