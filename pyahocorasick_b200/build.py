"""Build the native library in-tree: pyahocorasick_b200/_native/libacb200.so (sm_90a only).

    python -m pyahocorasick_b200.build [--force] [--verbose]

nvcc cross-compiles without a GPU, so the library can be built on a machine that has none.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
OUT_DIR = os.path.join(PKG, "_native")
LIB = os.path.join(OUT_DIR, "libacb200.so")
SOURCES = ["acb_host.cpp", "acb_device.cu"]
HEADERS = ["acb_hash.h", "acb_internal.h", os.path.join("..", "..", "include", "acb200.h")]

NVCC_FLAGS = [
    "-O3", "-std=c++17",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "-Xcompiler", "-fPIC,-O3,-Wall",
    "-shared",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (needed to build libacb200.so for sm_90a)")


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False, defines=(), out: str = LIB) -> str:
    """defines/out: experimental variants (e.g. defines=["ACB_EXP_X"], out=".../libacb200_x.so"), selected at
    run time with the environment variable ACB_LIB."""
    if not force and not defines and not needs_build():
        return LIB
    os.makedirs(OUT_DIR, exist_ok=True)
    cmd = [_nvcc()] + NVCC_FLAGS + [f"-D{d}" for d in defines] + (["-Xptxas", "-v"] if verbose else []) + ["-o", out] + SOURCES
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed building libacb200.so")
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
