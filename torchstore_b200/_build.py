"""In-tree build of libtstore_b200.so (nvcc, sm_90a: H100).  No torch extension machinery: the
library is a plain C-ABI shared object loaded with ctypes (see ``_native.py``)."""

from __future__ import annotations

import os
import shutil
import subprocess

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
REPO_ROOT = os.path.dirname(PKG_DIR)
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_DIR = os.path.join(PKG_DIR, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libtstore_b200.so")
SOURCES = ["copy_rects.cu", "plan.cu", "runtime.cu", "host_tier.cu"]
HEADERS = [os.path.join(CSRC, "tsb_internal.h"), os.path.join(REPO_ROOT, "include", "tstore_b200.h")]

NVCC_FLAGS = [
    "-gencode",
    "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "-O3",
    "-std=c++17",
    "--shared",
    "-Xcompiler",
    "-fPIC",
    "-cudart",
    "static",
]


def find_nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: cannot build libtstore_b200.so")


def needs_build() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    lib_mtime = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, s) for s in SOURCES] + HEADERS
    return any(os.path.getmtime(d) > lib_mtime for d in deps)


def build_native(force: bool = False, verbose: bool = False) -> str:
    """Compile csrc/*.cu into torchstore_b200/lib/libtstore_b200.so; returns its path."""
    if not force and not needs_build():
        return LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    tmp = LIB_PATH + ".tmp"
    cmd = [find_nvcc(), *NVCC_FLAGS, "-I", os.path.join(REPO_ROOT, "include"), "-I", CSRC, "-o", tmp]
    if verbose:
        cmd += ["-Xptxas", "-v"]
    cmd += [os.path.join(CSRC, s) for s in SOURCES]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError(f"nvcc failed ({proc.returncode}):\n{proc.stdout}\n{proc.stderr}")
    os.replace(tmp, LIB_PATH)
    if verbose:
        print(proc.stderr)
    return LIB_PATH


if __name__ == "__main__":
    print(build_native(force=True, verbose=True))
