"""Builds the C-ABI shared library in-tree: pydcop_b200/lib/libpydcop_b200.so (sm_90a, H100, only).

nvcc cross-compiles without a GPU, so the library can be built on a machine without one; it is a
build product and stays out of git.
"""
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIB_DIR = os.path.join(PKG, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libpydcop_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-fmad=false",           # keep the reference's operand order: no FMA contraction (bit parity)
    "--extended-lambda", "-shared", "-Xcompiler", "-fPIC", "-diag-suppress", "177",
]


def sources():
    out = []
    for root, _, files in os.walk(CSRC):
        out += [os.path.join(root, f) for f in files if f.endswith((".cu", ".cuh", ".h"))]
    out.append(os.path.join(os.path.dirname(PKG), "include", "pydcop_b200.h"))
    return out


def needs_build():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    return any(os.path.getmtime(s) > t for s in sources())


def nvcc_path():
    p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return p if os.path.exists(p) else None


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB_PATH
    nvcc = nvcc_path()
    if nvcc is None:
        raise RuntimeError("nvcc not found: cannot build libpydcop_b200.so")
    os.makedirs(LIB_DIR, exist_ok=True)
    # one translation unit per family: engine.cu (MaxSum, DSA, halo, cost), mgm.cu (MGM), mgm2.cu (MGM-2),
    # gdba.cu (GDBA), dpop.cu (DPOP), dba.cu (DBA), syncbb.cu (SyncBB), mixeddsa.cu (MixedDSA)
    units = [os.path.join(CSRC, f) for f in ("engine.cu", "mgm.cu", "mgm2.cu", "gdba.cu", "dpop.cu", "dba.cu",
                                              "syncbb.cu", "mixeddsa.cu")]
    cmd = [nvcc, *NVCC_FLAGS, "-o", LIB_PATH, *units, "-ldl"]
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stderr)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
