"""Builds libcrabml_cuda.so (sm_90a only) in-tree with nvcc.  Used by __graft_entry__.build()."""
from __future__ import annotations

import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "lib", "libcrabml_cuda.so")

NVCC_FLAGS = [
    "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
    # parity: no FMA contraction, IEEE div/sqrt, no flush-to-zero (the reference is plain f32 Rust)
    "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false",
    "-cudart", "static",
]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "host", "*.cpp")))


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "host", "*.hpp")) + \
        [os.path.join(os.path.dirname(HERE), "include", "crabml_cuda.h"), os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    objs = []
    procs = []
    objdir = os.path.join(HERE, "lib", "obj")
    os.makedirs(objdir, exist_ok=True)
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src) + ".o")
        objs.append(obj)
        cmd = [nvcc, *NVCC_FLAGS, "-x", "cu", "-c", src, "-o", obj] + (["-Xptxas", "-v"] if verbose else [])
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(f"--- {os.path.basename(src)} ---\n{out}\n")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    subprocess.check_call([nvcc, "-shared", "-cudart", "static", "-o", LIB, *objs, "-Xlinker", "--exclude-libs,ALL"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
