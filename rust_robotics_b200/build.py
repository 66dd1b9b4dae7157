"""Builds rust_robotics_b200/libpfgpu.so (sm_90a, H100) with nvcc.  Used by __graft_entry__.build()."""
import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(PKG, "csrc", "pfgpu.cu")
LIB = os.path.join(PKG, "libpfgpu.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "--fmad=false",                               # the numerical contract: no implicit a*b+c fusion (pf_contract_math.h)
    "-Xcompiler", "-fPIC,-ffp-contract=off",
    "-shared",
]


def sources():
    """everything the library depends on, this file included (a change of the flags above rebuilds it)"""
    d = os.path.join(PKG, "csrc")
    inc = os.path.join(os.path.dirname(PKG), "include")
    return [os.path.join(d, f) for f in os.listdir(d)] + [os.path.join(inc, f) for f in os.listdir(inc)] + [os.path.abspath(__file__)]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(s) > t for s in sources())


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB, SRC, "-lnccl"]
    env = dict(os.environ)
    env.pop("CC", None)
    env.pop("CXX", None)
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed building libpfgpu.so")
    if verbose:
        print(r.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
