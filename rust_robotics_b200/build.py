"""Builds rust_robotics_b200/libpfgpu.so (sm_90a, H100) with nvcc, and the GPU probe of the fast form's reciprocal and
square root (build/libfsm_probe.so, tests/test_gpu_fast_rcp_sqrt.py) with the same flags.  Used by __graft_entry__.build()."""
import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(PKG, "csrc", "pfgpu.cu")
LIB = os.path.join(PKG, "libpfgpu.so")
ROOT = os.path.dirname(PKG)
PROBE_SRC = os.path.join(ROOT, "tests", "host", "fsm_probe.cu")
PROBE_LIB = os.path.join(ROOT, "build", "libfsm_probe.so")

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


def build_probe(force=False):
    """tests/host/fsm_probe.cu -> build/libfsm_probe.so: a shared object of its own, so libpfgpu.so gains no test entry"""
    inc = os.path.join(ROOT, "include")
    deps = [PROBE_SRC, os.path.abspath(__file__)] + [os.path.join(inc, f) for f in os.listdir(inc)]
    if not force and os.path.exists(PROBE_LIB) and all(os.path.getmtime(s) <= os.path.getmtime(PROBE_LIB) for s in deps):
        return PROBE_LIB
    os.makedirs(os.path.dirname(PROBE_LIB), exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    env = dict(os.environ)
    env.pop("CC", None)
    env.pop("CXX", None)
    r = subprocess.run([nvcc] + NVCC_FLAGS + ["-o", PROBE_LIB, PROBE_SRC], capture_output=True, text=True, env=env)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed building libfsm_probe.so")
    return PROBE_LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
    print(build_probe(force="--force" in sys.argv))
