#!/usr/bin/env python3
"""sass_compare.py — checks that a change leaves the machine code of existing kernels alone: the SASS of every kernel in a baseline
libpfgpu.so is compared with the same kernel in a new one, once addresses, encodings and symbol names are normalised.

    python sass_compare.py --rev HEAD~1 [NEW_LIB]       # builds the library of a git revision in a temporary directory first
    python sass_compare.py BASE_LIB [NEW_LIB]

NEW_LIB defaults to rust_robotics_b200/libpfgpu.so (build it first).  Prints the kernel counts, the kernels that are missing or
changed, and the kernels that are new; exits 1 when a baseline kernel is missing or changed.  Needs nvcc and cuobjdump, no GPU.
Writes nothing into the tree.
"""
import argparse
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.abspath(__file__))
CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")


def kernels(lib):
    """{mangled name: normalised SASS lines}"""
    out = subprocess.run([CUOBJDUMP, "-sass", lib], capture_output=True, text=True, check=True).stdout
    fs, name, cur = {}, None, []
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                fs[name] = cur
            name, cur = m.group(1), []
            continue
        if name:
            line = re.sub(r"/\*[0-9a-f]{4,}\*/", "", line)      # instruction addresses and encodings
            cur.append(re.sub(r"_Z\w+", "SYM", line).strip())    # call targets and constant-bank symbols
    if name:
        fs[name] = cur
    return fs


def build_rev(rev, tmp):
    """the library of git revision `rev`, built from a clean export in tmp"""
    src = os.path.join(tmp, "src")
    os.makedirs(src)
    archive = subprocess.run(["git", "-C", ROOT, "archive", rev], capture_output=True, check=True).stdout
    subprocess.run(["tar", "-x", "-C", src], input=archive, check=True)
    subprocess.run([sys.executable, os.path.join(src, "rust_robotics_b200", "build.py")], check=True, stdout=subprocess.DEVNULL)
    return os.path.join(src, "rust_robotics_b200", "libpfgpu.so")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("base", nargs="?", help="baseline libpfgpu.so")
    ap.add_argument("new", nargs="?", default=os.path.join(ROOT, "rust_robotics_b200", "libpfgpu.so"))
    ap.add_argument("--rev", help="build the baseline from this git revision")
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        base = build_rev(a.rev, tmp) if a.rev else a.base
        if not base:
            ap.error("give a baseline library or --rev")
        old, new = kernels(base), kernels(a.new)
    missing = sorted(k for k in old if k not in new)
    changed = sorted(k for k in old if k in new and old[k] != new[k])
    print(f"{len(old)} baseline kernels, {len(new)} new-build kernels; missing {len(missing)}, changed {len(changed)}")
    for k in missing:
        print("missing:", k)
    for k in changed:
        print("changed:", k)
    for k in sorted(k for k in new if k not in old):
        print("new:", k)
    return 1 if missing or changed else 0


if __name__ == "__main__":
    sys.exit(main())
