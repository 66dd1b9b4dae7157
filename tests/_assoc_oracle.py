"""ctypes access to the unknown-association oracle (tests/host/fs2_assoc_oracle.c), built on top of oracle/liboracle*.so.
Test infrastructure only."""
import ctypes as C
import os
import subprocess

import numpy as np

import _oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "fs2_assoc_oracle.c")
CFLAGS = ["-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-fopenmp", "-Wall", "-Wextra",
          "-Wno-unused-function"]
_LIBS = {}


def load(libm=False):
    """the oracle library (contract math, or glibc libm with libm=True); liboracle*.so is built first if needed"""
    if libm in _LIBS:
        return _LIBS[libm]
    base = _oracle.load(libm=libm)          # builds oracle/ and keeps liboracle*.so loaded
    dep = os.path.join(_oracle.ORACLE_DIR, "liboracle_libm.so" if libm else "liboracle.so")
    out = os.path.join(ROOT, "tests", "host", "libfs2_assoc_oracle_libm.so" if libm else "libfs2_assoc_oracle.so")
    hdrs = [SRC, os.path.join(ROOT, "oracle", "fs_state.h"), os.path.join(ROOT, "include", "pf_contract_math.h"), dep]
    if not os.path.exists(out) or any(os.path.getmtime(h) > os.path.getmtime(out) for h in hdrs):
        subprocess.run(["/usr/bin/gcc"] + CFLAGS + (["-DPF_ORACLE_LIBM"] if libm else []) + ["-shared", "-o", out, SRC, dep, "-lm"],
                       check=True)
    L = C.CDLL(out)
    dp, u64p = C.POINTER(C.c_double), C.POINTER(C.c_uint64)
    L.orc_fs2_step_unknown.argtypes = [C.c_void_p, dp, dp, C.c_size_t, C.c_double, u64p]
    L.orc_fs2_step_unknown_with_noise.argtypes = [C.c_void_p, dp, dp, C.c_size_t, C.c_double, dp, dp, C.c_double, u64p]
    L.orc_fs2_assoc_d2.argtypes = [C.POINTER(_oracle.FsConfig), dp, dp, C.c_double, C.c_double, dp]
    _LIBS[libm] = (base, L)
    return base, L


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


class OracleFS2Assoc(_oracle.OracleFS):
    """OracleFS (variant 2) plus the unknown-association step; known-id steps (step()) may be interleaved"""

    def __init__(self, n, m, seed=42, libm=False, **cfg):
        base, self.A = load(libm)
        super().__init__(base, n, m, seed=seed, variant=2, **cfg)
        self.counts = np.zeros(3, dtype=np.uint64)

    def step_unknown(self, u, z, gate_d2=16.0, z0=None, z1=None, u01=None):
        """z: k (d, angle) pairs.  Returns whether it resampled; self.counts = (matched, born, dropped)."""
        uu = _oracle.f64(u)
        zz = _oracle.f64(z).reshape(-1, 2)
        if zz.size == 0:
            zz = np.zeros((1, 2))
            k = 0
        else:
            k = zz.shape[0]
        cnt = np.zeros(3, dtype=np.uint64)
        cp = cnt.ctypes.data_as(C.POINTER(C.c_uint64))
        if z0 is None:
            did = self.A.orc_fs2_step_unknown(self.h, _dp(uu), _dp(zz), k, float(gate_d2), cp)
        else:
            a, b = _oracle.f64(z0), _oracle.f64(z1)
            did = self.A.orc_fs2_step_unknown_with_noise(self.h, _dp(uu), _dp(zz), k, float(gate_d2), _dp(a), _dp(b), float(u01), cp)
        self.counts = cnt
        return bool(did)

    def assoc_d2(self, lm6, pose3, z):
        """the metric of one (landmark, pose, observation): None when det S == 0"""
        l, p = _oracle.f64(lm6), _oracle.f64(pose3)
        out = np.zeros(1)
        ok = self.A.orc_fs2_assoc_d2(C.byref(self.cfg), _dp(l), _dp(p), float(z[0]), float(z[1]), _dp(out))
        return float(out[0]) if ok else None
