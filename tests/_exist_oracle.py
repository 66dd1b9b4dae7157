"""ctypes access to the existence-counter oracle (tests/host/fs2_exist_oracle.c, which includes fs2_assoc_oracle.c).
Test infrastructure only."""
import ctypes as C
import os
import subprocess

import numpy as np

import _assoc_oracle
import _oracle

SRC = os.path.join(_assoc_oracle.ROOT, "tests", "host", "fs2_exist_oracle.c")
_LIBS = {}


def load(libm=False):
    if libm in _LIBS:
        return _LIBS[libm]
    _assoc_oracle.load(libm)                # builds liboracle*.so first if needed
    dep = os.path.join(_oracle.ORACLE_DIR, "liboracle_libm.so" if libm else "liboracle.so")
    out = os.path.join(_assoc_oracle.ROOT, "tests", "host", "libfs2_exist_oracle_libm.so" if libm else "libfs2_exist_oracle.so")
    hdrs = [SRC, _assoc_oracle.SRC, os.path.join(_assoc_oracle.ROOT, "oracle", "fs_state.h"), dep]
    if not os.path.exists(out) or any(os.path.getmtime(h) > os.path.getmtime(out) for h in hdrs):
        subprocess.run(["/usr/bin/gcc"] + _assoc_oracle.CFLAGS + (["-DPF_ORACLE_LIBM"] if libm else []) + ["-shared", "-o", out, SRC, dep, "-lm"],
                       check=True)
    L = C.CDLL(out)
    dp, u64p, vp = C.POINTER(C.c_double), C.POINTER(C.c_uint64), C.c_void_p
    L.orc_fs2_step_unknown.argtypes = [vp, dp, dp, C.c_size_t, C.c_double, u64p]
    L.orc_fs2_step_unknown_with_noise.argtypes = [vp, dp, dp, C.c_size_t, C.c_double, dp, dp, C.c_double, u64p]
    L.orc_fs2_ex_new.argtypes, L.orc_fs2_ex_new.restype = [vp, C.c_double], vp
    L.orc_fs2_ex_free.argtypes, L.orc_fs2_ex_free.restype = [vp], None
    L.orc_fs2_ex_reset.argtypes, L.orc_fs2_ex_reset.restype = [vp], None
    L.orc_fs2_step_unknown_ex.argtypes = [vp, vp, dp, dp, C.c_size_t, C.c_double, dp, dp, C.c_double, u64p, u64p]
    L.orc_fs2_ex_counts.argtypes, L.orc_fs2_ex_counts.restype = [vp, vp, C.POINTER(C.c_int32)], None
    _LIBS[libm] = L
    return L


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


class OracleFS2Exist(_assoc_oracle.OracleFS2Assoc):
    """OracleFS2Assoc plus existence counters (enable_existence); with them off it is OracleFS2Assoc"""

    def __init__(self, n, m, seed=42, libm=False, **cfg):
        super().__init__(n, m, seed=seed, libm=libm, **cfg)
        self.A = load(libm)
        self.ex, self.removed = None, 0

    def __del__(self):
        if getattr(self, "ex", None):
            self.A.orc_fs2_ex_free(self.ex)
            self.ex = None
        super().__del__()

    def enable_existence(self, r):
        """r > 0 (inf allowed): every tau = 1; 0: off"""
        if self.ex:
            self.A.orc_fs2_ex_free(self.ex)
        self.ex, self.removed = (self.A.orc_fs2_ex_new(self.h, float(r)) if r else None), 0

    def set_state(self, pose_w, lm=None):
        super().set_state(pose_w, lm)
        if getattr(self, "ex", None):
            self.A.orc_fs2_ex_reset(self.ex)

    def seed_map(self, *a, **kw):
        super().seed_map(*a, **kw)
        if self.ex:
            self.A.orc_fs2_ex_reset(self.ex)

    def existence_counts(self):
        """(n, m) int32: tau of every slot, 0 for an empty one"""
        out = np.zeros((self.n, self.m), dtype=np.int32)
        self.A.orc_fs2_ex_counts(self.h, self.ex, out.ctypes.data_as(C.POINTER(C.c_int32)))
        return out

    def step_unknown(self, u, z, gate_d2=16.0, z0=None, z1=None, u01=None):
        """as OracleFS2Assoc.step_unknown; with counters also self.removed = copies removed"""
        if not self.ex:
            return super().step_unknown(u, z, gate_d2, z0, z1, u01)
        uu, zz = _oracle.f64(u), _oracle.f64(z).reshape(-1, 2)
        k = zz.shape[0]
        if k == 0:
            zz = np.zeros((1, 2))
        cnt, rem = np.zeros(3, dtype=np.uint64), C.c_uint64()
        a, b = (_oracle.f64(z0), _oracle.f64(z1)) if z0 is not None else (None, None)
        did = self.A.orc_fs2_step_unknown_ex(self.h, self.ex, _dp(uu), _dp(zz), k, float(gate_d2), _dp(a) if a is not None else None,
                                             _dp(b) if b is not None else None, float(u01 or 0.0), cnt.ctypes.data_as(C.POINTER(C.c_uint64)),
                                             C.byref(rem))
        self.counts, self.removed = cnt, int(rem.value)
        return bool(did)
