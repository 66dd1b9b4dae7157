"""ctypes access to the augmented-MCL oracle (tests/host/pf_recovery_oracle.c, which includes oracle/pf_oracle.c unchanged).
Test infrastructure only."""
import ctypes as C
import os
import subprocess

import numpy as np

import _assoc_oracle
import _oracle
from _oracle import f64

SRC = os.path.join(_oracle.ROOT, "tests", "host", "pf_recovery_oracle.c")
_LIBS = {}


def load(libm=False):
    """the oracle library (contract math, or glibc libm with libm=True), built here on first use"""
    if libm not in _LIBS:
        out = os.path.join(_oracle.ROOT, "tests", "host", "libpf_recovery_oracle%s.so" % ("_libm" if libm else ""))
        deps = [SRC] + [os.path.join(_oracle.ROOT, d) for d in ("oracle/pf_oracle.c", "oracle/oracle.h", "include/pf_contract_math.h")]
        if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
            subprocess.run(["/usr/bin/gcc"] + _assoc_oracle.CFLAGS + (["-DPF_ORACLE_LIBM"] if libm else []) + ["-shared", "-o", out, SRC, "-lm"],
                           check=True)
        L = C.CDLL(out)
        vp, dp = C.c_void_p, _oracle.c_dp
        L.orc_rec_new.argtypes, L.orc_rec_new.restype = [C.POINTER(_oracle.PfConfig), C.c_uint64], vp
        L.orc_rec_free.restype = L.orc_rec_state.restype = L.orc_rec_upload.restype = None
        L.orc_rec_pf.argtypes, L.orc_rec_pf.restype = [vp], vp
        L.orc_pf_count.restype = L.orc_pf_last_indices.restype = C.c_size_t
        for name, args in (("orc_rec_free", [vp]), ("orc_rec_enable", [vp, C.c_double, C.c_double, dp]),
                           ("orc_rec_state", [vp, dp, C.POINTER(C.c_uint64)]), ("orc_rec_init_region_with_uniforms", [vp, dp, dp]),
                           ("orc_rec_init_state", [vp, dp]), ("orc_rec_upload", [vp, dp, C.c_size_t]),
                           ("orc_rec_predict_with_draws", [vp, dp, dp, dp, dp]), ("orc_rec_update", [vp, dp, C.c_size_t]),
                           ("orc_rec_resample_with_uniforms", [vp, dp, C.c_size_t]),
                           ("orc_pf_count", [vp]), ("orc_pf_get_particles", [vp, dp]), ("orc_pf_estimate", [vp, dp, dp]),
                           ("orc_pf_last_indices", [vp, _oracle.c_u32p, C.c_size_t]), ("orc_pf_set_fast_search", [vp, C.c_int]),
                           ("orc_pf_set_threads", [vp, C.c_int])):
            getattr(L, name).argtypes = args
        _LIBS[libm] = L
    return _LIBS[libm]


def _dp(a):
    return None if a is None else f64(a).ctypes.data_as(_oracle.c_dp)


class OracleRecovery:
    """PF (mode 0) or MCL (mode 1) oracle with augmented MCL; the keyword arguments are _oracle.OraclePF's.  Array arguments are
    held in locals while the call runs (_dp converts them)."""

    def __init__(self, n, threshold=0.5, range_noise=0.2, velocity_noise=2.0, yaw_rate_noise=np.deg2rad(40.0), dt=0.1, seed=42, mode=0,
                 max_particles=None, kld_epsilon=0.05, kld_z=2.326, libm=False, fast_search=True, threads=1):
        self.L = load(libm)
        self.cfg = _oracle.PfConfig(n, threshold, range_noise, velocity_noise, yaw_rate_noise, dt, mode, 0,
                                    max_particles if max_particles is not None else n, kld_epsilon, kld_z)
        self.r = self.L.orc_rec_new(C.byref(self.cfg), seed)
        if not self.r:
            raise ValueError("InvalidParameter")
        self.h = self.L.orc_rec_pf(self.r)
        self.cap = int(self.cfg.max_particles)
        self.L.orc_pf_set_fast_search(self.h, int(fast_search))
        self.L.orc_pf_set_threads(self.h, int(threads))

    def __del__(self):
        if getattr(self, "r", None):
            self.L.orc_rec_free(self.r)
            self.r = None

    def enable(self, a_slow, a_fast, region):
        reg = None if region is None else f64(region)
        return self.L.orc_rec_enable(self.r, float(a_slow), float(a_fast), _dp(reg))

    def state(self):
        """((w_slow, w_fast, p), injected by the last predict)"""
        out, inj = np.empty(3), C.c_uint64()
        self.L.orc_rec_state(self.r, _dp(out), C.byref(inj))
        return out, int(inj.value)

    def init_region(self, region, u3=None):
        reg, u = f64(region), None if u3 is None else f64(u3)
        return self.L.orc_rec_init_region_with_uniforms(self.r, _dp(reg), _dp(u))

    def init_state(self, s):
        s = f64(s)
        return self.L.orc_rec_init_state(self.r, _dp(s))

    def upload(self, aos5):
        a = f64(aos5)
        self.L.orc_rec_upload(self.r, _dp(a), a.shape[0])

    def predict(self, u, zv=None, zw=None, inj4=None):
        u, zv, zw, i4 = (None if a is None else f64(a) for a in (u, zv, zw, inj4))
        return self.L.orc_rec_predict_with_draws(self.r, _dp(u), _dp(zv), _dp(zw), _dp(i4))

    def update(self, obs):
        o = f64(obs).reshape(-1, 3)
        return self.L.orc_rec_update(self.r, _dp(o), o.shape[0])

    def resample(self, rs=None):
        r = None if rs is None else f64(rs)
        return bool(self.L.orc_rec_resample_with_uniforms(self.r, _dp(r), 0 if r is None else r.size))

    def step(self, u, obs):
        """try_step: predict, update, resample -> (estimate, resampled)"""
        assert self.predict(u) == 0 and self.update(obs) == 0
        did = self.resample()
        return self.estimate(), did

    def count(self):
        return int(self.L.orc_pf_count(self.h))

    def particles(self):
        a = np.empty((self.count(), 5))
        self.L.orc_pf_get_particles(self.h, _dp(a))
        return a

    def estimate(self):
        est = np.empty(4)
        self.L.orc_pf_estimate(self.h, _dp(est), None)
        return est

    def last_indices(self):
        idx = np.empty(self.cap, dtype=np.uint32)
        return idx[:self.L.orc_pf_last_indices(self.h, idx.ctypes.data_as(_oracle.c_u32p), idx.size)].copy()
